from .bert import BertConfig
from .bert_layers import (ACT2FN, BertEmbeddings, BertLayer_Body, BertLayer_Head, BertLayer_Tail,
                          BertLayerNorm, BertPooler, BertSpan, BertTailForClassification,
                          BertTailForMaskedLM, LinearActivation, advance_rng, default_rng, get_backend, set_backend)
from .layers import (BasicBlock, BottleNeck, ResHead, ResLayer, ResNet, ResTail, resnet18,
                     resnet34, resnet50, resnet101, resnet152, resnet_layer_configs)

__all__ = [
    "BertConfig", "BertEmbeddings", "BertLayer_Head", "BertLayer_Body", "BertLayer_Tail",
    "BertPooler", "BertTailForClassification", "BertTailForMaskedLM", "BertLayerNorm", "LinearActivation", "BertSpan",
    "ACT2FN", "set_backend", "get_backend", "advance_rng", "default_rng", "BasicBlock", "BottleNeck", "ResHead",
    "ResLayer", "ResTail", "ResNet", "resnet18", "resnet34", "resnet50", "resnet101", "resnet152",
    "resnet_layer_configs",
]
