from .bert_dataset import GlueDataset, MaskedLMDataset
from .data_generator import BaseGenerator, DataloaderGenerator, RandomTensorGenerator
from .dataset import (CIFAR10Dataset, RandomImageDataset, RandomMlpDataset, SynthMLMDataset,
                      SynthMNLIDataset)

__all__ = ["GlueDataset", "BaseGenerator", "DataloaderGenerator", "RandomTensorGenerator",
           "CIFAR10Dataset", "RandomImageDataset", "RandomMlpDataset", "SynthMNLIDataset", "SynthMLMDataset", "MaskedLMDataset"]
