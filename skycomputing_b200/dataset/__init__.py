from .bert_dataset import GlueDataset, MaskedLMDataset, PreTrainingDataset
from .data_generator import BaseGenerator, DataloaderGenerator, RandomTensorGenerator
from .dataset import (CIFAR10Dataset, RandomImageDataset, RandomMlpDataset, SynthMLMDataset,
                      SynthMNLIDataset, SynthPretrainingDataset, SynthQADataset)
from .squad_dataset import SquadDataset

__all__ = ["GlueDataset", "BaseGenerator", "DataloaderGenerator", "RandomTensorGenerator",
           "CIFAR10Dataset", "RandomImageDataset", "RandomMlpDataset", "SynthMNLIDataset", "SynthMLMDataset", "MaskedLMDataset",
           "SynthPretrainingDataset", "PreTrainingDataset", "SynthQADataset", "SquadDataset"]
