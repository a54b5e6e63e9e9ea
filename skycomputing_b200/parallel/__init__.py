from .comm import TorchDistComm
from .optim import FusedAdam, FusedLamb, FusedSGD, Lamb, TorchOptimizerAdapter, build_optimizer
from .pipeline import PipelineEngine, one_f_one_b_order, sequential_order
from .pipeline_model import BaseModule, LocalModule, RemoteModule, RpcModel

__all__ = ["TorchDistComm", "FusedSGD", "FusedAdam", "FusedLamb", "Lamb", "TorchOptimizerAdapter",
           "build_optimizer",            "PipelineEngine", "one_f_one_b_order", "sequential_order", "BaseModule", "LocalModule",
           "RemoteModule", "RpcModel"]
