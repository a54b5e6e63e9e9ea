from .hooks import Hook
from .hooks_collection import (CheckpointHook, DistributedTimerHelperHook, EvalHook,
                               ReallocateHook, StopHook)
from .metrics import TorchEvalAccumulator, TorchTokenAccumulator, classification_metrics, token_metrics
from .runner import MaskedLMLoss, PreTrainingLoss, Runner, build_loss

__all__ = ["Hook", "CheckpointHook", "DistributedTimerHelperHook", "EvalHook", "StopHook",
           "ReallocateHook", "Runner", "build_loss", "TorchEvalAccumulator",
           "classification_metrics", "MaskedLMLoss", "PreTrainingLoss", "TorchTokenAccumulator", "token_metrics"]
