from .hooks import Hook
from .hooks_collection import (CheckpointHook, DistributedTimerHelperHook, EvalHook,
                               ReallocateHook, StopHook)
from .metrics import (TorchEvalAccumulator, TorchSpanAccumulator, TorchTokenAccumulator,
                      classification_metrics, span_metrics, token_metrics)
from .runner import MaskedLMLoss, PreTrainingLoss, QuestionAnsweringLoss, Runner, build_loss

__all__ = ["Hook", "CheckpointHook", "DistributedTimerHelperHook", "EvalHook", "StopHook",
           "ReallocateHook", "Runner", "build_loss", "TorchEvalAccumulator",
           "classification_metrics", "MaskedLMLoss", "PreTrainingLoss", "TorchTokenAccumulator", "token_metrics",
           "QuestionAnsweringLoss", "TorchSpanAccumulator", "span_metrics"]
