from .checkpoint_hook import CheckpointHook
from .distributed_timer_helper_hook import DistributedTimerHelperHook
from .eval_hook import EvalHook
from .reallocate_hook import ReallocateHook
from .stop_hook import StopHook

__all__ = ["CheckpointHook", "DistributedTimerHelperHook", "EvalHook", "StopHook", "ReallocateHook"]
