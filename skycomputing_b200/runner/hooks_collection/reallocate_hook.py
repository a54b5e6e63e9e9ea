"""Periodic re-benchmark + re-allocation while training ("dynamic" in the literal sense).

The reference benchmarks and allocates once, before training (experiment/launch.py:79-138); its
WorkerManager carries unused elastic scaffolding (SURVEY §5.3).  This hook closes that loop: every
``interval`` iterations all ranks

1. re-run the device benchmark (so a GPU that started to throttle, or a changed ``slowdown``, is
   seen), all-gathered like the initial one;
2. re-run the allocator on a COPY of the worker pool;
3. if the predicted bottleneck (max over stages of device_time x sum of layer costs) improves by more
   than ``min_gain``, migrate: every rank publishes the state_dicts of its layers keyed by GLOBAL
   layer index (the checkpoint format, so the move is partition independent), the model is rebuilt
   under the new partition, every rank loads its new span, optimizer and engine are rebuilt
   (``Runner.rebuild``).

Everything is collective and deterministic (all ranks compute the same allocation from the same
gathered numbers).  Plain-SGD state is nothing; momentum buffers are reset by a migration.  The
rebuilt optimizer gets the same learning-rate schedule / gradient clipping and continues the
schedule at the step count of the old one (no second warmup).
"""
import copy
from typing import Callable, Optional

from ...registry import HOOKS
from ..hooks import Hook


def _dist():
    import torch.distributed as dist

    return dist if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 else None


def _layout(worker_manager) -> list:
    """[(physical device, layer range)] in pipeline order."""
    return [(w.device, tuple(map(tuple, w.chunks)) if getattr(w, "chunks", None)
             else (tuple(w.layer_range) if w.layer_range is not None else None))
            for w in worker_manager.worker_pool]


def _bottleneck(worker_manager, device_times: dict, layer_cost: list) -> float:
    """max over workers of (device time) x (summed cost of the layers it runs)."""
    worst, pos = 0.0, 0
    for i, w in enumerate(worker_manager.worker_pool):
        if getattr(w, "chunks", None):
            spans = list(w.chunks)
        elif w.layer_range is not None:
            spans = [tuple(w.layer_range)]
        else:
            spans = [(pos, pos + len(w.model_config))]
        pos += len(w.model_config)
        t = device_times[w.device if w.device is not None else i]
        worst = max(worst, t * sum(sum(layer_cost[b:e]) for b, e in spans))
    return worst


@HOOKS.register_module
class ReallocateHook(Hook):
    def __init__(self, interval: int, allocator_factory: Callable, optimizer_cfg: dict,
                 allocate_type: str = "dynamic", min_gain: float = 0.05,
                 on_migrate: Optional[Callable] = None, lr_schedule: Optional[dict] = None,
                 grad_clip: Optional[dict] = None):
        """``allocator_factory(worker_manager) -> Allocator`` builds an allocator (with its model
        and device benchmarkers) around the given pool copy; ``optimizer_cfg`` is the
        ``train_config['optim_cfg']`` dict used to rebuild the optimizer after a migration."""
        assert interval > 0
        self._interval = interval
        self._factory = allocator_factory
        self._optimizer_cfg = dict(optimizer_cfg)
        self._lr_schedule = lr_schedule
        self._grad_clip = grad_clip
        self._type = allocate_type
        self._min_gain = min_gain
        self._on_migrate = on_migrate
        self.migrations = 0
        self.last_decision: Optional[dict] = None

    def after_train_iter(self, runner):
        if runner.iter == 0 or runner.iter % self._interval != 0:
            return
        self.reallocate(runner)

    # ------------------------------------------------------------------ the collective
    def reallocate(self, runner) -> bool:
        from ...parallel import RpcModel, build_optimizer

        old_wm = runner.worker_manager
        new_wm = copy.deepcopy(old_wm)
        allocator = self._factory(new_wm)
        v = max((len(w.chunks) for w in old_wm.worker_pool if getattr(w, "chunks", None)), default=1)
        new_wm = allocator.allocate(self._type, virtual_stages=v)
        dev = allocator.last_device_times
        cost = allocator.last_layer_costs
        if not dev:  # "even" never benchmarks: nothing to compare
            return False
        before = _bottleneck(old_wm, dev, cost)
        after = _bottleneck(new_wm, dev, cost)
        gain = 0.0 if before <= 0 else (before - after) / before
        self.last_decision = dict(iter=runner.iter, before=before, after=after, gain=gain,
                                  old=_layout(old_wm), new=_layout(new_wm))
        if _layout(new_wm) == _layout(old_wm) or gain < self._min_gain:
            runner._log("reallocate: keep {} (predicted gain {:.1%})".format(_layout(old_wm), gain))
            return False
        runner._log("reallocate: {} -> {} (predicted gain {:.1%})".format(
            _layout(old_wm), _layout(new_wm), gain))
        # ---- migrate: layer-indexed state of every rank -> every rank
        local = {}
        for module in runner.model.model:
            if module.is_local:
                b, _e = module.layer_range if module.layer_range is not None else (0, 0)
                for off, layer_sd in enumerate(module.get_state_dict()):
                    local[b + off] = layer_sd
        d = _dist()
        if d is not None:
            gathered = [None] * d.get_world_size()
            d.all_gather_object(gathered, local)
        else:
            gathered = [local]
        per_layer = {}
        for part in gathered:
            per_layer.update(part)
        model = RpcModel(worker_manager=new_wm, this_rank=runner.rank)
        for module in model.model:
            if module.is_local:
                b, e = module.layer_range
                module.load_weights([per_layer[i] for i in range(b, e)])
        model.train(True)
        optimizer = build_optimizer(model.optim_module, dict(self._optimizer_cfg),
                                    lr_schedule=self._lr_schedule, grad_clip=self._grad_clip)
        old = runner.optimizer
        if old is not None and hasattr(old, "step_count") and hasattr(optimizer, "set_step_count"):
            optimizer.set_step_count(old.step_count())
        runner.rebuild(model, optimizer, worker_manager=new_wm)
        self.migrations += 1
        if self._on_migrate is not None:
            self._on_migrate(runner, self.last_decision)
        if d is not None:
            d.barrier()
        return True
