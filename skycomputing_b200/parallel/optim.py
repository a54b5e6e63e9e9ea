"""Per-stage optimizers.

``FusedSGD`` - one multi-tensor kernel launch per step over the stage's flat fp32 parameter banks:
``p -= lr * (g/scale + wd * p)`` (optional momentum), refresh of the bf16 compute shadow and
gradient zeroing in the same pass (csrc/kernels/elementwise_sm100.cu: sgd_multi_kernel).
Parameters that do not live in a native bank (torch.nn fallback layers) are updated by a regular
``torch.optim.SGD`` next to it.

``FusedAdam`` - the same one-launch design for ``Adam`` / ``AdamW`` (adam_multi_kernel): both
moments, master, shadow and gradient zeroing in one pass, the step count lives in device memory so
the update replays correctly inside the whole-step CUDA graph.

``build_optimizer`` keeps the reference's config contract (``optim_cfg = {optim_type: <any
torch.optim class name or "LAMB">, **kwargs}``, experiment/launch.py:152-155): SGD / Adam / AdamW /
LAMB on the native path map to the fused classes, everything else (or options the fused kernels do not cover:
nesterov, dampening, amsgrad, maximize) to the named ``torch.optim`` class over the fp32 masters
(the bf16 shadows are then refreshed lazily by version counter; such a step is NOT graph-safe and
the engines run it eagerly).  Optimizer state lives with the stage, as with the reference's
DistributedOptimizer.

``FusedLamb`` - LAMB (apex ``FusedLAMB`` semantics) in two launches per step over a per-parameter
segment table inside the banks (``lamb_moments`` / ``lamb_update``): a trust ratio per
``nn.Parameter``, weight decay off for names containing ``exclude_from_weight_decay``.  ``Lamb`` is
its torch counterpart (``backend="torch"``, CPU, and parameters outside the banks).

Learning-rate schedules and global-norm gradient clipping (``build_optimizer(..., lr_schedule=,
grad_clip=)``, both opt-in).  The fused optimizers keep them on the device so that a captured step
replays them: ``grad_sumsq_multi`` writes per-block sums of squares of the gradients,
``optim_finalize`` adds them up in a fixed order (plus, in a pipeline, the other stages' shares:
peer-memory slots or one ``all_reduce``, see ``set_norm_reduction``) and writes ``OptimScalars
{lr, clip_coef, grad_norm}``, which ``sgd_multi`` / ``adam_multi`` read.  ``lr = base_lr * f(k)``
with k = optimizer steps already taken, read from a device-side counter.
"""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
import torch.nn as nn

LR_SCHEDULES = {"constant": 1, "linear": 2, "cosine": 3}   # csrc/kernels/api.h LrScheduleType


def lr_factor(schedule: Optional[dict], k: int) -> float:
    """f(k) of the schedule (HF transformers formulas); lr = base_lr * f(k), k = steps taken."""
    if not schedule:
        return 1.0
    w, t = schedule["warmup_steps"], schedule["total_steps"]
    if k < w:
        return k / max(1, w)
    if schedule["type"] == "constant":
        return 1.0
    span = max(1, t - w)
    if schedule["type"] == "linear":
        return max(0.0, (t - k) / span)
    prog = min(1.0, (k - w) / span)   # clamped: the rate does not rise again after T
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))


def check_lr_schedule(cfg: Optional[dict]) -> Optional[dict]:
    """Normalised ``dict(type, warmup_steps, total_steps)`` or None; ValueError when invalid."""
    if cfg is None:
        return None
    cfg = dict(cfg)
    kind = cfg.pop("type", None)
    if kind not in LR_SCHEDULES:
        raise ValueError(f"lr_schedule type must be one of {sorted(LR_SCHEDULES)}, got {kind!r}")
    w = int(cfg.pop("warmup_steps", 0) or 0)
    t = cfg.pop("total_steps", None)
    if cfg:
        raise ValueError(f"unknown lr_schedule keys {sorted(cfg)}")
    if w < 0:
        raise ValueError(f"lr_schedule warmup_steps must be >= 0, got {w}")
    if t is None:
        if kind != "constant":
            raise ValueError(f"lr_schedule {kind!r} needs total_steps")
        t = w
    t = int(t)
    if kind != "constant" and t <= 0:
        raise ValueError(f"lr_schedule total_steps must be > 0, got {t}")
    if w > t:
        raise ValueError(f"lr_schedule warmup_steps ({w}) > total_steps ({t})")
    return dict(type=kind, warmup_steps=w, total_steps=t)


def check_grad_clip(cfg: Optional[dict]) -> Optional[float]:
    """``max_norm`` of ``dict(max_norm=x[, norm_type=2])`` or None; ValueError when invalid."""
    if cfg is None:
        return None
    cfg = dict(cfg)
    if "max_norm" not in cfg:
        raise ValueError("grad_clip needs max_norm")
    max_norm = float(cfg.pop("max_norm"))
    norm_type = float(cfg.pop("norm_type", 2.0))
    if cfg:
        raise ValueError(f"unknown grad_clip keys {sorted(cfg)}")
    if not max_norm > 0.0 or math.isinf(max_norm):
        raise ValueError(f"grad_clip max_norm must be a positive finite number, got {max_norm}")
    if norm_type != 2.0:
        raise ValueError(f"grad_clip supports the L2 norm only (norm_type=2), got {norm_type}")
    return max_norm


# index of local_sumsq, this rank's share of grad_norm^2, in OptimScalars {lr, clip_coef,
# grad_norm, local_sumsq} (csrc/kernels/api.h)
_LOCAL_SUMSQ = 3


class FusedOptimizer:
    """What the fused optimizers share: the stage's de-duplicated parameter banks, a torch
    optimizer for the parameters outside them, the device-side step counter, learning-rate
    schedule and global-norm clipping, and one ``step()``.  A subclass supplies three things:
    ``_state_buffers()`` ({state_dict key: one buffer or None per bank}), ``_fallback(module,
    params)`` (the torch optimizer class and its parameter groups for the parameters outside the
    banks) and ``_update(stream, grad_scale, scalars)``, which launches the update of every bank
    (``scalars``: the device OptimScalars pointer, or 0)."""

    def __init__(self, module: nn.Module, banks: Optional[list], defaults: dict, counter: bool):
        from ..models.bert_layers import native_param_banks
        from ..ops import native as nat

        self._nat = nat
        banks = native_param_banks(module) if banks is None else banks
        self.banks = list({id(b): b for b in banks}.values())
        for b in self.banks:
            b.ensure()
        self.param_groups = [defaults]
        params = list(module.parameters())
        self._device = self.banks[0].master().device if self.banks else (
            params[0].device if params else torch.device("cpu"))
        bank_params = {id(p) for b in self.banks for p in b.params}
        rest = [p for p in params if id(p) not in bank_params and p.requires_grad]
        cls, groups = self._fallback(module, rest) if rest else (None, None)
        self._rest_opt = cls(groups) if rest else None
        self._overwrite_ok = os.environ.get("SKY_SGD_OVERWRITE", "1") != "0"
        self._zeroing_decided = False
        self._desc_dev: Optional[torch.Tensor] = None
        self._desc_count = 0
        self._max_numel = 0
        # ids of the banks whose update an engine applies in their weight-gradient GEMMs
        # (set_update_in_wgrad): the descriptor table leaves them out
        self._in_wgrad: frozenset = frozenset()
        # device-side count of steps taken: Adam's bias correction and the learning-rate schedule
        self._step = torch.zeros(1, dtype=torch.int64, device=self._device) if counter else None
        self._step_offset = 0                     # schedule steps taken by an earlier optimizer
        # learning-rate schedule / gradient clipping (configure()); all None = the plain update
        self._sched: Optional[dict] = None
        self._max_norm: Optional[float] = None
        self._scalars: Optional[torch.Tensor] = None      # device OptimScalars
        self._partials: Optional[torch.Tensor] = None
        self._sumsq_blocks = 0
        self._rest_sumsq: Optional[torch.Tensor] = None
        self._norm_allreduce = False
        self._norm_group = None
        self._norm_exchange = None
        # banks / torch-path parameters left out of this rank's share of the squared norm: a tied
        # table's replica, whose (identical) gradient the table's rank counts
        self._norm_skip: frozenset = frozenset()
        self._norm_desc: Optional[torch.Tensor] = None
        self._norm_desc_count = 0
        self._norm_max_numel = 0
        self._stepped = False

    @property
    def graph_safe(self) -> bool:
        """True when step() is pure device work with static addresses (CUDA-graph capturable)."""
        return self._rest_opt is None

    def configure(self, lr_schedule: Optional[dict] = None, max_norm: Optional[float] = None) -> None:
        """Device-side learning-rate schedule and / or global-norm clipping (validated configs,
        see build_optimizer).  The step() of a captured graph then replays both correctly."""
        self._sched, self._max_norm = lr_schedule, max_norm
        if lr_schedule is None and max_norm is None:
            return
        self._scalars = torch.zeros(self._nat.ext().OPTIM_SCALARS_FLOATS, dtype=torch.float32,
                                    device=self._device)
        if lr_schedule is not None and self._step is None:
            self._step = torch.zeros(1, dtype=torch.int64, device=self._device)

    @property
    def needs_global_norm(self) -> bool:
        """True when step() needs the gradient norm over every pipeline stage."""
        return self._max_norm is not None

    @property
    def reports_scalars(self) -> bool:
        return self._scalars is not None

    def set_norm_reduction(self, group=None, allreduce: bool = False, exchange=None) -> None:
        """How step() adds up the stages' shares of the squared norm: ``exchange`` (a
        p2p.GradNormExchange: peer-memory slots, capturable), ``allreduce`` (one fp32
        ``dist.all_reduce`` over ``group``) or neither (single stage)."""
        self._norm_exchange = exchange
        self._norm_allreduce = bool(allreduce) and exchange is None
        self._norm_group = group

    def set_norm_exclude(self, params) -> None:
        """Leave ``params`` (and the banks that hold them) out of this rank's share of the global
        gradient norm: the replica of a tied table, counted on the table's rank."""
        ids = frozenset(id(p) for p in params)
        self._norm_skip = ids | frozenset(id(b) for b in self.banks
                                          if any(id(p) in ids for p in b.params))
        self._norm_desc = None
        self._partials = None

    def rebind_banks(self) -> None:
        """A bank's buffers moved (a tied replica's gradient now lives in exchange memory):
        rebuild the descriptor / segment tables on the next step.  Not inside a captured step."""
        self._desc_dev = None
        self._norm_desc = None
        self._partials = None
        if getattr(self, "_lamb", None) is not None:
            self._lamb = None

    def _norm_table(self):
        """(descriptor table, count, max numel) of the banks whose gradients make up this rank's
        share of the squared norm: the update table, or a table without the excluded banks."""
        d = self._descriptors()
        if not self._norm_skip:
            return d, self._desc_count, self._max_numel
        if self._norm_desc is None:
            self._decide_zeroing()
            descs = [b.sgd_descriptor() for b in self.banks
                     if id(b) not in self._in_wgrad and id(b) not in self._norm_skip]
            self._norm_desc_count = len(descs)
            self._norm_max_numel = max((x[4] for x in descs), default=0)
            if descs:
                raw = self._nat.ext().pack_sgd_descriptors(descs)
                host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
                self._norm_desc = host.to(self._device)
        return self._norm_desc, self._norm_desc_count, self._norm_max_numel

    def _compute_scalars(self, grad_scale: float, stream: int) -> None:
        """grad_sumsq_multi + optim_finalize: writes lr / clip_coef / grad_norm for this step,
        reading k from the step counter before step() advances it."""
        ext = self._nat.ext()
        partials, n_part, extra = 0, 0, 0
        if self._max_norm is not None:
            d, count, max_numel = self._norm_table() if self.banks else (None, 0, 0)
            if count:
                if self._partials is None:
                    blocks = ext.grad_sumsq_blocks(max_numel)
                    self._partials = torch.zeros(blocks * count, dtype=torch.float32,
                                                 device=self._device)
                    self._sumsq_blocks = blocks
                ext.grad_sumsq_multi(d.data_ptr(), count, self._sumsq_blocks,
                                     float(grad_scale), self._partials.data_ptr(), stream)
                partials, n_part = self._partials.data_ptr(), self._partials.numel()
            if self._rest_opt is not None:
                # torch fallback layers (eager anyway: such an optimizer is not graph-safe)
                grads = self._rest_grads(counted_only=True)
                self._rest_sumsq = (torch.stack([g.float().pow(2).sum() for g in grads]).sum()
                                    if grads else torch.zeros((), device=self._device)).reshape(1)
                extra = self._rest_sumsq.data_ptr()
        sched = self._sched
        common = dict(step=self._step.data_ptr() if self._step is not None else 0,
                      step_offset=int(self._step_offset),
                      schedule=LR_SCHEDULES[sched["type"]] if sched else 0,
                      warmup=sched["warmup_steps"] if sched else 0,
                      total=sched["total_steps"] if sched else 0,
                      base_lr=float(self.param_groups[0]["lr"]),
                      max_norm=float(self._max_norm or 0.0), out=self._scalars.data_ptr(),
                      stream=stream)
        ex = self._norm_exchange
        if ex is not None and self._max_norm is not None:
            ext.optim_finalize(partials, n_part, extra, regions=ex.regions_ptr, n_ranks=ex.n_ranks,
                               my_pos=ex.position, epoch=ex.epoch_ptr, error_flag=ex.error_ptr,
                               **common)
        elif self._norm_allreduce and self._max_norm is not None:
            import torch.distributed as dist

            ext.optim_finalize(partials, n_part, extra, **common)    # this rank's share
            local = self._scalars[_LOCAL_SUMSQ:_LOCAL_SUMSQ + 1]
            dist.all_reduce(local, group=self._norm_group)
            ext.optim_finalize(0, 0, local.data_ptr(), **common)
        else:
            ext.optim_finalize(partials, n_part, extra, **common)

    def _rest_grads(self, counted_only: bool = False) -> list:
        return [p.grad for g in self._rest_opt.param_groups for p in g["params"]
                if p.grad is not None and not (counted_only and id(p) in self._norm_skip)]

    def _rest_step(self) -> None:
        if self._scalars is not None:
            if self._max_norm is not None:
                for g in self._rest_grads():
                    g.mul_(self._scalars[1])
            if self._sched is not None:
                k = self.step_count() - 1      # the device counter was advanced for this step
                for grp in self._rest_opt.param_groups:
                    grp["lr"] = float(self.param_groups[0]["lr"]) * lr_factor(self._sched, k)
        self._rest_opt.step()
        self._rest_opt.zero_grad(set_to_none=False)

    def scalars(self) -> dict:
        """lr and global grad_norm of the last step (None where not configured / no step yet)."""
        if self._scalars is None or not self._stepped:
            return dict(lr=None, grad_norm=None)
        lr, _coef, norm, _local = self._scalars.tolist()
        return dict(lr=lr, grad_norm=norm if self._max_norm is not None else None)

    def step_count(self) -> int:
        """Optimizer steps taken, as the learning-rate schedule counts them."""
        return (int(self._step.item()) if self._step is not None else 0) + self._step_offset

    def set_step_count(self, k: int) -> None:
        """Continue the schedule at step k (a rebuilt optimizer after a layer migration); the
        device counter that also drives Adam's bias correction is left alone, because the moments
        restart with the new optimizer."""
        self._step_offset = int(k) - (int(self._step.item()) if self._step is not None else 0)

    def _decide_zeroing(self) -> None:
        """Banks that received a wgrad GEMM in the first backward pass will receive one in every
        step: their gradient need not be zeroed, the next step's first wgrad overwrites it
        (``overwrite_first``).  Decided once, before the first descriptor or segment table."""
        if not self._zeroing_decided:
            for b in self.banks:
                target = bool(getattr(b, "wgrad_target", False)) or id(b) in self._in_wgrad
                # a tied table has several gradient writers: always accumulate into zeros
                b.overwrite_first = target and self._overwrite_ok and not getattr(b, "tied", False)
            self._zeroing_decided = True

    def wgrad_sgd_args(self) -> Optional[tuple]:
        """(lr, weight_decay, grad_scale) of the update that weight-gradient GEMMs may apply in
        their epilogue when the engine's step is this optimizer's plain SGD update; None (the
        default) when step() must see every gradient first."""
        return None

    def set_update_in_wgrad(self, banks: list) -> None:
        """The engine applies the update of ``banks`` (a subset of ``self.banks``) in the last
        weight-gradient GEMM of every step: step() leaves them out of its descriptor table, and
        their gradients stay un-zeroed (the next step's first wgrad overwrites them).  ``[]``
        hands every bank back to step()."""
        ids = frozenset(id(b) for b in banks)
        if ids != self._in_wgrad:
            self._in_wgrad = ids
            self._desc_dev = None
            self._zeroing_decided = False

    def _descriptors(self) -> Optional[torch.Tensor]:
        """The SgdTensor table on the device of the banks step() updates (all of them but those
        updated in their weight-gradient GEMMs), built once; None when there are none."""
        if self._desc_dev is None and self.banks:
            self._decide_zeroing()
            bufs = self._state_buffers()
            mom2 = bufs.get("second_moment", [None] * len(self.banks))
            descs = [b.sgd_descriptor(m, v) for b, m, v in zip(self.banks, bufs["momentum"], mom2)
                     if id(b) not in self._in_wgrad]
            self._desc_count = len(descs)
            if descs:
                raw = self._nat.ext().pack_sgd_descriptors(descs)
                host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
                self._desc_dev = host.to(self.banks[0].master().device)
                self._max_numel = max(d[4] for d in descs)
        return self._desc_dev

    def step(self, grad_scale: float = 1.0) -> None:
        configured = self._scalars is not None
        stream = torch.cuda.current_stream().cuda_stream if self.banks or configured else 0
        sc = 0
        if configured:
            self._compute_scalars(grad_scale, stream)
            sc = self._scalars.data_ptr()
            self._stepped = True
        # the counter counts the steps that ran device work, and only those
        if self._step is not None and (self.banks or configured):
            self._nat.ext().advance_counter(self._step.data_ptr(), 1, stream)
        if self.banks:
            self._update(stream, float(grad_scale), sc)
            for b in self.banks:
                if b.overwrite_first:
                    b.fresh = True
        if self._rest_opt is not None:
            self._rest_step()

    def zero_grad(self, set_to_none: bool = False) -> None:
        for b in self.banks:
            b.grad().zero_()
            b.fresh = False
        if self._rest_opt is not None:
            self._rest_opt.zero_grad(set_to_none=False)

    def state_dict(self) -> dict:
        sd = {k: [None if t is None else t.detach().cpu() for t in bufs]
              for k, bufs in self._state_buffers().items()}
        sd.update(rest=None if self._rest_opt is None else self._rest_opt.state_dict(),
                  param_groups=self.param_groups)
        if self._step is not None:
            sd["step"] = int(self._step.item())
        if self._sched is not None:
            sd["lr_schedule_step"] = self.step_count()
        return sd

    def load_state_dict(self, sd: dict) -> None:
        for k, bufs in self._state_buffers().items():
            for t, s in zip(bufs, sd.get(k, [])):
                if t is not None and s is not None:
                    t.copy_(s)
        if self._rest_opt is not None and sd.get("rest") is not None:
            self._rest_opt.load_state_dict(sd["rest"])
        self.param_groups = sd.get("param_groups", self.param_groups)
        if self._step is not None and "step" in sd:
            self._step.fill_(int(sd["step"]))
        if "lr_schedule_step" in sd:
            self.set_step_count(int(sd["lr_schedule_step"]))


class FusedSGD(FusedOptimizer):
    """``torch.optim.SGD`` (plain or momentum) as one multi-tensor launch per step."""

    def __init__(self, module: nn.Module, lr: float = 1e-3, momentum: float = 0.0,
                 weight_decay: float = 0.0, dampening: float = 0.0, nesterov: bool = False,
                 banks: Optional[list] = None):
        if dampening != 0.0 or nesterov:
            raise ValueError("FusedSGD supports plain / momentum SGD only")
        self.lr, self.momentum, self.weight_decay = lr, momentum, weight_decay
        super().__init__(module, banks, dict(lr=lr, momentum=momentum, weight_decay=weight_decay),
                         counter=False)
        self._mom = [torch.zeros_like(b.master()) if momentum else None for b in self.banks]

    def _fallback(self, module, params):
        return torch.optim.SGD, [dict(params=params, lr=self.lr, momentum=self.momentum,
                                      weight_decay=self.weight_decay)]

    def _state_buffers(self) -> dict:
        return dict(momentum=self._mom)

    def wgrad_sgd_args(self) -> Optional[tuple]:
        """Plain SGD (no momentum, no schedule, no clipping) needs no gradient but a bank's own:
        the update of a bank can ride in its last weight-gradient GEMM.  grad_scale is 1: the
        engines step with it."""
        if self.momentum != 0.0 or self._scalars is not None or not self._overwrite_ok:
            return None
        return (float(self.param_groups[0]["lr"]), float(self.weight_decay), 1.0)

    def _update(self, stream, grad_scale, scalars):
        d = self._descriptors()
        if d is None:
            return   # every bank is updated in its weight-gradient GEMMs
        self._nat.ext().sgd_multi(
            d_tensors=d.data_ptr(), n=self._desc_count, max_numel=self._max_numel,
            lr=float(self.param_groups[0]["lr"]), momentum=float(self.momentum),
            weight_decay=float(self.weight_decay), grad_scale=grad_scale, zero_grad=True,
            stream=stream, scalars=scalars)


class FusedAdam(FusedOptimizer):
    """``torch.optim.Adam`` / ``AdamW`` (amsgrad=False) as one multi-tensor launch per step."""

    def __init__(self, module: nn.Module, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, decoupled: bool = False, amsgrad: bool = False,
                 maximize: bool = False, banks: Optional[list] = None, **unsupported):
        if amsgrad or maximize or unsupported:
            raise ValueError("FusedAdam covers plain Adam / AdamW only")
        self.lr, self.weight_decay = lr, weight_decay
        self.betas, self.eps, self.decoupled = (float(betas[0]), float(betas[1])), eps, decoupled
        super().__init__(module, banks, dict(lr=lr, betas=self.betas, eps=eps,
                                             weight_decay=weight_decay), counter=True)
        self._mom = [torch.zeros_like(b.master()) for b in self.banks]
        self._mom2 = [torch.zeros_like(b.master()) for b in self.banks]

    def _fallback(self, module, params):
        cls = torch.optim.AdamW if self.decoupled else torch.optim.Adam
        return cls, [dict(params=params, lr=self.lr, betas=self.betas, eps=self.eps,
                          weight_decay=self.weight_decay)]

    def _state_buffers(self) -> dict:
        return dict(momentum=self._mom, second_moment=self._mom2)

    def _update(self, stream, grad_scale, scalars):
        d = self._descriptors()
        self._nat.ext().adam_multi(
            d_tensors=d.data_ptr(), n=self._desc_count, max_numel=self._max_numel,
            lr=float(self.param_groups[0]["lr"]), beta1=self.betas[0], beta2=self.betas[1],
            eps=float(self.eps), weight_decay=float(self.weight_decay),
            decoupled=bool(self.decoupled), step=self._step.data_ptr(), grad_scale=grad_scale,
            zero_grad=True, stream=stream, scalars=scalars)


LAMB_DEFAULTS = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01,
                     exclude_from_weight_decay=("bias", "LayerNorm"))


def check_lamb_cfg(cfg: dict) -> dict:
    """LAMB options (``optim_cfg`` without ``optim_type``) completed with LAMB_DEFAULTS;
    ValueError for unknown keys or values outside their range."""
    cfg = dict(cfg)
    unknown = sorted(set(cfg) - set(LAMB_DEFAULTS))
    if unknown:
        raise ValueError(f"unknown LAMB options {unknown}; allowed: {sorted(LAMB_DEFAULTS)}")
    out = dict(LAMB_DEFAULTS, **cfg)
    lr, eps, wd = float(out["lr"]), float(out["eps"]), float(out["weight_decay"])
    try:
        b1, b2 = (float(b) for b in out["betas"])
    except (TypeError, ValueError):
        raise ValueError(f"LAMB betas must be two numbers, got {out['betas']!r}") from None
    if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0):
        raise ValueError(f"LAMB betas must lie in [0, 1), got {(b1, b2)}")
    if not eps > 0.0:
        raise ValueError(f"LAMB eps must be > 0, got {eps}")
    if not wd >= 0.0:
        raise ValueError(f"LAMB weight_decay must be >= 0, got {wd}")
    if not lr >= 0.0:
        raise ValueError(f"LAMB lr must be >= 0, got {lr}")
    excl = out["exclude_from_weight_decay"]
    if isinstance(excl, str) or not all(isinstance(s, str) and s for s in excl):
        raise ValueError("LAMB exclude_from_weight_decay must be a sequence of non-empty "
                         f"strings, got {excl!r}")
    return dict(lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd,
                exclude_from_weight_decay=tuple(excl))


def lamb_weight_decay(name: str, weight_decay: float, exclude, param=None) -> float:
    """λ of the parameter called ``name``: 0 when the name contains one of ``exclude``.  A word
    table tied to a decoder (``param.tied_name``) decides under that name, so that the table and
    its replica on another rank cannot be treated differently."""
    name = getattr(param, "tied_name", None) or name
    return 0.0 if any(s in name for s in exclude) else weight_decay


def lamb_param_groups(module: nn.Module, weight_decay: float, exclude, params=None) -> list:
    """Parameter groups of ``module`` (or of its ``params`` subset) by weight decay, named as in
    ``module.named_parameters()``: the decayed ones first, then the excluded ones."""
    keep = None if params is None else {id(p) for p in params}
    groups = {}
    for name, p in module.named_parameters():
        if not p.requires_grad or (keep is not None and id(p) not in keep):
            continue
        wd = lamb_weight_decay(name, weight_decay, exclude, p)
        g = groups.setdefault(wd, dict(params=[], names=[], weight_decay=wd))
        g["params"].append(p)
        g["names"].append(name)
    return sorted(groups.values(), key=lambda g: -g["weight_decay"])


class Lamb(torch.optim.Optimizer):
    """LAMB (You et al. 2019) with apex ``FusedLAMB``'s defaults: decoupled weight decay inside
    the update, bias correction, no NVLAMB.  Per tensor W with weight decay λ, at step t::

        m = β1 m + (1-β1) g,   v = β2 v + (1-β2) g²
        u = (m / (1-β1^t)) / (sqrt(v / (1-β2^t)) + eps) + λ W
        r = ||W|| / ||u||  if λ != 0 and both norms > 0, else 1
        W ← W - lr · r · u

    The torch path of ``optim_type="LAMB"`` and the reference of the fused kernels.  No host
    synchronisation: r stays a device tensor (``state[p]["trust_ratio"]``)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6,
                 weight_decay: float = 0.0):
        chk = check_lamb_cfg(dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        chk.pop("exclude_from_weight_decay")
        super().__init__(params, chk)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                st["step"] += 1
                t = st["step"]
                g = p.grad
                m, v = st["exp_avg"], st["exp_avg_sq"]
                m.mul_(b1).add_(g, alpha=1.0 - b1)
                v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
                u = (m / (1.0 - b1 ** t)) / ((v / (1.0 - b2 ** t)).sqrt() + eps)
                if wd != 0.0:
                    u.add_(p, alpha=wd)
                    wn, un = torch.linalg.vector_norm(p), torch.linalg.vector_norm(u)
                    r = torch.where((wn > 0) & (un > 0), wn / un, torch.ones_like(wn))
                else:
                    r = torch.ones((), dtype=p.dtype, device=p.device)
                st["trust_ratio"] = r
                p.sub_(u * (r * lr))
        return loss


class FusedLamb(FusedAdam):
    """LAMB (see ``Lamb``) over the stage's flat parameter banks in two launches per step.

    Every ``nn.Parameter`` inside a bank is one segment with its own λ and trust ratio (``wqkv``
    holds three).  ``lamb_moments`` updates m and v and writes fp32 partials of ||W||² and ||u||²
    per fixed-size chunk; ``lamb_update`` sums a segment's partials in fp64 in a fixed order, forms
    r and applies the update with the bf16 shadow refresh.  No host sync, no per-step host-to-device
    copy: graph-safe like ``FusedAdam``, whose moments and step counter it shares.  Parameters outside the banks are stepped by ``Lamb``."""

    def __init__(self, module: nn.Module, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6,
                 weight_decay: float = 0.01, exclude_from_weight_decay=("bias", "LayerNorm"),
                 banks: Optional[list] = None):
        chk = check_lamb_cfg(dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                  exclude_from_weight_decay=exclude_from_weight_decay))
        self.exclude = chk["exclude_from_weight_decay"]
        self._names = {id(p): n for n, p in module.named_parameters()}
        super().__init__(module, lr=chk["lr"], betas=chk["betas"], eps=chk["eps"],
                         weight_decay=chk["weight_decay"], decoupled=True, banks=banks)
        self.param_groups[0]["exclude_from_weight_decay"] = self.exclude
        self._lamb = None          # (segments, chunk table, n_chunks) on the device, built once
        self._seg_info: list = []
        self._lamb_partials: Optional[torch.Tensor] = None
        self._ratios: Optional[torch.Tensor] = None
        self._lamb_stepped = False

    def _fallback(self, module, params):
        groups = lamb_param_groups(module, self.weight_decay, self.exclude, params)
        return Lamb, [dict(g, lr=self.lr, betas=self.betas, eps=self.eps) for g in groups]

    def segments(self) -> list:
        """The segment table as dicts: name, bank (index into ``banks``), offset and numel in the
        bank's flat buffer, weight_decay, use_ratio, skip_zero, aligned (float4 path)."""
        if self._lamb is None:
            return lamb_segments(self.banks, self._names, self.weight_decay, self.exclude)
        return [dict(s) for s in self._seg_info]

    def _lamb_table(self):
        if self._lamb is None:
            self._decide_zeroing()
            ext = self._nat.ext()
            info = lamb_segments(self.banks, self._names, self.weight_decay, self.exclude)
            rows = []
            for s in info:
                b = self.banks[s["bank"]]
                i, off = s["bank"], s["offset"]
                shadow = b.shadow().data_ptr() + 2 * off if b.need_shadow else 0
                rows.append((b.master().data_ptr() + 4 * off, b.grad().data_ptr() + 4 * off,
                             self._mom[i].data_ptr() + 4 * off, self._mom2[i].data_ptr() + 4 * off,
                             shadow, s["numel"], s["weight_decay"], int(s["use_ratio"]),
                             int(s["skip_zero"])))
            seg_raw, chunk_raw, n_chunks, vec = ext.pack_lamb_segments(rows)
            for s, a in zip(info, vec):
                s["aligned"] = bool(a)
            dev = self._device
            segs = torch.frombuffer(bytearray(seg_raw), dtype=torch.uint8).to(dev)
            chunks = torch.frombuffer(bytearray(chunk_raw), dtype=torch.uint8).to(dev)
            self._lamb_partials = torch.zeros(2 * max(1, n_chunks), dtype=torch.float32, device=dev)
            self._ratios = torch.ones(max(1, len(info)), dtype=torch.float32, device=dev)
            self._lamb = (segs, chunks, n_chunks)
            self._seg_info = info
        return self._lamb

    def _update(self, stream, grad_scale, scalars):
        segs, chunks, n_chunks = self._lamb_table()
        ext = self._nat.ext()
        b1, b2 = self.betas
        ext.lamb_moments(segs.data_ptr(), chunks.data_ptr(), n_chunks, b1, b2, float(self.eps),
                         self._step.data_ptr(), grad_scale, self._lamb_partials.data_ptr(), stream,
                         scalars)
        ext.lamb_update(segs.data_ptr(), chunks.data_ptr(), n_chunks,
                        float(self.param_groups[0]["lr"]), b1, b2, float(self.eps),
                        self._step.data_ptr(), self._lamb_partials.data_ptr(),
                        self._ratios.data_ptr(), stream, scalars)
        self._lamb_stepped = True

    def trust_ratios(self) -> dict:
        """{parameter name: r} of the last step (one device-to-host copy; {} before the first
        step).  Parameters outside the banks report the ratio ``Lamb`` used for them."""
        out = {}
        if self._lamb_stepped:
            out.update(zip((s["name"] for s in self._seg_info), self._ratios.tolist()))
        if self._rest_opt is not None:
            for g in self._rest_opt.param_groups:
                for name, p in zip(g["names"], g["params"]):
                    r = self._rest_opt.state.get(p, {}).get("trust_ratio")
                    if r is not None:
                        out[name] = float(r)
        return out


def lamb_segments(banks: list, names: dict, weight_decay: float, exclude) -> list:
    """One segment per ``nn.Parameter`` of ``banks``, in bank order: dict(name, bank, offset,
    numel, weight_decay, use_ratio, skip_zero, aligned).  ``names`` maps id(param) to its name in
    the stage (``named_parameters()``); offsets are in elements of the bank's flat buffer and
    ``aligned`` (float4 path) holds when the offset is a multiple of 4 elements."""
    out = []
    for i, b in enumerate(banks):
        flat = b.master()
        for p in b.params:
            off = (p.data_ptr() - flat.data_ptr()) // flat.element_size()
            name = names.get(id(p), f"<bank {i}>.{len(out)}")
            wd = lamb_weight_decay(name, weight_decay, exclude, p)
            if p.numel() == 0:
                continue
            out.append(dict(name=name, bank=i, offset=int(off), numel=p.numel(), weight_decay=wd,
                            use_ratio=wd != 0.0, skip_zero=bool(b.overwrite_first),
                            aligned=off % 4 == 0))
    return out


class TorchOptimizerAdapter:
    """Any ``torch.optim`` class over the stage's parameters; same step()/zero_grad() surface."""

    # host-side bookkeeping (step counters, lazily created state, version-counter driven refresh of
    # the bf16 shadows): must not be captured into a CUDA graph
    graph_safe = False

    def __init__(self, optimizer: torch.optim.Optimizer):
        self.optimizer = optimizer
        self.param_groups = optimizer.param_groups
        self._sched: Optional[dict] = None
        self._scheduler = None
        self._max_norm: Optional[float] = None
        self._norm_allreduce = False
        self._norm_group = None
        self._last_lr: Optional[float] = None
        self._last_norm: Optional[torch.Tensor] = None
        self._norm_skip: frozenset = frozenset()

    def configure(self, lr_schedule: Optional[dict] = None, max_norm: Optional[float] = None) -> None:
        """Learning-rate schedule (a LambdaLR stepped after every step()) and / or global-norm
        clipping of ``p.grad`` before the step."""
        self._sched, self._max_norm = lr_schedule, max_norm
        if lr_schedule is not None:
            self._scheduler = torch.optim.lr_scheduler.LambdaLR(
                self.optimizer, lambda k: lr_factor(lr_schedule, k))

    needs_global_norm = property(lambda self: self._max_norm is not None)
    reports_scalars = property(lambda self: self._sched is not None or self._max_norm is not None)

    def set_norm_reduction(self, group=None, allreduce: bool = False, exchange=None) -> None:
        self._norm_allreduce = bool(allreduce) or exchange is not None
        self._norm_group = group

    def set_norm_exclude(self, params) -> None:
        """See FusedOptimizer.set_norm_exclude: still clipped, not counted in the norm."""
        self._norm_skip = frozenset(id(p) for p in params)

    def _clip(self) -> None:
        """torch.nn.utils.clip_grad_norm_ over every stage: local sum of squares, all_reduce of
        that one element, then the same coefficient on every rank."""
        params = [p for g in self.optimizer.param_groups for p in g["params"]]
        grads = [p.grad for p in params if p.grad is not None]
        counted = [p.grad for p in params if p.grad is not None and id(p) not in self._norm_skip]
        if counted:
            sumsq = torch.stack([torch.linalg.vector_norm(g.detach(), 2.0) for g in counted]
                                ).float().pow(2).sum()
        else:
            sumsq = torch.zeros((), dtype=torch.float32, device=params[0].device)
        if self._norm_allreduce:
            import torch.distributed as dist

            dist.all_reduce(sumsq, group=self._norm_group)
        norm = sumsq.sqrt()
        coef = torch.clamp(self._max_norm / (norm + 1e-6), max=1.0)
        for g in grads:
            g.mul_(coef.to(g.dtype))
        self._last_norm = norm

    def step(self, grad_scale: float = 1.0) -> None:
        if grad_scale != 1.0:
            for g in self.optimizer.param_groups:
                for p in g["params"]:
                    if p.grad is not None:
                        p.grad.mul_(grad_scale)
        if self._max_norm is not None:
            self._clip()
        self._last_lr = float(self.optimizer.param_groups[0]["lr"])
        self.optimizer.step()
        self.optimizer.zero_grad(set_to_none=False)
        if self._scheduler is not None:
            self._scheduler.step()

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.optimizer.zero_grad(set_to_none=False)

    def scalars(self) -> dict:
        return dict(lr=self._last_lr if self.reports_scalars else None,
                    grad_norm=None if self._last_norm is None else float(self._last_norm))

    def step_count(self) -> int:
        return int(self._scheduler.last_epoch) if self._scheduler is not None else 0

    def set_step_count(self, k: int) -> None:
        if self._scheduler is None:
            return
        self._scheduler.last_epoch = int(k)
        for g in self.optimizer.param_groups:
            g["lr"] = g["initial_lr"] * lr_factor(self._sched, int(k))
        self._scheduler._last_lr = [g["lr"] for g in self.optimizer.param_groups]

    def state_dict(self):
        sd = self.optimizer.state_dict()
        if self._scheduler is not None:
            sd = dict(sd, lr_schedule_step=self.step_count())
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        k = sd.pop("lr_schedule_step", None)
        self.optimizer.load_state_dict(sd)
        if k is not None:
            self.set_step_count(int(k))


def build_optimizer(module: nn.Module, optim_cfg: dict, prefer_fused: bool = True,
                    lr_schedule: Optional[dict] = None, grad_clip: Optional[dict] = None):
    """``lr_schedule = dict(type="constant"|"linear"|"cosine", warmup_steps=W, total_steps=T)``,
    ``grad_clip = dict(max_norm=x)`` (L2): both optional, invalid values raise ValueError here."""
    sched = check_lr_schedule(lr_schedule)
    max_norm = check_grad_clip(grad_clip)
    opt = _build_optimizer(module, optim_cfg, prefer_fused)
    if sched is not None or max_norm is not None:
        opt.configure(sched, max_norm)
    return opt


def _build_optimizer(module: nn.Module, optim_cfg: dict, prefer_fused: bool):
    cfg = dict(optim_cfg)
    optim_type = cfg.pop("optim_type", "SGD")
    params = [p for p in module.parameters() if p.requires_grad]
    from ..models.bert_layers import native_active

    fused = prefer_fused and any(native_active(p.device) for p in params)
    if optim_type == "LAMB":
        # no torch.optim class to fall back to: every option is checked here, on every backend
        cfg = check_lamb_cfg(cfg)
        if fused:
            return FusedLamb(module, **cfg)
        if params:
            excl = cfg.pop("exclude_from_weight_decay")
            return TorchOptimizerAdapter(
                Lamb(lamb_param_groups(module, cfg["weight_decay"], excl), **cfg))
    if optim_type in ("SGD", "Adam", "AdamW") and fused:
        try:
            if optim_type == "SGD":
                return FusedSGD(module, **cfg)
            if optim_type == "AdamW":
                cfg.setdefault("weight_decay", 1e-2)   # torch.optim.AdamW's default
            return FusedAdam(module, decoupled=optim_type == "AdamW", **cfg)
        except (ValueError, TypeError):
            cfg = dict(optim_cfg)
            cfg.pop("optim_type", None)
    if not params:
        return TorchOptimizerAdapter(torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.0))
    return TorchOptimizerAdapter(getattr(torch.optim, optim_type)(params, **cfg))
