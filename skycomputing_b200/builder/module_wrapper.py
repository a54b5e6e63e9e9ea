"""Per-stage runtime (``ModuleWrapper``): owns the contiguous slice of layers one device runs.

Capability parity with scaelum/builder/module_wrapper.py:22-299 - same constructor signature
(= ``worker.extra_config`` + rank), forward timing, simulated slow device (``slowdown``), forward /
backward time log lines, ``detect_mem`` - re-designed for one-process-per-GPU execution:

* no RRef fetch / CPU staging: inputs arrive as device tensors (or through a fused peer channel);
* time is measured on the DEVICE (CUDA events around the stage's kernels, resolved lazily so the
  hot path never synchronises) instead of ``time.time()`` around ``cuda.synchronize()``;
* ``slowdown`` is a device-side throttle: a spin kernel that holds the stream for
  ``slowdown x (elapsed device time of the stage)`` - the analogue of ``time.sleep(comp_time *
  slowdown)`` (module_wrapper.py:124-126) and of the backward throttle (:254-283) without blocking
  the host or cloning tensors (the reference pays two clones per boundary tensor per direction);
* adjacent ``BertLayer_Head/Body/Tail`` entries of one transformer block are fused into a single
  autograd node (``BertSpan``) running the sm_90a kernels.
"""
from __future__ import annotations

import contextlib
import subprocess
import time
from typing import List, Optional

import psutil
import torch
import torch.nn as nn

from ..logger import Logger
from ..timer import DistributedTimer
from .sequential_wrapper import SequentialWrapper


class _BackwardProbe(torch.autograd.Function):
    """Identity whose backward marks the start / end of this stage's backward pass.

    ``is_input_side=False`` (placed on stage outputs) fires FIRST in backward: it records the
    start time.  ``is_input_side=True`` (placed on stage inputs) fires LAST: it throttles for
    ``slowdown x elapsed`` and logs.  No tensor is cloned.
    """

    @staticmethod
    def forward(ctx, feat, owner, is_input_side):
        ctx.owner = owner
        ctx.is_input_side = is_input_side
        return feat.view_as(feat)

    @staticmethod
    def backward(ctx, grad_output):
        owner = ctx.owner
        if ctx.is_input_side:
            owner._on_backward_end()
        else:
            owner._on_backward_start()
        return grad_output, None, None


class BackwardSlowdownFunction(torch.autograd.Function):
    """Stand-alone form of the backward probe with the reference's call signature
    (scaelum/builder/module_wrapper.py:240-283): an identity on ``feat`` whose backward measures the
    interval since the previous probe through ``timer`` (a ``DistributedTimer``), throttles for
    ``interval * slowdown`` when ``do_slowdown`` and logs.  ``ModuleWrapper`` itself uses the
    clone-free ``_BackwardProbe`` pair with device events; this class exists for code that builds
    its own stages out of the reference's pieces.  Returns exactly one gradient per input (the
    reference returns seven for six, SURVEY §2.7)."""

    @staticmethod
    def forward(ctx, feat, rank, slowdown, timer, logger, do_slowdown):
        ctx.rank, ctx.slowdown, ctx.timer, ctx.logger = rank, slowdown, timer, logger
        ctx.do_slowdown = do_slowdown
        return feat.view_as(feat)

    @staticmethod
    def backward(ctx, grad_output):
        timer, logger = ctx.timer, ctx.logger
        if ctx.do_slowdown:
            if grad_output.is_cuda:
                torch.cuda.current_stream(grad_output.device).synchronize()
            if timer is not None:
                timer.add_timestamp()
                try:
                    interval = timer.get_prev_interval()
                except (IndexError, ValueError):  # first stamp of the run: nothing to compare with
                    interval = 0.0
                if ctx.slowdown and interval > 0:
                    time.sleep(interval * ctx.slowdown)
                if logger is not None:
                    logger.info("backward time on rank {}: {}".format(
                        ctx.rank, interval * (1 + (ctx.slowdown or 0))))
                timer.add_timestamp()
        elif timer is not None:
            timer.add_timestamp()
        return grad_output, None, None, None, None, None


class BackwardSlowdownModule(nn.Module):
    """nn.Module face of :class:`BackwardSlowdownFunction` (scaelum module_wrapper.py:286-299)."""

    def __init__(self, rank, slowdown, timer, logger, do_slowdown):
        super().__init__()
        self.rank, self.slowdown, self.timer, self.logger = rank, slowdown, timer, logger
        self.do_slowdown = do_slowdown

    def forward(self, data):
        return BackwardSlowdownFunction.apply(data, self.rank, self.slowdown, self.timer,
                                              self.logger, self.do_slowdown)


def _in_fusable(span) -> bool:
    """Can this span consume its input from a fused peer slot?  Yes when it starts a block (Head:
    QKV GEMM gated on the panel flags) or starts at Body (cut after BertLayer_Head: the FFN1 GEMM
    is gated, attn_out doubles as the residual of Tail); not when it starts at Tail (cut after
    Body: two tensors, 5x the bytes - stays on torch.distributed p2p)."""
    return span.head is not None or span.body is not None


def _out_fusable(span) -> bool:
    """Can this span write its output into the next stage's HBM?  When it ends a block (Tail:
    FFN2 GEMM + LayerNorm) or is Head alone (attention-output GEMM + LayerNorm)."""
    return span.tail is not None or (span.head is not None and span.body is None)


class ModuleWrapper(nn.Module):
    def __init__(
        self,
        rank: int,
        module: nn.Module,
        module_to_cuda: bool = False,
        output_to_cpu: bool = False,
        mem_limit: int = -1,
        slowdown: float = 0,
        timer_config: Optional[dict] = None,
        logging_config: Optional[dict] = None,
        cuda_device: int = -1,
        record_forward_time: bool = False,
        fuse_spans: bool = True,
    ):
        super().__init__()
        assert isinstance(module, SequentialWrapper), (
            "The module is of type {}, but expected SequentialWrapper".format(type(module)))
        assert mem_limit != 0 and mem_limit >= -1, (
            "mem_limit can only be -1 (auto-detect) or a positive number of MiB")
        assert not module_to_cuda or cuda_device >= 0, "GPU device index must be non-negative"
        self._rank = rank
        self._module = module
        self._module_to_cuda = module_to_cuda
        self._output_to_cpu = output_to_cpu
        self._mem_limit = mem_limit
        self._slowdown = slowdown
        self._gpu_index = cuda_device
        self._logger = Logger(**logging_config) if logging_config else None
        self._timer = DistributedTimer(**(timer_config or {}))
        self._record_forward_time = record_forward_time
        self._probes_suspended = False  # suspend_forward_probes(): forwards are not timed / logged
        self._fuse_spans = fuse_spans
        self._fwd_events: list = []     # (start_event, end_event) pairs, resolved lazily
        self._bwd_events: list = []
        self._forward_time_resolved: List[float] = []
        self._backward_time_resolved: List[float] = []
        self._bwd_start_evt = None
        self._bwd_t0 = 0.0
        self._tslot = None              # device uint64 slot for the throttle kernels
        self._plan = None               # execution plan with fused spans
        self.in_channel = None          # set by the pipeline engine (fused stage boundary)
        self.out_channel = None
        self.microbatch = 0
        # the micro-batch's labels, bound by the pipeline engine when the last layer consumes
        # them (a sparse masked-language-model head).  A binding holds for ONE forward call,
        # which takes and clears it: a later call without a binding (inference, fill-mask) passes
        # no labels and gets the dense logits
        self.labels = None
        children = list(module.children())
        for i, layer in enumerate(children[:-1]):
            if getattr(layer, "consumes_labels", False):
                raise ValueError("{} (layer {} of {}) consumes labels and must be the model's "
                                 "last layer".format(type(layer).__name__, i, len(children)))
        # the pipeline engine brackets backward itself (begin_backward/end_backward) because the
        # first stage has no differentiable input to hang the autograd probe on
        self.engine_managed_backward = False
        if self._module_to_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("module_to_cuda=True but no CUDA device is available")
            torch.cuda.set_device(cuda_device)
            self.cuda(cuda_device)

    # ------------------------------------------------------------------ properties
    @property
    def rank(self) -> int:
        return self._rank

    @property
    def gpu_index(self) -> int:
        return self._gpu_index

    @property
    def layers(self) -> SequentialWrapper:
        return self._module

    @property
    def consumes_labels(self) -> bool:
        """Does the last layer take the labels (``ModuleWrapper.labels``) as an input?"""
        last = self._module[-1] if len(self._module) else None
        return bool(getattr(last, "consumes_labels", False))

    @property
    def device(self) -> torch.device:
        for p in self._module.parameters():
            return p.device
        return torch.device("cpu")

    @property
    def forward_time(self) -> List[float]:
        """Seconds per recorded forward call (device time incl. simulated slowdown)."""
        self._resolve_events()
        return self._forward_time_resolved

    @property
    def backward_time(self) -> List[float]:
        self._resolve_events()
        return self._backward_time_resolved

    # ------------------------------------------------------------------ span fusion
    def _build_plan(self) -> list:
        from ..models.bert_layers import BertLayer_Body, BertLayer_Head, BertLayer_Tail, BertSpan

        layers = list(self._module.children())
        plan: list = []
        i = 0
        while i < len(layers):
            l = layers[i]
            if self._fuse_spans and isinstance(l, (BertLayer_Head, BertLayer_Body, BertLayer_Tail)):
                head = body = tail = None
                j = i
                if isinstance(layers[j], BertLayer_Head):
                    head = layers[j]
                    j += 1
                if j < len(layers) and isinstance(layers[j], BertLayer_Body) and (head is not None or j == i):
                    body = layers[j]
                    j += 1
                if j < len(layers) and isinstance(layers[j], BertLayer_Tail) and (body is not None or j == i):
                    tail = layers[j]
                    j += 1
                plan.append(BertSpan(head=head, body=body, tail=tail))
                i = j
            else:
                plan.append(l)
                i += 1
        return plan

    def _run_layers(self, args, labels=None):
        from ..models.bert_layers import BertSpan, _native_enabled

        first_tensor = next((a for a in args if torch.is_tensor(a)), None)
        use_native = first_tensor is not None and first_tensor.is_cuda and _native_enabled(first_tensor)
        with_labels = labels is not None and self.consumes_labels
        if not use_native:
            if not with_labels:
                return self._module(*args)
            inputs = self._module[:-1](*args)
            inputs = inputs if isinstance(inputs, (tuple, list)) else (inputs,)
            return self._module[-1](*inputs, labels=labels)
        if self._plan is None:
            self._plan = self._build_plan()
        inputs = args
        n = len(self._plan)
        for idx, step in enumerate(self._plan):
            if not isinstance(inputs, (tuple, list)):
                inputs = (inputs,)
            if isinstance(step, BertSpan):
                hidden = inputs[0] if step.head is not None or step.body is not None else inputs[1]
                if step.supports(hidden):
                    # fusable cuts: in front of a block (span starts with Head) or after
                    # BertLayer_Head (span starts with Body: attn_out arrives in the slot, FFN1 is
                    # the flag-gated consumer); behind a block (span ends with Tail) or after Head
                    # (Head-only span: the K4 GEMM + LayerNorm writes the peer slot)
                    step.in_channel = self.in_channel if (idx == 0 and _in_fusable(step)) else None
                    step.out_channel = self.out_channel if (idx == n - 1 and _out_fusable(step)) else None
                    step.microbatch = self.microbatch
                    inputs = step(*inputs)
                else:
                    for layer in step.layers:
                        inputs = layer(*inputs) if isinstance(inputs, (tuple, list)) else layer(inputs)
            elif with_labels and idx == n - 1:
                inputs = step(*inputs, labels=labels)
            else:
                inputs = step(*inputs)
        return inputs

    def fused_boundary_support(self, shape: Optional[tuple] = None) -> tuple:
        """(input side fusable, output side fusable): whole-block cuts on the native path.

        ``shape`` = the negotiated ``(micro-batch, seq, hidden)``: when given, the boundary spans
        must also ``supports()`` it - a span that would fall back to the eager per-layer path
        (e.g. a non-gelu activation) neither waits on the inbound flags nor writes the peer slot,
        so it must not be negotiated as fused."""
        if self._plan is None:
            self._plan = self._build_plan()
        from ..models.bert_layers import BertSpan

        first, last = self._plan[0], self._plan[-1]
        in_ok = isinstance(first, BertSpan) and _in_fusable(first)
        out_ok = isinstance(last, BertSpan) and _out_fusable(last)
        if shape is not None and shape[0] and shape[1] and shape[2]:
            probe = torch.empty(tuple(shape), device="meta")
            in_ok = in_ok and first.supports(probe)
            out_ok = out_ok and last.supports(probe)
        return in_ok, out_ok

    def spans(self) -> list:
        from ..models.bert_layers import BertSpan

        if self._plan is None:
            self._plan = self._build_plan()
        return [s for s in self._plan if isinstance(s, BertSpan)]

    # ------------------------------------------------------------------ timing / throttle
    def _on_cuda(self) -> bool:
        return self.device.type == "cuda"

    def _throttle_slot(self):
        if self._tslot is None:
            self._tslot = torch.zeros(1, dtype=torch.int64, device=self.device)
        return self._tslot

    def _device_throttle_begin(self):
        from ..ops import native as nat

        nat.ext().record_time(self._throttle_slot().data_ptr(), torch.cuda.current_stream().cuda_stream)

    def _device_throttle_end(self):
        from ..ops import native as nat

        nat.ext().spin_factor(self._throttle_slot().data_ptr(), float(self._slowdown),
                              torch.cuda.current_stream().cuda_stream)

    def _on_backward_start(self):
        if self._on_cuda():
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._bwd_start_evt = ev
            if self._slowdown > 0:
                self._device_throttle_begin()
        else:
            self._bwd_t0 = time.time()
            self._timer.add_timestamp()

    def _on_backward_end(self):
        if self._on_cuda():
            if self._slowdown > 0:
                self._device_throttle_end()
            if self._bwd_start_evt is not None:
                ev = torch.cuda.Event(enable_timing=True)
                ev.record()
                self._bwd_events.append((self._bwd_start_evt, ev))
                self._bwd_start_evt = None
        else:
            elapsed = time.time() - self._bwd_t0
            if self._slowdown > 0:
                time.sleep(max(0.0, elapsed * self._slowdown))
            total = elapsed * (self._slowdown + 1)
            self._backward_time_resolved.append(total)
            if self._logger:
                self._logger.info("backward time on rank {}: {}".format(self._rank, total))
            self._timer.add_timestamp()

    def _resolve_events(self) -> None:
        if not self._fwd_events and not self._bwd_events:
            return
        torch.cuda.synchronize(self.device)
        for s, e in self._fwd_events:
            t = s.elapsed_time(e) * 1e-3
            self._forward_time_resolved.append(t)
            if self._logger:
                self._logger.info("forward time on rank {}: {}".format(self._rank, t))
        for s, e in self._bwd_events:
            t = s.elapsed_time(e) * 1e-3
            self._backward_time_resolved.append(t)
            if self._logger:
                self._logger.info("backward time on rank {}: {}".format(self._rank, t))
        self._fwd_events, self._bwd_events = [], []

    def flush_logs(self) -> None:
        """Resolve pending device timings into the log file (one sync)."""
        self._resolve_events()

    @contextlib.contextmanager
    def suspend_forward_probes(self):
        """Forward calls inside the block (evaluation passes) are neither timed nor logged and
        leave ``forward_time`` as it was; a simulated slowdown still applies."""
        saved = self._probes_suspended
        self._probes_suspended = True
        try:
            yield
        finally:
            self._probes_suspended = saved

    def reset_timers(self) -> None:
        self._resolve_events()
        self._forward_time_resolved, self._backward_time_resolved = [], []

    # ------------------------------------------------------------------ forward
    def _move_in(self, data):
        if self._module_to_cuda and isinstance(data, torch.Tensor) and not data.is_cuda:
            data = data.to("cuda:{}".format(self._gpu_index), non_blocking=True)
        return data

    def _move_out(self, data):
        if self._output_to_cpu and isinstance(data, torch.Tensor):
            data = data.cpu()
        return data

    def begin_backward(self) -> None:
        self._on_backward_start()

    def end_backward(self) -> None:
        self._on_backward_end()

    def _probe(self, t, is_input_side: bool):
        if self.engine_managed_backward:
            return t
        if isinstance(t, torch.Tensor) and t.requires_grad and torch.is_grad_enabled():
            return _BackwardProbe.apply(t, self, is_input_side)
        return t

    def forward(self, *args):
        labels, self.labels = self.labels, None
        args = [self._move_in(a) for a in args]
        need_probe = self._record_forward_time or self._slowdown > 0 or self._logger is not None
        timed = not self._probes_suspended
        cuda = self._on_cuda()
        if need_probe:
            args = [self._probe(a, True) for a in args]
            if cuda:
                if timed:
                    s_evt = torch.cuda.Event(enable_timing=True)
                    s_evt.record()
                if self._slowdown > 0:
                    self._device_throttle_begin()
            else:
                t0 = time.time()
        out = self._run_layers(args, labels)
        if need_probe:
            if cuda:
                if self._slowdown > 0:
                    self._device_throttle_end()
                if timed:
                    e_evt = torch.cuda.Event(enable_timing=True)
                    e_evt.record()
                    self._fwd_events.append((s_evt, e_evt))
                    if len(self._fwd_events) > 4096:
                        self._resolve_events()
            else:
                comp = time.time() - t0
                if self._slowdown > 0:
                    time.sleep(comp * self._slowdown)
                total = time.time() - t0
                if timed:
                    if self._logger:
                        self._logger.info("forward time on rank {}: {}".format(self._rank, total))
                    self._forward_time_resolved.append(total)
        single = not isinstance(out, (tuple, list))
        outs = (out,) if single else tuple(out)
        if need_probe:
            outs = tuple(self._probe(o, False) for o in outs)
        outs = tuple(self._move_out(o) for o in outs)
        return outs

    # ------------------------------------------------------------------ memory probe
    def detect_mem(self, destroy_module: bool = False) -> float:
        """Available device memory in MiB (``mem_limit`` overrides, as in the reference)."""
        if destroy_module:
            self._module = SequentialWrapper()
            self._plan = None
            if self._module_to_cuda or torch.cuda.is_available():
                try:
                    torch.cuda.empty_cache()
                except Exception:
                    pass
        if self._mem_limit > 0:
            return self._mem_limit
        if self._module_to_cuda and torch.cuda.is_available():
            return self._detect_gpu_ram()
        return self._detect_cpu_ram()

    def _detect_gpu_ram(self) -> float:
        try:
            free_b, _total = torch.cuda.mem_get_info(self._gpu_index)
            return free_b / 1024 / 1024 - 500  # keep the reference's 500 MiB safety margin
        except Exception:
            out = subprocess.check_output(
                "nvidia-smi --query-gpu=memory.free --format=csv".split()).decode("ascii")
            vals = [int(x.split()[0]) for x in out.strip().split("\n")[1:]]
            return vals[self._gpu_index] - 500

    def _detect_cpu_ram(self) -> float:
        return psutil.virtual_memory().available / 1024 / 1024
