"""What the pipeline engines share: weight-gradient placement, the device timeline, batch checks.

Both ``PipelineEngine`` (one span per rank, sequential / 1F1B) and ``LoopedPipelineEngine`` (v
chunks per rank on a ring) keep the input-gradient chain of a stage on the critical path and move
everything that only feeds the optimizer (weight / bias / LayerNorm-parameter gradients) off it:

* ``lazy_stream`` (multi-GPU default): backward only queues those gradients; the queue is launched
  on a SIDE STREAM in front of the next backward, i.e. in front of the kernel that will wait for
  the next incoming gradient, so they fill what would otherwise be pipeline bubble and never
  delay the gradient the previous stage waits for;
* ``immediate`` (single-GPU default): every weight gradient is launched at once on a side stream
  forked at the producing kernel;
* ``lazy`` / ``inline``: same queue flushed on the main stream / no deferral (debugging).

The side stream is forked from / joined to the main stream with events, which CUDA-graph capture
records as parallel branches.  Reference context: scaelum/runner/runner.py:137 runs one monolithic
``dist_autograd.backward``; nothing there distinguishes the two kinds of gradient.
"""
from __future__ import annotations

import os
from typing import Optional

import torch


class EngineBase:
    """Mixin state + helpers; concrete engines set ``device``, ``m``, ``is_first``, ``is_last``,
    ``mb_batch`` and call ``_init_common()`` from their constructor."""

    def _init_common(self) -> None:
        self._defer_wgrad = False
        self._wgrad_stream = None
        self._wgrad_forked = False
        self._wgrad_keepalive: list = []
        self._wgrad_tslot: Optional[torch.Tensor] = None
        # inline | lazy | lazy_stream | immediate | auto (see the module docstring)
        self._wgrad_mode = os.environ.get("SKY_WGRAD", "auto")
        self._wgrad_side_stream_enabled = False
        self._wgrad_immediate = False
        # device-side timeline (SKY_TRACE=1 or enable_trace()): one %globaltimer stamp in front of
        # and behind every F / B / W / optimizer phase, written by 1-thread kernels so that the
        # stamps survive CUDA-graph capture
        self._trace = os.environ.get("SKY_TRACE", "0") == "1"
        self._nvtx = os.environ.get("SKY_NVTX", "0") == "1"
        self._trace_buf: Optional[torch.Tensor] = None
        self._trace_tags: list = []
        self._trace_capacity = 0
        self._norm_exchange = None

    # ------------------------------------------------------------------ global gradient norm
    def _norm_info(self) -> tuple:
        """(needs the global gradient norm, can reduce it through peer memory): gathered with the
        other setup flags so that every rank picks the same reduction."""
        from .optim import FusedSGD

        needs = bool(getattr(self.optimizer, "needs_global_norm", False))
        return needs, needs and isinstance(self.optimizer, FusedSGD)

    def _setup_grad_norm(self, position: int, num_positions: int, rank_of_position,
                         infos) -> None:
        """Clipping needs the norm over every stage: a peer-memory exchange when the boundaries
        are fused and every rank runs a fused optimizer (capturable), one all_reduce otherwise.
        Created here, in setup, never during capture.  Collective."""
        needs = {bool(i[0]) for i in infos}
        if len(needs) > 1:
            raise ValueError("gradient clipping must be configured on every pipeline rank or none")
        if num_positions < 2 or not needs.pop():
            return
        if self.fused is not None and all(i[1] for i in infos):
            from .p2p import GradNormExchange

            self._norm_exchange = GradNormExchange(
                position, num_positions, list(rank_of_position), self.device,
                self.fused.epoch_ptr, self.fused.error_ptr, group=self.group)
            self.optimizer.set_norm_reduction(group=self.group, exchange=self._norm_exchange)
        else:
            self.optimizer.set_norm_reduction(group=self.group, allreduce=True)

    def _sends_before_optimizer(self) -> bool:
        """The optimizer's reduction of the norm must not overtake outstanding p2p sends (an NCCL
        all_reduce behind them would dead-lock): engines with such sends wait for them first."""
        return bool(getattr(self.optimizer, "needs_global_norm", False))

    def _close_grad_norm(self) -> None:
        if self._norm_exchange is not None:
            self._norm_exchange.close()
            self._norm_exchange = None
            self.optimizer.set_norm_reduction()

    # ------------------------------------------------------------------ backend
    def _native_active(self) -> bool:
        from ..models.bert_layers import get_backend
        from ..ops import native as nat

        return self.device.type == "cuda" and get_backend() != "torch" and nat.available()

    # ------------------------------------------------------------------ weight gradients
    def _configure_wgrad(self, multi: bool) -> None:
        if not self._native_active():
            return
        from ..ops.functions import set_wgrad_deferral, set_wgrad_stream

        mode = self._wgrad_mode
        if mode == "auto":
            mode = "lazy_stream" if multi else "immediate"  # not measured on H100
        if mode in ("lazy", "lazy_stream") and multi:
            self._defer_wgrad = True
            self._wgrad_side_stream_enabled = mode == "lazy_stream"
            set_wgrad_deferral(True)
        elif mode in ("immediate", "lazy_stream"):
            self._wgrad_stream = torch.cuda.Stream(device=self.device)
            self._wgrad_immediate = True
            set_wgrad_stream(self._wgrad_stream)

    def _slowdown_factor(self) -> float:
        return 0.0

    def _flush_wgrads(self) -> None:
        if not self._defer_wgrad:
            return
        from ..ops.functions import flush_wgrads, pending_wgrads

        if pending_wgrads() == 0:
            return
        if not self._wgrad_side_stream_enabled:
            self._mark(("W", -1, "begin"))
            flush_wgrads()
            self._mark(("W", -1, "end"))
            return
        if self._wgrad_stream is None:
            self._wgrad_stream = torch.cuda.Stream(device=self.device)
        main = torch.cuda.current_stream(self.device)
        self._wgrad_stream.wait_stream(main)
        slow = self._slowdown_factor()
        with torch.cuda.stream(self._wgrad_stream):
            self._mark(("W", -1, "begin"))
            if slow > 0:
                # a simulated slow device is slow for its weight gradients too (own time slot: the
                # stage's forward/backward throttle may be running on the main stream right now)
                from ..ops import native as nat

                if self._wgrad_tslot is None:
                    self._wgrad_tslot = torch.zeros(1, dtype=torch.int64, device=self.device)
                side = self._wgrad_stream.cuda_stream
                nat.ext().record_time(self._wgrad_tslot.data_ptr(), side)
            self._wgrad_keepalive.extend(flush_wgrads())
            if slow > 0:
                nat.ext().spin_factor(self._wgrad_tslot.data_ptr(), slow, side)
            self._mark(("W", -1, "end"))
        self._wgrad_forked = True

    def _join_wgrads(self) -> None:
        if self._wgrad_immediate:
            from ..ops.functions import wgrad_keepalive

            torch.cuda.current_stream(self.device).wait_stream(self._wgrad_stream)
            wgrad_keepalive().clear()
            return
        if self._wgrad_forked:
            torch.cuda.current_stream(self.device).wait_stream(self._wgrad_stream)
            self._wgrad_forked = False
        self._wgrad_keepalive.clear()

    def _release_wgrad_switches(self) -> None:
        """The deferral / side stream are process-wide switches of ops.functions: hand them back
        so that code running without an engine afterwards gets inline gradients again."""
        if self._defer_wgrad or self._wgrad_immediate:
            from ..ops.functions import set_wgrad_deferral, set_wgrad_stream

            if self._defer_wgrad:
                set_wgrad_deferral(False)
            set_wgrad_stream(None)
            self._defer_wgrad = self._wgrad_immediate = False

    # ------------------------------------------------------------------ device timeline
    def enable_trace(self) -> None:
        assert getattr(self, "_graph", None) is None, "enable_trace() must precede CUDA-graph capture"
        self._trace = True

    def _trace_slots(self) -> int:
        return 8 * (2 * self.m + 4) + 64

    def _mark(self, tag) -> None:
        if self._nvtx and self.device.type == "cuda":
            # NVTX ranges for nsys / ncu --nvtx (host-side: they bracket the LAUNCHES of a phase)
            if tag[2] == "begin":
                torch.cuda.nvtx.range_push(f"{tag[0]}{tag[1]}")
            else:
                torch.cuda.nvtx.range_pop()
        if not self._trace or self.device.type != "cuda":
            return
        from ..ops import native as nat

        if self._trace_buf is None:
            self._trace_buf = torch.zeros(self._trace_slots(), dtype=torch.int64, device=self.device)
        i = len(self._trace_tags)
        if i >= self._trace_buf.numel():
            return
        self._trace_tags.append(tag)
        nat.ext().record_time(self._trace_buf.data_ptr() + 8 * i,
                              torch.cuda.current_stream(self.device).cuda_stream)

    def trace(self) -> list:
        """[(tag, ns)] of the LAST executed step: tags are ('F'|'B'|'W'|'OPT', j, 'begin'|'end')."""
        if self._trace_buf is None:
            return []
        torch.cuda.synchronize(self.device)
        t = self._trace_buf.cpu().tolist()
        return [(tag, t[i]) for i, tag in enumerate(self._trace_tags)]

    # ------------------------------------------------------------------ batch shape
    def _check_batch(self, inputs, labels) -> None:
        """The micro-batch shape is fixed by the first step (static graph buffers, peer slots,
        cached p2p metas): a batch of another size must fail HERE, with a message, and not as a
        shape error inside ``copy_`` or as a neighbour stage hanging in a full-size receive."""
        want = self.mb_batch * self.m
        if not want:
            return
        for what, t in (("inputs", inputs[0] if (self.is_first and inputs) else None),
                        ("labels", labels if self.is_last else None)):
            if torch.is_tensor(t) and t.dim() > 0 and t.shape[0] != want:
                raise ValueError(
                    "{} have batch size {}, but this pipeline was set up for {} = {} micro-batches "
                    "x {} samples on its first step; drop short batches (drop_last=True) or build "
                    "a new engine".format(what, t.shape[0], want, self.m, self.mb_batch))
