"""What the pipeline engines share.

``PipelineEngine`` (one span per rank, sequential / 1F1B) and ``LoopedPipelineEngine`` (v chunks
per rank on a ring) differ in their micro-batch orders and transports.  The base owns the rest:
construction and ``close()``; ``train_step`` with the whole-step CUDA graph (``_run_graphed``,
which the single-GPU evaluation graph uses too); the step's preamble, last-stage loss, backward
and optimizer step; the fused-boundary input and the torch.distributed p2p helpers; ``eval_step``;
the global gradient norm; the device timeline; batch checks; and the placement of weight
gradients.

Both engines keep the input-gradient chain of a stage on the critical path and move everything
that only feeds the optimizer (weight / bias / LayerNorm-parameter gradients) off it:

* ``lazy_stream`` (multi-GPU default): backward only queues those gradients; the queue is launched
  on a SIDE STREAM in front of the next backward, i.e. in front of the kernel that will wait for
  the next incoming gradient, so they fill what would otherwise be pipeline bubble and never
  delay the gradient the previous stage waits for;
* ``immediate`` (single-GPU default): every weight gradient is launched at once on a side stream
  forked at the producing kernel;
* ``lazy`` / ``inline``: same queue flushed on the main stream / no deferral (debugging).

When the optimizer's step is plain SGD (``FusedSGD`` without momentum, schedule or clipping), the
encoder weight banks are not updated by the optimizer's pass at the end of the step: the wgrad
GEMM that produces a bank's last gradient of the step applies the update in its epilogue (the
backward of the last micro-batch of each local stage is "armed", ``_arm_wgrad_sgd``), and the
optimizer's one launch covers the remaining banks.

The side stream is forked from / joined to the main stream with events, which CUDA-graph capture
records as parallel branches.  Reference context: scaelum/runner/runner.py:137 runs one monolithic
``dist_autograd.backward``; nothing there distinguishes the two kinds of gradient.
"""
from __future__ import annotations

import contextlib
import os
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist


def graph_state(warmup: int, key=None) -> dict:
    """Static buffers and CUDA graph of one captured body (see ``EngineBase._run_graphed``):
    ``warmup`` eager calls before the capture, ``key`` what the graph was captured for, and the
    native kernel launches the capture recorded."""
    return dict(warmup=warmup, key=key, inputs=None, labels=None, graph=None, eager=0, launches=0)


class EngineBase:
    """State + helpers of both engines.  A concrete engine sets ``is_first``, ``is_last``, ``P``
    and ``schedule``, calls ``EngineBase.__init__`` from its constructor and provides ``_setup``,
    ``_step_body`` and ``forward_only``."""

    def __init__(self, stages: Sequence, device: torch.device, optimizer, loss_fn,
                 micro_batches: int, boundary: str, use_cuda_graph: bool, group,
                 advance_rng: bool) -> None:
        self.stages = list(stages)
        for st in self.stages:
            st.engine_managed_backward = True
        self.device = device
        self.optimizer = optimizer
        self.loss_fn = loss_fn
        self.m = micro_batches
        self.boundary = boundary
        self.group = group
        self._advance_rng = advance_rng
        self._want_graph = use_cuda_graph and device.type == "cuda"
        self.graphable = False
        self._setup_done = False
        self.mb_batch = self.seq = 0
        self.fused = None
        self.in_fused = self.out_fused = False
        self._loss_acc: Optional[torch.Tensor] = None
        self._pending_sends: list = []
        self._step = graph_state(warmup=3)     # the whole training step
        self._eval: Optional[dict] = None      # the evaluation graph (PipelineEngine, 1 GPU)
        self._defer_wgrad = False
        self._wgrad_stream = None
        self._wgrad_forked = False
        self._wgrad_keepalive: list = []
        self._wgrad_tslot: Optional[torch.Tensor] = None
        # plain-SGD update in the weight-gradient GEMMs (_setup_wgrad_sgd): (lr, weight_decay,
        # grad_scale), and the banks of every local stage it applies to
        self._wgrad_sgd: Optional[tuple] = None
        self._wgrad_sgd_banks: List[list] = [[] for _ in self.stages]
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

    # the captured training step (None until it is captured), the native kernel launches of one
    # replay, and its static input / label buffers
    @property
    def _graph(self) -> Optional[torch.cuda.CUDAGraph]:
        return self._step["graph"]

    @property
    def launches_per_step(self) -> int:
        return self._step["launches"]

    @property
    def _static_inputs(self) -> Optional[list]:
        return self._step["inputs"]

    @property
    def _static_labels(self) -> Optional[torch.Tensor]:
        return self._step["labels"]

    def close(self) -> None:
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)  # nothing of ours may still touch a peer region
        self._eval = None   # the evaluation graph is rebuilt by the next engine
        self._close_grad_norm()
        if self.fused is not None:
            self.fused.close()
            self.fused = None
        self._release_wgrad_switches()
        if self._wgrad_sgd is not None:
            self.optimizer.set_update_in_wgrad([])   # step() updates every bank again
            self._wgrad_sgd = None

    # ------------------------------------------------------------------ setup
    def _setup_batch_shape(self, inputs, src: Optional[int]) -> None:
        """``mb_batch`` and ``seq`` of the first stage's micro-batches, broadcast from rank ``src``
        (None: a single rank).  Collective."""
        shape = [0, 0]
        if self.is_first and inputs is not None:
            x = inputs[0]
            shape = [x.shape[0] // self.m, int(x.shape[1]) if x.dim() > 1 else 0]
        if src is not None:
            box = [shape]
            dist.broadcast_object_list(box, src=src, group=self.group)
            shape = box[0]
        self.mb_batch, self.seq = shape

    def _setup_graphable(self, capturable: bool) -> None:
        """``capturable``: the step runs native kernels only and every link of this rank is fused
        (or absent), i.e. nothing but the optimizer can keep the step out of a CUDA graph."""
        # only an optimizer whose step() is pure device work may be captured (a torch.optim class
        # behind TorchOptimizerAdapter keeps host-side state and refreshes the bf16 shadows through
        # a host-side version check: replaying it would train on stale weights)
        self.graphable = self._want_graph and capturable and \
            bool(getattr(self.optimizer, "graph_safe", False))
        if self.graphable:
            # device timers cannot be recorded inside a captured graph
            for st in self.stages:
                st._record_forward_time = False
                st._logger = None

    # ------------------------------------------------------------------ one optimisation step
    def train_step(self, inputs: Optional[Sequence[torch.Tensor]] = None,
                   labels: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """Run one optimisation step; returns the (mean) loss tensor on the last stage."""
        if not self._setup_done:
            self._setup(inputs)
            self._loss_acc = torch.zeros((), dtype=torch.float32, device=self.device)
        self._check_batch(inputs, labels)
        if self.graphable:
            self._run_graphed(self._step, self._step_body,
                              inputs if self.is_first else None, labels if self.is_last else None)
        else:
            self._step_body(inputs, labels)
        return self._loss_acc if self.is_last else None

    def _run_graphed(self, state: dict, body, inputs, labels) -> None:
        """``body(inputs, labels)`` through the CUDA graph of ``state`` (``graph_state``): the
        arguments are copied into static buffers, the first ``warmup`` calls run eagerly on them
        (allocations, lazily created attributes), the next one captures and, since capture only
        records, replays right away so that its batch is processed; every later call replays."""
        if state["inputs"] is None:
            state["inputs"] = [t.clone() for t in inputs] if inputs is not None else []
            state["labels"] = labels.clone() if labels is not None else None
        for s, t in zip(state["inputs"], inputs or ()):
            s.copy_(t, non_blocking=True)
        if state["labels"] is not None and labels is not None:
            state["labels"].copy_(labels, non_blocking=True)
        if state["graph"] is None and state["eager"] < state["warmup"]:
            body(state["inputs"], state["labels"])
            state["eager"] += 1
            return
        if state["graph"] is None:
            from ..ops import native as nat

            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            before = nat.launch_count()
            with torch.cuda.graph(g):
                body(state["inputs"], state["labels"])
            state["launches"] = nat.launch_count() - before
            state["graph"] = g
        state["graph"].replay()

    def _begin_step(self, inputs, labels):
        """Start of a step body: boundary epoch, dropout RNG, loss accumulator, timeline; returns
        the per-micro-batch input chunks (first stage) and label chunks (last stage)."""
        from ..models.bert_layers import advance_rng

        if self.fused is not None:
            self.fused.begin_step()
        if self._advance_rng and self._native_active():
            advance_rng()
        self._loss_acc.zero_()
        self._trace_tags = []
        self._mark(("STEP", 0, "begin"))
        chunks = [t.chunk(self.m, dim=0) for t in inputs] if self.is_first else None
        label_chunks = labels.chunk(self.m, dim=0) if (self.is_last and labels is not None) else None
        return chunks, label_chunks

    # ------------------------------------------------------------------ labels of the last layer
    @staticmethod
    def _bind_labels(st, label_chunks, j: int) -> None:
        """Before stage ``st`` runs micro-batch ``j``: its labels when the stage's last layer
        consumes them (a sparse masked-language-model head), none otherwise.  Inside a captured
        step the chunks are views of the static label buffer."""
        consumes = getattr(st, "consumes_labels", False)
        st.labels = label_chunks[j] if (label_chunks is not None and consumes) else None

    @staticmethod
    def _head_outputs(st, outs, labels):
        """(logits, labels) that the loss / the evaluation accumulator read from the last stage's
        outputs: a label-consuming last layer returns its own labels, one per decoded row, as
        ``outs[1]`` (viewed as [sequences, rows per sequence]); backward still starts at
        ``outs[0]``."""
        if getattr(st, "consumes_labels", False):
            return outs[0], outs[1].view(labels.shape[0], -1)
        return outs[0], labels

    def _last_stage_loss(self, st, outs, labels):
        """The loss of one micro-batch on the last stage, added into ``_loss_acc``."""
        logits, labels = self._head_outputs(st, outs, labels)
        if hasattr(self.loss_fn, "fused") and logits.is_cuda and self._loss_acc.dtype == torch.float32:
            # (dlogits,) instead of a scalar loss: see _NativeCrossEntropy.fused
            return (self.loss_fn.fused(logits, labels, 1.0 / self.m, self._loss_acc.view(1)),)
        loss = self.loss_fn(logits, labels) / self.m
        self._loss_acc += loss.detach().float()
        return loss

    @staticmethod
    def _backward_from_loss(outs, loss) -> None:
        if isinstance(loss, tuple):
            torch.autograd.backward([outs[0]], [loss[0].to(outs[0].dtype)])
        else:
            loss.backward()

    @staticmethod
    def _backward_from_grads(outs, grads) -> None:
        """Backward from the received gradients of the outputs that require grad."""
        ts, gs = [], []
        for o, g in zip(outs, grads):
            if g is not None and torch.is_tensor(o) and o.requires_grad:
                ts.append(o)
                gs.append(g.to(o.dtype))
        torch.autograd.backward(ts, gs)

    def _optimizer_step(self, pending: list) -> None:
        """The optimizer step at the end of a step; ``pending`` (outstanding p2p sends) is waited
        for and emptied."""
        self._mark(("OPT", 0, "begin"))
        if pending and self._sends_before_optimizer():
            self.comm.wait(pending)
            pending.clear()
        self.optimizer.step()
        self._mark(("OPT", 0, "end"))
        if pending:
            self.comm.wait(pending)
            pending.clear()

    # ------------------------------------------------------------------ boundaries
    def _fused_inputs(self, slot: int):
        """(activation, additive mask) of inbound fused-boundary slot ``slot``."""
        from ..ops import native as nat

        ch = self.fused.prev
        rows = self.mb_batch * self.seq
        # the additive mask rides next to the activation slot under its own flag
        nat.ext().wait_flags(ch.local.mask_flag_ptr(slot), 1, ch.epoch_ptr, 1, ch.error_ptr,
                             torch.cuda.current_stream().cuda_stream)
        x = ch.act_view(slot, rows, ch.cols).view(self.mb_batch, self.seq, ch.cols)
        x.requires_grad_(True)
        mask = ch.mask_view(slot, rows).view(self.mb_batch, 1, 1, self.seq)
        return (x, mask)

    @staticmethod
    def _diff_flags(tensors) -> List[bool]:
        """Which boundary tensors carry gradients: floating tensors, except a trailing additive
        mask when several tensors cross the boundary.  Both sides of a link apply this rule, so
        gradient messages need no metadata handshake."""
        n = len(tensors)
        return [torch.is_tensor(t) and t.is_floating_point() and (i < n - 1 or n == 1)
                for i, t in enumerate(tensors)]

    def _prep_inputs(self, tensors):
        for t, d in zip(tensors, self._diff_flags(tensors)):
            if d:
                t.requires_grad_(True)
        return tuple(tensors)

    def _grad_metas(self, outs):
        return [(o.dtype, tuple(o.shape)) if d else None
                for o, d in zip(outs, self._diff_flags(outs))]

    def _in_grads(self, args):
        out = []
        for a, d in zip(args, self._diff_flags(args)):
            if not d:
                out.append(None)
            else:
                out.append(a.grad if a.grad is not None else torch.zeros_like(a))
        return out

    # ------------------------------------------------------------------ evaluation
    def eval_step(self, inputs: Optional[Sequence[torch.Tensor]], labels: Optional[torch.Tensor],
                  accum, micro_batches: Optional[int] = None) -> None:
        """One evaluation batch: ``forward_only`` and, on the last stage, ``accum.add(logits,
        labels)`` per micro-batch, with the forward-time probes of every local stage suspended."""
        m = int(micro_batches or self.m)
        if self.is_first and inputs[0].shape[0] % m:
            raise ValueError("an evaluation batch of {} samples cannot be split into {} equal "
                             "micro-batches".format(inputs[0].shape[0], m))
        with contextlib.ExitStack() as stack:
            for st in self.stages:
                stack.enter_context(st.suspend_forward_probes())
            self._eval_pass(inputs, labels, accum, m)

    def _eval_pass(self, inputs, labels, accum, m: int) -> None:
        """The evaluation batch of ``eval_step``; PipelineEngine may replay it from a graph."""
        self._eval_body(inputs, labels, accum, m)

    def _eval_body(self, inputs, labels, accum, m: int) -> None:
        res = self.forward_only(inputs, micro_batches=m, labels=labels if self.is_last else None)
        if self.is_last:
            res = [res] if m == 1 else res
            for outs, lab in zip(res, labels.chunk(m, dim=0)):
                accum.add(*self._head_outputs(self.stages[-1], outs, lab))

    # ------------------------------------------------------------------ global gradient norm
    def _norm_info(self) -> tuple:
        """(needs the global gradient norm, can reduce it through peer memory): gathered with the
        other setup flags so that every rank picks the same reduction."""
        from .optim import FusedOptimizer

        needs = bool(getattr(self.optimizer, "needs_global_norm", False))
        return needs, needs and isinstance(self.optimizer, FusedOptimizer)

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
        self._setup_wgrad_sgd()

    def _setup_wgrad_sgd(self) -> None:
        """Let the wgrad GEMMs of the encoder weight banks apply the optimizer's update when it is
        plain SGD (``wgrad_sgd_args``): a bank then moves 10 B per parameter in that epilogue
        (read and write the master, write the shadow) instead of 4 B there (the gradient) and
        14 B in the optimizer's serial pass.  Other optimizers keep their step unchanged."""
        args_of = getattr(self.optimizer, "wgrad_sgd_args", None)
        args = args_of() if args_of is not None else None
        if args is None:
            return
        from ..models.bert_layers import native_param_banks

        owned = {id(b) for b in self.optimizer.banks}
        per_stage = [[b for b in native_param_banks(st)
                      if getattr(b, "update_in_wgrad_ok", False) and id(b) in owned]
                     for st in self.stages]
        if not any(per_stage):
            return
        self.optimizer.set_update_in_wgrad([b for banks in per_stage for b in banks])
        self._wgrad_sgd = args
        self._wgrad_sgd_banks = per_stage

    @contextlib.contextmanager
    def _arm_wgrad_sgd(self, stage_index: int, j: int):
        """Around the backward of micro-batch ``j`` on local stage ``stage_index``: the last
        micro-batch's backward produces the step's last gradient of every bank of the stage (no
        forward of the stage follows it in the step), so its wgrad GEMMs apply the update; the
        earlier ones accumulate as usual."""
        banks = self._wgrad_sgd_banks[stage_index] if j == self.m - 1 else []
        for b in banks:
            b.wgrad_sgd = self._wgrad_sgd
        try:
            yield
        finally:
            for b in banks:
                b.wgrad_sgd = None

    def _slowdown_factor(self) -> float:
        return max(float(getattr(st, "_slowdown", 0) or 0) for st in self.stages)

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
        return 8 * (2 * len(self.stages) * self.m + 4) + 64

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
