"""SPMD pipeline engine: one process per GPU, each owning one contiguous layer span.

What the reference does with RPC (scaelum/model/rpc_model.py:44-55, runner.py:127-139: the master
issues one remote forward per stage, stages pull activations through CPU, distributed autograd
walks back, a DistributedOptimizer steps every owner) happens here inside every rank:

    for each micro-batch (sequential or 1F1B order):
        obtain the stage input  (own data | fused peer slot | NCCL/gloo recv)
        run the stage           (ModuleWrapper -> fused sm_90a spans)
        hand the output on      (LayerNorm wrote it into the next GPU already | send)
        ... backward symmetric  (dgrad GEMM writes into the previous GPU | send)
    optimizer step              (FusedSGD: one launch)

Boundaries are FUSED (parallel/p2p.py) when the cut sits between two whole transformer blocks on
the native path, and fall back to torch.distributed p2p (nccl / gloo) otherwise.  When every link
of a rank is fused (or absent) the whole step - all micro-batches, backward, optimizer, RNG/epoch
counters - is captured into ONE CUDA graph and replayed; cross-GPU synchronisation then happens
exclusively through in-kernel flag waits.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch
import torch.distributed as dist

from ..builder.module_wrapper import ModuleWrapper
from .engine_base import EngineBase, graph_state


def one_f_one_b_order(stage: int, num_stages: int, micro_batches: int) -> List[tuple]:
    """[('F', j) | ('B', j)] for this stage (non-interleaved 1F1B)."""
    warm = min(num_stages - stage - 1, micro_batches)
    order: List[tuple] = [("F", j) for j in range(warm)]
    f, b = warm, 0
    for _ in range(micro_batches - warm):
        order.append(("F", f))
        f += 1
        order.append(("B", b))
        b += 1
    while b < micro_batches:
        order.append(("B", b))
        b += 1
    return order


def sequential_order(stage: int, num_stages: int, micro_batches: int) -> List[tuple]:
    """One micro-batch in flight at a time (reference semantics when micro_batches == 1)."""
    order: List[tuple] = []
    for j in range(micro_batches):
        order += [("F", j), ("B", j)]
    return order


class PipelineEngine(EngineBase):
    def __init__(self, stage: ModuleWrapper, stage_index: int, num_stages: int,
                 stage_to_rank: Sequence[int], device: torch.device, optimizer,
                 loss_fn: Optional[Callable] = None, micro_batches: int = 1,
                 schedule: str = "1f1b", boundary: str = "auto", use_cuda_graph: bool = True,
                 group=None, advance_rng: bool = True):
        assert schedule in ("1f1b", "sequential"), schedule
        assert boundary in ("auto", "fused", "nccl", "gloo", "dist"), boundary
        super().__init__([stage], device, optimizer, loss_fn, micro_batches, boundary,
                         use_cuda_graph, group, advance_rng)
        self.stage = stage
        self.s, self.P = stage_index, num_stages
        self.stage_to_rank = list(stage_to_rank)
        self.schedule = schedule
        self.is_first, self.is_last = stage_index == 0, stage_index == num_stages - 1
        self.prev_rank = None if self.is_first else self.stage_to_rank[stage_index - 1]
        self.next_rank = None if self.is_last else self.stage_to_rank[stage_index + 1]
        self.comm = None
        self._eval_comm_obj = None      # forward-only transport when training needs none

    # ------------------------------------------------------------------ setup
    def _setup(self, inputs: Optional[Sequence[torch.Tensor]]) -> None:
        multi = self.P > 1
        self._setup_batch_shape(inputs, self.stage_to_rank[0] if multi else None)
        want_fused = self.boundary in ("auto", "fused") and self._native_active() and multi
        in_ok = out_ok = False
        hidden = 0
        if want_fused:
            spans = self.stage.spans()
            if spans:
                hidden = self._hidden_size(spans[0])
            in_ok, out_ok = self.stage.fused_boundary_support((self.mb_batch, self.seq, hidden))
            shape_ok = self.seq % 8 == 0 and hidden % 64 == 0 and (self.mb_batch * self.seq) % 128 == 0
            if spans and spans[0].head is not None:
                shape_ok = shape_ok and spans[0].head.attention.self.attention_head_size == 64
            in_ok, out_ok = in_ok and shape_ok, out_ok and shape_ok
        if multi:
            flags: List[tuple] = [None] * dist.get_world_size(self.group)  # type: ignore[list-item]
            dist.all_gather_object(flags, (self.s, in_ok, out_ok, hidden, self._norm_info()),
                                   group=self.group)
            by_stage = {f[0]: f for f in flags}
            if not self.is_first:
                self.in_fused = want_fused and by_stage[self.s - 1][2] and in_ok
            if not self.is_last:
                self.out_fused = want_fused and by_stage[self.s + 1][1] and out_ok
            any_fused = any(
                by_stage[k][2] and by_stage[k + 1][1] for k in range(self.P - 1)) and want_fused
            if any_fused:
                # collective: every rank participates in the handle exchange
                from .p2p import FusedBoundaryManager

                hid = max(f[3] for f in flags)
                self.fused = FusedBoundaryManager(
                    self.s, self.P, self.stage_to_rank, self.m, self.mb_batch * self.seq, hid,
                    self.mb_batch * self.seq, self.device, group=self.group)
            if (not self.is_first and not self.in_fused) or (not self.is_last and not self.out_fused):
                from .comm import TorchDistComm

                self.comm = TorchDistComm(self.device, group=self.group)
            self._setup_grad_norm(self.s, self.P, self.stage_to_rank, [f[4] for f in flags])
            self._setup_tie(self.stage_to_rank[0], self.stage_to_rank[-1])
        self._setup_graphable(self._native_active() and (self.is_first or self.in_fused) and
                              (self.is_last or self.out_fused))
        self._configure_wgrad(multi)
        self._order = (one_f_one_b_order if self.schedule == "1f1b" else sequential_order)(
            self.s, self.P, self.m)
        self._setup_done = True

    @staticmethod
    def _hidden_size(span) -> int:
        if span.head is not None:
            return span.head.attention.output.dense.weight.shape[0]
        if span.body is not None:
            return span.body.intermediate.dense_act.weight.shape[1]
        return span.tail.output.dense.weight.shape[0]

    # ------------------------------------------------------------------ per micro-batch work
    def _stage_inputs(self, j: int, chunks):
        if self.is_first:
            return tuple(c[j] for c in chunks)
        if self.in_fused:
            return self._fused_inputs(j)
        return None  # filled by the comm path

    def _forward(self, j: int, args, labels_chunks):
        st = self.stage
        st.microbatch = j
        self._bind_labels(st, labels_chunks, j)
        st.in_channel = self.fused.prev if self.in_fused else None
        st.out_channel = self.fused.next if self.out_fused else None
        if self.out_fused and not self.is_first:
            # the mask travels with the activation (own flag); relay it as early as possible
            self.fused.next.send_mask(args[-1], j)
        self._mark(("F", j, "begin"))
        outs = st(*args)
        self._mark(("F", j, "end"))
        if self.out_fused and self.is_first:
            self.fused.next.send_mask(outs[-1], j)  # produced by the embeddings of this stage
        loss = self._last_stage_loss(st, outs, labels_chunks[j]) if self.is_last else None
        return outs, loss

    def _backward(self, j: int, outs, loss, grads, args):
        st = self.stage
        st.microbatch = j
        st.in_channel = self.fused.prev if self.in_fused else None
        st.out_channel = self.fused.next if self.out_fused else None
        # Weight gradients of the PREVIOUS micro-batch run now, i.e. in front of the kernel that
        # will wait for this micro-batch's incoming gradient: during the 1F1B cool-down they fill
        # what would otherwise be pipeline bubble, and they never delay the input gradient that
        # the previous stage is waiting for.
        self._flush_wgrads()
        self._mark(("B", j, "begin"))
        st.begin_backward()
        with self._arm_wgrad_sgd(0, j):
            if self.is_last:
                self._backward_from_loss(st, outs, loss)
            elif self.out_fused:
                dummy = outs[0]
                torch.autograd.backward([dummy], [torch.zeros_like(dummy)])
            else:
                self._backward_from_grads(outs, grads)
        st.end_backward()
        self._mark(("B", j, "end"))
        if self.is_first or self.in_fused:
            return None
        return self._in_grads(args)

    # ------------------------------------------------------------------ comm helpers (unfused)
    def _recv_forward(self):
        outs, reqs = self.comm.recv(self.prev_rank, "fwd")
        self.comm.wait(reqs)
        return self._prep_inputs(outs)

    def _send_forward(self, outs):
        self._pending_sends += self.comm.send([o.detach() if torch.is_tensor(o) else None
                                               for o in outs], self.next_rank, "fwd")

    def _recv_backward(self, outs):
        grads, reqs = self.comm.recv(self.next_rank, "bwd", metas=self._grad_metas(outs))
        self.comm.wait(reqs)
        return grads

    def _send_backward(self, in_grads):
        self._pending_sends += self.comm.send(in_grads, self.prev_rank, "bwd", with_meta=False)

    def _send_forward_recv_backward(self, outs):
        g, reqs = self.comm.exchange([o.detach() if torch.is_tensor(o) else None for o in outs],
                                     self.next_rank, "fwd", self.next_rank, "bwd",
                                     recv_metas=self._grad_metas(outs), send_with_meta=True)
        self.comm.wait(reqs)
        return g

    def _send_backward_recv_forward(self, in_grads):
        metas = self.comm.cached_meta(self.prev_rank, "fwd")
        x, reqs = self.comm.exchange(in_grads, self.prev_rank, "bwd", self.prev_rank, "fwd",
                                     recv_metas=metas)
        self.comm.wait(reqs)
        return self._prep_inputs(x)

    # ------------------------------------------------------------------ one optimisation step
    def _step_body(self, inputs, labels):
        chunks, label_chunks = self._begin_step(inputs, labels)
        need_recv_f = not self.is_first and not self.in_fused
        need_send_f = not self.is_last and not self.out_fused
        need_recv_b = need_send_f
        need_send_b = need_recv_f
        saved = {}
        order = self._order
        pending_in = None       # input received together with a backward send
        pending_grad = None     # gradient received together with a forward send
        for idx, (kind, j) in enumerate(order):
            nxt = order[idx + 1] if idx + 1 < len(order) else None
            if kind == "F":
                if need_recv_f:
                    args = pending_in if pending_in is not None else self._recv_forward()
                    pending_in = None
                else:
                    args = self._stage_inputs(j, chunks)
                outs, loss = self._forward(j, args, label_chunks)
                saved[j] = (args, outs, loss)
                if need_send_f:
                    if nxt is not None and nxt[0] == "B":
                        pending_grad = self._send_forward_recv_backward(outs)
                    else:
                        self._send_forward(outs)
            else:
                args, outs, loss = saved.pop(j)
                grads = None
                if need_recv_b:
                    grads = pending_grad if pending_grad is not None else self._recv_backward(outs)
                    pending_grad = None
                in_grads = self._backward(j, outs, loss, grads, args)
                if need_send_b:
                    if nxt is not None and nxt[0] == "F":
                        pending_in = self._send_backward_recv_forward(in_grads)
                    else:
                        self._send_backward(in_grads)
        self._flush_wgrads()
        self._join_wgrads()
        if self.fused is not None:
            self.fused.end_of_backward()
        self._optimizer_step(self._pending_sends)

    # ------------------------------------------------------------------ forward only (eval)
    def _eval_comm(self):
        """The p2p transport of forward-only passes: the training one when this rank has it,
        otherwise one of its own (fused boundaries carry training steps only)."""
        if self.comm is not None:
            return self.comm
        if self._eval_comm_obj is None:
            from .comm import TorchDistComm

            self._eval_comm_obj = TorchDistComm(self.device, group=self.group)
        return self._eval_comm_obj

    @torch.no_grad()
    def forward_only(self, inputs: Optional[Sequence[torch.Tensor]] = None, micro_batches: int = 1,
                     labels: Optional[torch.Tensor] = None):
        """Forward through the pipeline without gradients.  The batch is split into
        ``micro_batches`` chunks; sends are asynchronous and waited for at the end of the pass, so
        stage s runs chunk j + 1 while stage s + 1 runs chunk j.  ``labels`` (last stage) reach a
        label-consuming last layer.  Returns on the last stage the stage outputs
        (``micro_batches == 1``) or the list of per-chunk outputs, None elsewhere."""
        m = int(micro_batches)
        st = self.stage
        st.in_channel = st.out_channel = None
        chunks = [t.chunk(m, dim=0) for t in inputs] if self.is_first else None
        label_chunks = labels.chunk(m, dim=0) if (self.is_last and labels is not None) else None
        if self.P == 1:
            results = []
            for j in range(m):
                self._bind_labels(st, label_chunks, j)
                results.append(st(*(c[j] for c in chunks)))
            return results[0] if m == 1 else results
        comm = self._eval_comm()
        comm.forget("eval")   # every pass announces its own shapes
        results, pending, keep = [], [], []
        for j in range(m):
            st.microbatch = j
            self._bind_labels(st, label_chunks, j)
            if self.is_first:
                args = tuple(c[j] for c in chunks)
            else:
                args, reqs = comm.recv(self.prev_rank, "eval")
                comm.wait(reqs)
            outs = st(*args)
            if self.is_last:
                results.append(outs)
            else:
                keep.append(outs)
                pending += comm.send(list(outs), self.next_rank, "eval")
        comm.wait(pending)
        if not self.is_last:
            return None
        return results[0] if m == 1 else results

    def _eval_pass(self, inputs, labels, accum, m: int) -> None:
        """On one GPU with the native kernels and ``use_cuda_graph`` the whole batch (forward +
        accumulation) is captured into its own CUDA graph after one eager pass and replayed; it
        touches neither the dropout RNG, the boundary epochs, the training loss nor the optimizer.
        One evaluation graph per engine: a batch of other shapes, another ``m`` or another
        accumulator replaces it."""
        # the graph reads the bf16 weight copies in place: only an optimizer that refreshes them
        # on the device (graph_safe) keeps a captured evaluation current
        if not (self.P == 1 and self._want_graph and self._native_active() and
                bool(getattr(self.optimizer, "graph_safe", False))):
            self._eval_body(inputs, labels, accum, m)
            return
        # the accumulator object is part of the key: the graph adds into its buffer, which the
        # key keeps alive
        key = (tuple((tuple(t.shape), t.dtype) for t in inputs), tuple(labels.shape), m, accum)
        if self._eval is None or self._eval["key"] != key:
            self._eval = graph_state(warmup=1, key=key)
        self._run_graphed(self._eval, lambda x, y: self._eval_body(x, y, accum, m), inputs, labels)
