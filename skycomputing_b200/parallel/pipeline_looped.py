"""Looped ("breadth-first") pipeline engine: v virtual stages per rank.

A plain 1F1B step costs ``m x T + (P - 1) x (F + B)``: the fill / drain term is a whole stage's
forward + backward per pipeline hop and dominates at 8 GPUs.  Here every rank owns v NON-adjacent chunks of the model (virtual stage k = chunk k // P
of rank k % P, ``Allocator.looped_allocate``), the ranks form a ring, and a micro-batch visits
every rank v times.  Each rank runs, per step,

    for c in chunks:            for j in micro-batches:  forward (c, j)
    for c in reversed(chunks):  for j in micro-batches:  backward(c, j)

(the breadth-first order of Lamy-Poirier, "Breadth-first pipeline parallelism", 2022).  A hop now
costs 1/v of a rank's work, so the step is ``m x T + (P - 1) x (F + B) / v`` as long as
``m >= P``; activation memory grows to all micro-batches of all chunks, which 80 GB of HBM absorb
easily for the models this framework targets.  Weight gradients use the same deferral as the
plain engine.

Transport: ``boundary="auto"`` / ``"fused"`` uses the plain engine's peer-memory boundary when
every chunk of every rank supports it on the native path: the ranks form a RING of
``FusedChannel``s (incl. the wrap-around link), one slot per (chunk, micro-batch), and the whole
step is captured into one CUDA graph.  The Runner selects it by default (``SKY_LOOPED_FUSED=0``
turns it off); tests/test_multi_gpu.py runs it on 2, 4 and 8 GPUs.  Otherwise the boundaries are
``torch.distributed`` point-to-point (gloo on CPU, NCCL on GPUs): both ends of a link post their
transfers in the same (chunk, micro-batch) order, so plain FIFO matching is enough; the CPU tests
(tests/test_pipeline_cpu.py) run this path.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch
import torch.distributed as dist

from .comm import TorchDistComm
from .engine_base import EngineBase


def looped_order(num_chunks: int, micro_batches: int) -> List[tuple]:
    """[('F' | 'B', chunk, micro_batch)] for one rank."""
    order = [("F", c, j) for c in range(num_chunks) for j in range(micro_batches)]
    order += [("B", c, j) for c in reversed(range(num_chunks)) for j in range(micro_batches)]
    return order


class LoopedPipelineEngine(EngineBase):
    def __init__(self, stages: Sequence, virtual_indices: Sequence[int], num_ranks: int,
                 ring: Sequence[int], device: torch.device, optimizer,
                 loss_fn: Optional[Callable] = None, micro_batches: int = 1, group=None,
                 advance_rng: bool = True, boundary: str = "dist", use_cuda_graph: bool = True):
        """``stages[i]`` is the ModuleWrapper of virtual stage ``virtual_indices[i]``; ``ring[p]`` is
        the process rank at ring position p (virtual stage k lives at position k % num_ranks)."""
        super().__init__(stages, device, optimizer, loss_fn, micro_batches, boundary,
                         use_cuda_graph, group, advance_rng)
        self.vidx = list(virtual_indices)
        self.P = num_ranks
        self.v = len(self.stages)
        self.total = self.P * self.v
        assert self.P >= 2, "a looped pipeline needs at least two ranks"
        assert self.vidx == sorted(self.vidx) and len(set(k % self.P for k in self.vidx)) == 1
        self.pos = self.vidx[0] % self.P
        self.s = self.pos                                 # ring position (trace / log naming)
        assert self.vidx == [c * self.P + self.pos for c in range(self.v)], self.vidx
        self.ring = list(ring)
        self.prev_rank = self.ring[(self.pos - 1) % self.P]
        self.next_rank = self.ring[(self.pos + 1) % self.P]
        self.is_first = self.vidx[0] == 0                 # owns the stage that reads the data
        self.is_last = self.vidx[-1] == self.total - 1    # owns the stage that computes the loss
        self._comm: Optional[TorchDistComm] = None       # created on first use (p2p path only)
        self._order = looped_order(self.v, self.m)
        self.schedule = "looped"

    # ------------------------------------------------------------------ helpers
    @property
    def comm(self) -> TorchDistComm:
        """torch.distributed p2p transport.  Forward-only passes use it even when training runs
        on the fused ring; one communicator per direction, as on the training path (collective
        on first use)."""
        if self._comm is None:
            self._comm = TorchDistComm(self.device, group=self.group, directional=True)
        return self._comm

    # ------------------------------------------------------------------ setup (collective)
    def _setup(self, inputs) -> None:
        self._configure_wgrad(True)
        want_fused = self.boundary in ("auto", "fused") and self._native_active()
        self._setup_batch_shape(inputs, self.ring[0])
        ok, hidden = False, 0
        if want_fused:
            ok = True
            for c, st in enumerate(self.stages):
                k = self.vidx[c]
                spans = st.spans()
                if spans:
                    sp = spans[0]
                    if sp.head is not None:
                        hidden = sp.head.attention.output.dense.weight.shape[0]
                        ok = ok and sp.head.attention.self.attention_head_size == 64
                in_ok, out_ok = st.fused_boundary_support((self.mb_batch, self.seq, hidden))
                ok = ok and (in_ok or k == 0) and (out_ok or k == self.total - 1)
            ok = ok and self.seq % 8 == 0 and hidden > 0 and hidden % 64 == 0 and \
                (self.mb_batch * self.seq) % 128 == 0
        flags = [None] * dist.get_world_size(self.group)
        dist.all_gather_object(flags, (bool(ok), int(hidden), self._norm_info()), group=self.group)
        if want_fused and all(f[0] for f in flags):
            from .p2p import FusedBoundaryManager

            rows = self.mb_batch * self.seq
            self.fused = FusedBoundaryManager(self.pos, self.P, self.ring, self.v * self.m, rows,
                                              max(f[1] for f in flags), rows, self.device,
                                              group=self.group, ring=True)
            self.in_fused = self.out_fused = True
            self._setup_graphable(True)
        if self.fused is None:
            # collective: one communicator per direction so crossed sends cannot dead-lock NCCL
            self._comm = TorchDistComm(self.device, group=self.group, directional=True)
        # one optimizer over all local chunks (optim_module): one share of the norm per position
        self._setup_grad_norm(self.pos, self.P, self.ring, [f[2] for f in flags])
        self._setup_tie(self.ring[0], self.ring[self.P - 1])
        self._setup_done = True

    def _step_body(self, inputs, labels) -> None:
        if self.fused is not None:
            self._step_body_fused(inputs, labels)
        else:
            self._step_body_p2p(inputs, labels)

    def _step_body_fused(self, inputs, labels) -> None:
        """The same (chunk, micro-batch) order with every boundary in peer memory: no host-side
        transfers at all, the kernels of neighbouring ranks hand panels to each other."""
        chunks_in, label_chunks = self._begin_step(inputs, labels)
        saved = {}
        for kind, c, j in self._order:
            k = self.vidx[c]
            st = self.stages[c]
            # a link's slots are numbered by the CONSUMER's chunk: inbound = this chunk, outbound =
            # the chunk of virtual stage k + 1 (the same number except on the wrap-around link
            # from the last ring position to the first, where it is c + 1)
            slot = c * self.m + j
            out_slot = ((k + 1) // self.P) * self.m + j
            first_stage, last_stage = k == 0, k == self.total - 1
            st.microbatch = (slot, out_slot)
            st.in_channel = None if first_stage else self.fused.prev
            st.out_channel = None if last_stage else self.fused.next
            if kind == "F":
                args = tuple(t[j] for t in chunks_in) if first_stage else self._fused_inputs(slot)
                if not last_stage and not first_stage:
                    self.fused.next.send_mask(args[-1], out_slot)   # the mask travels with the slot
                self._bind_labels(st, label_chunks if last_stage else None, j)
                self._mark(("F", slot, "begin"))
                outs = st(*args)
                self._mark(("F", slot, "end"))
                if not last_stage and first_stage:
                    self.fused.next.send_mask(outs[-1], out_slot)   # produced by the embeddings here
                loss = self._last_stage_loss(st, outs, label_chunks[j]) if last_stage else None
                saved[(c, j)] = (outs, loss)
            else:
                outs, loss = saved.pop((c, j))
                self._flush_wgrads()
                self._mark(("B", slot, "begin"))
                st.begin_backward()
                with self._arm_wgrad_sgd(c, j):
                    if last_stage:
                        self._backward_from_loss(st, outs, loss)
                    else:
                        torch.autograd.backward([outs[0]], [torch.zeros_like(outs[0])])
                st.end_backward()
                self._mark(("B", slot, "end"))
        self._flush_wgrads()
        self._join_wgrads()
        self.fused.end_of_backward()
        self._optimizer_step([])

    def _step_body_p2p(self, inputs, labels) -> None:
        """The (chunk, micro-batch) order over torch.distributed p2p, one tagged FIFO per chunk."""
        if self._advance_rng and self._native_active():
            from ..models.bert_layers import advance_rng

            advance_rng()
        self._loss_acc.zero_()
        chunks_in = [t.chunk(self.m, dim=0) for t in inputs] if self.is_first else None
        label_chunks = labels.chunk(self.m, dim=0) if (self.is_last and labels is not None) else None
        saved = {}
        for kind, c, j in self._order:
            k = self.vidx[c]
            st = self.stages[c]
            st.microbatch = c * self.m + j
            st.in_channel = st.out_channel = None
            first_stage, last_stage = k == 0, k == self.total - 1
            if kind == "F":
                if first_stage:
                    args = tuple(t[j] for t in chunks_in)
                else:
                    got, reqs = self.comm.recv(self.prev_rank, f"fwd{c}")
                    self.comm.wait(reqs)
                    args = self._prep_inputs(got)
                self._bind_labels(st, label_chunks if last_stage else None, j)
                outs = st(*args)
                loss = None
                if last_stage:
                    loss = self.loss_fn(*self._head_outputs(st, outs, label_chunks[j])) / self.m
                    self._loss_acc += loss.detach().float()
                else:
                    self._pending_sends += self.comm.send(
                        [o.detach() if torch.is_tensor(o) else None for o in outs],
                        self.next_rank, f"fwd{c}")
                saved[(c, j)] = (args, outs, loss)
            else:
                args, outs, loss = saved.pop((c, j))
                self._flush_wgrads()
                st.begin_backward()
                with self._arm_wgrad_sgd(c, j):
                    if last_stage:
                        self._backward_from_loss(st, outs, loss)
                    else:
                        grads, reqs = self.comm.recv(self.next_rank, f"bwd{c}",
                                                     metas=self._grad_metas(outs))
                        self.comm.wait(reqs)
                        self._backward_from_grads(outs, grads)
                st.end_backward()
                if not first_stage:
                    self._pending_sends += self.comm.send(self._in_grads(args), self.prev_rank,
                                                          f"bwd{c}", with_meta=False)
        self._flush_wgrads()
        self._join_wgrads()
        # _optimizer_step without its OPT marks: this path records no phases on the timeline
        if self._sends_before_optimizer():
            self.comm.wait(self._pending_sends)
            self._pending_sends = []
        self._exchange_tied_grads()
        self.optimizer.step()
        self.comm.wait(self._pending_sends)
        self._pending_sends = []

    # ------------------------------------------------------------------ plain forward (eval)
    @torch.no_grad()
    def forward_only(self, inputs: Optional[Sequence[torch.Tensor]] = None, micro_batches: int = 1,
                     labels: Optional[torch.Tensor] = None):
        """Breadth-first forward of every (chunk, micro-batch) without gradients; sends are
        asynchronous and waited for at the end of the pass.  ``labels`` (rank of the last virtual
        stage) reach a label-consuming last layer.  Returns on the rank that owns the last
        virtual stage its outputs (``micro_batches == 1``) or the list of per-chunk outputs."""
        m = int(micro_batches)
        comm = self.comm
        chunks_in = [t.chunk(m, dim=0) for t in inputs] if self.is_first else None
        label_chunks = labels.chunk(m, dim=0) if (self.is_last and labels is not None) else None
        results, pending, keep = [], [], []
        for c, st in enumerate(self.stages):
            comm.forget(f"eval{c}")
            k = self.vidx[c]
            st.in_channel = st.out_channel = None
            for j in range(m):
                st.microbatch = c * m + j
                self._bind_labels(st, label_chunks if k == self.total - 1 else None, j)
                if k == 0:
                    args = tuple(t[j] for t in chunks_in)
                else:
                    args, reqs = comm.recv(self.prev_rank, f"eval{c}")
                    comm.wait(reqs)
                outs = st(*args)
                if k == self.total - 1:
                    results.append(outs)
                else:
                    keep.append(outs)
                    pending += comm.send(list(outs), self.next_rank, f"eval{c}")
        comm.wait(pending)
        if not results:
            return None
        return results[0] if m == 1 else results
