"""Peer-memory stage boundaries over NVLink / NVSwitch (CUDA IPC), the fused data path.

Every pipeline rank owns, in ITS OWN HBM and mapped by its neighbours through CUDA IPC:

* an inbound ACTIVATION region written by the previous stage (one ``[M_mb, H]`` bf16 slot + one
  ``[B_mb*S]`` fp32 mask slot per micro-batch) with one ``uint32`` flag per 128-row panel,
* an inbound GRADIENT region written by the next stage, same shape, own flags.

Producers are kernels of the neighbour GPU: the last GEMM of stage *i* (FFN2 with bias + dropout +
residual + LayerNorm in its GEMM epilogue) stores its output tiles straight into stage *i+1*'s
activation slot, and the first dgrad GEMM of stage *i+1*
(``QKV-dgrad + residual``) stores its output tiles straight into stage *i*'s gradient slot; both
bump the panel flags with ``red.release.sys``.  Consumers (the QKV GEMM's TMA producer warp / the
LayerNorm-backward warps) poll the flags with ``ld.acquire.sys``.  Flags are cumulative and never
reset: slot *j* is written exactly once per step, so after step *s* a complete panel reads
``s * signals_per_panel`` and consumers wait for ``epoch * signals_per_panel`` where ``epoch`` is
a device-side step counter (CUDA-graph friendly).

Slot re-use: a GRADIENT slot is only re-written in step *s+1* after this rank's own step-*s+1*
forward traffic, which is stream-ordered behind everything that read the slot.  An ACTIVATION slot
has one reader that is NOT ordered by opposite-direction traffic: the deferred QKV weight gradient
(side stream, flushed after the dgrad GEMM has already published the input gradient).  It is
covered by a one-word ACK per link and step: the consumer bumps the producer's ack word with
``red.release.sys`` once its weight gradients of the step have joined, and the producer waits for
``ack >= epoch`` (the word starts at 1) before its first forward of the next step.  The wait is
free in practice - the consumer of a link finishes its backward before its producer does.

Reference: replaces the CPU-staged TensorPipe hop ``rref.to_here()`` of
scaelum/builder/module_wrapper.py:148-175 and the distributed-autograd gradient hop of
scaelum/runner/runner.py:137.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import native as nat


class _DevView:
    """``__cuda_array_interface__`` shim so torch can wrap raw (IPC) device memory."""

    def __init__(self, ptr: int, shape: tuple, typestr: str):
        self.__cuda_array_interface__ = {
            "shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2,
            "strides": None,
        }


def tensor_from_ptr(ptr: int, shape: tuple, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    if dtype == torch.bfloat16:
        t = torch.as_tensor(_DevView(ptr, shape, "<i2"), device=device)
        return t.view(torch.bfloat16)
    typestr = {torch.float32: "<f4", torch.int32: "<i4", torch.int64: "<i8"}[dtype]
    return torch.as_tensor(_DevView(ptr, shape, typestr), device=device)


class BoundaryRegion:
    """One inbound region (activation or gradient) living in this rank's HBM."""

    def __init__(self, n_slots: int, rows: int, cols: int, mask_elems: int, device: torch.device):
        self.n_slots, self.rows, self.cols, self.mask_elems = n_slots, rows, cols, mask_elems
        self.panels = (rows + 127) // 128
        self.slot_bytes = rows * cols * 2
        self.mask_bytes = ((mask_elems * 4 + 255) // 256) * 256
        # panel flags followed by ONE extra flag that guards the mask slot
        self.flag_bytes = (((self.panels + 1) * 4 + 255) // 256) * 256
        self.stride = self.slot_bytes + self.mask_bytes + self.flag_bytes
        # one trailing 256-byte line holds the per-link ack word (see the module docstring)
        self.nbytes = n_slots * self.stride + 256
        self.ptr, self.handle = nat.ext().ipc_alloc(self.nbytes)
        self.device = device
        tensor_from_ptr(self.ack_ptr(), (1,), torch.int32, device).fill_(1)

    def layout(self) -> dict:
        return dict(n_slots=self.n_slots, rows=self.rows, cols=self.cols, stride=self.stride,
                    slot_bytes=self.slot_bytes, mask_bytes=self.mask_bytes, panels=self.panels)

    def data_ptr(self, slot: int, base: Optional[int] = None) -> int:
        return (self.ptr if base is None else base) + slot * self.stride

    def mask_ptr(self, slot: int, base: Optional[int] = None) -> int:
        return self.data_ptr(slot, base) + self.slot_bytes

    def flags_ptr(self, slot: int, base: Optional[int] = None) -> int:
        return self.data_ptr(slot, base) + self.slot_bytes + self.mask_bytes

    def mask_flag_ptr(self, slot: int, base: Optional[int] = None) -> int:
        return self.flags_ptr(slot, base) + 4 * self.panels

    def ack_ptr(self, base: Optional[int] = None) -> int:
        return (self.ptr if base is None else base) + self.n_slots * self.stride

    def free(self) -> None:
        if self.ptr:
            nat.ext().dev_free(self.ptr)
            self.ptr = 0


class FusedChannel:
    """This rank's view of the link to ONE neighbour stage (previous or next)."""

    def __init__(self, device: torch.device, epoch_ptr: int, error_ptr: int):
        self.device = device
        self.epoch_ptr = epoch_ptr
        self.error_ptr = error_ptr
        # local inbound region (activations from prev, or gradients from next)
        self.local: Optional[BoundaryRegion] = None
        # peer's inbound region that WE write (gradients to prev, or activations to next)
        self.peer_base = 0
        self.peer_layout: Optional[dict] = None
        self.rows = self.cols = 0
        self.act_wait_mult = nat.ext().LN_SIGNALS_PER_PANEL
        self.grad_wait_mult = 1

    # ---- inbound activation side (this rank is the consumer stage) --------------------------
    def act_view(self, mb: int, rows: int, cols: int) -> torch.Tensor:
        return tensor_from_ptr(self.local.data_ptr(mb), (rows, cols), torch.bfloat16, self.device)

    def mask_view(self, mb: int, n: int) -> torch.Tensor:
        return tensor_from_ptr(self.local.mask_ptr(mb), (n,), torch.float32, self.device)

    def act_flags_ptr(self, mb: int) -> int:
        return self.local.flags_ptr(mb)

    # ---- inbound gradient side (this rank is the producer stage of the forward link) --------
    def grad_view(self, mb: int, rows: int, cols: int) -> torch.Tensor:
        return tensor_from_ptr(self.local.data_ptr(mb), (rows, cols), torch.bfloat16, self.device)

    def grad_flags_ptr(self, mb: int) -> int:
        return self.local.flags_ptr(mb)

    # ---- outbound pointers into the peer's region --------------------------------------------
    def _peer(self, mb: int, what: str) -> int:
        lay = self.peer_layout
        base = self.peer_base + mb * lay["stride"]
        if what == "data":
            return base
        if what == "mask":
            return base + lay["slot_bytes"]
        return base + lay["slot_bytes"] + lay["mask_bytes"]

    def peer_act_ptr(self, mb: int) -> int:
        return self._peer(mb, "data")

    def peer_act_flags_ptr(self, mb: int) -> int:
        return self._peer(mb, "flags")

    def peer_mask_ptr(self, mb: int) -> int:
        return self._peer(mb, "mask")

    def peer_grad_ptr(self, mb: int) -> int:
        return self._peer(mb, "data")

    def peer_grad_flags_ptr(self, mb: int) -> int:
        return self._peer(mb, "flags")

    @property
    def grad_ld(self) -> int:
        return self.peer_layout["cols"]

    # ---- activation-slot acknowledgement (one word per link, lives in the PRODUCER's gradient
    # region, which the consumer has mapped for its gradient stores anyway) --------------------
    def ack_consumed(self) -> None:
        """Consumer side (channel to the previous stage): everything of this step that read the
        inbound activation slots is stream-ordered before this call."""
        lay = self.peer_layout
        nat.ext().signal_flags(self.peer_base + lay["n_slots"] * lay["stride"], 1, 1,
                               torch.cuda.current_stream().cuda_stream)

    def wait_consumer_ack(self) -> None:
        """Producer side (channel to the next stage): the consumer has finished every read of the
        slots it received in the previous step."""
        nat.ext().wait_flags(self.local.ack_ptr(), 1, self.epoch_ptr, 1, self.error_ptr,
                             torch.cuda.current_stream().cuda_stream)

    def send_mask(self, mask: torch.Tensor, mb: int) -> None:
        """Copy the additive attention mask next to the activation slot of the next stage."""
        m = mask.reshape(-1).contiguous().float()
        nbytes = ((m.numel() * 4 + 15) // 16) * 16
        if nbytes != m.numel() * 4:
            pad = torch.zeros(nbytes // 4, dtype=torch.float32, device=m.device)
            pad[: m.numel()] = m
            m = pad
        mask_flag = self._peer(mb, "flags") + 4 * self.peer_layout["panels"]
        nat.ext().peer_copy_signal(m.data_ptr(), self.peer_mask_ptr(mb), nbytes, mask_flag, 1, 1,
                                   torch.cuda.current_stream().cuda_stream)


class FusedBoundaryManager:
    """Allocates this rank's inbound regions and exchanges IPC handles with its neighbours."""

    def __init__(self, stage_index: int, num_stages: int, stage_to_rank: List[int],
                 micro_batches: int, rows: int, cols: int, mask_elems: int,
                 device: torch.device, group=None, ring: bool = False):
        """``ring=True`` (looped pipelines): every stage has a previous and a next neighbour
        (stage 0's previous is the last stage); ``micro_batches`` is then the number of slots,
        one per (chunk, micro-batch)."""
        self.stage_index, self.num_stages = stage_index, num_stages
        self.stage_to_rank = stage_to_rank
        self.device = device
        self.micro_batches = micro_batches
        self.state = torch.zeros(4, dtype=torch.int32, device=device)  # [epoch, error, -, -]
        self.epoch_ptr = self.state.data_ptr()
        self.error_ptr = self.state.data_ptr() + 4
        self.prev: Optional[FusedChannel] = None   # link to stage-1 (we consume activations)
        self.next: Optional[FusedChannel] = None   # link to stage+1 (we consume gradients)
        self._opened: List[int] = []
        self._regions: List[BoundaryRegion] = []
        ext = nat.ext()
        has_prev, has_next = stage_index > 0, stage_index < num_stages - 1
        if ring and num_stages > 1:
            has_prev = has_next = True
        prev_idx = (stage_index - 1) % num_stages
        next_idx = (stage_index + 1) % num_stages
        my_rank = dist.get_rank(group)
        if has_prev:
            self.prev = FusedChannel(device, self.epoch_ptr, self.error_ptr)
            self.prev.local = BoundaryRegion(micro_batches, rows, cols, mask_elems, device)
            self._regions.append(self.prev.local)
        if has_next:
            self.next = FusedChannel(device, self.epoch_ptr, self.error_ptr)
            self.next.local = BoundaryRegion(micro_batches, rows, cols, 0, device)
            self._regions.append(self.next.local)
        block_n = ext.gemm_pick_block_n(rows, cols)
        grad_mult = ext.gemm_tiles_per_panel(cols, block_n)
        # forward producer = the GEMM + LayerNorm kernel (one signal per column tile of a panel)
        # when the row fits a cluster, else the standalone LayerNorm kernel (one per 8 rows)
        act_mult = (nat.gemm_ln_tiles_per_panel(rows, cols) if nat.gemm_ln_supported(rows, cols)
                    else ext.LN_SIGNALS_PER_PANEL)
        for ch in (self.prev, self.next):
            if ch is not None:
                ch.grad_wait_mult = grad_mult
                ch.act_wait_mult = act_mult
                ch.rows, ch.cols = rows, cols
        # exchange handles: everybody publishes {to_prev: handle of my act region, to_next: grad}
        mine: Dict[str, object] = {"rank": my_rank, "gpu": self._gpu_uuid(device)}
        if has_prev:
            mine["act"] = (self.prev.local.handle, self.prev.local.layout())
        if has_next:
            mine["grad"] = (self.next.local.handle, self.next.local.layout())
        world = dist.get_world_size(group)
        gathered: List[dict] = [None] * world  # type: ignore[list-item]
        dist.all_gather_object(gathered, mine, group=group)
        by_rank = {g["rank"]: g for g in gathered}
        # a neighbour's GPU is identified by UUID, not by assuming rank == CUDA ordinal: the
        # ordinal of the same physical GPU differs between processes under CUDA_VISIBLE_DEVICES
        for idx, present in ((prev_idx, has_prev), (next_idx, has_next)):
            if present:
                ext.enable_peer_access(self._local_device_of(by_rank[stage_to_rank[idx]]["gpu"],
                                                             stage_to_rank[idx]))
        if has_next:   # I write activations into next stage's "act" region
            handle, lay = by_rank[stage_to_rank[next_idx]]["act"]
            self.next.peer_base = ext.ipc_open(handle)
            self.next.peer_layout = lay
            self._opened.append(self.next.peer_base)
        if has_prev:   # I write gradients into prev stage's "grad" region
            handle, lay = by_rank[stage_to_rank[prev_idx]]["grad"]
            self.prev.peer_base = ext.ipc_open(handle)
            self.prev.peer_layout = lay
            self._opened.append(self.prev.peer_base)
        torch.cuda.synchronize(device)   # the ack words are initialised before anybody proceeds
        dist.barrier(group=group)

    @staticmethod
    def _gpu_uuid(device: torch.device) -> str:
        return str(torch.cuda.get_device_properties(device).uuid)

    @staticmethod
    def _local_device_of(uuid: str, rank: int) -> int:
        """CUDA ordinal, in THIS process, of the GPU with that UUID (the peer rank's device)."""
        for i in range(torch.cuda.device_count()):
            if str(torch.cuda.get_device_properties(i).uuid) == uuid:
                return i
        raise RuntimeError(
            f"the GPU of rank {rank} ({uuid}) is not visible to this process: fused stage "
            "boundaries need every neighbour's GPU in CUDA_VISIBLE_DEVICES (peer access)")

    def begin_step(self) -> None:
        """Advance the flag epoch; as a producer, wait for last step's consumer acknowledgement."""
        self.advance_epoch()
        if self.next is not None:
            self.next.wait_consumer_ack()

    def end_of_backward(self) -> None:
        """Call once all reads of this step's inbound activation slots are stream-ordered before
        the current point (i.e. after the weight-gradient side stream has joined)."""
        if self.prev is not None:
            self.prev.ack_consumed()

    def advance_epoch(self) -> None:
        nat.ext().advance_epoch(self.epoch_ptr, 1, torch.cuda.current_stream().cuda_stream)

    def error_code(self) -> int:
        return int(self.state[1].item())

    def close(self) -> None:
        ext = nat.ext()
        torch.cuda.synchronize(self.device)
        for p in self._opened:
            try:
                ext.ipc_close(p)
            except Exception:
                pass
        self._opened = []
        for r in self._regions:
            r.free()
        self._regions = []


class GradNormExchange:
    """Peer-memory all-reduce of ONE fp32 per step: the stages' shares of the squared gradient
    norm, summed in pipeline-position order so that every rank computes a bit-identical clip
    coefficient.  Runs inside the captured step (``optim_finalize`` kernel, csrc/kernels/
    elementwise_sm100.cu, which also documents the slot protocol).

    Every rank owns one small region in its own HBM (``flags[P]`` in the first 256 bytes, then
    ``slots[2][P]`` fp32, double-buffered by epoch parity) and maps the regions of ALL other ranks,
    not only of its neighbours.  The flag epoch and the error word are the boundary manager's: a
    peer that never publishes makes the wait time out and sets error 4, which
    ``Runner._check_boundary_health`` reports.  Collective: every rank of ``group`` constructs it.
    """

    def __init__(self, position: int, num_positions: int, rank_of_position: List[int],
                 device: torch.device, epoch_ptr: int, error_ptr: int, group=None):
        ext = nat.ext()
        self.position, self.n_ranks = position, num_positions
        self.device = device
        self.epoch_ptr, self.error_ptr = epoch_ptr, error_ptr
        self.nbytes = 256 + ((2 * num_positions * 4 + 255) // 256) * 256
        self.ptr, handle = ext.ipc_alloc(self.nbytes)
        self._opened: List[int] = []
        mine = {"rank": dist.get_rank(group), "gpu": FusedBoundaryManager._gpu_uuid(device),
                "handle": handle}
        gathered: List[dict] = [None] * dist.get_world_size(group)  # type: ignore[list-item]
        dist.all_gather_object(gathered, mine, group=group)
        by_rank = {g["rank"]: g for g in gathered}
        bases = []
        for pos in range(num_positions):
            r = rank_of_position[pos]
            if pos == position:
                bases.append(self.ptr)
                continue
            ext.enable_peer_access(FusedBoundaryManager._local_device_of(by_rank[r]["gpu"], r))
            base = ext.ipc_open(by_rank[r]["handle"])
            self._opened.append(base)
            bases.append(base)
        self._bases = torch.tensor(bases, dtype=torch.int64, device=device)
        self.regions_ptr = self._bases.data_ptr()
        torch.cuda.synchronize(device)
        dist.barrier(group=group)   # every region is mapped before anybody may write into it

    def close(self) -> None:
        if not self.ptr:
            return
        ext = nat.ext()
        torch.cuda.synchronize(self.device)
        for p in self._opened:
            try:
                ext.ipc_close(p)
            except Exception:
                pass
        self._opened = []
        ext.dev_free(self.ptr)
        self.ptr = 0


class TiedGradExchange:
    """One summed gradient per step for a word-embedding table tied to a masked-language-model
    decoder on another rank: the first rank holds the table, the last rank a replica.  Both must
    step on ``g = g_embeddings + g_decoder``; then any optimizer keeps the copies bit-identical.
    Runs inside the captured step (``tied_grad_push`` / ``tied_grad_reduce`` kernels, csrc/kernels/
    elementwise_sm100.cu).

    Each of the two ranks owns one region in its own HBM, mapped by the other: 256 bytes of words
    (``[0]`` the inbound flag, ``[1]`` the done counter of the kernel this rank launches), then one
    fp32 buffer of the table's size: on the first rank the INBOX, on the last rank the replica's
    gradient itself (the bank's gradient is rebound to it, so the sum can be stored into it).

    Per step: the last rank pushes its gradient into the inbox and bumps the first rank's flag; the
    first rank, after its own backward, waits for that flag (>= epoch), computes the sum once,
    stores it into its own gradient and into the replica's, and bumps the last rank's flag, which
    the last rank waits for before its optimizer.  A timeout sets error 5 in the boundary manager's
    error word.  The single inbox is safe to reuse: step k+1's push follows the last rank's wait
    for step k's sum, which the first rank released only after it had read the inbox.  Collective:
    every rank of ``group`` constructs it (``bank`` None on the others)."""

    HEADER = 256

    def __init__(self, bank, is_first: bool, peer_rank: Optional[int], device: torch.device,
                 epoch_ptr: int, error_ptr: int, group=None):
        ext = nat.ext()
        self.bank, self.is_first, self.device = bank, is_first, device
        self.epoch_ptr, self.error_ptr = epoch_ptr, error_ptr
        self.ptr = self.peer_base = 0
        self.buffer: Optional[torch.Tensor] = None
        mine = {"rank": dist.get_rank(group), "gpu": None, "handle": None}
        if bank is not None:
            bank.ensure()
            self.numel = bank.flat.numel()
            nbytes = self.HEADER + ((self.numel * 4 + 255) // 256) * 256
            self.ptr, handle = ext.ipc_alloc(nbytes)
            tensor_from_ptr(self.ptr, (self.HEADER // 4,), torch.int32, device).zero_()
            self.buffer = tensor_from_ptr(self.ptr + self.HEADER, tuple(bank.flat.shape),
                                          torch.float32, device)
            self.buffer.zero_()
            if not is_first:
                self.buffer.copy_(bank.flat_grad)
                bank.flat_grad = self.buffer
                bank._bind_grads()
            mine.update(gpu=FusedBoundaryManager._gpu_uuid(device), handle=handle)
        gathered: List[dict] = [None] * dist.get_world_size(group)  # type: ignore[list-item]
        dist.all_gather_object(gathered, mine, group=group)
        if bank is not None:
            peer = {g["rank"]: g for g in gathered}[peer_rank]
            ext.enable_peer_access(FusedBoundaryManager._local_device_of(peer["gpu"], peer_rank))
            self.peer_base = ext.ipc_open(peer["handle"])
        torch.cuda.synchronize(device)
        dist.barrier(group=group)   # both regions are zeroed and mapped before either is written

    def push(self) -> None:
        """Last rank, once its weight gradients have joined."""
        nat.ext().tied_grad_push(src=self.bank.grad().data_ptr(), dst=self.peer_base + self.HEADER,
                                 n=self.numel, flag=self.peer_base, done=self.ptr + 4,
                                 stream=torch.cuda.current_stream().cuda_stream)

    def wait(self) -> None:
        """Last rank, before its optimizer: the summed gradient has arrived."""
        nat.ext().wait_flags(self.ptr, 1, self.epoch_ptr, 1, self.error_ptr,
                             torch.cuda.current_stream().cuda_stream)

    def reduce(self) -> None:
        """First rank, after its last backward (embedding backward included) has joined."""
        nat.ext().tied_grad_reduce(g=self.bank.grad().data_ptr(), inbox=self.ptr + self.HEADER,
                                   peer_g=self.peer_base + self.HEADER, n=self.numel,
                                   wait_flag=self.ptr, epoch=self.epoch_ptr,
                                   error_flag=self.error_ptr, publish_flag=self.peer_base,
                                   done=self.ptr + 4,
                                   stream=torch.cuda.current_stream().cuda_stream)

    def close(self) -> None:
        """Hands the replica its own gradient memory again (not zeroed), then unmaps and frees."""
        if not self.ptr:
            return
        ext = nat.ext()
        torch.cuda.synchronize(self.device)
        if not self.is_first and self.bank.flat_grad is self.buffer:
            self.bank.flat_grad = self.buffer.clone()
            self.bank._bind_grads()
        try:
            ext.ipc_close(self.peer_base)
        except Exception:
            pass
        self.buffer = None
        ext.dev_free(self.ptr)
        self.ptr = self.peer_base = 0
