"""Stage-to-stage transport behind one interface.

``TorchDistComm`` moves boundary tensors with ``torch.distributed`` point-to-point operations -
``gloo`` for the CPU plumbing tests (the "fake NVLink"), ``nccl`` send/recv on the GPU box for
every boundary that cannot be fused into a GEMM / LayerNorm epilogue (and as the baseline the
fused path is measured against).  Opposite-direction transfers of the 1F1B steady state are
issued as ONE ``batch_isend_irecv`` group so NCCL cannot dead-lock on crossed sends.

``directional=True`` (looped pipelines on NCCL; collective constructor): messages travel on two
extra communicators, one per direction (sender rank < receiver rank, and the reverse).  NCCL
executes the p2p operations of one communicator in posting order and a send larger than its
staging buffer only completes against a posted receive, so on a ring of TWO ranks - where the next
and the previous neighbour are the same peer - two ranks that both have a send at the head of the
same communicator dead-lock.  A communicator that carries one direction only cannot cross.

Tensor metadata (count / dtype / shape) is exchanged once per (peer, direction) and cached.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

_DTYPES = [torch.float32, torch.bfloat16, torch.float16, torch.int64, torch.int32, torch.bool,
           torch.float64, torch.uint8]


def _encode_meta(tensors: Sequence[Optional[torch.Tensor]]) -> torch.Tensor:
    vals = [len(tensors)]
    for t in tensors:
        if t is None:
            vals += [-1, 0]
            continue
        vals += [_DTYPES.index(t.dtype), t.dim(), *t.shape]
    out = torch.full((64,), -7, dtype=torch.int64)
    assert len(vals) <= 64, "too many boundary tensors / dims for the meta message"
    out[: len(vals)] = torch.tensor(vals, dtype=torch.int64)
    return out


def _decode_meta(meta: torch.Tensor) -> List[Optional[Tuple[torch.dtype, tuple]]]:
    vals = meta.tolist()
    n, pos, out = vals[0], 1, []
    for _ in range(n):
        code = vals[pos]
        if code == -1:
            out.append(None)
            pos += 2
            continue
        nd = vals[pos + 1]
        shape = tuple(vals[pos + 2: pos + 2 + nd])
        out.append((_DTYPES[code], shape))
        pos += 2 + nd
    return out


class TorchDistComm:
    def __init__(self, device: torch.device, group=None, directional: bool = False):
        self.device = device
        self.group = group
        self.backend = dist.get_backend(group)
        self._meta_sent: Dict[tuple, bool] = {}
        self._meta_recv: Dict[tuple, list] = {}
        self._rank = dist.get_rank(group)
        self._up = self._down = None
        if directional and self.backend == "nccl" and group is None:
            self._up = dist.new_group(backend="nccl")      # sender rank < receiver rank
            self._down = dist.new_group(backend="nccl")    # sender rank > receiver rank

    def _grp(self, sender: int, receiver: int):
        if self._up is None:
            return self.group
        return self._up if sender < receiver else self._down

    # -- metadata ---------------------------------------------------------------------------
    def _meta_device(self) -> torch.device:
        return self.device if self.backend == "nccl" else torch.device("cpu")

    def _send_meta(self, tensors, dst: int, key: tuple) -> None:
        if key in self._meta_sent:
            return
        dist.send(_encode_meta(tensors).to(self._meta_device()), dst,
                  group=self._grp(self._rank, dst))
        self._meta_sent[key] = True

    def _recv_meta(self, src: int, key: tuple) -> list:
        if key not in self._meta_recv:
            buf = torch.empty(64, dtype=torch.int64, device=self._meta_device())
            dist.recv(buf, src, group=self._grp(src, self._rank))
            self._meta_recv[key] = _decode_meta(buf.cpu())
        return self._meta_recv[key]

    # -- blocking-ish primitives --------------------------------------------------------------
    def send(self, tensors: Sequence[Optional[torch.Tensor]], dst: int, direction: str,
             with_meta: bool = True) -> list:
        if with_meta:
            self._send_meta(tensors, dst, (dst, direction))
        reqs = []
        for t in tensors:
            if t is not None:
                reqs.append(dist.isend(t.contiguous(), dst, group=self._grp(self._rank, dst)))
        return reqs

    def recv(self, src: int, direction: str, metas: Optional[list] = None) -> Tuple[list, list]:
        """`metas` ([(dtype, shape) | None]) skips the metadata message (the caller knows the
        layout, e.g. gradients mirror the tensors it sent)."""
        if metas is None:
            metas = self._recv_meta(src, (src, direction))
        outs, reqs = [], []
        for m in metas:
            if m is None:
                outs.append(None)
                continue
            dtype, shape = m
            buf = torch.empty(shape, dtype=dtype, device=self.device)
            reqs.append(dist.irecv(buf, src, group=self._grp(src, self._rank)))
            outs.append(buf)
        return outs, reqs

    def exchange(self, send_tensors, dst: int, send_dir: str, src: int, recv_dir: str,
                 recv_metas: list, send_with_meta: bool = False):
        """Send to `dst` and receive from `src` as ONE batched p2p group (1F1B steady state).

        The layout of what is received must be known (`recv_metas`): waiting for a metadata
        message here would dead-lock, because the peer only answers after it got our payload."""
        if send_with_meta:
            self._send_meta(send_tensors, dst, (dst, send_dir))
        metas = recv_metas
        ops, outs = [], []
        for t in send_tensors:
            if t is not None:
                ops.append(dist.P2POp(dist.isend, t.contiguous(), dst, self.group))
        for m in metas:
            if m is None:
                outs.append(None)
                continue
            dtype, shape = m
            buf = torch.empty(shape, dtype=dtype, device=self.device)
            ops.append(dist.P2POp(dist.irecv, buf, src, self.group))
            outs.append(buf)
        reqs = dist.batch_isend_irecv(ops) if ops else []
        return outs, reqs

    def forget(self, direction: str) -> None:
        """Drop the cached metadata of ``direction`` (both ends of a link call this at the same
        point, e.g. at the start of every forward-only pass, whose batch shape may change)."""
        for cache in (self._meta_sent, self._meta_recv):
            for key in [k for k in cache if k[1] == direction]:
                del cache[key]

    def cached_meta(self, src: int, direction: str) -> Optional[list]:
        return self._meta_recv.get((src, direction))

    @staticmethod
    def wait(reqs) -> None:
        for r in reqs:
            r.wait()
