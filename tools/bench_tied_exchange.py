"""Timing of the tied word-embedding gradient exchange against its byte floors (needs >= 2 GPUs;
run under torchrun with 2 processes):

    python -m torch.distributed.run --nproc-per-node=2 tools/bench_tied_exchange.py [--iters 20]

Each kernel is timed on its own.  ``tied_grad_push`` (rank 1, the last stage): the replica's
gradient, V x H fp32 = 125 MB at BERT's padded vocabulary, into rank 0's inbox; its floor is 125 MB
over NVLink.  ``tied_grad_reduce`` (rank 0, the first stage), timed after every push has been
published, so its flag wait is satisfied at once: g + inbox into its own gradient and into rank
1's; its floor is the larger of 250 MB read + 125 MB written of local HBM (3.35 TB/s, the H100 SXM
data sheet's figure) and 125 MB of peer writes.  The NVLink rate is that of a plain peer copy of
the same size, measured in the same run.  Prints one JSON line; CUDA-event means over ``--iters``
launches after 3 warm-up launches."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from skycomputing_b200.ops import native as nat  # noqa: E402
from skycomputing_b200.ops.functions import ParamBank  # noqa: E402
from skycomputing_b200.parallel.p2p import TiedGradExchange  # noqa: E402

V, H = 30528, 1024
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    if world != 2:
        raise SystemExit("run with exactly 2 processes")
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    w = torch.nn.Parameter(torch.zeros(V, H, device=dev))
    bank = ParamBank([w], need_shadow=False)
    bank.ensure()
    bank.flat_grad.normal_()
    state = torch.zeros(4, dtype=torch.int32, device=dev)      # [epoch, error, -, -]
    ex = TiedGradExchange(bank, rank == 0, 1 - rank, dev, state.data_ptr(), state.data_ptr() + 4)
    nbytes = V * H * 4

    s = torch.cuda.current_stream().cuda_stream
    epoch = state[0:1]

    def timed(fn, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / iters

    n_push = 3 + a.iters
    # 1. push alone (rank 1): n_push pushes into the inbox; nothing waits for them
    push_ms = None
    if rank == 1:
        for _ in range(3):
            ex.push()
        push_ms = timed(ex.push, a.iters)
    torch.cuda.synchronize()
    dist.barrier()
    # 2. reduce alone (rank 0): every push has arrived (the flag reads n_push), so the reduce's
    # wait is satisfied at once and only its sum and its stores are timed; epoch k <= n_push
    reduce_ms = None
    if rank == 0:
        def reduce_step():
            nat.ext().advance_epoch(state.data_ptr(), 1, s)
            ex.reduce()
        for _ in range(3):
            reduce_step()
        reduce_ms = timed(reduce_step, a.iters)
        assert int(epoch.item()) <= n_push
    torch.cuda.synchronize()
    dist.barrier()
    # 3. NVLink reference: a plain peer copy of the same size into the inbox (rank 1)
    copy_ms = None
    if rank == 1:
        dst = ex.peer_base + ex.HEADER
        src = bank.grad().data_ptr()
        scratch = torch.zeros(64, dtype=torch.int32, device=dev)
        copy = lambda: nat.ext().peer_copy_signal(src, dst, nbytes, scratch.data_ptr(), 0, 0, s)  # noqa: E731
        for _ in range(3):
            copy()
        copy_ms = timed(copy, a.iters)
    torch.cuda.synchronize()
    dist.barrier()
    info = dict(rank=rank, push_ms=push_ms, reduce_ms=reduce_ms, peer_copy_ms=copy_ms,
                error=int(state[1].item()))
    gathered = [None] * world
    dist.all_gather_object(gathered, info)
    if rank == 0:
        push_ms, copy_ms = gathered[1]["push_ms"], gathered[1]["peer_copy_ms"]
        reduce_ms = gathered[0]["reduce_ms"]
        nvlink = nbytes / (copy_ms * 1e-3)                      # bytes/s of a plain peer copy
        hbm_floor_ms = 3 * nbytes / HBM * 1e3                   # 250 MB read + 125 MB written
        peer_floor_ms = nbytes / nvlink * 1e3                   # 125 MB peer writes
        reduce_floor_ms = max(hbm_floor_ms, peer_floor_ms)      # both streams overlap
        print(json.dumps(dict(
            card=torch.cuda.get_device_name(dev), bytes=nbytes,
            push_ms=push_ms, push_floor_ms=peer_floor_ms, push_floor_over_time=peer_floor_ms / push_ms,
            nvlink_gb_s=nvlink / 1e9,
            reduce_ms=reduce_ms, reduce_hbm_floor_ms=hbm_floor_ms, reduce_peer_floor_ms=peer_floor_ms,
            reduce_floor_over_time=reduce_floor_ms / reduce_ms,
            error=max(g["error"] for g in gathered))), flush=True)
    ex.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
