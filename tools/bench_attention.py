"""wgmma attention kernels: S = 128 single-tile kernels, the tiled kernels at other lengths, and
the eager PyTorch attention they replace (bf16, same tokens), per forward / backward call.
CUDA-graph replays; one JSON line per configuration -> bench_out/bench_attention.json.

The first row is the BERT-large training step's configuration (B = 32, 16 heads, S = 128, additive
padding mask, dropout 0.1 on the probabilities from an RngState).  Every row also gives the HBM
bytes a call must move at least (forward: QKV in, ctx and lse out; backward: QKV, dO, O and lse in,
dQKV out; the 4-byte-per-token mask is left out), the time those bytes take at the 3.35 TB/s
data-sheet bandwidth of the H100 SXM, and the share of that floor the kernel reaches."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from skycomputing_b200.ops import native as nat  # noqa: E402
from tools.triage_gemm import timeit  # noqa: E402


def eager(qkv, B, S, heads):
    H = qkv.shape[1] // 3
    q, k, v = qkv.view(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
    return (p @ v).permute(0, 2, 1, 3).reshape(B * S, H)


HBM_BYTES_PER_S = 3.35e12


def byte_floor_us(B, S, heads, H):
    tok = B * S
    lse = B * heads * S * 4
    fwd = tok * 3 * H * 2 + tok * H * 2 + lse
    bwd = tok * 3 * H * 2 + 2 * tok * H * 2 + lse + tok * 3 * H * 2
    return fwd / HBM_BYTES_PER_S * 1e6, bwd / HBM_BYTES_PER_S * 1e6


def main():
    rows = []
    heads, H = 16, 1024
    print(json.dumps(dict(gpu=torch.cuda.get_device_name())), flush=True)
    configs = [(128, 32, True)] + [(S, B, False) for S, B in
                                   ((128, 32), (64, 64), (256, 16), (384, 8), (512, 8))]
    for S, B, step in configs:
        torch.manual_seed(0)
        qkv = torch.randn(B * S, 3 * H, device="cuda").bfloat16()
        dctx = torch.randn(B * S, H, device="cuda").bfloat16()
        mask, kw = None, {}
        if step:
            lens = torch.randint(S // 2, S + 1, (B,), device="cuda")
            mask = (torch.arange(S, device="cuda")[None, :] >= lens[:, None]).float() * -10000.0
            kw = dict(dropout_p=0.1, rng=nat.RngState(1), rng_stream=0)
        ctx, lse = nat.attention_fwd(qkv, mask, B, S, heads, **kw)
        tf = timeit(lambda: nat.attention_fwd(qkv, mask, B, S, heads, **kw)) * 1e3
        tb = timeit(lambda: nat.attention_bwd(qkv, mask, ctx, lse, dctx, B, S, heads, **kw)) * 1e3
        te = timeit(lambda: eager(qkv, B, S, heads)) * 1e3
        qg = qkv.clone().requires_grad_(True)

        def eager_fb():
            o = eager(qg, B, S, heads)
            o.backward(dctx)
            qg.grad = None

        teb = timeit(eager_fb, iters=5) * 1e3 - te
        flops_f = 4.0 * B * heads * S * S * 64
        ff, fb = byte_floor_us(B, S, heads, H)
        row = dict(S=S, B=B, tokens=B * S, kernels="single-tile" if S == 128 else "tiled",
                   config="training step (mask, dropout 0.1)" if step else "no mask, no dropout",
                   fwd_us=round(tf, 1), bwd_us=round(tb, 1), fwd_tflops=round(flops_f / tf / 1e6, 1),
                   bwd_tflops=round(2.5 * flops_f / tb / 1e6, 1),
                   fwd_byte_floor_us=round(ff, 1), bwd_byte_floor_us=round(fb, 1),
                   fwd_share_of_byte_floor=round(ff / tf, 3),
                   bwd_share_of_byte_floor=round(fb / tb, 3),
                   eager_fwd_us=round(te, 1), eager_bwd_us=round(teb, 1))
        rows.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(rows, open("bench_out/bench_attention.json", "w"), indent=1)


if __name__ == "__main__":
    main()
