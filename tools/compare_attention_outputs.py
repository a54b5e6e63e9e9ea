"""Comparison of the attention kernels' outputs between two builds of the project.

    python tools/compare_attention_outputs.py dump --root TREE --out DIR [--seq S]
    python tools/compare_attention_outputs.py compare DIR_A DIR_B

``dump`` imports the package from TREE (a source tree with a built extension) and runs the
attention forward and backward at the BERT-large training step's configuration (B = 32, 16 heads,
head size 64, additive padding mask) on seeded inputs, without dropout and with dropout 0.1 from an
``RngState``.  The sequence length is ``--seq`` (default 128, the single-tile kernels; any other
length runs the tiled kernels).  It stores the raw bits of ``ctx``, ``lse`` and ``dqkv`` as
DIR/<name>.npy.  ``compare`` reports, per output, whether the bits agree, the largest absolute
difference, the largest difference in bf16 ulps of the value and relative to the output's largest
magnitude (bf16 outputs) or relative to the value (fp32 ``lse``).  ``dqkv_torchfwd_*`` runs the
backward on a forward (``lse`` and ``ctx``) computed by torch, so it compares the backward kernels
alone on identical inputs.
"""
from __future__ import annotations

import argparse
import os
import sys

B, HEADS, D = 32, 16, 64


def _torch_forward(torch, qkv, mask, ctx_like, S):
    """lse (log2 domain) from torch in fp32, and a seeded random bf16 ctx (the backward reads ctx
    only for delta = rowsum(dO * O)); neither depends on the build."""
    import math

    q, k, _ = qkv.float().view(B, S, 3, HEADS, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(D) + mask.view(B, 1, 1, S)
    lse = (torch.logsumexp(s, -1) / math.log(2.0)).reshape(-1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(99)
    ctx = torch.randn(ctx_like.shape, device="cuda", generator=g).to(torch.bfloat16)
    return ctx, lse


def dump(root: str, out_dir: str, S: int) -> None:
    sys.path.insert(0, os.path.abspath(root))
    import numpy as np
    import torch

    from skycomputing_b200.ops import native as nat

    assert nat.available(), f"no built extension under {root}"
    H = HEADS * D
    g = torch.Generator(device="cuda").manual_seed(4321)
    qkv = torch.randn(B * S, 3 * H, device="cuda", generator=g).to(torch.bfloat16)
    dctx = torch.randn(B * S, H, device="cuda", generator=g).to(torch.bfloat16)
    lens = torch.randint(48, S + 1, (B,), device="cuda", generator=g)
    mask = (torch.arange(S, device="cuda")[None, :] >= lens[:, None]).float() * -10000.0
    outs = {}
    for tag, p in (("p0", 0.0), ("p0.1", 0.1)):
        rng = nat.RngState(77) if p > 0 else None
        kw = dict(dropout_p=p, rng=rng, rng_stream=3)
        ctx, lse = nat.attention_fwd(qkv, mask, B, S, HEADS, **kw)
        outs[f"ctx_{tag}"] = ctx
        outs[f"lse_{tag}"] = lse
        outs[f"dqkv_{tag}"] = nat.attention_bwd(qkv, mask, ctx, lse, dctx, B, S, HEADS, **kw)
        # the backward alone, on a forward (ctx, lse) computed by torch, the same in every build
        ctx_t, lse_t = _torch_forward(torch, qkv, mask, ctx, S)
        outs[f"dqkv_torchfwd_{tag}"] = nat.attention_bwd(qkv, mask, ctx_t, lse_t, dctx, B, S,
                                                         HEADS, **kw)
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for k, v in outs.items():
        bits = v.contiguous().view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32)
        np.save(os.path.join(out_dir, f"{k}.npy"), bits.cpu().numpy())
        np.save(os.path.join(out_dir, f"{k}.f32.npy"), v.float().cpu().numpy())
    print(f"wrote {len(outs)} outputs to {out_dir}")


def compare(a: str, b: str) -> int:
    import numpy as np

    names = sorted(f[:-4] for f in os.listdir(a) if f.endswith(".npy") and not f.endswith(".f32.npy"))
    bad = 0
    for n in names:
        x, y = np.load(os.path.join(a, n + ".npy")), np.load(os.path.join(b, n + ".npy"))
        fx = np.load(os.path.join(a, n + ".f32.npy"))
        fy = np.load(os.path.join(b, n + ".f32.npy"))
        if x.shape != y.shape:
            print(f"{n:12s} SHAPE {x.shape} vs {y.shape}")
            bad += 1
            continue
        same = np.array_equal(x, y)
        d = np.abs(fx.astype(np.float64) - fy.astype(np.float64))
        mag = np.maximum(np.abs(fx), np.abs(fy)).astype(np.float64)
        if x.dtype == np.int16:
            # one bf16 ulp of a value v is 2^(floor(log2|v|) - 7)
            ulp = np.exp2(np.floor(np.log2(np.maximum(mag, 1e-30))) - 7)
            rel = (f"max {float(np.max(d / ulp)):.0f} bf16 ulp of the value, max |diff| / max |x| "
                   f"{float(d.max() / max(float(mag.max()), 1e-30)):.2g}")
        else:
            rel = f"max rel {float(np.max(d / np.maximum(mag, 1e-30))):.2g}"
        print(f"{n:12s} {'bit-identical' if same else 'DIFFERENT'}  elements differing "
              f"{int((x != y).sum())} of {x.size}  max |diff| {float(d.max()):.3g}  {rel}")
        bad += not same
    print("all bit-identical" if not bad else f"{bad} of {len(names)} outputs differ")
    return 1 if bad else 0


def main() -> int:
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    d.add_argument("--out", required=True)
    d.add_argument("--seq", type=int, default=128)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args.root, args.out, args.seq)
        return 0
    return compare(args.a, args.b)


if __name__ == "__main__":
    sys.exit(main())
