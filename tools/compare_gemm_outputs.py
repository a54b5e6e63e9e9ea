"""Bit-for-bit comparison of the GEMM epilogues between two builds of the project.

    python tools/compare_gemm_outputs.py dump --root TREE --out DIR
    python tools/compare_gemm_outputs.py compare DIR_A DIR_B

``dump`` imports the package from TREE (a source tree with a built extension), runs every GEMM the
BERT-large training step issues at its shapes (32 x 128 tokens) on seeded inputs, plus the
dropout, tanh / fp32 and ragged variants, the GEMM + LayerNorm kernel (y, z, mean and rstd at
K = 1024 and 4096, with and without dropout, at BLOCK_N = 256 and 128) and the opt-in schedules
(CTA pairs, 4-CTA clusters, stream-K) with a bf16 epilogue and with fp32 accumulation, and stores
each output's raw bits as DIR/<name>.npy.  ``compare`` reports, per output, whether the bits agree
and the largest difference.
"""
from __future__ import annotations

import argparse
import os
import sys


def dump(root: str, out_dir: str) -> None:
    sys.path.insert(0, os.path.abspath(root))
    import numpy as np
    import torch

    from skycomputing_b200.ops import native as nat

    assert nat.available(), f"no built extension under {root}"
    T, H, I = 4096, 1024, 4096
    g = torch.Generator(device="cuda").manual_seed(1234)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)

    x, x1 = rnd(T, H), rnd(T, H)
    inter = rnd(T, I)
    wqkv, wo = rnd(3 * H, H, scale=0.03), rnd(H, H, scale=0.03)
    w1, w2 = rnd(I, H, scale=0.03), rnd(H, I, scale=0.03)
    bqkv, b1, bo = (torch.randn(n, device="cuda", generator=g) * 0.1 for n in (3 * H, I, H))
    g2, dqkv, dh = rnd(T, H), rnd(T, 3 * H), rnd(T, I)
    rng = nat.RngState(99)
    outs = {}
    outs["qkv_fwd"] = nat.gemm(x, wqkv, bias=bqkv)
    pre = torch.empty(T, I, dtype=torch.bfloat16, device="cuda")
    outs["ffn1_fwd"] = nat.gemm(x, w1, bias=b1, act=nat.ACT_GELU, out2=pre)
    outs["ffn1_pre"] = pre
    outs["ffn2_dgrad_dgelu"] = nat.gemm(g2, w2, b_mn=True, aux=inter, act=nat.ACT_DGELU_MUL_AUX)
    outs["ffn1_dgrad_res"] = nat.gemm(dh, w1, b_mn=True, aux=x1, add_aux=True)
    outs["wo_dgrad"] = nat.gemm(g2, wo, b_mn=True)
    outs["qkv_dgrad_res"] = nat.gemm(dqkv, wqkv, b_mn=True, aux=x1, add_aux=True)
    outs["wo_dense_dropout_res"] = nat.gemm(x, wo, bias=bo, aux=x1, add_aux=True, dropout_p=0.1,
                                            rng=rng, rng_stream=3)
    for name, (dy, act) in {"wqkv": (dqkv, x), "wo": (g2, x), "w1": (dh, x), "w2": (g2, inter)}.items():
        dw = nat.gemm(dy, act, a_mn=True, b_mn=True, out_dtype=torch.float32)
        outs[f"{name}_wgrad"] = dw.clone()
        nat.gemm(dy, act, a_mn=True, b_mn=True, out=dw, accumulate=True)
        outs[f"{name}_wgrad_acc"] = dw
    for name, kw in {"pair1": dict(pair=1), "pair2": dict(pair=2),
                     "streamk": dict(pair=0, stream_k=1)}.items():
        outs[f"qkv_fwd_{name}"] = nat.gemm(x, wqkv, bias=bqkv, **kw)
        dw = outs["w1_wgrad"].clone()
        nat.gemm(dh, x, a_mn=True, b_mn=True, out=dw, accumulate=True, **kw)
        outs[f"w1_wgrad_acc_{name}"] = dw
    gamma = 1 + 0.1 * torch.randn(H, device="cuda", generator=g)
    beta = 0.1 * torch.randn(H, device="cuda", generator=g)
    for k, (a_in, w) in {1024: (x, wo), 4096: (inter, w2)}.items():
        for p in (0.0, 0.1):
            for bn in (256, 128):
                res = nat.gemm_ln(a_in, w, gamma, beta, bias=bo, residual=x1, dropout_p=p, rng=rng,
                                  rng_stream=5, block_n=bn)
                tag = f"ln_k{k}{'_dropout' if p else ''}_bn{bn}"
                outs.update({f"{tag}_{n}": v for n, v in zip(("y", "z", "mean", "rstd"), res)})
    outs["pooler_tanh_f32"] = nat.gemm(x[:32], wo, bias=bo, act=nat.ACT_TANH, out_dtype=torch.float32)
    outs["ragged_gelu"] = nat.gemm(x[:4000], w1[:1000], bias=b1[:1000], act=nat.ACT_GELU)
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
        same = x.shape == y.shape and np.array_equal(x, y)
        fx = np.load(os.path.join(a, n + ".f32.npy"))
        fy = np.load(os.path.join(b, n + ".f32.npy"))
        diff = float(np.nanmax(np.abs(fx - fy))) if fx.shape == fy.shape else float("nan")
        ndiff = int((x != y).sum()) if x.shape == y.shape else -1
        print(f"{n:28s} {'bit-identical' if same else 'DIFFERENT'}  elements differing {ndiff}"
              f"  max |diff| {diff:.3g}")
        bad += not same
    print("all bit-identical" if not bad else f"{bad} of {len(names)} outputs differ")
    return 1 if bad else 0


def main() -> int:
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    d.add_argument("--out", required=True)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args.root, args.out)
        return 0
    return compare(args.a, args.b)


if __name__ == "__main__":
    sys.exit(main())
