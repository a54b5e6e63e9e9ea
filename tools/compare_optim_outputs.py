"""Bit-for-bit comparison of the fused optimizers between two builds of the project.

    python tools/compare_optim_outputs.py dump --root TREE --out DIR
    python tools/compare_optim_outputs.py compare DIR_A DIR_B

``dump`` imports the package from TREE (a source tree with a built extension) and steps
FusedSGD (plain and with momentum, both with weight decay), FusedAdam, FusedAdam (AdamW) and
FusedLamb over one encoder layer's banks at BERT-large width (H = 1024, I = 4096) plus one bank of
21 elements (a scalar tail, and an unaligned LAMB segment); each with and without a cosine
schedule plus global-norm clipping, eagerly and by replaying a captured CUDA graph; four steps on
seeded gradients.  It stores the masters, gradients, moments, bf16 shadows, step counter,
OptimScalars and LAMB trust ratios: a SHA-256 digest of each array's bytes in DIR/<case>.json and
a seeded sample of its values in DIR/<case>.npz.  ``compare`` reports, per array, whether the bits
agree and, where they do not, the largest difference over the sample.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys

H, I = 1024, 4096
STEPS = 4
GRAD_SCALE = 0.5
SAMPLE = 4096            # elements per array kept to size a difference


def _stage(torch, ParamBank):
    """One encoder layer's parameters in banks (named as in the model) plus an odd-sized bank."""
    g = torch.Generator(device="cuda").manual_seed(7)
    mod = torch.nn.Module()

    def param(name, *shape, scale=0.03):
        p = torch.nn.Parameter(torch.randn(*shape, device="cuda", generator=g) * scale)
        mod.register_parameter(name, p)
        return p

    q, k, v = (param(f"attention_self_{n}_weight", H, H) for n in ("query", "key", "value"))
    qb, kb, vb = (param(f"attention_self_{n}_bias", H) for n in ("query", "key", "value"))
    banks = [ParamBank([q, k, v]), ParamBank([qb, kb, vb], need_shadow=False),
             ParamBank([param("attention_output_dense_weight", H, H)]),
             ParamBank([param("attention_output_dense_bias", H)], need_shadow=False),
             ParamBank([param("attention_output_LayerNorm_weight", H, scale=1.0)],
                       need_shadow=False),
             ParamBank([param("attention_output_LayerNorm_bias", H)], need_shadow=False),
             ParamBank([param("intermediate_dense_weight", I, H)]),
             ParamBank([param("intermediate_dense_bias", I)], need_shadow=False),
             ParamBank([param("output_dense_weight", H, I)]),
             ParamBank([param("output_dense_bias", H)], need_shadow=False),
             ParamBank([param("odd_weight", 7, 3, scale=0.5)])]
    for i in (0, 2, 6, 8):
        banks[i].wgrad_target = True        # left un-zeroed by the optimizer (overwrite_first)
    return mod, banks


def _optimizers(optim):
    return {
        "sgd": lambda m, b: optim.FusedSGD(m, lr=0.05, weight_decay=0.01, banks=b),
        "sgd_momentum": lambda m, b: optim.FusedSGD(m, lr=0.05, momentum=0.9, weight_decay=0.01,
                                                    banks=b),
        "adam": lambda m, b: optim.FusedAdam(m, lr=1e-3, weight_decay=0.01, banks=b),
        "adamw": lambda m, b: optim.FusedAdam(m, lr=1e-3, weight_decay=0.01, decoupled=True,
                                              banks=b),
        "lamb": lambda m, b: optim.FusedLamb(m, lr=1e-3, weight_decay=0.01, banks=b),
    }


def dump(root: str, out_dir: str) -> None:
    sys.path.insert(0, os.path.abspath(root))
    import numpy as np
    import torch

    from skycomputing_b200.ops import native as nat
    from skycomputing_b200.ops.functions import ParamBank
    from skycomputing_b200.parallel import optim

    assert nat.available(), f"no built extension under {root}"
    os.makedirs(out_dir, exist_ok=True)
    sched = optim.check_lr_schedule(dict(type="cosine", warmup_steps=1, total_steps=6))
    for kind, make in _optimizers(optim).items():
        for config in ("plain", "schedule_clip"):
            for mode in ("eager", "graph"):
                mod, banks = _stage(torch, ParamBank)
                opt = make(mod, banks)
                if config == "schedule_clip":
                    opt.configure(sched, 1.0)
                gen = torch.Generator(device="cuda").manual_seed(11)
                graph = None
                for step in range(STEPS):
                    for b in opt.banks:
                        b.grad().copy_(torch.randn(b.grad().shape, device="cuda", generator=gen))
                    if mode == "eager" or step == 0:
                        opt.step(GRAD_SCALE)       # the first step builds the tables
                        continue
                    if graph is None:
                        graph = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(graph):
                            opt.step(GRAD_SCALE)
                    graph.replay()
                torch.cuda.synchronize()
                arrays = {}
                sd = opt.state_dict()
                for i, b in enumerate(opt.banks):
                    arrays[f"bank{i}_master"] = b.master()
                    arrays[f"bank{i}_grad"] = b.grad()
                    if b.need_shadow:
                        arrays[f"bank{i}_shadow"] = b.shadow()
                    for key in ("momentum", "second_moment"):
                        t = sd.get(key, [None] * len(opt.banks))[i]
                        if t is not None:
                            arrays[f"bank{i}_{key}"] = t
                if opt._step is not None:
                    arrays["step"] = opt._step
                if opt._scalars is not None:
                    arrays["scalars"] = opt._scalars
                if kind == "lamb":
                    arrays["trust_ratios"] = opt._ratios
                digests, samples = {}, {}
                for k, t in arrays.items():
                    flat = t.detach().reshape(-1)
                    raw = flat.contiguous().view(torch.uint8).cpu().numpy().tobytes()
                    digests[k] = hashlib.sha256(raw).hexdigest()
                    idx = torch.randint(0, flat.numel(), (min(SAMPLE, flat.numel()),),
                                        generator=torch.Generator().manual_seed(3))
                    samples[k] = flat[idx.to(flat.device)].double().cpu().numpy()
                with open(os.path.join(out_dir, f"{kind}_{config}_{mode}.json"), "w") as f:
                    json.dump(digests, f, indent=1, sort_keys=True)
                np.savez(os.path.join(out_dir, f"{kind}_{config}_{mode}.npz"), **samples)
                print(f"{kind}_{config}_{mode}: {len(arrays)} arrays", flush=True)


def compare(a: str, b: str) -> int:
    import numpy as np

    cases = sorted(f[:-5] for f in os.listdir(a) if f.endswith(".json"))
    bad = total = 0
    for case in cases:
        with open(os.path.join(a, case + ".json")) as f:
            x = json.load(f)
        with open(os.path.join(b, case + ".json")) as f:
            y = json.load(f)
        sx, sy = np.load(os.path.join(a, case + ".npz")), np.load(os.path.join(b, case + ".npz"))
        for k in sorted(x):
            total += 1
            if x[k] != y.get(k):
                bad += 1
                diff = (float(np.nanmax(np.abs(sx[k] - sy[k])))
                        if k in sy.files and sx[k].shape == sy[k].shape else float("nan"))
                print(f"{case:28s} {k:24s} DIFFERENT  max |diff| over a sample {diff:.3g}")
        print(f"{case:28s} {len(x)} arrays checked")
    print(f"all {total} arrays bit-identical" if not bad else f"{bad} of {total} arrays differ")
    return 1 if bad or not cases else 0


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
