"""Per-kernel breakdown of the single-GPU BERT-large training step (torch.profiler, CUDA activities).

    python tools/profile_step.py [--out DIR] [--graph] [--layers 24] [--batch 32] [--steps 3] [--warmup 3]

Geometry of ``bench.py --gpus 1``: BERT-large (H=1024, A=16, I=4096), 32 x 128 tokens, dropout 0.1,
fused SGD.  The profiled steps run eagerly (the same kernels the captured step replays, without the
graph) or, with ``--graph``, as replays of the step that ``bench.py`` captures, after warm-up steps
that are not profiled.  The wall time of the same number of unprofiled steps is recorded too.  Writes ``DIR/profile_step.json``: per kernel
(template instantiation) and per kernel family the calls per step, us per call, us per step and
share of the summed kernel time, and for the four matrix-multiply kernels the FLOP per step from
the model's shapes with the achieved rate against the 989 TFLOP/s data-sheet dense BF16 rate of
the H100 SXM.  The card's name, power limit and maximum SM clock are recorded with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BF16 = 989e12   # H100 SXM data sheet, dense BF16, 700 W card
SEQ = 128


def model_flops(layers: int, batch: int, hidden=1024, inter=4096, heads=16, head_dim=64) -> dict:
    """FLOP per training step of each matrix-multiply kernel family, from the model's shapes."""
    t = batch * SEQ
    # forward: QKV and FFN1 run on the plain GEMM, the attention-output and FFN2 projections
    # (each followed by LayerNorm) on the GEMM + LayerNorm kernel; backward: dgrad and wgrad of
    # all four on the plain GEMM
    qkv, wo, ffn1, ffn2 = (2 * t * hidden * 3 * hidden, 2 * t * hidden * hidden,
                           2 * t * hidden * inter, 2 * t * inter * hidden)
    gemm = (qkv + ffn1) + 2 * (qkv + wo + ffn1 + ffn2)
    gemm_ln = wo + ffn2
    one = 2 * batch * heads * SEQ * SEQ * head_dim   # one S x S x d product, all heads
    return {"gemm_wgmma_kernel": layers * gemm, "gemm_ln_wgmma_kernel": layers * gemm_ln,
            "attention_fwd_kernel": layers * 2 * one,        # Q K^T, P V
            "attention_bwd_kernel": layers * 5 * one}        # Q K^T, dO V^T, P^T dO, dS^T Q, dS K


def short_name(name: str) -> str:
    n = name.replace("sky::", "").replace("(anonymous namespace)::", "")
    n = re.sub(r"^void ", "", n)
    return re.sub(r"\(.*$", "", n)


def family(name: str) -> str:
    return re.sub(r"<.*$", "", short_name(name))


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still worth keeping
        return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def _captured_step(sky, model_config, batch):
    """The single-GPU training step as bench.py builds it (Runner engine, one CUDA graph per
    step after its eager warm-up steps); returns a callable that runs one step."""
    import torch
    import torch.distributed as dist

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29541")
    device = torch.device("cuda", 0)
    if not dist.is_initialized():
        dist.init_process_group(backend="nccl", rank=0, world_size=1, device_id=device)
    import tempfile

    log_root = tempfile.mkdtemp(prefix="sky_profile_")
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(slowdown=0, mem_limit=-1, cuda_device=0, module_to_cuda=True,
                          output_to_cpu=False, timer_config=dict(root=log_root)))])
    wm = sky.Allocator(model_config, wm, None, None, granularity="block",
                       solver="heuristic").allocate("even", virtual_stages=1)
    model = sky.RpcModel(wm, this_rank=0)
    optimizer = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=1e-3))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=optimizer,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root=log_root), logging_cfg=None, micro_batches=1,
                        schedule="sequential", boundary="auto", use_cuda_graph=True,
                        device=device, async_loss=True)
    model.train(True)
    eng = runner.engine
    ds = sky.SynthMNLIDataset(num_samples=batch, max_seq_length=SEQ, seed=0)
    data = [t[:batch].contiguous().to(device) for t in (ds.input_ids, ds.segment_ids, ds.input_mask)]
    labels = ds.labels[:batch].contiguous().to(device)

    def step():
        return eng.train_step(data, labels)

    for _ in range(5):   # eager steps and the capture happen in here
        step()
    torch.cuda.synchronize()
    assert eng._graph is not None, "the engine did not capture the step"
    return step


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "profile"))
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--graph", action="store_true",
                    help="profile replays of the captured step (the engine bench.py times) "
                         "instead of eager steps")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import skycomputing_b200 as sky
    from skycomputing_b200.models import BertConfig, advance_rng, set_backend
    from skycomputing_b200.ops import native as nat

    if not torch.cuda.is_available() or not nat.available():
        raise RuntimeError("profile_step.py needs a CUDA device and the built native extension")
    set_backend("native")
    torch.manual_seed(0)
    cfg = BertConfig.bert_large()
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * args.layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=1024, num_classes=3)])
    B = args.batch
    if args.graph:
        step = _captured_step(sky, mc, B)
    else:
        stage = sky.build_module_from_cfg(0, mc, dict(module_to_cuda=True, cuda_device=0))
        stage._record_forward_time = False
        stage.train()
        opt = sky.build_optimizer(stage, dict(optim_type="SGD", lr=1e-3))
        loss_fn = sky.build_loss(dict(type="CrossEntropyLoss"), torch.device("cuda", 0))
        ids = torch.randint(1000, 30522, (B, SEQ), device="cuda")
        tt = torch.zeros(B, SEQ, dtype=torch.long, device="cuda")
        mask = torch.ones(B, SEQ, dtype=torch.long, device="cuda")
        labels = torch.randint(0, 3, (B,), device="cuda")

        def step():
            advance_rng()
            loss = loss_fn(stage(ids, tt, mask)[0], labels)
            loss.backward()
            opt.step()
            return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    # wall time of the same steps without the profiler (device events)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    wall_us = e0.elapsed_time(e1) * 1e3 / args.steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()

    per = defaultdict(lambda: [0, 0.0])   # instantiation -> [calls, total us]
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        dur = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if dur <= 0:
            continue
        k = short_name(ev.name)
        per[k][0] += 1
        per[k][1] += dur
    total_us = sum(v[1] for v in per.values()) / args.steps
    flops = model_flops(args.layers, B)

    def row(calls, us):
        return {"calls_per_step": calls / args.steps, "us_per_call": us / calls,
                "us_per_step": us / args.steps, "share_of_kernel_time": us / args.steps / total_us}

    kernels = {k: row(*v) for k, v in sorted(per.items(), key=lambda kv: -kv[1][1])}
    fam = defaultdict(lambda: [0, 0.0])
    for k, v in per.items():
        f = family(k)
        fam[f][0] += v[0]
        fam[f][1] += v[1]
    families = {}
    for f, v in sorted(fam.items(), key=lambda kv: -kv[1][1]):
        r = row(*v)
        if f in flops:
            r["flop_per_step"] = flops[f]
            r["tflop_per_s"] = flops[f] / (r["us_per_step"] * 1e-6) / 1e12
            r["share_of_bf16_peak"] = r["tflop_per_s"] * 1e12 / PEAK_BF16
        families[f] = r
    result = {
        "gpu": gpu_info(),
        "geometry": {"model": f"BERT-large L={args.layers}", "batch": B, "seq_len": SEQ,
                     "dropout": 0.1, "optimizer": "fused SGD", "profiled_steps": args.steps,
                     "mode": "CUDA-graph replays of the captured step" if args.graph else
                             "eager steps (same kernels as the captured step)"},
        "wall_us_per_step": wall_us,
        "kernel_us_per_step": total_us,
        "note": "shares are of the summed kernel time; the weight-gradient GEMMs run on a side "
                "stream next to the data-gradient chain, so the sum can exceed the wall time",
        "bound": "dense BF16 data-sheet rate 989 TFLOP/s (H100 SXM, 700 W) for the matrix-multiply "
                 "kernels; the others are not rated here",
        "families": families,
        "kernels": kernels,
    }
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "profile_step.json")
    with open(path, "w") as fh:
        json.dump(result, fh, indent=1)
    print(f"wall time per step: {wall_us / 1e3:.2f} ms, summed kernel time per step: "
          f"{total_us / 1e3:.2f} ms  ({path})")
    for f, r in list(families.items())[:12]:
        rate = f"  {r['tflop_per_s']:.0f} TFLOP/s" if "tflop_per_s" in r else ""
        print(f"  {f:34s} {r['calls_per_step']:6.0f} x {r['us_per_call']:8.1f} us = "
              f"{r['us_per_step'] / 1e3:7.2f} ms  {100 * r['share_of_kernel_time']:5.1f} %{rate}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
