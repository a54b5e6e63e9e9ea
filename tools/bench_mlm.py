"""Masked-language-model pretraining cost on one GPU, at the geometry of ``bench.py --gpus 1``
(BERT-large, 24 blocks, 32 sequences of 128 tokens, one CUDA graph per step).

    python tools/bench_mlm.py [--steps 20] [--rounds 5] [--layers 24] [--max-predictions P]
                              [--out FILE]

Reports, after the card's name and power limit (read in the same run):
* ms/step of training with the BertTailForMaskedLM head + MaskedLMLoss against the pooler +
  classifier tail + CrossEntropyLoss, medians over ``--rounds`` alternating windows of
  ``--steps`` graph replays each (both models live on the card at once);
* the vocab_ce kernel (training mode, 4096 x 30528 bf16 logits) against its byte floor: read and
  write 2 x M x V bf16 at 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth).  The kernel does
  not read rows whose label is ignore_index, so with the 15 % MLM labelling it moves less than
  that floor; both label densities are timed;
* the decoder GEMM ([4096, 1024] x [30528, 1024]^T + bias, bf16 out) in TFLOP/s.
With ``--max-predictions P`` the sparse head (``BertTailForMaskedLM(max_predictions=P)``, only the
labelled positions decoded) joins the alternating windows as a third arm, each arm's peak memory
(weights, optimizer state, activations and graph pool, measured from its construction through its
warm-up) is reported, and the mlm_gather / mlm_scatter kernels are timed against their byte
floors at the benchmark's geometry with the dataset's 15 % labelling (graph replays: the
wrappers' host time exceeds these kernels' device time).
Kernel times are CUDA-event means over 50 launches after 5 warm-up launches.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import skycomputing_b200 as sky  # noqa: E402
from skycomputing_b200.models import set_backend  # noqa: E402
from skycomputing_b200.ops import native as nat  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, S, V = 32, 128, 30528


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def build_runner(layers: int, mlm: bool, max_predictions=None):
    cfg = sky.BertConfig.bert_large()
    if mlm:
        cfg.vocab_size = V
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    head = dict(layer_type="BertTailForMaskedLM", config=cfg.__dict__)
    if max_predictions is not None:
        head["max_predictions"] = max_predictions
    tail = ([head] if mlm else
            [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=cfg.hidden_size, num_classes=3)])
    mc = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + tail
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_bench_mlm")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=1e-4, momentum=0.9))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=1, device=torch.device("cuda", 0),
                        loss_cfg=dict(type="MaskedLMLoss" if mlm else "CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_bench_mlm"), logging_cfg=None,
                        micro_batches=1, use_cuda_graph=True)
    model.train(True)
    if mlm:
        ds = sky.SynthMLMDataset(num_samples=B, max_seq_length=S, vocab_size=V, seed=0)
    else:
        ds = sky.SynthMNLIDataset(num_samples=B, max_seq_length=S, seed=0)
    data, labels = next(iter(torch.utils.data.DataLoader(ds, batch_size=B)))
    inputs = [t.cuda() for t in data]
    labels = labels.cuda()
    return runner, inputs, labels


def step_window(runner, inputs, labels, steps: int) -> float:
    eng = runner.engine
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        eng.train_step(inputs, labels)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_ms(fn, iters: int = 50, warmup: int = 5) -> float:
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def graph_kernel_ms(fn, iters: int = 50, replays: int = 20) -> float:
    """Device time of a call whose host side (allocations, argument checks) takes longer than its
    kernel: ``iters`` calls captured in one CUDA graph, mean over ``replays`` replays."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / (replays * iters)


def slot_kernels(P: int) -> dict:
    """mlm_gather / mlm_scatter at the benchmark's geometry against their byte floors."""
    H = 1024
    ds = sky.SynthMLMDataset(num_samples=B, max_seq_length=S, vocab_size=V, seed=0)
    _, labels = next(iter(torch.utils.data.DataLoader(ds, batch_size=B)))
    labels = labels.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    hidden = torch.randn(B * S, H, generator=g, device="cuda").to(torch.bfloat16)
    x_c, slot_of_row, _ = nat.mlm_gather(hidden, labels, P, V)
    dx_c = torch.randn(B * P, H, generator=g, device="cuda").to(torch.bfloat16)
    decoded = min(int((labels != -100).sum()), B * P)
    # gather: labels read, the decoded rows read, the slots written, the two maps written
    gather_bytes = B * S * 8 + decoded * H * 2 + B * P * H * 2 + B * S * 4 + B * P * 8
    # scatter: the slot map read, the decoded slots read, every row of dhidden written
    scatter_bytes = B * S * 4 + decoded * H * 2 + B * S * H * 2
    out = {}
    for name, fn, nbytes in (
            ("mlm_gather", lambda: nat.mlm_gather(hidden, labels, P, V), gather_bytes),
            ("mlm_scatter", lambda: nat.mlm_scatter(dx_c, slot_of_row), scatter_bytes)):
        t = graph_kernel_ms(fn)
        floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
        out[name] = dict(ms=t, bytes=nbytes, byte_floor_ms=floor_ms, floor_over_time=floor_ms / t)
        print("{} B={} S={} H={} P={}: {:.1f} us, byte floor {:.2f} us ({:.2f} of the floor's "
              "time)".format(name, B, S, H, P, t * 1e3, floor_ms * 1e3, floor_ms / t), flush=True)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--max-predictions", type=int, default=None)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not (torch.cuda.is_available() and nat.available()):
        raise SystemExit("bench_mlm needs a GPU and the native extension")
    torch.cuda.set_device(0)
    set_backend("native")
    res = dict(card=card())
    print("card: {name}, power limit {power_limit}, max SM clock {max_sm_clock}".format(**res["card"]),
          flush=True)

    # --- whole steps, alternating windows ---
    P = args.max_predictions
    runs, peak_mib = {}, {}
    for name in ("cls", "mlm") + (("mlm_sparse",) if P else ()):
        if P:
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
        runs[name] = build_runner(args.layers, name != "cls", P if name == "mlm_sparse" else None)
        runner, inputs, labels = runs[name]
        for _ in range(args.warmup):
            runner.engine.train_step(inputs, labels)
        torch.cuda.synchronize()
        assert runner.engine._graph is not None, name
        if P:
            peak_mib[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    times = {name: [] for name in runs}
    for _ in range(args.rounds):
        for name, (runner, inputs, labels) in runs.items():
            times[name].append(step_window(runner, inputs, labels, args.steps))
    loss = {name: float(r[0].engine.train_step(r[1], r[2])) for name, r in runs.items()}
    for runner, _, _ in runs.values():
        runner.engine.close()
    del runs
    torch.cuda.empty_cache()
    steps = {name: dict(median_ms=statistics.median(t), windows_ms=t) for name, t in times.items()}
    steps["mlm_over_cls"] = steps["mlm"]["median_ms"] / steps["cls"]["median_ms"]
    res["step"] = dict(steps, loss=loss, layers=args.layers, batch=B, seq=S)
    print("step ms (median of {} windows x {} steps): cls {:.3f}, mlm {:.3f} ({:.2f}x)".format(
        args.rounds, args.steps, steps["cls"]["median_ms"], steps["mlm"]["median_ms"],
        steps["mlm_over_cls"]), flush=True)
    if P:
        steps["mlm_sparse_over_cls"] = steps["mlm_sparse"]["median_ms"] / steps["cls"]["median_ms"]
        res["step"].update(mlm_sparse_over_cls=steps["mlm_sparse_over_cls"], max_predictions=P)
        res["peak_mib"] = peak_mib
        print("sparse head (P = {}): mlm_sparse {:.3f} ms ({:.2f}x), {:.3f} ms less than the dense "
              "head".format(P, steps["mlm_sparse"]["median_ms"], steps["mlm_sparse_over_cls"],
                            steps["mlm"]["median_ms"] - steps["mlm_sparse"]["median_ms"]), flush=True)
        print("peak MiB: " + ", ".join("{} {:.0f}".format(k, v) for k, v in peak_mib.items()),
              flush=True)
        res["mlm_slots"] = slot_kernels(P)

    # --- vocab_ce kernel ---
    M = B * S
    floor_ms = 2 * M * V * 2 / HBM_BYTES_PER_S * 1e3
    g = torch.Generator(device="cuda").manual_seed(0)
    logits = (torch.randn(M, V, generator=g, device="cuda") * 2).to(torch.bfloat16)
    acc = torch.zeros(1, device="cuda")
    res["vocab_ce"] = dict(M=M, V=V, byte_floor_ms=floor_ms)
    for frac in (0.15, 1.0):
        labels = torch.randint(0, V, (M,), generator=g, device="cuda")
        labels[torch.rand(M, generator=g, device="cuda") >= frac] = -100
        rows = int((labels != -100).sum())
        t = kernel_ms(lambda: nat.vocab_ce(logits, labels, loss_acc=acc, in_place=True))
        moved = (rows * V * 2 + M * V * 2) / (t * 1e-3)    # labelled rows read, every row written
        res["vocab_ce"]["labelled_{:.2f}".format(frac)] = dict(
            ms=t, labelled_rows=rows, floor_over_time=floor_ms / t, moved_bytes_per_s=moved)
        print("vocab_ce M={} V={} labelled {:.0%}: {:.1f} us, byte floor {:.1f} us ({:.2f} of "
              "the floor's time), {:.2f} TB/s moved".format(M, V, frac, t * 1e3, floor_ms * 1e3,
                                                            floor_ms / t, moved / 1e12), flush=True)

    # --- decoder GEMM ---
    H = 1024
    y = (torch.randn(M, H, generator=g, device="cuda")).to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    bias = torch.zeros(V, device="cuda")
    out = torch.empty(M, V, dtype=torch.bfloat16, device="cuda")
    t = kernel_ms(lambda: nat.gemm(y, w, bias=bias, out=out))
    tflops = 2.0 * M * V * H / (t * 1e-3) / 1e12
    res["decoder_gemm"] = dict(M=M, N=V, K=H, ms=t, tflops=tflops)
    print("decoder GEMM {}x{}x{}: {:.1f} us, {:.0f} TFLOP/s".format(M, V, H, t * 1e3, tflops),
          flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
