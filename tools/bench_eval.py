"""Evaluation throughput on one GPU at the BERT-large geometry of bench.py (24 blocks, S = 128).

    python tools/bench_eval.py [--batches 32 256] [--iters 20] [--rounds 5] [--out FILE]

For every batch size it reports
* evaluation sequences/s of ``PipelineEngine.eval_step`` (forward + classify_eval), eager against
  the evaluation CUDA graph;
* the forward of the model in training mode (dropout, autograd, everything saved for backward),
  in eval mode with autograd (what an evaluation ran before the inference path existed) and
  through the inference path (eval mode, no autograd: no FFN1 pre-activation copy, no
  pre-LayerNorm sums, no attention LSE), with the peak memory of each;
* the card name and power limit, read in the same run.
Times are CUDA-event medians over ``--rounds`` alternating windows of ``--iters`` calls each;
the forwards are timed call by call (see ``timed_each``).
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import skycomputing_b200 as sky  # noqa: E402
from skycomputing_b200.runner.metrics import LazyEvalAccumulator  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def build_runner(layers: int, use_graph: bool):
    cfg = sky.BertConfig.bert_large()
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=cfg.hidden_size, num_classes=3)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_bench_eval")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=1e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=1, loss_cfg=dict(type="CrossEntropyLoss"),
                      timer_cfg=dict(root="/tmp/sky_bench_eval"), logging_cfg=None,
                      micro_batches=1, use_cuda_graph=use_graph, device=torch.device("cuda", 0))


def batch(B: int, S: int = 128):
    g = torch.Generator().manual_seed(B)
    ids = torch.randint(1000, 30522, (B, S), generator=g).cuda()
    return [ids, torch.zeros_like(ids), torch.ones_like(ids)], \
        torch.randint(0, 3, (B,), generator=g).cuda()


def timed(fn, iters: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / iters


def timed_each(fn, iters: int) -> float:
    """Device time of ``fn`` per call, each call bracketed by its own events.  A forward with
    autograd leaves reference cycles (an output saved by its own node) that hold the saved
    activations until the garbage collector runs: collect between calls, outside the events."""
    pairs = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        pairs.append((e0, e1))
        gc.collect()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in pairs) * 1e-3 / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval needs a GPU"
    torch.cuda.set_device(0)
    info = card()
    runners = {False: build_runner(args.layers, False), True: build_runner(args.layers, True)}
    # both runners are built from the same seed: the same weights
    results = []
    for B in args.batches:
        inputs, labels = batch(B)
        steps = {}
        for graph, r in runners.items():
            r.model.train(False)
            acc = LazyEvalAccumulator()

            def step(r=r, acc=acc):
                r.engine.eval_step(inputs, labels, acc, micro_batches=1)
            for _ in range(3):
                step()
            steps[graph] = step
        stage = runners[False].model.local_stage

        def fwd_train():
            stage.train(True)
            with torch.enable_grad():
                stage(*inputs)

        def fwd_eval_autograd():
            stage.train(False)
            with torch.enable_grad():
                stage(*inputs)

        def fwd_infer():
            stage.train(False)
            with torch.no_grad():
                stage(*inputs)

        fwds = dict(train=fwd_train, eval_autograd=fwd_eval_autograd, inference=fwd_infer)
        peak = {}
        for name, fn in fwds.items():
            fn()
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
            gc.collect()
        t = {k: [] for k in ("eval_eager", "eval_graph", *fwds)}
        for _ in range(args.rounds):
            t["eval_eager"].append(timed(steps[False], args.iters))
            t["eval_graph"].append(timed(steps[True], args.iters))
            for name, fn in fwds.items():
                t[name].append(timed_each(fn, args.iters))
        med = {k: statistics.median(v) for k, v in t.items()}
        spread = {k: max(v) - min(v) for k, v in t.items()}
        stage.train(False)
        results.append(dict(
            batch=B, seq=128,
            eval_seq_per_s_eager=B / med["eval_eager"], eval_seq_per_s_graph=B / med["eval_graph"],
            eval_ms_eager=med["eval_eager"] * 1e3, eval_ms_graph=med["eval_graph"] * 1e3,
            forward_ms=dict((k, med[k] * 1e3) for k in fwds),
            forward_peak_gib=peak,
            spread_ms=dict((k, v * 1e3) for k, v in spread.items())))
        print(json.dumps(results[-1]), flush=True)
    graphed = runners[True].engine._eval is not None and runners[True].engine._eval["graph"] is not None
    out = dict(card=info, layers=args.layers, rounds=args.rounds, iters=args.iters,
               eval_graph_captured=graphed, results=results)
    for r in runners.values():
        r.engine.close()
    line = json.dumps(out)
    print("BENCH_EVAL " + line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
