"""Extractive question-answering fine-tuning cost on one GPU: BERT-large, 24 blocks, 32 sequences,
one CUDA graph per step.

    python tools/bench_qa.py [--steps 10] [--rounds 5] [--layers 24] [--out FILE]

Reports, after the card's name and power limit (read in the same run):
* ms/step of training at S = 384 with the BertTailForQuestionAnswering head + QuestionAnsweringLoss
  against the pooler + classifier tail + CrossEntropyLoss at the same S, and the classification
  step at S = 128 for scale; SGD (momentum 0.9) and AdamW, medians over ``--rounds`` alternating
  windows of ``--steps`` graph replays each.  One optimizer's arms live on the card at once;
* each arm's peak memory from its construction through its warm-up;
* the four span-head kernels at B = 32, S = 384, H = 1024 from graph replays against their byte
  floors at 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth): qa_logits_fwd reads the bf16
  hidden states once (25.2 MB), qa_logits_bwd reads them and writes the input gradient (50.3 MB);
  qa_span_ce and qa_span_eval touch only the [32, 2, 384] logits (latency-bound).
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import skycomputing_b200 as sky  # noqa: E402
from skycomputing_b200.models import set_backend  # noqa: E402
from skycomputing_b200.ops import native as nat  # noqa: E402
from bench_mlm import card, graph_kernel_ms, step_window  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, H = 32, 1024


def build_runner(layers: int, qa: bool, S: int, optim: str):
    cfg = sky.BertConfig.bert_large()
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    tail = ([dict(layer_type="BertTailForQuestionAnswering", config=cfg.__dict__)] if qa else
            [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=cfg.hidden_size, num_classes=3)])
    mc = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + tail
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_bench_qa")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=0)
    optim_cfg = (dict(optim_type="SGD", lr=1e-4, momentum=0.9) if optim == "SGD" else
                 dict(optim_type=optim, lr=1e-5))
    opt = sky.build_optimizer(model.optim_module, optim_cfg)
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=1, device=torch.device("cuda", 0),
                        loss_cfg=dict(type="QuestionAnsweringLoss" if qa else "CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_bench_qa"), logging_cfg=None,
                        micro_batches=1, use_cuda_graph=True)
    model.train(True)
    if qa:
        ds = sky.SynthQADataset(num_samples=B, max_seq_length=S, vocab_size=cfg.vocab_size, seed=0)
    else:
        ds = sky.SynthMNLIDataset(num_samples=B, max_seq_length=S, seed=0)
    data, labels = next(iter(torch.utils.data.DataLoader(ds, batch_size=B)))
    return runner, [t.cuda() for t in data], labels.cuda()


def kernels() -> dict:
    S = 384
    g = torch.Generator(device="cuda").manual_seed(0)
    hidden = torch.randn(B, S, H, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(2, H, device="cuda", generator=g) * 0.02
    b = torch.zeros(2, device="cuda")
    dw, db = torch.zeros_like(w), torch.zeros_like(b)
    ds = sky.SynthQADataset(num_samples=B, max_seq_length=S, seed=0)
    labels = torch.stack([ds[i][1] for i in range(B)]).cuda()
    logits = nat.qa_logits(hidden, w, b)
    _, dl = nat.qa_span_ce(logits, labels)
    acc = nat.SpanEvalAccumulator(30, 10 ** 6, "cuda")
    res = {}
    floors = dict(qa_logits_fwd=B * S * H * 2 + B * 2 * S * 4,
                  qa_logits_bwd=2 * B * S * H * 2 + B * 2 * S * 4,
                  qa_span_ce=2 * B * 2 * S * 4, qa_span_eval=B * 2 * S * 4)
    fns = dict(qa_logits_fwd=lambda: nat.qa_logits(hidden, w, b),
               qa_logits_bwd=lambda: nat.qa_logits_bwd(hidden, dl, w, dw, db),
               qa_span_ce=lambda: nat.qa_span_ce(logits, labels),
               qa_span_eval=lambda: acc.add(logits, labels))
    for name, fn in fns.items():
        ms = graph_kernel_ms(fn)
        floor_us = floors[name] / HBM_BYTES_PER_S * 1e6
        res[name] = dict(us=ms * 1e3, bytes=floors[name], floor_us=floor_us,
                         share_of_floor=floor_us / (ms * 1e3))
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    set_backend("native")
    nat.enable_launch_counter()
    res = dict(card=card(), geometry=dict(B=B, layers=args.layers), steps=args.steps,
               rounds=args.rounds, arms={})
    print("card: {name}, power limit {power_limit}, max SM clock {max_sm_clock}".format(**res["card"]),
          flush=True)
    arms = (("qa_s384", True, 384), ("cls_s384", False, 384), ("cls_s128", False, 128))
    for optim in ("SGD", "AdamW"):
        runners, peak = {}, {}
        for name, qa, S in arms:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            runners[name] = build_runner(args.layers, qa, S, optim)
            r, x, y = runners[name]
            # past the step graph's capture (the 4th step): an engine captures while its
            # weight-gradient stream is the process-wide one
            for _ in range(5):
                r.engine.train_step(x, y)
            torch.cuda.synchronize()
            peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        times = {name: [] for name, _, _ in arms}
        for _ in range(args.rounds):
            for name, _, _ in arms:
                times[name].append(step_window(*runners[name], args.steps))
        for name, qa, S in arms:
            med = statistics.median(times[name])
            res["arms"]["{}_{}".format(name, optim)] = dict(
                ms_per_step=med, windows=times[name], peak_mib=peak[name],
                sequences_per_s=B / med * 1e3)
            print("{:>9} {:5}  {:8.2f} ms/step  {:7.1f} seq/s  peak {:8.0f} MiB".format(
                name, optim, med, B / med * 1e3, peak[name]), flush=True)
        for r, _, _ in runners.values():
            r.engine.close()
        del runners
        gc.collect()
        torch.cuda.empty_cache()
    res["kernels"] = kernels()
    for name, k in res["kernels"].items():
        print("{:>14}  {:7.2f} us  floor {:6.2f} us  ({:.0%} of the byte floor's rate)".format(
            name, k["us"], k["floor_us"], k["share_of_floor"]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
