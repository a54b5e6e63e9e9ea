"""Step time of LAMB against SGD and AdamW on one GPU, and the two LAMB kernels against their
byte floor.

    python tools/bench_lamb.py [--steps 20] [--reps 6] [--layers 24]

Workload = bench.py's single-GPU geometry: BERT-large (L=24, H=1024, A=16, I=4096), 32 sequences
of 128 tokens per step, dropout 0.1, whole step replayed from one CUDA graph.  Three runners are
built in the same process (SGD lr=1e-3 as in bench.py, AdamW, LAMB); after warm-up and capture
their graphs are replayed in alternating timed windows (``--reps`` windows each, ``--steps`` steps
per window, CUDA events).  Then ``lamb_moments`` and ``lamb_update`` are timed alone over many
launches and compared with the bytes each pass must move, from the segment table, over the H100
SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import skycomputing_b200 as sky  # noqa: E402
from skycomputing_b200.models import BertConfig, set_backend  # noqa: E402
from skycomputing_b200.ops import native as nat  # noqa: E402

DATASHEET_BYTES_PER_S = 3.35e12
SEQ_LEN, BATCH = 128, 32


def _card() -> dict:
    info = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=10).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def _runner(layers: int, optim_cfg: dict, log_root: str):
    cfg = BertConfig(30522, hidden_size=1024, num_hidden_layers=layers, num_attention_heads=16,
                     intermediate_size=4096)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=1024, num_classes=3)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          output_to_cpu=False, timer_config=dict(root=log_root)))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_cfg))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root=log_root), logging_cfg=None, micro_batches=1,
                        schedule="sequential", device=torch.device("cuda", 0))
    model.train(True)
    return runner, opt


def _window(eng, inputs, labels, steps: int) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        eng.train_step(inputs, labels)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def _time_launches(fn, n: int) -> float:
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def lamb_bytes(segments) -> tuple:
    """Bytes the two passes must move: moments reads p, g, m, v and writes m, v (+ the zeroed g
    unless skip_zero); update reads p, m, v and writes p (+ the bf16 shadow)."""
    b1 = sum(s["numel"] * (24 + (0 if s["skip_zero"] else 4)) for s in segments)
    b2 = sum(s["numel"] * (16 + (2 if s["shadow"] else 0)) for s in segments)
    return b1, b2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--kernel-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lamb.py needs a CUDA device")
    torch.cuda.set_device(0)
    set_backend("native")
    nat.enable_launch_counter()
    torch.manual_seed(0)
    log_root = os.environ.get("SKY_TRACE_DIR", "/tmp/sky_bench_lamb")
    ds = sky.SynthMNLIDataset(num_samples=BATCH, max_seq_length=SEQ_LEN, seed=0)
    inputs = [ds.input_ids.cuda(), ds.segment_ids.cuda(), ds.input_mask.cuda()]
    labels = ds.labels.cuda()
    arms = {
        "sgd": dict(optim_type="SGD", lr=1e-3),
        "adamw": dict(optim_type="AdamW", lr=1e-4, weight_decay=0.01),
        "lamb": dict(optim_type="LAMB", lr=1e-3, weight_decay=0.01),
    }
    runners = {}
    for name, cfg in arms.items():
        runner, opt = _runner(a.layers, cfg, log_root)
        for _ in range(5):                       # 3 eager steps, capture, one replay
            runner.engine.train_step(inputs, labels)
        torch.cuda.synchronize()
        assert runner.engine._graph is not None, "the step was not captured"
        runners[name] = (runner, opt)
    times = {name: [] for name in arms}
    names = list(arms)
    for rep in range(a.reps):
        order = names[rep % len(names):] + names[:rep % len(names)]
        for name in order:
            times[name].append(_window(runners[name][0].engine, inputs, labels, a.steps))
    med = {k: statistics.median(v) for k, v in times.items()}

    # the two LAMB kernels alone, on the LAMB runner's segment table
    opt = runners["lamb"][1]
    ext = nat.ext()
    segs, chunks, n_chunks = opt._lamb_table()
    info = opt.segments()
    for s in info:
        s["shadow"] = opt.banks[s["bank"]].need_shadow
    b1, b2 = lamb_bytes(info)
    stream = torch.cuda.current_stream().cuda_stream
    beta1, beta2 = opt.betas
    mom_ms = _time_launches(lambda: ext.lamb_moments(
        segs.data_ptr(), chunks.data_ptr(), n_chunks, beta1, beta2, float(opt.eps),
        opt._step.data_ptr(), 1.0, opt._lamb_partials.data_ptr(), stream, 0), a.kernel_iters)
    upd_ms = _time_launches(lambda: ext.lamb_update(
        segs.data_ptr(), chunks.data_ptr(), n_chunks, 0.0, beta1, beta2, float(opt.eps),
        opt._step.data_ptr(), opt._lamb_partials.data_ptr(), opt._ratios.data_ptr(), stream, 0),
        a.kernel_iters)
    n_params = sum(s["numel"] for s in info)
    floor1, floor2 = b1 / DATASHEET_BYTES_PER_S * 1e3, b2 / DATASHEET_BYTES_PER_S * 1e3
    out = dict(
        card=_card(), layers=a.layers, batch=BATCH, seq=SEQ_LEN, steps_per_window=a.steps,
        windows=a.reps,
        step_ms={k: times[k] for k in names}, median_ms=med,
        range_ms={k: [min(v), max(v)] for k, v in times.items()},
        lamb_minus_sgd_ms=med["lamb"] - med["sgd"], lamb_minus_adamw_ms=med["lamb"] - med["adamw"],
        launches_per_step={k: runners[k][0].engine.launches_per_step for k in names},
        params=n_params, segments=len(info), chunks=n_chunks, chunk_elems=ext.LAMB_CHUNK,
        moments_bytes=b1, update_bytes=b2, bytes_per_param=(b1 + b2) / n_params,
        moments_ms=mom_ms, update_ms=upd_ms,
        moments_floor_ms=floor1, update_floor_ms=floor2,
        moments_share_of_datasheet_bw=floor1 / mom_ms, update_share_of_datasheet_bw=floor2 / upd_ms)
    print("LAMB " + json.dumps(out), flush=True)
    for runner, _ in runners.values():
        runner.engine.close()


if __name__ == "__main__":
    main()
