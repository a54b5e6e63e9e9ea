"""Cost of global-norm gradient clipping + a learning-rate schedule on one GPU.

    python tools/bench_grad_clip.py [--steps 20] [--reps 6] [--layers 24]

Workload = bench.py's single-GPU geometry: BERT-large (L=24, H=1024, A=16, I=4096), 32 sequences
of 128 tokens per step, SGD lr=1e-3, dropout 0.1, whole step replayed from one CUDA graph.  Two
runners are built in the same process, one plain and one with ``grad_clip=dict(max_norm=1.0)``
and a linear warmup / decay schedule; after warm-up and capture their graphs are replayed in
alternating timed windows (``--reps`` windows each, ``--steps`` steps per window, CUDA events).
Then ``grad_sumsq_multi`` (the extra pass over the gradients) and ``optim_finalize`` are timed
alone over many launches, and the sum-of-squares pass is compared with the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s) for the 4 bytes per parameter it reads.  Prints one JSON line.
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


def _runner(layers: int, step_cfg: dict, log_root: str):
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
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=1e-3), **step_cfg)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--kernel-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grad_clip.py needs a CUDA device")
    torch.cuda.set_device(0)
    set_backend("native")
    nat.enable_launch_counter()
    torch.manual_seed(0)
    log_root = os.environ.get("SKY_TRACE_DIR", "/tmp/sky_bench_grad_clip")
    ds = sky.SynthMNLIDataset(num_samples=BATCH, max_seq_length=SEQ_LEN, seed=0)
    inputs = [ds.input_ids.cuda(), ds.segment_ids.cuda(), ds.input_mask.cuda()]
    labels = ds.labels.cuda()
    total = a.reps * a.steps + 10
    modes = {
        "off": dict(),
        "on": dict(grad_clip=dict(max_norm=1.0),
                   lr_schedule=dict(type="linear", warmup_steps=total // 10, total_steps=total)),
    }
    runners = {}
    for name, cfg in modes.items():
        runner, opt = _runner(a.layers, cfg, log_root)
        for _ in range(5):                       # 3 eager steps, capture, one replay
            runner.engine.train_step(inputs, labels)
        torch.cuda.synchronize()
        assert runner.engine._graph is not None, "the step was not captured"
        runners[name] = (runner, opt)
    times = {name: [] for name in modes}
    for rep in range(a.reps):
        order = ("off", "on") if rep % 2 == 0 else ("on", "off")
        for name in order:
            times[name].append(_window(runners[name][0].engine, inputs, labels, a.steps))
    med = {k: statistics.median(v) for k, v in times.items()}
    diffs = [b - o for o, b in zip(times["off"], times["on"])]

    # the two extra kernels alone, on the clipping optimizer's banks
    opt = runners["on"][1]
    ext = nat.ext()
    d = opt._descriptors()
    n_params = sum(b.master().numel() for b in opt.banks)
    stream = torch.cuda.current_stream().cuda_stream
    sumsq_ms = _time_launches(lambda: ext.grad_sumsq_multi(
        d.data_ptr(), len(opt.banks), opt._sumsq_blocks, 1.0, opt._partials.data_ptr(), stream),
        a.kernel_iters)
    fin_ms = _time_launches(lambda: ext.optim_finalize(
        opt._partials.data_ptr(), opt._partials.numel(), 0, max_norm=1.0,
        out=opt._scalars.data_ptr(), stream=stream), a.kernel_iters)
    nbytes = 4 * n_params
    out = dict(
        card=_card(), layers=a.layers, batch=BATCH, seq=SEQ_LEN, steps_per_window=a.steps,
        windows=a.reps,
        step_ms_off=times["off"], step_ms_on=times["on"],
        median_ms_off=med["off"], median_ms_on=med["on"],
        overhead_ms_median=statistics.median(diffs), overhead_ms_min=min(diffs),
        overhead_ms_max=max(diffs),
        launches_per_step_off=runners["off"][0].engine.launches_per_step,
        launches_per_step_on=runners["on"][0].engine.launches_per_step,
        params=n_params, sumsq_bytes=nbytes, sumsq_ms=sumsq_ms,
        sumsq_bytes_per_s=nbytes / (sumsq_ms * 1e-3),
        sumsq_share_of_datasheet_bw=(nbytes / DATASHEET_BYTES_PER_S) / (sumsq_ms * 1e-3),
        sumsq_partials=opt._partials.numel(), finalize_ms=fin_ms)
    print("GRADCLIP " + json.dumps(out), flush=True)
    for runner, _ in runners.values():
        runner.engine.close()


if __name__ == "__main__":
    main()
