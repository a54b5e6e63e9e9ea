"""Where does the GEMM + LayerNorm kernel lose time against the plain GEMM?

Prints the card, its power limit and how many clusters of the fused kernel the device can hold at
once (cudaOccupancyMaxActiveClusters with the kernel's real dynamic shared memory), then times, at
the BERT-large attention-output (K = 1024) and FFN2 (K = 4096) shapes for 4096 and 2048 tokens:

    fused          the GEMM + LayerNorm kernel as the training step launches it
    fused_mainloop the same launch with debug=1: main loop only, the epilogue is skipped
    gemm_alone     the plain GEMM with the same bias, dropout and residual epilogue
    gemm_mainloop  the plain GEMM with debug=1
    two_kernels    the plain GEMM, then layernorm_fwd

Each time is the median (and range) of 5 CUDA-event timings of 50 back-to-back launches replayed
from a CUDA graph, after warm-up.  One JSON line per shape; bench_out/diagnose_gemm_ln.json
collects them.
"""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from skycomputing_b200.ops import native as nat  # noqa: E402
from tools.triage_gemm import timeit  # noqa: E402

REPEATS = 5


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable ({e})"
    return dict(card=name, power_limit_and_max_sm_clock=q,
                sms=torch.cuda.get_device_properties(0).multi_processor_count)


def timed(fn):
    ts = sorted(timeit(fn, iters=50) * 1e3 for _ in range(REPEATS))
    return dict(median=round(statistics.median(ts), 2), min=round(ts[0], 2), max=round(ts[-1], 2))


def main():
    assert torch.cuda.is_available(), "diagnose_gemm_ln.py needs a GPU"
    torch.manual_seed(0)
    head = card()
    for bn in (256, 128):
        clusters, size = nat.ext().gemm_ln_max_active_clusters(1024, bn)
        head[f"N1024_bn{bn}"] = dict(max_active_clusters=clusters, ctas_per_cluster=size)
    print(json.dumps(head), flush=True)
    rows = [head]
    rng = nat.RngState(1)
    for name, M, N, K in (("attn_out 4096 tok", 4096, 1024, 1024),
                          ("ffn2 4096 tok", 4096, 1024, 4096),
                          ("attn_out 2048 tok", 2048, 1024, 1024),
                          ("ffn2 2048 tok", 2048, 1024, 4096)):
        a = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        res = torch.randn(M, N, device="cuda").bfloat16()
        bias = torch.randn(N, device="cuda")
        g, b = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
        y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ep = dict(bias=bias, dropout_p=0.1, rng=rng, rng_stream=3)
        bn = nat.ext().gemm_ln_block_n(M, N, True)

        def fused(debug=0):
            nat.gemm_ln(a, w, g, b, residual=res, block_n=bn, debug=debug, **ep)

        def gemm_alone(debug=0):
            return nat.gemm(a, w, aux=res, add_aux=True, debug=debug, **ep)

        def two_kernels():
            nat.layernorm_fwd(gemm_alone(), g, b, y=y)

        row = dict(shape=name, M=M, N=N, K=K, block_n=bn,
                   fused_in_training_step=nat.ext().gemm_ln_block_n(M, N) != 0,
                   fused_us=timed(fused), fused_mainloop_us=timed(lambda: fused(1)),
                   gemm_alone_us=timed(gemm_alone), gemm_mainloop_us=timed(lambda: gemm_alone(1)),
                   two_kernels_us=timed(two_kernels))
        row["fused_over_gemm_alone"] = round(row["fused_us"]["median"]
                                             / row["gemm_alone_us"]["median"], 3)
        row["fused_tflops"] = round(2.0 * M * N * K / row["fused_us"]["median"] / 1e6, 1)
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = os.environ.get("DIAG_OUT", "bench_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "diagnose_gemm_ln.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
