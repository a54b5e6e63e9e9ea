"""LAMB in 2-stage pipelines over NCCL and over the fused peer-memory boundaries, with global-norm
clipping: every transport trains the same losses, and every rank computes the same global norm
(the trust ratios are per tensor and stage-local, so LAMB adds no cross-stage exchange)."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world: int, *extra) -> dict:
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "check_pipeline.py"), *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


def test_lamb_pipelines_agree_across_transports():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    common = ("--optim", "lamb", "--layers", "4", "--micro-batches", "2", "--batch", "16",
              "--max-grad-norm", "0.5", "--lr-schedule", "linear")
    runs = {"nccl": _run(2, "--boundary", "nccl", *common),
            "fused": _run(2, "--boundary", "fused", *common)}
    ref = runs["nccl"]["losses"]
    assert len(ref) == 6 and ref[-1] != ref[0]
    for name, r in runs.items():
        assert r["err_any"] == 0, name
        assert r["norms_identical"], (name, r["rank_norms"])
        assert r["losses"][0] == ref[0], name
        for a, b in zip(r["losses"], ref):
            assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (name, r["losses"], ref)
    assert runs["fused"]["fused_any"] and runs["fused"]["graph_all"]
