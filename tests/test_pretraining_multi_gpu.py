"""The pretraining head (masked-LM + next-sentence) across a 2-GPU pipeline (needs >= 2 GPUs,
skipped otherwise), through ``tools/check_mlm_pipeline.py --nsp``: plain 1F1B and looped engines,
fused (peer-memory) and NCCL boundaries, dense and sparse head, tied and untied decoder.  The
losses match one GPU, a tied decoder's two copies stay bit-identical every step, and the boundary
error word stays 0."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_GPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world: int, *extra) -> dict:
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "check_mlm_pipeline.py"), "--nsp", *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


_SINGLE: dict = {}


def _single(*extra) -> dict:
    if extra not in _SINGLE:
        _SINGLE[extra] = _run(1, *extra)
    return _SINGLE[extra]


@pytest.mark.skipif(N_GPU < 2, reason="needs two GPUs")
@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("boundary", ["auto", "nccl"])
@pytest.mark.parametrize("engine", ["plain", "looped"])
def test_pretraining_two_gpu_pipeline(engine, boundary, sparse, tie):
    common = (("--max-predictions", "20") if sparse else ()) + (("--tie",) if tie else ())
    layout = ("--virtual-stages", "2") if engine == "looped" else ("--cut", "blocks")
    two = _run(2, "--boundary", boundary, *layout, *common)
    one = _single(*common)
    assert two["err_any"] == 0
    assert two["engine"] == ("LoopedPipelineEngine" if engine == "looped" else "PipelineEngine")
    if boundary == "auto":
        assert two["fused_any"] and two["graph_all"]
    if tie:
        first, last = two["tied_checksums"]
        assert len(first) == len(last) == 6 and first == last
    assert len(two["losses"]) == len(one["losses"]) == 6
    assert two["losses"][0] == pytest.approx(one["losses"][0], rel=1e-5)
    for a, b in zip(two["losses"], one["losses"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (two["losses"], one["losses"])
