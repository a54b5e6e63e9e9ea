"""The sparse masked-language-model head (max_predictions = 20) as a 2-GPU pipeline (needs >= 2
GPUs, skipped otherwise): the labels reach the head on the last stage, with the cut between two
blocks (fused peer-memory boundary, one CUDA graph per step) or directly in front of the head
(torch.distributed p2p).  Against the 1-GPU run with the same sparse head, seeds and data, at the
tolerance of tests/test_mlm_multi_gpu.py."""
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
           os.path.join(ROOT, "tools", "check_mlm_pipeline.py"), "--max-predictions", "20", *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


@pytest.fixture(scope="module")
def single():
    if N_GPU < 2:
        pytest.skip("needs two GPUs")
    return _run(1)


@pytest.mark.skipif(N_GPU < 2, reason="needs two GPUs")
@pytest.mark.parametrize("cut", ["blocks", "head"])
def test_two_gpu_sparse_mlm_pipeline_matches_single_gpu(single, cut):
    two = _run(2, "--cut", cut)
    assert two["err_any"] == 0
    if cut == "blocks":
        assert two["fused_any"] and two["graph_all"] and two["layers"] == [7, 7]
    else:
        assert sorted(two["layers"]) == [1, 13]
        assert two["last_stage_first_layer"] == "BertTailForMaskedLM"
    assert len(single["losses"]) == len(two["losses"]) == 6
    assert two["losses"][0] == single["losses"][0]            # bit for bit
    for a, b in zip(two["losses"], single["losses"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (cut, two["losses"], single["losses"])
