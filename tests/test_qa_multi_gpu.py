"""The question-answering head across a 2-GPU pipeline (needs >= 2 GPUs, skipped otherwise),
through ``tools/check_mlm_pipeline.py --qa`` at S = 384: the cut between blocks (fused boundary,
CUDA graph) or directly in front of the head.  The losses match one GPU and the boundary error
word stays 0."""
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
           os.path.join(ROOT, "tools", "check_mlm_pipeline.py"), "--qa", *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


@pytest.mark.skipif(N_GPU < 2, reason="needs two GPUs")
@pytest.mark.parametrize("cut", ["blocks", "head"])
def test_qa_two_gpu_pipeline(cut):
    two = _run(2, "--cut", cut)
    one = _run(1)
    assert two["err_any"] == 0
    if cut == "blocks":
        assert two["fused_any"] and two["graph_all"]
    else:
        assert two["last_stage_first_layer"] == "BertTailForQuestionAnswering"
    assert len(two["losses"]) == len(one["losses"]) == 6
    assert two["losses"][0] == pytest.approx(one["losses"][0], rel=1e-5)
    for a, b in zip(two["losses"], one["losses"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (two["losses"], one["losses"])
