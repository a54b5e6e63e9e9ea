"""A decoder tied to the word embeddings across a 2-GPU pipeline (needs >= 2 GPUs, skipped
otherwise): the table on the first rank, a replica on the last.  Plain 1F1B and looped engines
(the head in the last chunk of the last rank), fused boundaries (peer-memory exchange of the
summed gradient inside the captured step) and torch.distributed p2p boundaries (one all_reduce over
the two ranks), dense and sparse head, with and without clipping, SGD and LAMB: the tied N-GPU
losses (and clipping norms) match one GPU, the checksums of both copies are identical after every
step, and the boundary error word stays 0."""
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
           os.path.join(ROOT, "tools", "check_mlm_pipeline.py"), "--tie", *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


_SINGLE: dict = {}


def _single(*extra) -> dict:
    """The 1-GPU run with the same optimizer / head / clipping (a pipeline layout does not apply)."""
    if extra not in _SINGLE:
        _SINGLE[extra] = _run(1, *extra)
    return _SINGLE[extra]


CASES = [
    # (engine / cut, boundary, exchange, extra arguments)
    ("blocks", "auto", "peer", ()),
    ("blocks", "nccl", "all_reduce", ()),
    ("head", "auto", "all_reduce", ()),
    ("blocks", "auto", "peer", ("--max-predictions", "20")),
    ("head", "auto", "all_reduce", ("--max-predictions", "20")),
    ("blocks", "auto", "peer", ("--max-grad-norm", "0.5")),
    ("blocks", "nccl", "all_reduce", ("--max-grad-norm", "0.5")),
    ("looped", "auto", "peer", ()),
    ("looped", "nccl", "all_reduce", ()),
    ("looped", "auto", "peer", ("--max-grad-norm", "0.5")),
]


@pytest.mark.skipif(N_GPU < 2, reason="needs two GPUs")
@pytest.mark.parametrize("optim", ["SGD", "LAMB"])
@pytest.mark.parametrize("cut,boundary,exchange,extra", CASES)
def test_tied_two_gpu_pipeline(cut, boundary, exchange, extra, optim):
    common = ("--optim", optim) + tuple(extra)
    layout = ("--virtual-stages", "2") if cut == "looped" else ("--cut", cut)
    two = _run(2, "--boundary", boundary, *layout, *common)
    one = _single(*common)
    assert two["err_any"] == 0
    assert two["tied_exchange"] == exchange
    assert two["engine"] == ("LoopedPipelineEngine" if cut == "looped" else "PipelineEngine")
    if exchange == "peer":
        assert two["fused_any"] and two["graph_all"]
    first, last = two["tied_checksums"]
    assert len(first) == len(last) == 6 and first == last        # bit-identical copies
    assert two["losses"][0] == one["losses"][0]
    for a, b in zip(two["losses"], one["losses"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (cut, two["losses"], one["losses"])
    if "--max-grad-norm" in extra:
        # the norm counts the table once: the replica is left out of the last rank's share
        assert two["grad_norms"][0] == pytest.approx(one["grad_norms"][0], rel=1e-3)
        for a, b in zip(two["grad_norms"], one["grad_norms"]):
            assert a == pytest.approx(b, rel=3e-2)
