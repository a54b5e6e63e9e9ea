"""The whole-step CUDA-graph driver that both pipeline engines share (EngineBase._run_graphed),
driven on CPU: CUDAGraph, graph capture, synchronize and the native launch counter are replaced by
recorders, the stages and the optimizer by fakes, and the engines run their real step bodies."""
import contextlib

import pytest
import torch

from skycomputing_b200.ops import native as nat
from skycomputing_b200.parallel.pipeline import PipelineEngine
from skycomputing_b200.parallel.pipeline_looped import LoopedPipelineEngine


class _Stage(torch.nn.Module):
    def __init__(self, log):
        super().__init__()
        self.log = log
        self.w = torch.nn.Parameter(torch.ones(()))

    def forward(self, *args):
        self.log.append("F")
        return (args[0].float() * self.w, args[-1])

    def begin_backward(self):
        pass

    def end_backward(self):
        pass

    def spans(self):
        return []

    def suspend_forward_probes(self):
        return contextlib.nullcontext()


class _Opt:
    graph_safe = True

    def __init__(self, log):
        self.log = log

    def step(self):
        self.log.append("opt")


@pytest.fixture
def fake_cuda(monkeypatch):
    """Recorders for everything the driver asks of CUDA; each forward counts as one launch."""
    log = []

    class Graph:
        def replay(self):
            log.append("replay")

    @contextlib.contextmanager
    def capture(g):
        assert isinstance(g, Graph)
        log.append("capture")
        yield
        log.append("capture_end")

    monkeypatch.setattr(torch.cuda, "CUDAGraph", Graph)
    monkeypatch.setattr(torch.cuda, "graph", capture)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: log.append("sync"))
    monkeypatch.setattr(nat, "launch_count", lambda: log.count("F"))
    return log


def _loss(out, lab):
    return (out.sum(-1) - lab).pow(2).mean()


def _spy_body(eng, log, name="_step_body"):
    """Record every body call with the tensors it was given (identity and values)."""
    body = getattr(eng, name)

    def spy(inputs, labels, *rest):
        log.append(("body", inputs, labels,
                    [t.clone() for t in inputs or ()], None if labels is None else labels.clone()))
        return body(inputs, labels, *rest)

    setattr(eng, name, spy)


def _plain(log, graph=True):
    eng = PipelineEngine(_Stage(log), 0, 1, [0], torch.device("cpu"), _Opt(log), loss_fn=_loss,
                         micro_batches=2, advance_rng=False)
    if graph:   # what a single native GPU would report; setup then decides to capture
        eng._native_active = lambda: True
        eng._want_graph = True
        eng._wgrad_mode = "inline"
    return eng


class _Chan:
    def send_mask(self, mask, slot):
        pass


class _Fused:
    prev, next = _Chan(), _Chan()

    def begin_step(self):
        pass

    def end_of_backward(self):
        pass


def _looped(log, pos, graph=True):
    """Ring position ``pos`` of a 2 x 2 looped pipeline on the fused ring, set up by hand."""
    P, v = 2, 2
    eng = LoopedPipelineEngine([_Stage(log) for _ in range(v)], [c * P + pos for c in range(v)],
                               P, [0, 1], torch.device("cpu"), _Opt(log), loss_fn=_loss,
                               micro_batches=2, advance_rng=False)
    eng.fused, eng.in_fused, eng.out_fused = _Fused(), True, True
    eng._fused_inputs = lambda slot: (torch.ones(2, 3, requires_grad=True), torch.zeros(2))
    eng._setup = lambda inputs: setattr(eng, "_setup_done", True)
    eng.graphable = graph
    return eng


def _engines(log, graph=True):
    """(engine, feeds inputs, feeds labels) for both engines; the looped engine at the ring
    position that reads the data and at the one that computes the loss."""
    return [(_plain(log, graph), True, True), (_looped(log, 0, graph), True, False),
            (_looped(log, 1, graph), False, True)]


def _batch(k):
    return [torch.full((4, 3), float(k))], torch.full((4,), float(k))


@pytest.mark.parametrize("which", range(3))
def test_three_eager_steps_then_one_capture_then_replays(fake_cuda, which):
    log = fake_cuda
    eng, first, last = _engines(log)[which]
    _spy_body(eng, log)
    for k in range(1, 7):
        log.clear()
        inputs, labels = _batch(k)
        ret = eng.train_step(inputs if first else None, labels if last else None)
        assert (ret is eng._loss_acc) if last else ret is None
        calls = [e for e in log if isinstance(e, tuple)]
        if k <= 3:
            # eager, on the static buffers, into which this call's batch was copied first
            assert eng.graphable and eng._graph is None and len(calls) == 1
            _, got_in, got_lab, vals_in, val_lab = calls[0]
            assert got_in is eng._static_inputs and got_lab is eng._static_labels
            if first:
                assert len(vals_in) == 1 and torch.equal(vals_in[0], inputs[0])
            else:
                assert vals_in == []
            if last:
                assert torch.equal(val_lab, labels)
            else:
                assert val_lab is None
            assert "opt" in log and "replay" not in log and "capture" not in log
        elif k == 4:
            # capture once, count its launches, replay right away
            names = [e if isinstance(e, str) else e[0] for e in log if e != "F" and e != "opt"]
            assert names == ["sync", "capture", "body", "capture_end", "replay"]
            assert calls[0][1] is eng._static_inputs and calls[0][2] is eng._static_labels
            assert eng._graph is not None and eng.launches_per_step == log.count("F") > 0
            if first:
                assert torch.equal(eng._static_inputs[0], inputs[0])
            if last:
                assert torch.equal(eng._static_labels, labels)
        else:
            assert log == ["replay"]
            if first:    # the replay reads this step's batch
                assert torch.equal(eng._static_inputs[0], inputs[0])
            if last:
                assert torch.equal(eng._static_labels, labels)
    assert eng._step["eager"] == 3


@pytest.mark.parametrize("which", range(3))
def test_an_engine_that_cannot_capture_runs_the_body_every_step(fake_cuda, which):
    log = fake_cuda
    eng, first, last = _engines(log, graph=False)[which]
    _spy_body(eng, log)
    for k in range(1, 6):
        log.clear()
        inputs, labels = _batch(k)
        inputs, labels = (inputs if first else None), (labels if last else None)
        eng.train_step(inputs, labels)
        calls = [e for e in log if isinstance(e, tuple)]
        assert len(calls) == 1 and calls[0][1] is inputs and calls[0][2] is labels
        assert log.count("opt") == 1
        assert not {"sync", "capture", "replay"} & {e for e in log if isinstance(e, str)}
    assert not eng.graphable and eng._graph is None and eng.launches_per_step == 0


class _Accum:
    def __init__(self, log):
        self.log = log

    def add(self, logits, labels):
        self.log.append("add")


def test_evaluation_graph_one_eager_pass_then_capture_then_replays(fake_cuda):
    log = fake_cuda
    eng = _plain(log)
    eng.optimizer.graph_safe = True
    _spy_body(eng, log, "_eval_body")
    acc = _Accum(log)
    for k in range(1, 5):
        log.clear()
        inputs, labels = _batch(k)
        eng.eval_step(inputs, labels, acc)
        calls = [e for e in log if isinstance(e, tuple)]
        state = eng._eval
        if k == 1:
            assert len(calls) == 1 and calls[0][1] is state["inputs"] and calls[0][2] is state["labels"]
            assert torch.equal(calls[0][3][0], inputs[0]) and torch.equal(calls[0][4], labels)
            assert state["graph"] is None and log.count("add") == 2 and "replay" not in log
        elif k == 2:
            names = [e if isinstance(e, str) else e[0] for e in log if e not in ("F", "add")]
            assert names == ["sync", "capture", "body", "capture_end", "replay"]
            assert state["graph"] is not None
        else:
            assert log == ["replay"] and torch.equal(state["inputs"][0], inputs[0])
    # the training step's graph is not the evaluation's
    assert eng._graph is None and eng.launches_per_step == 0
    # another batch shape or accumulator replaces the graph, with one eager pass again
    first = eng._eval
    log.clear()
    eng.eval_step([torch.ones(6, 3)], torch.ones(6), acc)
    assert eng._eval is not first and eng._eval["graph"] is None
    assert [e[0] for e in log if isinstance(e, tuple)] == ["body"] and "replay" not in log
    log.clear()
    second = eng._eval
    eng.eval_step([torch.ones(6, 3)], torch.ones(6), _Accum(log))
    assert eng._eval is not second and eng._eval["graph"] is None and "replay" not in log
    eng.close()
    assert eng._eval is None
