"""Host-side scheduling of the parameter-gradient kernels (ops/functions.py), exercised on CPU with
the kernel wrappers replaced by recorders: deferral queue order, overwrite-first stores, bias column
sums riding in the LayerNorm parameter-gradient launch."""
import torch

from skycomputing_b200.ops import functions as F


class _Recorder:
    def __init__(self):
        self.calls = []

    def gemm(self, a, b, **kw):
        self.calls.append(("gemm", kw.get("accumulate"), kw["out"].data_ptr()))

    def colsum_(self, x, out):
        self.calls.append(("colsum", out.data_ptr()))

    def ln_param_grad(self, dy, z, mean, rstd, dgamma, dbeta, x2=None, out2=None):
        self.calls.append(("ln", dgamma.data_ptr(), None if out2 is None else out2.data_ptr()))


def _bank(*shape):
    return F.ParamBank([torch.nn.Parameter(torch.zeros(*shape))], need_shadow=False)


def test_deferred_queue_keeps_program_order_and_flushes_once(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(F, "nat", rec)
    w, b, g, bn, bo = _bank(4, 3), _bank(4), _bank(3), _bank(3), _bank(3)
    x = torch.zeros(5, 3)
    F.set_wgrad_deferral(True)
    try:
        F._wgrad(torch.zeros(5, 4), x, w, b)
        F._ln_pgrad(x, x, torch.zeros(5), torch.zeros(5), g, bn, x, bo)
        F._wgrad(torch.zeros(5, 4), x, w, None)          # bias handled elsewhere: no colsum
        assert rec.calls == [] and F.pending_wgrads() == 3
        items = F.flush_wgrads()
        assert len(items) == 3 and F.pending_wgrads() == 0
        kinds = [c[0] for c in rec.calls]
        assert kinds == ["gemm", "colsum", "ln", "gemm"]
        assert rec.calls[2] == ("ln", g.grad().data_ptr(), bo.grad().data_ptr())
        assert F.flush_wgrads() == []
    finally:
        F.set_wgrad_deferral(False)


def test_overwrite_first_store_then_accumulate(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(F, "nat", rec)
    w, b = _bank(4, 3), _bank(4)
    x, g = torch.zeros(5, 3), torch.zeros(5, 4)
    F._wgrad(g, x, w, b)                                  # first backward ever: accumulate into zeros
    assert w.wgrad_target and rec.calls[0][:2] == ("gemm", True)
    w.overwrite_first = True                              # what FusedSGD decides after that step
    w.fresh = True                                        # ... and sets after every optimizer step
    rec.calls.clear()
    F._wgrad(g, x, w, b)                                  # micro-batch 0 of the next step: store
    F._wgrad(g, x, w, b)                                  # micro-batch 1: accumulate
    assert [c[1] for c in rec.calls if c[0] == "gemm"] == [False, True]
    assert not w.fresh
    b2 = _bank(4, 3)                                      # a bank the optimizer did not mark
    b2.fresh = True
    rec.calls.clear()
    F._wgrad(g, x, b2, None)
    assert rec.calls == [("gemm", True, b2.grad().data_ptr())]


def test_fused_sgd_marks_only_wgrad_targets(monkeypatch):
    """FusedSGD.step sets `fresh` on banks it decided to leave un-zeroed, and only on those."""
    from skycomputing_b200.parallel import optim

    class FakeExt:
        def pack_sgd_descriptors(self, descs):
            self.descs = descs
            return bytes(48 * len(descs))

        def sgd_multi(self, **kw):
            self.stepped = kw

    fake = FakeExt()
    monkeypatch.setattr(F.nat, "ext", lambda: fake)
    monkeypatch.delenv("SKY_SGD_OVERWRITE", raising=False)
    w, b = _bank(4, 3), _bank(4)
    w.wgrad_target = True
    opt = optim.FusedSGD(torch.nn.Module(), lr=0.1, banks=[w, b])
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    opt.step()
    assert [d[5] for d in opt._nat.ext().descs] == [1, 0]
    assert w.fresh and not b.fresh
    opt.zero_grad()
    assert not w.fresh


def test_looped_fused_step_body_order_and_slots(monkeypatch):
    """The (GPU-only) fused step body of the looped engine, driven with fakes on CPU: breadth-first
    order, slot = consumer chunk * m + micro-batch, masks relayed once per slot, first / last virtual stage
    special cases, one optimizer step."""
    from skycomputing_b200.parallel.pipeline_looped import LoopedPipelineEngine

    log = []

    class Stage(torch.nn.Module):
        def __init__(self, name):
            super().__init__()
            self.name = name
            self.w = torch.nn.Parameter(torch.ones(()))

        def forward(self, *args):
            log.append(("F", self.name, self.microbatch, self.in_channel is not None,
                        self.out_channel is not None))
            x = args[0].float() * self.w
            return (x, args[-1])

        def begin_backward(self):
            log.append(("B", self.name, self.microbatch))

        def end_backward(self):
            pass

    class Chan:
        def __init__(self, name):
            self.name = name

        def send_mask(self, mask, slot):
            log.append(("mask", self.name, slot))

    class Fused:
        prev, next = Chan("prev"), Chan("next")

        def begin_step(self):          # advance the epoch + wait for the consumer's ack
            log.append(("epoch",))

        def end_of_backward(self):     # acknowledge the inbound activation slots
            log.append(("ack",))

    class Opt:
        def step(self):
            log.append(("opt",))

    P, v, m = 2, 2, 2
    for pos in (0, 1):
        log.clear()
        stages = [Stage(f"c{c}") for c in range(v)]
        eng = LoopedPipelineEngine(stages, [c * P + pos for c in range(v)], P, [0, 1],
                                   torch.device("cpu"), Opt(),
                                   loss_fn=lambda out, lab: out.mean(), micro_batches=m,
                                   advance_rng=False)
        eng.fused, eng._setup_done = Fused(), True
        eng._loss_acc = torch.zeros(())
        monkeypatch.setattr(eng, "_fused_inputs",
                            lambda slot: (torch.ones(2, 3, requires_grad=True), torch.zeros(2)))
        data = [torch.ones(4, 3, requires_grad=True), torch.zeros(4)]
        eng._step_body_fused(data if pos == 0 else None, torch.zeros(4) if pos == 1 else None)
        # (inbound slot, outbound slot): a link's slots are numbered by the CONSUMER's chunk, so
        # the wrap-around link (ring position P-1 -> 0) writes into the slots of chunk c + 1
        wrap = m if pos == P - 1 else 0
        fwd = [e for e in log if e[0] == "F"]
        assert [(e[1], e[2]) for e in fwd] == [("c0", (0, 0 + wrap)), ("c0", (1, 1 + wrap)),
                                               ("c1", (2, 2 + wrap)), ("c1", (3, 3 + wrap))]
        bwd = [e for e in log if e[0] == "B"]
        assert [(e[1], e[2][0]) for e in bwd] == [("c1", 2), ("c1", 3), ("c0", 0), ("c0", 1)]
        # virtual stage 0 has no inbound channel, the last one no outbound channel
        assert fwd[0][3] == (pos != 0) and fwd[-1][4] == (pos != 1)
        masks = [e for e in log if e[0] == "mask"]
        assert all(e[1] == "next" for e in masks)
        assert sorted(e[2] for e in masks) == ([0, 1, 2, 3] if pos == 0 else [2, 3])
        assert log[0] == ("epoch",) and log[-1] == ("opt",) and log.count(("opt",)) == 1
        # the slot acknowledgement goes out after the last backward and before the optimizer
        assert log[-2] == ("ack",) and log.count(("ack",)) == 1
        if pos == 1:
            assert float(eng._loss_acc) > 0
