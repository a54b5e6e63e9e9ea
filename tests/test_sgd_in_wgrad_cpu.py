"""The plain-SGD update in the weight-gradient GEMMs, host side, on CPU with fakes of the kernels:
which optimizer configurations allow it, which backward of each engine arms which banks, the order
of an armed wgrad behind the dgrad that reads its shadow (also when deferred), and the optimizer's
remaining descriptor table with its one ``sgd_multi`` launch per step."""
import pytest
import torch

from skycomputing_b200.ops import functions as F
from skycomputing_b200.parallel import optim

ARGS = (0.1, 0.0, 1.0)


class FakeExt:
    OPTIM_SCALARS_FLOATS = 4

    def __init__(self):
        self.tables, self.launches = [], []

    def pack_sgd_descriptors(self, descs):
        self.tables.append(list(descs))
        return bytes(48 * len(descs))

    def sgd_multi(self, **kw):
        self.launches.append(("sgd_multi", kw["n"]))

    def adam_multi(self, **kw):
        self.launches.append(("adam_multi", kw["n"]))

    def advance_counter(self, *a):
        self.launches.append(("advance_counter",))

    def optim_finalize(self, *a, **kw):
        self.launches.append(("optim_finalize",))


@pytest.fixture
def fake(monkeypatch):
    ext = FakeExt()
    monkeypatch.setattr(F.nat, "ext", lambda: ext)
    monkeypatch.setattr(torch.cuda, "current_stream",
                        lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    monkeypatch.delenv("SKY_SGD_OVERWRITE", raising=False)
    return ext


def _bank(*shape, weight=True):
    b = F.ParamBank([torch.nn.Parameter(torch.zeros(*shape))], need_shadow=False)
    b.update_in_wgrad_ok = weight
    return b


# ------------------------------------------------------------------ eligibility
def test_only_plain_sgd_offers_the_update(fake, monkeypatch):
    banks = [_bank(4, 3)]
    opt = optim.FusedSGD(torch.nn.Module(), lr=0.25, weight_decay=0.5, banks=banks)
    assert opt.wgrad_sgd_args() == (0.25, 0.5, 1.0)
    assert optim.FusedSGD(torch.nn.Module(), lr=0.1, momentum=0.9,
                          banks=banks).wgrad_sgd_args() is None
    for cfg in (dict(lr_schedule=dict(type="constant", warmup_steps=0, total_steps=0)),
                dict(max_norm=1.0)):
        o = optim.FusedSGD(torch.nn.Module(), lr=0.1, banks=banks)
        o.configure(**cfg)
        assert o.wgrad_sgd_args() is None, cfg
    assert optim.FusedAdam(torch.nn.Module(), banks=banks).wgrad_sgd_args() is None
    assert optim.FusedLamb(torch.nn.Module(), banks=banks).wgrad_sgd_args() is None
    monkeypatch.setenv("SKY_SGD_OVERWRITE", "0")     # gradients zeroed by the optimizer's pass
    assert optim.FusedSGD(torch.nn.Module(), lr=0.1, banks=banks).wgrad_sgd_args() is None


def test_span_marks_its_weight_banks_only():
    sp = F.SpanParams()
    w, b = sp._bank([torch.nn.Parameter(torch.zeros(4, 3))]), \
        sp._bank([torch.nn.Parameter(torch.zeros(4))], False)
    assert w.update_in_wgrad_ok and not b.update_in_wgrad_ok
    assert not F.ParamBank([torch.nn.Parameter(torch.zeros(4, 3))]).update_in_wgrad_ok


# ------------------------------------------------------------------ the optimizer's table
def test_remaining_banks_in_one_launch(fake):
    w0, b0, w1 = _bank(4, 3), _bank(4, weight=False), _bank(6, 3)
    opt = optim.FusedSGD(torch.nn.Module(), lr=0.1, banks=[w0, b0, w1])
    opt.set_update_in_wgrad([w0, w1])
    for _ in range(3):
        opt.step()
    assert len(fake.tables) == 1                          # built once
    assert [d[0] for d in fake.tables[0]] == [b0.flat.data_ptr()]
    assert fake.launches == [("sgd_multi", 1)] * 3
    # updated in backward: left un-zeroed, the next step's first wgrad overwrites them
    assert w0.overwrite_first and w1.overwrite_first and w0.fresh and w1.fresh
    assert not b0.overwrite_first and not b0.fresh
    opt.set_update_in_wgrad([])                           # handed back: every bank again
    opt.step()
    assert [d[0] for d in fake.tables[-1]] == [b.flat.data_ptr() for b in (w0, b0, w1)]
    assert fake.launches[-1] == ("sgd_multi", 3)


def test_no_launch_when_every_bank_is_updated_in_backward(fake):
    w0, w1 = _bank(4, 3), _bank(6, 3)
    opt = optim.FusedSGD(torch.nn.Module(), lr=0.1, banks=[w0, w1])
    opt.set_update_in_wgrad([w0, w1])
    opt.step()
    assert fake.launches == [] and w0.fresh and w1.fresh


# ------------------------------------------------------------------ wgrad / dgrad order
class _Recorder:
    def __init__(self):
        self.calls = []

    def gemm(self, a, b, **kw):
        self.calls.append(("gemm", kw.get("accumulate"), kw.get("sgd_master") is not None,
                           kw.get("sgd_lr")))

    def colsum_(self, x, out):
        self.calls.append(("colsum",))

    def cast_f32_to_bf16_(self, src, dst):
        pass


def test_armed_wgrad_follows_its_dgrad(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(F, "nat", rec)
    w, b = _bank(4, 3), _bank(4, weight=False)
    g, x = torch.zeros(5, 4), torch.zeros(5, 3)
    dgrad = lambda: rec.calls.append(("dgrad",)) or "dx"   # noqa: E731
    assert F._wgrad_dgrad(g, x, w, b, dgrad) == "dx"
    assert [c[0] for c in rec.calls] == ["gemm", "colsum", "dgrad"]
    assert rec.calls[0][2] is False
    rec.calls.clear()
    w.wgrad_sgd = ARGS
    assert F._wgrad_dgrad(g, x, w, b, dgrad) == "dx"
    assert [c[0] for c in rec.calls] == ["dgrad", "gemm", "colsum"]
    assert rec.calls[1][2:] == (True, ARGS[0])


def test_deferred_wgrad_keeps_the_arming_it_was_queued_with(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(F, "nat", rec)
    w = _bank(4, 3)
    g, x = torch.zeros(5, 4), torch.zeros(5, 3)
    F.set_wgrad_deferral(True)
    try:
        F._wgrad_dgrad(g, x, w, None, lambda: None)       # an earlier micro-batch: accumulates
        w.wgrad_sgd = ARGS
        F._wgrad_dgrad(g, x, w, None, lambda: None)       # the last one: armed
        w.wgrad_sgd = None                                # disarmed before the flush
        assert rec.calls == []
        F.flush_wgrads()
    finally:
        F.set_wgrad_deferral(False)
    assert [c[2] for c in rec.calls] == [False, True]


# ------------------------------------------------------------------ engines
class _Stage(torch.nn.Module):
    """Records, when backward reaches it, which bank arming is in force."""

    def __init__(self, name, bank, log):
        super().__init__()
        self.name, self.bank, self.log = name, bank, log
        self.w = torch.nn.Parameter(torch.ones(()))

    def forward(self, *args):
        x = args[0].float() * self.w
        mb = self.microbatch
        x.register_hook(lambda grad: self.log.append((self.name, mb, self.bank.wgrad_sgd)))
        return (x, args[-1])

    def begin_backward(self):
        pass

    def end_backward(self):
        pass


class _Opt:
    def step(self):
        pass


@pytest.mark.parametrize("m", [1, 2, 3])
def test_plain_engine_arms_the_last_micro_batch(m):
    from skycomputing_b200.parallel.pipeline import PipelineEngine, one_f_one_b_order

    log = []
    bank = _bank(4, 3)
    st = _Stage("s", bank, log)
    eng = PipelineEngine(st, 0, 1, [0], torch.device("cpu"), _Opt(),
                         loss_fn=lambda out, lab: out.mean(), micro_batches=m,
                         use_cuda_graph=False, advance_rng=False)
    eng._setup_done, eng._order = True, one_f_one_b_order(0, 1, m)
    eng._loss_acc = torch.zeros(())
    eng._wgrad_sgd, eng._wgrad_sgd_banks = ARGS, [[bank]]
    eng._step_body([torch.ones(2 * m, 3), torch.zeros(2 * m)], torch.zeros(2 * m))
    assert log == [("s", j, ARGS if j == m - 1 else None) for j in range(m)]
    assert bank.wgrad_sgd is None


def test_looped_engine_arms_each_chunks_last_micro_batch():
    from skycomputing_b200.parallel.pipeline_looped import LoopedPipelineEngine

    class Chan:
        def send_mask(self, mask, slot):
            pass

    class Fused:
        prev, next = Chan(), Chan()

        def begin_step(self):
            pass

        def end_of_backward(self):
            pass

    log = []
    P, v, m, pos = 2, 2, 2, 0
    banks = [_bank(4, 3) for _ in range(v)]
    stages = [_Stage(f"c{c}", banks[c], log) for c in range(v)]
    eng = LoopedPipelineEngine(stages, [c * P + pos for c in range(v)], P, [0, 1],
                               torch.device("cpu"), _Opt(), loss_fn=lambda out, lab: out.mean(),
                               micro_batches=m, advance_rng=False)
    eng.fused, eng._setup_done = Fused(), True
    eng._loss_acc = torch.zeros(())
    eng._fused_inputs = lambda slot: (torch.ones(2, 3, requires_grad=True), torch.zeros(2))
    eng._wgrad_sgd, eng._wgrad_sgd_banks = ARGS, [[b] for b in banks]
    eng._step_body_fused([torch.ones(4, 3), torch.zeros(4)], None)
    # backward order: chunk 1's micro-batches, then chunk 0's; slot = chunk * m + micro-batch
    assert [(n, mb[0], a) for n, mb, a in log] == [("c1", 2, None), ("c1", 3, ARGS),
                                                   ("c0", 0, None), ("c0", 1, ARGS)]
    assert all(b.wgrad_sgd is None for b in banks)


def test_engine_setup_selects_the_stages_weight_banks(fake, monkeypatch):
    from skycomputing_b200.models import bert_layers
    from skycomputing_b200.parallel.pipeline_looped import LoopedPipelineEngine

    w0, b0, w1 = _bank(4, 3), _bank(4, weight=False), _bank(6, 3)
    foreign = _bank(2, 3)                                 # not one of the optimizer's banks
    stages = [torch.nn.Module(), torch.nn.Module()]
    stages[0].banks_, stages[1].banks_ = [w0, b0], [w1, foreign]
    monkeypatch.setattr(bert_layers, "native_param_banks", lambda st: st.banks_)
    for momentum, armed in ((0.0, True), (0.9, False)):
        opt = optim.FusedSGD(torch.nn.Module(), lr=0.1, momentum=momentum, banks=[w0, b0, w1])
        eng = LoopedPipelineEngine(stages, [0, 2], 2, [0, 1], torch.device("cpu"), opt,
                                   micro_batches=2, advance_rng=False)
        eng._setup_wgrad_sgd()
        if not armed:
            assert eng._wgrad_sgd is None and opt._in_wgrad == frozenset()
            continue
        assert eng._wgrad_sgd == (0.1, 0.0, 1.0)
        assert eng._wgrad_sgd_banks == [[w0], [w1]]
        fake.launches.clear()
        opt.step()
        assert fake.launches == [("sgd_multi", 1)]
        eng.close()                                       # step() covers every bank again
        opt.step()
        assert fake.launches[-1] == ("sgd_multi", 3)
