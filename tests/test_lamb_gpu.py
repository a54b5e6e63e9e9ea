"""FusedLamb on the sm_90a path against an fp64 LAMB written here: a small native stage and an
odd-shaped bank (unaligned segments, scalar path), with and without clipping / a schedule and with
grad_scale != 1; per-parameter trust ratios; bit-identical graph replay; gradient zeroing and bf16
shadows; one full BERT-large stage; the Runner with FusedLamb and with the torch Lamb."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BETAS, EPS = (0.9, 0.999), 1e-6


def _stage(layers=1, hidden=256, vocab=1000, inter=512, heads=4):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import BertConfig, set_backend

    set_backend("native")
    cfg = BertConfig(vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                     intermediate_size=inter, max_position_embeddings=512,
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type=t, config=cfg.__dict__)
           for t in ("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail")] * layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                  hidden_size=hidden, num_classes=3)])
    torch.manual_seed(0)
    stage = sky.build_module_from_cfg(0, mc, dict(module_to_cuda=True, cuda_device=0))
    with torch.no_grad():
        for n, p in stage.named_parameters():
            p.copy_(torch.randn_like(p) * 0.02 + (1.0 if n.endswith("LayerNorm.weight") else 0.0))
    return stage


class _Ref:
    """fp64 LAMB over named tensors (apex FusedLAMB defaults), clipping and schedule included."""

    def __init__(self, named, lr, wd, exclude=("bias", "LayerNorm"), sched=None, max_norm=None):
        self.w = {n: p.detach().double().clone() for n, p in named}
        self.m = {n: torch.zeros_like(w) for n, w in self.w.items()}
        self.v = {n: torch.zeros_like(w) for n, w in self.w.items()}
        self.lam = {n: 0.0 if any(s in n for s in exclude) else wd for n in self.w}
        self.lr, self.sched, self.max_norm, self.t = lr, sched, max_norm, 0
        self.ratios = {}

    def step(self, grads, grad_scale=1.0):
        from skycomputing_b200.parallel.optim import lr_factor

        g = {n: x.double() * grad_scale for n, x in grads.items()}
        if self.max_norm is not None:
            norm = math.sqrt(sum(float(x.pow(2).sum()) for x in g.values()))
            coef = min(1.0, self.max_norm / (norm + 1e-6))
            g = {n: x * coef for n, x in g.items()}
        lr = self.lr * lr_factor(self.sched, self.t)
        self.t += 1
        b1, b2 = BETAS
        for n, w in self.w.items():
            m = self.m[n] = b1 * self.m[n] + (1 - b1) * g[n]
            v = self.v[n] = b2 * self.v[n] + (1 - b2) * g[n] * g[n]
            u = (m / (1 - b1 ** self.t)) / ((v / (1 - b2 ** self.t)).sqrt() + EPS) + self.lam[n] * w
            wn, un = float(w.norm()), float(u.norm())
            r = wn / un if (self.lam[n] != 0 and wn > 0 and un > 0) else 1.0
            self.ratios[n] = r
            self.w[n] = w - lr * r * u


def _check(opt, named, ref, rtol=2e-5, atol=2e-6):
    for n, p in named:
        torch.testing.assert_close(p.detach().double(), ref.w[n], rtol=rtol, atol=atol, msg=n)
    got = opt.trust_ratios()
    assert sorted(got) == sorted(ref.ratios)
    for n, r in ref.ratios.items():
        assert got[n] == pytest.approx(r, rel=1e-5), n


CASES = [(None, None, 1.0), (0.5, "linear", 1.0), (None, None, 0.5), (0.5, "cosine", 2.0)]


@pytest.mark.parametrize("max_norm,kind,grad_scale", CASES)
def test_native_stage_matches_fp64(max_norm, kind, grad_scale):
    import skycomputing_b200 as sky
    from skycomputing_b200.parallel.optim import FusedLamb

    stage = _stage()
    sched = dict(type=kind, warmup_steps=1, total_steps=6) if kind else None
    opt = sky.build_optimizer(stage, dict(optim_type="LAMB", lr=0.01, weight_decay=0.01),
                              lr_schedule=sched,
                              grad_clip=dict(max_norm=max_norm) if max_norm else None)
    assert isinstance(opt, FusedLamb) and opt.graph_safe
    named = list(stage.named_parameters())
    ref = _Ref(named, 0.01, 0.01, sched=sched, max_norm=max_norm)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(4):
        grads = {n: torch.randn(p.shape, generator=gen, device="cuda") * 0.1 for n, p in named}
        for n, p in named:
            p.grad.copy_(grads[n])
        opt.step(grad_scale=grad_scale)
        ref.step(grads, grad_scale)
        if max_norm:
            assert opt.scalars()["grad_norm"] > max_norm       # clipping is active
    _check(opt, named, ref)
    r = opt.trust_ratios()
    qkv = [r[n] for n, _ in named if n.endswith(("query.weight", "key.weight", "value.weight"))]
    assert len(qkv) == 3 and len(set(qkv)) == 3                # Q, K, V: one ratio each
    assert all(v == 1.0 for n, v in r.items() if "bias" in n or "LayerNorm" in n)
    assert any(n.endswith("word_embeddings.weight") for n in r)
    assert opt.step_count() == 4


def _odd_bank():
    from skycomputing_b200.ops.functions import ParamBank

    torch.manual_seed(3)
    mod = torch.nn.Module()
    mod.a = torch.nn.Parameter(torch.randn(3, 5, device="cuda") * 0.5)
    mod.b = torch.nn.Parameter(torch.randn(7000, 5, device="cuda") * 0.5)   # 3 chunks, offset 15
    mod.bias = torch.nn.Parameter(torch.randn(2, 5, device="cuda"))
    return mod, ParamBank([mod.a, mod.b, mod.bias])


@pytest.mark.parametrize("max_norm,kind,grad_scale", CASES)
def test_odd_shaped_bank_matches_fp64(max_norm, kind, grad_scale):
    from skycomputing_b200.parallel.optim import FusedLamb, check_lr_schedule

    mod, bank = _odd_bank()
    sched = check_lr_schedule(dict(type=kind, warmup_steps=1, total_steps=6)) if kind else None
    opt = FusedLamb(mod, lr=0.02, weight_decay=0.05, banks=[bank])
    if sched or max_norm:
        opt.configure(sched, max_norm)
    named = list(mod.named_parameters())
    ref = _Ref(named, 0.02, 0.05, sched=sched, max_norm=max_norm)
    gen = torch.Generator(device="cuda").manual_seed(2)
    for _ in range(4):
        grads = {n: torch.randn(p.shape, generator=gen, device="cuda") for n, p in named}
        for n, p in named:
            p.grad.copy_(grads[n])
        opt.step(grad_scale=grad_scale)
        ref.step(grads, grad_scale)
    assert [s["aligned"] for s in opt.segments()] == [True, False, False]
    _check(opt, named, ref)
    assert torch.equal(bank.shadow(), bank.master().to(torch.bfloat16))
    assert opt.trust_ratios()["a"] != opt.trust_ratios()["b"]


def _snapshot(opt):
    return ([b.master().clone() for b in opt.banks], [b.shadow().clone() for b in opt.banks],
            [m.clone() for m in opt._mom], [v.clone() for v in opt._mom2], opt._step.clone())


def _restore(opt, snap):
    masters, shadows, moms, mom2s, step = snap
    for b, x, s in zip(opt.banks, masters, shadows):
        b.master().copy_(x)
        b._shadow.copy_(s)
    for m, x in zip(opt._mom, moms):
        m.copy_(x)
    for v, x in zip(opt._mom2, mom2s):
        v.copy_(x)
    opt._step.copy_(step)


@pytest.mark.parametrize("clip", [False, True])
def test_graph_replay_is_bit_identical_to_eager_steps(clip):
    import skycomputing_b200 as sky

    stage = _stage()
    opt = sky.build_optimizer(stage, dict(optim_type="LAMB", lr=0.01),
                              lr_schedule=dict(type="linear", warmup_steps=1, total_steps=6)
                              if clip else None, grad_clip=dict(max_norm=0.5) if clip else None)
    params = list(stage.parameters())
    gen = torch.Generator(device="cuda").manual_seed(5)
    grads = [torch.randn(p.shape, generator=gen, device="cuda") * 0.1 for p in params]

    def one_step():
        for p, g in zip(params, grads):
            p.grad.copy_(g)
        opt.step()

    one_step()                                   # eager step 1: builds the table
    torch.cuda.synchronize()
    snap = _snapshot(opt)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one_step()                               # captured, not executed
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    replayed = _snapshot(opt)
    ratios = opt.trust_ratios()
    assert int(opt._step.item()) == 4
    _restore(opt, snap)
    for _ in range(3):
        one_step()
    torch.cuda.synchronize()
    eager = _snapshot(opt)
    for a, b in zip(replayed[:4], eager[:4]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert int(opt._step.item()) == 4 and opt.trust_ratios() == ratios


def test_gradient_zeroing_and_shadows():
    import skycomputing_b200 as sky

    stage = _stage()
    from skycomputing_b200.models.bert_layers import native_param_banks

    banks = native_param_banks(stage)
    kept = [banks[0], banks[6]]                  # wqkv and the FFN1 weight
    for b in kept:
        b.wgrad_target = True                    # their next wgrad overwrites the gradient
    opt = sky.build_optimizer(stage, dict(optim_type="LAMB", lr=0.01))
    gen = torch.Generator(device="cuda").manual_seed(6)
    for _ in range(2):
        for b in opt.banks:
            b.grad().copy_(torch.randn(b.grad().shape, generator=gen, device="cuda"))
        before = [b.grad().clone() for b in opt.banks]
        opt.step()
        torch.cuda.synchronize()
        for b, g0 in zip(opt.banks, before):
            if any(b is k for k in kept):
                assert b.overwrite_first and torch.equal(b.grad(), g0)
            else:
                assert not b.overwrite_first and not b.grad().any()
            if b.need_shadow:
                assert torch.equal(b.shadow(), b.master().to(torch.bfloat16))
                assert torch.equal(b._shadow, b.master().to(torch.bfloat16))


def test_full_bert_large_stage_ratios_match_fp64():
    import skycomputing_b200 as sky

    stage = _stage(layers=24, hidden=1024, vocab=30522, inter=4096, heads=16)
    opt = sky.build_optimizer(stage, dict(optim_type="LAMB", lr=1e-3, weight_decay=0.01))
    named = list(stage.named_parameters())
    assert len(opt.segments()) == len(named) == 393
    gen = torch.Generator(device="cuda").manual_seed(7)
    grads = {}
    for n, p in named:
        grads[n] = torch.randn(p.shape, generator=gen, device="cuda") * 1e-3
        p.grad.copy_(grads[n])
    w0 = {n: p.detach().clone() for n, p in named}
    opt.step()
    got = opt.trust_ratios()
    b1, b2 = BETAS
    for n, _ in named:
        w, g = w0[n].double(), grads[n].double()
        u = ((1 - b1) * g / (1 - b1)) / (((1 - b2) * g * g / (1 - b2)).sqrt() + EPS)
        lam = 0.0 if ("bias" in n or "LayerNorm" in n) else 0.01
        u = u + lam * w
        wn, un = float(w.norm()), float(u.norm())
        r = wn / un if (lam and wn > 0 and un > 0) else 1.0
        assert got[n] == pytest.approx(r, rel=1e-5), n
    emb = [n for n, _ in named if n.endswith("word_embeddings.weight")][0]
    assert dict(named)[emb].numel() > 31_000_000 and got[emb] != 1.0


def _runner_losses(optim: str, use_graph: bool, steps: int = 6):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import BertConfig, set_backend

    set_backend("native")
    cfg = BertConfig(30522, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=1024, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type=t, config=cfg.__dict__)
           for t in ("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail")] * 2
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                  hidden_size=256, num_classes=3)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_lamb_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(500 + off)
        with torch.no_grad():
            for n, p in layer.named_parameters():
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="LAMB", lr=5e-3),
                              prefer_fused=optim == "fused",
                              lr_schedule=dict(type="cosine", warmup_steps=2, total_steps=6),
                              grad_clip=dict(max_norm=0.5))
    assert type(opt).__name__ == ("FusedLamb" if optim == "fused" else "TorchOptimizerAdapter")
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_lamb_test"), logging_cfg=None,
                        micro_batches=2, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    ds = sky.SynthMNLIDataset(num_samples=32, max_seq_length=128, seed=3, full_length=False)
    losses = []
    for step in range(steps):
        sl = slice((step % 2) * 16, (step % 2 + 1) * 16)
        losses.append(runner.train_iteration(
            [ds.input_ids[sl], ds.segment_ids[sl], ds.input_mask[sl]], ds.labels[sl]))
        torch.cuda.synchronize()
    graphed = runner.engine._graph is not None
    runner.engine.close()
    return losses, graphed


def test_runner_fused_and_torch_lamb_agree():
    fused, g1 = _runner_losses("fused", False)
    torch_, g2 = _runner_losses("torch", False)
    assert not g1 and not g2
    assert fused[0] == torch_[0]
    assert fused[-1] != fused[0]                          # it trained
    for a, b in zip(fused, torch_):
        assert a == pytest.approx(b, rel=3e-3)


def test_runner_with_and_without_graph_agree():
    eager = _runner_losses("fused", False)
    graph = _runner_losses("fused", True)
    assert graph[1] and not eager[1]
    assert eager[0][0] == graph[0][0]
    for a, b in zip(eager[0], graph[0]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)
