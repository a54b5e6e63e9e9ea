"""LAMB on CPU / gloo: the ``Lamb`` optimizer against an fp64 implementation of the formula
written here, the fused optimizer's per-parameter segment table, config validation, clipping and
schedules, a 2-stage pipeline against one stage, checkpoint resume and the launcher's OPTIM key."""
import os
import runpy

import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.parallel.optim import FusedLamb, Lamb, TorchOptimizerAdapter, lr_factor
from tests._dist_helpers import run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ref_lamb_step(w, g, m, v, t, lr, wd, b1=0.9, b2=0.999, eps=1e-6):
    """One LAMB step in fp64 (apex FusedLAMB defaults); returns (w, m, v, r)."""
    w, g, m, v = (x.double() for x in (w, g, m, v))
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    u = (m / (1 - b1 ** t)) / (torch.sqrt(v / (1 - b2 ** t)) + eps) + wd * w
    wn, un = float(w.norm()), float(u.norm())
    r = wn / un if (wd != 0 and wn > 0 and un > 0) else 1.0
    return w - lr * r * u, m, v, r


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.dense = torch.nn.Linear(6, 5)
        self.LayerNorm = torch.nn.LayerNorm(5)
        self.zero = torch.nn.Parameter(torch.zeros(4, 3))        # ||W|| = 0: r = 1
        self.still = torch.nn.Parameter(torch.randn(7))          # zero gradient


@pytest.mark.parametrize("wd,grad_scale", [(0.0, 1.0), (0.05, 1.0), (0.05, 0.25)])
def test_lamb_matches_fp64_formula(wd, grad_scale):
    torch.manual_seed(0)
    net = _Net().double()
    excl = ("bias", "LayerNorm")
    opt = sky.build_optimizer(net, dict(optim_type="LAMB", lr=0.02, weight_decay=wd,
                                        exclude_from_weight_decay=excl))
    assert isinstance(opt, TorchOptimizerAdapter) and isinstance(opt.optimizer, Lamb)
    names = [n for n, _ in net.named_parameters()]
    ref = {n: [p.detach().clone(), torch.zeros_like(p), torch.zeros_like(p)]
           for n, p in net.named_parameters()}
    gen = torch.Generator().manual_seed(1)
    for t in range(1, 5):
        grads = {n: torch.randn(p.shape, generator=gen, dtype=torch.float64)
                 for n, p in net.named_parameters()}
        grads["still"].zero_()
        for n, p in net.named_parameters():
            p.grad = grads[n].clone()
        opt.step(grad_scale=grad_scale)
        ratios = {}
        for n in names:
            lam = 0.0 if any(s in n for s in excl) else wd
            w, m, v = ref[n]
            w, m, v, ratios[n] = ref_lamb_step(w, grads[n] * grad_scale, m, v, t, 0.02, lam)
            ref[n] = [w, m, v]
        for n, p in net.named_parameters():
            torch.testing.assert_close(p.detach(), ref[n][0], rtol=1e-12, atol=1e-14, msg=n)
        for grp in opt.optimizer.param_groups:
            for n, p in zip(grp["names"], grp["params"]):
                assert float(opt.optimizer.state[p]["trust_ratio"]) == pytest.approx(
                    ratios[n], rel=1e-12), n
        if t == 1:
            first = ratios
    if wd:
        assert first["zero"] == 1.0 and ratios["zero"] != 1.0      # ||W|| = 0 at the first step
        assert ratios["dense.weight"] != 1.0 and ratios["still"] != 1.0
        assert ratios["dense.bias"] == 1.0 and ratios["LayerNorm.weight"] == 1.0


def test_lamb_zero_gradient_without_decay_keeps_the_weight():
    p = torch.nn.Parameter(torch.randn(5, dtype=torch.float64))
    before = p.detach().clone()
    opt = Lamb([p], lr=0.1, weight_decay=0.0)
    p.grad = torch.zeros_like(p)
    opt.step()
    assert float(opt.state[p]["trust_ratio"]) == 1.0          # ||u|| = 0
    assert torch.equal(p.detach(), before)


def _bert_stage(layers=1):
    from skycomputing_b200.models import BertConfig, set_backend

    set_backend("native")
    c = BertConfig(1000, hidden_size=64, num_hidden_layers=layers, num_attention_heads=4,
                   intermediate_size=128, max_position_embeddings=32)
    enc = [dict(layer_type=t, config=c.__dict__)
           for t in ("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail")] * layers
    mc = ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=c.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                  hidden_size=64, num_classes=3)])
    try:
        return sky.build_module_from_cfg(0, mc, dict(module_to_cuda=False))
    finally:
        set_backend("torch")


def test_segment_table_of_a_bert_stage():
    stage = _bert_stage()
    opt = FusedLamb(stage, weight_decay=0.01)
    segs = opt.segments()
    named = dict(stage.named_parameters())
    assert sorted(s["name"] for s in segs) == sorted(named)      # one segment per nn.Parameter
    for s in segs:
        bank = opt.banks[s["bank"]]
        p = named[s["name"]]
        assert s["numel"] == p.numel()
        assert s["offset"] == (p.data_ptr() - bank.master().data_ptr()) // 4
        decays = not ("bias" in s["name"] or "LayerNorm" in s["name"])
        assert s["weight_decay"] == (0.01 if decays else 0.0), s["name"]
        assert s["use_ratio"] == decays and s["aligned"]
    by_bank = {}
    for s in segs:
        by_bank.setdefault(s["bank"], []).append(s)
    qkv = [v for v in by_bank.values() if len(v) == 3]
    assert len(qkv) == 2                                         # wqkv and bqkv
    for group in qkv:
        assert [s["name"].split(".")[-2] for s in group] == ["query", "key", "value"]
        n = group[0]["numel"]
        assert [s["offset"] for s in group] == [0, n, 2 * n]
    assert FusedLamb(stage, exclude_from_weight_decay=()).segments()[3]["weight_decay"] == 0.01


def test_odd_shaped_bank_has_an_unaligned_segment():
    from skycomputing_b200.ops.functions import ParamBank

    a = torch.nn.Parameter(torch.randn(3, 5))
    b = torch.nn.Parameter(torch.randn(7, 5))
    mod = torch.nn.Module()
    mod.a, mod.b = a, b
    bank = ParamBank([a, b], need_shadow=False)
    opt = FusedLamb(mod, banks=[bank], exclude_from_weight_decay=())
    segs = opt.segments()
    assert [(s["offset"], s["numel"], s["aligned"]) for s in segs] == [(0, 15, True),
                                                                        (15, 35, False)]


@pytest.mark.parametrize("bad", [
    dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(betas=(0.9,)), dict(eps=0.0),
    dict(eps=-1e-6), dict(weight_decay=-0.01), dict(lr=-1e-3), dict(amsgrad=True),
    dict(exclude_from_weight_decay="bias"), dict(exclude_from_weight_decay=("bias", 3)),
])
def test_invalid_configurations_raise(bad):
    with pytest.raises(ValueError):
        sky.build_optimizer(torch.nn.Linear(3, 2), dict(optim_type="LAMB", **bad))
    if "amsgrad" not in bad:
        with pytest.raises(ValueError):
            FusedLamb(torch.nn.Linear(3, 2), banks=[], **bad)


def test_clipping_and_schedule_with_lamb():
    torch.manual_seed(0)
    net = _Net()
    ref_net = _Net()
    ref_net.load_state_dict(net.state_dict())
    sched = dict(type="linear", warmup_steps=1, total_steps=5)
    opt = sky.build_optimizer(net, dict(optim_type="LAMB", lr=0.05), lr_schedule=sched,
                              grad_clip=dict(max_norm=0.1))
    ref = Lamb([dict(params=[p for n, p in ref_net.named_parameters()
                             if "bias" not in n and "LayerNorm" not in n], weight_decay=0.01),
                dict(params=[p for n, p in ref_net.named_parameters()
                             if "bias" in n or "LayerNorm" in n], weight_decay=0.0)], lr=0.05)
    ref_sched = torch.optim.lr_scheduler.LambdaLR(ref, lambda k: lr_factor(sched, k))
    gen = torch.Generator().manual_seed(2)
    for k in range(5):
        grads = [torch.randn(p.shape, generator=gen) for p in net.parameters()]
        for p, q, g in zip(net.parameters(), ref_net.parameters(), grads):
            p.grad, q.grad = g.clone(), g.clone()
        norm = float(torch.nn.utils.clip_grad_norm_(list(ref_net.parameters()), 0.1))
        opt.step()
        ref.step()
        ref_sched.step()
        sc = opt.scalars()
        assert sc["grad_norm"] == pytest.approx(norm, rel=1e-6) and norm > 0.1
        assert sc["lr"] == pytest.approx(0.05 * lr_factor(sched, k))
        for p, q in zip(net.parameters(), ref_net.parameters()):
            torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-7)
    assert opt.step_count() == 5


# ---------------------------------------------------------------------------------------------
# pipelines and checkpoints (gloo)
# ---------------------------------------------------------------------------------------------
LAMB_CFG = dict(optim_type="LAMB", lr=0.01, weight_decay=0.01)


def _model_cfg(layers=2):
    c = sky.BertConfig(100, hidden_size=32, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=64, max_position_embeddings=32, hidden_dropout_prob=0.0,
                       attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type=t, config=c.__dict__)
           for t in ("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail")] * layers
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
            + [dict(layer_type="BertPooler", config=c.__dict__),
               dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                    hidden_size=32, num_classes=3)])


def _train(rank, world, steps, tmp, hooks=(), epochs=1, same_batch=False, ps=False):
    cfg = _model_cfg()
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    wm = sky.Allocator(cfg, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=rank)
    for mod in model.model:
        if mod.is_local:
            for off, layer in enumerate(mod.module.layers.children()):
                g = torch.Generator().manual_seed(100 + mod.layer_range[0] + off)
                with torch.no_grad():
                    for p in layer.parameters():
                        p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    opt = sky.build_optimizer(model.optim_module, LAMB_CFG, grad_clip=dict(max_norm=0.05),
                              lr_schedule=dict(type="linear", warmup_steps=1, total_steps=6))
    assert isinstance(opt.optimizer, Lamb)
    runner = sky.Runner(model=model, parameter_server=sky.ParameterServer(cfg, lazy=True)
                        if (ps and rank == 0) else None, worker_manager=wm, optimizer=opt,
                        max_epochs=epochs, max_iters=steps, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=4,
                        schedule="1f1b")
    for h in hooks:
        runner.register_hook(h)
    losses = []
    orig = runner.train_iteration

    def spy(data, labels):
        out = orig(data, labels)
        if out is not None:
            losses.append(out)
        return out

    runner.train_iteration = spy
    loader = sky.build_dataloader_from_cfg(
        dataset_cfg=dict(type="SynthMNLIDataset", num_samples=64, max_seq_length=16,
                         vocab_size=100, seed=5),
        dataloader_cfg=dict(batch_size=8, shuffle=False))
    if same_batch:                      # a resumed run restarts the loader: feed one batch always
        loader = [next(iter(loader))] * steps
    runner.train(loader)
    runner.engine.close()
    params = {}
    for mod in runner.model.model:
        if mod.is_local:
            for off, sd in enumerate(mod.get_state_dict()):
                for name, val in sd.items():
                    params[f"{mod.layer_range[0] + off}.{name}"] = val.detach().clone().float()
    return dict(losses=losses, params=params)


def _merge(results):
    losses = [r["losses"] for r in results if r["losses"]][0]
    params = {}
    for r in results:
        params.update(r["params"])
    return losses, params


def test_two_stage_pipeline_matches_one_stage(tmp_path):
    one = _merge(run_distributed(_train, 1, 4, str(tmp_path)))
    two = _merge(run_distributed(_train, 2, 4, str(tmp_path)))
    assert one[0] == pytest.approx(two[0], rel=1e-5)
    assert sorted(one[1]) == sorted(two[1])
    for k in one[1]:
        torch.testing.assert_close(two[1][k], one[1][k], rtol=1e-5, atol=1e-7, msg=k)


def test_checkpoint_resume_continues_bit_identically(tmp_path):
    tmp = str(tmp_path)
    save = os.path.join(tmp, "ckpt")
    full = _merge(run_distributed(_train, 2, 5, tmp, (), 1, True, True))
    run_distributed(_train, 2, 3, tmp, (sky.CheckpointHook(save_path=save, save_interval=1),),
                    1, True, True)
    ckpt = os.path.join(save, sorted(f for f in os.listdir(save) if ".extra." not in f)[0])
    resumed = _merge(run_distributed(
        _train, 2, 5, tmp, (sky.CheckpointHook(load_checkpoint_from=ckpt,
                                               resume_training_state=True,
                                               strict_optimizer=True),), 2, True, True))
    assert len(resumed[0]) == 2
    assert resumed[0] == full[0][3:]
    for k in full[1]:
        assert torch.equal(resumed[1][k], full[1][k]), k


@pytest.mark.parametrize("env,want", [
    ({}, dict(optim_type="SGD", lr=0.001)),
    (dict(OPTIM="lamb", LR="0.002"), dict(optim_type="LAMB", lr=0.002)),
    (dict(OPTIM="adamw"), dict(optim_type="AdamW", lr=0.001)),
])
def test_launcher_config_optim_keys(monkeypatch, env, want):
    for k in ("OPTIM", "LR"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = runpy.run_path(os.path.join(ROOT, "experiment", "config.py"))
    assert cfg["train_config"]["optim_cfg"] == want
    if want["optim_type"] == "LAMB":
        opt = sky.build_optimizer(torch.nn.Linear(3, 2), cfg["train_config"]["optim_cfg"])
        assert isinstance(opt.optimizer, Lamb)


def test_launcher_config_rejects_unknown_optim(monkeypatch):
    monkeypatch.setenv("OPTIM", "rmsprop")
    with pytest.raises(ValueError):
        runpy.run_path(os.path.join(ROOT, "experiment", "config.py"))
