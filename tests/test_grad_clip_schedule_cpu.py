"""Learning-rate schedules and global-norm gradient clipping on CPU / gloo: the schedule formulas
against LambdaLR, pipelines of 2 / 3 stages (plain and looped) against one stage and against a
hand-written clip_grad_norm_ + LambdaLR loop, the launcher's config keys, checkpoint resume and
layer migration continuing the schedule, and config validation."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.parallel.optim import lr_factor
from tests._dist_helpers import free_port, run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_LR = 1.0
MAX_NORM = 0.02          # far below the gradient norm of these models: every step clips
SCHED = dict(type="linear", warmup_steps=1, total_steps=6)
CLIP = dict(max_norm=MAX_NORM)


# the HF transformers formulas, written out independently of the package
def _ref_lambda(kind, w, t):
    def f(k):
        if k < w:
            return k / max(1, w)
        if kind == "constant":
            return 1.0
        if kind == "linear":
            return max(0.0, (t - k) / max(1, t - w))
        p = min(1.0, (k - w) / max(1, t - w))
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * p)))
    return f


@pytest.mark.parametrize("kind", ["constant", "linear", "cosine"])
@pytest.mark.parametrize("w", [0, 10, 40])
def test_schedule_matches_lambdalr(kind, w):
    t = 40
    cfg = dict(type=kind, warmup_steps=w, total_steps=t)
    p = torch.nn.Parameter(torch.zeros(3))
    opt = torch.optim.SGD([p], lr=BASE_LR)
    ref = torch.optim.lr_scheduler.LambdaLR(opt, _ref_lambda(kind, w, t))
    mod = torch.nn.Linear(3, 2)
    ours = sky.build_optimizer(mod, dict(optim_type="SGD", lr=BASE_LR), lr_schedule=cfg)
    for k in range(60):
        want = ref.get_last_lr()[0]
        assert BASE_LR * lr_factor(cfg, k) == pytest.approx(want, rel=1e-12, abs=1e-15), k
        mod.weight.grad = torch.ones_like(mod.weight)
        mod.bias.grad = torch.ones_like(mod.bias)
        ours.step()
        assert ours.scalars()["lr"] == pytest.approx(want, rel=1e-12, abs=1e-15), k
        opt.step()
        ref.step()
    if kind != "constant":
        assert lr_factor(cfg, 60) == 0.0                  # no rise again after T


@pytest.mark.parametrize("bad_sched,bad_clip", [
    (dict(type="step", warmup_steps=0, total_steps=10), None),
    (dict(type="linear", warmup_steps=11, total_steps=10), None),
    (dict(type="linear", warmup_steps=0, total_steps=0), None),
    (dict(type="cosine", warmup_steps=0), None),
    (dict(type="linear", warmup_steps=0, total_steps=5, gamma=0.1), None),
    (None, dict(max_norm=0.0)),
    (None, dict(max_norm=-1.0)),
    (None, dict(max_norm=1.0, norm_type=1)),
    (None, dict(max_norm=1.0, norm_type=float("inf"))),
    (None, dict()),
])
def test_invalid_configurations_raise(bad_sched, bad_clip):
    with pytest.raises(ValueError):
        sky.build_optimizer(torch.nn.Linear(3, 2), dict(optim_type="SGD", lr=0.1),
                            lr_schedule=bad_sched, grad_clip=bad_clip)


def test_defaults_change_nothing():
    opt = sky.build_optimizer(torch.nn.Linear(3, 2), dict(optim_type="SGD", lr=0.1))
    assert not opt.reports_scalars and not opt.needs_global_norm
    assert "lr_schedule_step" not in opt.state_dict()


# ---------------------------------------------------------------------------------------------
# pipelines against one stage against a hand-written loop
# ---------------------------------------------------------------------------------------------
def _model_cfg(layers=2):
    c = sky.BertConfig(100, hidden_size=32, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=64, max_position_embeddings=32, hidden_dropout_prob=0.0,
                       attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=c.__dict__),
           dict(layer_type="BertLayer_Body", config=c.__dict__),
           dict(layer_type="BertLayer_Tail", config=c.__dict__)] * layers
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
            + [dict(layer_type="BertPooler", config=c.__dict__),
               dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                    hidden_size=32, num_classes=3)])


def _seed(model):
    for mod in model.model:
        if not mod.is_local:
            continue
        for off, layer in enumerate(mod.module.layers.children()):
            g = torch.Generator().manual_seed(100 + mod.layer_range[0] + off)
            with torch.no_grad():
                for p in layer.parameters():
                    p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def _loader(steps):
    return sky.build_dataloader_from_cfg(
        dataset_cfg=dict(type="SynthMNLIDataset", num_samples=8 * steps, max_seq_length=16,
                         vocab_size=100, seed=5),
        dataloader_cfg=dict(batch_size=8, shuffle=False))


def _workers(world, tmp):
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    return wm


def _layer_params(model) -> dict:
    out = {}
    for mod in model.model:
        if mod.is_local:
            for off, sd in enumerate(mod.get_state_dict()):
                for name, v in sd.items():
                    out[f"{mod.layer_range[0] + off}.{name}"] = v.detach().clone().float()
    return out


def _train(rank, world, granularity, virtual_stages, steps, tmp, hooks=(), layers=2,
           clip=CLIP, sched=SCHED, ps=False, epochs=1):
    cfg = _model_cfg(layers)
    wm = sky.Allocator(cfg, _workers(world, tmp), granularity=granularity).allocate(
        "even", virtual_stages=virtual_stages)
    model = sky.RpcModel(wm, this_rank=rank)
    _seed(model)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=BASE_LR),
                              lr_schedule=sched, grad_clip=clip)
    runner = sky.Runner(model=model, parameter_server=sky.ParameterServer(cfg, lazy=True)
                        if (ps and rank == 0) else None, worker_manager=wm, optimizer=opt,
                        max_epochs=epochs, max_iters=steps,
                        loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=4,
                        schedule="1f1b")
    for h in hooks:
        runner.register_hook(h(cfg) if callable(h) and not isinstance(h, sky.Hook) else h)
    losses, lrs, norms = [], [], []
    orig = runner.train_iteration

    def spy(data, labels):
        out = orig(data, labels)
        if out is not None:
            losses.append(out)
        sc = runner.optimizer.scalars()
        lrs.append(sc["lr"])
        norms.append(sc["grad_norm"])
        return out

    runner.train_iteration = spy
    runner.train(_loader(steps))
    runner.engine.close()
    return dict(losses=losses, lrs=lrs, norms=norms, params=_layer_params(runner.model),
                schedule=runner.engine.schedule)


def _hand_loop(rank, world, steps, tmp, split_at=None):
    """clip_grad_norm_ + LambdaLR around the same layers on one process (split_at: clip the
    layers below / above that index separately, as stage-local clipping would)."""
    cfg = _model_cfg(2)
    wm = sky.Allocator(cfg, _workers(1, tmp)).allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    _seed(model)
    stage = model.local_stage
    params = [p for p in stage.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, lr=BASE_LR)
    sched = torch.optim.lr_scheduler.LambdaLR(
        opt, _ref_lambda(SCHED["type"], SCHED["warmup_steps"], SCHED["total_steps"]))
    groups = [params]
    if split_at is not None:
        layers = list(stage.layers.children())
        low = {id(p) for layer in layers[:split_at] for p in layer.parameters()}
        groups = [[p for p in params if id(p) in low], [p for p in params if id(p) not in low]]
    ce = torch.nn.CrossEntropyLoss()
    losses, norms = [], []
    for data, labels in _loader(steps):
        total = 0.0
        for chunk in zip(*(t.chunk(4) for t in data), labels.chunk(4)):
            loss = ce(stage(*chunk[:-1])[0], chunk[-1]) / 4
            loss.backward()
            total += float(loss.detach())
        norms.append([float(torch.nn.utils.clip_grad_norm_(g, MAX_NORM)) for g in groups])
        opt.step()
        sched.step()
        opt.zero_grad()
        losses.append(total)
    return dict(losses=losses, norms=norms, params=_layer_params(model))


def _merge(results):
    out = {}
    for r in results:
        out.update(r["params"])
    return out


def _assert_same_training(a, b, rel=1e-5):
    assert a["losses"] == pytest.approx(b["losses"], rel=rel)
    pa, pb = _merge(a["all"]), _merge(b["all"])
    assert sorted(pa) == sorted(pb)
    for k in pa:
        torch.testing.assert_close(pa[k], pb[k], rtol=rel, atol=1e-7, msg=k)


def _last(results):
    r = dict([x for x in results if x["losses"]][0])
    r["all"] = results
    return r


def test_pipelines_clip_globally_and_follow_the_schedule(tmp_path):
    tmp = str(tmp_path)
    steps = 4
    hand = run_distributed(_hand_loop, 1, steps, tmp)[0]
    hand["all"] = [hand]
    one = _last(run_distributed(_train, 1, "layer", 1, steps, tmp))
    two = _last(run_distributed(_train, 2, "layer", 1, steps, tmp))
    three = _last(run_distributed(_train, 3, "block", 1, steps, tmp))
    # every step clipped: the global norm is far above max_norm
    assert all(n > 5 * MAX_NORM for n in one["norms"])
    assert one["norms"] == pytest.approx([n[0] for n in hand["norms"]], rel=1e-5)
    assert one["lrs"] == pytest.approx([BASE_LR * lr_factor(SCHED, k) for k in range(steps)])
    _assert_same_training(one, hand)
    _assert_same_training(two, one)
    _assert_same_training(three, one)
    # every rank reports the same global norm
    for run in (two, three):
        for r in run["all"]:
            assert r["norms"] == pytest.approx(one["norms"], rel=1e-5)
    # clipping each stage on its own would have trained something else
    local = run_distributed(_hand_loop, 1, steps, tmp, 5)[0]
    assert max(float((local["params"][k] - hand["params"][k]).abs().max())
               for k in hand["params"]) > 5e-4


def test_looped_pipeline_clips_like_the_plain_one(tmp_path):
    tmp = str(tmp_path)
    plain = _last(run_distributed(_train, 2, "block", 1, 4, tmp, (), 6))
    looped = _last(run_distributed(_train, 2, "block", 2, 4, tmp, (), 6))
    assert looped["schedule"] == "looped" and plain["schedule"] != "looped"
    _assert_same_training(looped, plain)
    assert looped["norms"] == pytest.approx(plain["norms"], rel=1e-5)


def test_launcher_logs_lr_and_grad_norm(tmp_path):
    env = dict(os.environ, TINY="1", LAYER_NUM="4", CORE_NUM="3", DEVICE="cpu", MAX_ITERS="4",
               PROJECT=str(tmp_path), ALLOCATE_TYPE="even", MICRO_BATCHES="2", BATCH_SIZE="8",
               MAX_GRAD_NORM="0.5", LR_SCHEDULE="linear", WARMUP_STEPS="2")
    out = subprocess.run([sys.executable, "-m", "skycomputing_b200.launch", "-c",
                          os.path.join(ROOT, "experiment", "config.py"), "--spawn", "2", "-p",
                          str(free_port())], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    d = os.path.join(str(tmp_path), "logs", "3nodes_4layers", "even")
    rows = [json.loads(line) for line in open(os.path.join(d, "metrics.jsonl"))]
    assert len(rows) == 4
    sched = dict(type="linear", warmup_steps=2, total_steps=4)
    assert [r["lr"] for r in rows] == pytest.approx([1e-3 * lr_factor(sched, k) for k in range(4)])
    assert all(r["grad_norm"] > 0 for r in rows)
    log = open(os.path.join(d, "allocation.log")).read()
    assert log.count("grad norm:") == 4 and log.count("lr:") == 4


def test_checkpoint_resume_continues_the_schedule(tmp_path):
    tmp = str(tmp_path)
    save = os.path.join(tmp, "ckpt")
    run_distributed(_train, 2, "block", 1, 3, tmp,
                    (sky.CheckpointHook(save_path=save, save_interval=1),), 2, CLIP, SCHED, True)
    ckpt = os.path.join(save, sorted(f for f in os.listdir(save) if ".extra." not in f)[0])
    resumed = _last(run_distributed(
        _train, 2, "block", 1, 5, tmp,
        (sky.CheckpointHook(load_checkpoint_from=ckpt, resume_training_state=True),), 2, CLIP,
        SCHED, True, 2))
    # the run resumes at iteration 3 with the schedule's step 3, not with a second warmup
    assert len(resumed["losses"]) == 2
    assert resumed["lrs"] == pytest.approx([BASE_LR * lr_factor(SCHED, k) for k in (3, 4)])


class _FakeDeviceBench:
    def __init__(self, wm):
        self._wm = wm

    def benchmark(self):
        from skycomputing_b200.utils import generate_worker_name

        return {generate_worker_name(w.rank): dict(time=3.0 if w.device == 1 else 1.0, avai_mem=1e9)
                for w in self._wm.worker_pool}


class _FakeModelBench:
    def __init__(self, n):
        self._n = n

    def benchmark(self):
        return [1.0] * self._n, [1.0] * self._n


def _migrating_hook(cfg):
    def factory(pool):
        return sky.Allocator(cfg, pool, _FakeModelBench(len(cfg)), _FakeDeviceBench(pool),
                             granularity="block", solver="exact")

    return sky.ReallocateHook(interval=2, allocator_factory=factory,
                              optimizer_cfg=dict(optim_type="SGD", lr=BASE_LR),
                              allocate_type="dynamic", min_gain=0.05, lr_schedule=SCHED,
                              grad_clip=CLIP)


def test_reallocation_continues_the_schedule(tmp_path):
    tmp = str(tmp_path)
    plain = _last(run_distributed(_train, 2, "block", 1, 5, tmp, (), 4))
    moved = _last(run_distributed(_train, 2, "block", 1, 5, tmp, (_migrating_hook,), 4))
    assert moved["lrs"] == pytest.approx([BASE_LR * lr_factor(SCHED, k) for k in range(5)])
    _assert_same_training(moved, plain)
