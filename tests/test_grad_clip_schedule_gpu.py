"""Global-norm clipping and learning-rate schedules on the fused sm_90a path: the grad_sumsq_multi
reduction against an fp64 sum, the fused SGD / Adam / AdamW updates against torch.optim +
clip_grad_norm_ + LambdaLR (eagerly and replayed from one CUDA graph), inf gradients, a one-GPU
Runner with and without the whole-step graph, and (with 2 / 4 GPUs) the pipelines whose stages
exchange their shares of the norm."""
import json
import math
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_GPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


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


def _stage():
    import skycomputing_b200 as sky
    from skycomputing_b200.models import BertConfig, set_backend

    set_backend("native")
    cfg = BertConfig(1000, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                     intermediate_size=512, max_position_embeddings=128,
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    mc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
          dict(layer_type="BertLayer_Body", config=cfg.__dict__),
          dict(layer_type="BertLayer_Tail", config=cfg.__dict__)]
    torch.manual_seed(0)
    return sky.build_module_from_cfg(0, mc, dict(module_to_cuda=True, cuda_device=0))


def test_grad_sumsq_multi_matches_fp64_and_is_replay_stable():
    from skycomputing_b200.ops import native as nat

    ext = nat.ext()
    g = torch.Generator(device="cuda").manual_seed(3)
    sizes = [1, 3, 5, 7, 1023, 4097, 100003, 262147] + [int(s) for s in
                                                         torch.randint(1, 5000, (57,))]
    grads = [torch.randn(n, generator=g, device="cuda") * 0.3 for n in sizes]
    params = [torch.zeros(n, device="cuda") for n in sizes]
    descs = [(p.data_ptr(), q.data_ptr(), 0, 0, n, 0, 0) for p, q, n in zip(params, grads, sizes)]
    d = torch.frombuffer(bytearray(ext.pack_sgd_descriptors(descs)), dtype=torch.uint8).cuda()
    blocks = ext.grad_sumsq_blocks(max(sizes))
    partials = torch.zeros(blocks * len(sizes), device="cuda")
    scalars = torch.zeros(ext.OPTIM_SCALARS_FLOATS, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    scale = 0.5
    want = sum(float((q.double() * scale).pow(2).sum()) for q in grads)
    seen = []
    for _ in range(3):
        partials.fill_(float("nan"))
        ext.grad_sumsq_multi(d.data_ptr(), len(sizes), blocks, scale, partials.data_ptr(), stream)
        ext.optim_finalize(partials.data_ptr(), partials.numel(), 0, max_norm=1.0,
                           out=scalars.data_ptr(), stream=stream)
        torch.cuda.synchronize()
        seen.append((partials.clone(), scalars.clone()))
    assert float(partials.double().sum()) == pytest.approx(want, rel=1e-5)
    lr, coef, norm, local = scalars.tolist()
    assert local == pytest.approx(want, rel=1e-5)
    assert norm == pytest.approx(math.sqrt(want), rel=1e-5)
    assert coef == pytest.approx(1.0 / (math.sqrt(want) + 1e-6), rel=1e-5)
    for p_, s_ in seen[1:]:
        assert torch.equal(p_, seen[0][0]) and torch.equal(s_, seen[0][1])   # bit for bit


CASES = [
    ("SGD", dict(lr=1e-2, momentum=0.9, weight_decay=1e-4)),
    ("Adam", dict(lr=2e-3, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.01)),
    ("AdamW", dict(lr=1e-3, weight_decay=0.05)),
]


def _pair(optim_type, kw, kind, max_norm=1.0):
    import skycomputing_b200 as sky

    stage = _stage()
    sched = dict(type=kind, warmup_steps=2, total_steps=5)
    opt = sky.build_optimizer(stage, dict(optim_type=optim_type, **kw), lr_schedule=sched,
                              grad_clip=dict(max_norm=max_norm))
    assert opt.graph_safe and opt.reports_scalars
    params = list(stage.parameters())
    ref_params = [torch.nn.Parameter(p.detach().clone()) for p in params]
    ref = getattr(torch.optim, optim_type)(ref_params, **kw)
    ref_sched = torch.optim.lr_scheduler.LambdaLR(ref, _ref_lambda(kind, 2, 5))
    return opt, params, ref, ref_params, ref_sched


def _ref_step(ref, ref_params, ref_sched, grads, max_norm=1.0):
    for r, gr in zip(ref_params, grads):
        r.grad = gr.clone()
    norm = float(torch.nn.utils.clip_grad_norm_(ref_params, max_norm))
    lr = ref_sched.get_last_lr()[0]
    ref.step()
    ref_sched.step()
    return lr, norm


@pytest.mark.parametrize("kind", ["constant", "linear", "cosine"])
@pytest.mark.parametrize("optim_type,kw", CASES)
def test_fused_optimizer_with_clip_and_schedule_matches_torch(optim_type, kw, kind):
    opt, params, ref, ref_params, ref_sched = _pair(optim_type, kw, kind)
    g = torch.Generator(device="cuda").manual_seed(1)
    for step in range(6):
        grads = [torch.randn(p.shape, generator=g, device="cuda") * 0.1 for p in params]
        for p, gr in zip(params, grads):
            p.grad.copy_(gr)
        opt.step()
        lr, norm = _ref_step(ref, ref_params, ref_sched, grads)
        sc = opt.scalars()
        assert norm > 1.0                                   # clipping is active
        assert sc["grad_norm"] == pytest.approx(norm, rel=1e-5)
        assert sc["lr"] == pytest.approx(lr, rel=1e-6, abs=1e-12)
        for p, r in zip(params, ref_params):
            torch.testing.assert_close(p.detach(), r.detach(), rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("kind", ["constant", "linear", "cosine"])
@pytest.mark.parametrize("optim_type,kw", CASES)
def test_fused_optimizer_with_clip_and_schedule_replays_from_a_graph(optim_type, kw, kind):
    opt, params, ref, ref_params, ref_sched = _pair(optim_type, kw, kind)
    g = torch.Generator(device="cuda").manual_seed(2)
    grads = [torch.randn(p.shape, generator=g, device="cuda") * 0.1 for p in params]

    def one_step():
        for p, gr in zip(params, grads):
            p.grad.copy_(gr)
        opt.step()

    one_step()                                   # eager step 1
    _ref_step(ref, ref_params, ref_sched, grads)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one_step()                               # captured, not executed
    lrs = []
    for _ in range(5):                           # steps 2..6
        graph.replay()
        lr, norm = _ref_step(ref, ref_params, ref_sched, grads)
        torch.cuda.synchronize()
        sc = opt.scalars()
        assert sc["lr"] == pytest.approx(lr, rel=1e-6, abs=1e-12)
        assert sc["grad_norm"] == pytest.approx(norm, rel=1e-5)
        lrs.append(sc["lr"])
    if kind != "constant":
        assert len(set(lrs)) > 2                 # the rate changed between replays
    for p, r in zip(params, ref_params):
        torch.testing.assert_close(p.detach(), r.detach(), rtol=2e-5, atol=2e-6)
    assert opt.step_count() == 6


@pytest.mark.parametrize("optim_type,kw", CASES)
def test_inf_gradient_propagates_like_torch(optim_type, kw):
    opt, params, ref, ref_params, ref_sched = _pair(optim_type, kw, "linear")
    g = torch.Generator(device="cuda").manual_seed(4)
    grads = [torch.randn(p.shape, generator=g, device="cuda") * 0.1 for p in params]
    grads[0].view(-1)[7] = float("inf")
    for _ in range(3):                           # warmup: lr 0 at the first step
        for p, gr in zip(params, grads):
            p.grad.copy_(gr)
        opt.step()
        _lr, norm = _ref_step(ref, ref_params, ref_sched, grads)
    assert math.isinf(norm) and math.isinf(opt.scalars()["grad_norm"])
    for p, r in zip(params, ref_params):
        torch.testing.assert_close(p.detach(), r.detach(), rtol=2e-5, atol=2e-6, equal_nan=True)


def _runner_losses(use_graph: bool, steps: int = 6):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import BertConfig, set_backend

    set_backend("native")
    cfg = BertConfig(30522, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=1024, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * 2
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                  hidden_size=256, num_classes=3)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_clip_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(500 + off)
        with torch.no_grad():
            for n, p in layer.named_parameters():
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=0.05, momentum=0.9),
                              lr_schedule=dict(type="cosine", warmup_steps=2, total_steps=6),
                              grad_clip=dict(max_norm=0.5))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_clip_test"), logging_cfg=None,
                        micro_batches=2, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    ds = sky.SynthMNLIDataset(num_samples=32, max_seq_length=128, seed=3, full_length=False)
    losses, norms, lrs = [], [], []
    for step in range(steps):
        sl = slice((step % 2) * 16, (step % 2 + 1) * 16)
        losses.append(runner.train_iteration(
            [ds.input_ids[sl], ds.segment_ids[sl], ds.input_mask[sl]], ds.labels[sl]))
        torch.cuda.synchronize()
        sc = opt.scalars()
        norms.append(sc["grad_norm"])
        lrs.append(sc["lr"])
    graphed = runner.engine._graph is not None
    runner.engine.close()
    return losses, norms, lrs, graphed


def test_runner_with_and_without_graph_agree():
    eager = _runner_losses(False)
    graph = _runner_losses(True)
    assert graph[3] and not eager[3]
    assert eager[2] == pytest.approx(graph[2], rel=1e-6)
    assert eager[2][0] == 0.0 and eager[2][2] == pytest.approx(0.05, rel=1e-6)
    assert eager[0][0] == graph[0][0]
    for a, b in zip(eager[0], graph[0]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)
    assert all(n > 0.5 for n in eager[1])                 # every step clipped
    for a, b in zip(eager[1], graph[1]):
        assert a == pytest.approx(b, rel=1e-2)


# ---------------------------------------------------------------------------------------------
# pipelines over 2 / 4 GPUs: every stage's share of the norm, through NCCL or peer memory
# ---------------------------------------------------------------------------------------------
def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world: int, *extra) -> dict:
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "check_pipeline.py"), *extra]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


@pytest.mark.parametrize("world", [2, 4])
def test_pipelines_with_clip_and_schedule_agree_across_transports(world):
    if N_GPU < world:
        pytest.skip(f"needs {world} GPUs")
    common = ("--layers", str(2 * world), "--micro-batches", str(world), "--batch",
              str(8 * world), "--max-grad-norm", "0.5", "--lr-schedule", "linear")
    runs = {
        "1f1b/nccl": _run(world, "--boundary", "nccl", *common),
        "1f1b/fused": _run(world, "--boundary", "fused", *common),
        "looped/fused": _run(world, "--virtual-stages", "2", *common),
    }
    ref = runs["1f1b/nccl"]["losses"]
    assert len(ref) == 6
    for name, r in runs.items():
        assert r["err_any"] == 0, name
        if name != "1f1b/nccl":
            assert r["fused_any"] and r["graph_all"], name
        # every rank computed the same global norm, bit for bit, at every step
        assert r["norms_identical"], (name, r["rank_norms"])
        assert all(n > 0.5 for n in r["rank_norms"][0]), name
        assert r["losses"][0] == ref[0], name
        for a, b in zip(r["losses"], ref):
            assert a == pytest.approx(b, rel=3e-3, abs=3e-3), (name, r["losses"], ref)
