"""The plain-SGD update in the weight-gradient GEMM's epilogue on the device.

Kernel: the wgrad GEMM with the update gives bit for bit the master and shadow that the wgrad
GEMM into an fp32 gradient followed by ``sgd_multi`` gives, storing or accumulating, with weight
decay and a gradient scale, on tiles ragged in M and N and at BERT-large's four weight-gradient
shapes at 4096 tokens; it leaves the gradient buffer alone and rejects the combinations it does
not support.

Training step: BERT layers trained through the engine with the update in the wgrad GEMMs against
the same model trained through the optimizer's pass (a constant learning-rate schedule with no
warm-up keeps every bank in that pass and gives the same lr bits), eagerly and from the captured
whole-step graph, with one and two micro-batches.  After the first step the weight banks' masters
and shadows and the loss are bit-identical: a dgrad that read a freshly updated shadow would change
the gradients of every layer below it.  Bias, LayerNorm and embedding gradients are summed with
float atomics, so later steps agree to a tolerance."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nat():
    from skycomputing_b200.ops import native as nat

    return nat


def _sgd_multi(p, grad, shadow, lr, wd, gs):
    nat = _nat()
    ext = nat.ext()
    descs = [(p.data_ptr(), grad.data_ptr(), 0, shadow.data_ptr(), p.numel(), 0, 0)]
    d = torch.frombuffer(bytearray(ext.pack_sgd_descriptors(descs)), dtype=torch.uint8).cuda()
    ext.sgd_multi(d_tensors=d.data_ptr(), n=1, max_numel=p.numel(), lr=lr, momentum=0.0,
                  weight_decay=wd, grad_scale=gs, zero_grad=False,
                  stream=torch.cuda.current_stream().cuda_stream, scalars=0)


# (M, N, K, block_n): M = output features, N = input features, K = tokens
SHAPES = [(1024, 1024, 4096, 0), (3072, 1024, 4096, 0), (4096, 1024, 4096, 0),
          (1024, 4096, 4096, 0), (200, 136, 256, 128), (200, 392, 256, 256),
          (136, 264, 128, 256)]


@pytest.mark.parametrize("M,N,K,block_n", SHAPES)
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("wd,gs", [(0.0, 1.0), (0.01, 0.5)])
def test_update_in_wgrad_matches_wgrad_then_sgd_multi(M, N, K, block_n, accumulate, wd, gs):
    nat = _nat()
    gen = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    dy = torch.randn(K, M, generator=gen, device="cuda").to(torch.bfloat16)
    x = torch.randn(K, N, generator=gen, device="cuda").to(torch.bfloat16)
    p0 = torch.randn(M, N, generator=gen, device="cuda") * 0.02
    g0 = torch.randn(M, N, generator=gen, device="cuda") if accumulate else \
        torch.full((M, N), float("nan"), device="cuda")
    lr = 0.0123
    # the two-pass reference: wgrad into the fp32 gradient, then the optimizer's pass
    grad = g0.clone()
    nat.gemm(dy, x, a_mn=True, b_mn=True, out=grad, accumulate=accumulate, block_n=block_n)
    p_ref = p0.clone()
    s_ref = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    _sgd_multi(p_ref, grad, s_ref, lr, wd, gs)
    # one pass
    grad2 = g0.clone()
    p = p0.clone()
    s = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    nat.gemm(dy, x, a_mn=True, b_mn=True, out=grad2, accumulate=accumulate, block_n=block_n,
             sgd_master=p, sgd_shadow=s, sgd_lr=lr, sgd_weight_decay=wd, sgd_grad_scale=gs)
    torch.cuda.synchronize()
    assert not torch.equal(p, p0)
    assert torch.equal(p, p_ref)
    assert torch.equal(s.view(torch.int16), s_ref.view(torch.int16))
    assert torch.equal(grad2.view(torch.int32), g0.view(torch.int32))   # gradient not stored


def test_update_in_wgrad_rejects_unsupported_combinations():
    nat = _nat()
    M, N, K = 256, 256, 128
    dy = torch.zeros(K, M, dtype=torch.bfloat16, device="cuda")
    x = torch.zeros(K, N, dtype=torch.bfloat16, device="cuda")
    grad = torch.zeros(M, N, device="cuda")
    p = torch.zeros(M, N, device="cuda")
    s = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    upd = dict(sgd_master=p, sgd_shadow=s, sgd_lr=0.1)
    bad = [dict(stream_k=1), dict(pair=1), dict(pair=2),
           dict(bias=torch.zeros(N, device="cuda"))]
    for kw in bad:
        with pytest.raises(RuntimeError, match="code 980"):
            nat.gemm(dy, x, a_mn=True, b_mn=True, out=grad, **upd, **kw)
    with pytest.raises(RuntimeError, match="code 980"):      # not a weight gradient's majors
        nat.gemm(dy.t().contiguous(), x, b_mn=True, out=grad, **upd)
    with pytest.raises(RuntimeError, match="code 980"):      # bf16 output
        nat.gemm(dy, x, a_mn=True, b_mn=True, out=torch.zeros(M, N, dtype=torch.bfloat16,
                                                               device="cuda"), **upd)
    with pytest.raises(RuntimeError, match="code 981"):      # misaligned master
        flat = torch.zeros(M * N + 1, device="cuda")
        nat.gemm(dy, x, a_mn=True, b_mn=True, out=grad, sgd_master=flat[1:].view(M, N),
                 sgd_shadow=s, sgd_lr=0.1)
    torch.cuda.synchronize()
    assert torch.count_nonzero(p) == 0


# ------------------------------------------------------------------ training step
def _model():
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
                          timer_config=dict(root="/tmp/sky_sgd_in_wgrad_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(700 + off)
        with torch.no_grad():
            for n, prm in layer.named_parameters():
                prm.copy_((torch.randn(prm.shape, generator=gen) * 0.02).to(prm.device))
                if n.endswith("LayerNorm.weight"):
                    prm.fill_(1.0)
    return sky, wm, model


def _state(opt):
    return [(b.flat.clone(), None if b._shadow is None else b._shadow.clone(),
             b.update_in_wgrad_ok) for b in opt.banks]


def _train(fused: bool, m: int, graph: bool, steps: int, lr: float = 0.05):
    sky, wm, model = _model()
    sched = None if fused else dict(type="constant", warmup_steps=0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=lr),
                              lr_schedule=sched)
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_sgd_in_wgrad_test"), logging_cfg=None,
                        micro_batches=m, schedule="1f1b", use_cuda_graph=graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    eng = runner.engine
    ds = sky.SynthMNLIDataset(num_samples=32, max_seq_length=128, seed=5, full_length=False)
    losses, first = [], None
    for step in range(steps):
        sl = slice((step % 2) * 16, (step % 2 + 1) * 16)
        data = [t[sl].cuda() for t in (ds.input_ids, ds.segment_ids, ds.input_mask)]
        loss = eng.train_step(data, ds.labels[sl].cuda())
        torch.cuda.synchronize()
        losses.append(float(loss))
        if step == 0:
            first = _state(opt)
    out = dict(losses=losses, first=first, last=_state(opt), armed=eng._wgrad_sgd is not None,
               graphed=eng._graph is not None, lr=opt.scalars()["lr"])
    eng.close()
    return out


@pytest.mark.parametrize("m,graph", [(1, False), (2, False), (1, True), (2, True)])
def test_training_step_matches_the_optimizer_pass(m, graph):
    steps = 6 if graph else 4
    ref = _train(False, m, graph, steps)
    got = _train(True, m, graph, steps)
    assert got["armed"] and not ref["armed"]
    assert got["graphed"] == graph and ref["graphed"] == graph
    assert ref["lr"] == float(np.float32(0.05))          # the schedule's lr: the same bits
    assert got["losses"][0] == ref["losses"][0]
    n_weights = 0
    for (p, s, weight), (p_ref, s_ref, _) in zip(got["first"], ref["first"]):
        if weight:
            n_weights += 1
            assert torch.equal(p, p_ref)
            assert torch.equal(s.view(torch.int16), s_ref.view(torch.int16))
    assert n_weights == 8                                  # wqkv, wo, w1, w2 of both layers
    # later steps: the float-atomic sums of the bias, LayerNorm and embedding gradients differ
    # from run to run in their last bits, and the steps amplify that (up to ~4e-4 of a bank's norm
    # after 4-6 steps, measured on H100); a missed or repeated update moves a bank by a whole step
    # (~1e-2 of its norm at this learning rate)
    for (p, _, _), (p_ref, _, _) in zip(got["last"], ref["last"]):
        assert float((p - p_ref).norm() / p_ref.norm()) < 2e-3
    for a, b in zip(got["losses"], ref["losses"]):
        assert a == pytest.approx(b, rel=1e-3, abs=1e-4)
