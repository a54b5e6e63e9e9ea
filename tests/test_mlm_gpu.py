"""Masked-language-model pretraining on the GPU: the vocab_ce kernel against torch fp32, its
determinism, its eval mode, the native BertTailForMaskedLM against the eager layer, and a
one-GPU BERT-large pipeline with the MLM head (graph-safe optimizer, graph = eager, clipping,
learning)."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    if not native.available():
        pytest.skip("native extension not built")
    return native


def _case(M, V, pad, seed, ignore_frac=0.3, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = (torch.randn(M, V + pad, generator=g, device="cuda") * scale).to(torch.bfloat16)
    logits = base[:, :V]
    labels = torch.randint(0, V, (M,), generator=g, device="cuda")
    labels[torch.rand(M, generator=g, device="cuda") < ignore_frac] = -100
    return base, logits, labels


def _torch_ref(logits, labels, scale):
    x = logits.float().requires_grad_(True)
    n = int((labels != -100).sum())
    if n == 0:
        return torch.zeros(()), torch.zeros_like(x)
    loss = F.cross_entropy(x, labels, ignore_index=-100)
    (g,) = torch.autograd.grad(loss * scale, x)
    return loss.detach(), g


# ---------------------------------------------------------------------------------------------
# training mode
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [3, 1000, 30528])
@pytest.mark.parametrize("M", [1, 37, 4096])
# (0, True) is the training layout: contiguous rows, 16-byte vectors, gradient over the logits
@pytest.mark.parametrize("pad,in_place", [(0, False), (8, False), (0, True), (5, True)])
def test_vocab_ce_matches_torch(nat, V, M, pad, in_place):
    base, logits, labels = _case(M, V, pad, seed=V + M + pad)
    if M == 1:
        labels[0] = V - 1
    want_loss, want_g = _torch_ref(logits, labels, 0.5)
    pad_cols = base[:, V:].clone()
    acc = torch.full((1,), 2.0, device="cuda")
    src = logits.clone() if not in_place else logits
    loss, dl = nat.vocab_ce(src, labels, grad_scale=0.5, loss_acc=acc, in_place=in_place)
    torch.cuda.synchronize()
    if in_place:
        assert dl.data_ptr() == logits.data_ptr()
    assert float(loss) == pytest.approx(float(want_loss), rel=1e-5, abs=1e-6)
    assert float(acc) == pytest.approx(2.0 + 0.5 * float(want_loss), rel=1e-5)
    ign = labels == -100
    assert torch.count_nonzero(dl[ign]) == 0                       # exactly 0
    # bf16 output: 8 mantissa bits
    torch.testing.assert_close(dl.float(), want_g, rtol=1.6e-2,
                               atol=1e-2 * float(want_g.abs().max()) + 1e-30)
    assert torch.equal(base[:, V:], pad_cols)                    # padding columns untouched


def test_vocab_ce_all_ignored_and_large_logits(nat):
    _, logits, labels = _case(64, 1000, 0, seed=1)
    labels.fill_(-100)
    acc = torch.zeros(1, device="cuda")
    loss, dl = nat.vocab_ce(logits, labels, grad_scale=1.0, loss_acc=acc)
    assert float(loss) == 0.0 and float(acc) == 0.0 and torch.count_nonzero(dl) == 0
    # torch gives NaN for an empty mean
    assert torch.isnan(F.cross_entropy(logits.float(), labels, ignore_index=-100))
    big = (torch.randn(256, 30528, device="cuda") * 3e4).to(torch.bfloat16)
    big[:, 7] = 2.0e5
    lab = torch.randint(0, 30528, (256,), device="cuda")
    lab[::3] = 7
    loss, dl = nat.vocab_ce(big, lab)
    want_loss, want_g = _torch_ref(big, lab, 1.0)
    assert math.isfinite(float(loss))
    assert float(loss) == pytest.approx(float(want_loss), rel=1e-5)
    torch.testing.assert_close(dl.float(), want_g, rtol=1.6e-2, atol=1e-6)


def test_vocab_ce_is_deterministic_and_graph_replays_agree(nat):
    _, logits, labels = _case(4096, 30528, 0, seed=9)
    a = nat.vocab_ce(logits, labels, grad_scale=0.25)
    b = nat.vocab_ce(logits, labels, grad_scale=0.25)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    acc = torch.zeros(1, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nat.vocab_ce(logits, labels, grad_scale=0.25, loss_acc=acc)   # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = nat.vocab_ce(logits, labels, grad_scale=0.25, loss_acc=acc)
    acc.zero_()
    g.replay()
    first = (out[0].clone(), out[1].clone(), acc.clone())
    acc.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(first[0], out[0]) and torch.equal(first[1], out[1])
    assert torch.equal(first[2], acc) and torch.equal(out[0], a[0]) and torch.equal(out[1], a[1])


def test_vocab_ce_rejects_bad_arguments(nat):
    with pytest.raises(RuntimeError, match="code 950"):
        nat.ext().vocab_ce(logits=1024, ldl=nat.ext().vocab_ce_max_v() + 8, labels=1024, M=1,
                           V=nat.ext().vocab_ce_max_v() + 8, dlogits=1024, workspace=1024)
    with pytest.raises(RuntimeError, match="code 952"):
        nat.ext().vocab_ce(logits=1024, ldl=8, labels=1024, M=1, V=8, workspace=1024)
    # the tensor-level wrapper names the vocabulary limit before anything is launched
    V = nat.ext().vocab_ce_max_v() + 8
    with pytest.raises(ValueError, match="at most"):
        nat.vocab_ce(torch.zeros(2, V, dtype=torch.bfloat16, device="cuda"),
                     torch.zeros(2, dtype=torch.int64, device="cuda"))


def test_vocab_ce_launch_count(nat):
    _, logits, labels = _case(8, 1000, 0, seed=2)
    acc = nat.TokenEvalAccumulator(1000, "cuda")
    nat.enable_launch_counter()
    for fn, want in ((lambda: nat.vocab_ce(logits, labels), 3),
                     (lambda: acc.add(logits, labels), 2),
                     (lambda: acc.add(logits[:0], labels[:0]), 0),
                     (lambda: nat.vocab_ce(logits[:0], labels[:0]), 2)):
        nat.reset_launch_counter()
        fn()
        assert nat.launch_count() == want
    # an empty training batch: loss 0 (count + finalize only)
    loss, dl = nat.vocab_ce(logits[:0], labels[:0])
    assert float(loss) == 0.0 and dl.shape == (0, 1000)


# ---------------------------------------------------------------------------------------------
# eval mode
# ---------------------------------------------------------------------------------------------
def test_token_accumulator_matches_torch(nat):
    from skycomputing_b200.runner.metrics import TorchTokenAccumulator

    _, logits, labels = _case(2048, 30528, 8, seed=3)
    logits[5] = 0.0
    logits[5, 17] = logits[5, 40] = 4.0                  # a tie: the first index wins
    labels[5] = 17
    labels[6] = 40000                                     # invalid
    labels[7] = -7                                        # invalid
    acc, ref = nat.TokenEvalAccumulator(30528, "cuda"), TorchTokenAccumulator(30528, "cuda")
    for part in (slice(0, 1000), slice(1000, 2048)):
        acc.add(logits[part], labels[part])
        ref.add(logits[part], labels[part])
    a, r = acc.read(), ref.read()
    assert a["count"] == r["count"] and a["correct"] == r["correct"] and a["invalid"] == r["invalid"] == 2
    assert a["loss_sum"] == pytest.approx(r["loss_sum"], rel=1e-5)
    one = nat.TokenEvalAccumulator(30528, "cuda")
    one.add(logits[5:6], labels[5:6])
    assert one.read()["correct"] == 1
    nan = logits[:4].clone()
    nan[0, 100] = float("nan")
    lab = torch.tensor([100, 1, -100, 2], device="cuda")
    acc2, ref2 = nat.TokenEvalAccumulator(30528, "cuda"), TorchTokenAccumulator(30528, "cuda")
    acc2.add(nan, lab)
    ref2.add(nan, lab)
    assert acc2.read()["correct"] == ref2.read()["correct"] and acc2.read()["count"] == 3


# ---------------------------------------------------------------------------------------------
# the native head against the eager layer
# ---------------------------------------------------------------------------------------------
def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def test_native_mlm_head_matches_eager():
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    cfg = sky.BertConfig(30528, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                         intermediate_size=4096)
    torch.manual_seed(0)
    head = sky.build_layer("BertTailForMaskedLM", config=cfg.__dict__).cuda()
    with torch.no_grad():
        for n, p in head.named_parameters():
            p.copy_(torch.randn_like(p) * 0.02)
            if n.endswith("LayerNorm.weight"):
                p.fill_(1.0)
    ref = copy.deepcopy(head)
    x = torch.randn(8, 128, 1024, device="cuda").to(torch.bfloat16)
    gy = (torch.randn(8, 128, 30528, device="cuda") * 1e-3).to(torch.bfloat16)
    set_backend("native")
    try:
        xn = x.clone().requires_grad_(True)
        out = head(xn, None)
        assert out.dtype == torch.bfloat16 and out.shape == (8, 128, 30528)
        out.backward(gy)
        torch.cuda.synchronize()
        set_backend("torch")
        xr = x.float().requires_grad_(True)
        want = ref(xr, None)
        want.backward(gy.float())
    finally:
        set_backend("auto")
    assert _rel(out, want) < 2e-2
    assert _rel(xn.grad, xr.grad) < 3e-2
    for (n, p), (_, q) in zip(head.named_parameters(), ref.named_parameters()):
        assert _rel(p.grad, q.grad) < 3e-2, n
    head.eval()
    with torch.no_grad():
        assert torch.equal(head(x, None), out.detach())     # inference path: the same logits


# ---------------------------------------------------------------------------------------------
# one GPU: BERT-large encoder layers + the MLM head
# ---------------------------------------------------------------------------------------------
def _mlm_runner(use_graph, grad_clip=None, lr=0.05, layers=2, micro_batches=2, optim=None):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    cfg = sky.BertConfig(30528, hidden_size=1024, num_hidden_layers=layers, num_attention_heads=16,
                         intermediate_size=4096, hidden_dropout_prob=0.0,
                         attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertTailForMaskedLM", config=cfg.__dict__)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_mlm_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(700 + off)
        with torch.no_grad():
            for n, p in layer.named_parameters():
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module,
                              optim or dict(optim_type="SGD", lr=lr, momentum=0.9),
                              grad_clip=grad_clip)
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="MaskedLMLoss"),
                        timer_cfg=dict(root="/tmp/sky_mlm_test"), logging_cfg=None,
                        micro_batches=micro_batches, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner, opt


def _batches(n, batch=16, seed=0, max_step=4, vocab=30528):
    import skycomputing_b200 as sky

    ds = sky.SynthMLMDataset(num_samples=n * batch, max_seq_length=128, vocab_size=vocab,
                             seed=seed, max_step=max_step)
    return list(torch.utils.data.DataLoader(ds, batch_size=batch))


def test_mlm_graph_step_equals_eager_and_optimizer_is_graph_safe():
    data = _batches(5)
    out = {}
    for use_graph in (False, True):
        runner, opt = _mlm_runner(use_graph)
        assert opt.graph_safe
        losses = [runner.train_iteration(d, l) for d, l in data]
        out[use_graph] = (losses, runner.engine._graph is not None)
        runner.engine.close()
    assert out[True][1] and not out[False][1]
    assert out[True][0][0] == out[False][0][0]
    for a, b in zip(out[False][0], out[True][0]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)


def test_evaluate_mlm_through_the_eval_graph():
    """Runner.evaluate on an MLM model: the evaluation CUDA graph captures the native token
    accumulator (vocab_ce in eval mode), a short last batch is padded with 2-D ignore labels, and
    the totals match the torch accumulator over the same micro-batches of eval-mode logits."""
    import skycomputing_b200 as sky
    from skycomputing_b200.runner.metrics import TorchTokenAccumulator, token_metrics

    ds = sky.SynthMLMDataset(num_samples=2 * 16 + 5, max_seq_length=128, vocab_size=30528, seed=1)
    loader = lambda: torch.utils.data.DataLoader(ds, batch_size=16)  # noqa: E731
    runner, _ = _mlm_runner(True)
    got = runner.evaluate(loader())
    again = runner.evaluate(loader())                  # replays the same graph
    assert runner.engine._eval["graph"] is not None
    assert again == got
    assert set(got) == {"n", "loss", "accuracy", "perplexity"}
    stage = runner.model.local_stage
    stage.eval()
    ref = TorchTokenAccumulator(30528, "cuda")
    with torch.no_grad():
        for data, labels in loader():
            n = data[0].shape[0]
            data = [torch.cat([t, t.new_zeros((16 - n,) + tuple(t.shape[1:]))]) for t in data]
            labels = torch.cat([labels, labels.new_full((16 - n, 128), -100)])
            for chunk, lab in zip(zip(*(t.chunk(2) for t in data)), labels.chunk(2)):
                ref.add(stage(*[t.cuda() for t in chunk])[0], lab.cuda())
    runner.engine.close()
    r = ref.read()
    want = token_metrics(r["loss_sum"], r["count"], r["correct"])
    assert got["n"] == want["n"] == sum(int((ds[i][1] != -100).sum()) for i in range(len(ds)))
    assert got["accuracy"] == want["accuracy"]
    assert got["loss"] == pytest.approx(want["loss"], rel=1e-5)


def test_clipping_norm_includes_the_head():
    from skycomputing_b200.models.bert_layers import native_param_banks

    (d, l), = _batches(1)
    runner, opt = _mlm_runner(False, grad_clip=dict(max_norm=1e9), lr=0.0, micro_batches=1)
    head = list(runner.model.local_stage.layers.children())[-1]
    head_ids = {id(p) for p in head.parameters()}
    assert head_ids <= {id(p) for b in native_param_banks(runner.model.local_stage) for p in b.params}
    runner.train_iteration(d, l)
    torch.cuda.synchronize()
    reported = opt.scalars()["grad_norm"]
    # the same batch by hand (lr 0: the weights did not move); the fused step zeroed the grads
    stage = runner.model.local_stage
    logits = stage(*[t.cuda() for t in d])[0]
    runner.loss_function(logits, l.cuda()).backward()
    torch.cuda.synchronize()
    params = [p for p in stage.parameters() if p.grad is not None]
    total = math.sqrt(sum(float(p.grad.double().pow(2).sum()) for p in params))
    head_only = math.sqrt(sum(float(p.grad.double().pow(2).sum()) for p in head.parameters()))
    runner.engine.close()
    assert head_only > 0.05 * total
    assert reported == pytest.approx(total, rel=2e-2)


def test_mlm_loss_falls_on_synthetic_data():
    # 1020 body tokens of the 30528-token vocabulary, step 1: every token is seen often enough
    # in 300 steps for the next-token rule to be learnt
    data = _batches(300, max_step=1, vocab=1024)
    runner, opt = _mlm_runner(True, optim=dict(optim_type="Adam", lr=1e-3))
    assert opt.graph_safe
    losses = [runner.train_iteration(d, l) for d, l in data]
    runner.engine.close()
    assert all(math.isfinite(x) for x in losses)
    assert sum(losses[-10:]) / 10 < 0.8 * sum(losses[:10]) / 10, losses[::10]
