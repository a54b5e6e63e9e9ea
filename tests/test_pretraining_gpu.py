"""Masked-LM + next-sentence pretraining on the GPU: the [CLS]-row join kernels and the
next-sentence cross entropy against torch, the native BertTailForPreTraining against its eager
fp32 path at BERT-large width (B = 32, S = 128; dense and sparse, tied and untied), and a one-GPU pipeline with the
head (graph = eager, bit-equal replays, evaluation against the torch accumulators, SGD and LAMB
lowering the training loss on SynthPretrainingDataset)."""
import math

import pytest
import torch

from skycomputing_b200.ops.functions import mlm_slots_ref, split_pretraining_labels

pytestmark = pytest.mark.gpu
V_LARGE = 30528


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    if not native.available():
        pytest.skip("native extension not built")
    return native


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


# ---------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,H", [(32, 128, 1024), (3, 16, 64)])
def test_scatter_joins_the_cls_gradient(nat, B, S, H):
    g = torch.Generator(device="cuda").manual_seed(B + S + H)
    labels = torch.randint(0, 1000, (B, S), generator=g, device="cuda")
    labels[torch.rand(B, S, generator=g, device="cuda") >= 0.15] = -100
    labels[0, 0] = 5   # a decoded [CLS] row gets the sum, rounded once
    P = 20
    hidden = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
    _, slot, _ = nat.mlm_gather(hidden, labels, P, 1000)
    dx_c = torch.randn(B * P, H, device="cuda").to(torch.bfloat16)
    dcls = torch.randn(B, H, device="cuda").to(torch.bfloat16)
    plain = nat.mlm_scatter(dx_c, slot)
    # without dcls: the old kernel's output (a pure copy)
    want_plain = torch.zeros_like(plain)
    want_plain[slot >= 0] = dx_c[slot[slot >= 0].long()]
    assert torch.equal(plain, want_plain)
    joined = nat.mlm_scatter(dx_c, slot, dcls)
    want = plain.clone().view(B, S, H)
    want[:, 0] = (want[:, 0].float() + dcls.float()).to(torch.bfloat16)
    assert torch.equal(joined.view(B, S, H), want)
    dense = torch.randn(B, S, H, device="cuda").to(torch.bfloat16)
    want = dense.clone()
    want[:, 0] = (want[:, 0].float() + dcls.float()).to(torch.bfloat16)
    nat.cls_grad_add_(dense, dcls)
    assert torch.equal(dense, want)


def test_masked_softmax_ce_matches_torch(nat):
    M, C = 32, 2
    logits = torch.randn(M, C, device="cuda") * 3
    labels = torch.randint(0, C, (M,), device="cuda")
    labels[::5] = -100
    acc = torch.zeros(1, device="cuda")
    loss, d = nat.masked_softmax_ce(logits, labels, grad_scale=0.5, loss_acc=acc)
    x = logits.double().requires_grad_(True)
    want = torch.nn.functional.cross_entropy(x, labels, ignore_index=-100)
    (want * 0.5).backward()
    want = want.detach()
    assert float(loss) == pytest.approx(float(want), rel=1e-6)
    assert float(acc) == pytest.approx(0.5 * float(want), rel=1e-6)
    assert torch.allclose(d.double(), x.grad, rtol=1e-5, atol=1e-7)
    assert torch.count_nonzero(d[::5]) == 0
    loss2, d2 = nat.masked_softmax_ce(logits, labels, grad_scale=0.5)
    assert torch.equal(loss2, loss) and torch.equal(d2, d)
    # no labelled row: loss 0 and a zero gradient
    loss, d = nat.masked_softmax_ce(logits, torch.full_like(labels, -100))
    assert float(loss) == 0.0 and torch.count_nonzero(d) == 0
    # an out-of-range label: NaN loss, its row 0, the other rows as without it
    bad = labels.clone()
    bad[1] = 7
    loss, d = nat.masked_softmax_ce(logits, bad)
    assert math.isnan(float(loss)) and torch.count_nonzero(d[1]) == 0
    # graph capture: bit-equal replays
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nat.masked_softmax_ce(logits, labels)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gl, gd = nat.masked_softmax_ce(logits, labels)
    graph.replay()
    first = (gl.clone(), gd.clone())
    graph.replay()
    assert torch.equal(gl, first[0]) and torch.equal(gd, first[1])


def test_cross_entropy_loss_is_unchanged(nat):
    from skycomputing_b200.runner import build_loss

    fn = build_loss(dict(type="CrossEntropyLoss"), torch.device("cuda", 0))
    logits = torch.randn(32, 3, device="cuda")
    labels = torch.randint(0, 3, (32,), device="cuda")
    acc = torch.zeros(1, device="cuda")
    d = fn.fused(logits, labels, 0.5, acc)
    loss, want = nat.softmax_ce(logits, labels, grad_scale=0.5)
    assert torch.equal(d, want) and float(acc) == float(loss) * 0.5


# ---------------------------------------------------------------------------------------------
# the head at BERT-large width against its eager fp32 path
# ---------------------------------------------------------------------------------------------
def _head(P=None, tie=False):
    """The native head and its eager twin with the same weights; ``tie``: each decodes with the
    word-embedding table of its own BertEmbeddings."""
    import skycomputing_b200 as sky
    from skycomputing_b200.models.bert_layers import tie_decoder_to_embeddings

    cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                         intermediate_size=4096)
    kw = dict(tie_word_embeddings=tie)
    if P is not None:
        kw["max_predictions"] = P
    head = sky.build_layer("BertTailForPreTraining", config=cfg.__dict__, **kw).cuda()
    eager = sky.build_layer("BertTailForPreTraining", config=cfg.__dict__, **kw).cuda()
    if tie:
        embs = [sky.build_layer("BertEmbeddings", config=cfg.__dict__).cuda() for _ in range(2)]
        assert tie_decoder_to_embeddings([embs[0], head])
        assert tie_decoder_to_embeddings([embs[1], eager])
    gen = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for n, p in head.named_parameters():
            p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
            if n.endswith("LayerNorm.weight"):
                p.fill_(1.0)
    if tie:
        embs[1].load_state_dict(embs[0].state_dict())
    eager.load_state_dict(head.state_dict())
    return head, eager


def _pretraining_labels(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    lab = torch.full((B, S + 1), -100, dtype=torch.int64)
    for b in range(B):
        pos = torch.randperm(S - 3, generator=g)[:19] + 1
        lab[b, pos] = torch.randint(0, V_LARGE, (19,), generator=g)
    lab[:, S] = torch.randint(0, 2, (B,), generator=g)
    return lab.cuda()


@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("P", [None, 20])
def test_native_head_matches_the_eager_head(nat, P, tie):
    from skycomputing_b200.models import set_backend

    B, S, H = 32, 128, 1024
    head, eager = _head(P, tie)
    x = torch.randn(B, S, H, device="cuda").to(torch.bfloat16)
    labels = _pretraining_labels(B, S, 0)
    dmlm = torch.randn(B * (P or S), V_LARGE, device="cuda") * 1e-3
    dnsp = torch.randn(B, 2, device="cuda")
    set_backend("native")
    try:
        xn = x.clone().requires_grad_(True)
        out = head(xn, None, labels) if P else head(xn, None)
        mlm, nsp = out[0], out[-1]
        assert nsp.shape == (B, 2) and nsp.dtype == torch.float32
        torch.autograd.backward([mlm, nsp], [dmlm.view_as(mlm).to(mlm.dtype), dnsp])
        torch.cuda.synchronize()
        set_backend("torch")
        xe = x.float().requires_grad_(True)
        oute = eager(xe, None, labels) if P else eager(xe, None)
        torch.autograd.backward([oute[0], oute[-1]], [dmlm.view_as(oute[0]), dnsp])
    finally:
        set_backend("auto")
    if P:
        want = mlm_slots_ref(split_pretraining_labels(labels)[0], P, -100, V_LARGE)[2]
        assert torch.equal(out[1], want) and torch.equal(oute[1], want)
    assert _rel(mlm, oute[0]) < 2e-2
    assert _rel(nsp, oute[-1]) < 2e-2
    assert _rel(xn.grad, xe.grad) < 3e-2
    # the [CLS] rows carry the pooler's gradient on top of the masked-LM one
    assert _rel(xn.grad[:, 0], xe.grad[:, 0]) < 3e-2
    for (n, p), (_, q) in zip(head.named_parameters(), eager.named_parameters()):
        assert _rel(p.grad, q.grad) < 3e-2, n
    # inference: the same outputs without autograd
    head.eval()
    set_backend("native")
    try:
        with torch.no_grad():
            inf = head(x, None, labels) if P else head(x, None)
    finally:
        set_backend("auto")
    assert torch.equal(inf[0], mlm.detach()) and torch.equal(inf[-1], nsp.detach())


# ---------------------------------------------------------------------------------------------
# one GPU: 2 BERT-large blocks + the pretraining head
# ---------------------------------------------------------------------------------------------
def _runner(use_graph, P=None, optim=None, micro_batches=2):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=2, num_attention_heads=16,
                         intermediate_size=4096, hidden_dropout_prob=0.0,
                         attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * 2
    head = dict(layer_type="BertTailForPreTraining", config=cfg.__dict__)
    if P is not None:
        head["max_predictions"] = P
    mc = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + [head]
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_pretraining_test")))])
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
                              optim or dict(optim_type="SGD", lr=0.05, momentum=0.9))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="PreTrainingLoss"),
                        timer_cfg=dict(root="/tmp/sky_pretraining_test"), logging_cfg=None,
                        micro_batches=micro_batches, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner, opt


def _batches(n, batch=32, seed=0):
    import skycomputing_b200 as sky

    ds = sky.SynthPretrainingDataset(num_samples=n * batch, max_seq_length=128,
                                     vocab_size=V_LARGE, seed=seed)
    return list(torch.utils.data.DataLoader(ds, batch_size=batch))


@pytest.mark.parametrize("P", [None, 20])
def test_pipeline_graph_matches_eager(nat, P):
    data = _batches(4)
    out = {}
    for name, use_graph in (("eager", False), ("graph", True)):
        runner, opt = _runner(use_graph, P)
        out[name] = [runner.train_iteration(d, l) for d, l in data]
        assert (runner.engine._graph is not None) == use_graph
        runner.engine.close()
    assert all(math.isfinite(x) for x in out["graph"])
    assert out["graph"][0] == out["eager"][0]
    for a, b in zip(out["eager"], out["graph"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)


def test_graph_replays_are_bit_equal(nat):
    data = _batches(1)
    losses = []
    for _ in range(2):
        runner, _ = _runner(True, 20, optim=dict(optim_type="SGD", lr=0.0))
        losses.append([runner.train_iteration(*data[0]) for _ in range(3)])
        runner.engine.close()
    assert losses[0] == losses[1]
    assert losses[0][1] == losses[0][2]    # lr 0: every replay computes the same step


def test_evaluate_matches_the_torch_accumulators(nat):
    import skycomputing_b200 as sky
    from skycomputing_b200.runner.metrics import (TorchEvalAccumulator, TorchTokenAccumulator,
                                                  pretraining_metrics)

    ds = sky.SynthPretrainingDataset(num_samples=2 * 32 + 5, max_seq_length=128,
                                     vocab_size=V_LARGE, seed=1)
    loader = lambda: torch.utils.data.DataLoader(ds, batch_size=32)  # noqa: E731
    for P in (None, 20):
        runner, _ = _runner(True, P)
        got = runner.evaluate(loader())
        assert runner.evaluate(loader()) == got           # replays the same graph
        tok, cls = TorchTokenAccumulator(V_LARGE, "cuda"), TorchEvalAccumulator(2, "cuda")
        head = runner.model.local_stage.layers[-1]
        runner.model.eval()
        with torch.no_grad():
            for data, labels in loader():
                # the short last batch padded as evaluate pads it (the head's native path needs
                # a batch that is a multiple of 8)
                pad = 32 - labels.shape[0]
                data = [torch.cat([t, t.new_zeros((pad,) + tuple(t.shape[1:]))]) for t in data]
                labels = torch.cat([labels, labels.new_full((pad, labels.shape[1]), -100)])
                # in the micro-batches evaluate runs (2 per batch)
                for chunk, lab in zip(zip(*(t.chunk(2) for t in data)), labels.chunk(2)):
                    outs = runner.model.local_module(*[t.cuda() for t in chunk])
                    mlm_l, nsp_l = split_pretraining_labels(lab.cuda())
                    tok.add(outs[0], mlm_l)
                    cls.add(outs[-1], nsp_l)
        want = pretraining_metrics(dict(mlm=tok.read(), nsp=cls.read()))
        assert got["mlm_n"] == want["mlm_n"] and got["nsp_n"] == want["nsp_n"] == len(ds)
        assert got["mlm_loss"] == pytest.approx(want["mlm_loss"], rel=1e-5)
        assert got["nsp_loss"] == pytest.approx(want["nsp_loss"], rel=1e-5)
        assert got["nsp_accuracy"] == want["nsp_accuracy"]
        assert got["mlm_accuracy"] == want["mlm_accuracy"]
        assert got["loss"] == pytest.approx(got["mlm_loss"] + got["nsp_loss"], rel=1e-12)
        assert isinstance(head, sky.models.BertTailForPreTraining)
        runner.engine.close()


@pytest.mark.parametrize("optim", [dict(optim_type="SGD", lr=0.01, momentum=0.9),
                                   dict(optim_type="LAMB", lr=2e-3)])
def test_training_lowers_the_loss(nat, optim):
    import skycomputing_b200 as sky

    # ids below 1024 of the 30528-token vocabulary, step 1: the progressions repeat often enough
    # to be learnt in a few dozen steps
    ds = sky.SynthPretrainingDataset(num_samples=60 * 32, max_seq_length=128, vocab_size=1024,
                                     seed=0, max_step=1)
    runner, _ = _runner(True, 20, optim=optim)
    losses = [runner.train_iteration(d, l)
              for d, l in torch.utils.data.DataLoader(ds, batch_size=32)]
    runner.engine.close()
    assert all(math.isfinite(x) for x in losses)
    assert sum(losses[-10:]) / 10 < 0.9 * sum(losses[:10]) / 10, losses[::5]
