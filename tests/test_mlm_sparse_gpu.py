"""Sparse masked-language-model decoding on the GPU: the mlm_gather / mlm_scatter kernels against
the reference slot helper (bit for bit, across calls and graph replays, bad arguments), the
native sparse head against the dense head and the eager head at BERT-large geometry, and a
one-GPU BERT-large pipeline with the sparse head (graph = eager, graph-safe optimizer, the dense
head's losses, launch count, evaluation, overflow)."""
import copy
import math

import pytest
import torch

from skycomputing_b200.ops.functions import mlm_slots_ref

pytestmark = pytest.mark.gpu
V_LARGE = 30528


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    if not native.available():
        pytest.skip("native extension not built")
    return native


def _labels(B, S, density, seed, V=1000):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.randint(0, V, (B, S), generator=g, device="cuda")
    lab[torch.rand(B, S, generator=g, device="cuda") >= density] = -100
    return lab


def _want_gather(hidden, labels, P, V):
    row, slot, lab = mlm_slots_ref(labels, P, -100, V)
    x = torch.zeros(row.numel(), hidden.shape[1], dtype=hidden.dtype, device=hidden.device)
    x[row >= 0] = hidden[row[row >= 0]]
    return x, slot, lab


def _want_scatter(dx_c, slot):
    d = torch.zeros(slot.numel(), dx_c.shape[1], dtype=dx_c.dtype, device=dx_c.device)
    d[slot >= 0] = dx_c[slot[slot >= 0]]
    return d


# ---------------------------------------------------------------------------------------------
# kernels against the reference slot helper
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("S", [16, 128, 200, 512])
@pytest.mark.parametrize("H", [64, 1024])
@pytest.mark.parametrize("P_kind", ["1", "20", "S"])
def test_gather_and_scatter_match_the_reference(nat, B, S, H, P_kind):
    P = S if P_kind == "S" else int(P_kind)
    V = 1000
    for k, density in enumerate((0.0, 0.15, 1.0)):
        seed = B * 100003 + S * 101 + H + P + k
        labels = _labels(B, S, density, seed, V)
        hidden = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
        x_c, slot, lab = nat.mlm_gather(hidden, labels, P, V)
        wx, wslot, wlab = _want_gather(hidden, labels, P, V)
        assert slot.dtype == torch.int32 and x_c.shape == (B * P, H)
        assert torch.equal(slot.long(), wslot), (density, P)
        assert torch.equal(lab, wlab), (density, P)
        assert torch.equal(x_c, wx), (density, P)
        again = nat.mlm_gather(hidden, labels, P, V)
        assert all(torch.equal(a, b) for a, b in zip(again, (x_c, slot, lab)))
        dx_c = torch.randn(B * P, H, device="cuda").to(torch.bfloat16)
        d = nat.mlm_scatter(dx_c, slot)
        assert torch.equal(d, _want_scatter(dx_c, wslot))
        assert torch.equal(nat.mlm_scatter(dx_c, slot), d)


def test_one_graph_replays_batches_with_different_label_counts(nat):
    B, S, H, P, V = 8, 128, 1024, 20, 30528
    hidden = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
    dx_c = torch.randn(B * P, H, device="cuda").to(torch.bfloat16)
    static = _labels(B, S, 0.15, 1, V)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x_c, slot, lab = nat.mlm_gather(hidden, static, P, V)
        nat.mlm_scatter(dx_c, slot)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        x_c, slot, lab = nat.mlm_gather(hidden, static, P, V)
        d = nat.mlm_scatter(dx_c, slot)
    seen = []
    for k, density in enumerate((0.15, 0.0, 1.0, 0.05, 0.3)):
        batch = _labels(B, S, density, 10 + k, V)
        static.copy_(batch)
        g.replay()
        torch.cuda.synchronize()
        wx, wslot, wlab = _want_gather(hidden, batch, P, V)
        assert torch.equal(slot.long(), wslot) and torch.equal(lab, wlab), density
        assert torch.equal(x_c, wx) and torch.equal(d, _want_scatter(dx_c, wslot)), density
        seen.append(int((batch != -100).sum()))
    assert len(set(seen)) == len(seen)
    static.copy_(_labels(B, S, 0.15, 10, V))
    g.replay()
    first = (x_c.clone(), d.clone())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(first[0], x_c) and torch.equal(first[1], d)


def test_bad_arguments_return_error_codes(nat):
    x = torch.zeros(4 * 16, 64, dtype=torch.bfloat16, device="cuda")
    lab = torch.full((4, 16), -100, dtype=torch.int64, device="cuda")
    out = torch.zeros(4 * 20, 64, dtype=torch.bfloat16, device="cuda")
    sor = torch.zeros(4 * 16, dtype=torch.int32, device="cuda")
    sl = torch.zeros(4 * 20, dtype=torch.int64, device="cuda")
    ok = dict(hidden=x.data_ptr(), labels=lab.data_ptr(), B=4, S=16, H=64, P=20, ignore_index=-100,
              V=100, slot_of_row=sor.data_ptr(), slot_labels=sl.data_ptr(), x_c=out.data_ptr())
    for change, code in ((dict(H=60), 960), (dict(P=0), 960), (dict(B=0), 960),
                         (dict(P=nat.ext().mlm_max_predictions() + 1), 960),
                         (dict(hidden=0), 961), (dict(slot_labels=0), 961),
                         (dict(x_c=out.data_ptr() + 2), 962)):
        with pytest.raises(RuntimeError, match="code {}".format(code)):
            nat.ext().mlm_gather(**dict(ok, **change))
    sc = dict(dx_c=out.data_ptr(), slot_of_row=sor.data_ptr(), rows=64, H=64, dhidden=x.data_ptr())
    for change, code in ((dict(H=12), 960), (dict(rows=0), 960), (dict(slot_of_row=0), 961),
                         (dict(dhidden=x.data_ptr() + 8), 962)):
        with pytest.raises(RuntimeError, match="code {}".format(code)):
            nat.ext().mlm_scatter(**dict(sc, **change))
    # the layer validates max_predictions against the kernel's limit
    from skycomputing_b200.models.bert_layers import BertTailForMaskedLM
    assert nat.ext().mlm_max_predictions() == BertTailForMaskedLM.MAX_PREDICTIONS_LIMIT
    nat.ext().mlm_gather(**ok)          # the unchanged arguments launch
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        nat.mlm_gather(x, lab.int(), 20, 100)


# ---------------------------------------------------------------------------------------------
# the head at BERT-large geometry: sparse against dense, and against the eager head
# ---------------------------------------------------------------------------------------------
def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _heads(P):
    import skycomputing_b200 as sky

    cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                         intermediate_size=4096)
    torch.manual_seed(0)
    dense = sky.build_layer("BertTailForMaskedLM", config=cfg.__dict__).cuda()
    with torch.no_grad():
        for n, p in dense.named_parameters():
            p.copy_(torch.randn_like(p) * 0.02)
            if n.endswith("LayerNorm.weight"):
                p.fill_(1.0)
    sparse = sky.build_layer("BertTailForMaskedLM", config=cfg.__dict__, max_predictions=P).cuda()
    sparse.load_state_dict(dense.state_dict())
    return dense, sparse, copy.deepcopy(sparse)


def _masked_labels(B, S, per_seq, seed, V=V_LARGE):
    """``per_seq`` labelled body positions per sequence, as the BERT masking produces."""
    g = torch.Generator().manual_seed(seed)
    lab = torch.full((B, S), -100, dtype=torch.int64)
    for b in range(B):
        pos = torch.randperm(S - 2, generator=g)[:per_seq] + 1
        lab[b, pos] = torch.randint(0, V, (per_seq,), generator=g)
    return lab.cuda()


def test_sparse_head_matches_the_dense_head_at_bert_large(nat):
    from skycomputing_b200.models import set_backend

    B, S, H, P = 8, 128, 1024, 20
    dense, sparse, eager = _heads(P)
    x = torch.randn(B, S, H, device="cuda").to(torch.bfloat16)
    labels = _masked_labels(B, S, 19, 0)
    set_backend("native")
    try:
        xd = x.clone().requires_grad_(True)
        ld = dense(xd, None)
        loss_d, g_d = nat.vocab_ce(ld.detach().view(-1, V_LARGE), labels.view(-1))
        ld.backward(g_d.view_as(ld))
        xs = x.clone().requires_grad_(True)
        ls, slot_labels = sparse(xs, None, labels)
        assert ls.shape == (B * P, V_LARGE) and ls.dtype == torch.bfloat16
        loss_s, g_s = nat.vocab_ce(ls.detach(), slot_labels)
        ls.backward(g_s)
        torch.cuda.synchronize()
        set_backend("torch")
        xe = x.float().requires_grad_(True)
        le, lab_e = eager(xe, None, labels)
        le.backward(g_s.float())
    finally:
        set_backend("auto")
    row, slot, want_lab = mlm_slots_ref(labels, P, -100, V_LARGE)
    assert torch.equal(slot_labels, want_lab) and torch.equal(lab_e, want_lab)
    assert float(loss_s) == pytest.approx(float(loss_d), rel=1e-6)
    decoded = row >= 0
    # the GEMMs' K order of an output element does not depend on M (stream-K is off by default):
    # a decoded row's logits and input gradient are the dense head's, bit for bit
    assert torch.equal(ls[decoded], ld.view(-1, V_LARGE)[row[decoded]])
    gs, gd = xs.grad.view(-1, H), xd.grad.view(-1, H)
    assert torch.count_nonzero(gs[slot < 0]) == 0
    assert torch.equal(gs[slot >= 0], gd[slot >= 0])
    for (n, p), (_, q) in zip(dense.named_parameters(), sparse.named_parameters()):
        assert _rel(q.grad, p.grad) < 1e-4, n
    # against the fp32 eager head: the bounds of the dense head's test
    assert _rel(ls, le) < 2e-2
    assert _rel(xs.grad, xe.grad) < 3e-2
    for (n, p), (_, q) in zip(sparse.named_parameters(), eager.named_parameters()):
        assert _rel(p.grad, q.grad) < 3e-2, n
    # inference (eval, no autograd): the same outputs; without labels the dense logits
    sparse.eval()
    dense.eval()
    set_backend("native")
    try:
        with torch.no_grad():
            li, lab_i = sparse(x, None, labels)
            assert torch.equal(li, ls.detach()) and torch.equal(lab_i, slot_labels)
            assert torch.equal(sparse(x, None), dense(x, None))
    finally:
        set_backend("auto")


# ---------------------------------------------------------------------------------------------
# one GPU: 2 BERT-large blocks + the sparse head
# ---------------------------------------------------------------------------------------------
def _runner(use_graph, P=None, micro_batches=2, optim=None):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=2, num_attention_heads=16,
                         intermediate_size=4096, hidden_dropout_prob=0.0,
                         attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * 2
    head = dict(layer_type="BertTailForMaskedLM", config=cfg.__dict__)
    if P is not None:
        head["max_predictions"] = P
    mc = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + [head]
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_mlm_sparse_test")))])
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
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="MaskedLMLoss"),
                        timer_cfg=dict(root="/tmp/sky_mlm_sparse_test"), logging_cfg=None,
                        micro_batches=micro_batches, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner, opt


def _batches(n, batch=16, seed=0):
    import skycomputing_b200 as sky

    ds = sky.SynthMLMDataset(num_samples=n * batch, max_seq_length=128, vocab_size=V_LARGE,
                             seed=seed)
    return list(torch.utils.data.DataLoader(ds, batch_size=batch))


def test_sparse_head_pipeline_on_one_gpu(nat):
    nat.enable_launch_counter()
    data = _batches(5)
    out = {}
    for name, use_graph, P in (("dense", True, None), ("eager", False, 20), ("graph", True, 20)):
        runner, opt = _runner(use_graph, P)
        assert opt.graph_safe
        losses = [runner.train_iteration(d, l) for d, l in data]
        out[name] = dict(losses=losses, graph=runner.engine._graph is not None,
                         launches=runner.engine.launches_per_step)
        # after training, a direct call (no labels bound) decodes every position
        runner.model.eval()
        with torch.no_grad():
            logits = runner.model(*[t.cuda() for t in data[0][0]])
        assert logits.shape == (16, 128, V_LARGE), name
        runner.engine.close()
    assert out["graph"]["graph"] and out["dense"]["graph"] and not out["eager"]["graph"]
    assert all(math.isfinite(x) for x in out["graph"]["losses"])
    assert out["graph"]["losses"][0] == out["eager"]["losses"][0]
    for a, b in zip(out["eager"]["losses"], out["graph"]["losses"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)
    for a, b in zip(out["dense"]["losses"], out["graph"]["losses"]):
        assert b == pytest.approx(a, rel=1e-2)
    # mlm_gather in forward, mlm_scatter in backward: 2 launches per micro-batch
    assert out["graph"]["launches"] == out["dense"]["launches"] + 2 * 2


def test_sparse_head_evaluate_matches_dense_and_overflow_is_loud(nat):
    import skycomputing_b200 as sky

    ds = sky.SynthMLMDataset(num_samples=2 * 16 + 5, max_seq_length=128, vocab_size=V_LARGE, seed=1)
    loader = lambda: torch.utils.data.DataLoader(ds, batch_size=16)  # noqa: E731
    got = {}
    for P in (None, 20):
        runner, _ = _runner(True, P)
        got[P] = runner.evaluate(loader())
        assert runner.engine._eval["graph"] is not None
        assert runner.evaluate(loader()) == got[P]          # replays the same graph
        runner.engine.close()
    assert got[20]["n"] == got[None]["n"] == sum(int((ds[i][1] != -100).sum())
                                                 for i in range(len(ds)))
    assert got[20]["loss"] == pytest.approx(got[None]["loss"], rel=1e-5)
    assert got[20]["accuracy"] == got[None]["accuracy"]
    # 19 labelled positions per sequence, P = 10: evaluate raises, the training loss is NaN
    runner, _ = _runner(True, 10)
    with pytest.raises(ValueError, match="max_predictions"):
        runner.evaluate(loader())
    (d, l), = _batches(1)
    assert math.isnan(runner.train_iteration(d, l))
    runner.engine.close()
