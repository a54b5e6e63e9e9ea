"""Extractive question answering on sm_90a: the four span-head kernels against fp64 references,
determinism across calls and graph replays, argument errors, the native accumulator against
TorchSpanAccumulator, the native head against its eager path, a one-GPU pipeline (graph, replays,
evaluation), training on SynthQADataset and fine-tuning from a pretraining checkpoint."""
from __future__ import annotations

import math

import pytest
import torch

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


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp(min=1e-30)))
    return torch.pow(2.0, e - 7)


def _span_labels(B, S, seed, ignore_frac=0.2):
    g = torch.Generator().manual_seed(seed)
    lo = torch.randint(0, S // 4, (B,), generator=g)
    hi = torch.randint(S // 2, S, (B,), generator=g)
    start = lo + torch.randint(0, 8, (B,), generator=g)
    end = torch.minimum(start + torch.randint(0, 6, (B,), generator=g), hi)
    lab = torch.stack([start, end, lo, hi, hi], 1)
    pad = torch.rand(B, generator=g) < ignore_frac
    lab[pad] = -100
    return lab


GEOMS = [(32, 384, 1024), (32, 128, 1024), (3, 72, 64)]


# ---------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,H", GEOMS)
def test_logits_forward_and_backward_against_fp64(nat, B, S, H):
    g = torch.Generator(device="cuda").manual_seed(B * S + H)
    hidden = torch.randn(B, S, H, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(2, H, device="cuda", generator=g) * 0.05
    b = torch.randn(2, device="cuda", generator=g)
    logits = nat.qa_logits(hidden, w, b)
    ref = torch.einsum("bsh,ch->bcs", hidden.double(), w.double()) + b.double().view(1, 2, 1)
    assert logits.shape == (B, 2, S) and _rel(logits, ref) <= 1e-5
    dl = torch.randn(B, 2, S, device="cuda", generator=g)
    dw = torch.zeros(2, H, device="cuda")
    db = torch.zeros(2, device="cuda")
    dh = nat.qa_logits_bwd(hidden, dl, w, dw, db)
    dh_ref = torch.einsum("bcs,ch->bsh", dl.double(), w.double())
    err = (dh.double() - dh_ref).abs()
    assert bool((err <= _bf16_ulp(dh_ref)).all()), float(err.max())
    dw_ref = torch.einsum("bcs,bsh->ch", dl.double(), hidden.double())
    assert _rel(dw, dw_ref) <= 1e-5 and _rel(db, dl.double().sum((0, 2))) <= 1e-5
    # the bank gradients accumulate; two calls give identical bits
    dw2, db2 = dw.clone(), db.clone()
    dh2 = nat.qa_logits_bwd(hidden, dl, w, dw2, db2)
    assert torch.equal(dh, dh2) and _rel(dw2, 2 * dw_ref) <= 1e-5
    assert torch.equal(nat.qa_logits(hidden, w, b), logits)


def _ce_ref(logits, lab, S):
    tot = 0.0
    for c in (0, 1):
        keep = (lab[:, c] >= 0) & (lab[:, c] < S)
        if keep.any():
            rows = logits[keep, c].double()
            tot += float((torch.logsumexp(rows, 1) - rows.gather(1, lab[keep, c:c + 1])[:, 0]).mean())
    return tot / 2


@pytest.mark.parametrize("B,S,H", GEOMS)
def test_span_ce_against_fp64(nat, B, S, H):
    g = torch.Generator(device="cuda").manual_seed(S)
    logits = torch.randn(B, 2, S, device="cuda", generator=g) * 3
    lab = _span_labels(B, S, seed=S).cuda()
    lab[0, 1] = -100                                   # an ignored end row alone
    acc = torch.zeros(1, device="cuda")
    loss, d = nat.qa_span_ce(logits, lab, grad_scale=0.5, loss_acc=acc)
    assert float(loss) == pytest.approx(_ce_ref(logits, lab, S), rel=1e-6)
    assert float(acc) == pytest.approx(0.5 * float(loss), rel=1e-6)
    x = logits.double().requires_grad_(True)
    ref = 0.0
    for c in (0, 1):
        keep = lab[:, c] != -100
        ref = ref + torch.nn.functional.cross_entropy(x[keep, c], lab[keep, c]) / 2
    (ref * 0.5).backward()
    assert _rel(d, x.grad) <= 1e-5
    assert torch.all(d[0, 1] == 0)
    loss2, d2 = nat.qa_span_ce(logits, lab, grad_scale=0.5)
    assert torch.equal(loss, loss2) and torch.equal(d, d2)
    none = lab.clone()
    none[:, :2] = -100
    l0, d0 = nat.qa_span_ce(logits, none)
    assert float(l0) == 0.0 and torch.all(d0 == 0)
    bad = lab.clone()
    bad[1, 0] = S
    lb, db_ = nat.qa_span_ce(logits, bad)
    assert math.isnan(float(lb)) and torch.all(db_[1, 0] == 0)


@pytest.mark.parametrize("B,S,H", GEOMS)
def test_span_eval_matches_the_torch_accumulator(nat, B, S, H):
    from skycomputing_b200.runner.metrics import TorchSpanAccumulator

    g = torch.Generator(device="cuda").manual_seed(B + S)
    # integer-valued logits: many equal scores exercise the tie rule; a few NaNs
    logits = torch.randint(-4, 5, (B, 2, S), device="cuda", generator=g).float()
    lab = _span_labels(B, S, seed=B + S).cuda()
    # NaN logits in the span search of two sequences whose gold labels are ignored (a NaN in a
    # counted row makes the loss sums NaN on both sides)
    lab[0] = torch.tensor([-100, -100, 0, 10, 12])
    lab[1 % B, :2] = -100
    logits[0, 0, 3] = float("nan")
    logits[1 % B, 1, 5] = float("nan")
    lab[-1] = torch.tensor([2, 1, 5, 3, 9])           # empty start range, gold end < start
    if B > 2:
        lab[1, 1] = S                                 # an invalid label
    L = 7
    cap = B + 4
    acc = nat.SpanEvalAccumulator(L, cap, "cuda")
    ref = TorchSpanAccumulator(L, cap)
    for _ in range(2):                               # the cursor appends
        acc.add(logits, lab)
        ref.add(logits, lab)
    got, want = acc.read(), ref.read()
    for k in ("count", "start_correct", "end_correct", "exact", "invalid", "overflow"):
        assert got[k] == want[k], k
    assert got["overflow"] == max(0, 2 * B - cap)
    assert torch.equal(got["spans"], want["spans"])
    assert torch.equal(got["scores"], want["scores"])
    for k in ("start_loss_sum", "end_loss_sum", "f1_sum"):
        assert got[k] == pytest.approx(want[k], rel=1e-6, abs=1e-9), k
    acc.reset()
    acc.add(logits, lab)
    again = acc.read()
    assert torch.equal(again["spans"], got["spans"][:B])
    assert again["f1_sum"] * 2 == got["f1_sum"]


def test_graph_replays_are_bit_equal_and_append(nat):
    B, S, H = 8, 128, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    hidden = torch.randn(B, S, H, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(2, H, device="cuda", generator=g) * 0.05
    b = torch.zeros(2, device="cuda")
    lab = _span_labels(B, S, seed=5).cuda()
    dw = torch.zeros(2, H, device="cuda")
    db = torch.zeros(2, device="cuda")
    loss_acc = torch.zeros(1, device="cuda")
    acc = nat.SpanEvalAccumulator(30, 3 * B, "cuda")
    outs = {}

    def body():
        dw.zero_()
        db.zero_()
        loss_acc.zero_()
        logits = nat.qa_logits(hidden, w, b)
        _, d = nat.qa_span_ce(logits, lab, loss_acc=loss_acc)
        outs["dh"] = nat.qa_logits_bwd(hidden, d, w, dw, db)
        acc.add(logits, lab)

    body()
    torch.cuda.synchronize()
    eager = (outs["dh"].clone(), dw.clone(), db.clone(), loss_acc.clone())
    acc.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    res = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        res.append((outs["dh"].clone(), dw.clone(), db.clone(), loss_acc.clone()))
    for a, b_ in zip(res[0], res[1]):
        assert torch.equal(a, b_)
    for a, b_ in zip(res[0], eager):
        assert torch.equal(a, b_)
    t = acc.read()
    assert t["spans"].shape[0] == 2 * B and torch.equal(t["spans"][:B], t["spans"][B:])


def test_argument_errors_and_launch_counter(nat):
    x = torch.zeros(2, 4, 12, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(2, 12, device="cuda")
    out = torch.zeros(2, 2, 4, device="cuda")
    e = nat.ext()
    with pytest.raises(RuntimeError, match="990"):
        e.qa_logits_fwd(hidden=x.data_ptr(), B=2, S=4, H=12, w=w.data_ptr(), b=w.data_ptr(),
                        logits=out.data_ptr())
    x16 = torch.zeros(2, 4, 16, dtype=torch.bfloat16, device="cuda")
    w16 = torch.zeros(2, 16, device="cuda")
    with pytest.raises(RuntimeError, match="991"):
        e.qa_logits_fwd(hidden=x16.data_ptr(), B=2, S=4, H=16, w=w16.data_ptr(), b=0,
                        logits=out.data_ptr())
    with pytest.raises(RuntimeError, match="992"):
        e.qa_logits_fwd(hidden=x16.data_ptr() + 2, B=2, S=4, H=16, w=w16.data_ptr(),
                        b=w16.data_ptr(), logits=out.data_ptr())
    lab = torch.zeros(2, 5, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="990"):
        e.qa_span_eval(logits=out.data_ptr(), labels=lab.data_ptr(), B=2, S=4,
                       max_answer_length=0, ignore_index=-100, acc=out.data_ptr(),
                       pred_spans=0, pred_scores=0, capacity=0)
    with pytest.raises(RuntimeError, match="991"):
        e.qa_span_ce(logits=out.data_ptr(), labels=0, B=2, S=4, ignore_index=-100,
                     dlogits=out.data_ptr())
    nat.enable_launch_counter()
    nat.reset_launch_counter()
    logits = nat.qa_logits(x16, w16, w16[0, :2].contiguous())
    _, d = nat.qa_span_ce(logits, lab)
    nat.qa_logits_bwd(x16, d, w16, torch.zeros_like(w16), torch.zeros(2, device="cuda"))
    nat.SpanEvalAccumulator(30, 2, "cuda").add(logits, lab)
    assert nat.launch_count() == 5


# ---------------------------------------------------------------------------------------------
# head
# ---------------------------------------------------------------------------------------------
def test_native_head_matches_the_eager_head(nat):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    torch.manual_seed(0)
    cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                         intermediate_size=4096)
    head = sky.build_layer("BertTailForQuestionAnswering", config=cfg.__dict__).cuda()
    x = torch.randn(4, 384, 1024, device="cuda").to(torch.bfloat16)
    gl = torch.randn(4, 2, 384, device="cuda")
    out = {}
    for backend in ("torch", "native"):
        set_backend(backend)
        for p in head.parameters():
            p.grad = None
        xh = x.clone().requires_grad_(True)
        logits = head(xh, None)
        logits.backward(gl)
        out[backend] = (logits.detach().float(), xh.grad.float(),
                        head.qa_outputs.weight.grad.clone(), head.qa_outputs.bias.grad.clone())
    set_backend("native")
    assert _rel(out["native"][0], out["torch"][0]) <= 1e-5
    assert _rel(out["native"][1], out["torch"][1]) <= 1e-2         # bf16 input gradient
    assert _rel(out["native"][2], out["torch"][2]) <= 1e-5
    assert _rel(out["native"][3], out["torch"][3]) <= 1e-5
    head.eval()
    with torch.no_grad():
        assert torch.equal(head(x, None), out["native"][0])
    loss = sky.build_loss(dict(type="QuestionAnsweringLoss"), torch.device("cuda", 0))
    assert hasattr(loss, "fused")


# ---------------------------------------------------------------------------------------------
# one GPU
# ---------------------------------------------------------------------------------------------
def _runner(use_graph, optim=None, head="BertTailForQuestionAnswering", small=False,
            loss="QuestionAnsweringLoss", micro_batches=2):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    if small:
        cfg = sky.BertConfig(1024, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                             intermediate_size=1024, hidden_dropout_prob=0.0,
                             attention_probs_dropout_prob=0.0)
    else:
        cfg = sky.BertConfig(V_LARGE, hidden_size=1024, num_hidden_layers=2,
                             num_attention_heads=16, intermediate_size=4096,
                             hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * 2
    mc = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + [
        dict(layer_type=head, config=cfg.__dict__)]
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_qa_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(900 + off)
        with torch.no_grad():
            for n, p in layer.named_parameters():
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module,
                              optim or dict(optim_type="SGD", lr=0.05, momentum=0.9))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type=loss),
                        timer_cfg=dict(root="/tmp/sky_qa_test"), logging_cfg=None,
                        micro_batches=micro_batches, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner, mc


def _loader(n, S=384, seed=0, batch=32, vocab=V_LARGE):
    import skycomputing_b200 as sky

    ds = sky.SynthQADataset(num_samples=n, max_seq_length=S, vocab_size=vocab, seed=seed)
    return torch.utils.data.DataLoader(ds, batch_size=batch)


def test_pipeline_graph_matches_eager_and_replays_are_bit_equal(nat):
    data = list(_loader(4 * 32))
    out = {}
    for name, use_graph in (("eager", False), ("graph", True)):
        runner, _ = _runner(use_graph)
        out[name] = [runner.train_iteration(d, l) for d, l in data]
        assert (runner.engine._graph is not None) == use_graph
        runner.engine.close()
    assert all(math.isfinite(x) for x in out["graph"])
    assert out["graph"][0] == out["eager"][0]
    for a, b in zip(out["eager"], out["graph"]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)
    losses = []
    for _ in range(2):
        runner, _ = _runner(True, optim=dict(optim_type="SGD", lr=0.0))
        losses.append([runner.train_iteration(*data[0]) for _ in range(3)])
        runner.engine.close()
    assert losses[0] == losses[1] and losses[0][1] == losses[0][2]


def test_evaluation_matches_the_torch_accumulator_and_leaves_training_bit_identical(nat):
    from skycomputing_b200.models import bert_layers
    from skycomputing_b200.runner.metrics import TorchSpanAccumulator, span_metrics

    data = list(_loader(3 * 32))
    dev = _loader(2 * 32 + 5, seed=1)
    runner, _ = _runner(True)
    b = [runner.train_iteration(d, l) for d, l in data[:2]]
    # the weights and the dropout RNG after two graphed steps
    state = [t.detach().clone() for t in runner.model.local_stage.parameters()]
    rng = [r.state.clone() for r in bert_layers._RNG.values()]
    got = runner.evaluate(dev)
    assert runner.evaluate(dev) == got                   # the same graph, the cursor reset
    after = [t.detach().clone() for t in runner.model.local_stage.parameters()]
    assert len(after) == len(state) and all(torch.equal(x, y) for x, y in zip(state, after))
    assert all(torch.equal(r.state, s0) for r, s0 in zip(bert_layers._RNG.values(), rng))
    assert got["n"] == 2 * 32 + 5
    ref = TorchSpanAccumulator(30, 3 * 32)
    runner.model.eval()
    with torch.no_grad():
        for d, lab in dev:
            pad = 32 - lab.shape[0]
            d = [torch.cat([t, t.new_zeros((pad,) + tuple(t.shape[1:]))]) for t in d]
            lab = torch.cat([lab, lab.new_full((pad, 5), -100)])
            for chunk, lb in zip(zip(*(t.chunk(2) for t in d)), lab.chunk(2)):
                outs = runner.model.local_module(*[t.cuda() for t in chunk])
                ref.add(outs[0] if isinstance(outs, (tuple, list)) else outs, lb)
    want = span_metrics(ref.read())
    for k in ("n", "start_accuracy", "end_accuracy", "exact"):
        assert got[k] == want[k], k
    for k in ("loss", "f1"):
        assert got[k] == pytest.approx(want[k], rel=1e-5), k
    runner.model.train(True)
    b.append(runner.train_iteration(*data[2]))      # the training graph after the evaluation
    assert all(math.isfinite(x) for x in b)
    runner.engine.close()


@pytest.mark.parametrize("optim", [dict(optim_type="SGD", lr=0.05, momentum=0.9),
                                   dict(optim_type="AdamW", lr=3e-4)])
def test_training_lowers_the_loss_and_raises_exact(nat, optim):
    # a 60-token body vocabulary: every token is q1 / q2 often enough to be learnt quickly
    runner, _ = _runner(True, optim=optim, small=True)
    dev = _loader(128, S=64, seed=1, vocab=64)
    before = runner.evaluate(dev)["exact"]
    losses = [runner.train_iteration(d, l) for d, l in _loader(300 * 32, S=64, vocab=64)]
    after = runner.evaluate(dev)
    runner.engine.close()
    assert all(math.isfinite(x) for x in losses)
    assert sum(losses[-20:]) < sum(losses[:20])
    if optim["optim_type"] == "AdamW":
        assert after["exact"] > before, (before, after)


def test_fine_tune_from_a_pretraining_checkpoint(nat, tmp_path):
    import skycomputing_b200 as sky
    from skycomputing_b200.dynamics.parameter_server import ParameterServer
    from skycomputing_b200.runner.hooks_collection.checkpoint_hook import CheckpointHook

    pre, pre_cfg = _runner(True, head="BertTailForPreTraining", loss="PreTrainingLoss")
    pre.parameter_server = ParameterServer(pre_cfg)
    path = str(tmp_path / "pre.pth")
    CheckpointHook(save_path=str(tmp_path)).save(pre, path)
    saved = torch.load(path)
    pre.engine.close()
    qa, qa_cfg = _runner(True)
    qa.parameter_server = ParameterServer(qa_cfg)
    CheckpointHook(load_checkpoint_from=path, from_pretraining=True).before_run(qa)
    now = qa.model.local_stage.layers.state_dict()
    assert all(torch.equal(now[k].cpu(), saved[k].cpu()) for k in saved if int(k.split(".")[0]) < 7)
    losses = [qa.train_iteration(d, l) for d, l in _loader(2 * 32)]
    assert all(math.isfinite(x) for x in losses)
    qa.engine.close()
    assert isinstance(qa.model.local_stage.layers[-1], sky.models.BertTailForQuestionAnswering)
