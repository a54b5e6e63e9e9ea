"""Evaluation on the GPU: the classify_eval kernel against the torch accumulator, the inference
span forward, the evaluation CUDA graph, training unaffected by evaluation, and a model that
learns a task it is then evaluated on."""
import json
import math
import os
import socket
import subprocess
import sys

import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.runner.metrics import TorchEvalAccumulator

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_GPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _nat():
    from skycomputing_b200.ops import native as nat

    return nat


# ---------------------------------------------------------------------------------------------
# classify_eval kernel
# ---------------------------------------------------------------------------------------------
def _batches(C, M, n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        logits = torch.randn(M, C, generator=g) * 3
        if i == 1:
            logits = logits.round()              # many ties: the first maximum must win
        if i == 2:
            # padded rows: _on_gpu slices them on the device, so the kernel sees row stride C + 5
            logits = torch.cat([logits, torch.randn(M, 5, generator=g)], 1)
        labels = torch.randint(0, C, (M,), generator=g)
        labels[i::4] = -100                      # ignored rows
        out.append((logits, labels))
    return out


def _on_gpu(logits, C):
    """(device view, host reference) of a batch; a padded batch stays a strided view on the GPU."""
    dev = logits.cuda()[:, :C]
    assert dev.stride(0) == logits.shape[1]
    return dev, logits[:, :C]


@pytest.mark.parametrize("C", [2, 3, 7, 1024])
@pytest.mark.parametrize("M", [1, 31, 256])
def test_classify_eval_matches_the_torch_accumulator(C, M):
    nat = _nat()
    acc = nat.EvalAccumulator(C, "cuda")
    ref = TorchEvalAccumulator(C)
    for logits, labels in _batches(C, M, 3, seed=C * 1000 + M):
        dev, host = _on_gpu(logits, C)
        acc.add(dev, labels.cuda())
        ref.add(host, labels)
    a, b = acc.read(), ref.read()
    assert a["count"] == b["count"] and a["invalid"] == b["invalid"] == 0
    assert torch.equal(a["confusion"], b["confusion"])
    assert a["loss_sum"] == pytest.approx(b["loss_sum"], rel=1e-6, abs=1e-9)


def test_classify_eval_nan_row_and_invalid_labels():
    nat = _nat()
    logits = torch.randn(6, 7, generator=torch.Generator().manual_seed(3))
    logits[2, 5] = float("nan")
    logits[2, 3] = float("nan")                   # two NaNs: the first one is the argmax
    labels = torch.tensor([0, 1, 2, 3, 9, -100])  # 9: invalid
    acc, ref = nat.EvalAccumulator(7, "cuda"), TorchEvalAccumulator(7)
    acc.add(logits.cuda(), labels.cuda())
    ref.add(logits, labels)
    a, b = acc.read(), ref.read()
    assert a["invalid"] == b["invalid"] == 1 and a["count"] == b["count"] == 4
    assert torch.equal(a["confusion"], b["confusion"])
    assert int(a["confusion"][2, 3]) == 1
    assert math.isnan(a["loss_sum"]) and math.isnan(b["loss_sum"])


def test_classify_eval_graph_replays_are_bit_identical():
    nat = _nat()
    C, M = 3, 256
    batches = [(_on_gpu(l, C)[0], t.cuda()) for l, t in _batches(C, M, 4, seed=11)]
    acc = nat.EvalAccumulator(C, "cuda")
    acc.reset()
    for logits, labels in batches:
        acc.add(logits, labels)
    eager = acc.buffer.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        acc.reset()
        for logits, labels in batches:
            acc.add(logits, labels)
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(acc.buffer, eager)


def test_classify_eval_rejects_more_than_1024_classes():
    nat = _nat()
    C = 1025
    buf = torch.zeros(3 + C * C, dtype=torch.int64, device="cuda")
    logits = torch.zeros(4, C, device="cuda")
    labels = torch.zeros(4, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="classify_eval failed with code 940"):
        nat.ext().classify_eval(logits=logits.data_ptr(), ldl=C, labels=labels.data_ptr(), M=4,
                                C=C, ignore_index=-100, acc=buf.data_ptr(),
                                stream=torch.cuda.current_stream().cuda_stream)
    with pytest.raises(ValueError):
        nat.EvalAccumulator(C, "cuda")


# ---------------------------------------------------------------------------------------------
# inference forward of the native spans
# ---------------------------------------------------------------------------------------------
def _stack(layer_types, cfg):
    from skycomputing_b200.builder import SequentialWrapper, build_layer

    return SequentialWrapper(*[build_layer(t, config=cfg.__dict__) for t in layer_types])


@pytest.mark.parametrize("S", [128, 96])
@pytest.mark.parametrize("types", [("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail"),
                                   ("BertLayer_Head",), ("BertLayer_Body", "BertLayer_Tail")])
def test_inference_span_forward_is_bit_identical(S, types, monkeypatch):
    """BERT-large block geometry (H = 1024, 16 heads, FFN 4096); S = 96 runs the tiled attention."""
    from skycomputing_b200.builder import ModuleWrapper
    from skycomputing_b200.models import set_backend
    from skycomputing_b200.ops.functions import BertSpanFn

    cfg = sky.BertConfig.bert_large()
    torch.manual_seed(0)
    set_backend("native")
    try:
        mw = ModuleWrapper(rank=0, module=_stack(types, cfg), module_to_cuda=True, cuda_device=0)
        mw.eval()
        B, H = 8, cfg.hidden_size
        m = torch.ones(B, S, device="cuda")
        m[0, S - 30:] = 0
        mask = ((1.0 - m) * -10000.0).view(B, 1, 1, S)
        if types[0] == "BertLayer_Body":
            args = [torch.randn(B, S, H, device="cuda").bfloat16(), mask]
        else:
            args = [torch.randn(B, S, H, device="cuda"), mask]
        calls = []
        real = BertSpanFn.infer
        monkeypatch.setattr(BertSpanFn, "infer",
                            staticmethod(lambda *a: calls.append(1) or real(*a)))
        with torch.enable_grad():
            ref = mw(*[a.clone().requires_grad_(a.is_floating_point() and a.dim() == 3)
                       for a in args])
        assert not calls
        with torch.no_grad():
            lean = mw(*args)
        assert calls                             # the inference path ran
        for r, l in zip(ref, lean):
            if torch.is_tensor(r) and r.is_floating_point():
                assert torch.equal(r.detach(), l)
    finally:
        set_backend("auto")


# ---------------------------------------------------------------------------------------------
# Runner.evaluate on one GPU
# ---------------------------------------------------------------------------------------------
def _model_cfg(layers=2, dropout=0.0, vocab=1000, classes=3):
    c = sky.BertConfig(vocab, hidden_size=256, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=1024, hidden_dropout_prob=dropout,
                       attention_probs_dropout_prob=dropout)
    enc = [dict(layer_type="BertLayer_Head", config=c.__dict__),
           dict(layer_type="BertLayer_Body", config=c.__dict__),
           dict(layer_type="BertLayer_Tail", config=c.__dict__)] * layers
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
            + [dict(layer_type="BertPooler", config=c.__dict__),
               dict(layer_type="BertTailForClassification", hidden_dropout_prob=dropout,
                    hidden_size=256, num_classes=classes)])


def _runner(use_graph=True, dropout=0.0, vocab=1000, optim=None, micro_batches=2, seed=500):
    mc = _model_cfg(dropout=dropout, vocab=vocab)
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_eval_test")))])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    for off, layer in enumerate(model.local_stage.layers.children()):
        gen = torch.Generator().manual_seed(seed + off)
        with torch.no_grad():
            for n, p in layer.named_parameters():
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module,
                              optim or dict(optim_type="SGD", lr=0.05, momentum=0.9))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_eval_test"), logging_cfg=None,
                        micro_batches=micro_batches, use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner


def _dev_loader(n=3 * 32 + 5, batch=32, seed=11, vocab=1000):
    ds = sky.SynthMNLIDataset(num_samples=n, max_seq_length=128, vocab_size=vocab, seed=seed,
                              full_length=False, label_rule="token")
    return torch.utils.data.DataLoader(ds, batch_size=batch)


def test_evaluate_graph_equals_eager():
    eager = _runner(use_graph=False)
    a = eager.evaluate(_dev_loader())
    assert getattr(eager.engine, "_eval", None) is None
    eager.engine.close()
    graphed = _runner(use_graph=True)
    b = graphed.evaluate(_dev_loader())
    c = graphed.evaluate(_dev_loader())          # a second pass replays the same graph
    assert graphed.engine._eval["graph"] is not None
    graphed.engine.close()
    assert a["n"] == 101
    assert a == b == c                           # bit for bit, loss included


def test_evaluate_matches_the_torch_backend():
    """Native (bf16 GEMMs, fp32 accumulation) against the fp32 torch layers, same weights.

    Tolerance from bf16: every GEMM input is rounded to 8 mantissa bits (relative error 2^-9),
    and about ten roundings lie between the embeddings and the logits, so logits may differ by a
    few 1e-2 relative to their scale; the mean loss is then within 2e-2 of the fp32 one, and a
    prediction may only flip on a row whose two largest fp32 logits are closer than twice the
    observed logit difference."""
    from skycomputing_b200.models import set_backend

    nat_runner = _runner(use_graph=True)
    got = nat_runner.evaluate(_dev_loader())
    nat_logits = []
    stage = nat_runner.model.local_stage
    stage.eval()
    with torch.no_grad():
        for data, _ in _dev_loader():
            nat_logits.append(stage(*[t.cuda() for t in data])[0].float())
    nat_runner.engine.close()
    set_backend("torch")
    try:
        ref_runner = _runner(use_graph=True)
        want = ref_runner.evaluate(_dev_loader())
        stage = ref_runner.model.local_stage
        stage.eval()
        ref_logits = []
        with torch.no_grad():
            for data, _ in _dev_loader():
                ref_logits.append(stage(*[t.cuda() for t in data])[0].float())
        ref_runner.engine.close()
    finally:
        set_backend("auto")
    nl, rl = torch.cat(nat_logits), torch.cat(ref_logits)
    diff = float((nl - rl).abs().max())
    assert diff <= 5e-2 * float(rl.abs().max()) + 1e-3
    top2 = rl.topk(2, dim=1).values
    fragile = int(((top2[:, 0] - top2[:, 1]) < 2 * diff).sum())
    assert got["n"] == want["n"] == 101
    assert abs(got["loss"] - want["loss"]) <= 2e-2 * max(1.0, want["loss"])
    assert abs(got["accuracy"] - want["accuracy"]) * got["n"] <= fragile


def _tensors(obj, out, prefix=""):
    if torch.is_tensor(obj):
        out[prefix] = obj.detach().clone()
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _tensors(v, out, f"{prefix}/{k}")
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _tensors(v, out, f"{prefix}/{i}")
    return out


def test_evaluation_inside_graphed_training_changes_nothing_training_reads():
    """Whole-step CUDA graph, dropout on, an evaluation after step 6 of 12.

    Two training runs from the same seed already differ in the last bits after a few steps
    (observed on H100 at the third step, without any evaluation), so the bit-for-bit check is on
    the state: every parameter, the optimizer state, the dropout RNG counters and the step graph's
    static buffers are the same tensors with the same bits after the evaluation as before it.  The
    loss trajectories of a run with and without the evaluation then agree within that rounding."""
    from skycomputing_b200.models import bert_layers

    span_streams = bert_layers._RNG_STREAM_COUNTER[0]

    def state(runner):
        eng = runner.engine
        out = _tensors(dict(runner.model.local_stage.state_dict()), {}, "params")
        _tensors(runner.optimizer.state_dict(), out, "optim")
        _tensors([r.state for r in bert_layers._RNG.values()], out, "rng")
        _tensors([eng._static_inputs, eng._static_labels, eng._loss_acc], out, "static")
        return out

    def run(evaluate: bool):
        # both runs start from the same dropout streams: span stream ids and the step counter
        bert_layers._RNG_STREAM_COUNTER[0] = span_streams
        for rng in bert_layers._RNG.values():
            rng.state[1].zero_()
        runner = _runner(use_graph=True, dropout=0.1)
        ds = sky.SynthMNLIDataset(num_samples=64, max_seq_length=128, vocab_size=1000, seed=3,
                                  full_length=False)
        losses = []
        for step in range(12):
            if evaluate and step == 6:
                torch.cuda.synchronize()
                before = state(runner)
                metrics = runner.evaluate(_dev_loader(n=40))
                assert runner.engine._eval["graph"] is not None and metrics["n"] == 40
                after = state(runner)
                assert sorted(before) == sorted(after)
                for k in before:
                    assert torch.equal(before[k], after[k]), k
            sl = slice((step % 4) * 16, (step % 4 + 1) * 16)
            losses.append(runner.train_iteration(
                [ds.input_ids[sl], ds.segment_ids[sl], ds.input_mask[sl]], ds.labels[sl]))
        torch.cuda.synchronize()
        assert runner.engine._graph is not None
        runner.engine.close()
        return losses

    plain, mixed = run(False), run(True)
    assert plain[0] == mixed[0]
    for a, b in zip(plain, mixed):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)   # the bound of the graph-vs-eager test


# measured on one NVIDIA H100 80GB HBM3 (700 W power limit), four runs: dev accuracy 0.318 before
# and 1.000 after the 300 steps (dev loss 1.100 -> 0.001-0.003; chance is 1/3).  The threshold
# leaves a wide margin below the measurement and stays far above chance.
LEARNED_ACCURACY = 0.9


def test_a_small_model_learns_the_token_task():
    vocab = 30                      # tokens 3..29 -> 27 token ids, label = id % 3
    runner = _runner(use_graph=True, dropout=0.1, vocab=vocab,
                     optim=dict(optim_type="AdamW", lr=5e-4, weight_decay=0.01))
    train = sky.SynthMNLIDataset(num_samples=32 * 300, max_seq_length=128, vocab_size=vocab,
                                 seed=21, full_length=False, label_rule="token")
    loader = torch.utils.data.DataLoader(train, batch_size=32, shuffle=True,
                                         generator=torch.Generator().manual_seed(0))
    runner._max_iters = 300
    before = runner.evaluate(_dev_loader(n=512, batch=64, seed=22, vocab=vocab))
    runner.train(loader)
    after = runner.evaluate(_dev_loader(n=512, batch=64, seed=22, vocab=vocab))
    runner.engine.close()
    print("token task: dev accuracy {:.4f} -> {:.4f}, loss {:.4f} -> {:.4f}".format(
        before["accuracy"], after["accuracy"], before["loss"], after["loss"]))
    assert after["n"] == 512
    assert after["accuracy"] >= LEARNED_ACCURACY, after


# ---------------------------------------------------------------------------------------------
# two GPUs: a fused-boundary pipeline evaluates like one stage
# ---------------------------------------------------------------------------------------------
def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _check(world: int) -> dict:
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "check_eval.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("CHECK ")][-1]
    return json.loads(line[len("CHECK "):])


@pytest.mark.multigpu
def test_two_stage_fused_pipeline_evaluates_like_one_stage():
    if N_GPU < 2:
        pytest.skip("needs 2 GPUs")
    one, two = _check(1), _check(2)
    assert two["fused_any"] and two["same_on_all_ranks"]
    assert two["before"] == one["before"]        # same weights, same kernels: bit-identical
    assert two["after"]["n"] == one["after"]["n"]
    assert two["after"]["loss"] == pytest.approx(one["after"]["loss"], rel=2e-2)

