"""Extractive question answering on the CPU (torch backend, gloo): the span head's eager path,
the span loss, the span accumulator against a brute-force search, the synthetic and SQuAD
datasets, the official answer scores, a two-stage pipeline against one stage, fine-tuning from a
pretraining checkpoint and the estimator entry."""
from __future__ import annotations

import json
import math

import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.dataset.squad_dataset import SquadDataset, exact_match_score, f1_score
from skycomputing_b200.dynamics.allocator import group_units
from skycomputing_b200.dynamics.estimator import Estimator
from skycomputing_b200.dynamics.parameter_server import ParameterServer
from skycomputing_b200.ops.functions import split_span_labels
from skycomputing_b200.runner import QuestionAnsweringLoss, TorchSpanAccumulator, span_metrics
from skycomputing_b200.runner.metrics import eval_accumulator
from tests._dist_helpers import run_distributed

V, H, S = 64, 64, 16


def _cfg(layers=1):
    return sky.BertConfig(V, hidden_size=H, num_hidden_layers=layers, num_attention_heads=4,
                          intermediate_size=2 * H, max_position_embeddings=32,
                          hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


def _model_cfg(head="BertTailForQuestionAnswering", layers=2):
    c = _cfg(layers).__dict__
    enc = [dict(layer_type="BertLayer_Head", config=c), dict(layer_type="BertLayer_Body", config=c),
           dict(layer_type="BertLayer_Tail", config=c)] * layers
    return [dict(layer_type="BertEmbeddings", config=c)] + enc + [dict(layer_type=head, config=c)]


# ---------------------------------------------------------------------------------------------
# head and loss
# ---------------------------------------------------------------------------------------------
def test_head_matches_hf_formulas_in_fp64():
    torch.manual_seed(0)
    head = sky.build_layer("BertTailForQuestionAnswering", config=_cfg().__dict__)
    assert set(head.state_dict()) == {"qa_outputs.weight", "qa_outputs.bias"}
    assert head.objective == "span" and head.max_answer_length == 30
    x = torch.randn(3, S, H)
    logits = head(x, None)
    assert logits.shape == (3, 2, S) and logits.dtype == torch.float32
    w, b = head.qa_outputs.weight.double(), head.qa_outputs.bias.double()
    ref = x.double() @ w.t() + b                     # HF: [B, S, 2], split into start / end
    assert torch.allclose(logits[:, 0].double(), ref[..., 0], atol=1e-5)
    assert torch.allclose(logits[:, 1].double(), ref[..., 1], atol=1e-5)
    with pytest.raises(ValueError):
        sky.build_layer("BertTailForQuestionAnswering", config=_cfg().__dict__, max_answer_length=0)


def _hf_loss(logits, start, end):
    """HF total_loss for labels in range: the mean of the two token cross entropies."""
    ls = torch.nn.functional.cross_entropy(logits[:, 0].double(), start)
    le = torch.nn.functional.cross_entropy(logits[:, 1].double(), end)
    return (ls + le) / 2


def test_loss_matches_hf_and_handles_ignored_invalid_and_empty_rows():
    torch.manual_seed(1)
    logits = torch.randn(5, 2, S, requires_grad=True)
    start = torch.randint(0, S, (5,))
    end = torch.randint(0, S, (5,))
    lab = torch.stack([start, end, torch.zeros(5, dtype=torch.long), torch.full((5,), S - 1),
                       torch.full((5,), S - 1)], 1)
    loss_fn = QuestionAnsweringLoss()
    loss = loss_fn(logits, lab)
    assert float(loss.detach()) == pytest.approx(float(_hf_loss(logits.detach(), start, end)), rel=1e-6)
    # ignored rows: each mean over its own labelled rows, exact-zero gradient on ignored rows
    lab2 = lab.clone()
    lab2[1, 0] = -100
    lab2[3, 1] = -100
    loss2 = loss_fn(logits, lab2)
    keep_s, keep_e = lab2[:, 0] != -100, lab2[:, 1] != -100
    ref = (torch.nn.functional.cross_entropy(logits[keep_s, 0].double(), start[keep_s])
           + torch.nn.functional.cross_entropy(logits[keep_e, 1].double(), end[keep_e])) / 2
    assert float(loss2.detach()) == pytest.approx(float(ref), rel=1e-6)
    loss2.backward()
    assert torch.all(logits.grad[1, 0] == 0) and torch.all(logits.grad[3, 1] == 0)
    # no labelled row: 0; an invalid label: NaN
    none = lab.clone()
    none[:, :2] = -100
    assert float(loss_fn(logits, none)) == 0.0
    bad = lab.clone()
    bad[2, 1] = S
    assert math.isnan(float(loss_fn(logits, bad)))
    bad[2, 1] = -3
    assert math.isnan(float(loss_fn(logits, bad)))


def test_split_span_labels_columns():
    lab = torch.arange(10).view(2, 5)
    cols = split_span_labels(lab)
    assert [c.tolist() for c in cols] == [[0, 5], [1, 6], [2, 7], [3, 8], [4, 9]]


def test_build_loss_on_cpu_is_the_torch_loss():
    loss = sky.build_loss(dict(type="QuestionAnsweringLoss"), torch.device("cpu"))
    assert type(loss) is QuestionAnsweringLoss


# ---------------------------------------------------------------------------------------------
# span accumulator
# ---------------------------------------------------------------------------------------------
def _brute(st, en, lo, hi, ehi, L):
    best = None
    for i in range(max(lo, 0), min(hi, len(st) - 1) + 1):
        for j in range(i, min(i + L - 1, ehi, len(st) - 1) + 1):
            v = float(torch.tensor(st[i], dtype=torch.float32) + torch.tensor(en[j], dtype=torch.float32))
            if v != v:
                v = float("-inf")
            if best is None or v > best[2]:
                best = (i, j, v)
    return best or (-1, -1, float("-inf"))


def test_span_search_against_brute_force():
    g = torch.Generator().manual_seed(3)
    for trial in range(40):
        n = 12
        st = torch.randint(-3, 3, (n,), generator=g).float()     # many ties
        en = torch.randint(-3, 3, (n,), generator=g).float()
        if trial % 5 == 0:
            st[int(torch.randint(0, n, (1,), generator=g))] = float("nan")
        lo = int(torch.randint(-2, n, (1,), generator=g))
        hi = int(torch.randint(lo, n + 2, (1,), generator=g))
        ehi = int(torch.randint(0, n + 2, (1,), generator=g))
        L = int(torch.randint(1, 5, (1,), generator=g))
        got = TorchSpanAccumulator.best_span(st, en, lo, hi, ehi, L)
        want = _brute(st.tolist(), en.tolist(), lo, hi, ehi, L)
        assert got == want, (trial, got, want)
    # empty range, and the smallest (i, j) among equal scores
    z = torch.zeros(6)
    assert TorchSpanAccumulator.best_span(z, z, 4, 2, 5, 3) == (-1, -1, float("-inf"))
    assert TorchSpanAccumulator.best_span(z, z, 1, 5, 5, 3) == (1, 1, 0.0)
    # every score NaN: still the first valid pair, with score -inf
    nan = torch.full((6,), float("nan"))
    assert TorchSpanAccumulator.best_span(nan, z, 2, 5, 5, 3) == (2, 2, float("-inf"))


def test_span_f1_formula():
    f1 = TorchSpanAccumulator.span_f1
    assert f1(3, 5, 3, 5) == 1.0
    assert f1(-1, -1, 3, 5) == 0.0
    assert f1(0, 2, 3, 5) == 0.0
    p, r = 2 / 4, 2 / 3                               # pred [2, 5], gold [4, 6]: overlap 4..5
    assert f1(2, 5, 4, 6) == pytest.approx(2 * p * r / (p + r))


def test_accumulator_totals_and_predictions():
    torch.manual_seed(4)
    B = 6
    logits = torch.randn(B, 2, S)
    lab = torch.tensor([[2, 4, 1, 10, 12], [5, 5, 1, 10, 12], [-100, -100, 1, 10, 12],
                        [3, S, 1, 10, 12], [0, 1, 0, 15, 15], [-100] * 5])
    acc = TorchSpanAccumulator(max_answer_length=4, capacity=5)
    acc.add(logits, lab)
    t = acc.read()
    assert t["count"] == 3 and t["invalid"] == 1 and t["overflow"] == 1
    assert t["spans"].shape == (5, 2) and t["scores"].shape == (5,)
    rows = [0, 1, 4]
    ce = sum(float(torch.logsumexp(logits[b, c].double(), 0) - logits[b, c, int(lab[b, c])])
             for b in rows for c in (0, 1))
    assert t["start_loss_sum"] + t["end_loss_sum"] == pytest.approx(ce, rel=1e-9)
    for b in range(5):
        want = _brute(logits[b, 0].tolist(), logits[b, 1].tolist(), *lab[b, 2:].tolist(), 4)
        assert tuple(t["spans"][b].tolist()) == want[:2]
    m = span_metrics(t)
    assert m["n"] == 3 and m["loss"] == pytest.approx(ce / 6)
    assert set(m) == {"n", "loss", "start_accuracy", "end_accuracy", "exact", "f1"}
    assert span_metrics(dict(t, count=0))["loss"] is None


def test_eval_accumulator_follows_the_head_declaration():
    logits, lab = torch.randn(2, 2, S), torch.zeros(2, 5, dtype=torch.long)
    loader = torch.utils.data.DataLoader(list(range(8)), batch_size=4)
    head = sky.build_layer("BertTailForQuestionAnswering", config=_cfg().__dict__)
    acc = eval_accumulator(head, -100, loader)
    acc.add(logits, lab)
    assert isinstance(acc.inner, TorchSpanAccumulator)
    # without the declaration the same shapes reach the token accumulator
    acc = eval_accumulator(torch.nn.Linear(H, 2), -100, loader)
    acc.add(logits, lab[:, :2])
    assert not isinstance(acc.inner, TorchSpanAccumulator)


# ---------------------------------------------------------------------------------------------
# datasets and answer scores
# ---------------------------------------------------------------------------------------------
def test_synth_qa_dataset_layout_and_determinism():
    ds = sky.SynthQADataset(num_samples=40, max_seq_length=S, vocab_size=V, seed=0,
                            max_answer_tokens=4)
    again = sky.SynthQADataset(num_samples=40, max_seq_length=S, vocab_size=V, seed=0,
                               max_answer_tokens=4)
    other = sky.SynthQADataset(num_samples=40, max_seq_length=S, vocab_size=V, seed=1,
                               max_answer_tokens=4)
    lengths = set()
    for i in range(len(ds)):
        (ids, tt, mask), lab = ds[i]
        (ids2, _, _), lab2 = again[i]
        assert torch.equal(ids, ids2) and torch.equal(lab, lab2)
        n = int(mask.sum())
        lengths.add(n)
        assert ids[0] == 1 and ids[3] == 2 and ids[n - 1] == 2 and torch.all(ids[n:] == 0)
        assert torch.all(tt[:4] == 0) and torch.all(tt[4:n] == 1) and torch.all(tt[n:] == 0)
        start, end, lo, hi, ehi = lab.tolist()
        q1, q2 = int(ids[1]), int(ids[2])
        ctx = ids[4:n - 1].tolist()
        assert ctx.count(q1) == 1 and ctx.count(q2) == 1
        assert ids[start - 1] == q1 and ids[end + 1] == q2 and 1 <= end - start + 1 <= 4
        assert (lo, hi, ehi) == (4, n - 2, n - 2)
    assert len(lengths) > 3
    assert any(not torch.equal(ds[i][0][0], other[i][0][0]) for i in range(len(ds)))


def _squad_files(tmp_path, impossible=False):
    words = ("[PAD] [UNK] [CLS] [SEP] [MASK] the cat sat on a mat in paris , which is big . "
             "where did what was it city 1895 ( ) - 1943 year born").split()
    vocab = tmp_path / "vocab.txt"
    vocab.write_text("\n".join(words) + "\n")
    context = ("The cat sat on a mat in Paris, which is big. The cat was born (1895-1943) in "
               "Paris. The mat is big.")
    qas = [dict(id="q1", question="Where did the cat sit?",
                answers=[dict(text="on a mat", answer_start=context.index("on a mat")),
                         dict(text="a mat", answer_start=context.index("a mat"))]),
           dict(id="q2", question="What year?",
                answers=[dict(text="1895", answer_start=context.index("1895"))])]
    if impossible:
        qas[1]["is_impossible"] = True
    data = dict(version="1.1", data=[dict(title="t", paragraphs=[dict(context=context, qas=qas)])])
    js = tmp_path / "squad.json"
    js.write_text(json.dumps(data))
    return str(js), str(vocab), context


def test_squad_dataset_windows_labels_and_text(tmp_path):
    js, vocab, context = _squad_files(tmp_path)
    for split in ("train", "dev"):
        ds = SquadDataset(js, vocab, max_seq_length=24, doc_stride=6, max_query_length=8,
                          split=split)
        assert len(ds) > 2 * 2                          # several windows per question
        per_q = {}
        for idx in range(len(ds)):
            (ids, tt, mask), lab = ds[idx]
            ex, start, q, _ = ds.features[idx]
            per_q.setdefault(ex, []).append(start)
            gs, ge, lo, hi, ehi = lab.tolist()
            n = int(mask.sum())
            assert ids[0] == 2 and ids[q - 1] == 3 and ids[n - 1] == 3
            assert torch.all(tt[:q] == 0) and torch.all(tt[q:n] == 1)
            assert ehi == n - 2 and q <= lo and hi <= ehi
            if gs >= 0 and (gs, ge) != (0, 0):
                # the gold tokens are the answer's tokens, and the words they cover contain it
                gold = ds.examples[ex][1][0]
                toks = ds.tokenizer.convert_ids_to_tokens(ids[gs:ge + 1].tolist())
                assert toks == ds.tokenizer.tokenize(gold)
                assert gold.lower() in ds.answer_text(idx, gs, ge).lower()
            elif split == "dev":
                assert (gs, ge) == (-100, -100)
        for starts in per_q.values():
            assert starts == sorted(starts) and all(b - a == 6 for a, b in zip(starts, starts[1:]))
        # every document position is the start range of exactly one window (max context)
        for ex in per_q:
            owned = []
            for idx in range(len(ds)):
                e, start, q, _ = ds.features[idx]
                if e == ex:
                    lo, hi = ds.labels[idx, 2:4].tolist()
                    owned.extend(range(start + lo - q, start + hi - q + 1))
            assert sorted(owned) == list(range(len(owned)))


def test_squad_improved_span_and_v2_rejected(tmp_path):
    js, vocab, _ = _squad_files(tmp_path)
    ds = SquadDataset(js, vocab, max_seq_length=64, doc_stride=32, max_query_length=8)
    idx = [i for i, f in enumerate(ds.features) if f[0] == 1]
    gs, ge = ds.labels[idx[0], :2].tolist()
    assert gs == ge and ds.tokenizer.convert_ids_to_tokens([int(ds.input_ids[idx[0], gs])]) == ["1895"]
    js2, vocab2, _ = _squad_files(tmp_path, impossible=True)
    with pytest.raises(ValueError, match="is_impossible"):
        SquadDataset(js2, vocab2, max_seq_length=64)


def test_official_scores_and_text_scores(tmp_path):
    assert exact_match_score("The Cat!", "cat") == 1.0
    assert exact_match_score("a cat sat", "cat") == 0.0
    p, r = 1 / 2, 1 / 1                                # "cat sat" vs "the cat"
    assert f1_score("cat sat", "the cat") == pytest.approx(2 * p * r / (p + r))
    assert f1_score("dog", "cat") == 0.0
    js, vocab, _ = _squad_files(tmp_path)
    ds = SquadDataset(js, vocab, max_seq_length=64, doc_stride=32, max_query_length=8, split="dev")
    assert len(ds) == 2
    # q1: "on a mat" exact; q2: predict "(1895-1943)", which normalises to "18951943" != "1895"
    spans, scores = [], []
    for idx in range(2):
        gs, ge = ds.labels[idx, :2].tolist()
        if idx == 0:
            spans.append((gs, ge))
        else:
            q = ds.features[idx][2]
            toks = ds.tokenizer.convert_ids_to_tokens(ds.input_ids[idx, q:].tolist())
            spans.append((q + toks.index("("), q + toks.index(")")))
        scores.append(1.0)
    out = ds.text_scores(torch.tensor(spans), torch.tensor(scores))
    assert out["text_exact_match"] == pytest.approx(50.0)
    assert out["text_f1"] == pytest.approx(50.0)


# ---------------------------------------------------------------------------------------------
# pipeline, evaluation, checkpoints, estimator
# ---------------------------------------------------------------------------------------------
def _runner(rank, world, tmp, cut, mc=None, loss="QuestionAnsweringLoss"):
    cfg = mc or _model_cfg()
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    alloc = sky.Allocator(cfg, wm, granularity="layer")
    units = group_units(cfg, "layer")
    n = len(units)
    at = {"one": n, "head": n - 1, "blocks": 4}[cut]
    wm = alloc._assign(list(range(world)), [0, at, n] if world > 1 else [0, n], units)
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=rank)
    for module in model.model:
        if not module.is_local:
            continue
        b = module.layer_range[0] if module.layer_range is not None else 0
        for off, layer in enumerate(module.module.layers.children()):
            gen = torch.Generator().manual_seed(100 + b + off)
            with torch.no_grad():
                for name, p in layer.named_parameters():
                    p.copy_(torch.randn(p.shape, generator=gen) * 0.02)
                    if name.endswith("LayerNorm.weight"):
                        p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="Adam", lr=2e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=0, loss_cfg=dict(type=loss),
                      timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                      schedule="1f1b")


def _train_and_eval(rank, world, tmp, cut):
    runner = _runner(rank, world, tmp, cut)
    train = sky.SynthQADataset(num_samples=8 * 6, max_seq_length=S, vocab_size=V, seed=0,
                               max_answer_tokens=4)
    losses = [runner.train_iteration(d, l) for d, l in torch.utils.data.DataLoader(train, batch_size=8)]
    dev = sky.SynthQADataset(num_samples=21, max_seq_length=S, vocab_size=V, seed=1,
                             max_answer_tokens=4)
    out = runner.evaluate(torch.utils.data.DataLoader(dev, batch_size=8), name="dev")
    runner.engine.close()
    return dict(losses=[x for x in losses if x is not None], eval=out)


@pytest.mark.parametrize("cut", ["blocks", "head"])
def test_two_rank_pipeline_matches_one_stage(tmp_path, cut):
    one = run_distributed(_train_and_eval, 1, str(tmp_path), "one")[0]
    two = run_distributed(_train_and_eval, 2, str(tmp_path), cut)
    last = 1 if two[1]["losses"] else 0
    assert len(one["losses"]) == len(two[last]["losses"]) == 6
    assert all(math.isfinite(x) for x in one["losses"])
    assert two[last]["losses"] == pytest.approx(one["losses"], rel=1e-4)
    assert one["eval"]["n"] == 21
    for r in range(2):
        assert two[r]["eval"]["n"] == 21
        for k in ("exact", "start_accuracy", "end_accuracy"):
            assert two[r]["eval"][k] == one["eval"][k]
        for k in ("loss", "f1"):
            assert two[r]["eval"][k] == pytest.approx(one["eval"][k], rel=1e-4)


def test_tiny_launcher_config_selects_the_qa_task(monkeypatch):
    import os
    import runpy

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for k in ("TASK", "INIT_FROM", "SAVE_PATH", "SEQ_LEN", "SQUAD_TRAIN", "SQUAD_DEV", "VOCAB_FILE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("TASK", "squad")
    monkeypatch.setenv("TINY", "1")
    monkeypatch.setenv("EVAL_EVERY", "2")
    cfg = runpy.run_path(os.path.join(root, "experiment", "config.py"))
    assert cfg["model_config"][-1]["layer_type"] == "BertTailForQuestionAnswering"
    assert cfg["data_config"]["dataset_cfg"]["type"] == "SynthQADataset"
    assert cfg["data_config"]["eval_datasets"]["dev"]["seed"] == 1
    assert cfg["train_config"]["loss_cfg"]["type"] == "QuestionAnsweringLoss"
    monkeypatch.setenv("TINY", "0")
    monkeypatch.delenv("EVAL_EVERY")
    cfg = runpy.run_path(os.path.join(root, "experiment", "config.py"))
    assert cfg["data_config"]["dataset_cfg"]["max_seq_length"] == 384
    monkeypatch.setenv("SQUAD_TRAIN", "train.json")
    monkeypatch.setenv("VOCAB_FILE", "vocab.txt")
    cfg = runpy.run_path(os.path.join(root, "experiment", "config.py"))
    assert cfg["data_config"]["dataset_cfg"]["type"] == "SquadDataset"


def _from_pretraining(rank, world, tmp):
    from skycomputing_b200.runner.hooks_collection.checkpoint_hook import CheckpointHook

    pre_cfg = _model_cfg(head="BertTailForPreTraining")
    pre = _runner(rank, world, tmp, "one", mc=pre_cfg, loss="PreTrainingLoss")
    pre.parameter_server = ParameterServer(pre_cfg)
    path = tmp + "/pre.pth"
    CheckpointHook(save_path=tmp).save(pre, path)
    saved = torch.load(path)
    pre.engine.close()
    qa = _runner(rank, world, tmp, "one")
    qa.parameter_server = ParameterServer(_model_cfg())
    torch.manual_seed(1234)
    init = {k: v.clone() for k, v in qa.model.local_stage.layers.state_dict().items()}
    logs = []
    qa._log = logs.append
    CheckpointHook(load_checkpoint_from=path, from_pretraining=True).before_run(qa)
    now = qa.model.local_stage.layers.state_dict()
    res = dict(logs=logs)
    res["encoder_equal"] = all(torch.equal(now[k], saved[k]) for k in saved
                               if int(k.split(".")[0]) < 7)
    res["head_init"] = all(torch.equal(now[k], init[k]) for k in init if k.startswith("7."))
    qa.engine.close()
    return res


def test_fine_tune_from_a_pretraining_checkpoint(tmp_path):
    res = run_distributed(_from_pretraining, 1, str(tmp_path))[0]
    assert res["encoder_equal"] and res["head_init"]
    (msg,) = [m for m in res["logs"] if "pretraining checkpoint" in m]
    for part in ("transform.*", "decoder.*", "pooler.*", "seq_relationship.*",
                 "layer 7 (BertTailForQuestionAnswering)"):
        assert part in msg, msg


def test_estimator_entry():
    cfg = dict(layer_type="BertTailForQuestionAnswering", config=_cfg().__dict__)
    data = (torch.zeros(4, S, H),)
    flops, mem, outs = Estimator.analytic_layer_cost(cfg, data)
    assert flops == 2.0 * 4 * S * H * 2
    assert outs == [((4, 2, S), torch.float32)]
    assert mem > 0
