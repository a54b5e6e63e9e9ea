"""Evaluation on held-out data (CPU, gloo): metrics, Runner.evaluate across pipeline layouts,
padding of the short final batch, training unaffected by evaluation, hooks, launcher, GLUE dev."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import skycomputing_b200 as sky
from skycomputing_b200.runner.metrics import (PreTrainingAccumulator, TorchEvalAccumulator,
                                              TorchTokenAccumulator, classification_metrics,
                                              eval_accumulator)
from tests._dist_helpers import free_port, run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------
def test_classification_metrics_by_hand():
    # rows = labels, columns = predictions: tn=5 fp=2 / fn=1 tp=4
    m = classification_metrics([[5, 2], [1, 4]], loss_sum=6.0, count=12)
    assert m["n"] == 12 and m["loss"] == pytest.approx(0.5)
    assert m["accuracy"] == pytest.approx(9 / 12)
    assert m["f1"] == pytest.approx(2 * 4 / (2 * 4 + 2 + 1))
    assert m["mcc"] == pytest.approx((4 * 5 - 2 * 1) / ((4 + 2) * (4 + 1) * (5 + 2) * (5 + 1)) ** 0.5)
    assert m["confusion"] == [[5, 2], [1, 4]]
    # everything predicted negative: no true / false positives -> f1 and mcc denominators are 0
    z = classification_metrics([[3, 0], [2, 0]], 1.0, 5)
    assert z["f1"] == 0.0 and z["mcc"] == 0.0 and z["accuracy"] == pytest.approx(0.6)
    # a perfect classifier
    p = classification_metrics([[3, 0], [0, 2]], 0.0, 5)
    assert p["f1"] == 1.0 and p["mcc"] == pytest.approx(1.0)
    # three classes: no f1 / mcc
    t = classification_metrics([[1, 0, 0], [0, 2, 1], [0, 0, 3]], 7.0, 7)
    assert "f1" not in t and "mcc" not in t and t["accuracy"] == pytest.approx(6 / 7)
    # an empty pass does not raise
    e = classification_metrics([[0, 0], [0, 0]], 0.0, 0)
    assert e["n"] == 0 and e["loss"] is None and e["accuracy"] is None
    assert e["f1"] == 0.0 and e["mcc"] == 0.0


def test_torch_accumulator_skips_ignored_and_counts_invalid():
    acc = TorchEvalAccumulator(3)
    logits = torch.tensor([[1.0, 2.0, 0.0], [0.5, 0.5, 0.1], [3.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    acc.add(logits, torch.tensor([1, 0, -100, 5]))
    r = acc.read()
    assert r["count"] == 2 and r["invalid"] == 1
    # row 1 ties between classes 0 and 1: the first maximum wins
    assert r["confusion"].tolist() == [[1, 0, 0], [0, 1, 0], [0, 0, 0]]
    want = F.cross_entropy(logits[:2].double(), torch.tensor([1, 0]), reduction="sum")
    assert r["loss_sum"] == pytest.approx(float(want), rel=1e-12)


@pytest.mark.parametrize("layer_type", ["BertTailForClassification", "BertTailForMaskedLM",
                                        "BertTailForPreTraining"])
def test_declared_objective_picks_the_torch_accumulator_on_the_cpu(layer_type):
    c = sky.BertConfig(100, hidden_size=32, num_hidden_layers=1, num_attention_heads=4,
                       intermediate_size=64, max_position_embeddings=32).__dict__
    kw = (dict(hidden_dropout_prob=0.1, hidden_size=32, num_classes=3)
          if layer_type == "BertTailForClassification" else dict(config=c))
    head = sky.build_layer(layer_type, **kw)
    acc = eval_accumulator(head, -100, None)   # only a span head reads the loader
    assert acc.objective == head.objective
    pooled = layer_type == "BertTailForClassification"
    with torch.no_grad():
        logits = head(torch.randn(2, 32) if pooled else torch.randn(2, 4, 32))
    # the accumulator is made on the first batch: labels [B], [B, S] and [B, S + 1]
    S_labels = 5 if layer_type == "BertTailForPreTraining" else 4
    acc.add(logits, torch.zeros((2,) if pooled else (2, S_labels), dtype=torch.long))
    inner = acc.inner
    if layer_type == "BertTailForClassification":
        assert type(inner) is TorchEvalAccumulator and inner.C == 3
    elif layer_type == "BertTailForMaskedLM":
        assert type(inner) is TorchTokenAccumulator and inner.V == 100
    else:
        assert type(inner) is PreTrainingAccumulator
        assert type(inner.mlm) is TorchTokenAccumulator and inner.mlm.V == 100
        assert type(inner.nsp) is TorchEvalAccumulator and inner.nsp.C == 2


# ---------------------------------------------------------------------------------------------
# Runner.evaluate across pipeline layouts
# ---------------------------------------------------------------------------------------------
def _model_cfg(layers=2, dropout=0.1):
    c = sky.BertConfig(100, hidden_size=32, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=64, max_position_embeddings=32, hidden_dropout_prob=dropout,
                       attention_probs_dropout_prob=dropout)
    enc = [dict(layer_type="BertLayer_Head", config=c.__dict__),
           dict(layer_type="BertLayer_Body", config=c.__dict__),
           dict(layer_type="BertLayer_Tail", config=c.__dict__)] * layers
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
            + [dict(layer_type="BertPooler", config=c.__dict__),
               dict(layer_type="BertTailForClassification", hidden_dropout_prob=dropout,
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


def _workers(world, tmp):
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    return wm


def _dataset(n, seed=7, bad_label_at=None):
    ds = sky.SynthMNLIDataset(num_samples=n, max_seq_length=16, vocab_size=100, seed=seed,
                              label_rule="token")
    if bad_label_at is not None:
        ds.labels[bad_label_at] = 7
    return ds


def _loader(ds, batch=8, shuffle=False, seed=0):
    kw = dict(generator=torch.Generator().manual_seed(seed)) if shuffle else {}
    return torch.utils.data.DataLoader(ds, batch_size=batch, shuffle=shuffle, **kw)


def _runner(rank, world, tmp, granularity="layer", virtual_stages=1, layers=2, dropout=0.1,
            max_iters=0, micro_batches=2, ps=False, logging=False):
    cfg = _model_cfg(layers, dropout)
    wm = sky.Allocator(cfg, _workers(world, tmp), granularity=granularity).allocate(
        "even", virtual_stages=virtual_stages)
    model = sky.RpcModel(wm, this_rank=rank)
    _seed(model)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=0.05))
    log = dict(mode="a", filename=os.path.join(tmp, "allocation.log")) if logging else None
    return sky.Runner(model=model, parameter_server=sky.ParameterServer(cfg, lazy=True)
                      if (ps and rank == 0) else None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=max_iters, loss_cfg=dict(type="CrossEntropyLoss"),
                      timer_cfg=dict(root=tmp), logging_cfg=log, micro_batches=micro_batches,
                      schedule="1f1b")


def _evaluate(rank, world, tmp, granularity, virtual_stages, layers):
    runner = _runner(rank, world, tmp, granularity, virtual_stages, layers)
    out = runner.evaluate(_loader(_dataset(37)), name="dev")
    again = runner.evaluate(_loader(_dataset(37)), name="dev")
    assert again == out                        # passes are independent of each other
    assert runner.model.training is True       # the previous mode is restored
    assert runner.iter == 0 and runner.val_iter == 5
    runner.engine.close()
    return out


def _plain_loop(rank, world, tmp, layers):
    """The same model on one process, evaluated with F.cross_entropy / argmax by hand."""
    runner = _runner(0, 1, tmp, layers=layers)
    stage = runner.model.local_stage
    stage.eval()
    conf = torch.zeros(3, 3, dtype=torch.int64)
    loss, n = 0.0, 0
    with torch.no_grad():
        for data, labels in _loader(_dataset(37)):
            logits = torch.cat([stage(*chunk)[0] for chunk in zip(*(t.chunk(2) for t in data))])
            loss += float(F.cross_entropy(logits.double(), labels, reduction="sum"))
            for lab, pred in zip(labels.tolist(), logits.argmax(1).tolist()):
                conf[lab, pred] += 1
            n += labels.numel()
    return dict(confusion=conf.tolist(), loss=loss / n, n=n)


def test_evaluate_is_the_same_on_every_pipeline_layout(tmp_path):
    tmp = str(tmp_path)
    one = run_distributed(_evaluate, 1, tmp, "layer", 1, 2)
    two = run_distributed(_evaluate, 2, tmp, "layer", 1, 2)
    three = run_distributed(_evaluate, 3, tmp, "block", 1, 2)
    looped = run_distributed(_evaluate, 2, tmp, "block", 2, 4)
    looped_ref = run_distributed(_evaluate, 1, tmp, "block", 1, 4)
    ref = one[0]
    assert ref["n"] == 37                      # 4 full batches + 5 padded to 8
    for run in (two, three):
        for r in run:                          # every rank gets the last stage's metrics
            assert r == ref
    for r in looped:
        assert r == looped_ref[0]
    hand = run_distributed(_plain_loop, 1, tmp, 2)[0]
    assert hand["n"] == ref["n"] and hand["confusion"] == ref["confusion"]
    assert ref["loss"] == pytest.approx(hand["loss"], rel=1e-6)
    assert ref["accuracy"] == pytest.approx(sum(hand["confusion"][i][i] for i in range(3)) / 37)


def _evaluate_bad_label(rank, world, tmp):
    runner = _runner(rank, world, tmp)
    with pytest.raises(ValueError, match="outside"):
        runner.evaluate(_loader(_dataset(20, bad_label_at=13)))
    return True


def test_out_of_range_label_raises_on_every_rank(tmp_path):
    assert run_distributed(_evaluate_bad_label, 1, str(tmp_path)) == [True]
    assert run_distributed(_evaluate_bad_label, 2, str(tmp_path)) == [True, True]


def test_micro_batches_must_divide_the_eval_batch(tmp_path):
    runner = _runner(0, 1, str(tmp_path))
    with pytest.raises(ValueError, match="micro-batches"):
        runner.evaluate(_loader(_dataset(12), batch=6), micro_batches=4)


# ---------------------------------------------------------------------------------------------
# evaluation does not change training
# ---------------------------------------------------------------------------------------------
def _params(model) -> dict:
    out = {}
    for mod in model.model:
        if mod.is_local:
            for off, sd in enumerate(mod.get_state_dict()):
                for name, v in sd.items():
                    out[f"{mod.layer_range[0] + off}.{name}"] = v.detach().clone()
    return out


def _train_with_eval(rank, world, tmp, evaluate):
    runner = _runner(rank, world, tmp, max_iters=8, dropout=0.1)
    losses = []
    orig = runner.train_iteration

    def spy(data, labels):
        out = orig(data, labels)
        if out is not None:
            losses.append(out)
        return out

    runner.train_iteration = spy
    hook = sky.EvalHook(dict(dev=_loader(_dataset(20, seed=9))), interval=4, at_end=False)
    if evaluate:
        runner.register_hook(hook)
    runner.train(_loader(_dataset(64, seed=3), shuffle=True))
    runner.engine.close()
    return dict(losses=losses, params=_params(runner.model), evals=len(hook.history))


@pytest.mark.parametrize("world", [1, 2])
def test_train_eval_train_equals_train(tmp_path, world):
    plain = run_distributed(_train_with_eval, world, str(tmp_path), False)
    mixed = run_distributed(_train_with_eval, world, str(tmp_path), True)
    for a, b in zip(plain, mixed):
        assert b["evals"] == 2 and a["evals"] == 0
        assert a["losses"] == b["losses"]
        assert sorted(a["params"]) == sorted(b["params"])
        for k in a["params"]:
            assert torch.equal(a["params"][k], b["params"][k]), k


# ---------------------------------------------------------------------------------------------
# hooks
# ---------------------------------------------------------------------------------------------
class _Recorder(sky.Hook):
    def __init__(self):
        self.calls = []

    def before_val_epoch(self, runner):
        self.calls.append(("before_val_epoch", runner.iter))

    def after_val_epoch(self, runner):
        self.calls.append(("after_val_epoch", runner.iter))

    def before_val_iter(self, runner):
        self.calls.append(("before_val_iter", runner.val_iter))

    def after_val_iter(self, runner):
        self.calls.append(("after_val_iter", runner.val_iter))

    def after_train_iter(self, runner):
        self.calls.append(("after_train_iter", runner.iter))


def test_val_hooks_fire_in_order(tmp_path):
    runner = _runner(0, 1, str(tmp_path))
    rec = _Recorder()
    runner.register_hook(rec)
    runner.evaluate(_loader(_dataset(20)))
    assert rec.calls == [("before_val_epoch", 0),
                         ("before_val_iter", 0), ("after_val_iter", 1),
                         ("before_val_iter", 1), ("after_val_iter", 2),
                         ("before_val_iter", 2), ("after_val_iter", 3),
                         ("after_val_epoch", 0)]


def test_checkpoint_and_stop_hooks_ignore_evaluation(tmp_path):
    tmp = str(tmp_path)
    runner = _runner(0, 1, tmp, ps=True)
    ckpt = os.path.join(tmp, "ckpt")
    runner.register_hook(sky.CheckpointHook(save_path=ckpt, save_interval=1))
    stop = sky.StopHook(root=tmp, check_interval=1)
    runner.register_hook(stop)
    stop.before_run(runner)
    sky.StopHook.stop(tmp)          # a pending stop request is for the training loop
    runner.evaluate(_loader(_dataset(20)))
    assert not os.path.exists(ckpt) or not os.listdir(ckpt)
    assert not runner._stop and runner.iter == 0


def test_eval_hook_interval_and_save_best(tmp_path):
    runner = _runner(0, 1, str(tmp_path), max_iters=8)
    scripted = iter([0.5, 0.4, 0.6])
    seen = []

    def fake_evaluate(loader, name="val"):
        seen.append((runner.iter, name))
        return dict(n=1, loss=1.0, accuracy=next(scripted))

    runner.evaluate = fake_evaluate
    hook = sky.EvalHook(dict(dev=object()), interval=3, at_end=True, save_best="best.pth")
    saves = []
    hook._saver.save = lambda r, path: saves.append((r.iter, path))
    runner.register_hook(hook)
    runner.train(_loader(_dataset(64, seed=3)))
    runner.engine.close()
    assert seen == [(3, "dev"), (6, "dev"), (8, "dev")]
    # 0.5 (first) and 0.6 improve, 0.4 does not
    assert saves == [(3, "best.pth"), (8, "best.pth")]
    assert hook.best == 0.6


def test_eval_hook_by_epoch_without_duplicate_at_end(tmp_path):
    runner = _runner(0, 1, str(tmp_path), max_iters=4)
    seen = []
    runner.evaluate = lambda loader, name="val": seen.append(runner.iter) or dict(accuracy=0.0)
    runner.register_hook(sky.EvalHook(dict(dev=object()), by_epoch=True, at_end=True))
    runner.train(_loader(_dataset(32, seed=3)))
    runner.engine.close()
    assert seen == [4]


# ---------------------------------------------------------------------------------------------
# launcher + data
# ---------------------------------------------------------------------------------------------
def test_launcher_writes_val_metrics(tmp_path):
    env = dict(os.environ, TINY="1", LAYER_NUM="2", CORE_NUM="3", DEVICE="cpu", MAX_ITERS="4",
               PROJECT=str(tmp_path), ALLOCATE_TYPE="even", MICRO_BATCHES="2", BATCH_SIZE="8",
               EVAL_EVERY="2", EVAL_SAMPLES="20")
    out = subprocess.run([sys.executable, "-m", "skycomputing_b200.launch", "-c",
                          os.path.join(ROOT, "experiment", "config.py"), "--spawn", "2", "-p",
                          str(free_port())], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    d = os.path.join(str(tmp_path), "logs", "3nodes_2layers", "even")
    rows = [json.loads(line) for line in open(os.path.join(d, "metrics.jsonl"))]
    val = [r for r in rows if r.get("mode") == "val"]
    assert [r["iter"] for r in val] == [2, 4]
    assert all(r["name"] == "dev" and r["n"] == 20 and 0 <= r["accuracy"] <= 1 for r in val)
    assert len([r for r in rows if r.get("mode") != "val"]) == 4
    assert open(os.path.join(d, "allocation.log")).read().count("eval dev:") == 2


def test_synth_token_labels_are_a_function_of_the_tokens():
    a = sky.SynthMNLIDataset(num_samples=50, max_seq_length=16, vocab_size=100, seed=1,
                             label_rule="token")
    assert torch.equal(a.labels, a.input_ids[:, 1] % 3)
    b = sky.SynthMNLIDataset(num_samples=50, max_seq_length=16, vocab_size=100, seed=2,
                             label_rule="token")
    assert not torch.equal(a.input_ids, b.input_ids)
    r = sky.SynthMNLIDataset(num_samples=50, max_seq_length=16, vocab_size=100, seed=1)
    assert torch.equal(r.input_ids, a.input_ids)      # the default draws the same tokens
    with pytest.raises(ValueError):
        sky.SynthMNLIDataset(num_samples=4, label_rule="nope")


def test_glue_dev_split(tmp_path):
    from skycomputing_b200.dataset.bert_dataset import GlueDataset

    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "the", "cat", "sat", "dog", "ran", "a"]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab) + "\n")
    header = "\t".join(["index"] + ["c%d" % i for i in range(1, 8)] + ["s1", "s2", "label"])

    def rows(pairs):
        return header + "\n" + "\n".join(
            "\t".join([str(i)] + ["x"] * 7 + [a, b, lab]) for i, (a, b, lab) in enumerate(pairs))

    (tmp_path / "train.tsv").write_text(rows([("the cat", "sat", "neutral")] * 3))
    (tmp_path / "dev_matched.tsv").write_text(rows([("the dog", "ran", "entailment"),
                                                    ("a cat", "sat", "contradiction")]))
    (tmp_path / "dev_mismatched.tsv").write_text(rows([("a dog", "sat", "neutral")]))
    kw = dict(data_dir=str(tmp_path), bert_model="tiny", vocab_file=str(tmp_path / "vocab.txt"),
              max_seq_length=8, do_lower_case=True, processor="mnli", reference_order=False)
    train = GlueDataset(**kw)
    dev = GlueDataset(**kw, split="dev")
    mm = GlueDataset(**kw, split="dev_mismatched")
    assert (len(train), len(dev), len(mm)) == (3, 2, 1)
    assert [int(dev[i][1]) for i in range(2)] == [1, 0]
    (ids, tts, mask), _ = dev[0]
    assert ids.tolist()[:5] == [2, 4, 7, 3, 8] and int(mask.sum()) == 6
    # every split has its own feature cache
    names = sorted(os.listdir(tmp_path))
    assert "tiny_8_True" in names and "tiny_8_True_dev" in names and "tiny_8_True_dev_mismatched" in names
    with pytest.raises(ValueError):
        GlueDataset(**kw, split="test")


def test_suspended_probes_record_no_forward_time(tmp_path):
    from skycomputing_b200.builder import ModuleWrapper, SequentialWrapper

    mw = ModuleWrapper(rank=0, module=SequentialWrapper(torch.nn.Linear(4, 4)),
                       record_forward_time=True, slowdown=0.01,
                       timer_config=dict(root=str(tmp_path)))
    x = torch.randn(2, 4)
    mw(x)
    assert len(mw.forward_time) == 1
    with mw.suspend_forward_probes():
        for _ in range(3):
            mw(x)                    # still slowed down, but not timed
    assert len(mw.forward_time) == 1
    mw(x)
    assert len(mw.forward_time) == 2
