"""Masked-language-model pretraining on the CPU: MaskedLMLoss, the MLM datasets' masking, the
analytic cost of BertTailForMaskedLM, the token accumulator and a 2-stage gloo pipeline that
trains and evaluates the MLM head."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import skycomputing_b200 as sky
from skycomputing_b200.dynamics.allocator import group_units
from skycomputing_b200.runner.metrics import TorchTokenAccumulator, token_metrics
from tests._dist_helpers import run_distributed


# ---------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------
def test_masked_lm_loss_matches_torch_cross_entropy():
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(3, 5, 11, generator=g, requires_grad=True)
    labels = torch.randint(0, 11, (3, 5), generator=g)
    labels[torch.rand(3, 5, generator=g) < 0.6] = -100
    labels[0, 0] = 4
    loss = sky.build_loss(dict(type="MaskedLMLoss"), torch.device("cpu"))
    assert isinstance(loss, sky.MaskedLMLoss)
    got = loss(logits, labels)
    want = F.cross_entropy(logits.reshape(-1, 11), labels.reshape(-1), ignore_index=-100)
    assert float(got.detach()) == pytest.approx(float(want), rel=1e-6)
    g1, = torch.autograd.grad(got, logits)
    g2, = torch.autograd.grad(want, logits)
    assert torch.allclose(g1, g2, atol=1e-7)
    # no labelled token: 0 and a zero gradient where torch's mean gives NaN
    none = torch.full((3, 5), -100)
    z = loss(logits, none)
    assert float(z) == 0.0
    assert torch.isnan(F.cross_entropy(logits.reshape(-1, 11), none.reshape(-1), ignore_index=-100))
    gz, = torch.autograd.grad(z, logits)
    assert torch.count_nonzero(gz) == 0


def test_cross_entropy_loss_is_unchanged():
    assert type(sky.build_loss(dict(type="CrossEntropyLoss"), torch.device("cpu"))) is torch.nn.CrossEntropyLoss


# ---------------------------------------------------------------------------------------------
# datasets
# ---------------------------------------------------------------------------------------------
def _mask_stats(ds, special_ids):
    n_label = n_mask = n_rand = n_keep = n_body = 0
    for i in range(len(ds)):
        (ids, tt, am), lab = ds[i]
        orig = ds.input_ids[i]
        lab_pos = lab != -100
        assert int(lab_pos.sum()) >= 1
        assert not bool(torch.isin(orig[lab_pos], torch.tensor(special_ids)).any())
        assert bool((am[lab_pos] == 1).all())
        assert torch.equal(lab[lab_pos], orig[lab_pos])
        assert torch.equal(ids[~lab_pos], orig[~lab_pos])
        n_label += int(lab_pos.sum())
        n_body += int(((am == 1) & ~torch.isin(orig, torch.tensor(special_ids))).sum())
        n_mask += int((ids[lab_pos] == ds.mask_id).sum())
        n_keep += int((ids[lab_pos] == orig[lab_pos]).sum())
        n_rand += int(((ids[lab_pos] != ds.mask_id) & (ids[lab_pos] != orig[lab_pos])).sum())
        # deterministic for (seed, index)
        (ids2, _, _), lab2 = ds[i]
        assert torch.equal(ids, ids2) and torch.equal(lab, lab2)
    return n_label, n_body, n_mask, n_rand, n_keep


def _check_split(n_label, n_body, n_mask, n_rand, n_keep):
    assert n_label / n_body == pytest.approx(0.15, abs=0.02)
    assert n_mask / n_label == pytest.approx(0.8, abs=0.03)
    # a random replacement can draw the original token: it then counts as unchanged
    assert n_rand / n_label == pytest.approx(0.1, abs=0.03)
    assert n_keep / n_label == pytest.approx(0.1, abs=0.03)


def test_synth_mlm_dataset_masking():
    ds = sky.SynthMLMDataset(num_samples=300, max_seq_length=64, vocab_size=30528, seed=3)
    stats = _mask_stats(ds, [ds.cls_id, ds.sep_id, 0])
    _check_split(*stats)
    (ids, tt, am), lab = ds[0]
    assert ids.shape == tt.shape == am.shape == lab.shape == (64,)
    assert ids.dtype == lab.dtype == torch.int64
    # the task: the body is an arithmetic progression, so a masked token follows from its neighbours
    body = ds.input_ids[5, 1:-1] - ds.first
    d = (body[1:] - body[:-1]) % (30528 - ds.first)
    assert bool((d == d[0]).all()) and 1 <= int(d[0]) <= 4
    other = sky.SynthMLMDataset(num_samples=300, max_seq_length=64, vocab_size=30528, seed=4)
    assert not torch.equal(other.input_ids, ds.input_ids)
    ro = sky.SynthMLMDataset(num_samples=4, max_seq_length=16, vocab_size=100, reference_order=True)
    (a, b, c), _ = ro[1]
    assert bool((b == 1).all()) and bool((c == 0).all())   # (input_ids, input_mask, segment_ids)


def _write_corpus(d):
    words = ["the", "cat", "sat", "on", "mat", "a", "dog", "ran", "far", "away", "and", "slept",
             "##s", "big", "red", "."]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    vp = os.path.join(d, "vocab.txt")
    with open(vp, "w") as f:
        f.write("\n".join(vocab) + "\n")
    g = torch.Generator().manual_seed(1)
    tp = os.path.join(d, "corpus.txt")
    with open(tp, "w") as f:
        for _ in range(200):
            n = int(torch.randint(3, 15, (1,), generator=g))
            f.write(" ".join(words[int(i)] for i in torch.randint(0, 12, (n,), generator=g)) + " .\n")
    return tp, vp


def test_masked_lm_dataset_from_text(tmp_path):
    tp, vp = _write_corpus(str(tmp_path))
    ds = sky.MaskedLMDataset(tp, vp, max_seq_length=32, seed=5)
    assert len(ds) > 50
    (ids, tt, am), lab = ds[len(ds) - 1]        # the packed tail: padded
    assert bool((am == 0).any()) and bool((ids[am == 0] == ds.pad_id).all())
    assert int(ds.input_ids[0, 0]) == ds.cls_id
    stats = _mask_stats(ds, [ds.cls_id, ds.sep_id, ds.pad_id, ds.mask_id, 1])
    _check_split(*stats)
    again = sky.MaskedLMDataset(tp, vp, max_seq_length=32, seed=5)
    assert torch.equal(again[7][1], ds[7][1])
    other = sky.MaskedLMDataset(tp, vp, max_seq_length=32, seed=6)
    assert any(not torch.equal(other[i][1], ds[i][1]) for i in range(10))


# ---------------------------------------------------------------------------------------------
# analytic cost
# ---------------------------------------------------------------------------------------------
def _mlm_cfg(layers=1, vocab=96, H=32, dropout=0.1):
    c = sky.BertConfig(vocab, hidden_size=H, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=2 * H, max_position_embeddings=32,
                       hidden_dropout_prob=dropout, attention_probs_dropout_prob=dropout)
    enc = [dict(layer_type="BertLayer_Head", config=c.__dict__),
           dict(layer_type="BertLayer_Body", config=c.__dict__),
           dict(layer_type="BertLayer_Tail", config=c.__dict__)] * layers
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] + enc
            + [dict(layer_type="BertTailForMaskedLM", config=c.__dict__)])


def test_analytic_cost_of_the_mlm_head_matches_measured():
    cfg = _mlm_cfg(2)
    gen = sky.build_data_generator("DataloaderGenerator", generator_cfg=dict(
        dataset_cfg=dict(type="SynthMLMDataset", num_samples=4, max_seq_length=16, vocab_size=96),
        dataloader_cfg=dict(batch_size=4)))
    f_meas, m_meas = sky.ModelBenchmarker(cfg, gen, device="cpu").benchmark()
    f_ana, m_ana = sky.ModelBenchmarker(cfg, gen, device="cpu", analytic=True).benchmark()
    B, S, H, V = 4, 16, 32, 96
    assert f_meas[-1] == 2 * B * S * H * (H + V)
    assert f_ana == pytest.approx(f_meas, rel=1e-6, abs=1e-6)
    assert m_ana == pytest.approx(m_meas, rel=0.05)


# ---------------------------------------------------------------------------------------------
# token accumulator
# ---------------------------------------------------------------------------------------------
def test_token_accumulator_totals():
    g = torch.Generator().manual_seed(2)
    acc = TorchTokenAccumulator(7)
    logits = torch.randn(2, 6, 7, generator=g)
    logits[0, 1] = torch.tensor([1.0, 3.0, 3.0, 0.0, 0.0, 0.0, 0.0])   # tie: the first maximum wins
    labels = torch.randint(0, 7, (2, 6), generator=g)
    labels[0, 1] = 1
    labels[1, :3] = -100
    labels[1, 3] = 9                                                     # invalid
    acc.add(logits[:1], labels[:1])
    acc.add(logits[1:], labels[1:])
    r = acc.read()
    flat, lab = logits.reshape(-1, 7), labels.reshape(-1)
    ok = (lab >= 0) & (lab < 7)
    assert r["count"] == int(ok.sum()) == 8 and r["invalid"] == 1 and r["classes"] == 7
    assert r["correct"] == int((flat[ok].argmax(1) == lab[ok]).sum())
    want = F.cross_entropy(flat[ok].double(), lab[ok], reduction="sum")
    assert r["loss_sum"] == pytest.approx(float(want), rel=1e-6)
    m = token_metrics(r["loss_sum"], r["count"], r["correct"])
    assert m["perplexity"] == pytest.approx(float(torch.exp(want / 8)), rel=1e-6)
    assert token_metrics(0.0, 0, 0) == dict(n=0, loss=None, accuracy=None, perplexity=None)


# ---------------------------------------------------------------------------------------------
# 2-stage pipeline: train and evaluate the MLM head
# ---------------------------------------------------------------------------------------------
def _mlm_runner(rank, world, tmp):
    cfg = _mlm_cfg(1, vocab=64, H=64, dropout=0.0)
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    alloc = sky.Allocator(cfg, wm, granularity="layer")
    units = group_units(cfg, "layer")
    n = len(units)
    bounds = [0, n - 1, n] if world == 2 else [0, n]     # the cut right in front of the head
    wm = alloc._assign(list(range(world)), bounds, units)
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=rank)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="Adam", lr=2e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=0, loss_cfg=dict(type="MaskedLMLoss"),
                      timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                      schedule="1f1b")


def _train_and_eval(rank, world, tmp):
    runner = _mlm_runner(rank, world, tmp)
    # step 1: the next-token rule a one-layer model picks up within a few hundred steps
    train = sky.SynthMLMDataset(num_samples=8 * 250, max_seq_length=16, vocab_size=64, seed=0,
                                max_step=1)
    losses = []
    for data, labels in torch.utils.data.DataLoader(train, batch_size=8):
        loss = runner.train_iteration(data, labels)
        if loss is not None:
            losses.append(loss)
    dev = sky.SynthMLMDataset(num_samples=21, max_seq_length=16, vocab_size=64, seed=1, max_step=1)
    out = runner.evaluate(torch.utils.data.DataLoader(dev, batch_size=8), name="dev")
    labelled = sum(int((dev[i][1] != -100).sum()) for i in range(len(dev)))
    runner.engine.close()
    return dict(losses=losses, eval=out, labelled=labelled)


def test_two_stage_pipeline_trains_and_evaluates_the_mlm_head(tmp_path):
    res = run_distributed(_train_and_eval, 2, str(tmp_path))
    losses = res[1]["losses"]
    assert res[0]["losses"] == []
    assert len(losses) == 250
    first, last = sum(losses[:10]) / 10, sum(losses[-10:]) / 10
    assert last < 0.85 * first, losses
    ev = res[0]["eval"]
    assert res[1]["eval"] == ev                      # the same dict on both ranks
    assert set(ev) == {"n", "loss", "accuracy", "perplexity"}
    # 21 sequences: 2 full batches + 5 padded to 8 with 2-D ignore_index labels; each token once
    assert ev["n"] == res[0]["labelled"]
    assert ev["perplexity"] == pytest.approx(math.exp(ev["loss"]), rel=1e-9)
    assert 0.0 <= ev["accuracy"] <= 1.0
