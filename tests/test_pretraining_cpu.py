"""Masked-LM + next-sentence pretraining on the CPU (torch backend, gloo): the head's eager path
against an fp64 composition of HF's formulas, the one-tensor label layout and PreTrainingLoss, both
datasets, 2-rank pipelines against one stage (cut between blocks, in front of the head, looped;
dense and sparse; tied and untied), evaluation metrics, and the pretrain -> classification
checkpoint round trip."""
import math

import pytest
import torch
import torch.nn.functional as F

import skycomputing_b200 as sky
from skycomputing_b200.dynamics.allocator import group_units
from skycomputing_b200.dynamics.parameter_server import ParameterServer
from skycomputing_b200.ops.functions import join_pretraining_labels, split_pretraining_labels
from skycomputing_b200.runner import PreTrainingLoss
from tests._dist_helpers import run_distributed

V, H, S = 64, 64, 16


def _cfg(layers=1):
    return sky.BertConfig(V, hidden_size=H, num_hidden_layers=layers, num_attention_heads=4,
                          intermediate_size=2 * H, max_position_embeddings=32,
                          hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


def _model_cfg(P=None, tie=False, layers=2, head="BertTailForPreTraining"):
    c = _cfg(layers).__dict__
    enc = [dict(layer_type="BertLayer_Head", config=c), dict(layer_type="BertLayer_Body", config=c),
           dict(layer_type="BertLayer_Tail", config=c)] * layers
    tail = dict(layer_type=head, config=c)
    if P is not None:
        tail["max_predictions"] = P
    if tie:
        tail["tie_word_embeddings"] = True
    return [dict(layer_type="BertEmbeddings", config=c)] + enc + [tail]


# ---------------------------------------------------------------------------------------------
# head
# ---------------------------------------------------------------------------------------------
def _gelu(x):
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _ln(x, w, b, eps=1e-12):
    u = x.mean(-1, keepdim=True)
    s = ((x - u) ** 2).mean(-1, keepdim=True)
    return w * (x - u) / torch.sqrt(s + eps) + b


def test_head_matches_hf_formulas_in_fp64():
    torch.manual_seed(0)
    head = sky.build_layer("BertTailForPreTraining", config=_cfg().__dict__)
    assert isinstance(head, sky.models.BertTailForMaskedLM)
    assert {k.split(".")[0] for k in head.state_dict()} == {"transform", "decoder", "pooler",
                                                          "seq_relationship"}
    x = torch.randn(3, S, H)
    xh = x.clone().requires_grad_(True)
    mlm, nsp = head(xh)
    gm, gn = torch.randn_like(mlm), torch.randn_like(nsp)
    torch.autograd.backward([mlm, nsp], [gm, gn])
    p = {k: v.detach().double().requires_grad_(True) for k, v in head.named_parameters()}
    xd = x.double().requires_grad_(True)
    t = _ln(_gelu(xd @ p["transform.dense_act.weight"].T + p["transform.dense_act.bias"]),
            p["transform.LayerNorm.weight"], p["transform.LayerNorm.bias"])
    mlm_d = t @ p["decoder.weight"].T + p["decoder.bias"]
    pooled = torch.tanh(xd[:, 0] @ p["pooler.dense_act.weight"].T + p["pooler.dense_act.bias"])
    nsp_d = pooled @ p["seq_relationship.weight"].T + p["seq_relationship.bias"]
    torch.autograd.backward([mlm_d, nsp_d], [gm.double(), gn.double()])
    assert torch.allclose(mlm.double(), mlm_d, rtol=1e-4, atol=1e-5)
    assert torch.allclose(nsp.double(), nsp_d, rtol=1e-4, atol=1e-5)
    assert torch.allclose(xh.grad.double(), xd.grad, rtol=1e-4, atol=1e-5)
    for n, q in head.named_parameters():
        assert torch.allclose(q.grad.double(), p[n].grad, rtol=1e-4, atol=1e-5), n


def test_sparse_head_returns_slot_labels_and_nsp_logits():
    torch.manual_seed(0)
    head = sky.build_layer("BertTailForPreTraining", config=_cfg().__dict__, max_predictions=4)
    x = torch.randn(2, S, H)
    lab = torch.full((2, S + 1), -100)
    lab[0, 3], lab[1, 5], lab[:, S] = 7, 9, torch.tensor([0, 1])
    logits, slots, nsp = head(x, None, lab)
    assert logits.shape == (8, V) and nsp.shape == (2, 2)
    assert slots.tolist() == [7, -100, -100, -100, 9, -100, -100, -100]
    mlm_dense, nsp_dense = head(x)     # without labels: the dense outputs
    assert torch.allclose(logits[0], mlm_dense[0, 3], atol=1e-6)
    assert torch.equal(nsp, nsp_dense)
    with pytest.raises(ValueError, match="max_predictions"):
        sky.build_layer("BertTailForPreTraining", config=_cfg().__dict__)(x, None, lab)


def test_native_param_banks_list_every_bank_once():
    from skycomputing_b200.models.bert_layers import native_param_banks

    head = sky.build_layer("BertTailForPreTraining", config=_cfg().__dict__)
    banks = native_param_banks(head)
    params = [p for b in banks for p in b.params]
    assert len(params) == len({id(p) for p in params}) == len(list(head.parameters()))


# ---------------------------------------------------------------------------------------------
# labels and loss
# ---------------------------------------------------------------------------------------------
def test_label_helper_round_trip():
    lab = torch.arange(2 * 6).view(2, 6)
    mlm, nsp = split_pretraining_labels(lab)
    assert mlm.tolist() == [[0, 1, 2, 3, 4], [6, 7, 8, 9, 10]] and nsp.tolist() == [5, 11]
    assert torch.equal(join_pretraining_labels(mlm, nsp), lab)
    assert torch.equal(join_pretraining_labels(mlm.reshape(-1), nsp), lab)


def test_pretraining_loss_is_the_sum_of_the_two_means():
    torch.manual_seed(0)
    mlm, nsp = torch.randn(3, S, V), torch.randn(3, 2)
    lab = torch.full((3, S + 1), -100)
    lab[:, 2] = torch.tensor([1, 2, 3])
    lab[0, 5] = 4
    lab[:, S] = torch.tensor([0, 1, -100])
    got = PreTrainingLoss()((mlm, nsp), lab)
    m = F.cross_entropy(mlm.reshape(-1, V), lab[:, :S].reshape(-1), reduction="sum") / 4
    n = F.cross_entropy(nsp, lab[:, S], reduction="sum") / 2
    assert float(got) == pytest.approx(float(m + n), rel=1e-6)
    # every row ignored: 0, not NaN
    none = torch.full((3, S + 1), -100)
    assert float(PreTrainingLoss()((mlm, nsp), none)) == 0.0
    bad = lab.clone()
    bad[0, S] = 5
    with pytest.raises((IndexError, RuntimeError)):
        PreTrainingLoss()((mlm, nsp), bad)


# ---------------------------------------------------------------------------------------------
# datasets
# ---------------------------------------------------------------------------------------------
def test_synth_pretraining_dataset_layout():
    ds = sky.SynthPretrainingDataset(num_samples=64, max_seq_length=S, vocab_size=V, seed=3)
    nsp = []
    for i in range(len(ds)):
        (ids, tt, am), lab = ds[i]
        assert ids.shape == tt.shape == am.shape == (S,) and lab.shape == (S + 1,)
        seps = (ids == ds.sep_id).nonzero()[:, 0].tolist()
        assert ids[0] == ds.cls_id and seps[-1] == S - 1
        a_end = int(ds.len_a[i]) + 1
        assert ids[a_end] == ds.sep_id
        assert tt[:a_end + 1].eq(0).all() and tt[a_end + 1:].eq(1).all() and am.eq(1).all()
        mlm = lab[:S]
        assert mlm[[0, a_end, S - 1]].eq(-100).all()       # specials are never masked
        assert mlm.ne(-100).sum() == max(1, round(0.15 * (S - 3)))
        # unmasked body: A is a progression, B continues it exactly when the label is 0
        body = torch.where(mlm != -100, mlm, ids)
        seq = torch.cat([body[1:a_end], body[a_end + 1:S - 1]])
        span, first = V - ds.first, ds.first
        step = (seq[1] - seq[0]) % span if a_end > 2 else int(ds.step[i])
        cont = bool((((seq[1:] - seq[:-1]) % span) == step).all())
        assert cont == (int(lab[S]) == 0), i
        nsp.append(int(lab[S]))
        assert seq.ge(first).all()
        a2 = ds[i]
        assert torch.equal(a2[0][0], ids) and torch.equal(a2[1], lab)
    assert sum(nsp) == 32
    other = sky.SynthPretrainingDataset(num_samples=64, max_seq_length=S, vocab_size=V, seed=4)
    assert not torch.equal(other[0][0][0], ds[0][0][0])


def _corpus(tmp_path, docs):
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + ["w{}".format(i) for i in range(40)]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab) + "\n")
    text = "\n\n".join("\n".join(" ".join("w{}".format((d * 7 + s * 3 + k) % 40)
                                          for k in range(3 + s % 3)) for s in range(5))
                       for d in range(docs))
    (tmp_path / "corpus.txt").write_text(text + "\n")
    return str(tmp_path / "corpus.txt"), str(tmp_path / "vocab.txt")


def test_text_pretraining_dataset(tmp_path):
    text, vocab = _corpus(tmp_path, 4)
    ds = sky.dataset.PreTrainingDataset(text, vocab, max_seq_length=S, seed=1)
    assert len(ds) == 20
    nsp = []
    for i in range(len(ds)):
        (ids, tt, am), lab = ds[i]
        n = int(am.sum())
        seps = (ids[:n] == ds.sep_id).nonzero()[:, 0].tolist()
        assert ids[0] == ds.cls_id and len(seps) == 2 and seps[1] == n - 1 and n <= S
        assert tt[:seps[0] + 1].eq(0).all() and tt[seps[0] + 1:n].eq(1).all()
        assert tt[n:].eq(0).all() and ids[n:].eq(ds.pad_id).all()
        assert lab[[0, seps[0], n - 1]].eq(-100).all() and lab[n:S].eq(-100).all()
        nsp.append(int(lab[S]))
        again = sky.dataset.PreTrainingDataset(text, vocab, max_seq_length=S, seed=1)[i]
        assert torch.equal(again[0][0], ids) and torch.equal(again[1], lab)
    assert 0 < sum(nsp) < len(nsp)
    # 50/50 over many items: 40 documents of 5 sentences, 200 items
    many, _ = _corpus(tmp_path, 40)
    big = sky.dataset.PreTrainingDataset(many, vocab, max_seq_length=S, seed=2)
    share = sum(int(big[i][1][S]) for i in range(len(big))) / len(big)
    assert 0.4 < share < 0.6, share
    one, vocab = _corpus(tmp_path, 1)
    with pytest.raises(ValueError, match="at least two"):
        sky.dataset.PreTrainingDataset(one, vocab, max_seq_length=S)


# ---------------------------------------------------------------------------------------------
# pipelines, evaluation, checkpoints
# ---------------------------------------------------------------------------------------------
def _runner(rank, world, tmp, P, tie, cut, loss="PreTrainingLoss", head="BertTailForPreTraining",
            mc=None):
    cfg = mc or _model_cfg(P, tie, head=head)
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    if cut == "looped":
        wm = sky.Allocator(cfg, wm, granularity="layer").allocate("even", virtual_stages=2)
    else:
        alloc = sky.Allocator(cfg, wm, granularity="layer")
        units = group_units(cfg, "layer")
        n = len(units)
        at = {"one": n, "head": n - 1, "blocks": 4}[cut]
        wm = alloc._assign(list(range(world)), [0, at, n] if world > 1 else [0, n], units)
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=rank)
    # the same weights whatever the partition: seeded by global layer index
    for module in model.model:
        if not module.is_local:
            continue
        b = module.layer_range[0] if module.layer_range is not None else 0
        for off, layer in enumerate(module.module.layers.children()):
            gen = torch.Generator().manual_seed(100 + b + off)
            with torch.no_grad():
                for n, p in layer.named_parameters():
                    if n == "decoder.weight" and getattr(layer, "tie_word_embeddings", False):
                        continue   # the word-embedding table's (replica synced at setup)
                    p.copy_(torch.randn(p.shape, generator=gen) * 0.02)
                    if n.endswith("LayerNorm.weight"):
                        p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="Adam", lr=2e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=0, loss_cfg=dict(type=loss),
                      timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                      schedule="1f1b")


def _train_and_eval(rank, world, tmp, P, tie, cut):
    runner = _runner(rank, world, tmp, P, tie, cut)
    train = sky.SynthPretrainingDataset(num_samples=8 * 6, max_seq_length=S, vocab_size=V, seed=0)
    losses = [runner.train_iteration(d, l) for d, l in torch.utils.data.DataLoader(train, batch_size=8)]
    dev = sky.SynthPretrainingDataset(num_samples=21, max_seq_length=S, vocab_size=V, seed=1)
    out = runner.evaluate(torch.utils.data.DataLoader(dev, batch_size=8), name="dev")
    runner.engine.close()
    return dict(losses=[x for x in losses if x is not None], eval=out)


@pytest.mark.parametrize("cut", ["blocks", "head", "looped"])
@pytest.mark.parametrize("P,tie", [(None, False), (None, True), (4, False), (4, True)])
def test_two_rank_pipeline_matches_one_stage(tmp_path, cut, P, tie):
    one = run_distributed(_train_and_eval, 1, str(tmp_path), P, tie, "one")[0]
    two = run_distributed(_train_and_eval, 2, str(tmp_path), P, tie, cut)
    last = 1 if two[1]["losses"] else 0
    assert len(one["losses"]) == len(two[last]["losses"]) == 6
    assert two[last]["losses"] == pytest.approx(one["losses"], rel=1e-4)
    for r in range(2):
        for k in ("mlm_n", "nsp_n"):
            assert two[r]["eval"][k] == one["eval"][k]
        assert two[r]["eval"]["loss"] == pytest.approx(one["eval"]["loss"], rel=1e-4)


def test_sparse_and_dense_heads_agree_and_evaluation_is_direct(tmp_path):
    def run(P):
        return run_distributed(_train_and_eval, 1, str(tmp_path), P, False, "one")[0]

    dense, sparse = run(None), run(4)
    assert sparse["losses"] == pytest.approx(dense["losses"], rel=1e-5)
    assert sparse["eval"]["loss"] == pytest.approx(dense["eval"]["loss"], rel=1e-5)


def _eval_direct(rank, world, tmp):
    from skycomputing_b200.models.bert_layers import set_backend

    set_backend("torch")
    runner = _runner(rank, world, tmp, None, False, "one")
    dev = sky.SynthPretrainingDataset(num_samples=21, max_seq_length=S, vocab_size=V, seed=1)
    got = runner.evaluate(torch.utils.data.DataLoader(dev, batch_size=8), name="dev")
    runner.model.eval()
    mlm_sum = nsp_sum = 0.0
    mlm_n = nsp_ok = 0
    with torch.no_grad():
        for (ids, tt, am), lab in torch.utils.data.DataLoader(dev, batch_size=21):
            outs = runner.model.local_module(ids, tt, am)
            mlm, nsp = outs[0], outs[-1]
            ml, nl = split_pretraining_labels(lab)
            mlm_sum = float(F.cross_entropy(mlm.reshape(-1, V).double(), ml.reshape(-1),
                                            reduction="sum"))
            mlm_n = int((ml != -100).sum())
            nsp_sum = float(F.cross_entropy(nsp.double(), nl, reduction="sum"))
            nsp_ok = int((nsp.argmax(1) == nl).sum())
    runner.engine.close()
    return got, dict(mlm_loss=mlm_sum / mlm_n, mlm_n=mlm_n, nsp_loss=nsp_sum / 21,
                     nsp_accuracy=nsp_ok / 21)


def test_evaluation_metrics_match_a_direct_computation(tmp_path):
    got, want = run_distributed(_eval_direct, 1, str(tmp_path))[0]
    assert got["mlm_n"] == want["mlm_n"] and got["nsp_n"] == 21
    assert got["mlm_loss"] == pytest.approx(want["mlm_loss"], rel=1e-5)
    assert got["nsp_loss"] == pytest.approx(want["nsp_loss"], rel=1e-5)
    assert got["nsp_accuracy"] == want["nsp_accuracy"]
    assert got["loss"] == pytest.approx(got["mlm_loss"] + got["nsp_loss"])
    assert got["perplexity"] == pytest.approx(math.exp(got["mlm_loss"]))
    text = sky.runner.metrics.format_metrics(got)
    assert "nsp_accuracy=" in text and "mlm_loss=" in text


def _cls_cfg():
    c = _cfg(2).__dict__
    enc = [dict(layer_type="BertLayer_Head", config=c), dict(layer_type="BertLayer_Body", config=c),
           dict(layer_type="BertLayer_Tail", config=c)] * 2
    return ([dict(layer_type="BertEmbeddings", config=c)] + enc
            + [dict(layer_type="BertPooler", config=c),
               dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.0,
                    hidden_size=H, num_classes=3)])


def _round_trip(rank, world, tmp, head):
    from skycomputing_b200.runner.hooks_collection.checkpoint_hook import CheckpointHook

    pre = _runner(rank, world, tmp, None, False, "one", head=head,
                  loss="PreTrainingLoss" if head == "BertTailForPreTraining" else "MaskedLMLoss")
    pre.parameter_server = ParameterServer(_model_cfg(head=head))
    path = tmp + "/pre_{}.pth".format(head)
    CheckpointHook(save_path=tmp).save(pre, path)
    saved = torch.load(path)
    pre.engine.close()
    cls = _runner(rank, world, tmp, None, False, "one", loss="CrossEntropyLoss", mc=_cls_cfg())
    cls.parameter_server = ParameterServer(_cls_cfg())
    torch.manual_seed(1234)
    init = {k: v.clone() for k, v in cls.model.local_stage.layers.state_dict().items()}
    with pytest.raises(ValueError, match="from_pretraining=True"):
        CheckpointHook(load_checkpoint_from=path).before_run(cls)
    logs = []
    cls._log = logs.append
    CheckpointHook(load_checkpoint_from=path, from_pretraining=True).before_run(cls)
    now = cls.model.local_stage.layers.state_dict()
    ps = cls.parameter_server.full_state_dict()
    res = dict(logs=logs)
    res["encoder_equal"] = all(torch.equal(now[k], saved[k]) and torch.equal(ps[k], saved[k])
                               for k in saved if int(k.split(".")[0]) < 7)
    res["pooler_equal"] = all(
        torch.equal(now["7." + n], saved["7.pooler." + n]) and torch.equal(ps["7." + n],
                                                                           saved["7.pooler." + n])
        for n in ("dense_act.weight", "dense_act.bias")) if head == "BertTailForPreTraining" \
        else all(torch.equal(now["7." + n], init["7." + n]) for n in ("dense_act.weight",))
    res["classifier_init"] = all(torch.equal(now[k], init[k]) for k in init if k.startswith("8."))
    cls.engine.close()
    return res


@pytest.mark.parametrize("head", ["BertTailForPreTraining", "BertTailForMaskedLM"])
def test_pretrain_to_classification_round_trip(tmp_path, head):
    res = run_distributed(_round_trip, 1, str(tmp_path), head)[0]
    assert res["encoder_equal"] and res["pooler_equal"] and res["classifier_init"]
    (msg,) = [m for m in res["logs"] if "pretraining checkpoint" in m]
    assert "layer 7: decoder.*" in msg and "transform.*" in msg
    assert "layer 8 (BertTailForClassification)" in msg
    if head == "BertTailForPreTraining":
        assert "seq_relationship.*" in msg
    else:
        assert "layer 7 (BertPooler)" in msg


def _shape_mismatch(rank, world, tmp):
    from skycomputing_b200.runner.hooks_collection.checkpoint_hook import CheckpointHook

    pre = _runner(rank, world, tmp, None, False, "one")
    pre.parameter_server = ParameterServer(_model_cfg())
    path = tmp + "/pre_v64.pth"
    CheckpointHook(save_path=tmp).save(pre, path)
    pre.engine.close()
    # a vocabulary that is not a multiple of 8 (60): the pretraining run's table is [64, H]
    mc = _cls_cfg()
    mc[0] = dict(mc[0], config=dict(mc[0]["config"], vocab_size=60))
    cls = _runner(rank, world, tmp, None, False, "one", loss="CrossEntropyLoss", mc=mc)
    cls.parameter_server = ParameterServer(mc)
    try:
        CheckpointHook(load_checkpoint_from=path, from_pretraining=True).before_run(cls)
    except ValueError as e:
        return str(e)
    finally:
        cls.engine.close()
    return None


def test_unpadded_vocabulary_is_a_clear_error(tmp_path):
    msg = run_distributed(_shape_mismatch, 1, str(tmp_path))[0]
    assert msg is not None and "word_embeddings.weight" in msg and "[64, 64]" in msg, msg
    assert "[60, 64]" in msg


def test_launcher_pads_the_vocabulary_of_a_fine_tuning_run(monkeypatch):
    import os
    import runpy

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for env, want in ((dict(TASK="cls"), 30522), (dict(TASK="cls", INIT_FROM="x.pth"), 30528),
                      (dict(TASK="pretrain"), 30528)):
        for k in ("TASK", "INIT_FROM", "SAVE_PATH", "TINY"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        cfg = runpy.run_path(os.path.join(root, "experiment", "config.py"))
        assert cfg["model_config"][0]["config"]["vocab_size"] == want, env
        hooks = [h["type"] for h in cfg["train_config"]["hook_config"]]
        assert ("CheckpointHook" in hooks) == ("INIT_FROM" in env), env
