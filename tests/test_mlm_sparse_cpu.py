"""Sparse masked-language-model decoding on the CPU: the reference slot helper on hand-made
cases, ``max_predictions`` validation, where a label-consuming layer may sit, the sparse head
against the dense head on the torch backend, 2-stage gloo pipelines (plain 1F1B and looped) that
train and evaluate the sparse head like the dense one, its analytic cost and checkpoint exchange
with the dense head."""
import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.dynamics.allocator import group_units
from skycomputing_b200.ops.functions import mlm_slots_ref
from tests._dist_helpers import run_distributed

I = -100


# ---------------------------------------------------------------------------------------------
# the slot layout
# ---------------------------------------------------------------------------------------------
def test_slots_of_hand_made_sequences():
    labels = torch.tensor([
        [I, I, I, I, I],          # nothing labelled: every slot empty
        [4, 5, 6, 7, 8],          # all labelled, P = 3 < 5: overflow
        [I, 9, I, 2, 3],          # exactly P
        [1, I, I, I, I],          # fewer than P
    ])
    row, slot, lab = mlm_slots_ref(labels, 3, I, 50)
    assert row.tolist() == [-1, -1, -1, 5, 6, 7, 11, 13, 14, 15, -1, -1]
    assert lab.tolist() == [I, I, I, 4, 5, 50, 9, 2, 3, 1, I, I]
    assert slot.tolist() == [-1] * 5 + [3, 4, 5, -1, -1] + [-1, 6, -1, 7, 8] + [9, -1, -1, -1, -1]
    for t in (row, slot, lab):
        assert t.dtype == torch.int64


def test_one_label_too_many_drops_the_last_position_and_sets_the_sentinel():
    labels = torch.tensor([[I, 3, 4, I, 5, 6]])              # P + 1 = 4 labelled positions
    row, slot, lab = mlm_slots_ref(labels, 3, I, 10)
    assert row.tolist() == [1, 2, 4]                          # position 5 is dropped
    assert slot.tolist() == [-1, 0, 1, -1, 2, -1]
    assert lab.tolist() == [3, 4, 10]                         # label V in the last slot
    # exactly P: no sentinel
    assert mlm_slots_ref(labels[:, :5], 3, I, 10)[2].tolist() == [3, 4, 5]


def test_custom_ignore_index_and_p_above_the_sequence_length():
    labels = torch.tensor([[0, -1, 7, -1], [-1, -1, -1, 2]])
    row, slot, lab = mlm_slots_ref(labels, 6, -1, 9)
    assert row.tolist() == [0, 2, -1, -1, -1, -1, 7, -1, -1, -1, -1, -1]
    assert lab.tolist() == [0, 7, -1, -1, -1, -1, 2, -1, -1, -1, -1, -1]
    assert slot.tolist() == [0, -1, 1, -1, -1, -1, -1, 6]


# ---------------------------------------------------------------------------------------------
# the layer option
# ---------------------------------------------------------------------------------------------
def _cfg(layers=1, vocab=64, H=64):
    return sky.BertConfig(vocab, hidden_size=H, num_hidden_layers=layers, num_attention_heads=4,
                          intermediate_size=2 * H, max_position_embeddings=32,
                          hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


@pytest.mark.parametrize("bad", [0, -3, 33, 2.0, "20", True])
def test_max_predictions_is_validated(bad):
    with pytest.raises(ValueError, match="max_predictions"):
        sky.build_layer("BertTailForMaskedLM", config=_cfg().__dict__, max_predictions=bad)


def test_max_predictions_accepts_the_sequence_bound():
    for p in (None, 1, 20, 32):
        head = sky.build_layer("BertTailForMaskedLM", config=_cfg().__dict__, max_predictions=p)
        assert head.consumes_labels == (p is not None)


def test_max_predictions_is_capped_at_the_kernel_limit():
    cls = sky.models.bert_layers.BertTailForMaskedLM
    c = _cfg(H=32).__dict__
    c = dict(c, max_position_embeddings=2 * cls.MAX_PREDICTIONS_LIMIT)
    assert sky.build_layer("BertTailForMaskedLM", config=c,
                           max_predictions=cls.MAX_PREDICTIONS_LIMIT).max_predictions == 8192
    with pytest.raises(ValueError, match="8192"):
        sky.build_layer("BertTailForMaskedLM", config=c,
                        max_predictions=cls.MAX_PREDICTIONS_LIMIT + 1)


def _one_stage_runner(tmp, P):
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(name="w0", server_config={}, device=0, extra_config=dict(
        slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))])
    wm = sky.Allocator(_model_cfg(1, P=P), wm, granularity="layer").allocate("even")
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="Adam", lr=2e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=0, loss_cfg=dict(type="MaskedLMLoss"),
                      timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                      schedule="1f1b")


def test_inference_after_training_decodes_every_position(tmp_path):
    """The engine binds labels for one forward only: after a training step and an evaluation, a
    direct call of a one-stage model returns the dense [B, S, V] logits."""
    runner = _one_stage_runner(str(tmp_path), P=4)
    data, lab = _batch(n=4)
    runner.train_iteration(data, lab)
    runner.evaluate([(data, lab)], name="dev")
    stage = runner.model.local_stage
    assert stage.labels is None
    dense = sky.build_module_from_cfg(0, _model_cfg(1), {})
    dense.load_state_dict(stage.state_dict())
    runner.model.eval()
    dense.eval()
    other, _ = _batch(n=8, seed=3)          # another batch size: no label shape to trip over
    with torch.no_grad():
        for x in (data, other):
            out = runner.model(*x)
            assert out.shape == (x[0].shape[0], 16, 64)
            assert torch.equal(out, dense(*x)[0])
    runner.engine.close()


def _model_cfg(layers=1, P=None, vocab=64, H=64):
    c = _cfg(layers, vocab, H).__dict__
    enc = [dict(layer_type="BertLayer_Head", config=c), dict(layer_type="BertLayer_Body", config=c),
           dict(layer_type="BertLayer_Tail", config=c)] * layers
    head = dict(layer_type="BertTailForMaskedLM", config=c)
    if P is not None:
        head["max_predictions"] = P
    return [dict(layer_type="BertEmbeddings", config=c)] + enc + [head]


def test_a_label_consuming_layer_must_be_last():
    c = _cfg().__dict__
    cfg = [dict(layer_type="BertTailForMaskedLM", config=c, max_predictions=4),
           dict(layer_type="BertTailForMaskedLM", config=c)]
    with pytest.raises(ValueError, match="last layer"):
        sky.build_module_from_cfg(0, cfg, {})
    # within a pipeline: a stage that ends with it but is not the last stage
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(name=f"w{i}", server_config={}, device=i,
                                          extra_config=dict(slowdown=0, mem_limit=-1))
                                     for i in range(2)])
    mc = _model_cfg(1, P=4) + [dict(layer_type="BertTailForMaskedLM", config=c)]
    units = group_units(mc, "layer")
    wm = sky.Allocator(mc, wm, granularity="layer")._assign([0, 1], [0, len(units) - 1,
                                                                     len(units)], units)
    with pytest.raises(ValueError, match="last layer"):
        sky.RpcModel(wm, this_rank=0)
    # as the last layer it is accepted, and the stage reports it
    stage = sky.build_module_from_cfg(0, _model_cfg(1, P=4), {})
    assert stage.consumes_labels and not sky.build_module_from_cfg(0, _model_cfg(1), {}).consumes_labels


def _stages(P):
    torch.manual_seed(0)
    dense = sky.build_module_from_cfg(0, _model_cfg(1), {})
    sparse = sky.build_module_from_cfg(0, _model_cfg(1, P=P), {})
    sparse.load_state_dict(dense.state_dict())
    return dense, sparse


def _batch(n=4, seed=0):
    ds = sky.SynthMLMDataset(num_samples=n, max_seq_length=16, vocab_size=64, seed=seed)
    (ids, tt, am), lab = next(iter(torch.utils.data.DataLoader(ds, batch_size=n)))
    return (ids, tt, am), lab


def test_sparse_head_loss_and_gradients_equal_the_dense_head():
    dense, sparse = _stages(P=4)
    data, lab = _batch()
    loss_fn = sky.MaskedLMLoss()
    out_d = dense(*data)
    assert len(out_d) == 1 and out_d[0].shape == (4, 16, 64)
    ld = loss_fn(out_d[0], lab)
    ld.backward()
    sparse.labels = lab
    logits, slot_labels = sparse(*data)
    assert logits.shape == (4 * 4, 64) and slot_labels.shape == (16,)
    ls = loss_fn(logits, slot_labels)
    ls.backward()
    assert float(ls.detach()) == pytest.approx(float(ld.detach()), rel=1e-5)
    for (n, p), (_, q) in zip(dense.named_parameters(), sparse.named_parameters()):
        torch.testing.assert_close(q.grad, p.grad, rtol=1e-5, atol=1e-7, msg=n)
    # a binding holds for one forward: the next call, with none, computes the dense logits
    assert sparse.labels is None
    with torch.no_grad():
        assert torch.equal(sparse(*data)[0], dense(*data)[0])


def test_dense_checkpoint_loads_into_the_sparse_head():
    c = _cfg().__dict__
    dense = sky.build_layer("BertTailForMaskedLM", config=c)
    sparse = sky.build_layer("BertTailForMaskedLM", config=c, max_predictions=20)
    assert list(dense.state_dict()) == list(sparse.state_dict())
    sparse.load_state_dict(dense.state_dict(), strict=True)
    dense.load_state_dict(sparse.state_dict(), strict=True)
    x = torch.randn(2, 16, 64)
    with torch.no_grad():
        assert torch.equal(sparse(x), dense(x))


# ---------------------------------------------------------------------------------------------
# cost model
# ---------------------------------------------------------------------------------------------
def test_analytic_cost_of_the_sparse_head_matches_measured():
    P = 5
    cfg = _model_cfg(2, P=P, vocab=96, H=32)
    gen = sky.build_data_generator("DataloaderGenerator", generator_cfg=dict(
        dataset_cfg=dict(type="SynthMLMDataset", num_samples=4, max_seq_length=16, vocab_size=96),
        dataloader_cfg=dict(batch_size=4)))
    f_meas, m_meas = sky.ModelBenchmarker(cfg, gen, device="cpu").benchmark()
    f_ana, m_ana = sky.ModelBenchmarker(cfg, gen, device="cpu", analytic=True).benchmark()
    B, S, H, V = 4, 16, 32, 96
    assert f_meas[-1] == 2 * B * P * H * (H + V)
    assert f_ana == pytest.approx(f_meas, rel=1e-6, abs=1e-6)
    assert m_ana == pytest.approx(m_meas, rel=0.05)
    dense_f, dense_m = sky.ModelBenchmarker(_model_cfg(2, vocab=96, H=32), gen, device="cpu",
                                            analytic=True).benchmark()
    assert f_ana[-1] < dense_f[-1] / 3 and m_ana[-1] < dense_m[-1]


# ---------------------------------------------------------------------------------------------
# 2-stage pipelines: the sparse head trains and evaluates like the dense head
# ---------------------------------------------------------------------------------------------
def _runner(rank, world, tmp, P, virtual_stages):
    cfg = _model_cfg(1, P=P)
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    if virtual_stages > 1:
        wm = sky.Allocator(cfg, wm, granularity="layer").allocate("even",
                                                                  virtual_stages=virtual_stages)
    else:
        alloc = sky.Allocator(cfg, wm, granularity="layer")
        units = group_units(cfg, "layer")
        n = len(units)
        wm = alloc._assign(list(range(world)), [0, n - 1, n], units)   # cut in front of the head
    torch.manual_seed(0)
    model = sky.RpcModel(wm, this_rank=rank)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="Adam", lr=2e-3))
    return sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                      max_epochs=1, max_iters=0, loss_cfg=dict(type="MaskedLMLoss"),
                      timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                      schedule="1f1b")


def _train_and_eval(rank, world, tmp, P, virtual_stages):
    runner = _runner(rank, world, tmp, P, virtual_stages)
    train = sky.SynthMLMDataset(num_samples=8 * 12, max_seq_length=16, vocab_size=64, seed=0,
                                max_step=1)
    losses = []
    for data, labels in torch.utils.data.DataLoader(train, batch_size=8):
        loss = runner.train_iteration(data, labels)
        if loss is not None:
            losses.append(loss)
    dev = sky.SynthMLMDataset(num_samples=21, max_seq_length=16, vocab_size=64, seed=1, max_step=1)
    out = runner.evaluate(torch.utils.data.DataLoader(dev, batch_size=8), name="dev")
    err = None
    if P is not None:
        # one label more than P in every sequence: evaluate must raise and name max_predictions
        over = sky.SynthMLMDataset(num_samples=8, max_seq_length=16, vocab_size=64, seed=2,
                                   max_step=1)
        (ids, tt, am), lab = next(iter(torch.utils.data.DataLoader(over, batch_size=8)))
        lab[:, 1:2 + P] = ids[:, 1:2 + P]
        try:
            runner.evaluate([((ids, tt, am), lab)], name="over")
        except ValueError as e:
            err = str(e)
    schedule = runner.engine.schedule
    runner.engine.close()
    return dict(losses=losses, eval=out, err=err, schedule=schedule)


@pytest.mark.parametrize("virtual_stages", [1, 2])
def test_two_stage_pipeline_sparse_head_matches_dense(tmp_path, virtual_stages):
    dense = run_distributed(_train_and_eval, 2, str(tmp_path), None, virtual_stages)
    sparse = run_distributed(_train_and_eval, 2, str(tmp_path), 4, virtual_stages)
    assert (sparse[0]["schedule"] == "looped") == (virtual_stages > 1)
    last = 1 if sparse[1]["losses"] else 0
    d, s = dense[last]["losses"], sparse[last]["losses"]
    assert len(d) == len(s) == 12
    assert s == pytest.approx(d, rel=1e-5)
    for r in range(2):
        assert sparse[r]["eval"]["n"] == dense[r]["eval"]["n"]
        assert sparse[r]["eval"]["loss"] == pytest.approx(dense[r]["eval"]["loss"], rel=1e-5)
        assert sparse[r]["err"] is not None and "max_predictions" in sparse[r]["err"]
