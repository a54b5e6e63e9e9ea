"""A masked-language-model decoder tied to the word embeddings, on the CPU: validation, the shared
Parameter of a one-stage model, 2-rank gloo pipelines (plain 1F1B and looped) whose replica stays
bit-identical to the table, the checkpoint rule and reallocation."""
import os

import pytest
import torch

import skycomputing_b200 as sky
from skycomputing_b200.dynamics.allocator import group_units
from skycomputing_b200.models.bert_layers import BertTailForMaskedLM
from skycomputing_b200.runner.hooks_collection.checkpoint_hook import CheckpointHook
from skycomputing_b200.utils import get_state_dict, load_weights
from tests._dist_helpers import run_distributed

V, H = 64, 32


def _cfg(layers=2, tie=True, vocab=V, head_vocab=None, first=True):
    c = sky.BertConfig(vocab, hidden_size=H, num_hidden_layers=layers, num_attention_heads=4,
                       intermediate_size=2 * H, max_position_embeddings=32,
                       hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    hc = c.__dict__ if head_vocab is None else dict(c.__dict__, vocab_size=head_vocab)
    enc = [dict(layer_type="BertLayer_Head", config=c.__dict__),
           dict(layer_type="BertLayer_Body", config=c.__dict__),
           dict(layer_type="BertLayer_Tail", config=c.__dict__)] * layers
    head = dict(layer_type="BertTailForMaskedLM", config=hc, tie_word_embeddings=tie)
    return ([dict(layer_type="BertEmbeddings", config=c.__dict__)] if first else []) + enc + [head]


def _pool(world, tmp):
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([
        dict(name=f"w{i}", server_config={}, device=i,
             extra_config=dict(slowdown=0, mem_limit=-1, timer_config=dict(root=tmp)))
        for i in range(world)])
    return wm


def _seed(stage, first_index):
    """Deterministic weights per global layer index; a tied head's decoder is the table (or a
    replica of it) and is not seeded."""
    for off, layer in enumerate(stage.layers.children()):
        g = torch.Generator().manual_seed(100 + first_index + off)
        skip = {id(layer.decoder.weight)} if isinstance(layer, BertTailForMaskedLM) and \
            layer.tie_word_embeddings else set()
        with torch.no_grad():
            for p in layer.parameters():
                if id(p) not in skip:
                    p.copy_(torch.randn(p.shape, generator=g) * 0.1)


# ---------------------------------------------------------------------------------------------
# the option and its validation
# ---------------------------------------------------------------------------------------------
def test_tie_needs_embeddings_first_and_matching_shapes(tmp_path):
    def build(cfg):
        wm = sky.Allocator(cfg, _pool(1, str(tmp_path)), granularity="layer").even_allocate()
        return sky.RpcModel(wm, this_rank=0)

    with pytest.raises(ValueError, match="first layer"):
        build(_cfg(first=False))
    with pytest.raises(ValueError, match="vocab, hidden"):
        build(_cfg(head_vocab=V + 8))
    model = build(_cfg())
    assert model.tied_word_embeddings
    assert not build(_cfg(tie=False)).tied_word_embeddings
    # the head alone (benchmarkers, cost model) keeps its own decoder weight
    head = BertTailForMaskedLM(_cfg()[-1]["config"], tie_word_embeddings=True)
    assert head.is_replica and head.decoder.weight.shape == (V, H)


def test_untied_default_is_unchanged(tmp_path):
    stage = sky.build_module_from_cfg(0, _cfg(tie=False), {})
    emb, head = stage.layers[0], stage.layers[-1]
    assert head.decoder.weight is not emb.word_embeddings.weight
    assert not hasattr(head.decoder.weight, "tied_name")


# ---------------------------------------------------------------------------------------------
# one stage: one Parameter; its gradient is the sum of both uses
# ---------------------------------------------------------------------------------------------
def _batch(n=4, S=16, seed=0):
    ds = sky.SynthMLMDataset(num_samples=n, max_seq_length=S, vocab_size=V, seed=seed, max_step=1)
    (ids, tt, am), lab = next(iter(torch.utils.data.DataLoader(ds, batch_size=n)))
    return (ids, tt, am), lab


def test_one_stage_tied_gradient_is_the_sum_of_both_uses():
    tied = sky.build_module_from_cfg(0, _cfg(), {})
    untied = sky.build_module_from_cfg(0, _cfg(tie=False), {})
    _seed(tied, 0)
    emb, head = tied.layers[0], tied.layers[-1]
    assert head.decoder.weight is emb.word_embeddings.weight
    assert sum(1 for _ in tied.parameters()) == sum(1 for _ in untied.parameters()) - 1
    names = [n for n, p in tied.named_parameters() if p is emb.word_embeddings.weight]
    assert names == ["_module.0.word_embeddings.weight"]
    untied.load_state_dict(tied.state_dict())      # both entries are in the tied state_dict
    assert torch.equal(untied.layers[-1].decoder.weight, emb.word_embeddings.weight)
    loss = sky.MaskedLMLoss()
    inputs, labels = _batch()
    for stage in (tied, untied):
        loss(stage(*inputs)[0], labels).backward()
    want = untied.layers[0].word_embeddings.weight.grad + untied.layers[-1].decoder.weight.grad
    got = emb.word_embeddings.weight.grad
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-7)
    assert torch.allclose(head.decoder.bias.grad, untied.layers[-1].decoder.bias.grad)


def test_lamb_decides_the_tied_table_under_one_name():
    stage = sky.build_module_from_cfg(0, _cfg(), {})
    opt = sky.build_optimizer(stage, dict(optim_type="LAMB", lr=1e-3,
                                          exclude_from_weight_decay=("decoder", "bias")))
    groups = opt.optimizer.param_groups
    table = stage.layers[0].word_embeddings.weight
    decayed = [g for g in groups if any(p is table for p in g["params"])]
    assert len(decayed) == 1 and decayed[0]["weight_decay"] > 0   # not excluded as "decoder"
    assert sum(any(p is table for p in g["params"]) for g in groups) == 1


# ---------------------------------------------------------------------------------------------
# checkpoints
# ---------------------------------------------------------------------------------------------
class _FakeServer:
    def load_weights_from_file(self, path):
        pass

    def __len__(self):
        return 0


class _FakeRunner:
    def __init__(self, model):
        self.model, self.parameter_server, self.is_rank0, self.rank = model, _FakeServer(), True, 0
        self.engine, self.logged = None, []

    def _log(self, msg):
        self.logged.append(msg)


def _file(stage, path):
    sd = {}
    for i, layer_sd in enumerate(get_state_dict(stage)):
        sd.update({"{}.{}".format(i, k): v for k, v in layer_sd.items()})
    torch.save(sd, path)
    return sd


def test_checkpoint_keeps_both_entries_and_the_embedding_entry_wins(tmp_path):
    wm = sky.Allocator(_cfg(), _pool(1, str(tmp_path)), granularity="layer").even_allocate()
    model = sky.RpcModel(wm, this_rank=0)
    stage = model.local_stage
    _seed(stage, 0)
    n = len(list(stage.layers.children()))
    sd = _file(stage, str(tmp_path / "tied.pth"))
    assert torch.equal(sd["0.word_embeddings.weight"], sd["{}.decoder.weight".format(n - 1)])
    # round trip into a fresh tied model
    model2 = sky.RpcModel(wm, this_rank=0)
    runner = _FakeRunner(model2)
    CheckpointHook(load_checkpoint_from=str(tmp_path / "tied.pth")).before_run(runner)
    for a, b in zip(model2.local_stage.state_dict().values(), stage.state_dict().values()):
        assert torch.equal(a, b)
    assert runner.logged == []
    # an untied file: the embedding entry wins, reported once
    untied = sky.build_module_from_cfg(0, _cfg(tie=False), {})
    _seed(untied, 1000)
    usd = _file(untied, str(tmp_path / "untied.pth"))
    model3 = sky.RpcModel(wm, this_rank=0)
    runner = _FakeRunner(model3)
    with pytest.warns(UserWarning, match="untied"):
        CheckpointHook(load_checkpoint_from=str(tmp_path / "untied.pth")).before_run(runner)
    st = model3.local_stage
    assert torch.equal(st.layers[-1].decoder.weight.detach(), usd["0.word_embeddings.weight"])
    assert st.layers[-1].decoder.weight is st.layers[0].word_embeddings.weight
    assert len(runner.logged) == 1
    # loading per-layer dicts directly: the head skips its decoder entry
    with pytest.warns(UserWarning, match="untied"):
        load_weights(st, get_state_dict(untied))
    assert torch.equal(st.layers[0].word_embeddings.weight.detach(),
                       untied.layers[0].word_embeddings.weight.detach())


# ---------------------------------------------------------------------------------------------
# 2-stage gloo pipeline: replica bit-identical to the table, losses of the 1-stage model
# ---------------------------------------------------------------------------------------------
OPTIMS = {
    "sgd": dict(optim_type="SGD", lr=0.05, momentum=0.9),
    "adamw": dict(optim_type="AdamW", lr=2e-3),
    "lamb": dict(optim_type="LAMB", lr=2e-3),
}
SCHED = dict(type="cosine", warmup_steps=2, total_steps=8)
CLIP = dict(max_norm=0.5)


def _tied_run(rank, world, cut, optim, steps, tmp, ckpt):
    cfg = _cfg(layers=2)
    alloc = sky.Allocator(cfg, _pool(world, tmp), granularity="layer")
    if cut == "looped":
        # 4 virtual stages on 2 ranks: the table in chunk 0 of rank 0, the head in the last
        # chunk of rank 1
        wm = alloc.allocate("even", virtual_stages=2)
    else:
        units = group_units(cfg, "layer")
        n = len(units)
        bounds = {1: [0, n], 2: {"blocks": [0, 4, n], "head": [0, n - 1, n]}.get(cut)}[world]
        wm = alloc._assign(list(range(world)), bounds, units)
    model = sky.RpcModel(wm, this_rank=rank)
    opt = sky.build_optimizer(model.optim_module, dict(OPTIMS[optim]), lr_schedule=SCHED,
                              grad_clip=CLIP)
    runner = sky.Runner(model=model, parameter_server=_FakeServer(), worker_manager=wm,
                        optimizer=opt, max_epochs=1, max_iters=steps,
                        loss_cfg=dict(type="MaskedLMLoss"), timer_cfg=dict(root=tmp),
                        logging_cfg=None, micro_batches=2, schedule="1f1b")
    CheckpointHook(load_checkpoint_from=ckpt).before_run(runner)
    ds = sky.SynthMLMDataset(num_samples=8 * steps, max_seq_length=16, vocab_size=V, seed=3,
                             max_step=1)
    losses, copies, norms = [], [], []
    eng = runner.engine
    for data, labels in torch.utils.data.DataLoader(ds, batch_size=8):
        loss = runner.train_iteration(data, labels)
        if loss is not None:
            losses.append(loss)
        norms.append(opt.scalars()["grad_norm"])
        table, head = eng._local_tied_params()
        if world == 1:
            copies.append(table.detach().clone())
        elif eng.is_first:
            copies.append(table.detach().clone())
        elif eng.is_last:
            copies.append(head.decoder.weight.detach().clone())
    eng.close()
    return dict(losses=losses, copies=copies, norms=norms, engine=type(eng).__name__,
                chunks=len(eng.stages))


@pytest.fixture(scope="module")
def tied_ckpt(tmp_path_factory):
    d = tmp_path_factory.mktemp("tied")
    stage = sky.build_module_from_cfg(0, _cfg(layers=2), {})
    _seed(stage, 0)
    path = str(d / "init.pth")
    _file(stage, path)
    return path


@pytest.mark.parametrize("optim", sorted(OPTIMS))
@pytest.mark.parametrize("cut", ["blocks", "head", "looped"])
def test_two_stage_tied_pipeline_matches_one_stage(tmp_path, tied_ckpt, cut, optim):
    steps = 5
    ref = _tied_run(0, 1, None, optim, steps, str(tmp_path), tied_ckpt)
    res = run_distributed(_tied_run, 2, cut, optim, steps, str(tmp_path), tied_ckpt)
    if cut == "looped":
        assert res[0]["engine"] == res[1]["engine"] == "LoopedPipelineEngine"
        assert res[0]["chunks"] == res[1]["chunks"] == 2
    assert res[0]["losses"] == [] and len(res[1]["losses"]) == steps
    assert res[1]["losses"] == pytest.approx(ref["losses"], rel=2e-5, abs=1e-6)
    assert res[1]["norms"] == pytest.approx(ref["norms"], rel=2e-5)   # the table counted once
    for k, (t, r) in enumerate(zip(res[0]["copies"], res[1]["copies"])):
        assert torch.equal(t, r), "step {}: replica differs from the table".format(k)
        assert torch.allclose(t, ref["copies"][k], rtol=1e-4, atol=1e-6)
    assert not torch.equal(res[0]["copies"][0], res[0]["copies"][-1])


def _untied_into_tied(rank, world, tmp, ckpt):
    cfg = _cfg(layers=2)
    units = group_units(cfg, "layer")
    wm = sky.Allocator(cfg, _pool(world, tmp), granularity="layer")._assign(
        [0, 1], [0, len(units) - 1, len(units)], units)
    model = sky.RpcModel(wm, this_rank=rank)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=0.1))
    runner = sky.Runner(model=model, parameter_server=_FakeServer(), worker_manager=wm,
                        optimizer=opt, max_epochs=1, max_iters=1,
                        loss_cfg=dict(type="MaskedLMLoss"), timer_cfg=dict(root=tmp),
                        logging_cfg=None, micro_batches=1)
    import warnings

    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        CheckpointHook(load_checkpoint_from=ckpt).before_run(runner)
    table, head = runner.engine._local_tied_params()
    runner.engine._setup(None if rank else [torch.zeros(2, 16, dtype=torch.long)] * 3)
    mine = (table if rank == 0 else head.decoder.weight).detach().clone()
    runner.engine.close()
    return dict(copy=mine, warned=sum("untied" in str(x.message) for x in w))


def test_untied_checkpoint_into_a_two_stage_tied_model(tmp_path):
    untied = sky.build_module_from_cfg(0, _cfg(layers=2, tie=False), {})
    _seed(untied, 0)
    path = str(tmp_path / "untied.pth")
    sd = _file(untied, path)
    res = run_distributed(_untied_into_tied, 2, str(tmp_path), path)
    assert torch.equal(res[0]["copy"], sd["0.word_embeddings.weight"])
    assert torch.equal(res[1]["copy"], sd["0.word_embeddings.weight"])
    assert res[0]["warned"] == 0 and res[1]["warned"] == 1


# ---------------------------------------------------------------------------------------------
# reallocation keeps the tie
# ---------------------------------------------------------------------------------------------
class _FakeDeviceBench:
    def __init__(self, wm):
        self._wm = wm

    def benchmark(self):
        from skycomputing_b200.utils import generate_worker_name

        return {generate_worker_name(w.rank): dict(time=3.0 if w.device == 1 else 1.0, avai_mem=1e9)
                for w in self._wm.worker_pool}


class _FakeModelBench:
    def __init__(self, n):
        self._n = n

    def benchmark(self):
        return [1.0] * self._n, [1.0] * self._n


def _realloc_run(rank, world, use_hook, steps, tmp):
    cfg = _cfg(layers=4)
    wm = sky.Allocator(cfg, _pool(world, tmp), granularity="block").even_allocate()
    model = sky.RpcModel(wm, this_rank=rank)
    _seed(model.local_stage, model.local_module.layer_range[0])
    optim_cfg = dict(optim_type="SGD", lr=0.1)
    opt = sky.build_optimizer(model.local_stage, dict(optim_cfg))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=steps, loss_cfg=dict(type="MaskedLMLoss"),
                        timer_cfg=dict(root=tmp), logging_cfg=None, micro_batches=2,
                        schedule="1f1b")
    hook = None
    if use_hook:
        def factory(pool):
            return sky.Allocator(cfg, pool, _FakeModelBench(len(cfg)), _FakeDeviceBench(pool),
                                 granularity="block", solver="exact")

        hook = sky.ReallocateHook(interval=2, allocator_factory=factory, optimizer_cfg=optim_cfg,
                                  allocate_type="dynamic", min_gain=0.05)
        runner.register_hook(hook)
    ds = sky.SynthMLMDataset(num_samples=8 * steps, max_seq_length=16, vocab_size=V, seed=5,
                             max_step=1)
    losses = []
    orig = runner.train_iteration

    def spy(data, labels):
        out = orig(data, labels)
        if out is not None:
            losses.append(out)
        return out

    runner.train_iteration = spy
    runner.train(torch.utils.data.DataLoader(ds, batch_size=8))
    eng = runner.engine
    table, head = eng._local_tied_params()
    copy = table if eng.is_first else head.decoder.weight
    out = dict(losses=losses, copy=copy.detach().clone(), range=tuple(runner.model.local_module.layer_range),
               migrations=0 if hook is None else hook.migrations, group=eng._tied_group is not None)
    eng.close()
    return out


def test_reallocation_keeps_the_tie(tmp_path):
    tmp = str(tmp_path)
    plain = run_distributed(_realloc_run, 2, False, 5, tmp)
    moved = run_distributed(_realloc_run, 2, True, 5, tmp)
    assert moved[0]["migrations"] == 1 and plain[0]["range"] != moved[0]["range"]
    assert all(r["group"] for r in plain + moved)
    for run in (plain, moved):
        assert torch.equal(run[0]["copy"], run[1]["copy"])
    lp = [r["losses"] for r in plain if r["losses"]][0]
    lm = [r["losses"] for r in moved if r["losses"]][0]
    assert lm == pytest.approx(lp, rel=1e-5)
    assert torch.allclose(moved[0]["copy"], plain[0]["copy"], rtol=1e-5, atol=1e-7)
