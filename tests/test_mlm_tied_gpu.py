"""A masked-language-model decoder tied to the word embeddings on one H100: the native tied model
against the fp32 eager one (dense and sparse head), the shared parameter bank and its zeroing /
SGD-in-wgrad rules, the shadow after a step, graph = eager, evaluation, LAMB trust ratios, the
clipping norm, and the two exchange kernels in loopback (local buffers stand in for the peer)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

V, H = 30528, 1024


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    if not native.available():
        pytest.skip("native extension not built")
    return native


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _model_cfg(layers, tie=True, max_predictions=None):
    import skycomputing_b200 as sky

    cfg = sky.BertConfig(V, hidden_size=H, num_hidden_layers=max(layers, 1), num_attention_heads=16,
                         intermediate_size=4096, hidden_dropout_prob=0.0,
                         attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * layers
    head = dict(layer_type="BertTailForMaskedLM", config=cfg.__dict__, tie_word_embeddings=tie)
    if max_predictions is not None:
        head["max_predictions"] = max_predictions
    return [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + [head]


def _seed(stage, base=700):
    for off, layer in enumerate(stage.layers.children()):
        gen = torch.Generator().manual_seed(base + off)
        skip = {id(layer.decoder.weight)} if getattr(layer, "tie_word_embeddings", False) else set()
        with torch.no_grad():
            for n, p in layer.named_parameters():
                if id(p) in skip:
                    continue
                p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                if n.endswith("LayerNorm.weight"):
                    p.fill_(1.0)


def _batches(n, batch=16, seed=0, max_step=4):
    import skycomputing_b200 as sky

    ds = sky.SynthMLMDataset(num_samples=n * batch, max_seq_length=128, vocab_size=V, seed=seed,
                             max_step=max_step)
    return list(torch.utils.data.DataLoader(ds, batch_size=batch))


# ---------------------------------------------------------------------------------------------
# the native tied model against the fp32 eager tied model
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sparse", [False, True])
def test_native_tied_model_matches_eager(nat, sparse):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    P = 20 if sparse else None
    stage = sky.build_module_from_cfg(0, _model_cfg(0, max_predictions=P), {})
    ref = sky.build_module_from_cfg(0, _model_cfg(0, max_predictions=P), {})
    _seed(stage)
    _seed(ref)
    assert ref.layers[-1].decoder.weight is ref.layers[0].word_embeddings.weight
    stage.cuda()
    ref.cuda()
    (d, l), = _batches(1, batch=8)
    d, l = [t.cuda() for t in d], l.cuda()
    loss_fn = sky.MaskedLMLoss()
    out = {}
    try:
        for name, st, backend in (("native", stage, "native"), ("eager", ref, "torch")):
            set_backend(backend)
            if sparse:
                st.labels = l
            outs = st(*d)
            logits, labels = (outs[0], outs[1].view(l.shape[0], -1)) if sparse else (outs[0], l)
            loss = loss_fn(logits.float(), labels)
            loss.backward()
            torch.cuda.synchronize()
            out[name] = (logits.detach(), float(loss.detach()), st.layers[0].word_embeddings.weight.grad.clone(),
                         st.layers[-1].decoder.bias.grad.clone())
    finally:
        set_backend("auto")
    n, e = out["native"], out["eager"]
    assert _rel(n[0], e[0]) < 2e-2
    assert n[1] == pytest.approx(e[1], rel=2e-2)
    assert _rel(n[2], e[2]) < 3e-2          # the tied gradient: embeddings + decoder
    assert _rel(n[3], e[3]) < 3e-2


# ---------------------------------------------------------------------------------------------
# one GPU through the engine
# ---------------------------------------------------------------------------------------------
def _runner(use_graph, tie=True, optim=None, grad_clip=None, micro_batches=2, layers=1):
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name="gpu-0", server_config={}, device=0,
        extra_config=dict(module_to_cuda=True, cuda_device=0, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_mlm_tied_test")))])
    mc = _model_cfg(layers, tie=tie)
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=0)
    _seed(model.local_stage)
    opt = sky.build_optimizer(model.optim_module, optim or dict(optim_type="SGD", lr=0.05),
                              grad_clip=grad_clip)
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type="MaskedLMLoss"),
                        timer_cfg=dict(root="/tmp/sky_mlm_tied_test"), logging_cfg=None,
                        micro_batches=micro_batches, schedule="1f1b", use_cuda_graph=use_graph,
                        device=torch.device("cuda", 0))
    model.train(True)
    return runner, opt


def test_one_bank_never_overwrite_first_never_armed_and_fresh_shadow(nat):
    from skycomputing_b200.models.bert_layers import native_param_banks

    data = _batches(2)
    runner, opt = _runner(False)        # plain SGD: the encoder banks update in their wgrad GEMMs
    untied, _ = _runner(False, tie=False)
    stage = runner.model.local_stage
    banks = native_param_banks(stage)
    assert len(banks) == len(native_param_banks(untied.model.local_stage)) - 1
    untied.engine.close()
    emb, head = stage.layers[0], stage.layers[-1]
    bank = emb._native_params().word
    assert head._native_params().w_dec is bank and bank.tied and bank.need_shadow
    assert sum(b is bank for b in opt.banks) == 1
    runner.train_iteration(*data[0])
    eng = runner.engine
    assert eng._wgrad_sgd is not None                       # the SGD-in-wgrad path is active
    assert all(b is not bank for banks_ in eng._wgrad_sgd_banks for b in banks_)
    assert bank.wgrad_target and not bank.overwrite_first and bank.wgrad_sgd is None
    runner.train_iteration(*data[1])
    torch.cuda.synchronize()
    assert not bank.overwrite_first
    # the decoder reads the shadow the optimizer refreshed with the update
    assert torch.equal(bank._shadow, bank.flat.to(torch.bfloat16))
    assert torch.count_nonzero(bank.flat_grad) == 0          # zeroed by the optimizer
    eng.close()


def test_tied_graph_step_equals_eager_and_evaluates(nat):
    data = _batches(4)
    out = {}
    for use_graph in (False, True):
        runner, opt = _runner(use_graph)
        assert opt.graph_safe
        out[use_graph] = [runner.train_iteration(d, l) for d, l in data]
        if use_graph:
            assert runner.engine._graph is not None
            import skycomputing_b200 as sky

            ds = sky.SynthMLMDataset(num_samples=2 * 16 + 3, max_seq_length=128, vocab_size=V,
                                     seed=1)
            ev = runner.evaluate(torch.utils.data.DataLoader(ds, batch_size=16))
            again = runner.evaluate(torch.utils.data.DataLoader(ds, batch_size=16))
            assert ev == again and ev["n"] > 0 and math.isfinite(ev["loss"])
        runner.engine.close()
    assert out[True][0] == out[False][0]                      # bit for bit before any update
    for a, b in zip(out[False], out[True]):
        assert a == pytest.approx(b, rel=3e-3, abs=3e-3)


def test_lamb_has_one_trust_ratio_for_the_table(nat):
    runner, opt = _runner(True, optim=dict(optim_type="LAMB", lr=1e-3))
    for d, l in _batches(2):
        runner.train_iteration(d, l)
    r = opt.trust_ratios()
    runner.engine.close()
    assert [k for k in r if "word_embeddings.weight" in k] == ["_module.0.word_embeddings.weight"]
    assert not any(k.endswith("decoder.weight") for k in r)
    assert math.isfinite(r["_module.0.word_embeddings.weight"])


def test_clipping_norm_counts_the_table_once(nat):
    (d, l), = _batches(1)
    runner, opt = _runner(False, optim=dict(optim_type="SGD", lr=0.0),
                          grad_clip=dict(max_norm=1e9), micro_batches=1)
    runner.train_iteration(d, l)
    torch.cuda.synchronize()
    reported = opt.scalars()["grad_norm"]
    stage = runner.model.local_stage
    logits = stage(*[t.cuda() for t in d])[0]
    runner.loss_function(logits, l.cuda()).backward()
    torch.cuda.synchronize()
    params = list(stage.parameters())                        # unique: the table once
    total = math.sqrt(sum(float(p.grad.double().pow(2).sum()) for p in params if p.grad is not None))
    runner.engine.close()
    assert reported == pytest.approx(total, rel=2e-2)


# ---------------------------------------------------------------------------------------------
# the exchange kernels in loopback
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1027, V * H])
def test_exchange_kernels_in_loopback(nat, n):
    ext = nat.ext()
    s = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device="cuda").manual_seed(n)
    src = torch.randn(n, generator=gen, device="cuda")
    inbox = torch.full((n,), float("nan"), device="cuda")
    words = torch.zeros(8, dtype=torch.int32, device="cuda")   # [push flag, push done, reduce flag,
    #                                                             reduce done, epoch, error]
    base = words.data_ptr()
    ext.tied_grad_push(src=src.data_ptr(), dst=inbox.data_ptr(), n=n, flag=base, done=base + 4,
                       stream=s)
    torch.cuda.synchronize()
    assert torch.equal(inbox, src)
    assert words[:2].tolist() == [1, 0]
    g = torch.randn(n, generator=gen, device="cuda")
    want = g + inbox
    peer_g = torch.zeros(n, device="cuda")
    words[4] = 1                                              # epoch 1: the push flag is there
    ext.tied_grad_reduce(g=g.data_ptr(), inbox=inbox.data_ptr(), peer_g=peer_g.data_ptr(), n=n,
                         wait_flag=base, epoch=base + 16, error_flag=base + 20,
                         publish_flag=base + 8, done=base + 12, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(g.view(torch.int32), want.view(torch.int32))
    assert torch.equal(peer_g.view(torch.int32), want.view(torch.int32))
    assert words.tolist()[:6] == [1, 0, 1, 0, 1, 0]
    # a second round (epoch 2): the counters were reset, the flags count steps
    ext.tied_grad_push(src=src.data_ptr(), dst=inbox.data_ptr(), n=n, flag=base, done=base + 4,
                       stream=s)
    words[4] = 2
    ext.tied_grad_reduce(g=g.data_ptr(), inbox=inbox.data_ptr(), peer_g=peer_g.data_ptr(), n=n,
                         wait_flag=base, epoch=base + 16, error_flag=base + 20,
                         publish_flag=base + 8, done=base + 12, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(peer_g, want + src) and words.tolist()[:6] == [2, 0, 2, 0, 2, 0]


def test_exchange_kernels_reject_bad_arguments(nat):
    ext = nat.ext()
    x = torch.zeros(16, device="cuda")
    with pytest.raises(RuntimeError, match="code 930"):
        ext.tied_grad_push(src=x.data_ptr(), dst=0, n=16, flag=x.data_ptr(), done=x.data_ptr())
    with pytest.raises(RuntimeError, match="code 931"):
        ext.tied_grad_push(src=x.data_ptr() + 4, dst=x.data_ptr(), n=4, flag=x.data_ptr(),
                           done=x.data_ptr())


@pytest.mark.parametrize("optim", ["SGD", "LAMB"])
def test_norm_exclusion_leaves_the_replica_out_of_the_fused_norm(nat, optim):
    """What the last rank of a tied pipeline does: its replica's bank (here the table's bank, the
    mechanism is the same) and a parameter outside the banks (a torch fallback layer) are left out
    of this rank's share of the squared norm: grad_sumsq_multi runs over its own descriptor table
    and the fallback's sum skips the parameter."""
    import skycomputing_b200 as sky
    from skycomputing_b200.models import set_backend

    set_backend("native")
    try:
        stage = sky.build_module_from_cfg(0, _model_cfg(1), dict(module_to_cuda=True,
                                                                  cuda_device=0))
        _seed(stage)
        extra = torch.nn.Linear(16, 16).cuda()        # outside the banks: the torch fallback
        mod = torch.nn.ModuleList([stage, extra])
        opt = sky.build_optimizer(mod, dict(optim_type=optim, lr=0.0), grad_clip=dict(max_norm=1e-3))
        table = stage.layers[0].word_embeddings.weight
        opt.set_norm_exclude([table, extra.weight])
        (d, l), = _batches(1, batch=8)
        logits = stage(*[t.cuda() for t in d])[0]
        sky.MaskedLMLoss()(logits.float(), l.cuda()).backward()
        extra.weight.grad = torch.randn_like(extra.weight)
        extra.bias.grad = torch.randn_like(extra.bias)
        torch.cuda.synchronize()
        skip = {id(table), id(extra.weight)}
        params = [p for p in mod.parameters() if p.grad is not None]
        want = math.sqrt(sum(float(p.grad.double().pow(2).sum()) for p in params
                             if id(p) not in skip))
        full = math.sqrt(sum(float(p.grad.double().pow(2).sum()) for p in params))
        opt.step()
        torch.cuda.synchronize()
        got = opt.scalars()["grad_norm"]
    finally:
        set_backend("auto")
    assert got == pytest.approx(want, rel=1e-4)
    assert abs(full - want) > 1e-2 * want                  # the exclusion changed the norm
