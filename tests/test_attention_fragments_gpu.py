"""S = 128 attention kernels on wgmma accumulator fragments, at the BERT-large training geometry.

The small cases in test_kernels_gpu.py launch a handful of CTAs; here B = 32 and 16 heads put 512
CTAs on the GPU, so every SM runs several of them (the forward is resident two per SM).  The
reference is the fp32 attention with the exact dropout keep mask from the host replica of the RNG.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

B, S, HEADS, D = 32, 128, 16, 64
H = HEADS * D
P_DROP = 0.1
STREAM = 5


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    assert native.available(), "native extension must be built and a GPU present"
    return native


def _close(got, ref, rtol, atol, what):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs().max().item()
    lim = atol + rtol * ref.abs().max().item()
    assert err <= lim, f"{what}: max abs err {err} > {lim}"


def _inputs(seed, padded):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * S, 3 * H, device="cuda", generator=g).to(torch.bfloat16)
    dctx = torch.randn(B * S, H, device="cuda", generator=g).to(torch.bfloat16)
    mask = None
    if padded:
        # a different number of fully masked tail keys per sequence (none in some)
        lens = torch.randint(40, S + 1, (B,), device="cuda", generator=g)
        lens[0] = S
        keep = torch.arange(S, device="cuda")[None, :] < lens[:, None]
        mask = (1.0 - keep.float()) * -10000.0
    return qkv, dctx, mask


def _reference(qkv, mask, keep, p):
    q, k, v = qkv.float().view(B, S, 3, HEADS, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(D)
    if mask is not None:
        s = s + mask.view(B, 1, 1, S)
    lse2 = torch.logsumexp(s, -1) / math.log(2.0)  # log2 domain, as the kernels store it
    pr = torch.softmax(s, -1)
    if keep is not None:
        pr = pr * keep.to(pr.dtype) / (1.0 - p)
    o = pr @ v
    return o.permute(0, 2, 1, 3).reshape(B * S, H), lse2.reshape(-1)


@pytest.mark.parametrize("padded", [False, True], ids=["nomask", "padmask"])
@pytest.mark.parametrize("p", [0.0, P_DROP], ids=["p0", "p0.1"])
def test_attention_fragments_training_geometry(nat, padded, p):
    from skycomputing_b200.ops.dropout_ref import keep_mask_from_state

    qkv, dctx, mask = _inputs(100 + int(padded) + int(p > 0) * 2, padded)
    rng = nat.RngState(9001) if p > 0 else None
    kw = dict(dropout_p=p, rng=rng, rng_stream=STREAM)
    ctx, lse = nat.attention_fwd(qkv, mask, B, S, HEADS, **kw)
    dqkv = nat.attention_bwd(qkv, mask, ctx, lse, dctx, B, S, HEADS, **kw)
    keep = None
    if p > 0:
        keep = torch.from_numpy(keep_mask_from_state(rng.state, STREAM, (B, HEADS, S, S), p)).cuda()
    qf = qkv.float().requires_grad_(True)
    ref, ref_lse = _reference(qf, mask, keep, p)
    ref.backward(dctx.float())
    _close(ctx, ref, 2e-2, 2e-2, "ctx")
    _close(lse, ref_lse, 0.0, 2e-3, "lse")
    g, rg = dqkv.view(B * S, 3, H), qf.grad.view(B * S, 3, H)
    for i, name in enumerate(("dQ", "dK", "dV")):
        _close(g[:, i], rg[:, i], 3e-2, 3e-2, name)
    if padded:
        # keys that every query of a sequence ignores get no gradient
        dead = (mask != 0).view(B * S)
        assert dead.any()
        assert float(g[dead, 1].float().abs().max()) == 0.0
        assert float(g[dead, 2].float().abs().max()) == 0.0


@pytest.mark.parametrize("p", [0.0, P_DROP], ids=["p0", "p0.1"])
def test_attention_inference_ctx_matches_training_forward(nat, p):
    """``save_lse=False`` passes a null lse pointer; ctx must carry the same bits."""
    qkv, _, mask = _inputs(7, True)
    rng = nat.RngState(31) if p > 0 else None
    ctx_t, lse = nat.attention_fwd(qkv, mask, B, S, HEADS, dropout_p=p, rng=rng, rng_stream=STREAM)
    ctx_i, none = nat.attention_fwd(qkv, mask, B, S, HEADS, dropout_p=p, rng=rng,
                                    rng_stream=STREAM, save_lse=False)
    assert none is None and lse is not None
    assert torch.equal(ctx_t.view(torch.int16), ctx_i.view(torch.int16))


def test_attention_graph_replay_matches_eager(nat):
    """Forward + backward captured in a CUDA graph and replayed twice: bit-identical to an eager
    call with the same RNG state."""
    qkv, dctx, mask = _inputs(11, True)
    rng = nat.RngState(2024)
    kw = dict(dropout_p=P_DROP, rng=rng, rng_stream=STREAM)
    ctx_e, lse_e = nat.attention_fwd(qkv, mask, B, S, HEADS, **kw)
    dqkv_e = nat.attention_bwd(qkv, mask, ctx_e, lse_e, dctx, B, S, HEADS, **kw)
    torch.cuda.synchronize()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up outside the capture
        c, l_ = nat.attention_fwd(qkv, mask, B, S, HEADS, **kw)
        nat.attention_bwd(qkv, mask, c, l_, dctx, B, S, HEADS, **kw)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx_g, lse_g = nat.attention_fwd(qkv, mask, B, S, HEADS, **kw)
        dqkv_g = nat.attention_bwd(qkv, mask, ctx_g, lse_g, dctx, B, S, HEADS, **kw)
    for _ in range(2):
        for t in (ctx_g, lse_g, dqkv_g):
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ctx_g.view(torch.int16), ctx_e.view(torch.int16))
        assert torch.equal(lse_g.view(torch.int32), lse_e.view(torch.int32))
        assert torch.equal(dqkv_g.view(torch.int16), dqkv_e.view(torch.int16))
