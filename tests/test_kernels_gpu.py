"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    assert native.available(), "native extension must be built and a GPU present"
    return native


def _rand(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(dtype)


def _close(got, ref, rtol=2e-2, atol=2e-2):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs().max().item()
    denom = ref.abs().max().item() + 1e-6
    assert torch.isfinite(got).all(), "non-finite output"
    assert err <= atol + rtol * denom, f"max abs err {err} vs ref max {denom}"


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(256, 512, 320), (200, 264, 64), (1024, 1024, 1024), (32, 1024, 1024)])
def test_gemm_kk(nat, M, N, K, block_n):
    torch.manual_seed(0)
    a, b = _rand(M, K), _rand(N, K)
    bias = torch.randn(N, device="cuda")
    out = nat.gemm(a, b, bias=bias, block_n=block_n)
    ref = a.float() @ b.float().t() + bias
    _close(out, ref, atol=0.05 * math.sqrt(K) / 8)


def test_gemm_strided_views(nat):
    torch.manual_seed(1)
    big = _rand(512, 3 * 256)
    a = big[:, 256:512]  # row stride 768, inner stride 1
    b = _rand(384, 256)
    out = nat.gemm(a, b)
    _close(out, a.float() @ b.float().t(), atol=0.2)


def test_gemm_gelu_dual_output(nat):
    torch.manual_seed(2)
    M, N, K = 384, 768, 256
    a, b = _rand(M, K), _rand(N, K, scale=0.1)
    bias = torch.randn(N, device="cuda") * 0.1
    pre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    out = nat.gemm(a, b, bias=bias, act=nat.ACT_GELU, out2=pre)
    h = a.float() @ b.float().t() + bias
    _close(pre, h)
    _close(out, h * 0.5 * (1.0 + torch.erf(h / math.sqrt(2.0))))


def test_gemm_residual_and_dgelu(nat):
    torch.manual_seed(3)
    M, N, K = 256, 512, 512
    a, b = _rand(M, K, scale=0.2), _rand(N, K, scale=0.2)
    aux = _rand(M, N)
    out = nat.gemm(a, b, aux=aux, add_aux=True)
    _close(out, a.float() @ b.float().t() + aux.float())
    out = nat.gemm(a, b, aux=aux, act=nat.ACT_DGELU_MUL_AUX)
    x = aux.float()
    dg = 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    _close(out, (a.float() @ b.float().t()) * dg)


@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_dgrad_layout(nat, block_n):
    """dX[M,K] = dY[M,N] W[N,K]: A K-major, B MN-major (no transposed weight copy)."""
    torch.manual_seed(4)
    M, N, K = 384, 320, 512  # reduction over N
    dy, w = _rand(M, N), _rand(N, K, scale=0.2)
    out = nat.gemm(dy, w, b_mn=True, block_n=block_n)
    _close(out, dy.float() @ w.float(), atol=0.2)


@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_wgrad_layout_f32_accumulate(nat, block_n):
    """dW[N,K] (+)= dY^T[N,M] X[M,K]: both operands MN-major, fp32 output with accumulation."""
    torch.manual_seed(5)
    M, N, K = 640, 384, 512  # reduction over M (tokens)
    dy, x = _rand(M, N, scale=0.3), _rand(M, K, scale=0.3)
    dw = torch.ones(N, K, device="cuda", dtype=torch.float32)
    nat.gemm(dy, x, a_mn=True, b_mn=True, out=dw, accumulate=True, block_n=block_n)
    _close(dw, 1.0 + dy.float().t() @ x.float(), rtol=1e-2, atol=0.05)
    dw2 = nat.gemm(dy, x, a_mn=True, b_mn=True, out_dtype=torch.float32, block_n=block_n)
    _close(dw2, dy.float().t() @ x.float(), rtol=1e-2, atol=0.05)


def test_gemm_dropout_mask_consistent_with_layernorm_bwd(nat):
    torch.manual_seed(6)
    M, H = 256, 1024
    rng = nat.RngState(1234)
    a = torch.zeros(M, 64, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(H, 64, dtype=torch.bfloat16, device="cuda")
    ones = torch.ones(H, device="cuda")
    p = 0.1
    out = nat.gemm(a, b, bias=ones, dropout_p=p, rng=rng, rng_stream=7).float()
    keep = out != 0
    frac = keep.float().mean().item()
    assert abs(frac - (1 - p)) < 0.01, frac
    _close(out[keep], torch.full_like(out[keep], 1 / (1 - p)))
    # LayerNorm backward must regenerate the identical mask for dz_dropped
    z = _rand(M, H)
    dy = _rand(M, H)
    gamma = torch.ones(H, device="cuda")
    beta = torch.zeros(H, device="cuda")
    _, mean, rstd = nat.layernorm_fwd(z, gamma, beta)
    dg = torch.zeros(H, device="cuda")
    db = torch.zeros(H, device="cuda")
    dz, dzd = nat.layernorm_bwd(dy, z, mean, rstd, gamma, dg, db, dropout_p=p, rng=rng, rng_stream=7)
    expect = torch.where(keep, dz.float() / (1 - p), torch.zeros_like(dz.float()))
    _close(dzd, expect)
    # a different step gives a different mask
    rng.advance()
    out2 = nat.gemm(a, b, bias=ones, dropout_p=p, rng=rng, rng_stream=7).float()
    assert ((out2 != 0) != keep).float().mean().item() > 0.05


@pytest.mark.parametrize("H", [64, 256, 1024])
def test_layernorm_fwd_bwd(nat, H):
    torch.manual_seed(7)
    M = 300
    z = _rand(M, H, scale=2.0)
    gamma = torch.randn(H, device="cuda") * 0.5 + 1
    beta = torch.randn(H, device="cuda") * 0.1
    y, mean, rstd = nat.layernorm_fwd(z, gamma, beta, 1e-12)
    zf = z.float().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    bt = beta.clone().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(zf, (H,), g, bt, 1e-12)
    _close(y, ref)
    dy = _rand(M, H)
    ref.backward(dy.float())
    dg = torch.zeros(H, device="cuda")
    db = torch.zeros(H, device="cuda")
    dz, _ = nat.layernorm_bwd(dy, z, mean, rstd, gamma, dg, db)
    _close(dz, zf.grad)
    _close(dg, g.grad, rtol=2e-2, atol=0.3)
    _close(db, bt.grad, rtol=2e-2, atol=0.3)


def test_colsum(nat):
    x = _rand(1000, 768)
    out = torch.ones(768, device="cuda")
    nat.colsum_(x, out)
    _close(out, 1 + x.float().sum(0), rtol=1e-3, atol=1e-2)


def _attention_ref(qkv, mask, B, S, heads):
    H = qkv.shape[1] // 3
    d = H // heads
    q, k, v = qkv.float().view(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(d)
    if mask is not None:
        s = s + mask.view(B, 1, 1, S)
    p = torch.softmax(s, -1)
    o = p @ v
    return o.permute(0, 2, 1, 3).reshape(B * S, H)


@pytest.mark.parametrize("with_mask", [False, True])
def test_attention_fwd_bwd(nat, with_mask):
    torch.manual_seed(8)
    B, S, heads, d = 3, 128, 4, 64
    H = heads * d
    qkv = _rand(B * S, 3 * H)
    mask = None
    if with_mask:
        m = torch.ones(B, S, device="cuda")
        m[0, 100:] = 0
        m[2, 17:] = 0
        mask = (1.0 - m) * -10000.0
    ctx, lse = nat.attention_fwd(qkv, mask, B, S, heads)
    qf = qkv.float().requires_grad_(True)
    ref = _attention_ref(qf, mask, B, S, heads)
    _close(ctx, ref)
    dctx = _rand(B * S, H)
    ref.backward(dctx.float())
    dqkv = nat.attention_bwd(qkv, mask, ctx, lse, dctx, B, S, heads)
    _close(dqkv, qf.grad, rtol=3e-2, atol=3e-2)


def test_attention_dropout_statistics(nat):
    torch.manual_seed(9)
    B, S, heads, d = 2, 128, 2, 64
    H = heads * d
    qkv = torch.zeros(B * S, 3 * H, dtype=torch.bfloat16, device="cuda")
    qkv[:, 2 * H:] = 1.0  # V = 1 -> ctx = sum_j P_ij keep_ij / (1-p) ~ 1
    rng = nat.RngState(77)
    ctx, _ = nat.attention_fwd(qkv, None, B, S, heads, dropout_p=0.1, rng=rng, rng_stream=3)
    c = ctx.float()
    assert abs(c.mean().item() - 1.0) < 0.02
    assert 0.01 < c.std().item() < 0.1


def test_softmax_ce(nat):
    torch.manual_seed(10)
    logits = torch.randn(32, 3, device="cuda")
    labels = torch.randint(0, 3, (32,), device="cuda")
    loss, dl = nat.softmax_ce(logits, labels)
    lf = logits.clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf, labels)
    ref.backward()
    _close(loss, ref.detach().view(1), rtol=1e-4, atol=1e-5)
    _close(dl, lf.grad, rtol=1e-4, atol=1e-6)


def test_gemm_flag_handshake_single_gpu(nat):
    """Consumer GEMM launched FIRST on a side stream must wait for the producer's panel flags."""
    torch.manual_seed(11)
    M, H, I = 512, 256, 512
    x, w1, w2 = _rand(M, H), _rand(I, H, scale=0.1), _rand(H, I, scale=0.1)
    mid = torch.zeros(M, I, dtype=torch.bfloat16, device="cuda")
    flags = torch.zeros(M // 128, dtype=torch.int32, device="cuda")
    epoch = torch.ones(1, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty(M, H, dtype=torch.bfloat16, device="cuda")
    bn = 128
    tiles = nat.ext().gemm_tiles_per_panel(I, bn)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        nat.gemm(mid, w2, out=out, wait_flags=flags.data_ptr(), wait_epoch=epoch.data_ptr(),
                 wait_mult=tiles, error_flag=err.data_ptr(), max_ctas=8)
    nat.gemm(x, w1, out=mid, signal_flags=flags.data_ptr(), block_n=bn, max_ctas=16)
    torch.cuda.synchronize()
    assert err.item() == 0
    assert flags.tolist() == [tiles] * (M // 128)
    ref_mid = (x.float() @ w1.float().t()).to(torch.bfloat16)
    _close(out, ref_mid.float() @ w2.float().t(), atol=0.1)


@pytest.mark.parametrize("pair,stream_k", [(1, 0), (0, 1), (1, 1), (2, 0), (2, 1)])
@pytest.mark.parametrize("M,N,K", [(2048, 1024, 4096), (1000, 520, 1096), (4096, 1024, 1024)])
def test_gemm_pair_and_stream_k_schedules(nat, M, N, K, pair, stream_k):
    """2- / 4-CTA clusters (TMA multicast) and the stream-K schedule (split tiles reduced through the
    workspace by the last-arriving CTA) must match the classic schedule bit-for-bit in layout and
    closely in value; run twice so the second launch sees the counters the first one left."""
    torch.manual_seed(11)
    a, b = _rand(M, K), _rand(N, K)
    bias = torch.randn(N, device="cuda")
    ref = a.float() @ b.float().t() + bias
    for block_n in (128, 256):
        for _ in range(2):
            out = nat.gemm(a, b, bias=bias, block_n=block_n, pair=pair, stream_k=stream_k)
            _close(out, ref, atol=0.05 * math.sqrt(K) / 8)
    # dgrad / wgrad operand layouts
    dy = _rand(M, N)
    dx = nat.gemm(dy, b, b_mn=True, pair=pair, stream_k=stream_k)
    _close(dx, dy.float() @ b.float(), atol=0.05 * math.sqrt(N) / 8)
    if M % 8 == 0:
        dw = torch.zeros(N, K, device="cuda", dtype=torch.float32)
        for _ in range(2):
            nat.gemm(dy, a, a_mn=True, b_mn=True, out=dw, accumulate=True, pair=pair, stream_k=stream_k)
        _close(dw, 2 * (dy.float().t() @ a.float()), atol=0.05 * math.sqrt(M) / 4)


def test_gemm_stream_k_fused_epilogue(nat):
    """GELU + second output + residual paths on a split tile (only the finishing CTA applies them)."""
    torch.manual_seed(12)
    M, N, K = 512, 512, 2048
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    pre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    out = nat.gemm(a, b, bias=bias, act=nat.ACT_GELU, out2=pre, stream_k=1)
    h = a.float() @ b.float().t() + bias
    _close(pre, h)
    _close(out, h * 0.5 * (1.0 + torch.erf(h / math.sqrt(2.0))))
    res = _rand(M, N)
    out = nat.gemm(a, b, bias=bias, aux=res, add_aux=True, stream_k=1, pair=1)
    _close(out, h + res.float())


# ------------------------------------------------------------------------------------------
# GEMM + bias + dropout + residual + LayerNorm in one kernel (cluster-wide row statistics)
# ------------------------------------------------------------------------------------------
def _ln_ref(zf, gamma, beta, eps=1e-12):
    mu = zf.mean(-1, keepdim=True)
    var = ((zf - mu) ** 2).mean(-1, keepdim=True)
    return (zf - mu) / torch.sqrt(var + eps) * gamma + beta, mu.squeeze(-1), (1 / torch.sqrt(var + eps)).squeeze(-1)


@pytest.mark.parametrize("M,N,K,block_n", [
    (4096, 1024, 1024, 0),      # BERT-large attention output projection: 4-CTA clusters, 256-wide
    (2048, 1024, 4096, 0),      # BERT-large FFN2 at 16 sequences: 8-CTA clusters, 128-wide
    (4096, 1024, 4096, 256),
    (512, 256, 512, 0),         # 2-CTA clusters
    (300, 256, 192, 128),       # ragged M
    (128, 128, 64, 128),        # a cluster of one
    (256, 768, 256, 0),         # 3 / 6 CTAs per cluster (not a power of two)
])
def test_gemm_layernorm_epilogue(nat, M, N, K, block_n):
    torch.manual_seed(11)
    assert nat.ext().gemm_ln_block_n(M, N, True) != 0
    # the automatic policy only fuses launches that fill the GPU with 256-wide tiles
    assert nat.gemm_ln_supported(M, N) == (N % 256 == 0 and ((M + 127) // 128) * (N // 256) >= 96)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    res = _rand(M, N)
    gamma = 1.0 + 0.1 * torch.randn(N, device="cuda")
    beta = 0.1 * torch.randn(N, device="cuda")
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, bias=bias, residual=res, block_n=block_n)
    zf = a.float() @ w.float().t() + bias + res.float()
    yr, mur, rstdr = _ln_ref(zf, gamma, beta)
    _close(z, zf)
    _close(y, yr, rtol=2e-2, atol=3e-2)
    torch.testing.assert_close(mean, mur, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(rstd, rstdr, rtol=2e-3, atol=1e-4)
    # and against the two-kernel path it replaces (same bf16 rounding points except the stats)
    z2 = nat.gemm(a, w, bias=bias, aux=res, add_aux=True)
    y2, mean2, rstd2 = nat.layernorm_fwd(z2, gamma, beta)
    assert torch.equal(z, z2)
    _close(y, y2, rtol=1e-2, atol=2e-2)


def test_gemm_layernorm_epilogue_dropout_uses_the_gemm_mask(nat):
    torch.manual_seed(12)
    M, N, K, p = 512, 1024, 256, 0.1
    rng = nat.RngState(99)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    res = _rand(M, N)
    gamma, beta = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    # the mask of (rng, stream 5) for an [M, N] output, read off a GEMM of zeros + bias 1
    probe = nat.gemm(torch.zeros(M, 64, dtype=torch.bfloat16, device="cuda"),
                     torch.zeros(N, 64, dtype=torch.bfloat16, device="cuda"),
                     bias=torch.ones(N, device="cuda"), dropout_p=p, rng=rng, rng_stream=5).float()
    keep = probe != 0
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, bias=bias, residual=res, dropout_p=p,
                                   rng=rng, rng_stream=5)
    h = a.float() @ w.float().t() + bias
    zf = torch.where(keep, h / (1 - p), torch.zeros_like(h)) + res.float()
    _close(z, zf)
    _close(y, _ln_ref(zf, gamma, beta)[0], rtol=2e-2, atol=3e-2)
    # LayerNorm backward regenerates the same mask from (rng, stream)
    dy = _rand(M, N)
    dz, dzd = nat.layernorm_bwd(dy, z, mean, rstd, gamma, None, None, dropout_p=p, rng=rng,
                                rng_stream=5)
    _close(dzd, torch.where(keep, dz.float() / (1 - p), torch.zeros_like(dz.float())))


def test_gemm_layernorm_epilogue_signals_panels_like_a_stage_boundary(nat):
    """y redirected to a raw pointer + panel flags (single GPU stand-in for the peer slot): every
    128-row panel receives gemm_ln_tiles_per_panel signals; a consumer GEMM gated on those flags
    reads the complete tensor."""
    torch.manual_seed(13)
    M, N, K = 1024, 1024, 512
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    gamma, beta = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    slot = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    flags = torch.zeros(M // 128, dtype=torch.int32, device="cuda")
    epoch = torch.ones(1, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    mult = nat.ext().gemm_ln_tiles_per_panel(M, N, True)
    assert mult == 4
    y, z, _, _ = nat.gemm_ln(a, w, gamma, beta, y_ptr=slot.data_ptr(), y_ld=N,
                             signal_flags=flags.data_ptr())
    assert y is None
    w2 = _rand(256, N, scale=0.05)
    out = nat.gemm(slot, w2, wait_flags=flags.data_ptr(), wait_epoch=epoch.data_ptr(),
                   wait_mult=mult, error_flag=err.data_ptr())
    torch.cuda.synchronize()
    assert flags.tolist() == [mult] * (M // 128) and int(err.item()) == 0
    yr = _ln_ref(z.float(), gamma, beta)[0]
    _close(slot, yr, rtol=2e-2, atol=3e-2)
    _close(out, slot.float() @ w2.float().t(), atol=0.3)


# ------------------------------------------------------------------------------------------
# attention for any sequence length (flash-style tiled kernels; S = 128 has its own kernels)
# ------------------------------------------------------------------------------------------
def _attention_ref_masked(qkv, mask, B, S, heads, keep=None, p=0.0):
    H = qkv.shape[1] // 3
    d = H // heads
    q, k, v = qkv.float().view(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(d)
    if mask is not None:
        s = s + mask.view(B, 1, 1, S)
    pr = torch.softmax(s, -1)
    if keep is not None:
        pr = pr * keep.to(pr.dtype) / (1.0 - p)
    o = pr @ v
    return o.permute(0, 2, 1, 3).reshape(B * S, H)


@pytest.mark.parametrize("S", [64, 192, 256, 384, 512, 72])
def test_attention_tiled_any_sequence_length(nat, S):
    """64 (< one tile), 192 / 72 (ragged last tile), 256 / 384 / 512 (2-4 tiles): forward, lse and
    all three gradients against the fp32 reference, with a padding mask."""
    torch.manual_seed(20 + S)
    B, heads, d = 2, 3, 64
    H = heads * d
    assert nat.ext().attention_supported(S, d)
    qkv = _rand(B * S, 3 * H)
    m = torch.ones(B, S, device="cuda")
    m[0, S - S // 4:] = 0
    m[1, S // 2:] = 0
    mask = (1.0 - m) * -10000.0
    ctx, lse = nat.attention_fwd(qkv, mask, B, S, heads)
    qf = qkv.float().requires_grad_(True)
    ref = _attention_ref_masked(qf, mask, B, S, heads)
    _close(ctx, ref)
    # log-sum-exp (log2 domain) of the scaled, masked scores
    q, k, _ = qkv.float().view(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
    sc = q @ k.transpose(-1, -2) / math.sqrt(d) + mask.view(B, 1, 1, S)
    lse_ref = torch.logsumexp(sc, -1) / math.log(2.0)
    _close(lse.view(B, heads, S), lse_ref, rtol=1e-3, atol=2e-2)
    dctx = _rand(B * S, H)
    ref.backward(dctx.float())
    dqkv = nat.attention_bwd(qkv, mask, ctx, lse, dctx, B, S, heads)
    _close(dqkv[:, :H], qf.grad[:, :H], rtol=3e-2, atol=3e-2)           # dQ
    _close(dqkv[:, H:2 * H], qf.grad[:, H:2 * H], rtol=3e-2, atol=3e-2)  # dK
    _close(dqkv[:, 2 * H:], qf.grad[:, 2 * H:], rtol=3e-2, atol=3e-2)   # dV


@pytest.mark.parametrize("S", [128, 256, 72])
def test_attention_dropout_exact_mask_parity(nat, S):
    """Dropout on the probabilities: the host replica of the device RNG gives the exact keep mask
    of the [B, heads, S, S] site; forward and gradients must match the fp32 reference that applies
    that mask (S = 128: single-tile kernels, S = 256: tiled kernels - same element indexing,
    S = 72: a ragged tile whose fragment rows past the end still take part in the mask shuffles)."""
    from skycomputing_b200.ops.dropout_ref import keep_mask_from_state

    torch.manual_seed(31)
    B, heads, d, p = 2, 2, 64, 0.1
    H = heads * d
    rng = nat.RngState(4242)
    qkv = _rand(B * S, 3 * H)
    ctx, lse = nat.attention_fwd(qkv, None, B, S, heads, dropout_p=p, rng=rng, rng_stream=11)
    keep = torch.from_numpy(keep_mask_from_state(rng.state, 11, (B, heads, S, S), p)).cuda()
    assert abs(float(keep.float().mean()) - (1 - p)) < 1e-2
    qf = qkv.float().requires_grad_(True)
    ref = _attention_ref_masked(qf, None, B, S, heads, keep=keep, p=p)
    _close(ctx, ref)
    dctx = _rand(B * S, H)
    ref.backward(dctx.float())
    dqkv = nat.attention_bwd(qkv, None, ctx, lse, dctx, B, S, heads, dropout_p=p, rng=rng,
                             rng_stream=11)
    _close(dqkv, qf.grad, rtol=3e-2, atol=3e-2)


def test_attention_tiled_matches_single_tile_kernels_at_128(nat, monkeypatch):
    """SKY_ATTN_TILED is read once per process, so compare through a subprocess-free trick: the
    tiled launcher is reachable directly for S = 128 by passing a [B*2, 64]-folded problem - the
    same tokens seen as sequences of 64 must differ, while S = 128 through both paths must agree;
    here: tiled S = 256 on a batch whose second half of every sequence is masked out equals the
    single-tile S = 128 result on the first halves."""
    torch.manual_seed(33)
    B, heads, d = 2, 2, 64
    H = heads * d
    S2 = 256
    qkv = _rand(B * S2, 3 * H)
    m = torch.ones(B, S2, device="cuda")
    m[:, 128:] = 0
    mask = (1.0 - m) * -10000.0
    ctx2, _ = nat.attention_fwd(qkv, mask, B, S2, heads)                 # tiled kernels
    first = qkv.view(B, S2, 3 * H)[:, :128].reshape(B * 128, 3 * H).contiguous()
    ctx1, _ = nat.attention_fwd(first, None, B, 128, heads)              # single-tile kernels
    _close(ctx2.view(B, S2, H)[:, :128].reshape(B * 128, H), ctx1, rtol=1e-2, atol=1e-2)
