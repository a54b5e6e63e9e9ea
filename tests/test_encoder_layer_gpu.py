"""The encoder layer's kernels against fp64 references of the same operation: the wgmma GEMM in
the six calls a layer makes, the GEMM + LayerNorm kernel and the GEMM + standalone LayerNorm it
replaces, the S = 128 and the tiled attention kernels, and one whole BERT-large layer with
dropout on, stage by stage, over two micro-batches and end to end.

As in test_model_ends_gpu.py, every reference is computed in fp64 from exactly what the kernel
received and every element is checked against its own worst-case bound (tests/_fp64_bounds.py):
the output rounding, n * u * sum|terms| of each accumulation and the documented error of each
approximate intrinsic.  Dropout uses the exact keep masks of ``keep_mask_from_state``.  The GEMM
runs its production tile policy (``block_n`` = 0: no pair or stream-K override) and, explicitly,
``block_n`` = 128 and 256.
"""
import math

import pytest
import torch

from tests._encoder_layer_ref import PARAM_NAMES, layer_params, layer_ref
from tests._fp64_bounds import (BF16, DEV, DROP, EXPF_ULPS, F64, RSQRT_APPROX, U, U_TC, _bf16_out,
                                _keep, _ln_input_grad_ref, _within)

pytestmark = pytest.mark.gpu

ERF_AS = 1.5e-7              # Abramowitz-Stegun 7.1.26: |erf error| < 1.5e-7, absolute
EX2_APPROX = 2.0 ** -22      # PTX ISA: ex2.approx.f32 (exp2f under fast math) max relative error
LG2_APPROX = 2.0 ** -22      # PTX ISA: lg2.approx.f32 (log2f): 2^-22.6 absolute on [0.5, 2]
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
ACT_NONE, ACT_GELU, ACT_DGELU = 0, 1, 2
BLOCK_NS = (0, 128, 256)     # 0: the production pick


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    assert native.available(), "native extension must be built and a GPU present"
    return native


def _bf(t):
    return t.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------
# GELU and its derivative as the GEMM epilogue evaluates them (gelu_fast / dgelu_fast)
# ---------------------------------------------------------------------------------------------
def _gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _dgelu64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(
        2 * math.pi)


def _erf_err(z):
    """|erf_exp_fast(z) - erf(z)|: the A-S polynomial (1.5e-7 absolute), 1 - poly * e rounded, and
    poly * e = erfc(z) off relatively by __expf (2 + 1.173 z^2 ulp), the rounded argument z^2
    (relative 4u each on z, z^2: 5u z^2 absolute in the exponent) and rcp.approx + Horner (20u)."""
    return ERF_AS + U + torch.erfc(z) * ((2 + EXPF_ULPS * z * z) * 2.0 ** -23 + 5 * U * z * z
                                         + 20 * U)


def _gelu_err(x):
    """gelu_fast = 0.5 x (1 + copysign(erf)): the erf error scaled by 0.5 |x| and a few roundings.
    Where GELU(x) -> 0 (x < -5) the result is the difference 1 - erf(|z|) ~ 0, so the bound is
    ABSOLUTE, about |x| (1.5e-7 + u), not relative to the tiny GELU value."""
    return 0.5 * x.abs() * _erf_err(x.abs() / math.sqrt(2.0)) + 4 * U * (_gelu64(x).abs()
                                                                          + 0.5 * x.abs())


def _dgelu_err(x):
    """dgelu_fast = cdf + x pdf: half the erf error in the cdf, the __expf error of the density,
    and the fma rounding."""
    z = x.abs() / math.sqrt(2.0)
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    return (0.5 * _erf_err(z) + (x * pdf).abs() * ((2 + EXPF_ULPS * z * z) * 2.0 ** -23
                                                   + 5 * U * z * z + 4 * U)
            + 2 * U * _dgelu64(x).abs() + U)


# ---------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------
def _acc_err(K):
    """Relative (to sum|products|) error of a K-long fp32 tensor-core accumulation: each k16
    wgmma step adds 16 exact bf16 products to the accumulator as one fused sum, off by at most
    2 ulp of the largest magnitude involved (addend alignment + the final rounding), and there
    are K / 16 steps; + 32 ulp for the k-block tail and stream-K partial additions."""
    return (K / 8 + 32) * U_TC


def _reduce_depth(M):
    """Additions on the longest path of a column sum over M rows in ln_param_grad / colsum: one
    thread sums every (8 x grid.y)-th row (grid.y = min(64, ceil(M / 64))), then 8 shared-memory
    partials, then grid.y atomics onto the initial value."""
    ry = min(64, -(-M // 64))
    return -(-M // (8 * ry)) + 8 + ry + 1


def _ln_twopass_ref(zb, gamma, beta, eps):
    """layernorm_fwd of bf16 rows (exact inputs), as ``_ln_fwd_ref`` but with the kernel's
    summation depth: a warp per row, each lane sums H / 32 elements, then 5 shuffle levels."""
    H = zb.shape[1]
    g, b = gamma.to(F64), beta.to(F64)
    depth = H // 32 + 8
    mu = zb.mean(1, keepdim=True)
    var = ((zb - mu) ** 2).mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(var + eps)
    xh = (zb - mu) * rs
    y = xh * g + b
    d_mu = depth * U * zb.abs().mean(1, keepdim=True) + U * mu.abs()
    # (z - mu)^2 with mu off by d_mu: 2 d_mu sum|z - mu| <= 2 d_mu H sigma, plus the sum itself
    sig = torch.sqrt(var)
    var_rel = (2 * d_mu * sig + d_mu * d_mu) / (var + eps) + (depth + 6) * U
    rs_rel = 0.5 * 1.01 * var_rel + RSQRT_APPROX + U
    d_xh = rs * d_mu + xh.abs() * (rs_rel + 3 * U)
    d_y = g.abs() * d_xh + 2 * U * ((xh * g).abs() + b.abs())
    return (y, mu.squeeze(1), rs.squeeze(1)), (d_y, d_mu.squeeze(1), (rs * rs_rel).squeeze(1))


def _gemm_ref(a, b, a_mn=False, b_mn=False, bias=None, act=ACT_NONE, aux=None, add_aux=False,
              kf=None):
    """fp64 value and fp32 error of the epilogue chain acc (+ bias) (act) (dropout) (* dgelu(aux)
    | + aux), before the output rounding; also the pre-activation (out2) and its error."""
    A = (a.t() if a_mn else a).to(F64)
    Bm = (b.t() if b_mn else b).to(F64)
    v = A @ Bm.t()
    dv = _acc_err(A.shape[1]) * (A.abs() @ Bm.abs().t())
    if bias is not None:
        v = v + bias.to(F64)
        dv = dv + U * v.abs()                                  # one fp32 addition
    pre, d_pre = v, dv
    if act == ACT_GELU:
        v, dv = _gelu64(pre), 1.13 * d_pre + _gelu_err(pre)    # |gelu'| <= 1.13
    if kf is not None:
        v = v * kf
        dv = dv * kf + DROP * v.abs()
    if aux is not None:
        x = aux.to(F64)
        if act == ACT_DGELU:
            dg = _dgelu64(x)
            w = v * dg
            dv = dv * dg.abs() + v.abs() * _dgelu_err(x) + U * w.abs()
            v = w
        elif add_aux:
            v = v + x
            dv = dv + U * v.abs()
    return v, dv, pre, d_pre


def _inputs_for(kind, M, N, K, seed):
    """Operands of one of the layer's GEMM calls, scaled as in training; ``M`` tokens."""
    g = torch.Generator(device=DEV).manual_seed(seed)

    def rn(*shape, s=1.0):
        return _bf(torch.randn(*shape, device=DEV, generator=g) * s)

    bias = torch.randn(N, device=DEV, generator=g) * 0.5
    if kind == "qkv":
        return dict(a=rn(M, K), b=rn(N, K, s=K ** -0.5), bias=bias)
    if kind == "ffn1":
        # pre-activations out to +-8: row scales 1 .. 4 over the rows, a tail past x = -5
        a = torch.randn(M, K, device=DEV, generator=g)
        a = a * (1.0 + 1.5 * (torch.arange(M, device=DEV) % 16 == 0).float())[:, None]
        return dict(a=_bf(a), b=rn(N, K, s=1.5 * K ** -0.5), bias=bias, act=ACT_GELU)
    if kind == "dgrad_residual":
        return dict(a=rn(M, K), b=rn(K, N, s=K ** -0.5), b_mn=True, aux=rn(M, N),
                    add_aux=True)
    if kind == "dgrad_dgelu":
        return dict(a=rn(M, K), b=rn(K, N, s=K ** -0.5), b_mn=True, aux=rn(M, N, s=2.5),
                    act=ACT_DGELU)
    if kind == "dgrad":
        return dict(a=rn(M, K), b=rn(K, N, s=K ** -0.5), b_mn=True)
    raise KeyError(kind)


# (kind, N, K) of the layer's calls at H = 1024, I = 4096; the wgrad is tested on its own
LAYER_CALLS = [("qkv", 3072, 1024), ("ffn1", 4096, 1024), ("dgrad_residual", 1024, 3072),
               ("dgrad_dgelu", 4096, 1024), ("dgrad", 1024, 1024)]
GEMM_CASES = ([(kind, M, N, K) for M in (4096, 2048) for kind, N, K in LAYER_CALLS]
              + [(kind, 4000, 1000, 1096) for kind, _, _ in LAYER_CALLS])


@pytest.mark.parametrize("kind,M,N,K", GEMM_CASES)
def test_gemm_layer_call(nat, kind, M, N, K):
    """The GEMM as the layer calls it; M = 4000, N = 1000, K = 1096 has a ragged last row panel,
    column tile and k-block (1096 = 17 * 64 + 8)."""
    kw = _inputs_for(kind, M, N, K, seed=M + N + K + len(kind))
    ref, acc, pre, d_pre = _gemm_ref(**kw)
    bound = _bf16_out(ref, acc)
    worst = 0.0
    for bn in BLOCK_NS:
        out2 = torch.empty(M, N, dtype=torch.bfloat16, device=DEV) if kind == "ffn1" else None
        out = nat.gemm(kw["a"], kw["b"], b_mn=kw.get("b_mn", False), bias=kw.get("bias"),
                       act=kw.get("act", ACT_NONE), aux=kw.get("aux"),
                       add_aux=kw.get("add_aux", False), out2=out2, block_n=bn)
        tag = f"gemm {kind} M={M} N={N} K={K} block_n={bn}"
        worst = max(worst, _within(f"{tag} out", out, ref, bound))
        if out2 is not None:
            _within(f"{tag} out2", out2, pre, _bf16_out(pre, d_pre))
    if kind == "ffn1":
        assert float(pre.min()) < -5.0 and float(pre.max()) > 5.0, "no GELU tail exercised"
    assert 0 < worst <= 1


@pytest.mark.parametrize("M,N,K", [(4096, 4096, 1024), (4096, 1024, 4096), (4096, 3072, 1024),
                                   (2048, 4096, 1024), (4000, 1000, 1096)])
def test_gemm_wgrad_accumulates(nat, M, N, K):
    """dW = g^T act with both operands MN-major over M tokens into fp32: once with accumulate =
    False over a buffer of nonzero values (it must overwrite), then twice accumulating."""
    gen = torch.Generator(device=DEV).manual_seed(M + N + K)
    gs = [_bf(torch.randn(M, N, device=DEV, generator=gen)) for _ in range(3)]
    xs = [_bf(torch.randn(M, K, device=DEV, generator=gen)) for _ in range(3)]
    refs, bounds = [], []
    ref = torch.zeros(N, K, dtype=F64, device=DEV)
    bound = torch.zeros_like(ref)
    for i in range(3):
        v, dv, _, _ = _gemm_ref(gs[i], xs[i], a_mn=True, b_mn=True)
        # red.add onto the previous value: one more rounding of the running sum per partial
        bound = bound + dv + _acc_err(M) * ref.abs()
        ref = ref + v
        refs.append(ref)
        bounds.append(bound)
    for bn in BLOCK_NS:
        out = torch.randn(N, K, device=DEV, generator=gen) * 100
        for i in range(3):
            nat.gemm(gs[i], xs[i], a_mn=True, b_mn=True, out=out, accumulate=i > 0, block_n=bn)
            w = _within(f"wgrad M={M} N={N} K={K} block_n={bn} call {i}", out, refs[i],
                        bounds[i])
        assert 0 < w <= 1


# ---------------------------------------------------------------------------------------------
# GEMM + LayerNorm
# ---------------------------------------------------------------------------------------------
def _z_ref(a, w, bias, residual, kf):
    """z = dropout(a w^T + bias) + residual in fp64 and its fp32 error."""
    t, dt, _, _ = _gemm_ref(a, w, bias=bias)
    if kf is None:
        kf = torch.ones_like(t)
    tk = t * kf
    z = tk + residual.to(F64)
    dz = dt * kf + (DROP + U) * tk.abs() + U * z.abs()
    return z, dz


def _ln_onepass_ref(z, dz, gamma, beta, eps, depth):
    """The fused kernel's statistics: fp32 sums of z and z^2 (each row summed ``depth`` roundings
    deep: BLOCK_N / 4 per thread, 2 quad shuffles, one per cluster CTA), mean = s1 / N and
    var = max(s2 / N - mean^2, 0).  The one-pass variance cancels: its sum error
    depth * u * sum z^2 is relative depth * u * (mu^2 + sigma^2) / sigma^2 on the variance.
    Returns (y, mean, rstd) and their errors; y is normalised from the fp32 z."""
    N = z.shape[1]
    g, b = gamma.to(F64), beta.to(F64)
    mu = z.mean(1, keepdim=True)
    var = ((z - mu) ** 2).mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(var + eps)
    xh = (z - mu) * rs
    y = xh * g + b
    d_mu = (depth * U * z.abs().sum(1, keepdim=True) + dz.sum(1, keepdim=True)) / N + U * mu.abs()
    e2 = (z * z).mean(1, keepdim=True)
    d_s2 = depth * U * (z * z).sum(1, keepdim=True) + (2 * z.abs() * dz + dz * dz).sum(1, keepdim=True)
    d_var = d_s2 / N + U * e2 + 2 * mu.abs() * d_mu + d_mu * d_mu + U * (var + eps)
    rs_rel = 0.5 * 1.01 * d_var / (var + eps) + RSQRT_APPROX + U
    d_xh = rs * (dz + d_mu) + xh.abs() * (rs_rel + 3 * U)
    d_y = g.abs() * d_xh + 2 * U * ((xh * g).abs() + b.abs())
    return (y, mu.squeeze(1), rs.squeeze(1)), (d_y, d_mu.squeeze(1), (rs * rs_rel).squeeze(1))


def _ln_inputs(M, N, K, seed):
    """a, w, bias, residual, gamma, beta: rows of the residual carry mean offsets of 0, 3, 10 and
    30 standard deviations of z (cycled over the rows)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = _bf(torch.randn(M, K, device=DEV, generator=g))
    w = _bf(torch.randn(N, K, device=DEV, generator=g) * K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g) * 0.5
    off = torch.tensor([0.0, 3.0, 10.0, 30.0], device=DEV)[torch.arange(M, device=DEV) % 4]
    sign = 1.0 - 2.0 * (torch.arange(M, device=DEV) % 8 >= 4).float()
    residual = _bf(torch.randn(M, N, device=DEV, generator=g) + (off * sign * 1.5)[:, None])
    gamma = 1.0 + 0.2 * torch.randn(N, device=DEV, generator=g)
    beta = 0.1 * torch.randn(N, device=DEV, generator=g)
    return a, w, bias, residual, gamma, beta


LN_CASES = [(4096, 1024, 1024, 0), (4096, 1024, 1024, 128), (4096, 1024, 1024, 256),
            (4096, 1024, 4096, 0), (4096, 1024, 4096, 128), (4096, 1024, 4096, 256),
            (2048, 1024, 4096, 256)]


@pytest.mark.parametrize("M,N,K,block_n", LN_CASES)
def test_gemm_layernorm(nat, M, N, K, block_n):
    """The fused GEMM + LayerNorm with dropout 0.1 and a residual (M = 2048 forced: production
    takes the two-kernel path there), against fp64, and against GEMM + layernorm_fwd on the same
    inputs and masks.  Rows carry mean offsets up to 30 sigma."""
    a, w, bias, residual, gamma, beta = _ln_inputs(M, N, K, seed=M + K + block_n)
    eps, p, stream = 1e-12, 0.1, 77
    rng = nat.RngState(555 + K)
    rng.advance(2)
    kf = _keep(rng, stream, (M, N), p)
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, eps=eps, bias=bias, residual=residual,
                                   dropout_p=p, rng=rng, rng_stream=stream, block_n=block_n)
    bn = block_n or nat.ext().gemm_ln_block_n(M, N, True)
    zr, dz = _z_ref(a, w, bias, residual, kf)
    (yr, mu, rs), (d_y, d_mu, d_rs) = _ln_onepass_ref(zr, dz, gamma, beta, eps,
                                                      depth=bn // 4 + N // bn + 4)
    tag = f"gemm_ln M={M} N={N} K={K} block_n={block_n}"
    worst = _within(f"{tag} z", z, zr, _bf16_out(zr, dz))
    worst = max(worst, _within(f"{tag} mean", mean, mu, d_mu))
    worst = max(worst, _within(f"{tag} rstd", rstd, rs, d_rs))
    worst = max(worst, _within(f"{tag} y", y, yr, _bf16_out(yr, d_y)))
    sig_over_mu = (mu.abs() * rs)
    assert float(sig_over_mu.max()) > 25, "no row with a large mean offset"

    # the two-kernel path of the same layer: GEMM (bias, dropout, residual) -> layernorm_fwd
    z2 = nat.gemm(a, w, bias=bias, aux=residual, add_aux=True, dropout_p=p, rng=rng,
                  rng_stream=stream)
    _within(f"{tag} unfused z", z2, zr, _bf16_out(zr, dz))
    y2, mean2, rstd2 = nat.layernorm_fwd(z2, gamma, beta, eps)
    (y2r, mu2, rs2), (d_y2, d_mu2, d_rs2) = _ln_twopass_ref(z2.to(F64), gamma, beta, eps)
    _within(f"{tag} unfused y", y2, y2r, _bf16_out(y2r, d_y2))
    _within(f"{tag} unfused mean", mean2, mu2, d_mu2)
    _within(f"{tag} unfused rstd", rstd2, rs2, d_rs2)
    # both against each other: within the sum of their bounds and of the distance of their
    # references (bf16 z against fp32 z)
    _within(f"{tag} fused vs unfused y", y, y2.to(F64),
            _bf16_out(yr, d_y) + _bf16_out(y2r, d_y2) + (yr - y2r).abs())
    assert 0 < worst <= 1


def test_gemm_layernorm_constant_row(nat):
    """A row whose z is one constant (zero A row, no bias, constant residual): mean is exact,
    z - mean = 0 and y must be exactly beta, rstd = rsqrt(eps) at most."""
    M, N, K = 4096, 1024, 1024
    a, w, _, residual, gamma, beta = _ln_inputs(M, N, K, seed=9)
    a[5] = 0
    residual[5] = 0.7109375                      # a bf16 value
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, eps=1e-12, residual=residual)
    assert float(mean[5]) == 0.7109375
    assert torch.equal(y[5], _bf(beta)), "y of a constant row is not beta"
    assert float(rstd[5]) <= 1e6 * (1 + 1e-6)


# ---------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------
def _attn_split(t, B, S, heads):
    """[B*S, 3H] -> q, k, v as [B, heads, S, 64] fp64."""
    return t.to(F64).view(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)


def _scores(qkv, mask2, B, S, heads):
    """log2-domain scores s2 = q k^T / 8 * log2e + mask * log2e, and their fp32 error: 64
    tensor-core additions, the scale (fp32 0.125 * log2e, 2 roundings), the masked sum; the
    rounding of a score carries U |mask * log2e| (1e-3 for a -10000 key)."""
    q, k, v = _attn_split(qkv, B, S, heads)
    raw = q @ k.transpose(-1, -2)
    sc = 0.125 * LOG2E
    m2 = (mask2.to(F64) * LOG2E)[:, None, None, :]
    s2 = raw * sc + m2
    ds = 65 * U_TC * (q.abs() @ k.abs().transpose(-1, -2)) * sc + 3 * U * (raw * sc).abs() \
        + U * m2.abs() + U * s2.abs()
    return q, k, v, s2, ds


def _attn_fwd_ref(qkv, mask2, B, S, heads, kf):
    """ctx = (softmax * keep) V and lse (log2) with the kernel's error: e = exp2f(s - max)
    (EX2 + ln2 * the exponent error), their fp32 row sum, e rounded to bf16 for the P V wgmma,
    S tensor-core additions, the 1 / sum scaling; the tiled kernels rescale by exp2f(m_old -
    m_new) once per key tile."""
    q, k, v, s2, ds = _scores(qkv, mask2, B, S, heads)
    lse = torch.logsumexp(s2 * LN2, -1) * LOG2E
    P = torch.exp2(s2 - lse[..., None])
    ds_max = ds.amax(-1, keepdim=True)
    mx = s2.amax(-1, keepdim=True)
    rel_e = 1.01 * LN2 * (ds + ds_max + U * (s2 - mx).abs()) + EX2_APPROX
    tiles = (S + 127) // 128
    rel_sum = rel_e.amax(-1, keepdim=True) * tiles + (S + 2 + 4 * tiles) * U
    d_lse = ds_max.squeeze(-1) + 1.01 * rel_sum.squeeze(-1) * LOG2E + LG2_APPROX \
        + 2 * U * (lse.abs() + mx.squeeze(-1).abs())
    Pk = P * kf
    rel = 1.01 * (BF16 + rel_e.amax(-1, keepdim=True) * (1 + tiles) + rel_sum + DROP + 8 * U) \
        + (S + 1) * U_TC
    ctx = Pk @ v
    d_ctx = rel * (Pk @ v.abs())
    merge = lambda t: t.permute(0, 2, 1, 3).reshape(B * S, heads * 64)  # noqa: E731
    return merge(ctx), merge(d_ctx), lse.reshape(-1), d_lse.reshape(-1)


def _attn_bwd_ref(qkv, mask2, ctx, lse, dctx, B, S, heads, kf):
    """dQ, dK, dV from the kernel's saved lse and bf16 ctx: P = exp2f(s - lse), delta =
    rowsum(dO * ctx) over 64 fp32 products, dP = dO V^T (64 tensor-core additions), dS = P (dP *
    keep - delta) / 8; P * keep and dS rounded to bf16 for their wgmmas (S additions each)."""
    q, k, v, s2, ds = _scores(qkv, mask2, B, S, heads)
    split = lambda t: t.to(F64).view(B, S, heads, 64).permute(0, 2, 1, 3)  # noqa: E731
    do, o = split(dctx), split(ctx)
    lk = lse.to(F64).view(B, heads, S, 1)
    P = torch.exp2(s2 - lk)
    rel_p = 1.01 * LN2 * (ds + U * (s2 - lk).abs()) + EX2_APPROX
    Pk = P * kf
    e_pk = Pk * (1.01 * (rel_p + DROP + U) + BF16)
    dv = Pk.transpose(-1, -2) @ do
    d_dv = e_pk.transpose(-1, -2) @ do.abs() + (S + 1) * U_TC * (Pk.transpose(-1, -2) @ do.abs())
    dP = do @ v.transpose(-1, -2)
    d_dP = 65 * U_TC * (do.abs() @ v.abs().transpose(-1, -2))
    delta = (do * o).sum(-1, keepdim=True)
    d_delta = 66 * U * (do * o).abs().sum(-1, keepdim=True)
    inner = dP * kf - delta
    d_inner = kf * d_dP + (DROP + U) * (dP * kf).abs() + d_delta + U * inner.abs()
    dS = P * inner * 0.125
    e_ds = 1.01 * (P * d_inner * 0.125 + dS.abs() * (rel_p + 2 * U)) + BF16 * dS.abs()
    dq = dS @ k
    d_dq = e_ds @ k.abs() + (S + 1) * U_TC * (dS.abs() @ k.abs())
    dk = dS.transpose(-1, -2) @ q
    d_dk = e_ds.transpose(-1, -2) @ q.abs() + (S + 1) * U_TC * (dS.abs().transpose(-1, -2) @ q.abs())
    cat = lambda *ts: torch.stack(ts, 0).permute(1, 3, 0, 2, 4).reshape(B * S, 3 * heads * 64)  # noqa: E731
    return cat(dq, dk, dv), cat(d_dq, d_dk, d_dv)


def _attn_mask(B, S, seed):
    """Additive [B, S] mask: a different length per sequence, sequence 1 fully padded (every key
    -10000), sequence 0 unpadded."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, S + 1, (B,), generator=g)
    lens[0], lens[1] = S, 0
    keep = torch.arange(S)[None, :] < lens[:, None]
    return ((1.0 - keep.float()) * -10000.0).to(DEV)


def _check_attention_fwd(qkv, mask2, B, S, heads, kf, ctx, lse, tag):
    ref, d_ref, lse_r, d_lse = _attn_fwd_ref(qkv, mask2, B, S, heads, kf)
    worst = _within(f"{tag} ctx", ctx, ref, _bf16_out(ref, d_ref))
    return max(worst, _within(f"{tag} lse", lse, lse_r, d_lse))


def _check_attention_bwd(qkv, mask2, B, S, heads, kf, ctx, lse, dctx, dqkv, tag):
    g, d_g = _attn_bwd_ref(qkv, mask2, ctx, lse, dctx, B, S, heads, kf)
    H = heads * 64
    worst = 0.0
    for i, name in enumerate(("dQ", "dK", "dV")):
        sl = slice(i * H, (i + 1) * H)
        worst = max(worst, _within(f"{tag} {name}", dqkv[:, sl], g[:, sl],
                                   _bf16_out(g[:, sl], d_g[:, sl])))
    return worst


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,S", [(32, 128), (4, 512), (8, 200), (8, 72)])
def test_attention(nat, B, S, p):
    """S = 128 runs the single-tile kernels, 512 / 200 / 72 the tiled ones (ragged last tiles)."""
    heads = 16
    torch.manual_seed(1000 + S + B)
    qkv = _bf(torch.randn(B * S, 3 * heads * 64, device=DEV) * 1.5)
    mask2 = _attn_mask(B, S, seed=S)
    rng = nat.RngState(31 + S)
    rng.advance(4)
    stream, tag = 9, f"attention B={B} S={S} p={p}"
    ctx, lse = nat.attention_fwd(qkv, mask2, B, S, heads, dropout_p=p, rng=rng,
                                 rng_stream=stream)
    kf = _keep(rng, stream, (B, heads, S, S), p)
    worst = _check_attention_fwd(qkv, mask2, B, S, heads, kf, ctx, lse, tag)
    dctx = _bf(torch.randn(B * S, heads * 64, device=DEV))
    dqkv = nat.attention_bwd(qkv, mask2, ctx, lse, dctx, B, S, heads, dropout_p=p, rng=rng,
                             rng_stream=stream)
    worst = max(worst, _check_attention_bwd(qkv, mask2, B, S, heads, kf, ctx, lse, dctx, dqkv,
                                            tag))
    assert 0 < worst <= 1


# ---------------------------------------------------------------------------------------------
# one whole BERT-large layer (Head + Body + Tail as one span) with dropout 0.1
# ---------------------------------------------------------------------------------------------
S_LAYER, H_LAYER, HEADS_LAYER, I_LAYER = 128, 1024, 16, 4096


def _make_span(p=0.1):
    from skycomputing_b200.models import BertConfig
    from skycomputing_b200.models.bert_layers import (BertLayer_Body, BertLayer_Head,
                                                      BertLayer_Tail, BertSpan)

    torch.manual_seed(2024)
    cfg = BertConfig(30522, hidden_size=H_LAYER, num_attention_heads=HEADS_LAYER,
                     intermediate_size=I_LAYER, hidden_dropout_prob=p,
                     attention_probs_dropout_prob=p).__dict__
    head, body, tail = (m(cfg).to(DEV).train() for m in (BertLayer_Head, BertLayer_Body,
                                                        BertLayer_Tail))
    with torch.no_grad():
        for ln in (head.attention.output.LayerNorm, tail.output.LayerNorm):
            ln.weight.add_(0.2 * torch.randn_like(ln.weight))
            ln.bias.add_(0.1 * torch.randn_like(ln.bias))
    return BertSpan(head, body, tail), (head, body, tail)


def _layer_inputs(B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = _bf(torch.randn(B, S_LAYER, H_LAYER, device=DEV, generator=g)).requires_grad_(True)
    mask = _attn_mask(B, S_LAYER, seed=seed).view(B, 1, 1, S_LAYER)
    dy = _bf(torch.randn(B, S_LAYER, H_LAYER, device=DEV, generator=g))
    return x, mask, dy


def _banks(sp):
    return dict(wqkv=sp.wqkv, bqkv=sp.bqkv, wo=sp.wo, bo=sp.bo, g1=sp.g1, b1n=sp.b1n, w1=sp.w1,
                b1=sp.b1, w2=sp.w2, b2=sp.b2, g2=sp.g2, b2n=sp.b2n)


def _run_span(span, x, mask, dy):
    from skycomputing_b200.models import set_backend

    set_backend("native")
    try:
        out, _ = span(x, mask)
        saved = dict(out.grad_fn.saved)
        out.backward(dy)
    finally:
        set_backend("auto")
    return out.detach(), saved


def _ln_stage(tag, nat, fused, a, wbank, bbank, residual, gbank, betabank, kf, z, mean, rstd, y):
    """A dense + dropout + residual + LayerNorm stage of the span against fp64 fed its inputs."""
    w, bias, gamma, beta = wbank.shadow(), bbank.master(), gbank.master(), betabank.master()
    zr, dz = _z_ref(a, w, bias, residual, kf)
    if fused:
        N = w.shape[0]
        bn = nat.ext().gemm_ln_block_n(a.shape[0], N, True)
        (yr, mu, rs), (d_y, d_mu, d_rs) = _ln_onepass_ref(zr, dz, gamma, beta, 1e-12,
                                                          depth=bn // 4 + N // bn + 4)
    else:
        (yr, mu, rs), (d_y, d_mu, d_rs) = _ln_twopass_ref(z.to(F64), gamma, beta, 1e-12)
    w_ = _within(f"{tag} z", z, zr, _bf16_out(zr, dz))
    w_ = max(w_, _within(f"{tag} mean", mean, mu, d_mu))
    w_ = max(w_, _within(f"{tag} rstd", rstd, rs, d_rs))
    return max(w_, _within(f"{tag} y", y, yr, _bf16_out(yr, d_y)))


def _ln_bwd_stage(tag, nat, dy, z, mean, rstd, gbank, p, rng, stream, kf):
    """layernorm_bwd as the span calls it (dgamma / dbeta left to ln_param_grad): dz and the
    dropped dz of the site in front of it; returns both (kernel outputs) and the x-hat used."""
    dz, dzd = nat.layernorm_bwd(dy, z, mean, rstd, gbank.master(), None, None, dropout_p=p,
                                rng=rng, rng_stream=stream)
    rs = rstd.to(F64)[:, None]
    xh = (z.to(F64) - mean.to(F64)[:, None]) * rs
    ref, d_ref = _ln_input_grad_ref(dy.to(F64), torch.zeros_like(xh), xh, 2 * U * xh.abs(),
                                    gbank.master(), rs)
    w_ = _within(f"{tag} dz", dz, ref, _bf16_out(ref, d_ref))
    refd = ref * kf
    w_ = max(w_, _within(f"{tag} dz dropped", dzd, refd,
                         _bf16_out(refd, d_ref * kf + DROP * refd.abs())))
    return dz, dzd, xh, w_


def _gemm_stage(tag, nat, out, **kw):
    ref, acc, pre, d_pre = _gemm_ref(**kw)
    return _within(tag, out, ref, _bf16_out(ref, acc)), (pre, d_pre)


def _check_micro_batch(tag, nat, span, x, mask, dy, sv, y, fused):
    """Every forward stage from the saved intermediates, then the backward chain recomputed with
    the span's kernels, streams and wiring; returns the fp64 parameter-gradient contributions
    {name: (ref, bound, n_adds)} of this micro-batch."""
    sp = span.params
    rng, base, p = sp.rng, sp.rng_base, sp.p_hidden
    B = x.shape[0]
    T, H, heads = B * S_LAYER, H_LAYER, HEADS_LAYER
    xf = x.detach().reshape(T, H)
    mask2 = mask.reshape(B, S_LAYER)
    k_attn = _keep(rng, base + 1, (B, heads, S_LAYER, S_LAYER), sp.p_attn)
    k_o = _keep(rng, base + 2, (T, H), p)
    k_f = _keep(rng, base + 3, (T, H), p)
    assert torch.equal(sv["x"], xf) and torch.equal(sv["mask2"], mask2)

    # ---- forward, stage by stage ----
    worst, _ = _gemm_stage(f"{tag} qkv", nat, sv["qkv"], a=xf, b=sp.wqkv.shadow(),
                           bias=sp.bqkv.master())
    worst = max(worst, _check_attention_fwd(sv["qkv"], mask2, B, S_LAYER, heads, k_attn,
                                            sv["ctxt"], sv["lse"], f"{tag} attention"))
    worst = max(worst, _ln_stage(f"{tag} LN1", nat, fused, sv["ctxt"], sp.wo, sp.bo, xf, sp.g1,
                                 sp.b1n, k_o, sv["z1"], sv["mean1"], sv["rstd1"], sv["a"]))
    w_, (pre, d_pre) = _gemm_stage(f"{tag} ffn1", nat, sv["inter"], a=sv["a"], b=sp.w1.shadow(),
                                   bias=sp.b1.master(), act=ACT_GELU)
    worst = max(worst, w_, _within(f"{tag} ffn1 pre-activation", sv["h1"], pre,
                                   _bf16_out(pre, d_pre)))
    worst = max(worst, _ln_stage(f"{tag} LN2", nat, fused, sv["inter"], sp.w2, sp.b2, sv["a"],
                                 sp.g2, sp.b2n, k_f, sv["z2"], sv["mean2"], sv["rstd2"],
                                 y.reshape(T, H)))

    # ---- backward: the span's chain, recomputed kernel by kernel ----
    dy2 = dy.reshape(T, H)
    dz2, g2, xh2, w_ = _ln_bwd_stage(f"{tag} LN2 bwd", nat, dy2, sv["z2"], sv["mean2"],
                                     sv["rstd2"], sp.g2, p, rng, base + 3, k_f)
    worst = max(worst, w_)
    d_h1 = nat.gemm(g2, sp.w2.shadow(), b_mn=True, aux=sv["h1"], act=ACT_DGELU)
    w_, _ = _gemm_stage(f"{tag} FFN2 dgrad * dgelu", nat, d_h1, a=g2, b=sp.w2.shadow(), b_mn=True,
                        aux=sv["h1"], act=ACT_DGELU)
    worst = max(worst, w_)
    d_a = nat.gemm(d_h1, sp.w1.shadow(), b_mn=True, aux=dz2, add_aux=True)
    w_, _ = _gemm_stage(f"{tag} FFN1 dgrad + dz2", nat, d_a, a=d_h1, b=sp.w1.shadow(), b_mn=True,
                        aux=dz2, add_aux=True)
    worst = max(worst, w_)
    dz1, g1, xh1, w_ = _ln_bwd_stage(f"{tag} LN1 bwd", nat, d_a, sv["z1"], sv["mean1"],
                                     sv["rstd1"], sp.g1, p, rng, base + 2, k_o)
    worst = max(worst, w_)
    dctx = nat.gemm(g1, sp.wo.shadow(), b_mn=True)
    w_, _ = _gemm_stage(f"{tag} attention-output dgrad", nat, dctx, a=g1, b=sp.wo.shadow(),
                        b_mn=True)
    worst = max(worst, w_)
    dqkv = nat.attention_bwd(sv["qkv"], mask2, sv["ctxt"], sv["lse"], dctx, B, S_LAYER, heads,
                             dropout_p=sp.p_attn, rng=rng, rng_stream=base + 1)
    worst = max(worst, _check_attention_bwd(sv["qkv"], mask2, B, S_LAYER, heads, k_attn,
                                            sv["ctxt"], sv["lse"], dctx, dqkv,
                                            f"{tag} attention"))
    dx = x.grad.reshape(T, H)
    w_, _ = _gemm_stage(f"{tag} dx (QKV dgrad + dz1)", nat, dx, a=dqkv, b=sp.wqkv.shadow(),
                        b_mn=True, aux=dz1, add_aux=True)
    worst = max(worst, w_)
    # the span computed exactly this chain: its dx is the recomputed one, bit for bit
    dx_re = nat.gemm(dqkv, sp.wqkv.shadow(), b_mn=True, aux=dz1, add_aux=True)
    assert torch.equal(dx_re.view(torch.int16), dx.view(torch.int16)), f"{tag}: dx differs"

    # ---- parameter-gradient contributions: fp64 terms over the T tokens ----
    def wg(g, act):
        v, dv, _, _ = _gemm_ref(g, act, a_mn=True, b_mn=True)
        return v, dv, _acc_err(T)

    def cs(t, err=None):                   # column sums (ln_param_grad / colsum)
        t = t.to(F64)
        e = torch.zeros(t.shape[1], dtype=F64, device=DEV) if err is None else err.sum(0)
        n = _reduce_depth(T) * U
        return t.sum(0), n * t.abs().sum(0) + e, n

    d1, d2 = d_a.to(F64), dy2.to(F64)
    contrib = dict(
        wqkv=wg(dqkv, xf), bqkv=cs(dqkv), wo=wg(g1, sv["ctxt"]), bo=cs(g1),
        g1=cs(d1 * xh1, 3 * U * (d1 * xh1).abs()), b1n=cs(d1),
        w1=wg(d_h1, sv["a"]), b1=cs(d_h1), w2=wg(g2, sv["inter"]), b2=cs(g2),
        g2=cs(d2 * xh2, 3 * U * (d2 * xh2).abs()), b2n=cs(d2))
    return contrib, worst


def _check_param_grads(tag, sp, totals):
    worst = 0.0
    for name, bank in _banks(sp).items():
        ref, bound = totals[name]
        worst = max(worst, _within(f"{tag} grad {name}", bank.grad(), ref, bound))
    return worst


@pytest.mark.parametrize("B", [32, 16])
def test_layer_stage_by_stage_two_micro_batches(nat, B, monkeypatch):
    """BertSpan(head, body, tail) at the benchmark's geometry with dropout 0.1 in training mode:
    B = 32 takes the fused GEMM + LayerNorm, B = 16 GEMM + standalone LayerNorm.  Two
    micro-batches (the dropout step advanced between them): every stage of each is checked
    against fp64 fed the previous stage's saved values, and the weight gradients accumulate to
    the sum of both micro-batches' references."""
    from skycomputing_b200.models import advance_rng
    from skycomputing_b200.ops import functions

    gemm_ln = nat.gemm_ln
    monkeypatch.delenv("SKY_FUSE_LN", raising=False)
    T = B * S_LAYER
    fused = nat.gemm_ln_supported(T, H_LAYER)
    assert fused == (B == 32), "unexpected LayerNorm path for this batch size"
    span, _ = _make_span()
    sp = span.params
    totals = {}
    worst = 0.0
    masks = []
    for mb in range(2):
        if mb:
            advance_rng()
        x, mask, dy = _layer_inputs(B, seed=300 + 10 * B + mb)
        calls = []
        monkeypatch.setattr(functions.nat, "gemm_ln",
                            lambda *a, **k: calls.append(1) or gemm_ln(*a, **k))
        y, sv = _run_span(span, x, mask, dy)
        monkeypatch.setattr(functions.nat, "gemm_ln", gemm_ln)
        assert len(calls) == (2 if fused else 0), "the span took the other LayerNorm path"
        masks.append(_keep(sp.rng, sp.rng_base + 3, (T, H_LAYER), sp.p_hidden))
        tag = f"layer B={B} mb={mb}"
        contrib, w_ = _check_micro_batch(tag, nat, span, x, mask, dy, sv, y, fused)
        worst = max(worst, w_)
        for name, (ref, bound, per_add) in contrib.items():
            if name in totals:
                # accumulated onto the previous micro-batch's sum: every addition is also off by
                # up to one rounding of that sum
                r0, b0 = totals[name]
                totals[name] = (r0 + ref, b0 + bound + per_add * r0.abs())
            else:
                totals[name] = (ref, bound)
        worst = max(worst, _check_param_grads(tag, sp, totals))
    assert not torch.equal(masks[0], masks[1]), "advance_rng() did not change the dropout masks"
    assert 0 < worst <= 1


def _normwise(got, ref):
    return float((got.to(F64) - ref).norm() / ref.norm())


def test_layer_end_to_end_fused_and_unfused(nat, monkeypatch):
    """The whole layer at B = 32 against an fp64 autograd reference that starts from the same bf16
    input and weights and applies the same keep masks: normwise relative errors of the output, dx
    and every parameter gradient, for the fused LayerNorm path and SKY_FUSE_LN=0."""
    B = 32
    T = B * S_LAYER
    span, (head, body, tail) = _make_span()
    sp = span.params
    x, mask, dy = _layer_inputs(B, seed=77)
    runs = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("SKY_FUSE_LN", mode)
        assert nat.gemm_ln_supported(T, H_LAYER) == (mode == "1")
        for bank in sp.banks:
            bank.grad().zero_()
        x.grad = None
        y, _ = _run_span(span, x, mask, dy)
        got = {"out": y, "dx": x.grad.detach()}
        got.update({n: b.grad().clone() for n, b in _banks(sp).items()})
        runs[mode] = got
    # the reference: bf16 compute copies of the weights, fp32 biases / LayerNorm parameters
    weights = dict(wqkv=sp.wqkv.shadow(), wo=sp.wo.shadow(), w1=sp.w1.shadow(),
                   w2=sp.w2.shadow())
    prm = layer_params(head, body, tail, weights=weights)
    k_attn = _keep(sp.rng, sp.rng_base + 1, (B, HEADS_LAYER, S_LAYER, S_LAYER), sp.p_attn)
    k_o = _keep(sp.rng, sp.rng_base + 2, (T, H_LAYER), sp.p_hidden)
    k_f = _keep(sp.rng, sp.rng_base + 3, (T, H_LAYER), sp.p_hidden)
    xr = x.detach().to(F64).requires_grad_(True)
    yr, _ = layer_ref(xr, mask.reshape(B, S_LAYER).to(F64), prm, HEADS_LAYER, k_attn, k_o, k_f)
    gr = torch.autograd.grad(yr, [xr] + [prm[n] for n in PARAM_NAMES], dy.to(F64))
    ref = {"out": yr.detach(), "dx": gr[0]}
    ref.update({n: g.reshape(_banks(sp)[n].grad().shape) for n, g in zip(PARAM_NAMES, gr[1:])})
    print()
    for key in ref:
        e1, e0 = _normwise(runs["1"][key], ref[key]), _normwise(runs["0"][key], ref[key])
        print(f"[e2e] {key}: normwise relative error fused {e1:.3e}, unfused {e0:.3e}")
        assert e1 < 2e-2 and e0 < 2e-2, (key, e1, e0)
        assert e1 <= 1.25 * e0, f"{key}: the fused path is {e1 / e0:.2f}x the unfused error"
