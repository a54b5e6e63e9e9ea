"""The kernels at both ends of a training step against fp64 references of the same operation:
the embedding gather + LayerNorm + dropout and its scatter backward, the pooler on the wgmma GEMM
and on the small-linear kernels, the classifier, softmax cross entropy, the LayerNorm parameter
gradients, the standalone LayerNorm, ``dgelu_mul`` and the bf16 casts.

Every reference is computed in fp64 from exactly the values the kernel received (bf16 inputs
upcast, fp32 tables and saved statistics as they are), and every element is checked against a
bound of its own: the output rounding plus a worst-case accumulation term n * u * sum|terms|,
with sum|terms| computed by the same fp64 reference over absolute values.  Worst-case bounds
cannot flake on atomic ordering, and a wrong index, mask or scale gives an O(1) error.
"""
import math

import numpy as np
import pytest
import torch

from tests._fp64_bounds import (BF16, DEV, DROP, EXPF_ULPS, F64, RSQRT_APPROX, U, U_TC, _bf16_out,
                                _colsum_ref, _keep, _ln_fwd_ref, _ln_input_grad_ref, _within)

pytestmark = pytest.mark.gpu

TANH_APPROX = 2.0 ** -10.98   # PTX ISA: tanh.approx.f32 (MUFU.TANH) max relative error 2^-10.987


@pytest.fixture(scope="module")
def nat():
    from skycomputing_b200.ops import native

    assert native.available(), "native extension must be built and a GPU present"
    return native


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------
# embeddings
# ---------------------------------------------------------------------------------------------
def _embed_fwd_call(nat, ids, tts, am, word, pos, typ, gamma, beta, B, S, eps, p, rng, stream):
    """The kernel call of ``EmbeddingsFn.forward`` (same keyword arguments)."""
    H = word.shape[1]
    out = torch.empty((B * S, H), dtype=torch.bfloat16, device=DEV)
    ext_mask = torch.empty(B * S, dtype=torch.float32, device=DEV)
    mean = torch.empty(B * S, dtype=torch.float32, device=DEV)
    rstd = torch.empty(B * S, dtype=torch.float32, device=DEV)
    nat.ext().embed_fwd(ids=ids.data_ptr(), tts=tts.data_ptr(), amask=am.data_ptr(),
                        word=word.data_ptr(), pos=pos.data_ptr(), type=typ.data_ptr(),
                        gamma=gamma.data_ptr(), beta=beta.data_ptr(), out=out.data_ptr(),
                        ext_mask=ext_mask.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                        B=B, S=S, H=H, eps=eps, dropout_p=p,
                        rng_state=0 if rng is None else rng.ptr, rng_stream=stream,
                        stream=_stream())
    return out, ext_mask, mean, rstd


def _embed_rows(ids, tts, S, word, pos, typ):
    BS = ids.numel()
    s = torch.arange(BS, device=DEV) % S
    a, b, d = word.to(F64)[ids], pos.to(F64)[s], typ.to(F64)[tts]
    e_abs = a.abs() + b.abs() + d.abs()
    return a + b + d, 2 * U * e_abs, e_abs, s      # e = a + b + d: two fp32 additions


def _check_embed_fwd(tag, out, ext_mask, mean, rstd, ids, tts, am, S, word, pos, typ, gamma,
                     beta, eps, kf):
    e, e_err, e_abs, _ = _embed_rows(ids, tts, S, word, pos, typ)
    (y, mu, rs, _), (d_y, d_mu, d_rs) = _ln_fwd_ref(e, e_err, e_abs, gamma, beta, eps)
    y = y * kf
    d_y = d_y * kf + DROP * y.abs()
    worst = _within(f"{tag} out", out, y, _bf16_out(y, d_y))
    _within(f"{tag} mean", mean, mu, d_mu)
    _within(f"{tag} rstd", rstd, rs, d_rs)
    ext_ref = (1.0 - am.float()) * -10000.0
    assert torch.equal(ext_mask, ext_ref), f"{tag}: ext_mask differs"
    return worst


def _check_embed_bwd(tag, grads, inits, dout, ids, tts, S, word, pos, typ, gamma, mean, rstd,
                     kf):
    """grads / inits: (dword, dpos, dtype, dgamma, dbeta) after / before the backward."""
    BS, H = dout.shape
    e, e_err, _, s = _embed_rows(ids, tts, S, word, pos, typ)
    mu, rs = mean.to(F64)[:, None], rstd.to(F64)[:, None]   # the statistics the kernel was given
    xh = (e - mu) * rs
    xh_err = rs * e_err + 2 * U * xh.abs()
    dy = dout.to(F64) * kf
    dy_err = DROP * dy.abs()
    de, d_de = _ln_input_grad_ref(dy, dy_err, xh, xh_err, gamma, rs)
    # shared-memory partials are flushed once per CTA of 8 warps: at most BS / 8 more additions
    ctas = (BS + 7) // 8 + 1
    worst = 0.0
    for name, got, init, index, smem in (("dword", grads[0], inits[0], ids, False),
                                         ("dpos", grads[1], inits[1], s, False),
                                         ("dtype", grads[2], inits[2], tts, True)):
        init = init.to(F64)
        cnt = torch.bincount(index, minlength=init.shape[0]).to(F64)[:, None]
        ref = init.index_add(0, index, de)
        absum = init.abs().index_add(0, index, de.abs())
        err = torch.zeros_like(init).index_add(0, index, d_de)
        bound = (cnt + (ctas if smem else 1)) * U * absum + err
        worst = max(worst, _within(f"{tag} {name}", got, ref, bound))
    worst = max(worst, _colsum_ref(f"{tag} dgamma", grads[3], inits[3], dy * xh,
                                   dy.abs() * xh_err + dy_err * xh.abs() + U * (dy * xh).abs(),
                                   BS + ctas))
    worst = max(worst, _colsum_ref(f"{tag} dbeta", grads[4], inits[4], dy, dy_err, BS + ctas))
    return worst


# (B, S, H, vocabulary ids, token-type rows, p): every value of each axis meets every value of
# the others at least once; H = 4096 takes the t_smem = 0 fallback of embed_bwd, token types >= 4
# go to global atomics, "collide" draws every id from 3 values so the dword atomics collide
EMBED_CASES = [
    (32, 128, 1024, "uniform", 2, 0.1),
    (32, 128, 1024, "collide", 6, 0.1),
    (32, 128, 256, "uniform", 6, 0.0),
    (32, 128, 256, "collide", 2, 0.1),
    (32, 128, 4096, "uniform", 2, 0.1),
    (32, 128, 4096, "collide", 6, 0.0),
    (3, 37, 256, "uniform", 2, 0.0),
    (3, 37, 1024, "collide", 2, 0.0),
    (3, 37, 1024, "uniform", 6, 0.1),
    (3, 37, 4096, "uniform", 6, 0.1),
    (3, 37, 4096, "collide", 2, 0.1),
    (3, 37, 256, "collide", 6, 0.1),
]


def _embed_inputs(B, S, H, ids_kind, type_rows, V=30522, P=512):
    ids = (torch.randint(0, V, (B, S), device=DEV) if ids_kind == "uniform" else
           torch.tensor([0, 1234, V - 1], device=DEV)[torch.randint(0, 3, (B, S), device=DEV)])
    tts = torch.randint(0, type_rows, (B, S), device=DEV)
    am = torch.ones(B, S, dtype=torch.int64, device=DEV)
    for b in range(B):                       # padded tails of random length, one row unpadded
        if b % 3:
            am[b, int(torch.randint(1, S, ())):] = 0
    word = torch.randn(V, H, device=DEV)
    pos = torch.randn(P, H, device=DEV) * 0.5
    typ = torch.randn(type_rows, H, device=DEV) * 0.3 + 0.2
    gamma = 1.0 + 0.2 * torch.randn(H, device=DEV)
    beta = 0.1 * torch.randn(H, device=DEV)
    return ids, tts, am, (word, pos, typ, gamma, beta)


@pytest.mark.parametrize("B,S,H,ids_kind,type_rows,p", EMBED_CASES)
def test_embedding_forward_backward(nat, B, S, H, ids_kind, type_rows, p):
    torch.manual_seed(100 + H + B + type_rows)
    ids, tts, am, (word, pos, typ, gamma, beta) = _embed_inputs(B, S, H, ids_kind, type_rows)
    ids, tts, am = ids.reshape(-1), tts.reshape(-1), am.reshape(-1)
    eps, stream = 1e-12, 24
    rng = nat.RngState(4321 + H)
    rng.advance(3)
    out, ext_mask, mean, rstd = _embed_fwd_call(nat, ids, tts, am, word, pos, typ, gamma, beta,
                                                B, S, eps, p, rng, stream)
    kf = _keep(rng, stream, (B * S, H), p)
    tag = f"embed B={B} S={S} H={H} {ids_kind} T={type_rows} p={p}"
    w_fwd = _check_embed_fwd(tag, out, ext_mask, mean, rstd, ids, tts, am, S, word, pos, typ,
                             gamma, beta, eps, kf)

    dout = torch.randn(B * S, H, device=DEV).to(torch.bfloat16)
    # the gradients accumulate (+=): start them from nonzero values
    inits = [torch.randn_like(t) * 0.5 for t in (word, pos, typ, gamma, beta)]
    grads = [t.clone() for t in inits]
    nat.ext().embed_bwd(dout=dout.data_ptr(), ids=ids.data_ptr(), tts=tts.data_ptr(),
                        word=word.data_ptr(), pos=pos.data_ptr(), type=typ.data_ptr(),
                        gamma=gamma.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                        dword=grads[0].data_ptr(), dpos=grads[1].data_ptr(),
                        dtype=grads[2].data_ptr(), dgamma=grads[3].data_ptr(),
                        dbeta=grads[4].data_ptr(), B=B, S=S, H=H, type_rows=type_rows,
                        dropout_p=p, rng_state=rng.ptr, rng_stream=stream, stream=_stream())
    w_bwd = _check_embed_bwd(tag, grads, inits, dout, ids, tts, S, word, pos, typ, gamma, mean,
                             rstd, kf)
    assert w_fwd > 0 and w_bwd > 0


def test_embedding_index_dtypes_match_int64(nat):
    """int32 ids / token types with a bool or int32 attention mask give the int64 run's bits."""
    from skycomputing_b200.models import BertConfig, set_backend
    from skycomputing_b200.models.bert_layers import BertEmbeddings

    torch.manual_seed(5)
    B, S, H = 4, 128, 256
    emb = BertEmbeddings(BertConfig(30522, hidden_size=H).__dict__).to(DEV).eval()
    ids, tts, am, _ = _embed_inputs(B, S, H, "uniform", 2)
    set_backend("native")
    try:
        with torch.no_grad():
            ref, ref_mask = emb(ids, tts, am)
            for i_dt, m_dt in ((torch.int32, torch.bool), (torch.int32, torch.int32),
                               (torch.int64, torch.bool)):
                out, ext = emb(ids.to(i_dt), tts.to(i_dt), am.to(m_dt))
                assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (i_dt, m_dt)
                assert torch.equal(ext, ref_mask), (i_dt, m_dt)
    finally:
        set_backend("auto")


# ---------------------------------------------------------------------------------------------
# pooler on the wgmma GEMM
# ---------------------------------------------------------------------------------------------
def _pooler_fwd_ref(x0, w, b):
    """tanh(x0 w^T + b) from bf16 x0 / w and fp32 b: K tensor-core additions and the bias add,
    then tanh.approx (relative error 2^-10.987 of its result; tanh is 1-Lipschitz)."""
    K = x0.shape[1]
    x0, w, b = x0.to(F64), w.to(F64), b.to(F64)
    pre = x0 @ w.t() + b
    d_pre = (K + 2) * U_TC * (x0.abs() @ w.abs().t() + b.abs())
    y = torch.tanh(pre)
    return y, TANH_APPROX * (y.abs() + d_pre) + d_pre


def _check_pooler_bwd(tag, dy, y, x0, w_bf16, dw, dw0, db, db0, dx0):
    """PoolerFn.backward: g = dy (1 - y^2) in torch fp32 (3 roundings), rounded to bf16 for the
    GEMMs; db += sum_b g (torch), dW += gb^T x0 (tensor cores, K = B), dx0 = gb W as bf16."""
    B, H = x0.shape
    g = dy.to(F64) * (1 - y.to(F64) ** 2)
    gb = (dy.float() * (1.0 - y * y)).to(torch.bfloat16)   # exactly what the GEMMs received
    worst = _colsum_ref(f"{tag} db", db, db0, g, 3 * U * g.abs(), B + 1)
    gb, x0, w = gb.to(F64), x0.to(F64), w_bf16.to(F64)
    worst = max(worst, _within(f"{tag} dW", dw, dw0.to(F64) + gb.t() @ x0,
                               (B + 1) * U_TC * (dw0.to(F64).abs() + gb.abs().t() @ x0.abs())))
    ref = gb @ w
    worst = max(worst, _within(f"{tag} dx", dx0, ref,
                               _bf16_out(ref, (H + 1) * U_TC * (gb.abs() @ w.abs()))))
    return worst


@pytest.mark.parametrize("B", [8, 16, 32])
def test_pooler_on_gemm(nat, B):
    """PoolerFn (taken whenever B % 8 == 0): ACT_TANH with fp32 out on an A view of row stride
    S*H, the wgrad with K = B < one k-block into a nonzero fp32 buffer, the dgrad into strided
    bf16 rows; the other S - 1 token positions stay untouched."""
    from skycomputing_b200.ops.functions import PoolerFn, SmallLinearParams

    torch.manual_seed(200 + B)
    S, H = 128, 1024
    w = torch.nn.Parameter(torch.randn(H, H, device=DEV) * 0.03)
    bias = torch.nn.Parameter(torch.randn(H, device=DEV) * 0.5)
    lp = SmallLinearParams(w, bias, act_tanh=True, first_token=True)
    dw0 = torch.randn(H, H, device=DEV)
    db0 = torch.randn(H, device=DEV)
    lp.w.grad().copy_(dw0)
    lp.b.grad().copy_(db0)
    hidden = torch.randn(B, S, H, device=DEV).to(torch.bfloat16).requires_grad_(True)
    y = PoolerFn.apply(lp, hidden, *lp.all_params())
    tag = f"pooler gemm B={B}"
    ref, bound = _pooler_fwd_ref(hidden[:, 0].detach(), lp.w.shadow(), bias.detach())
    worst = _within(f"{tag} y", y, ref, bound)
    dy = torch.randn(B, H, device=DEV)
    y.backward(dy)
    dh = hidden.grad
    assert torch.count_nonzero(dh[:, 1:]) == 0, "dgrad wrote outside the first-token rows"
    worst = max(worst, _check_pooler_bwd(tag, dy, y.detach(), hidden[:, 0].detach(),
                                         lp.w.shadow(), lp.w.grad(), dw0, lp.b.grad(), db0,
                                         dh[:, 0]))
    # the dgrad alone into a strided view of a sentinel-filled buffer
    gb = (dy * (1.0 - y.detach() * y.detach())).to(torch.bfloat16)
    buf = torch.full((B, S, H), 3.0, dtype=torch.bfloat16, device=DEV)
    nat.gemm(gb, lp.w.shadow(), b_mn=True, out=buf.view(B, S * H)[:, :H])
    assert torch.equal(buf[:, 1:], torch.full_like(buf[:, 1:], 3.0)), "sentinel overwritten"
    ref = gb.to(F64) @ lp.w.shadow().to(F64)
    _within(f"{tag} dgrad into a strided view", buf[:, 0], ref,
            _bf16_out(ref, (H + 1) * U_TC * (gb.to(F64).abs() @ lp.w.shadow().to(F64).abs())))
    assert 0 < worst <= 1


# ---------------------------------------------------------------------------------------------
# small_linear_fwd / small_linear_bwd: the classifier and the pooler fallback
# ---------------------------------------------------------------------------------------------
def _small_linear_ref(x, kf, w, b, tanh):
    """y = act((x * keep) w^T + b): K fp32 additions, the input scaling (DROP), the products and
    the bias add."""
    K = x.shape[1]
    xk = x.to(F64) * kf
    w = w.to(F64)
    pre = xk @ w.t() + b.to(F64)
    d_pre = (K + 2 + DROP / U) * U * (xk.abs() @ w.abs().t() + b.to(F64).abs())
    if not tanh:
        return pre, d_pre, xk
    y = torch.tanh(pre)
    return y, TANH_APPROX * (y.abs() + d_pre) + d_pre, xk


def _check_small_linear_bwd(tag, dy, y, xk, kf, w, tanh, dx, dx_bf16, dw, dw0, db, db0):
    M, N = dy.shape
    dy, y, w = dy.to(F64), y.to(F64), w.to(F64)
    g = dy * (1 - y * y) if tanh else dy           # y: the kernel's output, as backward reads it
    dg = 3 * U * dy.abs() * (1 + y * y) if tanh else torch.zeros_like(g)
    ref = (g @ w) * kf
    acc = ((N + 1) * U * (g.abs() @ w.abs()) + dg @ w.abs()) * kf + DROP * ref.abs()
    worst = _within(f"{tag} dx", dx, ref, _bf16_out(ref, acc) if dx_bf16 else acc)
    worst = max(worst, _within(f"{tag} dw", dw, dw0.to(F64) + g.t() @ xk,
                               (M + 2 + DROP / U) * U * (dw0.to(F64).abs() + g.abs().t() @ xk.abs())
                               + dg.t() @ xk.abs()))
    worst = max(worst, _colsum_ref(f"{tag} db", db, db0, g, dg, M + 1))
    return worst


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("M", [8, 32, 37])
def test_small_linear_classifier(nat, M, p):
    """The classifier: fp32 input with input dropout (site index m * K + k), N = 3, fp32 dx."""
    torch.manual_seed(300 + M)
    N, K, stream = 3, 1024, 16
    rng = nat.RngState(99 + M)
    x = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) * 0.03
    b = torch.randn(N, device=DEV)
    y = torch.empty(M, N, device=DEV)
    nat.ext().small_linear_fwd(x=x.data_ptr(), x_bf16=False, ldx=K, w=w.data_ptr(),
                               b=b.data_ptr(), y=y.data_ptr(), M=M, N=N, K=K, act_tanh=0,
                               dropout_p=p, rng_state=rng.ptr, rng_stream=stream, stream=_stream())
    kf = _keep(rng, stream, (M, K), p)
    tag = f"classifier M={M} p={p}"
    ref, bound, xk = _small_linear_ref(x, kf, w, b, False)
    _within(f"{tag} y", y, ref, bound)
    dy = torch.randn(M, N, device=DEV)
    dx = torch.empty(M, K, device=DEV)
    dw0, db0 = torch.randn(N, K, device=DEV), torch.randn(N, device=DEV)
    dw, db = dw0.clone(), db0.clone()
    nat.ext().small_linear_bwd(x=x.data_ptr(), x_bf16=False, ldx=K, w=w.data_ptr(),
                               y=y.data_ptr(), dy=dy.data_ptr(), dx=dx.data_ptr(), dx_bf16=False,
                               lddx=K, dw=dw.data_ptr(), db=db.data_ptr(), M=M, N=N, K=K,
                               act_tanh=0, dropout_p=p, rng_state=rng.ptr, rng_stream=stream,
                               stream=_stream())
    _check_small_linear_bwd(tag, dy, y, xk, kf, w, False, dx, False, dw, dw0, db, db0)


@pytest.mark.parametrize("B", [4, 37])
def test_small_linear_pooler_fallback(nat, B):
    """The pooler when B % 8 != 0: bf16 first-token rows (ldx = S*H), tanh, bf16 dx written into
    the first-token rows of a zero-filled [B, S, H] buffer (lddx = S*H)."""
    torch.manual_seed(400 + B)
    S, H = 128, 1024
    hidden = torch.randn(B, S, H, device=DEV).to(torch.bfloat16)
    w = torch.randn(H, H, device=DEV) * 0.03
    b = torch.randn(H, device=DEV) * 0.5
    y = torch.empty(B, H, device=DEV)
    nat.ext().small_linear_fwd(x=hidden.data_ptr(), x_bf16=True, ldx=S * H, w=w.data_ptr(),
                               b=b.data_ptr(), y=y.data_ptr(), M=B, N=H, K=H, act_tanh=1,
                               dropout_p=0.0, rng_state=0, rng_stream=0, stream=_stream())
    tag = f"pooler fallback B={B}"
    kf = torch.ones(B, H, dtype=F64, device=DEV)
    ref, bound, xk = _small_linear_ref(hidden[:, 0], kf, w, b, True)
    _within(f"{tag} y", y, ref, bound)
    dy = torch.randn(B, H, device=DEV)
    dx = torch.zeros_like(hidden)
    dw0, db0 = torch.randn(H, H, device=DEV), torch.randn(H, device=DEV)
    dw, db = dw0.clone(), db0.clone()
    nat.ext().small_linear_bwd(x=hidden.data_ptr(), x_bf16=True, ldx=S * H, w=w.data_ptr(),
                               y=y.data_ptr(), dy=dy.data_ptr(), dx=dx.data_ptr(), dx_bf16=True,
                               lddx=S * H, dw=dw.data_ptr(), db=db.data_ptr(), M=B, N=H, K=H,
                               act_tanh=1, dropout_p=0.0, rng_state=0, rng_stream=0,
                               stream=_stream())
    assert torch.count_nonzero(dx[:, 1:]) == 0, "dx written outside the first-token rows"
    _check_small_linear_bwd(tag, dy, y, xk, kf, w, True, dx[:, 0], True, dw, dw0, db, db0)


# ---------------------------------------------------------------------------------------------
# softmax cross entropy
# ---------------------------------------------------------------------------------------------
def _softmax_ce_ref(logits, labels, gs, acc0=None, calls=1):
    """Mean cross entropy and (softmax - onehot) * gs / M in fp64, with worst-case errors of the
    kernel's fp32 row max / __expf / __logf / exp-sum and its fp64 sum of the rows (fast-math
    intrinsics: __expf is off by 2 + |1.173 x| ulp, __logf by 2^-21.41 absolute on [0.5, 2] and
    3 ulp elsewhere)."""
    M, C = logits.shape
    lf = logits.to(F64)
    lab = labels[:, None]
    mx = lf.amax(1, keepdim=True)
    se = torch.exp(lf - mx).sum(1, keepdim=True)
    lse = mx + torch.log(se)
    row = lse.squeeze(1) - lf.gather(1, lab).squeeze(1)
    ulp = 2.0 ** -23
    exp_rel = (2 + EXPF_ULPS * (lf - mx).abs()) * ulp + U * ((lf - mx).abs() + 1)
    se_rel = exp_rel.amax(1, keepdim=True) + (C + 1) * U
    log_err = torch.where(se <= 2, torch.full_like(se, 2.0 ** -21.41), 3 * ulp * torch.log(se))
    d_lse = 1.01 * se_rel + log_err + U * lse.abs()
    d_row = d_lse.squeeze(1) + U * (lse.squeeze(1).abs() + lf.gather(1, lab).squeeze(1).abs())
    mean = row.mean()
    # each fp32 row CE / M in fp64 (1 rounding), a fp64 sum of M terms (at most M - 1 roundings
    # on any term), then one rounding to fp32
    d_mean = ((M + 1) * 2.0 ** -53 * row.abs().sum() + d_row.sum()) / M + 2 * U * mean.abs()
    onehot = torch.zeros_like(lf).scatter_(1, lab, 1.0)
    p = torch.exp(lf - lse)
    d = (p - onehot) * gs / M
    p_err = p * ((3 + EXPF_ULPS * (lf - lse).abs()) * ulp + 1.01 * d_lse + U * (lf - lse).abs())
    # p - onehot, times grad_scale / M (fast-math division: 2 ulp)
    d_err = (p_err + 6 * U * (p - onehot).abs()) * gs / M
    out = dict(loss=mean, d_loss=d_mean, dlogits=d, d_dlogits=d_err)
    if acc0 is not None:
        a = float(acc0)
        out["acc"] = a + calls * mean * gs
        out["d_acc"] = calls * (gs * d_mean + 2 * U * (abs(a) + calls * (mean * gs).abs()))
    return out


@pytest.mark.parametrize("with_acc", [False, True])
@pytest.mark.parametrize("gs", [1.0, 1.0 / 7])
@pytest.mark.parametrize("C", [2, 3, 17])
@pytest.mark.parametrize("M", [1, 32, 300, 1000])
def test_softmax_ce(nat, M, C, gs, with_acc):
    """What the engine's fused loss uses (grad_scale = 1/m, loss_acc), and M > 256, where the
    kernel sums several 256-row chunks."""
    torch.manual_seed(500 + M + C)
    logits = torch.randn(M, C, device=DEV) * 3
    labels = torch.randint(0, C, (M,), device=DEV)
    acc0 = 0.25
    acc = torch.full((1,), acc0, device=DEV) if with_acc else None
    for _ in range(2):                     # twice: loss_acc accumulates
        loss, dl = nat.softmax_ce(logits, labels, grad_scale=gs, loss_acc=acc)
    gs32 = float(np.float32(gs))           # the fp32 scale the kernel received
    r = _softmax_ce_ref(logits, labels, gs32, acc0 if with_acc else None, calls=2)
    tag = f"softmax_ce M={M} C={C} gs={gs:.3g}"
    _within(f"{tag} loss", loss[0], r["loss"], r["d_loss"])
    _within(f"{tag} dlogits", dl, r["dlogits"], r["d_dlogits"])
    if with_acc:
        _within(f"{tag} loss_acc", acc[0], r["acc"], r["d_acc"])


def test_softmax_ce_rejects_bad_labels(nat):
    logits = torch.randn(8, 3, device=DEV)
    for bad in (torch.randint(0, 3, (8,), device=DEV, dtype=torch.int32),
                torch.randint(0, 3, (7,), device=DEV),
                torch.randint(0, 3, (8,))):
        with pytest.raises(ValueError, match="labels"):
            nat.softmax_ce(logits, bad)


def test_native_cross_entropy_ignores_minus_100(nat):
    """The native CrossEntropyLoss leaves rows labelled -100 out of the mean, as
    nn.CrossEntropyLoss() does; with every row ignored it gives 0 and a zero gradient."""
    from skycomputing_b200.runner import build_loss

    fn = build_loss(dict(type="CrossEntropyLoss"), torch.device(DEV))
    assert type(fn) is not torch.nn.CrossEntropyLoss
    torch.manual_seed(510)
    logits = (torch.randn(64, 3, device=DEV) * 3).requires_grad_(True)
    labels = torch.randint(0, 3, (64,), device=DEV)
    labels[::3] = -100
    loss = fn(logits, labels)
    loss.backward()
    x = logits.detach().to(F64).requires_grad_(True)
    want = torch.nn.CrossEntropyLoss()(x, labels)
    want.backward()
    assert float(loss.detach()) == pytest.approx(float(want.detach()), rel=1e-6)
    assert torch.allclose(logits.grad.to(F64), x.grad, rtol=1e-5, atol=1e-7)
    assert torch.count_nonzero(logits.grad[::3]) == 0
    logits.grad = None
    loss = fn(logits, torch.full_like(labels, -100))
    loss.backward()
    assert float(loss.detach()) == 0.0 and torch.count_nonzero(logits.grad) == 0


# ---------------------------------------------------------------------------------------------
# LayerNorm parameter gradients, standalone LayerNorm
# ---------------------------------------------------------------------------------------------
def _check_ln_param_grads(tag, dy, z, mean, rstd, dg, dg0, db, db0, x2=None, o2=None, o20=None):
    """Every column is summed over M rows by one thread (strided by 8 x grid.y <= 64 blocks), then
    8 shared-memory partials and <= 64 global atomics: at most M + 72 additions."""
    M = z.shape[0]
    n = M + 72
    dy = dy.to(F64)
    xh = (z.to(F64) - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
    t = dy * xh
    worst = _colsum_ref(f"{tag} dgamma", dg, dg0, t, 3 * U * t.abs(), n)
    worst = max(worst, _colsum_ref(f"{tag} dbeta", db, db0, dy, torch.zeros_like(dy), n))
    if x2 is not None:
        x2 = x2.to(F64)
        worst = max(worst, _colsum_ref(f"{tag} out2", o2, o20, x2, torch.zeros_like(x2), n))
    return worst


@pytest.mark.parametrize("with_x2", [False, True])
@pytest.mark.parametrize("H", [768, 1024])
@pytest.mark.parametrize("M", [384, 4096, 4100])
def test_ln_param_grad(nat, M, H, with_x2):
    """The kernel every encoder layer's backward runs (functions._ln_pgrad), with the dense
    layer's bias gradient fused in; M = 4096 saturates grid.y at 64."""
    torch.manual_seed(600 + M + H)
    z = (torch.randn(M, H, device=DEV) * 2 + 0.5).to(torch.bfloat16)
    dy = torch.randn(M, H, device=DEV).to(torch.bfloat16)
    zf = z.float()
    mean = zf.mean(1)
    rstd = torch.rsqrt(zf.var(1, unbiased=False) + 1e-12)
    dg0, db0 = torch.randn(H, device=DEV), torch.randn(H, device=DEV)
    dg, db = dg0.clone(), db0.clone()
    x2 = o2 = o20 = None
    if with_x2:
        x2 = torch.randn(M, H, device=DEV).to(torch.bfloat16)
        o20 = torch.randn(H, device=DEV)
        o2 = o20.clone()
    nat.ln_param_grad(dy, z, mean, rstd, dg, db, x2, o2)
    _check_ln_param_grads(f"ln_param_grad M={M} H={H}", dy, z, mean, rstd, dg, dg0, db, db0,
                          x2, o2, o20)


def test_ln_param_grad_rejects_h_not_multiple_of_8(nat):
    M, H = 16, 12
    z = torch.zeros(M, H, dtype=torch.bfloat16, device=DEV)
    stats = torch.ones(M, device=DEV)
    with pytest.raises(RuntimeError, match="916"):
        nat.ln_param_grad(z, z, stats, stats, torch.zeros(H, device=DEV),
                          torch.zeros(H, device=DEV))


@pytest.mark.parametrize("eps", [1e-12, 1e-5])
@pytest.mark.parametrize("M", [1, 300, 4100])
@pytest.mark.parametrize("H", [384, 512, 768, 1536, 2048])
def test_layernorm_standalone(nat, H, M, eps):
    """layernorm_fwd / layernorm_bwd (MLM head, and every LayerNorm the GEMM epilogue cannot
    take): H = 384 / 512 instantiate NV = 2, 1536 / 2048 NV = 8.  Row scales span 1e-3 .. 10, so
    the variance of some rows is near eps = 1e-5 and a wrong eps is an O(1) error."""
    torch.manual_seed(700 + H + M)
    scale = 10.0 ** (torch.rand(M, 1, device=DEV) * 4 - 3)
    z = ((torch.randn(M, H, device=DEV) + 0.5) * scale).to(torch.bfloat16)
    gamma = 1.0 + 0.2 * torch.randn(H, device=DEV)
    beta = 0.1 * torch.randn(H, device=DEV)
    y, mean, rstd = nat.layernorm_fwd(z, gamma, beta, eps)
    tag = f"layernorm H={H} M={M} eps={eps:g}"
    zf = z.to(F64)
    (yr, mu, rs, xh), (d_y, d_mu, d_rs) = _ln_fwd_ref(zf, torch.zeros_like(zf), zf.abs(), gamma,
                                                      beta, eps)
    _within(f"{tag} y", y, yr, _bf16_out(yr, d_y))
    _within(f"{tag} mean", mean, mu, d_mu)
    _within(f"{tag} rstd", rstd, rs, d_rs)

    dy = torch.randn(M, H, device=DEV).to(torch.bfloat16)
    dg0, db0 = torch.randn(H, device=DEV), torch.randn(H, device=DEV)
    dg, db = dg0.clone(), db0.clone()
    dz, _ = nat.layernorm_bwd(dy, z, mean, rstd, gamma, dg, db)
    rs_k = rstd.to(F64)[:, None]                    # the statistics the backward was given
    xh = (zf - mean.to(F64)[:, None]) * rs_k
    ref, d_dz = _ln_input_grad_ref(dy.to(F64), torch.zeros_like(zf), xh, 2 * U * xh.abs(), gamma,
                                   rs_k)
    _within(f"{tag} dz", dz, ref, _bf16_out(ref, d_dz))
    _check_ln_param_grads(tag, dy, z, mean, rstd, dg, dg0, db, db0)


# ---------------------------------------------------------------------------------------------
# dgelu_mul, casts
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [8, 4096 * 4096 // 16])
def test_dgelu_mul(nat, n):
    """y = g * gelu'(h) with h over +-8: erff (2 ulp) for the CDF, __expf for the density."""
    torch.manual_seed(800)
    g = torch.randn(n, device=DEV).to(torch.bfloat16)
    h = (torch.rand(n, device=DEV) * 16 - 8).to(torch.bfloat16)
    y = torch.empty_like(g)
    nat.ext().dgelu_mul(g.data_ptr(), h.data_ptr(), y.data_ptr(), n, _stream())
    gd, x = g.to(F64), h.to(F64)
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    ref = gd * (cdf + x * pdf)
    d_cdf = U * x.abs() + 2.0 ** -22 + 2 * U
    d_pdf = pdf * ((3 + EXPF_ULPS * 0.5 * x * x) * 2.0 ** -23 + U * x * x + 2 * U)
    acc = gd.abs() * (d_cdf + x.abs() * d_pdf + 2 * U * (x * pdf).abs()
                      + U * (cdf + x * pdf).abs()) + U * ref.abs()
    _within(f"dgelu_mul n={n}", y, ref, _bf16_out(ref, acc))


def test_dgelu_mul_rejects_n_not_multiple_of_8(nat):
    t = torch.zeros(16, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="914"):
        nat.ext().dgelu_mul(t.data_ptr(), t.data_ptr(), t.data_ptr(), 12, _stream())


def _cast_inputs(n):
    """Finite values over many binades, exact round-to-nearest-even ties (both directions), +-0,
    +-inf, NaN and subnormals; the last three elements (the scalar tail when n % 4 != 0) are
    values whose rounding differs from truncation."""
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, 30, (n,), generator=g).float())
    bits = x.view(torch.int32)
    tie = (torch.arange(n) % 7 == 3)
    bits[tie] = (bits[tie] & ~0xFFFF) | 0x8000               # exactly halfway: round to even
    special = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -3e-39,
                            1.1754942e-38, 65504.0, 3.3895314e38])
    k = min(n, special.numel())
    x[:k] = special[:k] if n > 3 else x[:k]
    up = torch.tensor([0x3F818000, 0x3F80C000, -0x407E4000], dtype=torch.int32).view(torch.float32)
    m = min(n, 3)
    x[n - m:] = up[3 - m:]                                     # 1.0117 (odd tie), 1.0059, -1.98..
    return x


@pytest.mark.parametrize("n", [1, 3, 4, 4097, 2 ** 20 + 3])
def test_casts_match_torch(nat, n):
    """cast_f32_to_bf16 (float4 body + scalar tail in block 0) and cast_bf16_to_f32 are
    bit-identical to torch, subnormals included; a NaN stays a NaN."""
    x = _cast_inputs(n)
    xd = x.to(DEV)
    out = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    nat.ext().cast_f32_to_bf16(xd.data_ptr(), out.data_ptr(), n, _stream())
    got = out.cpu().view(torch.int16)
    ref = x.to(torch.bfloat16).view(torch.int16)
    nan = torch.isnan(x)
    assert torch.isnan(out.cpu()[nan]).all()
    diff = (got != ref) & ~nan
    assert not diff.any(), f"{int(diff.sum())} differ, first at {int(diff.nonzero()[0])}"

    g = torch.Generator().manual_seed(n + 1)
    b = torch.randint(-32768, 32768, (n,), generator=g, dtype=torch.int32).to(torch.int16)
    b[: min(n, 4)] = torch.tensor([0x0001, 0x7F80, 0x7FC1, -0x8000], dtype=torch.int16)[: min(n, 4)]
    bf = b.view(torch.bfloat16)
    f = torch.empty(n, dtype=torch.float32, device=DEV)
    nat.ext().cast_bf16_to_f32(bf.to(DEV).data_ptr(), f.data_ptr(), n, _stream())
    assert torch.equal(f.cpu().view(torch.int32), bf.float().view(torch.int32))


# ---------------------------------------------------------------------------------------------
# end to end at the benchmark's geometry
# ---------------------------------------------------------------------------------------------
def test_embeddings_pooler_classifier_end_to_end(nat):
    """BertEmbeddings -> BertPooler (GEMM path) -> BertTailForClassification with dropout 0.1
    and the fused softmax_ce at B = 32, S = 128, H = 1024, V = 30522.  Each layer is checked
    against its fp64 reference fed the values that layer's kernels received, with the masks of
    the layers' own RNG streams."""
    from skycomputing_b200.models import BertConfig, set_backend
    from skycomputing_b200.models.bert_layers import (BertEmbeddings, BertPooler,
                                                      BertTailForClassification, default_rng)
    from skycomputing_b200.runner.runner import _NativeCrossEntropy

    torch.manual_seed(900)
    B, S, H, V, C, p = 32, 128, 1024, 30522, 3, 0.1
    cfg = BertConfig(V, hidden_size=H, hidden_dropout_prob=p).__dict__
    emb = BertEmbeddings(cfg).to(DEV).train()
    pool = BertPooler(cfg).to(DEV).train()
    tail = BertTailForClassification(p, H, C).to(DEV).train()
    ids, tts, am, _ = _embed_inputs(B, S, H, "uniform", 2, V=V)
    labels = torch.randint(0, C, (B,), device=DEV)
    scale = 0.25                                 # grad_scale = 1 / micro-batches
    loss_acc = torch.zeros(1, device=DEV)
    set_backend("native")
    try:
        hidden, ext_mask = emb(ids, tts, am)
        hidden.retain_grad()
        pooled = pool(hidden, ext_mask)
        pooled.retain_grad()
        logits = tail(pooled)
        dlogits = _NativeCrossEntropy().fused(logits, labels, scale, loss_acc)
        logits.backward(dlogits)
    finally:
        set_backend("auto")
    rng = default_rng(ids.device)
    assert pool._native.w._shadow is not None, "the pooler did not take the GEMM path"

    # forward
    word, pos, typ = (m.weight.detach() for m in (emb.word_embeddings, emb.position_embeddings,
                                                  emb.token_type_embeddings))
    gamma, beta = emb.LayerNorm.weight.detach(), emb.LayerNorm.bias.detach()
    fi, ft, fm = ids.reshape(-1), tts.reshape(-1), am.reshape(-1)
    k_emb = _keep(rng, emb._native.rng_base, (B * S, H), p)
    mean, rstd = _embed_stats(nat, emb, fi, ft, fm, B, S, p, rng)
    worst = _check_embed_fwd("e2e embed", hidden.detach().reshape(B * S, H), ext_mask.reshape(-1),
                             mean, rstd, fi, ft, fm, S, word, pos, typ, gamma, beta, 1e-12, k_emb)
    w_pool, b_pool = pool._native.w.shadow(), pool.dense_act.bias.detach()
    ref, bound = _pooler_fwd_ref(hidden.detach()[:, 0], w_pool, b_pool)
    worst = max(worst, _within("e2e pooler y", pooled, ref, bound))
    k_cls = _keep(rng, tail._native.rng_base, (B, H), p)
    w_cls, b_cls = tail.classifier.weight.detach(), tail.classifier.bias.detach()
    ref, bound, xk = _small_linear_ref(pooled.detach(), k_cls, w_cls, b_cls, False)
    _within("e2e classifier logits", logits, ref, bound)
    r = _softmax_ce_ref(logits.detach(), labels, scale, 0.0, calls=1)
    _within("e2e loss_acc", loss_acc[0], r["acc"], r["d_acc"])
    _within("e2e dlogits", dlogits, r["dlogits"], r["d_dlogits"])

    # backward: every parameter gradient started from zero
    zeros = torch.zeros_like
    _check_small_linear_bwd("e2e classifier", dlogits, logits.detach(), xk, k_cls, w_cls, False,
                            pooled.grad, False, tail.classifier.weight.grad, zeros(w_cls),
                            tail.classifier.bias.grad, zeros(b_cls))
    dh = hidden.grad.reshape(B, S, H)
    assert torch.count_nonzero(dh[:, 1:]) == 0
    worst = max(worst, _check_pooler_bwd("e2e pooler", pooled.grad, pooled.detach(),
                                         hidden.detach()[:, 0], w_pool,
                                         pool.dense_act.weight.grad,
                                         zeros(w_pool, dtype=torch.float32),
                                         pool.dense_act.bias.grad, zeros(b_pool), dh[:, 0]))
    grads = [m.weight.grad for m in (emb.word_embeddings, emb.position_embeddings,
                                      emb.token_type_embeddings)]
    grads += [emb.LayerNorm.weight.grad, emb.LayerNorm.bias.grad]
    worst = max(worst, _check_embed_bwd("e2e embed", grads, [zeros(g) for g in grads],
                                        hidden.grad.reshape(B * S, H), fi, ft, S, word, pos, typ,
                                        gamma, mean, rstd, k_emb))
    assert 0 < worst <= 1


def _embed_stats(nat, emb, ids, tts, am, B, S, p, rng):
    """(mean, rstd) of the embedding forward, which EmbeddingsFn keeps only inside its autograd
    context: the forward kernel is deterministic, so a second call reproduces them."""
    ep = emb._native
    _, _, mean, rstd = _embed_fwd_call(
        nat, ids, tts, am, ep.word.master(), ep.pos.master(), ep.type.master(), ep.gamma.master(),
        ep.beta.master(), B, S, ep.eps, p, rng, ep.rng_base)
    return mean, rstd
