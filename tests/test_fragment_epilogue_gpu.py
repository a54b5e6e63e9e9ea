"""GEMM epilogues at training-step sizes (M = 4096 tokens) against an fp32 torch reference.

At these shapes every CTA of the persistent GEMM handles several tiles in turn, so the operand
ring's stage / phase and the double-buffered bias tile are carried from one tile to the next; the
ragged shapes cover partial row and column tiles.  Every epilogue variant runs on the accumulator
fragments: bias, GELU with the pre-activation as a second output, residual add, dGELU x aux,
dropout (exact keep mask from the host replica of the device RNG), fp32 output and fp32
accumulation, and the GEMM + LayerNorm kernel.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(4096, 4096, 1024), (4096, 1024, 4096), (4000, 1000, 1024)]


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
    assert torch.isfinite(got).all(), "non-finite output"
    err = (got - ref).abs().max().item()
    denom = ref.abs().max().item() + 1e-6
    assert err <= atol + rtol * denom, f"max abs err {err} vs ref max {denom}"


def _operands(M, N, K, seed):
    torch.manual_seed(seed)
    s = 1.0 / math.sqrt(K)
    return _rand(M, K), _rand(N, K, scale=s), torch.randn(N, device="cuda") * 0.1


def _gelu(h):
    return h * 0.5 * (1.0 + torch.erf(h / math.sqrt(2.0)))


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bias(nat, M, N, K):
    a, b, bias = _operands(M, N, K, 1)
    out = nat.gemm(a, b, bias=bias)
    _close(out, a.float() @ b.float().t() + bias)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gelu_with_preactivation(nat, M, N, K):
    a, b, bias = _operands(M, N, K, 2)
    pre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    out = nat.gemm(a, b, bias=bias, act=nat.ACT_GELU, out2=pre)
    h = a.float() @ b.float().t() + bias
    _close(pre, h)
    _close(out, _gelu(h))


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_residual_add_dgrad_layout(nat, M, N, K):
    """dX = dY W + residual: B MN-major, as the backward of the QKV and FFN1 projections runs."""
    torch.manual_seed(3)
    dy, w = _rand(M, K), _rand(K, N, scale=1.0 / math.sqrt(K))
    aux = _rand(M, N)
    out = nat.gemm(dy, w, b_mn=True, aux=aux, add_aux=True)
    _close(out, dy.float() @ w.float() + aux.float())


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgelu_times_aux(nat, M, N, K):
    torch.manual_seed(4)
    dy, w = _rand(M, K), _rand(K, N, scale=1.0 / math.sqrt(K))
    aux = _rand(M, N)
    out = nat.gemm(dy, w, b_mn=True, aux=aux, act=nat.ACT_DGELU_MUL_AUX)
    x = aux.float()
    dg = 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    _close(out, (dy.float() @ w.float()) * dg)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dropout_exact_mask(nat, M, N, K):
    from skycomputing_b200.ops.dropout_ref import keep_mask_from_state

    a, b, bias = _operands(M, N, K, 5)
    res = _rand(M, N)
    p = 0.1
    rng = nat.RngState(2024)
    out = nat.gemm(a, b, bias=bias, aux=res, add_aux=True, dropout_p=p, rng=rng, rng_stream=9)
    keep = torch.from_numpy(keep_mask_from_state(rng.state, 9, (M, N), p)).cuda()
    h = a.float() @ b.float().t() + bias
    ref = torch.where(keep, h / (1 - p), torch.zeros_like(h)) + res.float()
    _close(out, ref)
    # the dropped elements are exactly the residual
    dropped = ~keep
    assert torch.equal(out[dropped], res[dropped])


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_fp32_out_and_accumulate(nat, M, N, K):
    """Weight-gradient layout: dW[N, K] (+)= dY^T X with both operands MN-major, fp32 output."""
    torch.manual_seed(6)
    dy, x = _rand(K, M, scale=0.3), _rand(K, N, scale=0.3)   # reduction over K "tokens"
    ref = dy.float().t() @ x.float()
    dw = nat.gemm(dy, x, a_mn=True, b_mn=True, out_dtype=torch.float32)
    _close(dw, ref, rtol=1e-2)
    acc = torch.full((M, N), 0.5, device="cuda", dtype=torch.float32)
    nat.gemm(dy, x, a_mn=True, b_mn=True, out=acc, accumulate=True)
    _close(acc, ref + 0.5, rtol=1e-2)
    nat.gemm(dy, x, a_mn=True, b_mn=True, out=acc, accumulate=True)
    _close(acc, 2 * ref + 0.5, rtol=1e-2)


@pytest.mark.parametrize("M,N,K", [(4096, 1024, 1024), (4096, 1024, 4096), (4000, 1024, 1024)])
@pytest.mark.parametrize("block_n", [128, 256])
def test_layernorm_epilogue(nat, M, N, K, block_n):
    from skycomputing_b200.ops.dropout_ref import keep_mask_from_state

    a, w, bias = _operands(M, N, K, 7)
    res = _rand(M, N)
    gamma = 1.0 + 0.1 * torch.randn(N, device="cuda")
    beta = 0.1 * torch.randn(N, device="cuda")
    p = 0.1
    rng = nat.RngState(77)
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, bias=bias, residual=res, dropout_p=p,
                                   rng=rng, rng_stream=4, block_n=block_n)
    keep = torch.from_numpy(keep_mask_from_state(rng.state, 4, (M, N), p)).cuda()
    h = a.float() @ w.float().t() + bias
    zr = torch.where(keep, h / (1 - p), torch.zeros_like(h)) + res.float()
    mur = zr.mean(dim=1)
    var = zr.var(dim=1, unbiased=False)
    rstdr = torch.rsqrt(var + 1e-12)
    _close(z, zr)
    torch.testing.assert_close(mean, mur, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(rstd, rstdr, rtol=2e-3, atol=1e-4)
    _close(y, (zr - mur[:, None]) * rstdr[:, None] * gamma + beta)
