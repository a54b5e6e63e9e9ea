"""fp64 references and worst-case error bounds shared by the kernel tests.

Every bound is the output rounding plus a worst-case accumulation term n * u * sum|terms|, with
sum|terms| computed by the same fp64 reference over absolute values, plus the documented error of
each approximate intrinsic.  ``_within`` checks every element against its own bound and prints
the largest |err| / bound as a ``[bound]`` line.
"""
import numpy as np
import torch

from skycomputing_b200.ops.dropout_ref import keep_mask_from_state

U = 2.0 ** -24          # fp32 round-to-nearest unit roundoff
U_TC = 2.0 ** -23       # tensor-core fp32 accumulation is not specified as round-to-nearest: 1 ulp
BF16 = 2.0 ** -8        # bf16 round-to-nearest: half an ulp of 8 significant bits, relative
RSQRT_APPROX = 2.0 ** -22     # PTX ISA: rsqrt.approx.f32 max relative error 2^-22.9
EXPF_ULPS = 1.173             # CUDA guide: __expf max error 2 + floor(|1.173 x|) ulp
# kept elements are scaled by the fp32 1 / (1 - p) under fast math: 1 - p (1 rounding), an
# approximate reciprocal (2 ulp) and the multiply: relative error <= 6u
DROP = 6 * U
F64 = torch.float64
DEV = "cuda"


def _within(name, got, ref, bound):
    """Every element of ``got`` within its own ``bound`` of ``ref``; returns max |err| / bound."""
    got = got.detach().to(F64).reshape(ref.shape if ref.dim() else (1,))
    ref = ref.reshape(got.shape)
    bound = torch.as_tensor(bound, dtype=F64).expand(ref.shape).reshape(got.shape)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    err = (got - ref).abs()
    bad = err > bound
    if bad.any():
        i = int(torch.argmax((err - bound).reshape(-1)))
        idx = np.unravel_index(i, tuple(ref.shape))
        raise AssertionError(
            f"{name}: {int(bad.sum())} of {ref.numel()} elements outside their bound; worst at "
            f"{idx}: got {got.reshape(-1)[i].item():.8g}, ref {ref.reshape(-1)[i].item():.8g}, "
            f"bound {bound.reshape(-1)[i].item():.3g}")
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    print(f"[bound] {name}: max |err|/bound = {worst:.3g}")
    return worst


def _bf16_out(ref, acc):
    """Bound of a bf16 output: its rounding (relative 2^-8 of the value) plus the fp32 error
    ``acc`` of the value before rounding, which the rounding can scale by at most 1 + 2^-8."""
    return BF16 * ref.abs() + (1 + BF16) * acc


def _keep(rng, stream, shape, p):
    """Kept-and-scaled factor of each element of a dropout site (1 everywhere when p = 0)."""
    if p <= 0:
        return torch.ones(shape, dtype=F64, device=DEV)
    keep = torch.from_numpy(keep_mask_from_state(rng.state, stream, shape, p)).to(DEV)
    # the kernels scale by an fp32 1 / (1 - p) of the fp32 p: its error is in DROP
    return keep.to(F64) / (1.0 - float(np.float32(p)))

# ---------------------------------------------------------------------------------------------
# LayerNorm statistics: shared by the embedding and standalone LayerNorm references
# ---------------------------------------------------------------------------------------------
def _ln_fwd_ref(e, e_err, e_abs, gamma, beta, eps):
    """fp64 LayerNorm of rows ``e`` that the kernel holds in fp32 with per-element error
    ``e_err``.  Returns (y, mean, rstd, xhat) and the worst-case fp32 errors (y, mean, rstd) of a
    kernel that sums each row of H elements in some order."""
    H = e.shape[1]
    g, b = gamma.to(F64), beta.to(F64)
    mu = e.mean(1, keepdim=True)
    var = ((e - mu) ** 2).mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(var + eps)
    xh = (e - mu) * rs
    y = xh * g + b
    # mean: H fp32 additions over |e| (+ the errors of e), then one multiply by 1/H
    d_mu = (H + 2) * U * e_abs.mean(1, keepdim=True) + e_err.mean(1, keepdim=True)
    # one e - mu is off by at most dl; the variance sum of (x + d)^2 is off by 2 dl sum|x| + H dl^2
    # with sum|x| <= H sigma, plus H additions of positive terms and a few roundings
    dl = e_err.amax(1, keepdim=True) + d_mu
    sig = torch.sqrt(var)
    var_rel = (2 * dl * sig + dl * dl) / (var + eps) + (H + 6) * U
    rs_rel = 0.5 * var_rel * 1.01 + RSQRT_APPROX
    d_xh = rs * (e_err + d_mu) + xh.abs() * (rs_rel + 3 * U)
    d_y = g.abs() * d_xh + 2 * U * ((xh * g).abs() + b.abs())
    return (y, mu.squeeze(1), rs.squeeze(1), xh), (d_y, (d_mu + U * mu.abs()).squeeze(1),
                                                 (rs * rs_rel).squeeze(1))


def _ln_input_grad_ref(dy, dy_err, xh, xh_err, gamma, rs):
    """fp64 LayerNorm input gradient (q - mean(q) - xhat mean(q xhat)) * rstd, q = dy * gamma,
    and its worst-case fp32 error: two H-long row sums plus the elementwise roundings."""
    H = dy.shape[1]
    g = gamma.to(F64)
    q = dy * g
    dq = dy_err * g.abs() + U * q.abs()
    c1 = q.mean(1, keepdim=True)
    c2 = (q * xh).mean(1, keepdim=True)
    dc1 = ((H + 1) * U * q.abs().sum(1, keepdim=True) + dq.sum(1, keepdim=True)) / H \
        + U * c1.abs()
    dc2 = ((H + 1) * U * (q * xh).abs().sum(1, keepdim=True)
           + (q.abs() * xh_err + xh.abs() * dq).sum(1, keepdim=True)) / H + U * c2.abs()
    dz = (q - c1 - xh * c2) * rs
    d_dz = rs * (dq + dc1 + xh.abs() * dc2 + c2.abs() * xh_err
                 + 4 * U * (q.abs() + c1.abs() + (xh * c2).abs()))
    return dz, d_dz


def _colsum_ref(name, got, init, terms, term_err, n_adds):
    """``got`` = init + column sums of ``terms`` accumulated in fp32 by at most ``n_adds``
    additions per column, each off by at most u * (|init| + sum|terms|)."""
    ref = init.to(F64) + terms.sum(0)
    bound = n_adds * U * (init.to(F64).abs() + terms.abs().sum(0)) + term_err.sum(0)
    return _within(name, got, ref, bound)
