"""The pair layout of the GEMM + LayerNorm kernel (N = 1024, 256-wide warpgroup tiles): 64-row
panels, one CTA pair per panel."""
import pytest
import torch

from tests.test_kernels_gpu import _close, _ln_ref, _rand, nat  # noqa: F401

pytestmark = pytest.mark.gpu


def test_pair_layout_fits_a_4096_token_launch_in_one_wave(nat):
    clusters, size = nat.ext().gemm_ln_max_active_clusters(1024, 256)
    assert size == 2
    assert clusters >= 4096 // 64


@pytest.mark.parametrize("M,K", [(64, 64), (960, 320), (1000, 1024), (4000, 1096)])
def test_pair_layout_ragged_rows(nat, M, K):
    """Every 128-row panel receives its 4 signals even when its second pair lies past M (M = 960
    and 64), y / mean / rstd match fp32 references, and z is the two-kernel path's z bit for bit."""
    torch.manual_seed(M + K)
    N = 1024
    assert nat.ext().gemm_ln_block_n(M, N, True) == 256
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    res = _rand(M, N)
    gamma = 1.0 + 0.1 * torch.randn(N, device="cuda")
    beta = 0.1 * torch.randn(N, device="cuda")
    panels = (M + 127) // 128
    flags = torch.zeros(panels, dtype=torch.int32, device="cuda")
    rng = nat.RngState(7)
    y, z, mean, rstd = nat.gemm_ln(a, w, gamma, beta, bias=bias, residual=res, dropout_p=0.1,
                                   rng=rng, rng_stream=4, signal_flags=flags.data_ptr())
    torch.cuda.synchronize()
    assert flags.tolist() == [nat.ext().gemm_ln_tiles_per_panel(M, N, True)] * panels == [4] * panels
    z2 = nat.gemm(a, w, bias=bias, aux=res, add_aux=True, dropout_p=0.1, rng=rng, rng_stream=4)
    assert torch.equal(z, z2)
    yr, mur, rstdr = _ln_ref(z.float(), gamma, beta)
    _close(y, yr, rtol=2e-2, atol=3e-2)
    torch.testing.assert_close(mean, mur, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(rstd, rstdr, rtol=2e-3, atol=1e-4)
