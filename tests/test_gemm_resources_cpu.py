"""Compile-only checks of the wgmma GEMM kernels' resources (no GPU needed).

Both GEMM kernels are built from the same prologue, producer, main-loop and epilogue steps, and
those steps must not cost the kernels registers: every kernel a training step runs stays free of
spills, and ptxas neither serialises a wgmma on a register hazard nor injects a warpgroup.arrive.
"""
import os
import re

import pytest

from tests.test_attention_fragments_cpu import NVCC, ROOT, _ptxas

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

# gemm_wgmma_kernel<BLOCK_N, A_MN, B_MN, OUT_F32, CL, SK> / gemm_ln_wgmma_kernel<BLOCK_N>
PLAIN = re.compile(r"\d+gemm_wgmma_kernelILi(\d+)ELb([01])ELb([01])ELb([01])ELi(\d)ELb([01])EE")
LN = re.compile(r"\d+gemm_ln_wgmma_kernelILi(\d+)EE")
# spill bytes (stores, loads) of the opt-in stream-K instantiations, by BLOCK_N
STREAM_K_SPILL_LIMIT = {128: (0, 0), 256: (146, 236)}


@pytest.fixture(scope="module")
def gemm_ptxas(tmp_path_factory):
    # one compile of the file for the whole module: it takes minutes without a GPU
    return _ptxas(os.path.join(ROOT, "csrc", "kernels", "gemm_sm100.cu"),
                  tmp_path_factory.mktemp("gemm"))


def _kernels(res, pattern):
    return {tuple(int(x) for x in m.groups()): v for k, v in res.items() if (m := pattern.search(k))}


def test_gemm_kernels_do_not_spill(gemm_ptxas):
    res, log = gemm_ptxas
    plain = _kernels(res, PLAIN)
    # 2 tile widths x 2 x 2 operand majors x 2 output types x 3 cluster sizes, plus stream-K at CL = 1
    assert len(plain) == 64, log
    for (bn, _, _, _, cl, sk), props in plain.items():
        if sk:
            assert cl == 1
            stores, loads = STREAM_K_SPILL_LIMIT[bn]
            assert props["spill_stores"] <= stores and props["spill_loads"] <= loads, (bn, props)
        else:
            assert props["spill"] == 0, (bn, cl, props)
    ln = _kernels(res, LN)
    assert sorted(ln) == [(128,), (256,)], log
    for bn, props in ln.items():
        assert props["spill"] == 0, (bn, props)


def test_gemm_wgmma_not_serialised(gemm_ptxas):
    _, log = gemm_ptxas
    # no wgmma made to wait on a register hazard (C7517), no injected warpgroup.arrive (C7519)
    assert "C7517" not in log, log
    assert "C7519" not in log, log
