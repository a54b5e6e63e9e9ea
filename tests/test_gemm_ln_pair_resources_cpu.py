"""Compile-only check of the GEMM + LayerNorm kernel's pair layout (no GPU needed): it keeps the
wide layout's register budget and does not spill."""
import os
import re

import pytest

from tests.test_attention_fragments_cpu import NVCC, ROOT, _ptxas

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def test_gemm_ln_pair_kernel_does_not_spill(tmp_path):
    res, log = _ptxas(os.path.join(ROOT, "csrc", "kernels", "gemm_sm100.cu"), tmp_path)
    pair = [v for k, v in res.items() if re.search(r"\d+gemm_ln_pair_kernelE", k)]
    wide = [v for k, v in res.items() if re.search(r"\d+gemm_ln_wgmma_kernelILi256EE", k)]
    assert len(pair) == 1 and len(wide) == 1, log
    assert pair[0]["spill"] == 0, pair[0]
    assert pair[0]["regs"] <= wide[0]["regs"], (pair[0], wide[0])
