"""Compile-only check of the weight-gradient GEMM with the SGD update in its epilogue (no GPU
needed): both tile widths keep the classic kernels' register budget and do not spill."""
import os
import re

import pytest

from tests.test_attention_fragments_cpu import NVCC, ROOT, _ptxas

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def test_wgrad_sgd_kernels_do_not_spill(tmp_path):
    res, log = _ptxas(os.path.join(ROOT, "csrc", "kernels", "gemm_sm100.cu"), tmp_path)
    upd = {int(m.group(1)): v for k, v in res.items()
           if (m := re.search(r"\d+gemm_wgrad_sgd_kernelILi(\d+)EE", k))}
    # the classic fp32 weight-gradient kernels (both operands MN-major, single CTAs, no stream-K)
    plain = {int(m.group(1)): v for k, v in res.items()
             if (m := re.search(r"\d+gemm_wgmma_kernelILi(\d+)ELb1ELb1ELb1ELi1ELb0EE", k))}
    assert sorted(upd) == [128, 256] and sorted(plain) == [128, 256], log
    for bn, props in upd.items():
        assert props["spill"] == 0, (bn, props)
        assert props["regs"] <= plain[bn]["regs"], (bn, props, plain[bn])
