"""Compile-only checks of the register-A wgmma and of the attention kernels' resources.

No GPU is needed: nvcc builds for sm_90a and ptxas reports registers and spills.  The S = 128
forward is meant to run two CTAs per SM, which needs at most 128 registers at 256 threads.
"""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

RS_PROBE = r"""
#include "kernels/sm100_ptx.cuh"
using namespace sky;
// P (registers) x V (MN-major, shared memory), the product the attention forward issues, and the
// 128-wide form
__global__ void __launch_bounds__(128) rs_probe(float* out) {
  __shared__ __align__(1024) uint8_t tile[16384];
  float d64[32], d128[64];
  for (int i = 0; i < 32; ++i) d64[i] = 0.f;
  for (int i = 0; i < 64; ++i) d128[i] = 0.f;
  uint32_t a[4];
  frag_to_a(d128, threadIdx.x & 7, a);
  acc_fence(d64);
  acc_fence(d128);
  wgmma_fence();
  for (int k = 0; k < 8; ++k) wgmma_rs_k16<64, 1>(d64, a, desc_mnmajor(smem_u32(tile), k, 16384, 0), 1u);
  for (int k = 0; k < 4; ++k) wgmma_rs_k16<128, 0>(d128, a, desc_kmajor(smem_u32(tile), k, 16384, 0), 1u);
  wgmma_commit();
  wgmma_wait<0>();
  for (int i = 0; i < 32; ++i) out[i * 128 + threadIdx.x] = d64[i] + d128[i] + d128[32 + i];
}
"""


def _ptxas(src_path, tmp_path):
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math",
           "-Xptxas", "-v", f"-I{os.path.join(ROOT, 'csrc')}", "-c", str(src_path), "-o",
           str(tmp_path / "probe.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    out = {}
    current = None
    for line in proc.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            props = out.setdefault(current, {})
            props["spill_stores"], props["spill_loads"] = int(m.group(1)), int(m.group(2))
            props["spill"] = props["spill_stores"] + props["spill_loads"]
        m = re.search(r"Used (\d+) registers", line)
        if m and current:
            out.setdefault(current, {})["regs"] = int(m.group(1))
    return out, proc.stderr


def test_register_a_wgmma_compiles_without_spills(tmp_path):
    src = tmp_path / "rs_probe.cu"
    src.write_text(RS_PROBE)
    res, _ = _ptxas(src, tmp_path)
    (props,) = [v for k, v in res.items() if "rs_probe" in k]
    assert props["spill"] == 0


ATTENTION_KERNELS = ("attention_fwd_kernel", "attention_bwd_kernel", "attention_fwd_tiled_kernel",
                     "attention_bwd_dq_kernel", "attention_bwd_dkv_kernel")


def test_attention_kernels_fit_their_occupancy(tmp_path):
    res, log = _ptxas(os.path.join(ROOT, "csrc", "kernels", "attention_sm100.cu"), tmp_path)
    props = {}
    for name in ATTENTION_KERNELS:
        found = [v for k, v in res.items() if re.search(rf"\d{name}E", k)]
        assert len(found) == 1, (name, log)
        props[name] = found[0]
        assert found[0]["spill"] == 0, (name, log)
    # 2 CTAs x 256 threads in the 64 K-register file
    assert props["attention_fwd_kernel"]["regs"] <= 128
    # no wgmma was made to wait on a register hazard (ptxas info C7517), and ptxas injected no
    # warpgroup.arrive to reach the accumulator registers (C7519)
    assert "C7517" not in log, log
    assert "C7519" not in log, log
