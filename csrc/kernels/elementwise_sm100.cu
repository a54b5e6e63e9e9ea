// Memory-bound sm_90a kernels: LayerNorm fwd/bwd (optionally gated on cross-GPU panel flags),
// bias-gradient column sums, fused embedding gather+LN+dropout and its scatter backward, the
// latency-bound pooler / classifier / cross-entropy heads, fused multi-tensor SGD / Adam with the
// gradient-norm reduction and optimizer scalars they read (global-norm clipping, learning-rate
// schedules), and the small runtime kernels (RNG step, flag epochs, device-side throttle, peer
// copy + signal).
//
// Reference parity (what these replace):
//   BertLayerNorm            scaelum/model/bert_layers.py:143-168   -> layernorm_{fwd,bwd}
//   BertEmbeddings.forward   scaelum/model/bert_layers.py:191-212   -> embed_{fwd,bwd}
//   BertPooler / classifier  scaelum/model/bert_layers.py:366-395   -> small_linear_{fwd,bwd}
//   nn.CrossEntropyLoss      scaelum/runner/runner.py:51-52,131     -> softmax_ce
//   optim.SGD step           experiment/launch.py:152-155           -> sgd_multi
//   time.sleep slowdown      scaelum/builder/module_wrapper.py:124-126,265-266 -> spin_* kernels
#include <algorithm>
#include <type_traits>

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "api.h"
#include "launch_util.h"
#include "sm100_ptx.cuh"

namespace sky {

namespace {

constexpr uint64_t kFlagTimeoutNs = 4000000000ull;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void warp_wait_panel(const uint32_t* flags, int panel, uint32_t target,
                                                int* error_flag, int lane) {
  if (lane == 0) {
    if (!wait_flag_ge(flags + panel, target, kFlagTimeoutNs)) {
      if (error_flag) atomicExch(error_flag, 2);
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, 8 bf16 (16B) per lane per step, row held in registers.
// H % 8 == 0, H <= 2048.  NV = number of 16B vectors per lane (compile-time).
// ------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 8;  // H <= 8*256
constexpr int kLnRowsPerCta = 8;  // one row per warp; a 128-row panel = 16 signals

template <int NV>
__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ z, __nv_bfloat16* __restrict__ y,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out,
                     const float* __restrict__ gamma, const float* __restrict__ beta, int M, int H,
                     float eps, const uint32_t* wait_flags, const uint32_t* wait_epoch,
                     uint32_t wait_mult, int* error_flag, uint32_t* signal_flags) {
  pdl_wait();
  pdl_launch_dependents();
  // Each CTA owns kLnRowsPerCta consecutive rows (8 warps x 4 rows) so that a finished CTA can
  // publish "32 rows of panel p are written" with one release.sys add (y may be peer memory).
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nvec = H / 8;  // 16B vectors per row
  const float inv_h = 1.f / static_cast<float>(H);
  const uint32_t target = wait_flags ? (*wait_epoch) * wait_mult : 0u;
  int last_panel = -1;
  const int row_base = blockIdx.x * kLnRowsPerCta;

  for (int r = warp; r < kLnRowsPerCta; r += 8) {
    const int row = row_base + r;
    if (row >= M) break;
    if (wait_flags != nullptr) {
      const int panel = row >> 7;
      if (panel != last_panel) {
        warp_wait_panel(wait_flags, panel, target, error_flag, lane);
        last_panel = panel;
      }
    }
    const uint4* zr = reinterpret_cast<const uint4*>(z + static_cast<long long>(row) * H);
    float x[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < nvec) {
        const uint4 u = zr[v];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 f = unpack_bf16x2(w[t]);
          x[i][2 * t] = f.x;
          x[i][2 * t + 1] = f.y;
          s += f.x + f.y;
        }
      }
    }
    const float mu = warp_sum(s) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < nvec) {
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float d = x[i][t] - mu;
          sq += d * d;
        }
      }
    }
    const float var = warp_sum(sq) * inv_h;
    const float rs = rsqrtf(var + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mu;
      if (rstd_out) rstd_out[row] = rs;
    }
    uint4* yr = reinterpret_cast<uint4*>(y + static_cast<long long>(row) * H);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < nvec) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
        uint4 o;
        o.x = pack_bf16x2((x[i][0] - mu) * rs * g0.x + b0.x, (x[i][1] - mu) * rs * g0.y + b0.y);
        o.y = pack_bf16x2((x[i][2] - mu) * rs * g0.z + b0.z, (x[i][3] - mu) * rs * g0.w + b0.w);
        o.z = pack_bf16x2((x[i][4] - mu) * rs * g1.x + b1.x, (x[i][5] - mu) * rs * g1.y + b1.y);
        o.w = pack_bf16x2((x[i][6] - mu) * rs * g1.z + b1.z, (x[i][7] - mu) * rs * g1.w + b1.w);
        yr[v] = o;
      }
    }
  }
  if (signal_flags != nullptr) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) red_release_sys_add(signal_flags + (row_base >> 7), 1u);
  }
}

// ------------------------------------------------------------------------------------------
// LayerNorm backward (input gradient).  One warp per row; parameter gradients are produced by
// ln_param_grad_kernel below (column-oriented, no per-lane column partials -> low registers).
// ------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ z,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     const float* __restrict__ gamma, __nv_bfloat16* __restrict__ dz,
                     __nv_bfloat16* __restrict__ dz_dropped, int M, int H, float dropout_p,
                     const uint64_t* rng_state, uint32_t rng_stream, const uint32_t* wait_flags,
                     const uint32_t* wait_epoch, uint32_t wait_mult, int* error_flag) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int warp_global = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int total_warps = gridDim.x * warps_per_block;
  const int nvec = H / 8;
  const float inv_h = 1.f / static_cast<float>(H);
  const uint32_t target = wait_flags ? (*wait_epoch) * wait_mult : 0u;
  int last_panel = -1;
  // the masked copy is written only when dz_dropped is given
  const Dropout drop =
      dropout_of(dz_dropped != nullptr ? dropout_p : 0.f, rng_state, rng_stream);

  for (int row = warp_global; row < M; row += total_warps) {
    if (wait_flags != nullptr) {
      const int panel = row >> 7;
      if (panel != last_panel) {
        warp_wait_panel(wait_flags, panel, target, error_flag, lane);
        last_panel = panel;
      }
    }
    const float mu = mean[row];
    const float rs = rstd[row];
    const uint4* zr = reinterpret_cast<const uint4*>(z + static_cast<long long>(row) * H);
    const uint4* dr = reinterpret_cast<const uint4*>(dy + static_cast<long long>(row) * H);
    float xh[NV][8], g[NV][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < nvec) {
        const uint4 uz = zr[v];
        const uint4 ud = dr[v];
        const uint32_t wz[4] = {uz.x, uz.y, uz.z, uz.w};
        const uint32_t wd[4] = {ud.x, ud.y, ud.z, ud.w};
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
        const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 fz = unpack_bf16x2(wz[t]);
          const float2 fd = unpack_bf16x2(wd[t]);
          const float x0 = (fz.x - mu) * rs, x1 = (fz.y - mu) * rs;
          xh[i][2 * t] = x0;
          xh[i][2 * t + 1] = x1;
          const float q0 = fd.x * gm[2 * t], q1 = fd.y * gm[2 * t + 1];
          g[i][2 * t] = q0;
          g[i][2 * t + 1] = q1;
          s1 += q0 + q1;
          s2 += q0 * x0 + q1 * x1;
        }
      }
    }
    const float c1 = warp_sum(s1) * inv_h;
    const float c2 = warp_sum(s2) * inv_h;
    uint4* dzr = reinterpret_cast<uint4*>(dz + static_cast<long long>(row) * H);
    uint4* dzd = drop.on
                     ? reinterpret_cast<uint4*>(dz_dropped + static_cast<long long>(row) * H)
                     : nullptr;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) o[t] = (g[i][t] - c1 - xh[i][t] * c2) * rs;
        dzr[v] = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]),
                            pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        if (drop.on) {
          const uint64_t base = (static_cast<uint64_t>(row) * H + v * 8) >> 2;
          const uint32_t m0 = dropout_keep4(drop.seed, base, drop.thr16);
          const uint32_t m1 = dropout_keep4(drop.seed, base + 1, drop.thr16);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            o[t] = (m0 >> t) & 1u ? o[t] * drop.scale : 0.f;
            o[4 + t] = (m1 >> t) & 1u ? o[4 + t] * drop.scale : 0.f;
          }
          dzd[v] = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]),
                              pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        }
      }
    }
  }
}

// dgamma[c] += sum_r dy[r,c] * xhat[r,c];  dbeta[c] += sum_r dy[r,c]
// block = 32 column groups (8 columns each) x 8 row lanes; grid.y splits the rows.
__global__ void __launch_bounds__(256)
ln_param_grad_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ z,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, int M, int H,
                     const __nv_bfloat16* __restrict__ x2, float* __restrict__ out2) {
  // x2 / out2 (optional): out2[c] += sum_r x2[r,c] - the bias gradient of the dense layer in front
  // of this LayerNorm (column sum of the LayerNorm input gradient), fused here to save a launch
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float redg[8][256 + 8];
  __shared__ float redb[8][256 + 8];
  __shared__ float red2[8][256 + 8];
  float a2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int cg = threadIdx.x & 31;
  const int rl = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + cg) * 8;
  float ag[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ab[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < H) {
    for (int r = blockIdx.y * 8 + rl; r < M; r += gridDim.y * 8) {
      const float mu = mean[r], rs = rstd[r];
      const uint4 ud = *reinterpret_cast<const uint4*>(dy + static_cast<long long>(r) * H + col);
      const uint4 uz = *reinterpret_cast<const uint4*>(z + static_cast<long long>(r) * H + col);
      const uint32_t wd[4] = {ud.x, ud.y, ud.z, ud.w};
      const uint32_t wz[4] = {uz.x, uz.y, uz.z, uz.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 fd = unpack_bf16x2(wd[t]);
        const float2 fz = unpack_bf16x2(wz[t]);
        ag[2 * t] += fd.x * (fz.x - mu) * rs;
        ag[2 * t + 1] += fd.y * (fz.y - mu) * rs;
        ab[2 * t] += fd.x;
        ab[2 * t + 1] += fd.y;
      }
      if (x2 != nullptr) {
        const uint4 ux = *reinterpret_cast<const uint4*>(x2 + static_cast<long long>(r) * H + col);
        const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 fx = unpack_bf16x2(wx[t]);
          a2[2 * t] += fx.x;
          a2[2 * t + 1] += fx.y;
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    redg[rl][cg * 8 + t] = ag[t];
    redb[rl][cg * 8 + t] = ab[t];
    red2[rl][cg * 8 + t] = a2[t];
  }
  __syncthreads();
  const int c = threadIdx.x;
  float sg = 0.f, sb = 0.f, s2 = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    sg += redg[r][c];
    sb += redb[r][c];
    s2 += red2[r][c];
  }
  const int gc = blockIdx.x * 256 + c;
  if (gc < H) {
    if (dgamma) atomicAdd(&dgamma[gc], sg);
    if (dbeta) atomicAdd(&dbeta[gc], sb);
    if (out2) atomicAdd(&out2[gc], s2);
  }
}

// ------------------------------------------------------------------------------------------
// Column sums of a bf16 [M,N] matrix into fp32 (+=).  block = (32 col-groups of 8) x 8 row lanes
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, int M, int N, long long ldx,
              float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8][256 + 8];
  const int cg = threadIdx.x & 31;
  const int rl = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + cg) * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    for (int r = blockIdx.y * 8 + rl; r < M; r += gridDim.y * 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + r * ldx + col);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = unpack_bf16x2(w[t]);
        acc[2 * t] += f.x;
        acc[2 * t + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) red[rl][cg * 8 + t] = acc[t];
  __syncthreads();
  const int c = threadIdx.x;  // 256 columns per block
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) s += red[r][c];
  const int gc = blockIdx.x * 256 + c;
  if (gc < N) atomicAdd(&out[gc], s);
}

// ------------------------------------------------------------------------------------------
// Embeddings
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_fwd_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ tts,
                 const int64_t* __restrict__ amask, const float* __restrict__ word,
                 const float* __restrict__ pos, const float* __restrict__ type,
                 const float* __restrict__ gamma, const float* __restrict__ beta,
                 __nv_bfloat16* __restrict__ out, float* __restrict__ ext_mask,
                 float* __restrict__ mean_out, float* __restrict__ rstd_out, int BS, int S, int H,
                 float eps, float dropout_p, const uint64_t* rng_state, uint32_t rng_stream) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int row0 = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int total_warps = gridDim.x * warps_per_block;
  const float inv_h = 1.f / static_cast<float>(H);
  const Dropout drop = dropout_of(dropout_p, rng_state, rng_stream);
  for (int row = row0; row < BS; row += total_warps) {
    const long long id = ids[row];
    const long long tt = tts[row];
    const int s = row % S;
    if (lane == 0 && ext_mask != nullptr)
      ext_mask[row] = amask ? (1.0f - static_cast<float>(amask[row])) * -10000.0f : 0.f;
    const float* wr = word + id * H;
    const float* pr = pos + static_cast<long long>(s) * H;
    const float* tr = type + tt * H;
    float sum = 0.f;
    for (int c = lane * 4; c < H; c += 128) {
      const float4 a = *reinterpret_cast<const float4*>(wr + c);
      const float4 b = *reinterpret_cast<const float4*>(pr + c);
      const float4 d = *reinterpret_cast<const float4*>(tr + c);
      sum += (a.x + b.x + d.x) + (a.y + b.y + d.y) + (a.z + b.z + d.z) + (a.w + b.w + d.w);
    }
    const float mu = warp_sum(sum) * inv_h;
    float sq = 0.f;
    for (int c = lane * 4; c < H; c += 128) {
      const float4 a = *reinterpret_cast<const float4*>(wr + c);
      const float4 b = *reinterpret_cast<const float4*>(pr + c);
      const float4 d = *reinterpret_cast<const float4*>(tr + c);
      const float e0 = a.x + b.x + d.x - mu, e1 = a.y + b.y + d.y - mu;
      const float e2 = a.z + b.z + d.z - mu, e3 = a.w + b.w + d.w - mu;
      sq += e0 * e0 + e1 * e1 + e2 * e2 + e3 * e3;
    }
    const float rs = rsqrtf(warp_sum(sq) * inv_h + eps);
    if (lane == 0) {
      mean_out[row] = mu;
      rstd_out[row] = rs;
    }
    __nv_bfloat16* orow = out + static_cast<long long>(row) * H;
    for (int c = lane * 4; c < H; c += 128) {
      const float4 a = *reinterpret_cast<const float4*>(wr + c);
      const float4 b = *reinterpret_cast<const float4*>(pr + c);
      const float4 d = *reinterpret_cast<const float4*>(tr + c);
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
      float o0 = (a.x + b.x + d.x - mu) * rs * g.x + be.x;
      float o1 = (a.y + b.y + d.y - mu) * rs * g.y + be.y;
      float o2 = (a.z + b.z + d.z - mu) * rs * g.z + be.z;
      float o3 = (a.w + b.w + d.w - mu) * rs * g.w + be.w;
      if (drop.on) {
        const uint32_t m =
            dropout_keep4(drop.seed, (static_cast<uint64_t>(row) * H + c) >> 2, drop.thr16);
        o0 = (m & 1u) ? o0 * drop.scale : 0.f;
        o1 = (m & 2u) ? o1 * drop.scale : 0.f;
        o2 = (m & 4u) ? o2 * drop.scale : 0.f;
        o3 = (m & 8u) ? o3 * drop.scale : 0.f;
      }
      uint2 pk;
      pk.x = pack_bf16x2(o0, o1);
      pk.y = pack_bf16x2(o2, o3);
      *reinterpret_cast<uint2*>(orow + c) = pk;
    }
  }
}

// backward: recompute xhat from the tables, LN backward, scatter-add into the fp32 grad tables.
__global__ void __launch_bounds__(256)
embed_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const int64_t* __restrict__ ids,
                 const int64_t* __restrict__ tts, const float* __restrict__ word,
                 const float* __restrict__ pos, const float* __restrict__ type,
                 const float* __restrict__ gamma, const float* __restrict__ mean,
                 const float* __restrict__ rstd, float* __restrict__ dword,
                 float* __restrict__ dpos, float* __restrict__ dtype_, float* __restrict__ dgamma,
                 float* __restrict__ dbeta, int BS, int S, int H, float dropout_p,
                 const uint64_t* rng_state, uint32_t rng_stream, const uint32_t* wait_flags,
                 const uint32_t* wait_epoch, uint32_t wait_mult, int* error_flag,
                 int type_rows_in_smem) {
  // Heavily shared targets (LayerNorm gamma/beta: every row; token-type rows: ~half of all
  // rows each) are accumulated in shared memory and flushed once per CTA; the first version
  // issued one global atomic per element and spent 400 us serialising on ~4K addresses.
  extern __shared__ float acc_smem[];  // [dgamma H][dbeta H][dtype type_rows_in_smem * H]
  float* s_dgamma = acc_smem;
  float* s_dbeta = acc_smem + H;
  float* s_dtype = acc_smem + 2 * H;
  for (int i = threadIdx.x; i < (2 + type_rows_in_smem) * H; i += blockDim.x) acc_smem[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int row0 = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int total_warps = gridDim.x * warps_per_block;
  const float inv_h = 1.f / static_cast<float>(H);
  const Dropout drop = dropout_of(dropout_p, rng_state, rng_stream);
  const uint32_t target = wait_flags ? (*wait_epoch) * wait_mult : 0u;
  int last_panel = -1;
  for (int row = row0; row < BS; row += total_warps) {
    if (wait_flags != nullptr) {
      const int panel = row >> 7;
      if (panel != last_panel) {
        warp_wait_panel(wait_flags, panel, target, error_flag, lane);
        last_panel = panel;
      }
    }
    const long long id = ids[row];
    const long long tt = tts[row];
    const int s = row % S;
    const float mu = mean[row], rs = rstd[row];
    const float* wr = word + id * H;
    const float* pr = pos + static_cast<long long>(s) * H;
    const float* tr = type + tt * H;
    const __nv_bfloat16* drow = dout + static_cast<long long>(row) * H;
    float s1 = 0.f, s2 = 0.f;
    // pass 1: row statistics of g = dy*gamma
    for (int c = lane * 4; c < H; c += 128) {
      const uint2 u = *reinterpret_cast<const uint2*>(drow + c);
      float2 d01 = unpack_bf16x2(u.x), d23 = unpack_bf16x2(u.y);
      float dy[4] = {d01.x, d01.y, d23.x, d23.y};
      if (drop.on) {
        const uint32_t m =
            dropout_keep4(drop.seed, (static_cast<uint64_t>(row) * H + c) >> 2, drop.thr16);
#pragma unroll
        for (int t = 0; t < 4; ++t) dy[t] = (m >> t) & 1u ? dy[t] * drop.scale : 0.f;
      }
      const float4 a = *reinterpret_cast<const float4*>(wr + c);
      const float4 b = *reinterpret_cast<const float4*>(pr + c);
      const float4 d = *reinterpret_cast<const float4*>(tr + c);
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float e[4] = {a.x + b.x + d.x, a.y + b.y + d.y, a.z + b.z + d.z, a.w + b.w + d.w};
      const float gm[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float xh = (e[t] - mu) * rs;
        const float q = dy[t] * gm[t];
        s1 += q;
        s2 += q * xh;
        atomicAdd(&s_dgamma[c + t], dy[t] * xh);
        atomicAdd(&s_dbeta[c + t], dy[t]);
      }
    }
    const float c1 = warp_sum(s1) * inv_h;
    const float c2 = warp_sum(s2) * inv_h;
    for (int c = lane * 4; c < H; c += 128) {
      const uint2 u = *reinterpret_cast<const uint2*>(drow + c);
      float2 d01 = unpack_bf16x2(u.x), d23 = unpack_bf16x2(u.y);
      float dy[4] = {d01.x, d01.y, d23.x, d23.y};
      if (drop.on) {
        const uint32_t m =
            dropout_keep4(drop.seed, (static_cast<uint64_t>(row) * H + c) >> 2, drop.thr16);
#pragma unroll
        for (int t = 0; t < 4; ++t) dy[t] = (m >> t) & 1u ? dy[t] * drop.scale : 0.f;
      }
      const float4 a = *reinterpret_cast<const float4*>(wr + c);
      const float4 b = *reinterpret_cast<const float4*>(pr + c);
      const float4 d = *reinterpret_cast<const float4*>(tr + c);
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float e[4] = {a.x + b.x + d.x, a.y + b.y + d.y, a.z + b.z + d.z, a.w + b.w + d.w};
      const float gm[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float xh = (e[t] - mu) * rs;
        const float de = (dy[t] * gm[t] - c1 - xh * c2) * rs;
        atomicAdd(&dword[id * H + c + t], de);
        atomicAdd(&dpos[static_cast<long long>(s) * H + c + t], de);
        if (tt < type_rows_in_smem)
          atomicAdd(&s_dtype[tt * H + c + t], de);
        else
          atomicAdd(&dtype_[tt * H + c + t], de);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    atomicAdd(&dgamma[i], s_dgamma[i]);
    atomicAdd(&dbeta[i], s_dbeta[i]);
  }
  for (int i = threadIdx.x; i < type_rows_in_smem * H; i += blockDim.x)
    atomicAdd(&dtype_[i], s_dtype[i]);
}

// ------------------------------------------------------------------------------------------
// Small dense layers (pooler, classifier): one warp per output column n, looping over rows.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_x(const void* x, bool x_bf16, long long idx) {
  return x_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[idx])
                : reinterpret_cast<const float*>(x)[idx];
}
__device__ __forceinline__ float drop1(uint64_t seed, uint64_t idx, uint32_t thr16, float scale,
                                       float v) {
  const uint32_t m = dropout_keep4(seed, idx >> 2, thr16);
  return ((m >> (idx & 3)) & 1u) ? v * scale : 0.f;
}

__global__ void __launch_bounds__(128)
small_linear_fwd_kernel(const void* __restrict__ x, bool x_bf16, long long ldx,
                        const float* __restrict__ w, const float* __restrict__ b,
                        float* __restrict__ y, int M, int N, int K, int act_tanh, float dropout_p,
                        const uint64_t* rng_state, uint32_t rng_stream) {
  // one warp per output element (m, n): lanes stride the reduction dimension
  const int lane = threadIdx.x & 31;
  const long long o = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (o >= static_cast<long long>(M) * N) return;
  const int m = static_cast<int>(o / N), n = static_cast<int>(o % N);
  const Dropout drop = dropout_of(dropout_p, rng_state, rng_stream);
  const float* wr = w + static_cast<long long>(n) * K;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) {
    float xv = load_x(x, x_bf16, m * ldx + k);
    if (drop.on)
      xv = drop1(drop.seed, static_cast<uint64_t>(m) * K + k, drop.thr16, drop.scale, xv);
    acc += xv * wr[k];
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    float v = acc + (b ? b[n] : 0.f);
    if (act_tanh) v = tanhf(v);
    y[o] = v;
  }
}

// dx[m,k] = sum_n dy'[m,n] w[n,k]; one thread per k, 8 rows at a time.
__global__ void __launch_bounds__(128)
small_linear_dx_kernel(const float* __restrict__ w, const float* __restrict__ y,
                       const float* __restrict__ dy, void* __restrict__ dx, bool dx_bf16,
                       long long lddx, int M, int N, int K, int act_tanh, float dropout_p,
                       const uint64_t* rng_state, uint32_t rng_stream) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int m0 = blockIdx.y * 8;
  if (k >= K) return;
  const Dropout drop = dropout_of(dropout_p, rng_state, rng_stream);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int n = 0; n < N; ++n) {
    const float wv = w[static_cast<long long>(n) * K + k];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + i;
      if (m < M) {
        float g = dy[static_cast<long long>(m) * N + n];
        if (act_tanh) {
          const float yv = y[static_cast<long long>(m) * N + n];
          g *= (1.f - yv * yv);
        }
        acc[i] += g * wv;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + i;
    if (m < M) {
      float v = acc[i];
      if (drop.on)
        v = drop1(drop.seed, static_cast<uint64_t>(m) * K + k, drop.thr16, drop.scale, v);
      if (dx_bf16)
        reinterpret_cast<__nv_bfloat16*>(dx)[m * lddx + k] = __float2bfloat16(v);
      else
        reinterpret_cast<float*>(dx)[m * lddx + k] = v;
    }
  }
}

// dw[n,k] += sum_m dy'[m,n] x[m,k];  db[n] += sum_m dy'[m,n]
__global__ void __launch_bounds__(128)
small_linear_dw_kernel(const void* __restrict__ x, bool x_bf16, long long ldx,
                       const float* __restrict__ y, const float* __restrict__ dy,
                       float* __restrict__ dw, float* __restrict__ db, int M, int N, int K,
                       int act_tanh, float dropout_p, const uint64_t* rng_state,
                       uint32_t rng_stream) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  const Dropout drop = dropout_of(dropout_p, rng_state, rng_stream);
  float acc = 0.f, accb = 0.f;
  for (int m = 0; m < M; ++m) {
    float g = dy[static_cast<long long>(m) * N + n];
    if (act_tanh) {
      const float yv = y[static_cast<long long>(m) * N + n];
      g *= (1.f - yv * yv);
    }
    accb += g;
    if (k < K) {
      float xv = load_x(x, x_bf16, m * ldx + k);
      if (drop.on)
        xv = drop1(drop.seed, static_cast<uint64_t>(m) * K + k, drop.thr16, drop.scale, xv);
      acc += g * xv;
    }
  }
  if (k < K) dw[static_cast<long long>(n) * K + k] += acc;
  if (db != nullptr && k == 0) db[n] += accb;
}

// ------------------------------------------------------------------------------------------
// Softmax cross entropy over rows of a few fp32 classes: the classification, next-sentence and
// span losses (launch_softmax_ce).  One CTA: its threads first count each group's labelled rows
// and the invalid labels (integer atomics: the counts do not depend on the order), then warp w
// owns rows w, w + 16, ... of each kCeChunk-row chunk and its lanes stride over the classes.
// A row's max and exp-sum are reduced with one fixed xor pattern, the rows' CE / n_g go into an
// fp64 chunk summed by a fixed tree, and thread 0 adds the chunk sums in chunk order.  An
// invalid label is never used as an index.  No float atomics, no host sync: graph replays are
// bit-identical.
// ------------------------------------------------------------------------------------------
constexpr int kCeWarps = 16;
constexpr int kCeChunk = 256;  // rows per fixed-order fp64 reduction chunk

// sums[0..n_arr) of the chunk's per-row values, a fixed tree over kCeChunk entries each
__device__ __forceinline__ void chunk_tree(double (*vals)[kCeChunk], int n_arr) {
  for (int s = kCeChunk / 2; s > 0; s >>= 1) {
    for (int i = threadIdx.x; i < n_arr * s; i += blockDim.x) {
      const int a = i / s, j = i - a * s;
      vals[a][j] += vals[a][j + s];
    }
    __syncthreads();
  }
}

// row r = item r / G, group r % G; G is a template parameter so that both are shifts
template <int G>
__global__ void __launch_bounds__(kCeWarps * 32)
softmax_ce_kernel(const float* __restrict__ logits, int ldl, const int64_t* __restrict__ labels,
                  int label_ld, int N, int C, long long ignore_index, float* __restrict__ dlogits,
                  float grad_scale, float* __restrict__ loss, float* __restrict__ loss_acc) {
  __shared__ double row_loss[1][kCeChunk];
  __shared__ int cnt[3];  // labelled rows of group 0, of group 1; invalid labels
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int R = N * G;
  if (threadIdx.x < 3) cnt[threadIdx.x] = 0;
  __syncthreads();
  int n0 = 0, n1 = 0, nbad = 0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const int g = r % G;
    const long long lab = labels[static_cast<long long>(r / G) * label_ld + g];
    if (lab == ignore_index) continue;
    if (lab < 0 || lab >= C) ++nbad;
    else if (g) ++n1;
    else ++n0;
  }
  if (n0) atomicAdd(&cnt[0], n0);
  if (n1) atomicAdd(&cnt[1], n1);
  if (nbad) atomicAdd(&cnt[2], nbad);
  __syncthreads();
  n0 = cnt[0];
  n1 = cnt[1];
  const float scale0 = n0 > 0 ? grad_scale / (G * static_cast<float>(n0)) : 0.f;
  const float scale1 = n1 > 0 ? grad_scale / (G * static_cast<float>(n1)) : 0.f;
  double total = 0.0;
  for (int base = 0; base < R; base += kCeChunk) {
    for (int rr = warp; rr < kCeChunk; rr += kCeWarps) {
      const int r = base + rr;
      double contrib = 0.0;
      if (r < R) {
        const int g = r % G;
        const float* l = logits + static_cast<long long>(r) * ldl;
        float* d = dlogits + static_cast<long long>(r) * C;
        const long long lab = labels[static_cast<long long>(r / G) * label_ld + g];
        if (lab == ignore_index || lab < 0 || lab >= C) {
          for (int c = lane; c < C; c += 32) d[c] = 0.f;
        } else {
          float mx = -INFINITY;
          for (int c = lane; c < C; c += 32) mx = fmaxf(mx, l[c]);
          mx = warp_max(mx);
          float se = 0.f;
          for (int c = lane; c < C; c += 32) se += expf(l[c] - mx);
          se = warp_sum(se);
          const float lse = mx + logf(se);
          const float sc = g ? scale1 : scale0;
          for (int c = lane; c < C; c += 32)
            d[c] = (expf(l[c] - lse) - (c == lab ? 1.f : 0.f)) * sc;
          contrib = static_cast<double>(lse - l[lab]) / (g ? n1 : n0);
        }
      }
      if (lane == 0) row_loss[0][rr] = contrib;
    }
    __syncthreads();
    chunk_tree(row_loss, 1);
    if (threadIdx.x == 0) total += row_loss[0][0];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float mean = static_cast<float>(total / G);
    if (cnt[2] > 0) mean = __int_as_float(0x7fc00000);  // NaN: an invalid label is never silent
    if (loss != nullptr) loss[0] = mean;
    // micro-batched training: the step loss is the sum of the scaled micro-batch losses
    if (loss_acc != nullptr) loss_acc[0] += mean * grad_scale;
  }
}

// Evaluation: per-row cross entropy + argmax of one batch of logits, added into an EvalAccum.
// One CTA of 16 warps; warp w owns rows w, w + 16, ... of each 512-row chunk, its lanes stride
// over the classes.  The row max / argmax and the exp-sum are reduced with one fixed xor pattern,
// the chunk's row losses are summed in a fixed fp64 tree and the chunk sums are added in chunk
// order by thread 0, so the result does not depend on scheduling (graph replays are bit-equal).
constexpr int kEvalWarps = 16;
constexpr int kEvalChunk = 512;

// (a, ia) is a better argmax candidate than (b, ib): NaN beats everything, then larger, then the
// smaller index (torch.argmax: the first maximum wins, a NaN counts as the maximum)
__device__ __forceinline__ bool eval_better(float a, int ia, float b, int ib) {
  const bool na = a != a, nb = b != b;
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

// argmax (eval_better) and lse = max + log(sum exp(l - max)) of one row of C > 0 classes,
// warp-wide: lanes stride over the classes, one fixed xor pattern reduces them
__device__ __forceinline__ void warp_row_stats(const float* __restrict__ l, int C, int lane,
                                               int* arg_out, float* lse_out) {
  float mx = -INFINITY;
  int arg = C;  // no candidate yet (C > 0: every row has one after the reduction)
  for (int c = lane; c < C; c += 32) {
    const float v = l[c];
    if (arg == C || eval_better(v, c, mx, arg)) {
      mx = v;
      arg = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float omx = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oarg = __shfl_xor_sync(0xffffffffu, arg, o);
    if (oarg < C && (arg == C || eval_better(omx, oarg, mx, arg))) {
      mx = omx;
      arg = oarg;
    }
  }
  float se = 0.f;
  for (int c = lane; c < C; c += 32) se += expf(l[c] - mx);
  se = warp_sum(se);
  *arg_out = arg;
  *lse_out = mx + logf(se);
}

__global__ void __launch_bounds__(kEvalWarps * 32)
classify_eval_kernel(const float* __restrict__ logits, long long ldl,
                     const int64_t* __restrict__ labels, int M, int C, long long ignore_index,
                     EvalAccum* __restrict__ acc) {
  __shared__ double row_loss[kEvalChunk];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long counted = 0, invalid = 0;
  double total = 0.0;
  for (int base = 0; base < M; base += kEvalChunk) {
    for (int r = warp; r < kEvalChunk; r += kEvalWarps) {
      const int m = base + r;
      double contrib = 0.0;
      if (m < M) {
        const float* l = logits + static_cast<long long>(m) * ldl;
        int arg;
        float lse;
        warp_row_stats(l, C, lane, &arg, &lse);
        const long long lab = labels[m];
        if (lab != ignore_index) {
          if (lab < 0 || lab >= C) {
            ++invalid;
          } else {
            const float loss = lse - l[lab];
            contrib = static_cast<double>(loss);
            ++counted;
            if (lane == 0) atomicAdd(&acc->confusion[lab * C + arg], 1ull);
          }
        }
      }
      if (lane == 0) row_loss[r] = contrib;
    }
    __syncthreads();
    for (int s = kEvalChunk / 2; s > 0; s >>= 1) {
      for (int i = threadIdx.x; i < s; i += blockDim.x) row_loss[i] += row_loss[i + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) total += row_loss[0];
    __syncthreads();
  }
  if (lane == 0) {
    if (counted) atomicAdd(&acc->count, counted);
    if (invalid) atomicAdd(&acc->invalid, invalid);
  }
  if (threadIdx.x == 0) acc->loss_sum += total;
}

// ------------------------------------------------------------------------------------------
// Vocabulary cross entropy over bf16 logits [M, V] (masked-language-model loss).
//   vocab_ce_count_kernel     1 CTA: n_valid = #labels != ignore_index (training mode only)
//   vocab_ce_row_kernel       1 CTA per row: the row is read from HBM once into shared memory,
//                             max (argmax) / exp-sum / loss from there, and in training mode the
//                             bf16 gradient is written from the shared copy (may alias the logits)
//   vocab_ce_finalize_kernel  1 CTA: the per-row results summed in a fixed order (fp64), added
//                             into loss_acc (training) or the VocabEvalAccum (eval)
// Rows whose label is ignore_index are not read at all.  No float atomics anywhere: graph replays
// are bit-identical.
// ------------------------------------------------------------------------------------------
constexpr int kVceThreads = 512;
constexpr int kVceWarps = kVceThreads / 32;
constexpr int kVceFinThreads = 1024;
enum : int { kVceCounted = 1, kVceCorrect = 2, kVceInvalid = 4 };

__global__ void __launch_bounds__(kVceFinThreads)
vocab_ce_count_kernel(const int64_t* __restrict__ labels, int M, long long ignore_index,
                      int* __restrict__ n_valid) {
  __shared__ int red[kVceFinThreads / 32];
  int n = 0;
  for (int m = threadIdx.x; m < M; m += blockDim.x) n += labels[m] != ignore_index ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kVceFinThreads / 32; ++w) t += red[w];
    *n_valid = t;
  }
}

__device__ __forceinline__ float bf16_at(uint4 v, int j) {
  const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
  return __bfloat162float(h[j]);
}

// kEval: argmax + counters, no gradient.  kVec: the row start is 16-byte aligned (16 B loads /
// stores for the first V/8*8 columns, scalar tail); otherwise every access is scalar.
template <bool kEval, bool kVec>
__global__ void __launch_bounds__(kVceThreads)
vocab_ce_row_kernel(const __nv_bfloat16* logits, long long ldl, const int64_t* __restrict__ labels,
                    int V, long long ignore_index, __nv_bfloat16* dlogits, float grad_scale,
                    const int* __restrict__ n_valid, double* __restrict__ row_loss,
                    int* __restrict__ row_flags) {
  extern __shared__ __align__(16) unsigned char vce_smem[];
  __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(vce_smem);
  __shared__ float red_v[kVceWarps];
  __shared__ int red_i[kVceWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long m = blockIdx.x;
  const long long lab = labels[m];
  const __nv_bfloat16* src = logits + m * ldl;
  const int V8 = kVec ? (V / 8) * 8 : 0;

  if (lab == ignore_index) {  // not read; zero gradient, nothing counted
    if (!kEval) {
      __nv_bfloat16* dst = dlogits + m * ldl;
      for (int c = tid * 8; c < V8; c += kVceThreads * 8)
        *reinterpret_cast<uint4*>(dst + c) = make_uint4(0, 0, 0, 0);
      for (int c = V8 + tid; c < V; c += kVceThreads) dst[c] = __float2bfloat16(0.f);
    }
    if (tid == 0) {
      row_loss[m] = 0.0;
      row_flags[m] = 0;
    }
    return;
  }

  // pass 1: HBM -> shared memory, thread-local max (eval: argmax candidate as in classify_eval)
  float mx = -INFINITY;
  int arg = V;  // no candidate yet
  auto take = [&](float v, int c) {
    if (kEval) {
      if (arg == V || eval_better(v, c, mx, arg)) {
        mx = v;
        arg = c;
      }
    } else {
      mx = fmaxf(mx, v);
    }
  };
  for (int c = tid * 8; c < V8; c += kVceThreads * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + c);
    *reinterpret_cast<uint4*>(row + c) = v;
#pragma unroll
    for (int j = 0; j < 8; ++j) take(bf16_at(v, j), c + j);
  }
  for (int c = V8 + tid; c < V; c += kVceThreads) {
    const __nv_bfloat16 v = src[c];
    row[c] = v;
    take(__bfloat162float(v), c);
  }
  // block max / argmax: fixed xor pattern, then the warps' results in warp order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float omx = __shfl_xor_sync(0xffffffffu, mx, o);
    if (kEval) {
      const int oarg = __shfl_xor_sync(0xffffffffu, arg, o);
      if (oarg < V && (arg == V || eval_better(omx, oarg, mx, arg))) {
        mx = omx;
        arg = oarg;
      }
    } else {
      mx = fmaxf(mx, omx);
    }
  }
  if (lane == 0) {
    red_v[warp] = mx;
    red_i[warp] = arg;
  }
  __syncthreads();  // also publishes the shared row
  mx = red_v[0];
  arg = red_i[0];
  for (int w = 1; w < kVceWarps; ++w) {
    if (kEval) {
      if (red_i[w] < V && (arg == V || eval_better(red_v[w], red_i[w], mx, arg))) {
        mx = red_v[w];
        arg = red_i[w];
      }
    } else {
      mx = fmaxf(mx, red_v[w]);
    }
  }
  __syncthreads();  // red_v is reused below

  // pass 2: sum exp(l - max) from shared memory
  const int V8s = (V / 8) * 8;  // the shared row is always 16-byte aligned
  float se = 0.f;
  for (int c = tid * 8; c < V8s; c += kVceThreads * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(row + c);
#pragma unroll
    for (int j = 0; j < 8; ++j) se += __expf(bf16_at(v, j) - mx);
  }
  for (int c = V8s + tid; c < V; c += kVceThreads) se += __expf(__bfloat162float(row[c]) - mx);
  se = warp_sum(se);
  if (lane == 0) red_v[warp] = se;
  __syncthreads();
  se = 0.f;
  for (int w = 0; w < kVceWarps; ++w) se += red_v[w];
  const float lse = mx + logf(se);
  const bool valid = lab >= 0 && lab < V;

  if (!kEval) {
    // dlogits = (softmax - onehot) * grad_scale / n_valid; an out-of-range label (neither
    // ignore_index nor in [0, V)) gets a zero gradient and a NaN loss
    const int nv = *n_valid;
    const float coef = valid ? grad_scale / static_cast<float>(nv) : 0.f;
    __nv_bfloat16* dst = dlogits + m * ldl;
    for (int c = tid * 8; c < V8; c += kVceThreads * 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(row + c);
      uint4 o;
      __nv_bfloat16* oh = reinterpret_cast<__nv_bfloat16*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p = __expf(bf16_at(v, j) - lse) - (c + j == lab ? 1.f : 0.f);
        oh[j] = __float2bfloat16(p * coef);
      }
      *reinterpret_cast<uint4*>(dst + c) = o;
    }
    for (int c = V8 + tid; c < V; c += kVceThreads) {
      const float p = __expf(__bfloat162float(row[c]) - lse) - (c == lab ? 1.f : 0.f);
      dst[c] = __float2bfloat16(p * coef);
    }
  }
  if (tid == 0) {
    if (valid) {
      row_loss[m] = static_cast<double>(lse - __bfloat162float(row[lab]));
      row_flags[m] = kVceCounted | (kEval && arg == lab ? kVceCorrect : 0);
    } else {
      row_loss[m] = kEval ? 0.0 : static_cast<double>(NAN);
      row_flags[m] = kVceInvalid;
    }
  }
}

__global__ void __launch_bounds__(kVceFinThreads)
vocab_ce_finalize_kernel(const double* __restrict__ row_loss, const int* __restrict__ row_flags,
                         int M, const int* __restrict__ n_valid, float grad_scale,
                         float* __restrict__ loss_out, float* __restrict__ loss_acc,
                         VocabEvalAccum* __restrict__ acc) {
  __shared__ double red[kVceFinThreads];
  __shared__ int cnt[3][kVceFinThreads / 32];
  double s = 0.0;
  int counted = 0, correct = 0, invalid = 0;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    s += row_loss[m];
    const int f = row_flags[m];
    counted += f & kVceCounted ? 1 : 0;
    correct += f & kVceCorrect ? 1 : 0;
    invalid += f & kVceInvalid ? 1 : 0;
  }
  red[threadIdx.x] = s;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    counted += __shfl_xor_sync(0xffffffffu, counted, o);
    correct += __shfl_xor_sync(0xffffffffu, correct, o);
    invalid += __shfl_xor_sync(0xffffffffu, invalid, o);
  }
  if ((threadIdx.x & 31) == 0) {
    cnt[0][threadIdx.x >> 5] = counted;
    cnt[1][threadIdx.x >> 5] = correct;
    cnt[2][threadIdx.x >> 5] = invalid;
  }
  __syncthreads();
  for (int k = kVceFinThreads / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  if (acc != nullptr) {
    unsigned long long c[3] = {0, 0, 0};
    for (int k = 0; k < 3; ++k)
      for (int w = 0; w < kVceFinThreads / 32; ++w) c[k] += cnt[k][w];
    acc->loss_sum += red[0];
    acc->count += c[0];
    acc->correct += c[1];
    acc->invalid += c[2];
  } else {
    // no labelled row: the loss is 0 (torch's mean over an empty selection would be NaN)
    const int nv = *n_valid;
    const float mean = nv > 0 ? static_cast<float>(red[0] / nv) : 0.f;
    if (loss_out != nullptr) loss_out[0] = mean;
    if (loss_acc != nullptr) loss_acc[0] += mean * grad_scale;
  }
}

// ------------------------------------------------------------------------------------------
// Sparse masked-language-model decoding: the rows the head decodes are the labelled positions.
//   mlm_gather_kernel   1 CTA per sequence: scans the S labels in position order (warp ballot +
//                       popc prefix), writes slot_of_row / slot_labels and copies the selected
//                       hidden rows into the slots (zero rows for empty slots)
//   mlm_scatter_kernel  grid-stride over dhidden: row r gets dx_c[slot_of_row[r]] or zeros
// Integer scans and pure copies: bit-identical on every call and replay.
// ------------------------------------------------------------------------------------------
constexpr int kMlmThreads = 256;
constexpr int kMlmWarps = kMlmThreads / 32;

__global__ void __launch_bounds__(kMlmThreads)
mlm_gather_kernel(const uint4* __restrict__ hidden, const int64_t* __restrict__ labels, int S,
                  int H8, int P, long long ignore_index, long long sentinel,
                  int* __restrict__ slot_of_row, int64_t* __restrict__ slot_labels,
                  uint4* __restrict__ x_c) {
  extern __shared__ int mlm_row_of_slot[];  // [P]: position of the slot's labelled token
  __shared__ int warp_cnt[kMlmWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t* lab = labels + static_cast<long long>(b) * S;
  int* sor = slot_of_row + static_cast<long long>(b) * S;
  int n = 0;  // labelled positions in front of the current chunk
  for (int base = 0; base < S; base += kMlmThreads) {
    const int pos = base + tid;
    const bool on = pos < S && lab[pos] != ignore_index;
    const unsigned m = __ballot_sync(0xffffffffu, on);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    int before = 0, chunk = 0;
#pragma unroll
    for (int w = 0; w < kMlmWarps; ++w) {
      before += w < warp ? warp_cnt[w] : 0;
      chunk += warp_cnt[w];
    }
    const int rank = n + before + __popc(m & ((1u << lane) - 1u));
    if (pos < S) {
      const bool kept = on && rank < P;
      sor[pos] = kept ? b * P + rank : -1;
      if (kept) mlm_row_of_slot[rank] = pos;
    }
    n += chunk;
    __syncthreads();  // warp_cnt is rewritten by the next chunk; the slot map is read below
  }
  const int filled = n < P ? n : P;
  int64_t* sl = slot_labels + static_cast<long long>(b) * P;
  for (int r = tid; r < P; r += kMlmThreads) {
    long long v = r < filled ? lab[mlm_row_of_slot[r]] : ignore_index;
    if (n > P && r == P - 1) v = sentinel;  // overflow: never silent
    sl[r] = v;
  }
  const long long src0 = static_cast<long long>(b) * S;
  uint4* dst = x_c + static_cast<long long>(b) * P * H8;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (int i = tid; i < P * H8; i += kMlmThreads) {
    const int r = i / H8, c = i - r * H8;
    dst[i] = r < filled ? hidden[(src0 + mlm_row_of_slot[r]) * H8 + c] : zero;
  }
}

// 8 bf16 lanes of a + b, each sum rounded once from fp32
__device__ __forceinline__ uint4 bf16x8_add(uint4 a, uint4 b) {
  const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
  const __nv_bfloat162* pb = reinterpret_cast<const __nv_bfloat162*>(&b);
  uint4 out;
  __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&out);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fa = __bfloat1622float2(pa[j]), fb = __bfloat1622float2(pb[j]);
    po[j] = __floats2bfloat162_rn(fa.x + fb.x, fa.y + fb.y);
  }
  return out;
}

// kCls: row b*S (a sequence's [CLS] position) also gets dcls[b], the pooler's input gradient, so
// that the input gradient of a head with a pooler branch is written once
template <bool kCls>
__global__ void __launch_bounds__(kMlmThreads)
mlm_scatter_kernel(const uint4* __restrict__ dx_c, const int* __restrict__ slot_of_row,
                   long long rows, int H8, uint4* __restrict__ dhidden,
                   const uint4* __restrict__ dcls, int S) {
  const long long total = rows * H8;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / H8;
    const int s = slot_of_row[r];
    uint4 v = s >= 0 ? dx_c[static_cast<long long>(s) * H8 + (i - r * H8)] : zero;
    if (kCls && r % S == 0) {
      const uint4 c = dcls[(r / S) * H8 + (i - r * H8)];
      v = s >= 0 ? bf16x8_add(v, c) : c;
    }
    dhidden[i] = v;
  }
}

// dhidden[b*S] += dcls[b] in place: the dense head's [CLS]-row join
__global__ void __launch_bounds__(kMlmThreads)
cls_grad_add_kernel(uint4* __restrict__ dhidden, const uint4* __restrict__ dcls, int B, int S,
                    int H8) {
  const long long total = static_cast<long long>(B) * H8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / H8;
    uint4* p = dhidden + b * S * H8 + (i - b * H8);
    *p = bf16x8_add(*p, dcls[i]);
  }
}

// ------------------------------------------------------------------------------------------
// Question-answering span head (HF BertForQuestionAnswering: qa_outputs = Linear(H, 2)).
//   qa_logits_fwd_kernel       one warp per row: the bf16 row (16-byte loads) dotted with w[0]
//                              and w[1] in fp32, plus the bias, stored as logits [B, 2, S]
//   qa_logits_bwd_kernel       CTA (x, y) owns 256 columns of rows [y * 128, (y + 1) * 128):
//                              dhidden = g0 w0 + g1 w1 (bf16, every row written once) and that
//                              row range's partial dW [2, H] / db [2]
//   qa_logits_finalize_kernel  the partials summed in row-block order (fp64), added into dW / db
//   qa_span_eval_kernel        one CTA: best span per row, totals, predictions at a device cursor
// The span loss is softmax_ce_kernel over the 2B rows, start and end as two groups.
// Warp reductions use one fixed xor pattern and every float sum a fixed order, no float atomics:
// two calls or graph replays give identical bits.
// ------------------------------------------------------------------------------------------
constexpr int kQaFwdWarps = 8;
constexpr int kQaColChunks = 32;  // bwd CTA: 32 x 8 threads, 32 16-byte chunks = 256 columns
constexpr int kQaRowLanes = 8;
constexpr int kQaRowUnroll = 4;   // rows a bwd thread loads before it computes

__device__ __forceinline__ void unpack_bf16x8(const uint4& u, float* x) {
  const float2 f0 = unpack_bf16x2(u.x), f1 = unpack_bf16x2(u.y);
  const float2 f2 = unpack_bf16x2(u.z), f3 = unpack_bf16x2(u.w);
  x[0] = f0.x;
  x[1] = f0.y;
  x[2] = f1.x;
  x[3] = f1.y;
  x[4] = f2.x;
  x[5] = f2.y;
  x[6] = f3.x;
  x[7] = f3.y;
}

__global__ void __launch_bounds__(kQaFwdWarps * 32)
qa_logits_fwd_kernel(const uint4* __restrict__ hidden, long long R, int S, int H8,
                     const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ logits) {
  const int lane = threadIdx.x & 31;
  const long long H = static_cast<long long>(H8) * 8;
  const float b0 = bias[0], b1 = bias[1];
  for (long long r = static_cast<long long>(blockIdx.x) * kQaFwdWarps + (threadIdx.x >> 5); r < R;
       r += static_cast<long long>(gridDim.x) * kQaFwdWarps) {
    const uint4* x = hidden + r * H8;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 2
    for (int v = lane; v < H8; v += 32) {
      float xf[8];
      unpack_bf16x8(x[v], xf);
      const float4* w0 = reinterpret_cast<const float4*>(w + v * 8);
      const float4* w1 = reinterpret_cast<const float4*>(w + H + v * 8);
      const float4 a0 = w0[0], a1 = w0[1], c0 = w1[0], c1 = w1[1];
      s0 += xf[0] * a0.x + xf[1] * a0.y + xf[2] * a0.z + xf[3] * a0.w +
            xf[4] * a1.x + xf[5] * a1.y + xf[6] * a1.z + xf[7] * a1.w;
      s1 += xf[0] * c0.x + xf[1] * c0.y + xf[2] * c0.z + xf[3] * c0.w +
            xf[4] * c1.x + xf[5] * c1.y + xf[6] * c1.z + xf[7] * c1.w;
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    if (lane == 0) {
      const long long b = r / S, s = r - b * S;
      logits[b * 2 * S + s] = s0 + b0;
      logits[b * 2 * S + S + s] = s1 + b1;
    }
  }
}

__global__ void __launch_bounds__(kQaColChunks * kQaRowLanes)
qa_logits_bwd_kernel(const uint4* __restrict__ hidden, const float* __restrict__ g, long long R,
                     int S, int H8, const float* __restrict__ w, uint4* __restrict__ dhidden,
                     float* __restrict__ partial) {
  __shared__ float red[kQaRowLanes][16][kQaColChunks];
  __shared__ float redb[kQaRowLanes][2];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c8 = blockIdx.x * kQaColChunks + tx;
  const bool col_ok = c8 < H8;
  const long long H = static_cast<long long>(H8) * 8;
  float w0[8], w1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    w0[i] = col_ok ? w[c8 * 8 + i] : 0.f;
    w1[i] = col_ok ? w[H + c8 * 8 + i] : 0.f;
  }
  float a0[8], a1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a0[i] = a1[i] = 0.f;
  float gb0 = 0.f, gb1 = 0.f;
  const long long r0 = static_cast<long long>(blockIdx.y) * kQaRowsPerCta;
  const long long r1 = r0 + kQaRowsPerCta < R ? r0 + kQaRowsPerCta : R;
  for (long long rb = r0 + ty; rb < r1; rb += kQaRowLanes * kQaRowUnroll) {
    uint4 u[kQaRowUnroll];
    float g0[kQaRowUnroll], g1[kQaRowUnroll];
#pragma unroll
    for (int k = 0; k < kQaRowUnroll; ++k) {
      const long long r = rb + k * kQaRowLanes;
      g0[k] = g1[k] = 0.f;
      u[k] = make_uint4(0u, 0u, 0u, 0u);
      if (r < r1) {
        const long long b = r / S, s = r - b * S;
        g0[k] = g[b * 2 * S + s];
        g1[k] = g[b * 2 * S + S + s];
        if (col_ok) u[k] = hidden[r * H8 + c8];
      }
    }
#pragma unroll
    for (int k = 0; k < kQaRowUnroll; ++k) {
      const long long r = rb + k * kQaRowLanes;
      if (r >= r1) continue;
      gb0 += g0[k];
      gb1 += g1[k];
      if (!col_ok) continue;
      float x[8], d[8];
      unpack_bf16x8(u[k], x);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        a0[i] = fmaf(g0[k], x[i], a0[i]);
        a1[i] = fmaf(g1[k], x[i], a1[i]);
        // g0 w0 + g1 w1 with the first product's rounding error added back, so that the one
        // rounding to bf16 is the only one that matters even when the two terms cancel
        const float p = __fmul_rn(g0[k], w0[i]);
        const float e = __fmaf_rn(g0[k], w0[i], -p);
        d[i] = __fadd_rn(__fmaf_rn(g1[k], w1[i], p), e);
      }
      dhidden[r * H8 + c8] = make_uint4(pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]),
                                        pack_bf16x2(d[4], d[5]), pack_bf16x2(d[6], d[7]));
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red[ty][i][tx] = a0[i];
    red[ty][8 + i][tx] = a1[i];
  }
  if (tx == 0) {
    redb[ty][0] = gb0;
    redb[ty][1] = gb1;
  }
  __syncthreads();
  float* out = partial + static_cast<long long>(blockIdx.y) * (2 * H + 2);
  for (int i = ty * kQaColChunks + tx; i < 16 * kQaColChunks; i += kQaColChunks * kQaRowLanes) {
    const int k = i / kQaColChunks, t = i - k * kQaColChunks;
    float s = 0.f;
#pragma unroll
    for (int y = 0; y < kQaRowLanes; ++y) s += red[y][k][t];
    const int cc = blockIdx.x * kQaColChunks + t;
    if (cc < H8) out[(k / 8) * H + cc * 8 + (k % 8)] = s;
  }
  if (blockIdx.x == 0 && ty == 0 && tx < 2) {
    float s = 0.f;
#pragma unroll
    for (int y = 0; y < kQaRowLanes; ++y) s += redb[y][tx];
    out[2 * H + tx] = s;
  }
}

// column i of the partials [n_blocks, n]: lane y of a 32 x 8 CTA sums blocks y, y + 8, ... in
// order, then the 8 lane sums are added in lane order
__global__ void __launch_bounds__(kQaColChunks * kQaRowLanes)
qa_logits_finalize_kernel(const float* __restrict__ partial, int n_blocks, int H,
                          float* __restrict__ dw, float* __restrict__ db) {
  __shared__ double red[kQaRowLanes][kQaColChunks];
  const int n = 2 * H + 2;
  const int i = blockIdx.x * kQaColChunks + threadIdx.x;
  double s = 0.0;
  if (i < n) {
#pragma unroll 4
    for (int k = threadIdx.y; k < n_blocks; k += kQaRowLanes)
      s += static_cast<double>(partial[static_cast<long long>(k) * n + i]);
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && i < n) {
    double t = 0.0;
#pragma unroll
    for (int y = 0; y < kQaRowLanes; ++y) t += red[y][threadIdx.x];
    if (i < 2 * H) dw[i] += static_cast<float>(t);
    else db[i - 2 * H] += static_cast<float>(t);
  }
}

// (v, i, j) is a better span than (w, k, l): a higher score, then the smaller (i, j); i < 0 marks
// "no candidate"
__device__ __forceinline__ bool qa_span_better(float v, int i, int j, float w, int k, int l) {
  if (i < 0) return false;
  if (k < 0) return true;
  return v > w || (v == w && (i < k || (i == k && j < l)));
}

__global__ void __launch_bounds__(kCeWarps * 32)
qa_span_eval_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int B,
                    int S, int L, long long ignore_index, SpanEvalAccum* __restrict__ acc,
                    int* __restrict__ pred_spans, float* __restrict__ pred_scores,
                    long long capacity) {
  __shared__ double vals[3][kCeChunk];  // start CE, end CE, F1 of the chunk's rows
  __shared__ unsigned long long cursor;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) cursor = acc->cursor;
  __syncthreads();
  unsigned long long counted = 0, start_ok = 0, end_ok = 0, exact = 0, invalid = 0, overflow = 0;
  double tot[3] = {0.0, 0.0, 0.0};
  for (int base = 0; base < B; base += kCeChunk) {
    for (int rr = warp; rr < kCeChunk; rr += kCeWarps) {
      const int b = base + rr;
      double ce_s = 0.0, ce_e = 0.0, f1 = 0.0;
      if (b < B) {
        const float* st = logits + static_cast<long long>(b) * 2 * S;
        const float* en = st + S;
        const int64_t* lab = labels + static_cast<long long>(b) * kQaLabelCols;
        const long long gs = lab[0], ge = lab[1];
        // the search range, clipped to the row: a padded row (ignore_index) is empty
        const long long lo = lab[2] > 0 ? lab[2] : 0;
        const long long hi = lab[3] < S - 1 ? lab[3] : S - 1;
        const long long ehi = lab[4] < S - 1 ? lab[4] : S - 1;
        float best = -INFINITY;
        int bi = -1, bj = -1;
        for (long long i = lo + lane; i <= hi; i += 32) {
          const float si = st[i];
          const long long jmax = i + L - 1 < ehi ? i + L - 1 : ehi;
          for (long long j = i; j <= jmax; ++j) {
            float v = si + en[j];
            if (v != v) v = -INFINITY;
            // i and j ascend within a lane: only a strictly higher score replaces the candidate
            if (bi < 0 || v > best) {
              best = v;
              bi = static_cast<int>(i);
              bj = static_cast<int>(j);
            }
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, best, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
          if (qa_span_better(ov, oi, oj, best, bi, bj)) {
            best = ov;
            bi = oi;
            bj = oj;
          }
        }
        if (lane == 0) {
          const unsigned long long slot = cursor + static_cast<unsigned long long>(b);
          if (slot < static_cast<unsigned long long>(capacity)) {
            pred_spans[2 * slot] = bi;
            pred_spans[2 * slot + 1] = bj;
            pred_scores[slot] = best;
          } else {
            ++overflow;
          }
        }
        const bool ok_s = gs >= 0 && gs < S, ok_e = ge >= 0 && ge < S;
        if ((gs != ignore_index && !ok_s) || (ge != ignore_index && !ok_e)) {
          if (lane == 0) ++invalid;
        } else if (ok_s && ok_e) {
          int arg_s, arg_e;
          float lse_s, lse_e;
          warp_row_stats(st, S, lane, &arg_s, &lse_s);
          warp_row_stats(en, S, lane, &arg_e, &lse_e);
          ce_s = static_cast<double>(lse_s - st[gs]);
          ce_e = static_cast<double>(lse_e - en[ge]);
          // SQuAD's token F1 on position intervals: overlap / predicted and overlap / gold length
          const long long ov_hi = bj < ge ? bj : ge, ov_lo = bi > gs ? bi : gs;
          const long long overlap = ov_hi - ov_lo + 1;
          if (bi >= 0 && overlap > 0) {
            const double p = static_cast<double>(overlap) / static_cast<double>(bj - bi + 1);
            const double r = static_cast<double>(overlap) / static_cast<double>(ge - gs + 1);
            f1 = 2.0 * p * r / (p + r);
          }
          if (lane == 0) {
            ++counted;
            start_ok += arg_s == gs ? 1 : 0;
            end_ok += arg_e == ge ? 1 : 0;
            exact += (bi == gs && bj == ge) ? 1 : 0;
          }
        }
      }
      if (lane == 0) {
        vals[0][rr] = ce_s;
        vals[1][rr] = ce_e;
        vals[2][rr] = f1;
      }
    }
    __syncthreads();
    chunk_tree(vals, 3);
    if (threadIdx.x == 0) {
      tot[0] += vals[0][0];
      tot[1] += vals[1][0];
      tot[2] += vals[2][0];
    }
    __syncthreads();
  }
  if (lane == 0) {
    if (counted) atomicAdd(&acc->count, counted);
    if (start_ok) atomicAdd(&acc->start_correct, start_ok);
    if (end_ok) atomicAdd(&acc->end_correct, end_ok);
    if (exact) atomicAdd(&acc->exact, exact);
    if (invalid) atomicAdd(&acc->invalid, invalid);
    if (overflow) atomicAdd(&acc->overflow, overflow);
  }
  if (threadIdx.x == 0) {
    acc->start_loss_sum += tot[0];
    acc->end_loss_sum += tot[1];
    acc->f1_sum += tot[2];
    acc->cursor = cursor + static_cast<unsigned long long>(B);
  }
}

// ------------------------------------------------------------------------------------------
// Optimizer
// ------------------------------------------------------------------------------------------
// kScalars: lr and the clip coefficient come from the device-side OptimScalars (schedule / global
// norm clipping); the gradient is clipped before weight decay and momentum, as torch does when
// clip_grad_norm_ runs ahead of optimizer.step().  kScalars == false is the plain update.
template <bool kScalars>
__device__ __forceinline__ float scaled_grad(float g, float grad_scale, float clip) {
  if constexpr (kScalars) return (g * grad_scale) * clip;
  return g * grad_scale;
}

// One bank of a multi-tensor update (blockIdx.y picks the bank): a grid-stride float4 body and a
// scalar tail in block 0.  upd(p, g, m, v) updates one element's master p in place from its raw
// gradient g, with m / v the element's momentum / second moment, loaded and stored only when the
// update uses them (has_mom / has_mom2).  The bf16 shadow refresh and the gradient zeroing
// follow every element's update.
template <typename Update>
__device__ __forceinline__ void multi_tensor_update(const SgdTensor& t, int zero_grad, bool has_mom,
                                                    bool has_mom2, Update upd) {
  const long long n4 = t.numel >> 2;
  float4* p4 = reinterpret_cast<float4*>(t.p);
  float4* g4 = reinterpret_cast<float4*>(t.g);
  float4* m4 = reinterpret_cast<float4*>(t.mom);
  float4* v4 = reinterpret_cast<float4*>(t.mom2);
  uint2* b4 = reinterpret_cast<uint2*>(t.p_bf16);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 p = p4[i], m = has_mom ? m4[i] : float4{}, v = has_mom2 ? v4[i] : float4{};
    const float4 g = g4[i];
    upd(p.x, g.x, m.x, v.x);
    upd(p.y, g.y, m.y, v.y);
    upd(p.z, g.z, m.z, v.z);
    upd(p.w, g.w, m.w, v.w);
    p4[i] = p;
    if (has_mom) m4[i] = m;
    if (has_mom2) v4[i] = v;
    if (b4 != nullptr) b4[i] = make_uint2(pack_bf16x2(p.x, p.y), pack_bf16x2(p.z, p.w));
    if (zero_grad && !t.skip_zero) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (blockIdx.x == 0) {
    for (long long i = (n4 << 2) + threadIdx.x; i < t.numel; i += blockDim.x) {
      float p = t.p[i], m = has_mom ? t.mom[i] : 0.f, v = has_mom2 ? t.mom2[i] : 0.f;
      upd(p, t.g[i], m, v);
      t.p[i] = p;
      if (has_mom) t.mom[i] = m;
      if (has_mom2) t.mom2[i] = v;
      if (t.p_bf16 != nullptr) reinterpret_cast<__nv_bfloat16*>(t.p_bf16)[i] = __float2bfloat16(p);
      // zeroed even under skip_zero: harmless, the next step's first wgrad overwrites it anyway
      if (zero_grad) t.g[i] = 0.f;
    }
  }
}

template <bool kScalars>
__global__ void __launch_bounds__(256)
sgd_multi_kernel(const SgdTensor* __restrict__ tensors, float lr, float momentum,
                 float weight_decay, float grad_scale, int zero_grad,
                 const OptimScalars* __restrict__ sc) {
  const SgdTensor t = tensors[blockIdx.y];
  float clip = 1.f;
  if constexpr (kScalars) {
    lr = sc->lr;
    clip = sc->clip_coef;
  }
  const bool has_mom = t.mom != nullptr;
  multi_tensor_update(t, zero_grad, has_mom, false, [&](float& p, float gi, float& m, float&) {
    float g = sgd_direction<kScalars>(gi, p, grad_scale, clip, weight_decay);
    if (has_mom) {
      m = __fmaf_rn(momentum, m, g);
      g = m;
    }
    p = sgd_apply(p, g, lr);
  });
}

// Adam / AdamW over the same descriptors (torch.optim.Adam semantics, experiment/launch.py:152-155
// accepts any torch.optim name): one launch per stage, moments + master + bf16 shadow + gradient
// zeroing in one pass = 28 B / parameter.  The bias corrections come from a device-side step
// counter, so a captured graph replays the right correction every step.
template <bool kScalars>
__global__ void __launch_bounds__(256)
adam_multi_kernel(const SgdTensor* __restrict__ tensors, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int decoupled, const uint64_t* __restrict__ step,
                  float grad_scale, int zero_grad, const OptimScalars* __restrict__ sc) {
  const SgdTensor t = tensors[blockIdx.y];
  float clip = 1.f;
  if constexpr (kScalars) {
    lr = sc->lr;   // scales step_size and the decoupled decay, as torch's lr does
    clip = sc->clip_coef;
  }
  const float tstep = static_cast<float>(*step);
  const float bc1 = 1.f - powf(beta1, tstep);
  const float bc2_rsqrt = rsqrtf(1.f - powf(beta2, tstep));
  const float step_size = lr / bc1;
  const float decay = decoupled ? 1.f - lr * weight_decay : 1.f;
  const float l2 = decoupled ? 0.f : weight_decay;
  multi_tensor_update(t, zero_grad, true, true, [&](float& p, float gi, float& m, float& v) {
    p *= decay;
    const float g = scaled_grad<kScalars>(gi, grad_scale, clip) + l2 * p;
    m = beta1 * m + (1.f - beta1) * g;
    v = beta2 * v + (1.f - beta2) * g * g;
    p -= step_size * m / (sqrtf(v) * bc2_rsqrt + eps);
  });
}

// Global-norm clipping, step 1: per-block sums of squares of g * grad_scale over the same
// descriptors (4 B read per parameter).  Each block reduces in a fixed order and stores its own
// partial, so a replay reproduces the result bit for bit.
__global__ void __launch_bounds__(256)
grad_sumsq_multi_kernel(const SgdTensor* __restrict__ tensors, float grad_scale,
                        float* __restrict__ partials) {
  const SgdTensor t = tensors[blockIdx.y];
  const long long n4 = t.numel >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(t.g);
  float acc = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 g = g4[i];
    const float x = g.x * grad_scale, y = g.y * grad_scale;
    const float z = g.z * grad_scale, w = g.w * grad_scale;
    acc += (x * x + y * y) + (z * z + w * w);
  }
  if (blockIdx.x == 0) {
    for (long long i = (n4 << 2) + threadIdx.x; i < t.numel; i += blockDim.x) {
      const float x = t.g[i] * grad_scale;
      acc += x * x;
    }
  }
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    partials[static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x] = s;
  }
}

__device__ __forceinline__ void st_relaxed_sys_f32(float* addr, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float ld_relaxed_sys_f32(const float* addr) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(addr) : "memory");
  return v;
}

__device__ double lr_factor(int schedule, double k, int warmup, int total) {
  if (schedule == kLrNone) return 1.0;
  if (k < warmup) return k / fmax(1.0, static_cast<double>(warmup));
  if (schedule == kLrConstant) return 1.0;
  const double span = fmax(1.0, static_cast<double>(total - warmup));
  if (schedule == kLrLinear) return fmax(0.0, (total - k) / span);
  const double prog = fmin(1.0, (k - warmup) / span);   // clamped: no rise again after T
  return fmax(0.0, 0.5 * (1.0 + cos(3.14159265358979323846 * prog)));
}

// Global-norm clipping, step 2 (+ the learning-rate schedule): one block.
//
// Peer exchange (ex.n_ranks > 1): thread 0 stores this rank's share into slot [epoch & 1][my_pos]
// of EVERY rank's region and bumps that region's flags[my_pos] with release semantics, then waits
// (acquire) until flags[q] >= epoch for every q and sums slot [epoch & 1][q] in position order.
// Flags count the steps a rank has published, so they equal the epoch after that step's store.
// Why two slots per rank are enough: rank q can only store epoch e + 2 (same parity as e) after
// its own step e + 1 finished the exchange, which needed this rank's epoch-(e + 1) store, and this
// rank makes that store in a later launch than the one that reads epoch e's slots.
__global__ void __launch_bounds__(256)
optim_finalize_kernel(const float* __restrict__ partials, int n_partials,
                      const float* __restrict__ extra_sumsq, NormExchangeArgs ex,
                      const uint64_t* __restrict__ step, long long step_offset, int schedule,
                      int warmup, int total, double base_lr, float max_norm, OptimScalars* __restrict__ out) {
  __shared__ double red[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_partials; i += blockDim.x) acc += partials[i];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  double local = red[0];
  if (extra_sumsq != nullptr) local += static_cast<double>(*extra_sumsq);
  const float local_f = static_cast<float>(local);
  double total_sumsq = local_f;
  if (ex.n_ranks > 1) {
    const uint32_t e = *ex.epoch;
    const int par = static_cast<int>(e & 1u) * ex.n_ranks;
    for (int q = 0; q < ex.n_ranks; ++q) {
      char* base = static_cast<char*>(ex.regions[q]);
      st_relaxed_sys_f32(reinterpret_cast<float*>(base + 256) + par + ex.my_pos, local_f);
      __threadfence_system();
      red_release_sys_add(reinterpret_cast<uint32_t*>(base) + ex.my_pos, 1u);
    }
    const char* mine = static_cast<const char*>(ex.regions[ex.my_pos]);
    const uint32_t* flags = reinterpret_cast<const uint32_t*>(mine);
    const float* slots = reinterpret_cast<const float*>(mine + 256) + par;
    total_sumsq = 0.0;
    for (int q = 0; q < ex.n_ranks; ++q) {
      if (!wait_flag_ge(flags + q, e, kFlagTimeoutNs)) {
        if (ex.error_flag) atomicExch(ex.error_flag, 4);
      }
      total_sumsq += static_cast<double>(ld_relaxed_sys_f32(slots + q));
    }
  }
  const float norm = static_cast<float>(sqrt(total_sumsq));
  float coef = 1.f;
  if (max_norm > 0.f) {
    // torch.nn.utils.clip_grad_norm_: clamp(max_norm / (norm + 1e-6), max=1); NaN stays NaN
    coef = __fdiv_rn(max_norm, __fadd_rn(norm, 1e-6f));
    if (!(coef != coef)) coef = fminf(coef, 1.f);
  }
  const double k = static_cast<double>(step != nullptr ? static_cast<long long>(*step) : 0ll) +
                   static_cast<double>(step_offset);
  out->lr = static_cast<float>(base_lr * lr_factor(schedule, k, warmup, total));
  out->clip_coef = coef;
  out->grad_norm = norm;
  out->local_sumsq = local_f;
}

// LAMB, two passes over the segment / chunk table (api.h).  Block b takes the contiguous chunk
// range [b * n / G, (b + 1) * n / G): every chunk is at most kLambChunk elements, so the blocks
// carry equal work whether a segment is a 1K bias or the 31M-element word-embedding table, and a
// block meets only the few segments its range crosses.  A chunk's partials depend only on the
// chunk, never on G or on which block ran it.
struct LambBias {
  float inv_bc1, inv_bc2;
};
__device__ __forceinline__ LambBias lamb_bias(const uint64_t* step, float beta1, float beta2) {
  const double t = static_cast<double>(*step);
  return {static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta1), t))),
          static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta2), t)))};
}
// the Adam-style update plus decay; both passes call this one function on the same m, v, p
__device__ __forceinline__ float lamb_u(float m, float v, float p, LambBias bc, float eps,
                                        float wd) {
  return (m * bc.inv_bc1) / (sqrtf(v * bc.inv_bc2) + eps) + wd * p;
}
__device__ __forceinline__ void lamb_chunk_range(int n_chunks, int& c0, int& c1) {
  c0 = static_cast<int>(static_cast<long long>(blockIdx.x) * n_chunks / gridDim.x);
  c1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * n_chunks / gridDim.x);
}

template <bool kScalars>
__global__ void __launch_bounds__(256)
lamb_moments_kernel(const LambSegment* __restrict__ segs, const int* __restrict__ chunk_seg,
                    int n_chunks, float beta1, float beta2, float eps,
                    const uint64_t* __restrict__ step, float grad_scale,
                    const OptimScalars* __restrict__ sc, float2* __restrict__ partials) {
  const float clip = kScalars ? sc->clip_coef : 1.f;
  const LambBias bc = lamb_bias(step, beta1, beta2);
  __shared__ float red[2][8];
  int c0, c1;
  lamb_chunk_range(n_chunks, c0, c1);
  for (int c = c0; c < c1; ++c) {
    const LambSegment s = segs[chunk_seg[c]];
    const long long base = static_cast<long long>(c - s.chunk0) * kLambChunk;
    const int len = static_cast<int>(min(static_cast<long long>(kLambChunk), s.numel - base));
    const float wd = s.weight_decay;
    float w2 = 0.f, u2 = 0.f;
    auto one = [&](float p, float gi, float& m, float& v) {
      const float g = scaled_grad<kScalars>(gi, grad_scale, clip);
      m = beta1 * m + (1.f - beta1) * g;
      v = beta2 * v + (1.f - beta2) * g * g;
      const float u = lamb_u(m, v, p, bc, eps, wd);
      w2 += p * p;
      u2 += u * u;
    };
    float* p = s.p + base;
    float* g = s.g + base;
    float* m = s.m + base;
    float* v = s.v + base;
    int scalar_from = 0;
    if (s.vec) {
      const int n4 = len >> 2;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 pp = reinterpret_cast<const float4*>(p)[i];
        const float4 gg = reinterpret_cast<const float4*>(g)[i];
        float4 mm = reinterpret_cast<const float4*>(m)[i];
        float4 vv = reinterpret_cast<const float4*>(v)[i];
        one(pp.x, gg.x, mm.x, vv.x);
        one(pp.y, gg.y, mm.y, vv.y);
        one(pp.z, gg.z, mm.z, vv.z);
        one(pp.w, gg.w, mm.w, vv.w);
        reinterpret_cast<float4*>(m)[i] = mm;
        reinterpret_cast<float4*>(v)[i] = vv;
        if (!s.skip_zero) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      scalar_from = n4 << 2;
    }
    for (int i = scalar_from + threadIdx.x; i < len; i += blockDim.x) {
      float mi = m[i], vi = v[i];
      one(p[i], g[i], mi, vi);
      m[i] = mi;
      v[i] = vi;
      if (!s.skip_zero) g[i] = 0.f;
    }
    w2 = warp_sum(w2);
    u2 = warp_sum(u2);
    if ((threadIdx.x & 31) == 0) {
      red[0][threadIdx.x >> 5] = w2;
      red[1][threadIdx.x >> 5] = u2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float a = 0.f, b = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        a += red[0][w];
        b += red[1][w];
      }
      partials[c] = make_float2(a, b);
    }
    __syncthreads();
  }
}

template <bool kScalars>
__global__ void __launch_bounds__(256)
lamb_update_kernel(const LambSegment* __restrict__ segs, const int* __restrict__ chunk_seg,
                   int n_chunks, float lr, float beta1, float beta2, float eps,
                   const uint64_t* __restrict__ step, const OptimScalars* __restrict__ sc,
                   const float2* __restrict__ partials, float* __restrict__ ratios) {
  if constexpr (kScalars) lr = sc->lr;
  const LambBias bc = lamb_bias(step, beta1, beta2);
  __shared__ double red[2][256];
  __shared__ float ratio_s;
  int c0, c1;
  lamb_chunk_range(n_chunks, c0, c1);
  int cur = -1;
  float r = 1.f;
  for (int c = c0; c < c1; ++c) {
    const int si = chunk_seg[c];
    const LambSegment s = segs[si];
    if (si != cur) {   // block-uniform: the trust ratio of a segment this block enters
      cur = si;
      r = 1.f;
      if (s.use_ratio) {
        double a = 0.0, b = 0.0;
        for (int k = threadIdx.x; k < s.n_chunks; k += blockDim.x) {
          const float2 q = partials[s.chunk0 + k];
          a += q.x;
          b += q.y;
        }
        red[0][threadIdx.x] = a;
        red[1][threadIdx.x] = b;
        __syncthreads();
        for (int h = 128; h > 0; h >>= 1) {
          if (threadIdx.x < h) {
            red[0][threadIdx.x] += red[0][threadIdx.x + h];
            red[1][threadIdx.x] += red[1][threadIdx.x + h];
          }
          __syncthreads();
        }
        if (threadIdx.x == 0) {
          const double wn = sqrt(red[0][0]), un = sqrt(red[1][0]);
          ratio_s = (wn > 0.0 && un > 0.0) ? static_cast<float>(wn / un) : 1.f;
        }
        __syncthreads();
        r = ratio_s;
      }
    }
    if (c == s.chunk0 && threadIdx.x == 0) ratios[si] = r;
    const long long base = static_cast<long long>(c - s.chunk0) * kLambChunk;
    const int len = static_cast<int>(min(static_cast<long long>(kLambChunk), s.numel - base));
    const float wd = s.weight_decay;
    const float step_lr = lr * r;
    float* p = s.p + base;
    const float* m = s.m + base;
    const float* v = s.v + base;
    int scalar_from = 0;
    if (s.vec) {
      const int n4 = len >> 2;
      uint2* b4 = s.p_bf16 ? reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(s.p_bf16) + base)
                           : nullptr;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 pp = reinterpret_cast<const float4*>(p)[i];
        const float4 mm = reinterpret_cast<const float4*>(m)[i];
        const float4 vv = reinterpret_cast<const float4*>(v)[i];
        pp.x -= step_lr * lamb_u(mm.x, vv.x, pp.x, bc, eps, wd);
        pp.y -= step_lr * lamb_u(mm.y, vv.y, pp.y, bc, eps, wd);
        pp.z -= step_lr * lamb_u(mm.z, vv.z, pp.z, bc, eps, wd);
        pp.w -= step_lr * lamb_u(mm.w, vv.w, pp.w, bc, eps, wd);
        reinterpret_cast<float4*>(p)[i] = pp;
        if (b4 != nullptr) b4[i] = make_uint2(pack_bf16x2(pp.x, pp.y), pack_bf16x2(pp.z, pp.w));
      }
      scalar_from = n4 << 2;
    }
    __nv_bfloat16* b = s.p_bf16 ? static_cast<__nv_bfloat16*>(s.p_bf16) + base : nullptr;
    for (int i = scalar_from + threadIdx.x; i < len; i += blockDim.x) {
      const float pi = p[i] - step_lr * lamb_u(m[i], v[i], p[i], bc, eps, wd);
      p[i] = pi;
      if (b != nullptr) b[i] = __float2bfloat16(pi);
    }
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ d,
                                     long long n) {
  const long long n4 = n >> 2;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(s)[i];
    reinterpret_cast<uint2*>(d)[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0)
    for (long long i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x)
      d[i] = __float2bfloat16(s[i]);
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ s, float* __restrict__ d,
                                     long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    d[i] = __bfloat162float(s[i]);
}

__global__ void __launch_bounds__(256)
dgelu_mul_kernel(const uint4* __restrict__ g, const uint4* __restrict__ h, uint4* __restrict__ y,
                 long long n8) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 a = g[i];
    const uint4 b = h[i];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
    const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 x = unpack_bf16x2(aw[t]);
      const float2 z = unpack_bf16x2(bw[t]);
      o[t] = pack_bf16x2(x.x * dgelu_erf(z.x), x.y * dgelu_erf(z.y));
    }
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------------------------------
// runtime helpers
// ------------------------------------------------------------------------------------------
__global__ void advance_counter_kernel(uint64_t* c, uint64_t inc) { *c += inc; }
__global__ void advance_epoch_kernel(uint32_t* c, uint32_t inc) { *c += inc; }
__global__ void signal_flags_kernel(uint32_t* flags, int n, uint32_t inc) {
  __threadfence_system();
  for (int i = threadIdx.x; i < n; i += blockDim.x) red_release_sys_add(flags + i, inc);
}
__global__ void wait_flags_kernel(const uint32_t* flags, int n, const uint32_t* epoch,
                                  uint32_t mult, int* error_flag) {
  const uint32_t target = (*epoch) * mult;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!wait_flag_ge(flags + i, target, kFlagTimeoutNs)) {
      if (error_flag) atomicExch(error_flag, 3);
    }
  }
}
__global__ void spin_ns_kernel(uint64_t ns) {
  const uint64_t t0 = globaltimer_ns();
  while (globaltimer_ns() - t0 < ns) __nanosleep(200);
}
__global__ void record_time_kernel(uint64_t* slot) { *slot = globaltimer_ns(); }
__global__ void spin_factor_kernel(const uint64_t* t_start, float factor) {
  const uint64_t now = globaltimer_ns();
  const uint64_t elapsed = now - *t_start;
  uint64_t budget = static_cast<uint64_t>(static_cast<double>(elapsed) * factor);
  if (budget > 2000000000ull) budget = 2000000000ull;  // never hold the GPU > 2 s
  while (globaltimer_ns() - now < budget) __nanosleep(200);
}
__global__ void __launch_bounds__(256)
peer_copy_signal_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long n16,
                        uint32_t* flags, int n_flags, uint32_t inc, unsigned int* done_counter) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n16;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      *done_counter = 0;
      __threadfence_system();
      for (int i = 0; i < n_flags; ++i) red_release_sys_add(flags + i, inc);
    }
  }
}

// ---- tied word-embedding gradient exchange (parallel/p2p.py: TiedGradExchange) ------------------
// After a block's stores: the last block of the grid to finish publishes `flag` (release.sys), so
// a reader that acquires the flag sees every block's stores.  `done` is reset for the next launch.
__device__ __forceinline__ void last_block_publish(uint32_t* flag, unsigned int* done) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {
      *done = 0;
      __threadfence_system();
      red_release_sys_add(flag, 1u);
    }
  }
}
// Last rank: the replica's gradient -> the first rank's inbox (16-byte peer stores), then +1 on the
// first rank's push flag.
__global__ void __launch_bounds__(256)
tied_grad_push_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n,
                      uint32_t* flag, unsigned int* done) {
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const float4* s4 = reinterpret_cast<const float4*>(src);
  float4* d4 = reinterpret_cast<float4*>(dst);
  for (long long i = t0; i < n4; i += stride) d4[i] = __ldcs(s4 + i);
  for (long long i = (n4 << 2) + t0; i < n; i += stride) dst[i] = src[i];
  last_block_publish(flag, done);
}
// First rank: wait until the push flag reaches *epoch (acquire.sys, 4 s timeout -> error 5), then
// s = g + inbox ONCE per element, stored into g and through the peer pointer into the replica's
// gradient, then +1 on the last rank's flag.  One writer of the sum: both copies bit-identical.
__global__ void __launch_bounds__(256)
tied_grad_reduce_kernel(float* __restrict__ g, const float* __restrict__ inbox,
                        float* __restrict__ peer_g, long long n, const uint32_t* wait_flag,
                        const uint32_t* epoch, int* error_flag, uint32_t* publish_flag,
                        unsigned int* done) {
  __shared__ int arrived;
  if (threadIdx.x == 0) {
    const uint32_t target = *epoch;
    bool ok = ld_acquire_sys(wait_flag) >= target;
    // after a timeout elsewhere in the step the run is failing: do not wait 4 s per block
    if (!ok && !(error_flag && *reinterpret_cast<volatile int*>(error_flag) != 0))
      ok = wait_flag_ge(wait_flag, target, kFlagTimeoutNs);
    if (!ok && error_flag) atomicExch(error_flag, 5);
    arrived = ok;
  }
  __syncthreads();
  if (arrived) {
    const long long n4 = n >> 2;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    float4* g4 = reinterpret_cast<float4*>(g);
    const float4* in4 = reinterpret_cast<const float4*>(inbox);
    float4* p4 = reinterpret_cast<float4*>(peer_g);
    for (long long i = t0; i < n4; i += stride) {
      const float4 a = g4[i];
      const float4 b = __ldcs(in4 + i);
      const float4 s = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
      g4[i] = s;
      p4[i] = s;
    }
    for (long long i = (n4 << 2) + t0; i < n; i += stride) {
      const float s = g[i] + inbox[i];
      g[i] = s;
      peer_g[i] = s;
    }
  }
  last_block_publish(publish_flag, done);
}

// SMs of the current device (grid caps of the grid-stride kernels are multiples of it)
inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

inline int grid_for_rows(int rows, int warps_per_block, int max_blocks) {
  int g = (rows + warps_per_block - 1) / warps_per_block;
  if (g > max_blocks) g = max_blocks;
  if (g < 1) g = 1;
  return g;
}

}  // namespace

#define SKY_LAUNCH_CHECK() return static_cast<int>(cudaGetLastError())

int launch_layernorm_fwd(const LayerNormFwdArgs& a, cudaStream_t stream) {
  if (a.M <= 0) return 0;
  if (a.H % 8 != 0 || a.H > kLnMaxVec * 256) return 910;
  const int grid = (a.M + kLnRowsPerCta - 1) / kLnRowsPerCta;
  const int nv = (a.H / 8 + 31) / 32;
#define SKY_LN_FWD(NV)                                                                          \
  launch_pdl(layernorm_fwd_kernel<NV>, dim3(grid), dim3(256), 0, stream,                        \
      reinterpret_cast<const __nv_bfloat16*>(a.z), reinterpret_cast<__nv_bfloat16*>(a.y), a.mean, \
      a.rstd, a.gamma, a.beta, a.M, a.H, a.eps, a.wait_flags, a.wait_epoch, a.wait_mult,        \
      a.error_flag, a.signal_flags)
  if (nv <= 1) SKY_LN_FWD(1);
  else if (nv <= 2) SKY_LN_FWD(2);
  else if (nv <= 4) SKY_LN_FWD(4);
  else SKY_LN_FWD(8);
#undef SKY_LN_FWD
  SKY_LAUNCH_CHECK();
}

int launch_layernorm_bwd(const LayerNormBwdArgs& a, cudaStream_t stream) {
  if (a.M <= 0) return 0;
  if (a.H % 8 != 0 || a.H > kLnMaxVec * 256) return 911;
  const int grid = grid_for_rows(a.M, 8, num_sms() * 8);
  const int nv = (a.H / 8 + 31) / 32;
#define SKY_LN_BWD(NV)                                                                           \
  launch_pdl(layernorm_bwd_kernel<NV>, dim3(grid), dim3(256), 0, stream,                         \
      reinterpret_cast<const __nv_bfloat16*>(a.dy), reinterpret_cast<const __nv_bfloat16*>(a.z), \
      a.mean, a.rstd, a.gamma, reinterpret_cast<__nv_bfloat16*>(a.dz),                           \
      reinterpret_cast<__nv_bfloat16*>(a.dz_dropped), a.M, a.H, a.dropout_p, a.rng_state,        \
      a.rng_stream, a.wait_flags, a.wait_epoch, a.wait_mult, a.error_flag)
  if (nv <= 1) SKY_LN_BWD(1);
  else if (nv <= 2) SKY_LN_BWD(2);
  else if (nv <= 4) SKY_LN_BWD(4);
  else SKY_LN_BWD(8);
#undef SKY_LN_BWD
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  // NOTE: when gated on peer flags, the row kernel above has already waited for every panel.
  if (a.dgamma != nullptr || a.dbeta != nullptr)
    return launch_ln_param_grad(a.dy, a.z, a.mean, a.rstd, a.dgamma, a.dbeta, a.M, a.H, nullptr,
                                nullptr, stream);
  SKY_LAUNCH_CHECK();
}

// dgamma += sum_rows dy * xhat, dbeta += sum_rows dy.  A separate entry point so that the engine
// can take it off the input-gradient critical path (it is queued with the weight gradients).
int launch_ln_param_grad(const void* dy, const void* z, const float* mean, const float* rstd,
                         float* dgamma, float* dbeta, int M, int H, const void* x2, float* out2,
                         cudaStream_t stream) {
  if (M <= 0) return 0;
  if (H % 8 != 0) return 916;  // 16-byte row loads
  dim3 g2((H + 255) / 256, 1);
  int ry = (M + 63) / 64;
  if (ry > 64) ry = 64;
  if (ry < 1) ry = 1;
  g2.y = ry;
  launch_pdl(ln_param_grad_kernel, g2, dim3(256), 0, stream,
             reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(z),
             mean, rstd, dgamma, dbeta, M, H, reinterpret_cast<const __nv_bfloat16*>(x2), out2);
  SKY_LAUNCH_CHECK();
}

int launch_dgelu_mul(const void* g, const void* h, void* y, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8 != 0) return 914;
  long long blocks = (n / 8 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  launch_pdl(dgelu_mul_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream,
      reinterpret_cast<const uint4*>(g), reinterpret_cast<const uint4*>(h),
      reinterpret_cast<uint4*>(y), n / 8);
  SKY_LAUNCH_CHECK();
}

int launch_colsum(const void* x, int M, int N, int ldx, float* out, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return 0;
  if (N % 8 != 0) return 912;
  dim3 grid((N + 255) / 256, 1);
  int ry = (M + 63) / 64;
  if (ry > 64) ry = 64;
  grid.y = ry;
  launch_pdl(colsum_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), M, N, static_cast<long long>(ldx),
                                          out);
  SKY_LAUNCH_CHECK();
}

int launch_embed_fwd(const EmbedArgs& a, cudaStream_t stream) {
  const int BS = a.B * a.S;
  if (BS <= 0) return 0;
  if (a.H % 4 != 0) return 913;
  const int grid = grid_for_rows(BS, 8, num_sms() * 8);
  embed_fwd_kernel<<<grid, 256, 0, stream>>>(
      a.input_ids, a.token_type, a.attn_mask, a.word, a.pos, a.type, a.gamma, a.beta,
      reinterpret_cast<__nv_bfloat16*>(a.out), a.ext_mask, a.mean, a.rstd, BS, a.S, a.H, a.eps,
      a.dropout_p, a.rng_state, a.rng_stream);
  SKY_LAUNCH_CHECK();
}

int launch_embed_bwd(const EmbedBwdArgs& a, cudaStream_t stream) {
  const int BS = a.B * a.S;
  if (BS <= 0) return 0;
  if (a.H % 4 != 0) return 913;
  const int grid = grid_for_rows(BS, 8, num_sms() * 2);
  int t_smem = a.type_rows < 4 ? a.type_rows : 4;
  if (t_smem < 0) t_smem = 0;
  const size_t smem = static_cast<size_t>(2 + t_smem) * a.H * sizeof(float);
  if (smem > 48 * 1024) {
    t_smem = 0;
  }
  const size_t smem_used = static_cast<size_t>(2 + t_smem) * a.H * sizeof(float);
  if (smem_used > 48 * 1024) return 915;
  embed_bwd_kernel<<<grid, 256, smem_used, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(a.dout), a.input_ids, a.token_type, a.word, a.pos,
      a.type, a.gamma, a.mean, a.rstd, a.dword, a.dpos, a.dtype_, a.dgamma, a.dbeta, BS, a.S, a.H,
      a.dropout_p, a.rng_state, a.rng_stream, a.wait_flags, a.wait_epoch, a.wait_mult,
      a.error_flag, t_smem);
  SKY_LAUNCH_CHECK();
}

int launch_small_linear_fwd(const void* x, bool x_bf16, int ldx, const float* w, const float* b,
                            float* y, int M, int N, int K, int act_tanh, float dropout_p,
                            const uint64_t* rng_state, uint32_t rng_stream, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return 0;
  const long long outs = static_cast<long long>(M) * N;
  const int grid = static_cast<int>((outs + 3) / 4);
  small_linear_fwd_kernel<<<grid, 128, 0, stream>>>(x, x_bf16, ldx, w, b, y, M, N, K, act_tanh,
                                                    dropout_p, rng_state, rng_stream);
  SKY_LAUNCH_CHECK();
}

int launch_small_linear_bwd(const void* x, bool x_bf16, int ldx, const float* w, const float* y,
                            const float* dy, void* dx, bool dx_bf16, int lddx, float* dw, float* db,
                            int M, int N, int K, int act_tanh, float dropout_p,
                            const uint64_t* rng_state, uint32_t rng_stream, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return 0;
  if (dx != nullptr) {
    dim3 grid((K + 127) / 128, (M + 7) / 8);
    small_linear_dx_kernel<<<grid, 128, 0, stream>>>(w, y, dy, dx, dx_bf16, lddx, M, N, K,
                                                     act_tanh, dropout_p, rng_state, rng_stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (dw != nullptr) {
    dim3 grid((K + 127) / 128, N);
    small_linear_dw_kernel<<<grid, 128, 0, stream>>>(x, x_bf16, ldx, y, dy, dw, db, M, N, K,
                                                     act_tanh, dropout_p, rng_state, rng_stream);
  }
  SKY_LAUNCH_CHECK();
}

int launch_softmax_ce(const float* logits, int ldl, const int64_t* labels, int label_ld, int N,
                      int G, int C, long long ignore_index, float* dlogits, float grad_scale,
                      float* loss, float* loss_acc, cudaStream_t stream) {
  if (N < 0 || C < 1 || (G != 1 && G != 2) || ldl < C || label_ld < G ||
      static_cast<long long>(N) * G * C > 0x7fffffffLL)
    return 985;
  if (N > 0 && (!logits || !labels || !dlogits)) return 986;
  auto kern = G == 2 ? softmax_ce_kernel<2> : softmax_ce_kernel<1>;
  kern<<<1, kCeWarps * 32, 0, stream>>>(logits, ldl, labels, label_ld, N, C, ignore_index, dlogits,
                                        grad_scale, loss, loss_acc);
  SKY_LAUNCH_CHECK();
}

int launch_classify_eval(const float* logits, int ldl, const int64_t* labels, int M, int C,
                         long long ignore_index, EvalAccum* acc, cudaStream_t stream) {
  if (C < 1 || C > kEvalMaxClasses) return 940;
  if (acc == nullptr || ldl < C) return 941;
  if (M <= 0) return 0;
  classify_eval_kernel<<<1, kEvalWarps * 32, 0, stream>>>(logits, ldl, labels, M, C, ignore_index,
                                                          acc);
  SKY_LAUNCH_CHECK();
}

size_t vocab_ce_workspace_bytes(int M) {
  return static_cast<size_t>(M > 0 ? M : 0) * (sizeof(double) + sizeof(int)) + 16;
}

namespace {
template <bool kEval, bool kVec>
int launch_vocab_ce_rows(const VocabCeArgs& a, size_t smem, double* row_loss, int* row_flags,
                         const int* n_valid, cudaStream_t stream) {
  auto kern = vocab_ce_row_kernel<kEval, kVec>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kVocabCeMaxV * 2);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = true;
  }
  kern<<<a.M, kVceThreads, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(a.logits), a.ldl, a.labels, a.V, a.ignore_index,
      reinterpret_cast<__nv_bfloat16*>(a.dlogits), a.grad_scale, n_valid, row_loss, row_flags);
  return static_cast<int>(cudaGetLastError());
}
}  // namespace

int vocab_ce_launches(const VocabCeArgs& a) {
  if (a.acc != nullptr) return a.M > 0 ? 2 : 0;
  return a.M > 0 ? 3 : 2;
}

int launch_vocab_ce(const VocabCeArgs& a, cudaStream_t stream) {
  const bool eval = a.acc != nullptr;
  if (a.V < 1 || a.V > kVocabCeMaxV) return 950;
  // an empty batch (M == 0) may come with null data pointers: nothing is read or written there
  if (a.M < 0 || a.ldl < a.V || a.workspace == nullptr) return 951;
  if (a.M > 0 && (a.logits == nullptr || a.labels == nullptr)) return 951;
  // exactly one of gradient (training) / accumulator (eval)
  if (eval ? a.dlogits != nullptr : (a.M > 0 && a.dlogits == nullptr)) return 952;
  if (a.M > 0 && a.dlogits != nullptr && a.dlogits != a.logits) {
    // a separate gradient buffer must not overlap the logits (in place is fine: each row is
    // staged in shared memory before it is overwritten)
    const char* l0 = static_cast<const char*>(a.logits);
    const char* d0 = static_cast<const char*>(a.dlogits);
    const long long bytes = (static_cast<long long>(a.M > 0 ? a.M - 1 : 0) * a.ldl + a.V) * 2;
    if (d0 < l0 + bytes && l0 < d0 + bytes) return 953;
  }
  char* ws = static_cast<char*>(a.workspace);
  double* row_loss = reinterpret_cast<double*>(ws);
  int* row_flags = reinterpret_cast<int*>(ws + static_cast<size_t>(a.M) * sizeof(double));
  int* n_valid = row_flags + a.M;
  if (!eval) {
    vocab_ce_count_kernel<<<1, kVceFinThreads, 0, stream>>>(a.labels, a.M, a.ignore_index,
                                                            n_valid);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (a.M > 0) {
    const size_t smem = ((static_cast<size_t>(a.V) * 2 + 15) / 16) * 16;
    const bool vec = (reinterpret_cast<uintptr_t>(a.logits) % 16 == 0) && (a.ldl % 8 == 0) &&
                     (eval || reinterpret_cast<uintptr_t>(a.dlogits) % 16 == 0);
    int rc = eval ? (vec ? launch_vocab_ce_rows<true, true>(a, smem, row_loss, row_flags, n_valid, stream)
                         : launch_vocab_ce_rows<true, false>(a, smem, row_loss, row_flags, n_valid, stream))
                  : (vec ? launch_vocab_ce_rows<false, true>(a, smem, row_loss, row_flags, n_valid, stream)
                         : launch_vocab_ce_rows<false, false>(a, smem, row_loss, row_flags, n_valid, stream));
    if (rc != 0) return rc;
  }
  if (eval && a.M == 0) return 0;
  vocab_ce_finalize_kernel<<<1, kVceFinThreads, 0, stream>>>(
      row_loss, row_flags, a.M, n_valid, a.grad_scale, a.loss_out, a.loss_acc, a.acc);
  SKY_LAUNCH_CHECK();
}

namespace {
bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }
}  // namespace

int launch_mlm_gather(const void* hidden, const int64_t* labels, int B, int S, int H, int P,
                      long long ignore_index, int V, int* slot_of_row, int64_t* slot_labels,
                      void* x_c, cudaStream_t stream) {
  if (B < 1 || S < 1 || H < 8 || H % 8 != 0 || P < 1 || P > kMlmMaxPredictions || V < 1)
    return 960;
  if (!hidden || !labels || !slot_of_row || !slot_labels || !x_c) return 961;
  if (!aligned16(hidden) || !aligned16(x_c)) return 962;
  mlm_gather_kernel<<<B, kMlmThreads, static_cast<size_t>(P) * sizeof(int), stream>>>(
      static_cast<const uint4*>(hidden), labels, S, H / 8, P, ignore_index, V, slot_of_row,
      slot_labels, static_cast<uint4*>(x_c));
  SKY_LAUNCH_CHECK();
}

int launch_mlm_scatter(const void* dx_c, const int* slot_of_row, long long rows, int H,
                       void* dhidden, cudaStream_t stream, const void* dcls, int S) {
  if (rows < 1 || H < 8 || H % 8 != 0) return 960;
  if (!dx_c || !slot_of_row || !dhidden) return 961;
  if (!aligned16(dx_c) || !aligned16(dhidden)) return 962;
  if (dcls != nullptr && (S < 1 || rows % S != 0)) return 960;
  if (dcls != nullptr && !aligned16(dcls)) return 962;
  const long long vec = rows * (H / 8);
  long long blocks = (vec + kMlmThreads - 1) / kMlmThreads;
  if (blocks > num_sms() * 8LL) blocks = num_sms() * 8LL;
  if (dcls == nullptr) {
    mlm_scatter_kernel<false><<<static_cast<unsigned>(blocks), kMlmThreads, 0, stream>>>(
        static_cast<const uint4*>(dx_c), slot_of_row, rows, H / 8, static_cast<uint4*>(dhidden),
        nullptr, 1);
  } else {
    mlm_scatter_kernel<true><<<static_cast<unsigned>(blocks), kMlmThreads, 0, stream>>>(
        static_cast<const uint4*>(dx_c), slot_of_row, rows, H / 8, static_cast<uint4*>(dhidden),
        static_cast<const uint4*>(dcls), S);
  }
  SKY_LAUNCH_CHECK();
}

int launch_cls_grad_add(void* dhidden, const void* dcls, int B, int S, int H,
                        cudaStream_t stream) {
  if (B < 1 || S < 1 || H < 8 || H % 8 != 0) return 982;
  if (!dhidden || !dcls) return 983;
  if (!aligned16(dhidden) || !aligned16(dcls)) return 984;
  const long long vec = static_cast<long long>(B) * (H / 8);
  long long blocks = (vec + kMlmThreads - 1) / kMlmThreads;
  if (blocks > num_sms() * 8LL) blocks = num_sms() * 8LL;
  cls_grad_add_kernel<<<static_cast<unsigned>(blocks), kMlmThreads, 0, stream>>>(
      static_cast<uint4*>(dhidden), static_cast<const uint4*>(dcls), B, S, H / 8);
  SKY_LAUNCH_CHECK();
}

namespace {
bool qa_shape_ok(int B, int S, int H) {
  return B >= 1 && S >= 1 && H >= 8 && H % 8 == 0 &&
         static_cast<long long>(B) * S <= 0x7fffffffLL;
}
}  // namespace

size_t qa_logits_bwd_workspace_bytes(int B, int S, int H) {
  if (!qa_shape_ok(B, S, H)) return 0;
  const long long R = static_cast<long long>(B) * S;
  const long long blocks = (R + kQaRowsPerCta - 1) / kQaRowsPerCta;
  return static_cast<size_t>(blocks * (2LL * H + 2) * sizeof(float));
}

int launch_qa_logits_fwd(const void* hidden, int B, int S, int H, const float* w,
                         const float* b, float* logits, cudaStream_t stream) {
  if (!qa_shape_ok(B, S, H)) return 990;
  if (!hidden || !w || !b || !logits) return 991;
  if (!aligned16(hidden) || !aligned16(w)) return 992;
  const long long R = static_cast<long long>(B) * S;
  const int grid = grid_for_rows(static_cast<int>(R), kQaFwdWarps, num_sms() * 16);
  qa_logits_fwd_kernel<<<grid, kQaFwdWarps * 32, 0, stream>>>(
      static_cast<const uint4*>(hidden), R, S, H / 8, w, b, logits);
  SKY_LAUNCH_CHECK();
}

int launch_qa_logits_bwd(const void* hidden, const float* dlogits, int B, int S, int H,
                         const float* w, void* dhidden, float* workspace, float* dw, float* db,
                         cudaStream_t stream) {
  if (!qa_shape_ok(B, S, H)) return 990;
  if (!hidden || !dlogits || !w || !dhidden || !workspace || !dw || !db) return 991;
  if (!aligned16(hidden) || !aligned16(dhidden)) return 992;
  const long long R = static_cast<long long>(B) * S;
  const int row_blocks = static_cast<int>((R + kQaRowsPerCta - 1) / kQaRowsPerCta);
  const int H8 = H / 8;
  dim3 grid((H8 + kQaColChunks - 1) / kQaColChunks, row_blocks);
  qa_logits_bwd_kernel<<<grid, dim3(kQaColChunks, kQaRowLanes), 0, stream>>>(
      static_cast<const uint4*>(hidden), dlogits, R, S, H8, w, static_cast<uint4*>(dhidden),
      workspace);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  const int n = 2 * H + 2;
  qa_logits_finalize_kernel<<<(n + kQaColChunks - 1) / kQaColChunks,
                              dim3(kQaColChunks, kQaRowLanes), 0, stream>>>(workspace, row_blocks,
                                                                             H, dw, db);
  SKY_LAUNCH_CHECK();
}

int launch_qa_span_eval(const float* logits, const int64_t* labels, int B, int S,
                        int max_answer_length, long long ignore_index, SpanEvalAccum* acc,
                        int* pred_spans, float* pred_scores, long long capacity,
                        cudaStream_t stream) {
  if (B < 1 || S < 1 || max_answer_length < 1 || capacity < 0 ||
      static_cast<long long>(B) * S > 0x3fffffffLL)
    return 990;
  if (!logits || !labels || !acc || (capacity > 0 && (!pred_spans || !pred_scores))) return 991;
  qa_span_eval_kernel<<<1, kCeWarps * 32, 0, stream>>>(logits, labels, B, S, max_answer_length,
                                                       ignore_index, acc, pred_spans, pred_scores,
                                                       capacity);
  SKY_LAUNCH_CHECK();
}

namespace {
// blocks per bank of sgd_multi / adam_multi / grad_sumsq_multi: one float4 per thread over the
// largest bank, at most two per SM
int multi_tensor_blocks(long long max_numel) {
  long long blocks = (max_numel / 4 + 255) / 256;
  if (blocks > num_sms() * 2) blocks = num_sms() * 2;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

// launch(std::true_type{}) when the device-side OptimScalars are given, launch(std::false_type{})
// otherwise: the kScalars instantiation of an optimizer kernel
template <typename Launch>
void dispatch_scalars(const OptimScalars* scalars, Launch launch) {
  if (scalars != nullptr)
    launch(std::true_type{});
  else
    launch(std::false_type{});
}
}  // namespace

int launch_sgd_multi(const SgdTensor* d_tensors, int n_tensors, long long max_numel, float lr,
                     float momentum, float weight_decay, float grad_scale, bool zero_grad,
                     cudaStream_t stream, const OptimScalars* scalars) {
  if (n_tensors <= 0) return 0;
  dim3 grid(static_cast<unsigned>(multi_tensor_blocks(max_numel)), n_tensors);
  dispatch_scalars(scalars, [&](auto k) {
    sgd_multi_kernel<decltype(k)::value><<<grid, 256, 0, stream>>>(
        d_tensors, lr, momentum, weight_decay, grad_scale, zero_grad ? 1 : 0, scalars);
  });
  SKY_LAUNCH_CHECK();
}

int launch_adam_multi(const SgdTensor* d_tensors, int n_tensors, long long max_numel, float lr,
                      float beta1, float beta2, float eps, float weight_decay, bool decoupled,
                      const uint64_t* step, float grad_scale, bool zero_grad, cudaStream_t stream,
                      const OptimScalars* scalars) {
  if (n_tensors <= 0) return 0;
  if (step == nullptr) return 906;
  dim3 grid(static_cast<unsigned>(multi_tensor_blocks(max_numel)), n_tensors);
  dispatch_scalars(scalars, [&](auto k) {
    adam_multi_kernel<decltype(k)::value><<<grid, 256, 0, stream>>>(
        d_tensors, lr, beta1, beta2, eps, weight_decay, decoupled ? 1 : 0, step, grad_scale,
        zero_grad ? 1 : 0, scalars);
  });
  SKY_LAUNCH_CHECK();
}

int grad_sumsq_blocks(long long max_numel) { return multi_tensor_blocks(max_numel); }

int launch_grad_sumsq_multi(const SgdTensor* d_tensors, int n_tensors, int blocks,
                            float grad_scale, float* partials, cudaStream_t stream) {
  if (n_tensors <= 0) return 0;
  if (blocks < 1 || partials == nullptr) return 907;
  dim3 grid(static_cast<unsigned>(blocks), n_tensors);
  grad_sumsq_multi_kernel<<<grid, 256, 0, stream>>>(d_tensors, grad_scale, partials);
  SKY_LAUNCH_CHECK();
}

int launch_optim_finalize(const float* partials, int n_partials, const float* extra_sumsq,
                          NormExchangeArgs ex, const uint64_t* step, long long step_offset,
                          int schedule, int warmup, int total, double base_lr, float max_norm,
                          OptimScalars* out, cudaStream_t stream) {
  if (out == nullptr || n_partials < 0) return 908;
  if (ex.n_ranks > 1 && (ex.regions == nullptr || ex.epoch == nullptr || ex.my_pos < 0 ||
                         ex.my_pos >= ex.n_ranks))
    return 909;
  optim_finalize_kernel<<<1, 256, 0, stream>>>(partials, n_partials, extra_sumsq, ex, step,
                                               step_offset, schedule, warmup, total, base_lr, max_norm, out);
  SKY_LAUNCH_CHECK();
}

long long lamb_chunks(long long numel) { return (numel + kLambChunk - 1) / kLambChunk; }

int lamb_prepare(LambSegment* segs, int n_segments, int* chunk_seg, long long cap, int* n_chunks) {
  if (n_segments < 0 || (n_segments > 0 && segs == nullptr) || n_chunks == nullptr) return 970;
  auto al = [](const void* q, uintptr_t a) { return reinterpret_cast<uintptr_t>(q) % a == 0; };
  long long total = 0;
  for (int i = 0; i < n_segments; ++i) {
    LambSegment& s = segs[i];
    if (!s.p || !s.g || !s.m || !s.v || s.numel < 1) return 970;
    if (!al(s.p, 4) || !al(s.g, 4) || !al(s.m, 4) || !al(s.v, 4)) return 970;
    if (s.p_bf16 != nullptr && !al(s.p_bf16, 2)) return 972;
    s.vec = al(s.p, 16) && al(s.g, 16) && al(s.m, 16) && al(s.v, 16) &&
            (s.p_bf16 == nullptr || al(s.p_bf16, 8));
    const long long c = lamb_chunks(s.numel);
    if (total + c > cap || total + c > 0x7fffffffLL) return 970;
    s.chunk0 = static_cast<int>(total);
    s.n_chunks = static_cast<int>(c);
    for (long long k = 0; k < c; ++k) chunk_seg[total + k] = i;
    total += c;
  }
  *n_chunks = static_cast<int>(total);
  return 0;
}

namespace {
// resident blocks of `kernel` (256 threads) on the whole device: the grid of both LAMB passes,
// so that the contiguous chunk ranges run in one wave
template <typename K>
int lamb_grid(K kernel, int n_chunks) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0) != cudaSuccess ||
      per_sm < 1)
    per_sm = 1;
  return n_chunks < per_sm * num_sms() ? n_chunks : per_sm * num_sms();
}
}  // namespace

int launch_lamb_moments(const LambSegment* segs, const int* chunk_seg, int n_chunks, float beta1,
                        float beta2, float eps, const uint64_t* step, float grad_scale,
                        float2* partials, cudaStream_t stream, const OptimScalars* scalars) {
  if (n_chunks == 0) return 0;
  if (n_chunks < 0 || segs == nullptr || chunk_seg == nullptr || partials == nullptr) return 970;
  if (step == nullptr) return 971;
  dispatch_scalars(scalars, [&](auto k) {
    constexpr bool kScalars = decltype(k)::value;
    static const int grid = lamb_grid(lamb_moments_kernel<kScalars>, 1 << 30);
    lamb_moments_kernel<kScalars><<<std::min(grid, n_chunks), 256, 0, stream>>>(
        segs, chunk_seg, n_chunks, beta1, beta2, eps, step, grad_scale, scalars, partials);
  });
  SKY_LAUNCH_CHECK();
}

int launch_lamb_update(const LambSegment* segs, const int* chunk_seg, int n_chunks, float lr,
                       float beta1, float beta2, float eps, const uint64_t* step,
                       const float2* partials, float* ratios, cudaStream_t stream,
                       const OptimScalars* scalars) {
  if (n_chunks == 0) return 0;
  if (n_chunks < 0 || segs == nullptr || chunk_seg == nullptr || partials == nullptr ||
      ratios == nullptr)
    return 970;
  if (step == nullptr) return 971;
  dispatch_scalars(scalars, [&](auto k) {
    constexpr bool kScalars = decltype(k)::value;
    static const int grid = lamb_grid(lamb_update_kernel<kScalars>, 1 << 30);
    lamb_update_kernel<kScalars><<<std::min(grid, n_chunks), 256, 0, stream>>>(
        segs, chunk_seg, n_chunks, lr, beta1, beta2, eps, step, scalars, partials, ratios);
  });
  SKY_LAUNCH_CHECK();
}

int launch_cast_f32_to_bf16(const float* src, void* dst, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  if (blocks < 1) blocks = 1;
  cast_f32_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  SKY_LAUNCH_CHECK();
}
int launch_cast_bf16_to_f32(const void* src, float* dst, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  cast_bf16_f32_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), dst, n);
  SKY_LAUNCH_CHECK();
}

int launch_advance_counter(uint64_t* counter, uint64_t inc, cudaStream_t stream) {
  advance_counter_kernel<<<1, 1, 0, stream>>>(counter, inc);
  SKY_LAUNCH_CHECK();
}
int launch_advance_epoch(uint32_t* counter, uint32_t inc, cudaStream_t stream) {
  advance_epoch_kernel<<<1, 1, 0, stream>>>(counter, inc);
  SKY_LAUNCH_CHECK();
}
int launch_signal_flags(uint32_t* flags, int n, uint32_t inc, cudaStream_t stream) {
  signal_flags_kernel<<<1, 64, 0, stream>>>(flags, n, inc);
  SKY_LAUNCH_CHECK();
}
int launch_wait_flags(const uint32_t* flags, int n, const uint32_t* epoch, uint32_t mult,
                      int* error_flag, cudaStream_t stream) {
  wait_flags_kernel<<<1, 64, 0, stream>>>(flags, n, epoch, mult, error_flag);
  SKY_LAUNCH_CHECK();
}
int launch_spin_ns(uint64_t ns, cudaStream_t stream) {
  spin_ns_kernel<<<1, 1, 0, stream>>>(ns);
  SKY_LAUNCH_CHECK();
}
int launch_record_time(uint64_t* slot, cudaStream_t stream) {
  record_time_kernel<<<1, 1, 0, stream>>>(slot);
  SKY_LAUNCH_CHECK();
}
int launch_spin_factor(const uint64_t* t_start_slot, float factor, cudaStream_t stream) {
  spin_factor_kernel<<<1, 1, 0, stream>>>(t_start_slot, factor);
  SKY_LAUNCH_CHECK();
}

int launch_peer_copy_signal(const void* src, void* dst, long long nbytes, uint32_t* flags,
                            int n_flags, uint32_t inc, cudaStream_t stream) {
  static unsigned int* d_counter = nullptr;
  if (d_counter == nullptr) {
    if (cudaMalloc(&d_counter, sizeof(unsigned int)) != cudaSuccess) return 920;
    cudaMemset(d_counter, 0, sizeof(unsigned int));
  }
  if (nbytes % 16 != 0) return 921;
  long long n16 = nbytes / 16;
  long long blocks = (n16 + 255) / 256;
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  if (blocks < 1) blocks = 1;
  peer_copy_signal_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), n16, flags, n_flags, inc,
      d_counter);
  SKY_LAUNCH_CHECK();
}

static int tied_grid(long long n) {
  long long blocks = ((n >> 2) + 255) / 256;
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  return blocks < 1 ? 1 : static_cast<int>(blocks);
}

int launch_tied_grad_push(const float* src, float* dst, long long n, uint32_t* flag,
                          unsigned int* done, cudaStream_t stream) {
  if (!src || !dst || !flag || !done || n <= 0) return 930;
  if (!aligned16(src) || !aligned16(dst)) return 931;
  tied_grad_push_kernel<<<tied_grid(n), 256, 0, stream>>>(src, dst, n, flag, done);
  SKY_LAUNCH_CHECK();
}
int launch_tied_grad_reduce(float* g, const float* inbox, float* peer_g, long long n,
                            const uint32_t* wait_flag, const uint32_t* epoch, int* error_flag,
                            uint32_t* publish_flag, unsigned int* done, cudaStream_t stream) {
  if (!g || !inbox || !peer_g || !wait_flag || !epoch || !publish_flag || !done || n <= 0)
    return 930;
  if (!aligned16(g) || !aligned16(inbox) || !aligned16(peer_g)) return 931;
  tied_grad_reduce_kernel<<<tied_grid(n), 256, 0, stream>>>(g, inbox, peer_g, n, wait_flag, epoch,
                                                             error_flag, publish_flag, done);
  SKY_LAUNCH_CHECK();
}

}  // namespace sky
