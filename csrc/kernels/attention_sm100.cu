// Fused self-attention for BERT geometry (S = 128 keys per sequence, head_dim = 64) on wgmma.
//
// One CTA of two warpgroups per (batch, head).  With S = 128 a whole score matrix is one 128x128
// tile, so no online-softmax tiling is needed.  Warpgroup w owns query rows 64w .. 64w + 63, and
// every MMA result stays in the wgmma accumulator registers:
//
//   forward : S = Q K^T (wgmma m64n128, K = 64) -> softmax (+mask, +dropout) on the fragments,
//             row max / row sum over the thread's columns and then its quad -> bf16 P as the
//             register A operand of O = P V (wgmma m64n64, K = 128) -> ctx through per-warp
//             staging buffers (128-byte rows)
//   backward: per 64-key half, S = Q K^T and dP = dO V^T (m64n64) -> P = exp2(s - lse),
//             dS = P (dP*keep - delta) on the fragments -> bf16 P / dS into swizzled smem (one copy
//             serves as K-major AND MN-major operand) -> dV = P^T dO, dK = dS^T Q (each warpgroup
//             64 keys), dQ = dS K (each warpgroup its 64 query rows) -> dqkv through the staging
//             buffers
//
// Fragment layout, staging buffer and the register-A wgmma are described in sm100_ptx.cuh.
// Q/K/V/dO tiles come straight out of the fused [tokens, 3H] QKV activation via 2D TMA boxes
// (no head split/merge copies), outputs are written head-merged.
//
// Reference parity: BertSelfAttention.forward, scaelum/model/bert_layers.py:249-275 (scores /
// sqrt(d) + mask, softmax, dropout on probabilities, P V, head merge) and its autograd backward.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>
#include <cstdlib>

#include "api.h"
#include "launch_util.h"
#include "sm100_ptx.cuh"

namespace sky {

int make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer,
                      uint64_t ld_elems, uint32_t box_inner, uint32_t box_outer);

namespace {

constexpr int kS = 128;   // sequence length handled by this kernel
constexpr int kD = 64;    // head dim
constexpr int kTile = kS * kD * 2;  // 16 KB: one [128 x 64] bf16 tile
constexpr int kThreads = 256;       // two warpgroups
constexpr float kLog2e = 1.4426950408889634f;

// byte offset of element (row, col) inside a [128 x 64]-bf16 SWIZZLE_128B tile (16B granularity)
__device__ __forceinline__ uint32_t sw128_offset(int row, int col) {
  const uint32_t chunk = static_cast<uint32_t>(col >> 3) ^ static_cast<uint32_t>(row & 7);
  return static_cast<uint32_t>(row) * 128u + (chunk << 4) + static_cast<uint32_t>(col & 7) * 2u;
}

struct AttnDev {
  const float* mask;  // [B,S] additive or null
  __nv_bfloat16* ctx;
  float* lse;  // [B*heads, S] log2-domain log-sum-exp
  const __nv_bfloat16* ctx_in;
  __nv_bfloat16* dqkv;
  int heads;
  int H;  // heads * 64
  float scale;
  float dropout_p;
  const uint64_t* rng_state;
  uint32_t rng_stream;
};

// ----------------------------------------------------------------------------------------------
// forward
// ----------------------------------------------------------------------------------------------
// Q, K, V, mask, barrier, 8 per-warp staging buffers: 68.6 KB with the alignment slack, so the
// 128-register budget of __launch_bounds__(256, 2) decides the occupancy (2 CTAs per SM)
constexpr int kFwdOffStage = 3 * kTile + 512 + 64;
constexpr int kFwdSmem = kFwdOffStage + 8 * kWarpStageBytes + 1024 /*align*/;

__global__ void __launch_bounds__(kThreads, 2)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTile;
  uint8_t* sV = smem + 2 * kTile;
  float* sMask = reinterpret_cast<float*>(smem + 3 * kTile);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 3 * kTile + 512);

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int lane = tid & 31;
  const int wg = warp >> 2;
  const int bh = blockIdx.x;
  const int b = bh / p.heads;
  const int h = bh % p.heads;
  uint8_t* s_stage = smem + kFwdOffStage + warp * kWarpStageBytes;
  // my fragment rows are query rows q0 and q0 + 8; my columns in every 8-column block 8j + fc + {0,1}
  const int wrow0 = wg * 64 + (warp & 3) * 16;
  const int q0 = wrow0 + (lane >> 2);
  const int fc = (lane & 3) * 2;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
  if (tid < kS) sMask[tid] = p.mask ? p.mask[b * kS + tid] * kLog2e : 0.f;
  __syncthreads();

  if (warp == 0 && elect_one_sync()) {
    mbar_expect_tx(&bars[0], 3 * kTile);
    tma_load_2d(sQ, &tmap_qkv, &bars[0], h * kD, b * kS);
    tma_load_2d(sK, &tmap_qkv, &bars[0], p.H + h * kD, b * kS);
    tma_load_2d(sV, &tmap_qkv, &bars[0], 2 * p.H + h * kD, b * kS);
  }
  mbar_wait(&bars[0], 0);

  // S[my 64 rows, 128 keys] = Q K^T
  float s[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  {
    const uint32_t aq = smem_u32(sQ), ak = smem_u32(sK);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kD / 16; ++k)
      wgmma_k16<128, 0, 0>(s, desc_kmajor(aq, k, kTile, wg * 64), desc_kmajor(ak, k, kTile, 0), 1u);
    wgmma_commit();
    wgmma_wait<0>();
  }

  // ---- softmax on the fragments: row max / row sum over my 32 columns, then over the quad ----
  const float sc = p.scale * kLog2e;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float m0 = sMask[8 * j + fc], m1 = sMask[8 * j + fc + 1];
    s[4 * j] = s[4 * j] * sc + m0;
    s[4 * j + 1] = s[4 * j + 1] * sc + m1;
    s[4 * j + 2] = s[4 * j + 2] * sc + m0;
    s[4 * j + 3] = s[4 * j + 3] * sc + m1;
    mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    s[4 * j] = exp2f(s[4 * j] - mx0);
    s[4 * j + 1] = exp2f(s[4 * j + 1] - mx0);
    s[4 * j + 2] = exp2f(s[4 * j + 2] - mx1);
    s[4 * j + 3] = exp2f(s[4 * j + 3] - mx1);
    sum0 += s[4 * j];
    sum0 += s[4 * j + 1];
    sum1 += s[4 * j + 2];
    sum1 += s[4 * j + 3];
  }
  // the row sum is taken before dropout: it normalises the un-dropped probabilities
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
  const bool has_dropout = p.dropout_p > 0.f;
  if (has_dropout) {
    // element index ((b * heads + h) * S + q) * S + key, as in the host replica (dropout_ref.py)
    const uint64_t seed = dropout_seed(p.rng_state, p.rng_stream);
    const uint32_t thr16 = static_cast<uint32_t>(p.dropout_p * 65536.f);
    const long long row_a = static_cast<long long>(bh) * kS + q0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t m = frag_keep_bits(seed, thr16, row_a, (j >> 3) * 64, kS, lane, j & 7);
      s[4 * j] = (m & 1u) ? s[4 * j] : 0.f;
      s[4 * j + 1] = (m & 2u) ? s[4 * j + 1] : 0.f;
      s[4 * j + 2] = (m & 4u) ? s[4 * j + 2] : 0.f;
      s[4 * j + 3] = (m & 8u) ? s[4 * j + 3] : 0.f;
    }
  }
  if (p.lse != nullptr && (lane & 3) == 0) {
    float* l = p.lse + static_cast<long long>(bh) * kS;
    l[q0] = mx0 + log2f(sum0);
    l[q0 + 8] = mx1 + log2f(sum1);
  }

  // O[my rows, d] = P V: A = bf16 P straight from the score fragments (8 K steps of 16 keys),
  // B = V (MN-major)
  uint32_t pa[kS / 16][4];
#pragma unroll
  for (int k = 0; k < kS / 16; ++k) frag_to_a(s, k, pa[k]);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  {
    const uint32_t av = smem_u32(sV);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kS / 16; ++k)
      wgmma_rs_k16<64, 1>(o, pa[k], desc_mnmajor(av, k, kTile, 0), 1u);
    wgmma_commit();
    wgmma_wait<0>();
  }

  const float keep_scale = has_dropout ? 1.f / (1.f - p.dropout_p) : 1.f;
  const float inv0 = keep_scale / sum0, inv1 = keep_scale / sum1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j] *= inv0;
    o[4 * j + 1] *= inv0;
    o[4 * j + 2] *= inv1;
    o[4 * j + 3] *= inv1;
  }
  frag_store_bf16(o, s_stage, lane, p.ctx, p.H, static_cast<long long>(b) * kS + wrow0, INT_MAX,
                  h * kD, p.H);
}

// ----------------------------------------------------------------------------------------------
// backward
// ----------------------------------------------------------------------------------------------
// 8 bf16 tiles (Q, K, V, dO, P0, P1, dS0, dS1) + mask, lse, delta + barrier + 8 per-warp staging
// buffers: 152.6 KB, one CTA per SM
constexpr int kBwdOffVec = 8 * kTile;  // sMask | sLse | sDelta, 128 floats each
constexpr int kBwdOffBar = kBwdOffVec + 3 * kS * 4;
constexpr int kBwdOffStage = kBwdOffBar + 64;
constexpr int kBwdSmem = kBwdOffStage + 8 * kWarpStageBytes + 1024 /*align*/;

__global__ void __launch_bounds__(kThreads, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                     const __grid_constant__ CUtensorMap tmap_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTile;
  uint8_t* sV = smem + 2 * kTile;
  uint8_t* sdO = smem + 3 * kTile;
  uint8_t* sP = smem + 4 * kTile;   // 2 blocks: keys 0..63 | 64..127
  uint8_t* sdS = smem + 6 * kTile;  // 2 blocks
  float* sMask = reinterpret_cast<float*>(smem + kBwdOffVec);
  float* sLse = sMask + kS;
  float* sDelta = sLse + kS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kBwdOffBar);

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int lane = tid & 31;
  const int wg = warp >> 2;
  const int bh = blockIdx.x;
  const int b = bh / p.heads;
  const int h = bh % p.heads;
  uint8_t* s_stage = smem + kBwdOffStage + warp * kWarpStageBytes;
  const int wrow0 = wg * 64 + (warp & 3) * 16;
  const int q0 = wrow0 + (lane >> 2);
  const int fc = (lane & 3) * 2;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
  if (tid < kS) sMask[tid] = p.mask ? p.mask[b * kS + tid] * kLog2e : 0.f;
  __syncthreads();

  if (warp == 0 && elect_one_sync()) {
    mbar_expect_tx(&bars[0], 4 * kTile);
    tma_load_2d(sQ, &tmap_qkv, &bars[0], h * kD, b * kS);
    tma_load_2d(sK, &tmap_qkv, &bars[0], p.H + h * kD, b * kS);
    tma_load_2d(sV, &tmap_qkv, &bars[0], 2 * p.H + h * kD, b * kS);
    tma_load_2d(sdO, &tmap_do, &bars[0], h * kD, b * kS);
  }

  // delta = rowsum(dO * O) and lse, one thread per query row while the loads run
  if (tid < kS) {
    float delta = 0.f;
    const long long off = (static_cast<long long>(b) * kS + tid) * p.H + h * kD;
    const uint4* o4 = reinterpret_cast<const uint4*>(p.ctx_in + off);
    // dO row read from global (also in smem, but swizzled; global read is simpler and cached)
    const uint4* d4 = reinterpret_cast<const uint4*>(
        reinterpret_cast<const __nv_bfloat16*>(p.ctx) + off);  // p.ctx aliases dctx in bwd
#pragma unroll
    for (int i = 0; i < kD / 8; ++i) {
      const uint4 a = o4[i];
      const uint4 g = d4[i];
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 x = unpack_bf16x2(aw[t]);
        const float2 y = unpack_bf16x2(gw[t]);
        delta += x.x * y.x + x.y * y.y;
      }
    }
    sDelta[tid] = delta;
    sLse[tid] = p.lse[static_cast<long long>(bh) * kS + tid];
  }
  __syncthreads();
  const float lse0 = sLse[q0], lse1 = sLse[q0 + 8];
  const float delta0 = sDelta[q0], delta1 = sDelta[q0 + 8];

  mbar_wait(&bars[0], 0);
  const uint32_t aQ = smem_u32(sQ), aK = smem_u32(sK), aV = smem_u32(sV), adO = smem_u32(sdO);
  const uint32_t aP = smem_u32(sP), adS = smem_u32(sdS);

  const float sc = p.scale * kLog2e;
  const bool has_dropout = p.dropout_p > 0.f;
  uint64_t seed = 0;
  uint32_t thr16 = 0;
  float dscale = 1.f;
  if (has_dropout) {
    seed = dropout_seed(p.rng_state, p.rng_stream);
    thr16 = static_cast<uint32_t>(p.dropout_p * 65536.f);
    dscale = 1.f / (1.f - p.dropout_p);
  }
  const long long row_a = static_cast<long long>(bh) * kS + q0;
#pragma unroll 1
  for (int kh = 0; kh < 2; ++kh) {  // 64 keys at a time: S and dP of those keys, my 64 queries
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      s[i] = 0.f;
      dp[i] = 0.f;
    }
    acc_fence(s);
    acc_fence(dp);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kD / 16; ++k)
      wgmma_k16<64, 0, 0>(s, desc_kmajor(aQ, k, kTile, wg * 64), desc_kmajor(aK, k, kTile, kh * 64),
                          1u);
#pragma unroll
    for (int k = 0; k < kD / 16; ++k)
      wgmma_k16<64, 0, 0>(dp, desc_kmajor(adO, k, kTile, wg * 64),
                          desc_kmajor(aV, k, kTile, kh * 64), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    uint8_t* bp = sP + kh * kTile;
    uint8_t* bd = sdS + kh * kTile;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + fc;  // key kh * 64 + col
      const float m0 = sMask[kh * 64 + col], m1 = sMask[kh * 64 + col + 1];
      float pr[4], ds[4];
      pr[0] = exp2f(s[4 * j] * sc + m0 - lse0);
      pr[1] = exp2f(s[4 * j + 1] * sc + m1 - lse0);
      pr[2] = exp2f(s[4 * j + 2] * sc + m0 - lse1);
      pr[3] = exp2f(s[4 * j + 3] * sc + m1 - lse1);
      if (has_dropout) {
        const uint32_t m = frag_keep_bits(seed, thr16, row_a, kh * 64, kS, lane, j);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const bool keep = (m >> t) & 1u;
          const float pj = pr[t];
          // dS uses the un-dropped P; the dropped/scaled P feeds dV
          ds[t] = pj * ((keep ? dp[4 * j + t] * dscale : 0.f) - (t < 2 ? delta0 : delta1)) *
                  p.scale;
          pr[t] = keep ? pj * dscale : 0.f;
        }
      } else {
#pragma unroll
        for (int t = 0; t < 4; ++t)
          ds[t] = pr[t] * (dp[4 * j + t] - (t < 2 ? delta0 : delta1)) * p.scale;
      }
      const uint32_t off0 = sw128_offset(q0, col), off1 = sw128_offset(q0 + 8, col);
      *reinterpret_cast<uint32_t*>(bp + off0) = pack_bf16x2(pr[0], pr[1]);
      *reinterpret_cast<uint32_t*>(bp + off1) = pack_bf16x2(pr[2], pr[3]);
      *reinterpret_cast<uint32_t*>(bd + off0) = pack_bf16x2(ds[0], ds[1]);
      *reinterpret_cast<uint32_t*>(bd + off1) = pack_bf16x2(ds[2], ds[3]);
    }
  }
  fence_proxy_async_smem();   // P / dS (generic-proxy stores) -> wgmma (async-proxy reads)
  __syncthreads();            // dV / dK need the P / dS rows of both warpgroups

  // dV[key, d] = sum_q P[q,key] dO[q,d] : A = P (MN-major, one key-chunk per block), B = dO (MN)
  // dK[key, d] = sum_q dS[q,key] Q[q,d] : A = dS (MN-major),                         B = Q  (MN)
  // warpgroup w: keys 64w .. 64w + 63 of dV / dK; query rows 64w .. 64w + 63 of
  // dQ[q, d] = sum_key dS[q,key] K[key,d] : A = dS (K-major, 2 K-blocks), B = K (MN-major)
  float dv[32], dk[32], dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    dv[i] = 0.f;
    dk[i] = 0.f;
    dq[i] = 0.f;
  }
  acc_fence(dv);
  acc_fence(dk);
  acc_fence(dq);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kS / 16; ++k)
    wgmma_k16<64, 1, 1>(dv, desc_mnmajor(aP, k, kTile, wg), desc_mnmajor(adO, k, kTile, 0), 1u);
#pragma unroll
  for (int k = 0; k < kS / 16; ++k)
    wgmma_k16<64, 1, 1>(dk, desc_mnmajor(adS, k, kTile, wg), desc_mnmajor(aQ, k, kTile, 0), 1u);
  wgmma_commit();
#pragma unroll
  for (int k = 0; k < kS / 16; ++k)
    wgmma_k16<64, 0, 1>(dq, desc_kmajor(adS, k, kTile, wg * 64), desc_mnmajor(aK, k, kTile, 0), 1u);
  wgmma_commit();

  const long long grow0 = static_cast<long long>(b) * kS + wrow0;  // my warp's keys / queries
  const int ld = 3 * p.H;
  wgmma_wait<1>();  // dV and dK leave while dQ is still in flight
  frag_store_bf16(dv, s_stage, lane, p.dqkv, ld, grow0, INT_MAX, 2 * p.H + h * kD, ld);
  frag_store_bf16(dk, s_stage, lane, p.dqkv, ld, grow0, INT_MAX, p.H + h * kD, ld);
  wgmma_wait<0>();
  frag_store_bf16(dq, s_stage, lane, p.dqkv, ld, grow0, INT_MAX, h * kD, ld);
}

}  // namespace

// S = 128 runs the single-tile kernels of this file; every other length (and S = 128 when
// SKY_ATTN_TILED=1, for A/B comparisons) the flash-style tiled kernels of attention_tiled_sm100.cu
static bool force_tiled() {
  static int v = -1;
  if (v < 0) {
    const char* e = std::getenv("SKY_ATTN_TILED");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

int launch_attention_fwd(const AttnArgs& a, cudaStream_t stream) {
  if (a.head_dim != kD) return 930;
  if (a.S != kS || force_tiled()) return launch_attention_fwd_tiled(a, stream);
  if (a.dropout_p > 0.f && a.rng_state == nullptr) return 903;
  const int H = a.heads * kD;
  CUtensorMap tm;
  int rc = make_tmap_bf16_2d(&tm, a.qkv, 3ull * H, static_cast<uint64_t>(a.B) * kS, 3ull * H, 64,
                             128);
  if (rc) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attention_fwd_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = true;
  }
  AttnDev d;
  d.mask = a.mask;
  d.ctx = reinterpret_cast<__nv_bfloat16*>(a.ctx);
  d.lse = a.lse;
  d.ctx_in = nullptr;
  d.dqkv = nullptr;
  d.heads = a.heads;
  d.H = H;
  d.scale = a.scale;
  d.dropout_p = a.dropout_p;
  d.rng_state = a.rng_state;
  d.rng_stream = a.rng_stream;
  cudaError_t le = launch_pdl(attention_fwd_kernel, dim3(a.B * a.heads), dim3(kThreads), kFwdSmem, stream, tm, d);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

int launch_attention_bwd(const AttnArgs& a, cudaStream_t stream) {
  if (a.head_dim != kD) return 930;
  if (a.S != kS || force_tiled()) return launch_attention_bwd_tiled(a, stream);
  if (a.dropout_p > 0.f && a.rng_state == nullptr) return 903;
  if (a.lse == nullptr || a.ctx == nullptr || a.dctx == nullptr) return 931;
  const int H = a.heads * kD;
  CUtensorMap tm, tdo;
  int rc = make_tmap_bf16_2d(&tm, a.qkv, 3ull * H, static_cast<uint64_t>(a.B) * kS, 3ull * H, 64,
                             128);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tdo, a.dctx, static_cast<uint64_t>(H), static_cast<uint64_t>(a.B) * kS,
                         static_cast<uint64_t>(H), 64, 128);
  if (rc) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = true;
  }
  AttnDev d;
  d.mask = a.mask;
  // in the backward kernel `ctx` carries dctx (gradient wrt attention output) and `ctx_in` the
  // saved forward output
  d.ctx = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a.dctx));
  d.ctx_in = reinterpret_cast<const __nv_bfloat16*>(a.ctx);
  d.lse = a.lse;
  d.dqkv = reinterpret_cast<__nv_bfloat16*>(a.dqkv);
  d.heads = a.heads;
  d.H = H;
  d.scale = a.scale;
  d.dropout_p = a.dropout_p;
  d.rng_state = a.rng_state;
  d.rng_stream = a.rng_stream;
  cudaError_t le = launch_pdl(attention_bwd_kernel, dim3(a.B * a.heads), dim3(kThreads), kBwdSmem, stream, tm, tdo, d);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace sky
