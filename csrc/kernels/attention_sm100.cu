// Fused self-attention on wgmma for head_dim = 64 and any sequence length S % 8 == 0.
//
// Every kernel runs two warpgroups (256 threads) on a 128-row tile; warpgroup w owns rows (query
// rows, or keys in the dK / dV kernel) 64w .. 64w + 63, and every MMA result stays in the wgmma
// accumulator registers.  The kernels are loops over the same fragment steps:
//
//   scores  S = Q K^T (m64nN, K = 64) for the warpgroup's 64 query rows, scaled and masked in the
//           log2 domain; row max / row sum over the thread's columns and then its quad
//   step A  S and dP = dO V^T of 64 keys -> P = exp2(s - lse), dS = P (dP*keep - delta) on the
//           fragments -> bf16 P / dS into swizzled smem (one copy serves as K-major AND MN-major
//           operand)
//   step B  dV += P^T dO, dK += dS^T Q for the warpgroup's 64 keys
//   step C  dQ += dS K for the warpgroup's 64 query rows
//
// S = 128 (the BERT geometry): one CTA per (batch, head); the whole score matrix is one tile.
//   forward : scores (m64n128) -> softmax (+mask, +dropout) on the fragments -> bf16 P as the
//             register A operand of O = P V (m64n64, K = 128)
//   backward: step A for both 64-key halves, then B and C
// Any other S (and S = 128 with SKY_ATTN_TILED=1): flash-style tiling over 128-row tiles.
//   forward : one CTA per (batch, head, query tile), loop over double-buffered key tiles with an
//             online softmax: running max and sum per fragment row, O rescaled by alpha before
//             O += P V
//   backward: dQ kernel (CTA per query tile, loop over key tiles: A then C) and dK/dV kernel (CTA
//             per key tile, loop over query tiles: A then B); the accumulators stay in registers
//             across the loop
//
// Q/K/V/dO tiles come straight out of the fused [tokens, 3H] QKV activation via 3D TMA boxes
// (C, S, B) (no head split/merge copies); outputs are written head-merged through per-warp
// staging buffers as 128-byte rows.  Ragged last tiles: TMA zero-fills rows past the end of a
// sequence, keys past the end get the additive mask -1e30, query rows past the end get
// lse = +1e30 and delta = 0 in the backward (so their P = dS = 0), and no row past the end is
// stored.  Dropout indexes its counter-based mask by ((b * heads + h) * S + q) * S + key, as the
// host replica does (skycomputing_b200/ops/dropout_ref.py).  Fragment layout, staging buffer and
// the register-A wgmma are described in sm100_ptx.cuh.
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

int make_tmap_bf16_3d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t middle,
                      uint64_t outer, uint64_t ld_middle_elems, uint64_t ld_outer_elems,
                      uint32_t box_inner, uint32_t box_middle);

namespace {

constexpr int kT = 128;             // query rows / keys per tile, and the single-tile S
constexpr int kD = 64;              // head dim
constexpr int kTile = kT * kD * 2;  // 16 KB: one [128 x 64] bf16 tile
constexpr int kThreads = 256;       // two warpgroups
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kNegBig = -1.0e30f;  // additive mask of keys past the end of the sequence

// byte offset of element (row, col) inside a [128 x 64]-bf16 SWIZZLE_128B tile (16B granularity)
__device__ __forceinline__ uint32_t sw128_offset(int row, int col) {
  const uint32_t chunk = static_cast<uint32_t>(col >> 3) ^ static_cast<uint32_t>(row & 7);
  return static_cast<uint32_t>(row) * 128u + (chunk << 4) + static_cast<uint32_t>(col & 7) * 2u;
}

struct AttnDev {
  const float* mask;            // [B, S] additive or null
  __nv_bfloat16* ctx;           // fwd: output [B*S, H]
  float* lse;                   // [B*heads, S] log2-domain log-sum-exp (fwd: out or null, bwd: in)
  const __nv_bfloat16* ctx_in;  // bwd: saved forward output
  const __nv_bfloat16* dctx;    // bwd: gradient of the attention output
  __nv_bfloat16* dqkv;          // bwd: [B*S, 3H]
  int S, heads, H, n_tiles;
  float scale, dropout_p;
  const uint64_t* rng_state;
  uint32_t rng_stream;
};

// SWIZZLE_128B tiles need 1024-byte alignment
__device__ __forceinline__ uint8_t* align_smem(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) &
                                    ~static_cast<uintptr_t>(1023));
}

// A thread's place in its warpgroup's fragments: its fragment rows are tile rows q0 and q0 + 8
// (q0 = wrow0 + lane / 4, wrow0 the warp's first row), its columns 8j + fc + {0, 1} of every
// 8-column block j.
struct Frag {
  int tid, warp, lane, wg, wrow0, q0, fc;
};
__device__ __forceinline__ Frag frag_of_thread() {
  Frag f;
  f.tid = threadIdx.x;
  f.warp = __shfl_sync(0xffffffffu, f.tid >> 5, 0);
  f.lane = f.tid & 31;
  f.wg = f.warp >> 2;
  f.wrow0 = f.wg * 64 + (f.warp & 3) * 16;
  f.q0 = f.wrow0 + (f.lane >> 2);
  f.fc = (f.lane & 3) * 2;
  return f;
}

// additive mask (log2 domain) of keys key0 .. key0 + 127 -> sMask; keys past the end get -1e30
__device__ __forceinline__ void load_mask(float* sMask, const AttnDev& p, int b, int S, int key0,
                                          int tid) {
  if (tid < kT) {
    const int k = key0 + tid;
    sMask[tid] = k < S ? (p.mask ? p.mask[b * S + k] * kLog2e : 0.f) : kNegBig;
  }
}

// acc (+)= A B^T over the head dim: A = rows a_row0 .. a_row0 + 63 of a K-major [128 x 64] tile,
// B = rows b_row0 .. b_row0 + N - 1 of another (S = Q K^T, dP = dO V^T).  Issue only.
template <int N>
__device__ __forceinline__ void mma_rows(float (&acc)[N / 2], uint32_t a, int a_row0, uint32_t b,
                                         int b_row0) {
#pragma unroll
  for (int k = 0; k < kD / 16; ++k)
    wgmma_k16<N, 0, 0>(acc, desc_kmajor(a, k, kTile, a_row0), desc_kmajor(b, k, kTile, b_row0), 1u);
}

// scores in the log2 domain: s = s * sc + the mask of its key (sMask indexed by fragment column)
template <int NREG>
__device__ __forceinline__ void scale_mask(float (&s)[NREG], const float* sMask, float sc, int fc) {
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    const float m0 = sMask[8 * j + fc], m1 = sMask[8 * j + fc + 1];
    s[4 * j] = s[4 * j] * sc + m0;
    s[4 * j + 1] = s[4 * j + 1] * sc + m1;
    s[4 * j + 2] = s[4 * j + 2] * sc + m0;
    s[4 * j + 3] = s[4 * j + 3] * sc + m1;
  }
}

// mx0 / mx1 = max of themselves and the thread's two fragment rows, then over the quad
template <int NREG>
__device__ __forceinline__ void row_max(const float (&s)[NREG], float& mx0, float& mx1) {
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
}

// s = exp2(s - row max); sum0 / sum1 += the thread's part of each row's sum
template <int NREG>
__device__ __forceinline__ void exp_rows(float (&s)[NREG], float mx0, float mx1, float& sum0,
                                         float& sum1) {
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    s[4 * j] = exp2f(s[4 * j] - mx0);
    s[4 * j + 1] = exp2f(s[4 * j + 1] - mx0);
    s[4 * j + 2] = exp2f(s[4 * j + 2] - mx1);
    s[4 * j + 3] = exp2f(s[4 * j + 3] - mx1);
    sum0 += s[4 * j];
    sum0 += s[4 * j + 1];
    sum1 += s[4 * j + 2];
    sum1 += s[4 * j + 3];
  }
}

__device__ __forceinline__ void quad_sum(float& sum0, float& sum1) {
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
}

// o (+)= P V over 128 keys: A = bf16 P straight from the score fragments (8 K steps of 16 keys),
// B = V (MN-major).  Waits for the result.
__device__ __forceinline__ void mma_pv(float (&o)[32], const float (&s)[64], uint32_t aV) {
  uint32_t pa[kT / 16][4];
#pragma unroll
  for (int k = 0; k < kT / 16; ++k) frag_to_a(s, k, pa[k]);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kT / 16; ++k)
    wgmma_rs_k16<64, 1>(o, pa[k], desc_mnmajor(aV, k, kTile, 0), 1u);
  wgmma_commit();
  wgmma_wait<0>();
}

// lse and delta = rowsum(dO * O) of the query rows q_base + tid (tid < 128) -> sLse / sDelta.
// Rows past the sequence end get lse = +1e30 and delta = 0, which makes their P and dS exactly 0.
__device__ __forceinline__ void load_bwd_rows(const AttnDev& p, int b, int h, int bh, int S,
                                              int q_base, int tid, float* sLse, float* sDelta) {
  if (tid >= kT) return;
  const int q = q_base + tid;
  float delta = 0.f, lse = 1.0e30f;
  if (q < S) {
    const long long off = (static_cast<long long>(b) * S + q) * p.H + h * kD;
    const uint4* o4 = reinterpret_cast<const uint4*>(p.ctx_in + off);
    const uint4* d4 = reinterpret_cast<const uint4*>(p.dctx + off);
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
    lse = p.lse[static_cast<long long>(bh) * S + q];
  }
  sDelta[tid] = delta;
  sLse[tid] = lse;
}

// lse / delta of a thread's two fragment rows
struct BwdRows {
  float lse0, lse1, delta0, delta1;
};

// Step A: S = Q K^T and dP = dO V^T of the warpgroup's 64 query rows (q_row0 of the Q / dO tiles)
// and keys k_row0 .. k_row0 + 63 of the K / V tiles; then on the fragments P = exp2(s - lse) and
// dS = P (dP * keep / (1 - p) - delta) * scale.  The dropped / scaled P (if kP) and dS go to the
// swizzled [128 x 64] blocks bp / bd, indexed [query][key].  sMask holds the keys' mask; row_a
// (the fragment's first query row), col0 (the first key) and S locate the dropout elements.
template <bool kP>
__device__ __forceinline__ void bwd_p_ds(const Frag& f, uint32_t aQ, uint32_t adO, uint32_t aK,
                                         uint32_t aV, int k_row0, const float* sMask,
                                         const BwdRows& r, float sc, float scale,
                                         const Dropout& dr, long long row_a, int col0, int S,
                                         uint8_t* bp, uint8_t* bd) {
  float s[32], dp[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    s[i] = 0.f;
    dp[i] = 0.f;
  }
  acc_fence(s);
  acc_fence(dp);
  wgmma_fence();
  mma_rows<64>(s, aQ, f.wg * 64, aK, k_row0);
  mma_rows<64>(dp, adO, f.wg * 64, aV, k_row0);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = 8 * j + f.fc;
    const float m0 = sMask[col], m1 = sMask[col + 1];
    float pr[4], ds[4];
    pr[0] = exp2f(s[4 * j] * sc + m0 - r.lse0);
    pr[1] = exp2f(s[4 * j + 1] * sc + m1 - r.lse0);
    pr[2] = exp2f(s[4 * j + 2] * sc + m0 - r.lse1);
    pr[3] = exp2f(s[4 * j + 3] * sc + m1 - r.lse1);
    if (dr.on) {
      const uint32_t m = frag_keep_bits(dr.seed, dr.thr16, row_a, col0, S, f.lane, j);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const bool keep = (m >> t) & 1u;
        const float pj = pr[t];
        // dS uses the un-dropped P; the dropped/scaled P feeds dV
        ds[t] = pj * ((keep ? dp[4 * j + t] * dr.scale : 0.f) - (t < 2 ? r.delta0 : r.delta1)) *
                scale;
        pr[t] = keep ? pj * dr.scale : 0.f;
      }
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t)
        ds[t] = pr[t] * (dp[4 * j + t] - (t < 2 ? r.delta0 : r.delta1)) * scale;
    }
    const uint32_t off0 = sw128_offset(f.q0, col), off1 = sw128_offset(f.q0 + 8, col);
    if (kP) {
      *reinterpret_cast<uint32_t*>(bp + off0) = pack_bf16x2(pr[0], pr[1]);
      *reinterpret_cast<uint32_t*>(bp + off1) = pack_bf16x2(pr[2], pr[3]);
    }
    *reinterpret_cast<uint32_t*>(bd + off0) = pack_bf16x2(ds[0], ds[1]);
    *reinterpret_cast<uint32_t*>(bd + off1) = pack_bf16x2(ds[2], ds[3]);
  }
}

// Step B: dV[key, d] += sum_q P[q,key] dO[q,d], dK[key, d] += sum_q dS[q,key] Q[q,d] over the
// tile's 128 query rows for the warpgroup's 64 keys: A = P / dS (MN-major, key chunk wg of the
// two blocks), B = dO / Q (MN-major).  Issue only.
__device__ __forceinline__ void mma_dkv(float (&dv)[32], float (&dk)[32], uint32_t aP, uint32_t adS,
                                        uint32_t adO, uint32_t aQ, int wg) {
#pragma unroll
  for (int k = 0; k < kT / 16; ++k)
    wgmma_k16<64, 1, 1>(dv, desc_mnmajor(aP, k, kTile, wg), desc_mnmajor(adO, k, kTile, 0), 1u);
#pragma unroll
  for (int k = 0; k < kT / 16; ++k)
    wgmma_k16<64, 1, 1>(dk, desc_mnmajor(adS, k, kTile, wg), desc_mnmajor(aQ, k, kTile, 0), 1u);
}

// Step C: dQ[q, d] += sum_key dS[q,key] K[key,d] over the tile's 128 keys for the warpgroup's 64
// query rows: A = dS (K-major, 2 K-blocks), B = K (MN-major).  Issue only.
__device__ __forceinline__ void mma_dq(float (&dq)[32], uint32_t adS, uint32_t aK, int wg) {
#pragma unroll
  for (int k = 0; k < kT / 16; ++k)
    wgmma_k16<64, 0, 1>(dq, desc_kmajor(adS, k, kTile, wg * 64), desc_mnmajor(aK, k, kTile, 0), 1u);
}

// ----------------------------------------------------------------------------------------------
// forward
// ----------------------------------------------------------------------------------------------
// S = 128: Q, K, V, mask, barrier, 8 per-warp staging buffers: 68.6 KB with the alignment slack,
// so the 128-register budget of __launch_bounds__(256, 2) decides the occupancy (2 CTAs per SM)
constexpr int kFwdOffStage = 3 * kTile + 512 + 64;
constexpr int kFwdSmem = kFwdOffStage + 8 * kWarpStageBytes + 1024 /*align*/;

__global__ void __launch_bounds__(kThreads, 2)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTile;
  uint8_t* sV = smem + 2 * kTile;
  float* sMask = reinterpret_cast<float*>(smem + 3 * kTile);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 3 * kTile + 512);

  const Frag f = frag_of_thread();
  const int bh = blockIdx.x;
  const int b = bh / p.heads;
  const int h = bh % p.heads;
  uint8_t* s_stage = smem + kFwdOffStage + f.warp * kWarpStageBytes;

  if (f.tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
  load_mask(sMask, p, b, kT, 0, f.tid);
  __syncthreads();

  if (f.warp == 0 && elect_one_sync()) {
    mbar_expect_tx(&bars[0], 3 * kTile);
    tma_load_3d(sQ, &tmap_qkv, &bars[0], h * kD, 0, b);
    tma_load_3d(sK, &tmap_qkv, &bars[0], p.H + h * kD, 0, b);
    tma_load_3d(sV, &tmap_qkv, &bars[0], 2 * p.H + h * kD, 0, b);
  }
  mbar_wait(&bars[0], 0);

  // S[my 64 rows, 128 keys] = Q K^T
  float s[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  wgmma_fence();
  mma_rows<128>(s, smem_u32(sQ), f.wg * 64, smem_u32(sK), 0);
  wgmma_commit();
  wgmma_wait<0>();

  scale_mask(s, sMask, p.scale * kLog2e, f.fc);
  float mx0 = -INFINITY, mx1 = -INFINITY;
  row_max(s, mx0, mx1);
  float sum0 = 0.f, sum1 = 0.f;
  exp_rows(s, mx0, mx1, sum0, sum1);
  // the row sum is taken before dropout: it normalises the un-dropped probabilities
  quad_sum(sum0, sum1);
  const Dropout dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  if (dr.on) frag_dropout(s, dr.seed, dr.thr16, 1.f, static_cast<long long>(bh) * kT + f.q0, 0, kT,
                          f.lane);
  if (p.lse != nullptr && (f.lane & 3) == 0) {
    float* l = p.lse + static_cast<long long>(bh) * kT;
    l[f.q0] = mx0 + log2f(sum0);
    l[f.q0 + 8] = mx1 + log2f(sum1);
  }

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mma_pv(o, s, smem_u32(sV));

  const float inv0 = dr.scale / sum0, inv1 = dr.scale / sum1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j] *= inv0;
    o[4 * j + 1] *= inv0;
    o[4 * j + 2] *= inv1;
    o[4 * j + 3] *= inv1;
  }
  frag_store_bf16(o, s_stage, f.lane, p.ctx, p.H, static_cast<long long>(b) * kT + f.wrow0, INT_MAX,
                  h * kD, p.H);
}

// tiled: Q, 2 x (K, V), mask, barriers, 8 per-warp staging buffers
constexpr int kFwdTOffStage = 5 * kTile + 512 + 64;
constexpr int kFwdTSmem = kFwdTOffStage + 8 * kWarpStageBytes + 1024 /*align*/;

__global__ void __launch_bounds__(kThreads, 1)
attention_fwd_tiled_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + kTile;  // [2 buffers][K, V]
  float* sMask = reinterpret_cast<float*>(smem + 5 * kTile);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * kTile + 512);
  uint64_t* bar_q = &bars[0];
  uint64_t* bar_kv = &bars[1];  // [2]

  const Frag f = frag_of_thread();
  const int qt = blockIdx.x % p.n_tiles;
  const int bh = blockIdx.x / p.n_tiles;
  const int b = bh / p.heads;
  const int h = bh % p.heads;
  uint8_t* s_stage = smem + kFwdTOffStage + f.warp * kWarpStageBytes;

  if (f.tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
  __syncthreads();

  const bool issuer = f.warp == 0 && elect_one_sync();
  if (issuer) {
    mbar_expect_tx(bar_q, kTile);
    tma_load_3d(sQ, &tmap_qkv, bar_q, h * kD, qt * kT, b);
    mbar_expect_tx(&bar_kv[0], 2 * kTile);
    tma_load_3d(sKV, &tmap_qkv, &bar_kv[0], p.H + h * kD, 0, b);
    tma_load_3d(sKV + kTile, &tmap_qkv, &bar_kv[0], 2 * p.H + h * kD, 0, b);
  }

  const float sc = p.scale * kLog2e;
  const Dropout dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  const long long row_a = static_cast<long long>(bh) * p.S + qt * kT + f.q0;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  // running max and (this thread's part of the) sum of the two fragment rows
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const uint32_t aQ = smem_u32(sQ);

  mbar_wait(bar_q, 0);
  for (int j = 0; j < p.n_tiles; ++j) {
    const int buf = j & 1;
    uint8_t* sK = sKV + buf * 2 * kTile;
    load_mask(sMask, p, b, p.S, j * kT, f.tid);
    if (issuer && j + 1 < p.n_tiles) {  // the other buffer's tile (j - 1) is fully consumed
      uint8_t* nK = sKV + (buf ^ 1) * 2 * kTile;
      mbar_expect_tx(&bar_kv[buf ^ 1], 2 * kTile);
      tma_load_3d(nK, &tmap_qkv, &bar_kv[buf ^ 1], p.H + h * kD, (j + 1) * kT, b);
      tma_load_3d(nK + kTile, &tmap_qkv, &bar_kv[buf ^ 1], 2 * p.H + h * kD, (j + 1) * kT, b);
    }
    mbar_wait(&bar_kv[buf], (j >> 1) & 1);
    __syncthreads();  // sMask visible

    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    acc_fence(s);
    wgmma_fence();
    mma_rows<128>(s, aQ, f.wg * 64, smem_u32(sK), 0);
    wgmma_commit();
    wgmma_wait<0>();

    scale_mask(s, sMask, sc, f.fc);
    float mx0 = m0, mx1 = m1;
    row_max(s, mx0, mx1);
    // 0 on the first tile (m = -inf, mx finite: key 0 of a sequence is never past its end)
    const float alpha0 = exp2f(m0 - mx0), alpha1 = exp2f(m1 - mx1);
    float sum0 = 0.f, sum1 = 0.f;
    exp_rows(s, mx0, mx1, sum0, sum1);
    l0 = l0 * alpha0 + sum0;  // before dropout, as in the single-tile kernel
    l1 = l1 * alpha1 + sum1;
    m0 = mx0;
    m1 = mx1;
    if (dr.on) frag_dropout(s, dr.seed, dr.thr16, 1.f, row_a, j * kT, p.S, f.lane);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= alpha0;
      o[4 * i + 1] *= alpha0;
      o[4 * i + 2] *= alpha1;
      o[4 * i + 3] *= alpha1;
    }
    mma_pv(o, s, smem_u32(sK + kTile));
    __syncthreads();  // K / V of this buffer and sMask consumed before they are refilled
  }

  quad_sum(l0, l1);
  const int q = qt * kT + f.q0;
  if (p.lse != nullptr && (f.lane & 3) == 0) {
    float* l = p.lse + static_cast<long long>(bh) * p.S;
    if (q < p.S) l[q] = m0 + log2f(l0);
    if (q + 8 < p.S) l[q + 8] = m1 + log2f(l1);
  }
  const float inv0 = dr.scale / l0, inv1 = dr.scale / l1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j] *= inv0;
    o[4 * j + 1] *= inv0;
    o[4 * j + 2] *= inv1;
    o[4 * j + 3] *= inv1;
  }
  frag_store_bf16(o, s_stage, f.lane, p.ctx, p.H,
                  static_cast<long long>(b) * p.S + qt * kT + f.wrow0, (b + 1) * p.S, h * kD, p.H);
}

// ----------------------------------------------------------------------------------------------
// backward
// ----------------------------------------------------------------------------------------------
// 8 bf16 tiles (Q, K, V, dO, P0, P1, dS0, dS1) + mask, lse, delta + barriers + 8 per-warp staging
// buffers: 152.6 KB, one CTA per SM.  The tiled dQ kernel leaves the P blocks unused.
constexpr int kBwdOffVec = 8 * kTile;  // sMask | sLse | sDelta, 128 floats each
constexpr int kBwdOffBar = kBwdOffVec + 3 * kT * 4;
constexpr int kBwdOffStage = kBwdOffBar + 64;
constexpr int kBwdSmem = kBwdOffStage + 8 * kWarpStageBytes + 1024 /*align*/;

struct BwdSmem {
  uint8_t *sQ, *sK, *sV, *sdO, *sP, *sdS;  // sP, sdS: 2 blocks each (keys 0..63 | 64..127)
  float *sMask, *sLse, *sDelta;
  uint64_t* bars;
  uint8_t* stage;
};
__device__ __forceinline__ BwdSmem bwd_smem(uint8_t* smem_raw, int warp) {
  uint8_t* smem = align_smem(smem_raw);
  BwdSmem m;
  m.sQ = smem;
  m.sK = smem + kTile;
  m.sV = smem + 2 * kTile;
  m.sdO = smem + 3 * kTile;
  m.sP = smem + 4 * kTile;
  m.sdS = smem + 6 * kTile;
  m.sMask = reinterpret_cast<float*>(smem + kBwdOffVec);
  m.sLse = m.sMask + kT;
  m.sDelta = m.sLse + kT;
  m.bars = reinterpret_cast<uint64_t*>(smem + kBwdOffBar);
  m.stage = smem + kBwdOffStage + warp * kWarpStageBytes;
  return m;
}

__device__ __forceinline__ void bwd_prologue(const BwdSmem& m, int nbars, int tid,
                                             const CUtensorMap* tmap_qkv,
                                             const CUtensorMap* tmap_do) {
  if (tid == 0) {
    tma_prefetch_desc(tmap_qkv);
    tma_prefetch_desc(tmap_do);
    for (int i = 0; i < nbars; ++i) mbar_init(&m.bars[i], 1);
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
}

// S = 128: one CTA per (batch, head)
__global__ void __launch_bounds__(kThreads, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                     const __grid_constant__ CUtensorMap tmap_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  const Frag f = frag_of_thread();
  const BwdSmem m = bwd_smem(smem_raw, f.warp);
  const int bh = blockIdx.x;
  const int b = bh / p.heads;
  const int h = bh % p.heads;

  bwd_prologue(m, 1, f.tid, &tmap_qkv, &tmap_do);
  load_mask(m.sMask, p, b, kT, 0, f.tid);
  __syncthreads();

  if (f.warp == 0 && elect_one_sync()) {
    mbar_expect_tx(&m.bars[0], 4 * kTile);
    tma_load_3d(m.sQ, &tmap_qkv, &m.bars[0], h * kD, 0, b);
    tma_load_3d(m.sK, &tmap_qkv, &m.bars[0], p.H + h * kD, 0, b);
    tma_load_3d(m.sV, &tmap_qkv, &m.bars[0], 2 * p.H + h * kD, 0, b);
    tma_load_3d(m.sdO, &tmap_do, &m.bars[0], h * kD, 0, b);
  }
  load_bwd_rows(p, b, h, bh, kT, 0, f.tid, m.sLse, m.sDelta);  // while the loads run
  __syncthreads();
  const BwdRows r{m.sLse[f.q0], m.sLse[f.q0 + 8], m.sDelta[f.q0], m.sDelta[f.q0 + 8]};

  mbar_wait(&m.bars[0], 0);
  const uint32_t aQ = smem_u32(m.sQ), aK = smem_u32(m.sK), aV = smem_u32(m.sV);
  const uint32_t adO = smem_u32(m.sdO), aP = smem_u32(m.sP), adS = smem_u32(m.sdS);
  const float sc = p.scale * kLog2e;
  const Dropout dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  const long long row_a = static_cast<long long>(bh) * kT + f.q0;
#pragma unroll 1
  for (int kh = 0; kh < 2; ++kh)
    bwd_p_ds<true>(f, aQ, adO, aK, aV, kh * 64, m.sMask + kh * 64, r, sc, p.scale, dr, row_a,
                   kh * 64, kT, m.sP + kh * kTile, m.sdS + kh * kTile);
  fence_proxy_async_smem();  // P / dS (generic-proxy stores) -> wgmma (async-proxy reads)
  __syncthreads();           // dV / dK need the P / dS rows of both warpgroups

  // warpgroup w: keys 64w .. 64w + 63 of dV / dK, query rows 64w .. 64w + 63 of dQ
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
  mma_dkv(dv, dk, aP, adS, adO, aQ, f.wg);
  wgmma_commit();
  mma_dq(dq, adS, aK, f.wg);
  wgmma_commit();

  const long long grow0 = static_cast<long long>(b) * kT + f.wrow0;  // my warp's keys / queries
  const int ld = 3 * p.H;
  wgmma_wait<1>();  // dV and dK leave while dQ is still in flight
  frag_store_bf16(dv, m.stage, f.lane, p.dqkv, ld, grow0, INT_MAX, 2 * p.H + h * kD, ld);
  frag_store_bf16(dk, m.stage, f.lane, p.dqkv, ld, grow0, INT_MAX, p.H + h * kD, ld);
  wgmma_wait<0>();
  frag_store_bf16(dq, m.stage, f.lane, p.dqkv, ld, grow0, INT_MAX, h * kD, ld);
}

// tiled dQ: one CTA per (batch, head, query tile), loop over key tiles
__global__ void __launch_bounds__(kThreads, 1)
attention_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                        const __grid_constant__ CUtensorMap tmap_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  const Frag f = frag_of_thread();
  const BwdSmem m = bwd_smem(smem_raw, f.warp);
  uint64_t* bar_q = &m.bars[0];
  uint64_t* bar_kv = &m.bars[1];
  const int qt = blockIdx.x % p.n_tiles;
  const int bh = blockIdx.x / p.n_tiles;
  const int b = bh / p.heads;
  const int h = bh % p.heads;

  bwd_prologue(m, 2, f.tid, &tmap_qkv, &tmap_do);
  __syncthreads();
  const bool issuer = f.warp == 0 && elect_one_sync();
  if (issuer) {
    mbar_expect_tx(bar_q, 2 * kTile);
    tma_load_3d(m.sQ, &tmap_qkv, bar_q, h * kD, qt * kT, b);
    tma_load_3d(m.sdO, &tmap_do, bar_q, h * kD, qt * kT, b);
  }
  load_bwd_rows(p, b, h, bh, p.S, qt * kT, f.tid, m.sLse, m.sDelta);
  __syncthreads();
  const BwdRows r{m.sLse[f.q0], m.sLse[f.q0 + 8], m.sDelta[f.q0], m.sDelta[f.q0 + 8]};
  const float sc = p.scale * kLog2e;
  const Dropout dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  const long long row_a = static_cast<long long>(bh) * p.S + qt * kT + f.q0;
  const uint32_t aQ = smem_u32(m.sQ), aK = smem_u32(m.sK), aV = smem_u32(m.sV);
  const uint32_t adO = smem_u32(m.sdO), adS = smem_u32(m.sdS);
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;

  mbar_wait(bar_q, 0);
  for (int j = 0; j < p.n_tiles; ++j) {
    load_mask(m.sMask, p, b, p.S, j * kT, f.tid);
    if (issuer) {
      mbar_expect_tx(bar_kv, 2 * kTile);
      tma_load_3d(m.sK, &tmap_qkv, bar_kv, p.H + h * kD, j * kT, b);
      tma_load_3d(m.sV, &tmap_qkv, bar_kv, 2 * p.H + h * kD, j * kT, b);
    }
    mbar_wait(bar_kv, j & 1);
    __syncthreads();  // sMask visible
#pragma unroll 1
    for (int kh = 0; kh < 2; ++kh)
      bwd_p_ds<false>(f, aQ, adO, aK, aV, kh * 64, m.sMask + kh * 64, r, sc, p.scale, dr, row_a,
                      j * kT + kh * 64, p.S, nullptr, m.sdS + kh * kTile);
    fence_proxy_async_smem();
    __syncthreads();  // dS rows visible to the warpgroup's wgmma
    wgmma_fence();
    mma_dq(dq, adS, aK, f.wg);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();  // K, V, sMask and dS consumed before the next tile overwrites them
  }
  const int ld = 3 * p.H;
  frag_store_bf16(dq, m.stage, f.lane, p.dqkv, ld,
                  static_cast<long long>(b) * p.S + qt * kT + f.wrow0, (b + 1) * p.S, h * kD, ld);
}

// tiled dK / dV: one CTA per (batch, head, key tile), loop over query tiles
__global__ void __launch_bounds__(kThreads, 1)
attention_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                         const __grid_constant__ CUtensorMap tmap_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  const Frag f = frag_of_thread();
  const BwdSmem m = bwd_smem(smem_raw, f.warp);
  uint64_t* bar_kv = &m.bars[0];
  uint64_t* bar_q = &m.bars[1];
  const int kt = blockIdx.x % p.n_tiles;
  const int bh = blockIdx.x / p.n_tiles;
  const int b = bh / p.heads;
  const int h = bh % p.heads;

  bwd_prologue(m, 2, f.tid, &tmap_qkv, &tmap_do);
  load_mask(m.sMask, p, b, p.S, kt * kT, f.tid);
  __syncthreads();
  const bool issuer = f.warp == 0 && elect_one_sync();
  if (issuer) {
    mbar_expect_tx(bar_kv, 2 * kTile);
    tma_load_3d(m.sK, &tmap_qkv, bar_kv, p.H + h * kD, kt * kT, b);
    tma_load_3d(m.sV, &tmap_qkv, bar_kv, 2 * p.H + h * kD, kt * kT, b);
  }
  const float sc = p.scale * kLog2e;
  const Dropout dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  const uint32_t aQ = smem_u32(m.sQ), aK = smem_u32(m.sK), aV = smem_u32(m.sV);
  const uint32_t adO = smem_u32(m.sdO), aP = smem_u32(m.sP), adS = smem_u32(m.sdS);
  float dv[32], dk[32];  // keys 64 wg .. 64 wg + 63 of the tile
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    dv[i] = 0.f;
    dk[i] = 0.f;
  }

  mbar_wait(bar_kv, 0);
  for (int i = 0; i < p.n_tiles; ++i) {
    if (issuer) {
      mbar_expect_tx(bar_q, 2 * kTile);
      tma_load_3d(m.sQ, &tmap_qkv, bar_q, h * kD, i * kT, b);
      tma_load_3d(m.sdO, &tmap_do, bar_q, h * kD, i * kT, b);
    }
    load_bwd_rows(p, b, h, bh, p.S, i * kT, f.tid, m.sLse, m.sDelta);  // overlaps the loads
    __syncthreads();
    const BwdRows r{m.sLse[f.q0], m.sLse[f.q0 + 8], m.sDelta[f.q0], m.sDelta[f.q0 + 8]};
    const long long row_a = static_cast<long long>(bh) * p.S + i * kT + f.q0;
    mbar_wait(bar_q, i & 1);
#pragma unroll 1
    for (int kh = 0; kh < 2; ++kh)
      bwd_p_ds<true>(f, aQ, adO, aK, aV, kh * 64, m.sMask + kh * 64, r, sc, p.scale, dr, row_a,
                     kt * kT + kh * 64, p.S, m.sP + kh * kTile, m.sdS + kh * kTile);
    fence_proxy_async_smem();
    __syncthreads();  // dV / dK need the P / dS rows of both warpgroups
    wgmma_fence();
    mma_dkv(dv, dk, aP, adS, adO, aQ, f.wg);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();  // Q, dO, P, dS, lse and delta consumed before the next query tile
  }

  const long long grow0 = static_cast<long long>(b) * p.S + kt * kT + f.wrow0;
  const int ld = 3 * p.H;
  frag_store_bf16(dv, m.stage, f.lane, p.dqkv, ld, grow0, (b + 1) * p.S, 2 * p.H + h * kD, ld);
  frag_store_bf16(dk, m.stage, f.lane, p.dqkv, ld, grow0, (b + 1) * p.S, p.H + h * kD, ld);
}

// ----------------------------------------------------------------------------------------------
// host
// ----------------------------------------------------------------------------------------------
// S = 128 runs the single-tile kernels; every other length (and S = 128 when SKY_ATTN_TILED=1,
// for A/B comparisons) the tiled kernels
bool use_tiled(int S) {
  static int v = -1;
  if (v < 0) {
    const char* e = std::getenv("SKY_ATTN_TILED");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return S != kT || v == 1;
}

// checks the arguments, fills the kernel parameters and the (C, S, B) tensor map of QKV
int prepare(const AttnArgs& a, AttnDev* d, CUtensorMap* tm_qkv) {
  if (a.head_dim != kD || a.S <= 0 || (a.S % 8) != 0) return 930;
  if (a.dropout_p > 0.f && a.rng_state == nullptr) return 903;
  d->mask = a.mask;
  d->ctx = reinterpret_cast<__nv_bfloat16*>(a.ctx);
  d->lse = a.lse;
  d->ctx_in = reinterpret_cast<const __nv_bfloat16*>(a.ctx);
  d->dctx = reinterpret_cast<const __nv_bfloat16*>(a.dctx);
  d->dqkv = reinterpret_cast<__nv_bfloat16*>(a.dqkv);
  d->S = a.S;
  d->heads = a.heads;
  d->H = a.heads * kD;
  d->n_tiles = (a.S + kT - 1) / kT;
  d->scale = a.scale;
  d->dropout_p = a.dropout_p;
  d->rng_state = a.rng_state;
  d->rng_stream = a.rng_stream;
  const uint64_t H = d->H;
  return make_tmap_bf16_3d(tm_qkv, a.qkv, 3 * H, a.S, a.B, 3 * H, 3 * H * a.S, 64, 128);
}

// sets the kernel's dynamic shared memory limit once, then launches `ctas` CTAs of 256 threads
template <auto Kern, class... Args>
int launch(int ctas, int smem, cudaStream_t stream, const Args&... args) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = true;
  }
  cudaError_t le = launch_pdl(Kern, dim3(ctas), dim3(kThreads), smem, stream, args...);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace

bool attention_supported(int S, int head_dim) { return head_dim == kD && S > 0 && (S % 8) == 0; }

int launch_attention_fwd(const AttnArgs& a, cudaStream_t stream) {
  AttnDev d;
  CUtensorMap tm;
  int rc = prepare(a, &d, &tm);
  if (rc) return rc;
  if (use_tiled(a.S))
    return launch<attention_fwd_tiled_kernel>(a.B * a.heads * d.n_tiles, kFwdTSmem, stream, tm, d);
  return launch<attention_fwd_kernel>(a.B * a.heads, kFwdSmem, stream, tm, d);
}

int launch_attention_bwd(const AttnArgs& a, cudaStream_t stream) {
  AttnDev d;
  CUtensorMap tm, tdo;
  int rc = prepare(a, &d, &tm);
  if (rc) return rc;
  if (a.lse == nullptr || a.ctx == nullptr || a.dctx == nullptr || a.dqkv == nullptr) return 931;
  const uint64_t H = d.H;
  rc = make_tmap_bf16_3d(&tdo, a.dctx, H, a.S, a.B, H, H * a.S, 64, 128);
  if (rc) return rc;
  if (!use_tiled(a.S))
    return launch<attention_bwd_kernel>(a.B * a.heads, kBwdSmem, stream, tm, tdo, d);
  const int ctas = a.B * a.heads * d.n_tiles;
  rc = launch<attention_bwd_dq_kernel>(ctas, kBwdSmem, stream, tm, tdo, d);
  if (rc) return rc;
  return launch<attention_bwd_dkv_kernel>(ctas, kBwdSmem, stream, tm, tdo, d);
}

}  // namespace sky
