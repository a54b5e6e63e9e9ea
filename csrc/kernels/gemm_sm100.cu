// Persistent warp-specialised wgmma GEMM for sm_90a (H100).
//
//   out[M,N] = epilogue( sum_k A[m,k] * B[n,k] )      bf16 x bf16 -> fp32 (registers) -> bf16 | fp32
//
//   * operands staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) into a 4..6 deep smem ring by one
//     producer warp,
//   * two consumer warpgroups, each issuing wgmma.mma_async m64 x BLOCK_N x 16 for its 64 rows of
//     the 128 x BLOCK_N tile; the accumulators live in registers (setmaxnreg moves the producer
//     warpgroup's registers to the consumers),
//   * the epilogue walks the tile in 64-column groups and applies bias / erf-GELU / GELU' /
//     dropout / residual add to the accumulator fragments in registers; bf16 results pass a small
//     per-warp staging buffer so that global stores stay whole 128-byte rows, fp32 results leave
//     straight from the fragments.  The target may be the NEXT PIPELINE STAGE's HBM (peer pointer
//     over NVLink); a per-128-row-panel flag is then bumped with red.release.sys so the consumer
//     GPU can start on that panel while we still compute,
//   * symmetric consumer side: the TMA producer can ld.acquire.sys-poll such flags before it
//     loads the A rows of a panel (GEMM -> GEMM boundary), see GemmArgs in api.h.
//
// Both operands may be K-major or MN-major (wgmma "transpose" bits), so forward
// (x W^T), dgrad (dy W) and wgrad (dy^T x) all run on this one kernel without transposes.
//
// Reference parity: replaces every nn.Linear / LinearActivation call in
// scaelum/model/bert_layers.py:60-108,227-229,281,311-313,319 and the autograd backward of those.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cstdlib>
#include <map>
#include <mutex>
#include <utility>

#include "api.h"
#include "launch_util.h"
#include "sm100_ptx.cuh"

namespace sky {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int MMA_K = 16;
// warpgroup 0: warp 0 = TMA producer (warps 1-3 only give up their registers);
// warpgroups 1, 2 (warps 4-11): wgmma consumers + epilogue, 64 rows of the tile each
constexpr int kNumThreads = 384;
constexpr int kEpiWarp0 = 4;
constexpr uint64_t kFlagTimeoutNs = 4000000000ull;  // 4 s
constexpr int kMaxSmemBytes = 227 * 1024;           // opt-in dynamic shared memory per block (H100)
// the per-warp bf16 staging buffer of the epilogues (kStageLd, kWarpStageBytes) is defined next
// to frag_store_bf16 in sm100_ptx.cuh

template <int BLOCK_N>
struct Cfg {
  static constexpr int kStages = BLOCK_N == 256 ? 4 : 6;
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBiasBytes = 2 * BLOCK_N * 4;  // double-buffered bias tile
  static constexpr int kOutStageBytes = 8 * kWarpStageBytes;  // one buffer per epilogue warp
  static constexpr int kOffBars = kStages * kStageBytes;
  static constexpr int kOffBias = kOffBars + 256;
  static constexpr int kOffOut = kOffBias + kBiasBytes;
  static constexpr int kSmemBytes = kOffOut + kOutStageBytes + 1024 /*align slack*/;
  static_assert(kSmemBytes <= kMaxSmemBytes, "GEMM shared memory over the per-block limit");
};

// ---- epilogue on accumulator fragments ----
// The fragment layout, the per-warp staging buffer, frag_store_bf16 and frag_dropout are in
// sm100_ptx.cuh (the attention kernels use them too).  Global memory is reached through the warp's
// staging buffer `s` for bf16 tiles (coalesced 128-byte rows) and straight from the fragments for
// fp32 (a quad covers 32 contiguous bytes of a row).  Column bounds are checked per 8-column block
// (one 16-byte bf16 piece, or the block's column pairs in the fp32 stores); that is exact only
// because the launchers require N % 8 == 0.  Relaxing that host check needs per-pair checks here
// first, or ragged tiles would write past column N.

// coalesced global read of a bf16 16 x 64 block (issued early, it hides behind the epilogue math)
__device__ __forceinline__ void aux_load(uint4 (&ax)[4], const __nv_bfloat16* aux, long long ld,
                                         long long grow0, int m, int col0, int n, int lane) {
  const int piece = lane & 7;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i * 4 + (lane >> 3);
    ax[i] = (grow0 + r < m && col0 + piece * 8 < n)
                ? *reinterpret_cast<const uint4*>(aux + (grow0 + r) * ld + col0 + piece * 8)
                : make_uint4(0, 0, 0, 0);
  }
}
// the block of aux_load -> staging -> fragment pairs (a[2j] = row fr, a[2j+1] = row fr + 8, bf16x2
// each), then f *= gelu'(aux) (mul_dgelu) or f += aux (add)
__device__ __forceinline__ void frag_apply_aux(float (&f)[32], const uint4 (&ax)[4], uint8_t* s,
                                               int lane, bool mul_dgelu, bool add) {
  const int piece = lane & 7;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<uint4*>(s + (i * 4 + (lane >> 3)) * kStageLd + piece * 16) = ax[i];
  __syncwarp();
  const uint8_t* mine = s + (lane >> 2) * kStageLd + (lane & 3) * 4;
  uint32_t a[16];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    a[2 * j] = *reinterpret_cast<const uint32_t*>(mine + j * 16);
    a[2 * j + 1] = *reinterpret_cast<const uint32_t*>(mine + 8 * kStageLd + j * 16);
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 xa = unpack_bf16x2(a[2 * j]);
    const float2 xb = unpack_bf16x2(a[2 * j + 1]);
    if (mul_dgelu) {
      f[4 * j] *= dgelu_fast(xa.x);
      f[4 * j + 1] *= dgelu_fast(xa.y);
      f[4 * j + 2] *= dgelu_fast(xb.x);
      f[4 * j + 3] *= dgelu_fast(xb.y);
    } else if (add) {
      f[4 * j] += xa.x;
      f[4 * j + 1] += xa.y;
      f[4 * j + 2] += xb.x;
      f[4 * j + 3] += xb.y;
    }
  }
}
// f += the bias of the group's 64 columns ct .. ct + 63 of the tile (staged in shared memory at sb)
__device__ __forceinline__ void frag_add_bias(float (&f)[32], const float* sb, int ct, int fc) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(sb + ct + j * 8 + fc);  // broadcast
    f[4 * j] = f[4 * j] + bb.x;
    f[4 * j + 1] = f[4 * j + 1] + bb.y;
    f[4 * j + 2] = f[4 * j + 2] + bb.x;
    f[4 * j + 3] = f[4 * j + 3] + bb.y;
  }
}

// Parameters both kernels read: the shape, the epilogue inputs they share, dropout and the
// stage-boundary flags (see GemmArgs in api.h).
struct GemmCommon {
  int M, N, K;
  const float* bias;
  const __nv_bfloat16* aux;
  long long ldaux;
  float dropout_p;
  const uint64_t* rng_state;
  uint32_t rng_stream;
  uint32_t* signal_flags;
  const uint32_t* wait_flags;
  const uint32_t* wait_epoch;
  uint32_t wait_mult;
  int* error_flag;
};

struct GemmDev : GemmCommon {
  void* out;
  void* out2;
  long long ldo, ldo2;
  int act;
  int add_aux;
  int accumulate;
  int debug;
  // stream-K: the flattened (tile, k-block) space is cut into one contiguous range per CTA (cluster);
  // tiles shared by several CTAs are reduced through `ws` by whichever CTA arrives last
  int stream_k;
  float* ws;           // partial accumulators: slot (2 * unit + which) * ctas_per_unit + cta_rank
  uint32_t* counters;  // per CTA tile: [2 * t] arrivals, [2 * t + 1] partials written
  // SGD update in the epilogue (gemm_wgrad_sgd_kernel only, see GemmArgs::sgd_master)
  float* sgd_p;
  __nv_bfloat16* sgd_shadow;
  float sgd_lr, sgd_weight_decay, sgd_grad_scale;
};

struct Work {
  int tile, kb0, kb1;
};

// Tile scheduler shared by the warp roles.  Classic mode: tiles unit, unit + U, ... with the
// whole K range.  Stream-K mode: k-blocks [unit * T / U, (unit + 1) * T / U) of T = tiles * nk.
struct Sched {
  int stream, unit, num_units, num_tiles, nk;
  long long total;
  int pos, end, tile;
  __device__ __forceinline__ long long bound(int u) const { return u * total / num_units; }
  __device__ __forceinline__ void init(int stream_k, int unit_, int num_units_, int num_tiles_,
                                       int nk_) {
    stream = stream_k;
    unit = unit_;
    num_units = num_units_;
    num_tiles = num_tiles_;
    nk = nk_;
    total = static_cast<long long>(num_tiles_) * nk_;
    pos = static_cast<int>(bound(unit_));
    end = static_cast<int>(bound(unit_ + 1));
    tile = unit_ - num_units_;
  }
  __device__ __forceinline__ bool next(Work& w) {
    if (!stream) {
      tile += num_units;
      if (tile >= num_tiles) return false;
      w.tile = tile;
      w.kb0 = 0;
      w.kb1 = nk;
      return true;
    }
    if (pos >= end) return false;
    w.tile = pos / nk;
    w.kb0 = pos - w.tile * nk;
    const int len = min(nk - w.kb0, end - pos);
    w.kb1 = w.kb0 + len;
    pos += len;
    return true;
  }
  // unit whose range contains flattened position x
  __device__ __forceinline__ int unit_of(long long x) const {
    int u = static_cast<int>(x * num_units / total);
    while (u + 1 < num_units && bound(u + 1) <= x) ++u;
    while (u > 0 && bound(u) > x) --u;
    return u;
  }
  __device__ __forceinline__ int first_tile(int u) const { return static_cast<int>(bound(u) / nk); }
};

// A position in the operand ring: the stage and the parity of its current fill.
template <int kStages>
struct Ring {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
};

// The operand ring in the 1024-byte aligned dynamic shared memory (SWIZZLE_128B tiles need that
// alignment): kStages A tiles, kStages B tiles, then the full and empty barriers at kOffBars.
struct Operands {
  uint8_t* base;  // the aligned shared memory
  uint8_t* a;
  uint8_t* b;
  uint64_t* full_bar;   // [kStages]
  uint64_t* empty_bar;  // [kStages]; the kernel's own barriers follow
};

// Prologue of both kernels, before their cluster / CTA sync: warp 0 prefetches the tensor maps,
// lane 0 of warp 1 initialises the ring barriers.  A stage is free again after `empty_count`
// arrivals: one per consumer warpgroup of every CTA that loads into it.  C = the ring's layout
// (kStages, kABytes, kOffBars).
template <int BLOCK_N, class C = Cfg<BLOCK_N>>
__device__ __forceinline__ Operands ring_prologue(uint8_t* smem_raw, const CUtensorMap* tmap_a,
                                                  const CUtensorMap* tmap_b, int warp_idx,
                                                  int lane, uint32_t empty_count) {
  Operands op;
  op.base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                       ~static_cast<uintptr_t>(1023));
  op.a = op.base;
  op.b = op.base + C::kStages * C::kABytes;
  op.full_bar = reinterpret_cast<uint64_t*>(op.base + C::kOffBars);
  op.empty_bar = op.full_bar + C::kStages;
  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(tmap_a);
    tma_prefetch_desc(tmap_b);
  }
  if (warp_idx == 1 && lane == 0) {
    for (int i = 0; i < C::kStages; ++i) {
      mbar_init(&op.full_bar[i], 1);
      mbar_init(&op.empty_bar[i], empty_count);
    }
    fence_barrier_init();
  }
  return op;
}

// Producer: wait until the inbound 128-row panel m_blk of A is complete (GEMM -> GEMM boundary).
// A timeout sets error code 1 and the loads go ahead.
__device__ __forceinline__ void wait_inbound_panel(const GemmCommon& p, int m_blk) {
  if (elect_one_sync()) {
    const uint32_t target = (*p.wait_epoch) * p.wait_mult;
    if (!wait_flag_ge(p.wait_flags + m_blk, target, kFlagTimeoutNs)) {
      if (p.error_flag) atomicExch(p.error_flag, 1);
    }
    fence_proxy_async();  // peer generic-proxy writes -> our async-proxy (TMA) reads
  }
  __syncwarp();
}

// Producer: TMA loads of k-block kb into ring stage `stage`, whose empty barrier the caller has
// waited on.  A: rows a_row0 .. a_row0 + 127; B: rows b_row0 .. of this CTA's share of the tile.
// cl_rank = rank in the cluster (CL, see gemm_wgmma_kernel).  no_loads (debug mode 3, single CTAs
// only) completes the stage without loading: the MMAs then read stale shared memory.
template <int BLOCK_N, bool A_MN, bool B_MN, int CL>
__device__ __forceinline__ void load_k_block(const Operands& op, int stage,
                                             const CUtensorMap* tmap_a, const CUtensorMap* tmap_b,
                                             int kb, int a_row0, int b_row0, uint32_t cl_rank,
                                             bool no_loads) {
  constexpr bool PAIR = CL >= 2;
  constexpr bool MC = CL == 4;
  using C = Cfg<BLOCK_N>;
  constexpr int kBRows = PAIR ? BLOCK_N / 2 : BLOCK_N;  // B rows fetched by ONE CTA
  uint64_t* full = &op.full_bar[stage];
  if (!PAIR && no_loads) {
    if (elect_one_sync()) mbar_arrive(full);
    __syncwarp();
    return;
  }
  if (elect_one_sync()) {
    const uint32_t cta_rank = cl_rank & 1u;  // rank in the pair
    const uint16_t mask_b = static_cast<uint16_t>(3u << (cl_rank & ~1u));  // my pair
    const uint16_t mask_a = static_cast<uint16_t>((1u << cl_rank) | (1u << (cl_rank ^ 2u)));
    mbar_expect_tx(full, C::kStageBytes);
    uint8_t* sa = op.a + stage * C::kABytes;
    uint8_t* sb = op.b + stage * C::kBBytes;
    // ---- A: my 128 rows (MC: my half of them, delivered to me and to the other pair) ----
    if constexpr (MC) {
      const int h = static_cast<int>(cl_rank >> 1);
      if constexpr (!A_MN)
        tma_load_2d_mc(sa + h * (64 * 128), tmap_a, full, kb * BLOCK_K, a_row0 + h * 64, mask_a);
      else
        tma_load_2d_mc(sa + h * (BLOCK_K * 128), tmap_a, full, a_row0 + h * 64, kb * BLOCK_K,
                       mask_a);
    } else if constexpr (!A_MN) {
      tma_load_2d(sa, tmap_a, full, kb * BLOCK_K, a_row0);
    } else {
#pragma unroll
      for (int c = 0; c < BLOCK_M / 64; ++c)
        tma_load_2d(sa + c * (BLOCK_K * 128), tmap_a, full, a_row0 + c * 64, kb * BLOCK_K);
    }
    // ---- B: the whole tile, or (clusters) my half of it multicast to my pair ----
    if constexpr (!PAIR) {
      if constexpr (!B_MN) {
        tma_load_2d(sb, tmap_b, full, kb * BLOCK_K, b_row0);
      } else {
#pragma unroll
        for (int c = 0; c < BLOCK_N / 64; ++c)
          tma_load_2d(sb + c * (BLOCK_K * 128), tmap_b, full, b_row0 + c * 64, kb * BLOCK_K);
      }
    } else {
      uint8_t* sbh = sb + cta_rank * (C::kBBytes / 2);
      if constexpr (!B_MN) {
        tma_load_2d_mc(sbh, tmap_b, full, kb * BLOCK_K, b_row0, mask_b);
      } else {
#pragma unroll
        for (int c = 0; c < kBRows / 64; ++c)
          tma_load_2d_mc(sbh + c * (BLOCK_K * 128), tmap_b, full, b_row0 + c * 64, kb * BLOCK_K,
                         mask_b);
      }
    }
  }  // elected lane
  __syncwarp();
}

// A consumer warpgroup hands a smem stage back to the producer(s): with clusters every CTA that
// multicasts into this stage waits for all CTAs' consumers, so the arrival goes to every CTA.
template <int CL>
__device__ __forceinline__ void release_stage(uint64_t* empty_bar) {
  if constexpr (CL == 1) {
    mbar_arrive(empty_bar);
  } else {
    const uint32_t a = smem_u32(empty_bar);
#pragma unroll
    for (uint32_t r = 0; r < CL; ++r) mbar_arrive_cluster(mapa_shared(a, r));
  }
}

// Main loop of one consumer warpgroup over k-blocks [kb0, kb1): acc (+)= A[64 rows] * B^T.
// One wgmma group stays in flight; a stage is released once the group that read it has retired.
// C = the ring's layout (stage strides kABytes, kBBytes).
template <int BLOCK_N, bool A_MN, bool B_MN, int CL, int kStages, class C = Cfg<BLOCK_N>>
__device__ __forceinline__ void consumer_mainloop(float (&acc)[BLOCK_N / 2], int kb0, int kb1,
                                                  uint32_t a_base, uint32_t b_base,
                                                  const Operands& op, Ring<kStages>& ring,
                                                  bool elected, bool skip_mma) {
  // K-major  SW128: 8-row atoms 1024B apart (SBO), LBO unused (1); K advance = 32B per MMA_K
  // MN-major SW128: 64-element MN chunks BLOCK_K*128B apart (LBO), 8-k-row groups 1024B apart
  //                 (SBO); K advance = 16 rows * 128B = 2048B per MMA_K
  constexpr uint32_t a_lbo = A_MN ? BLOCK_K * 128 : 16;
  constexpr uint32_t b_lbo = B_MN ? BLOCK_K * 128 : 16;
  constexpr uint32_t a_kadv = (A_MN ? MMA_K * 128 : MMA_K * 2) >> 4;
  constexpr uint32_t b_kadv = (B_MN ? MMA_K * 128 : MMA_K * 2) >> 4;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb, ring.advance()) {
    mbar_wait(&op.full_bar[ring.stage], ring.phase);
    if (!skip_mma) {
      const uint64_t desc_a = make_smem_desc_sw128(a_base + ring.stage * C::kABytes, a_lbo, 1024);
      const uint64_t desc_b = make_smem_desc_sw128(b_base + ring.stage * C::kBBytes, b_lbo, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / MMA_K; ++k)
        wgmma_k16<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, desc_a + k * a_kadv, desc_b + k * b_kadv,
                                                       (kb != kb0 || k != 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
    }
    if (prev >= 0 && elected) release_stage<CL>(&op.empty_bar[prev]);
    prev = ring.stage;
  }
  wgmma_wait<0>();
  if (prev >= 0 && elected) release_stage<CL>(&op.empty_bar[prev]);
}

// A consumer thread's place in the tile: consumer warpgroup wg owns rows 64 wg .. 64 wg + 63 of
// the tile, its warp q rows 16 q .. 16 q + 15 (warp_row = 64 wg + 16 q), and the thread the
// fragment rows fr and fr + 8 of those (see frag_store_bf16).
struct Consumer {
  int wg;
  int epi_tid;     // 0..255
  bool elected;    // thread 0 of its warpgroup: hands ring stages back
  int fr;
  int fc;          // fragment column pair inside every 8-column block
  int warp_row;
  uint8_t* stage;  // the warp's bf16 staging buffer
  Dropout dr;
};
__device__ __forceinline__ Consumer consumer_of(int warp_idx, int lane, uint8_t* out_stage,
                                                const GemmCommon& p) {
  const int e = warp_idx - kEpiWarp0;
  Consumer c;
  c.wg = e >> 2;
  c.epi_tid = threadIdx.x - kEpiWarp0 * 32;
  c.elected = (c.epi_tid & 127) == 0;
  c.fr = lane >> 2;
  c.fc = (lane & 3) * 2;
  c.warp_row = c.wg * 64 + (e & 3) * 16;
  c.stage = out_stage + e * kWarpStageBytes;
  c.dr = dropout_of(p.dropout_p, p.rng_state, p.rng_stream);
  return c;
}

// publish a finished tile of panel m_blk: all 256 epilogue threads' stores -> fence -> barrier ->
// one release.sys on the panel's flag
__device__ __forceinline__ void publish_panel(uint32_t* signal_flags, int m_blk, int epi_tid) {
  __threadfence_system();
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (epi_tid == 0) red_release_sys_add(signal_flags + m_blk, 1u);
}

// ---- SGD update in the weight-gradient epilogue (UPD, see gemm_body) ----
// The producer pulls a tile's fp32 masters (and, when accumulating, the gradient the epilogue adds
// to) into L2 this many k-blocks before the tile's main loop ends, so that the epilogue's reads do
// not wait on HBM.
constexpr int kSgdPrefetchKBlocks = 8;
// producer warp: one bulk L2 prefetch per row of the tile (rows >= M skipped); the rows are
// 16-byte aligned because the launcher checks the pointers and ldo % 8 == 0
__device__ __forceinline__ void prefetch_update_tile(const GemmDev& p, int row0, int col0,
                                                     int block_n, int lane) {
  const int cols = min(block_n, p.N - col0);
  if (cols <= 0) return;
  const uint32_t bytes = static_cast<uint32_t>(cols) * 4u;  // a multiple of 32: N % 8 == 0
  for (int r = lane; r < BLOCK_M && row0 + r < p.M; r += 32) {
    const long long off = static_cast<long long>(row0 + r) * p.ldo + col0;
    prefetch_l2_bulk(p.sgd_p + off, bytes);
    if (p.accumulate) prefetch_l2_bulk(reinterpret_cast<const float*>(p.out) + off, bytes);
  }
}
// f (the group's fp32 fragments of dW) -> the gradient g that the plain fp32 epilogue would leave in
// p.out (f, or p.out + f when accumulating); the master p is updated with sgd_multi_kernel's
// arithmetic and f gets the new p for the shadow store.  The gradient itself is not stored.
__device__ __forceinline__ void frag_sgd_update(float (&f)[32], const GemmDev& p, long long row_a,
                                                int col0, int fc) {
  const float* grad = reinterpret_cast<const float*>(p.out);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = row_a + 8 * h;
    if (row >= p.M) continue;
    const long long off = row * p.ldo + col0 + fc;
    float2 w[8], g0[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {  // every load of the row in flight before the math
      const bool in = col0 + j * 8 < p.N;  // covers fc, fc + 1 because N % 8 == 0
      w[j] = in ? *reinterpret_cast<const float2*>(p.sgd_p + off + j * 8) : make_float2(0.f, 0.f);
      g0[j] = (in && p.accumulate) ? *reinterpret_cast<const float2*>(grad + off + j * 8)
                                   : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (col0 + j * 8 >= p.N) continue;
      float gx = f[4 * j + 2 * h], gy = f[4 * j + 2 * h + 1];
      if (p.accumulate) {
        gx = g0[j].x + gx;
        gy = g0[j].y + gy;
      }
      w[j].x = sgd_apply(w[j].x, sgd_direction<false>(gx, w[j].x, p.sgd_grad_scale, 1.f,
                                                      p.sgd_weight_decay), p.sgd_lr);
      w[j].y = sgd_apply(w[j].y, sgd_direction<false>(gy, w[j].y, p.sgd_grad_scale, 1.f,
                                                      p.sgd_weight_decay), p.sgd_lr);
      *reinterpret_cast<float2*>(p.sgd_p + off + j * 8) = w[j];
      f[4 * j + 2 * h] = w[j].x;
      f[4 * j + 2 * h + 1] = w[j].y;
    }
  }
}

// CL = CTAs per cluster: 1 = independent CTAs; 2 = two CTAs that compute vertically neighbouring
// tiles (256 rows, the same BLOCK_N columns) and share the B operand: each fetches half of the B
// tile from L2 and TMA multicasts it to both; 4 = two such pairs on neighbouring N tiles that also
// share A the same way (each CTA fetches half of its 128 A rows and multicasts them to the CTA of
// the other pair that needs the same rows).
// SK = stream-K schedule compiled in (a separate instantiation: its bookkeeping costs registers in
// the epilogue, which the classic kernels - the ones every training step runs - must not pay).
// UPD = the fp32 result is a weight gradient that is not stored: the epilogue applies the SGD
// update to the master weights and their bf16 shadow instead (gemm_wgrad_sgd_kernel; no bias,
// activation, dropout or aux input, single CTAs, classic schedule).
template <int BLOCK_N, bool A_MN, bool B_MN, bool OUT_F32, int CL, bool SK, bool UPD>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tmap_a_, const CUtensorMap* tmap_b_,
                                          const GemmDev& p) {
  static_assert(!UPD || (OUT_F32 && CL == 1 && !SK), "the SGD epilogue needs fp32 single CTAs");
  const CUtensorMap& tmap_a = *tmap_a_;
  const CUtensorMap& tmap_b = *tmap_b_;
  constexpr bool PAIR = CL >= 2;
  constexpr bool MC = CL == 4;
  using C = Cfg<BLOCK_N>;
  constexpr int kStages = C::kStages;
  const uint32_t cl_rank = PAIR ? cluster_ctarank() : 0u;  // rank in the cluster
  const uint32_t cta_rank = cl_rank & 1u;                  // rank in the pair
  const uint32_t pair_idx = cl_rank >> 1;                  // which pair of the cluster (MC)

  extern __shared__ uint8_t smem_raw[];
  const int warp_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  // tile scheduler: a "unit" is one CTA (128 rows) or one CTA pair (256 rows)
  constexpr int UNIT_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  const int num_m_units = (p.M + UNIT_M - 1) / UNIT_M;
  const int num_n_blks = (p.N + BLOCK_N - 1) / BLOCK_N;
  // MC: a scheduling unit covers TWO neighbouring N tiles (one per pair); the host only selects
  // this mode when the number of N tiles is even
  const int num_n_units = MC ? num_n_blks / 2 : num_n_blks;
  const int num_tiles = num_m_units * num_n_units;
  const int num_k_blks = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int unit_id = static_cast<int>(blockIdx.x) / CL;
  const int num_units = static_cast<int>(gridDim.x) / CL;

  const Operands op = ring_prologue<BLOCK_N>(smem_raw, &tmap_a, &tmap_b, warp_idx, lane, 2 * CL);
  uint32_t* s_ticket = reinterpret_cast<uint32_t*>(op.empty_bar + kStages);
  float* s_bias = reinterpret_cast<float*>(op.base + C::kOffBias);
  __syncwarp();
  if constexpr (PAIR)
    cluster_sync_all();  // the peers' barriers must be initialised before anything signals them
  else
    __syncthreads();
  // everything above (barrier init, tensormap prefetch) overlapped the previous kernel's tail;
  // from here on we read what it produced
  pdl_wait();
  pdl_launch_dependents();

  if (warp_idx < kEpiWarp0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp_idx == 0) {
      // ===================================== TMA producer =====================================
      Ring<kStages> ring;
      Sched sched;
      sched.init(SK ? 1 : 0, unit_id, num_units, num_tiles, num_k_blks);
      Work w;
      while (sched.next(w)) {
        const int tile = w.tile;
        const int m_blk = (tile % num_m_units) * (PAIR ? 2 : 1) + static_cast<int>(cta_rank);
        const int n_blk =
            (tile / num_m_units) * (MC ? 2 : 1) + (MC ? static_cast<int>(pair_idx) : 0);
        const int b_row0 = n_blk * BLOCK_N + static_cast<int>(cta_rank) * (PAIR ? BLOCK_N / 2 : 0);
        if (p.wait_flags != nullptr && m_blk * BLOCK_M < p.M) wait_inbound_panel(p, m_blk);
        for (int kb = w.kb0; kb < w.kb1; ++kb, ring.advance()) {
          if constexpr (UPD) {
            if (kb == max(w.kb0, w.kb1 - kSgdPrefetchKBlocks))
              prefetch_update_tile(p, m_blk * BLOCK_M, n_blk * BLOCK_N, BLOCK_N, lane);
          }
          mbar_wait_cluster(&op.empty_bar[ring.stage], ring.phase ^ 1);
          load_k_block<BLOCK_N, A_MN, B_MN, CL>(op, ring.stage, &tmap_a, &tmap_b, kb,
                                                m_blk * BLOCK_M, b_row0, cl_rank, p.debug == 3);
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ============================ consumers: wgmma main loop + epilogue ============================
    // The epilogue runs on the accumulator fragments in registers, 64 columns at a time; bias for
    // the tile is staged once in shared memory, aux (residual / pre-activation) blocks are loaded
    // before the epilogue math, fp32 gradient accumulation uses red.global.add (no
    // read-modify-write).
    const Consumer c = consumer_of(warp_idx, lane, op.base + C::kOffOut, p);
    const bool has_aux = !UPD && p.aux != nullptr;
    int it = 0;
    Ring<kStages> ring;
    // both MN- and K-major A tiles keep rows 64..127 one 8 KB block after rows 0..63
    const uint32_t a_base = smem_u32(op.a) + c.wg * 8192;
    const uint32_t b_base = smem_u32(op.b);
    Sched sched;
    sched.init(SK ? 1 : 0, unit_id, num_units, num_tiles, num_k_blks);
    Work w;
    constexpr int kCtasPerUnit = CL;
    constexpr int kTileElems = BLOCK_M * BLOCK_N;
    float acc[BLOCK_N / 2];
    for (; sched.next(w); ++it) {
      const int tile = w.tile;
      const int m_blk = (tile % num_m_units) * (PAIR ? 2 : 1) + static_cast<int>(cta_rank);
      const int n_blk = (tile / num_m_units) * (MC ? 2 : 1) + (MC ? static_cast<int>(pair_idx) : 0);
      const long long warp_row0 = static_cast<long long>(m_blk) * BLOCK_M + c.warp_row;
      const long long row_a = warp_row0 + c.fr;  // and row_a + 8
      // ---- stage bias (overlaps the main loop of the other warpgroup) ----
      float* sb = s_bias + (it & 1) * BLOCK_N;
      if (c.epi_tid < BLOCK_N) {
        const int gc = n_blk * BLOCK_N + c.epi_tid;
        sb[c.epi_tid] = (p.bias != nullptr && gc < p.N) ? __ldg(p.bias + gc) : 0.f;
      }

      consumer_mainloop<BLOCK_N, A_MN, B_MN, CL>(acc, w.kb0, w.kb1, a_base, b_base, op, ring,
                                                 c.elected, !PAIR && p.debug == 4);

      // ---- stream-K: is this CTA the one that finishes the tile? ----
      // Every contributor takes a ticket once its share of the K range is accumulated.  All but the
      // last arrival park their raw fp32 accumulators in the workspace and bump `done`; the last
      // arrival waits for those writes (the writers are already past their main loop, so the
      // wait is short and cannot deadlock), adds them and runs the real epilogue.
      bool finisher = true;
      int n_contrib = 1, u_first = 0;
      float* ws_mine = nullptr;
      const bool partial = SK && !(w.kb0 == 0 && w.kb1 == num_k_blks) && !p.accumulate;
      const int ctile = n_blk * (num_m_units * (PAIR ? 2 : 1)) + m_blk;
      if (partial) {
        u_first = sched.unit_of(static_cast<long long>(tile) * num_k_blks);
        const int u_last = sched.unit_of(static_cast<long long>(tile + 1) * num_k_blks - 1);
        n_contrib = u_last - u_first + 1;
        asm volatile("bar.sync 1, 256;" ::: "memory");  // the previous tile's ticket has been read
        if (c.epi_tid == 0) *s_ticket = atomicAdd(p.counters + 2 * ctile, 1u);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        finisher = (*s_ticket == static_cast<uint32_t>(n_contrib - 1));
        const int which = (tile == sched.first_tile(unit_id)) ? 0 : 1;
        ws_mine = p.ws + static_cast<size_t>((2 * unit_id + which) * kCtasPerUnit + cl_rank) *
                             kTileElems;
        if (finisher) {
          if (c.epi_tid == 0) {
            const uint64_t t0 = globaltimer_ns();
            while (ld_acquire_sys(p.counters + 2 * ctile + 1) <
                   static_cast<uint32_t>(n_contrib - 1)) {
              if (globaltimer_ns() - t0 > kFlagTimeoutNs) {
                if (p.error_flag) atomicExch(p.error_flag, 2);
                break;
              }
            }
            p.counters[2 * ctile] = 0;  // leave the counters clean for the next launch
            p.counters[2 * ctile + 1] = 0;
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
      }
      // workspace layout of one 128 x BLOCK_N tile: [8-column block][consumer thread][4] floats,
      // the fragment registers as they are, so that a warp's float4 accesses are contiguous
      auto ws_ptr = [&](float* base, int j) {
        return reinterpret_cast<float4*>(base) + j * 256 + c.epi_tid;
      };
      // every consumer thread has staged its share of this tile's bias (and, through the barrier of
      // the previous tile, nobody still reads the buffer that was overwritten)
      asm volatile("bar.sync 1, 256;" ::: "memory");

#pragma unroll
      for (int g = 0; g < BLOCK_N / 64; ++g) {
        const int ct = g * 64;  // first column of the group inside the tile
        const int col0 = n_blk * BLOCK_N + ct;
        if (col0 >= p.N || p.debug == 1 || p.debug >= 3) continue;  // uniform across the CTA
        uint4 ax[4];
        if (has_aux) aux_load(ax, p.aux, p.ldaux, warp_row0, p.M, col0, p.N, lane);
        float f[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] = acc[g * 32 + i];
        if (partial) {
          if (!finisher) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              *ws_ptr(ws_mine, g * 8 + j) =
                  make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
            continue;
          }
          for (int u = u_first; u < u_first + n_contrib; ++u) {
            if (u == unit_id) continue;
            const int which_u = (tile == sched.first_tile(u)) ? 0 : 1;
            float* base =
                p.ws + static_cast<size_t>((2 * u + which_u) * kCtasPerUnit + cl_rank) * kTileElems;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 x = __ldcg(ws_ptr(base, g * 8 + j));
              f[4 * j] = f[4 * j] + x.x;
              f[4 * j + 1] = f[4 * j + 1] + x.y;
              f[4 * j + 2] = f[4 * j + 2] + x.z;
              f[4 * j + 3] = f[4 * j + 3] + x.w;
            }
          }
        }
        if constexpr (!UPD) {
          frag_add_bias(f, sb, ct, c.fc);
          if (p.act == ACT_GELU) {
            if (p.out2 != nullptr && p.debug != 2)
              frag_store_bf16(f, c.stage, lane, reinterpret_cast<__nv_bfloat16*>(p.out2), p.ldo2,
                              warp_row0, p.M, col0, p.N);
#pragma unroll
            for (int i = 0; i < 32; ++i) f[i] = gelu_fast(f[i]);
          } else if (p.act == ACT_TANH) {
#pragma unroll
            for (int i = 0; i < 32; ++i) f[i] = tanh_fast(f[i]);
          }
          if (c.dr.on) frag_dropout(f, c.dr.seed, c.dr.thr16, c.dr.scale, row_a, col0, p.N, lane);
          if (has_aux) frag_apply_aux(f, ax, c.stage, lane, p.act == ACT_DGELU_MUL_AUX, p.add_aux);
        }
        if (p.debug != 2) {
          if constexpr (UPD) {
            frag_sgd_update(f, p, row_a, col0, c.fc);
            frag_store_bf16(f, c.stage, lane, p.sgd_shadow, p.ldo, warp_row0, p.M, col0, p.N);
          } else if constexpr (OUT_F32) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const long long row = row_a + 8 * h;
              if (row < p.M) {
                float* o = reinterpret_cast<float*>(p.out) + row * p.ldo + col0 + c.fc;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  // covers columns fc, fc + 1 only because N % 8 == 0 (launch_gemm checks it)
                  if (col0 + j * 8 < p.N) {
                    if (p.accumulate)
                      red_add_v2_f32(o + j * 8, f[4 * j + 2 * h], f[4 * j + 2 * h + 1]);
                    else
                      *reinterpret_cast<float2*>(o + j * 8) =
                          make_float2(f[4 * j + 2 * h], f[4 * j + 2 * h + 1]);
                  }
                }
              }
            }
          } else {
            frag_store_bf16(f, c.stage, lane, reinterpret_cast<__nv_bfloat16*>(p.out), p.ldo,
                            warp_row0, p.M, col0, p.N);
          }
        }
      }
      if (partial && !finisher) {
        // publish the parked partial: all stores -> fence -> barrier -> one counter bump
        __threadfence();
        asm volatile("bar.sync 2, 256;" ::: "memory");
        if (c.epi_tid == 0) atomicAdd(p.counters + 2 * ctile + 1, 1u);
      }
      if (finisher && p.signal_flags != nullptr && m_blk * BLOCK_M < p.M)
        publish_panel(p.signal_flags, m_blk, c.epi_tid);
    }
  }

  __syncwarp();
  if constexpr (PAIR)
    cluster_sync_all();  // no CTA may leave while a peer still multicasts into / signals it
  else
    __syncthreads();
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool OUT_F32, int CL, bool SK>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                  const __grid_constant__ CUtensorMap tmap_b, const GemmDev p) {
  gemm_body<BLOCK_N, A_MN, B_MN, OUT_F32, CL, SK, false>(&tmap_a, &tmap_b, p);
}

// dW (+)= dY^T X with both operands MN-major over the tokens, and the SGD update of W in the
// epilogue instead of the store of dW (GemmArgs::sgd_master)
template <int BLOCK_N>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgrad_sgd_kernel(const __grid_constant__ CUtensorMap tmap_a,
                      const __grid_constant__ CUtensorMap tmap_b, const GemmDev p) {
  gemm_body<BLOCK_N, true, true, true, 1, false, true>(&tmap_a, &tmap_b, p);
}


// ------------------------------------------------------------------------------------------
// GEMM + bias + dropout + residual + LayerNorm in ONE kernel (SURVEY K4 / K6):
//
//     y = LayerNorm( dropout(A W^T + bias) + residual ) * gamma + beta        z = the pre-LN sum
//
// A LayerNorm row spans all N columns, a warpgroup's accumulator only 256 (or 128) of them, so the
// CTAs that own the columns of one row panel form a THREAD-BLOCK CLUSTER and exchange per-row
// partial sums through distributed shared memory.  Two layouts (L below) share one body:
//
//   wide  (LnCfg<BLOCK_N>)  128-row panels; the N / BLOCK_N CTAs of a panel form a 2..8-CTA cluster,
//                           each CTA owns 128 x BLOCK_N (warpgroup: 64 rows x BLOCK_N)
//   pair  (LnPairCfg)       N = 1024 only: 64-row panels, one CTA pair per panel, each CTA owns
//                           64 x 512 (warpgroup: the same 64 rows x 256 columns).  A 4-CTA
//                           cluster needs four free SMs in one GPC: an H100 SXM (132 SMs) holds
//                           30 such clusters of this kernel at once, so the 32 clusters of a
//                           4096-token wide launch ran in two waves; it holds 66 pairs, and the
//                           64 pairs of that launch run in one.
//
// The prologue, the producer (wide), the main loop and the epilogue steps of pass 1 are those of
// gemm_wgmma_kernel:
//
//   pass 1  on the accumulator fragments: + bias, dropout, + residual; store z (bf16, saved for
//           backward); accumulate row sum / sum of squares (the quad that holds a row combines
//           them with two shuffles); the fp32 sums stay in the accumulator registers
//   DSMEM   one thread per row and warpgroup stores the row's (sum, sumsq) into ALL CTAs of the
//           cluster (st.shared::cluster) and arrives on their mbarriers (release.cluster); each
//           CTA adds the partials in column order, so both layouts give the same statistics
//   pass 2  on the fragments again: normalise with the cluster-wide statistics,
//           gamma / beta, store y - straight into the NEXT PIPELINE STAGE's HBM when y is a peer
//           pointer, then one red.release.sys per CTA on the 128-row panel's flag (N / 256 per
//           panel at N = 1024 in both layouts).
//
// This is the forward stage boundary of the north star: the last GEMM of stage i stores its
// output tiles into stage i+1's HBM from inside the GEMM kernel; no separate LayerNorm launch.
// Reference ops replaced: scaelum/model/bert_layers.py:285-289 (BertSelfOutput) and :323-327
// (BertOutput); hop replaced: scaelum/builder/module_wrapper.py:148-175.
// ------------------------------------------------------------------------------------------
struct GemmLnDev : GemmCommon {
  void* y;
  void* z;
  long long ldy, ldz;
  const float* gamma;
  const float* beta;
  float* mean;
  float* rstd;
  float eps;
  int debug;  // 1 = main loop only: the epilogue discards the tile (see GemmArgs::debug)
};

constexpr int kLnMaxCluster = 8;

template <int BLOCK_N>
struct LnCfg {
  using C = Cfg<BLOCK_N>;  // the operand ring
  static constexpr bool kPair = false;
  static constexpr int kRows = BLOCK_M;  // rows of a panel (= of a CTA tile)
  static constexpr int kCols = BLOCK_N;  // columns of a CTA tile
  static constexpr int kVecBytes = 3 * BLOCK_N * 4;                 // bias, gamma, beta
  static constexpr int kStatsBytes = kLnMaxCluster * BLOCK_M * 8;   // float2 per (cta, row)
  static constexpr int kOffVec = C::kOffBars + 256;
  static constexpr int kOffOut = kOffVec + kVecBytes;
  static constexpr int kOffStats = kOffOut + C::kOutStageBytes;
  static constexpr int kSmemBytes = kOffStats + kStatsBytes + 1024 /*align slack*/;
  static_assert(kSmemBytes <= kMaxSmemBytes, "GEMM + LayerNorm shared memory over the per-block limit");
};

// The pair layout: its own operand ring (64 A rows, 512 B rows per stage) and, since a stage is
// 72 KB, only three stages; the epilogue's staging buffers reuse the ring once the main loop is
// done.  The statistics stay outside the ring: the peer writes them while we may still compute.
struct LnPairCfg {
  using C = LnPairCfg;
  static constexpr bool kPair = true;
  static constexpr int kRows = 64;
  static constexpr int kCols = 512;
  static constexpr int kStages = 3;
  static constexpr int kABytes = kRows * BLOCK_K * 2;
  static constexpr int kBBytes = kCols * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kOffBars = kStages * kStageBytes;
  static constexpr int kVecBytes = 3 * kCols * 4;   // bias, gamma, beta
  static constexpr int kStatsBytes = 4 * kRows * 8;  // float2 per (warpgroup of the pair, row)
  static constexpr int kOffVec = kOffBars + 256;
  static constexpr int kOffOut = 0;
  static constexpr int kOffStats = kOffVec + kVecBytes;
  static constexpr int kSmemBytes = kOffStats + kStatsBytes + 1024 /*align slack*/;
  static_assert(kSmemBytes <= kMaxSmemBytes, "GEMM + LayerNorm shared memory over the per-block limit");
  static_assert(8 * kWarpStageBytes <= kOffBars, "epilogue staging does not fit the operand ring");
};

// Producer of the pair layout: k-block kb of the CTA's tile into ring stage `stage`, whose empty
// barrier the caller has waited on.  A: the panel's 64 rows from a_row0; B: the CTA's 512 rows as
// two boxes.  A is not multicast inside the pair: with three stages, a stage that both CTAs must
// release before either can refill it stalled the main loop (measured on H100: 1.9x the plain
// GEMM's time at K = 4096, against 1.07x without multicast).
__device__ __forceinline__ void load_k_block_ln_pair(const Operands& op, int stage,
                                                     const CUtensorMap* tmap_a,
                                                     const CUtensorMap* tmap_b, int kb, int a_row0,
                                                     uint32_t cta) {
  using C = LnPairCfg;
  if (elect_one_sync()) {
    uint64_t* full = &op.full_bar[stage];
    mbar_expect_tx(full, C::kStageBytes);
    uint8_t* sa = op.a + stage * C::kABytes;
    uint8_t* sb = op.b + stage * C::kBBytes;
    tma_load_2d(sa, tmap_a, full, kb * BLOCK_K, a_row0);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      tma_load_2d(sb + h * (C::kBBytes / 2), tmap_b, full, kb * BLOCK_K,
                  static_cast<int>(cta) * C::kCols + h * (C::kCols / 2));
  }
  __syncwarp();
}

template <int BLOCK_N, class L>
__device__ __forceinline__ void gemm_ln_body(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b,
                                             const GemmLnDev& p) {
  using C = typename L::C;
  constexpr int kStages = C::kStages;
  constexpr bool kPair = L::kPair;
  const uint32_t cln = cluster_nctarank();  // CTAs per cluster (wide: column tiles per panel)
  const uint32_t cta = cluster_ctarank();   // this CTA's column tile
  const int m_blk = static_cast<int>(blockIdx.x / cln);  // panel of L::kRows rows
  const int panel128 = kPair ? m_blk / 2 : m_blk;         // the flags count 128-row panels
  // contributors of row statistics: wide: one per CTA, pair: one per warpgroup
  const uint32_t ncontrib = kPair ? 2 * cln : cln;

  extern __shared__ uint8_t smem_raw[];
  const int warp_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int num_k_blks = (p.K + BLOCK_K - 1) / BLOCK_K;

  const Operands op =
      ring_prologue<BLOCK_N, C>(smem_raw, tmap_a, tmap_b, warp_idx, lane, 2);
  uint64_t* stats_bar = op.empty_bar + kStages;
  float* s_bias = reinterpret_cast<float*>(op.base + L::kOffVec);
  float* s_gamma = s_bias + L::kCols;
  float* s_beta = s_gamma + L::kCols;
  float2* s_stats = reinterpret_cast<float2*>(op.base + L::kOffStats);   // [ncontrib][kRows]
  if (warp_idx == 1 && lane == 0) {
    mbar_init(stats_bar, ncontrib * L::kRows);   // one arrival per row-owner thread of every CTA
    fence_barrier_init();
  }
  __syncwarp();
  cluster_sync_all();   // peers' stats barriers exist before anybody arrives on them
  pdl_wait();
  pdl_launch_dependents();

  if (warp_idx < kEpiWarp0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp_idx == 0) {
      // ===================================== TMA producer =====================================
      Ring<kStages> ring;
      if (p.wait_flags != nullptr) wait_inbound_panel(p, panel128);
      for (int kb = 0; kb < num_k_blks; ++kb, ring.advance()) {
        mbar_wait(&op.empty_bar[ring.stage], ring.phase ^ 1);
        if constexpr (kPair) {
          load_k_block_ln_pair(op, ring.stage, tmap_a, tmap_b, kb, m_blk * L::kRows, cta);
        } else {
          load_k_block<BLOCK_N, false, false, 1>(op, ring.stage, tmap_a, tmap_b, kb,
                                                 m_blk * BLOCK_M, static_cast<int>(cta) * BLOCK_N,
                                                 0u, false);
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ============================ consumers: wgmma main loop + epilogue ============================
    const Consumer c = consumer_of(warp_idx, lane, op.base + L::kOffOut, p);
    // the warp's first row inside the CTA tile, the warpgroup's first column inside it
    const int warp_row = kPair ? c.warp_row - 64 * c.wg : c.warp_row;
    const int wg_col = kPair ? c.wg * BLOCK_N : 0;
    const int tile_col0 = static_cast<int>(cta) * L::kCols;
    const long long warp_row0 = static_cast<long long>(m_blk) * L::kRows + warp_row;
    const long long row_a = warp_row0 + c.fr;  // and row_a + 8
    const bool has_aux = p.aux != nullptr;
    for (int i = c.epi_tid; i < L::kCols; i += 256) {
      const int gc = tile_col0 + i;
      s_bias[i] = p.bias != nullptr ? __ldg(p.bias + gc) : 0.f;
      s_gamma[i] = __ldg(p.gamma + gc);
      s_beta[i] = __ldg(p.beta + gc);
    }

    float acc[BLOCK_N / 2];
    {
      Ring<kStages> ring;
      const uint32_t a_base = smem_u32(op.a) + (kPair ? 0 : c.wg * 8192);
      const uint32_t b_base = smem_u32(op.b) + (kPair ? c.wg * (C::kBBytes / 2) : 0);
      consumer_mainloop<BLOCK_N, false, false, 1, kStages, C>(
          acc, 0, num_k_blks, a_base, b_base, op, ring, c.elected, false);
    }
    // bias / gamma / beta staged; (pair) no warpgroup reads the ring any more
    asm volatile("bar.sync 1, 256;" ::: "memory");

    if (p.debug != 1) {
      // -------------- pass 1: z = dropout(acc + bias) + residual; row statistics --------------
      // the fp32 sums stay in the accumulator registers for pass 2
      float s1a = 0.f, s2a = 0.f, s1b = 0.f, s2b = 0.f;   // rows fr / fr + 8
#pragma unroll
      for (int g = 0; g < BLOCK_N / 64; ++g) {
        const int ct = wg_col + g * 64;  // first column of the group inside the CTA tile
        const int col0 = tile_col0 + ct;
        uint4 ax[4];
        if (has_aux) aux_load(ax, p.aux, p.ldaux, warp_row0, p.M, col0, p.N, lane);
        float f[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] = acc[g * 32 + i];
        frag_add_bias(f, s_bias, ct, c.fc);
        if (c.dr.on) frag_dropout(f, c.dr.seed, c.dr.thr16, c.dr.scale, row_a, col0, p.N, lane);
        if (has_aux) frag_apply_aux(f, ax, c.stage, lane, false, true);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1a += f[4 * j] + f[4 * j + 1];
          s2a = fmaf(f[4 * j], f[4 * j], fmaf(f[4 * j + 1], f[4 * j + 1], s2a));
          s1b += f[4 * j + 2] + f[4 * j + 3];
          s2b = fmaf(f[4 * j + 2], f[4 * j + 2], fmaf(f[4 * j + 3], f[4 * j + 3], s2b));
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[g * 32 + i] = f[i];
        if (p.z != nullptr)
          frag_store_bf16(f, c.stage, lane, reinterpret_cast<__nv_bfloat16*>(p.z), p.ldz,
                          warp_row0, p.M, col0, p.N);
      }
      // -------------- cluster-wide row statistics through distributed shared memory --------------
      // a row of the warpgroup's BLOCK_N columns lives in one quad: two shuffles give its sums,
      // then lane 0 (row fr) and lane 1 (row fr + 8) of the quad publish them to every CTA of
      // the cluster, in the slot of the warpgroup's column range
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        s1a += __shfl_xor_sync(0xffffffffu, s1a, o);
        s2a += __shfl_xor_sync(0xffffffffu, s2a, o);
        s1b += __shfl_xor_sync(0xffffffffu, s1b, o);
        s2b += __shfl_xor_sync(0xffffffffu, s2b, o);
      }
      const int contrib = kPair ? static_cast<int>(2 * cta) + c.wg : static_cast<int>(cta);
      const int row_a_in_tile = warp_row + c.fr;
      if ((lane & 3) < 2) {
        const int hb = lane & 1;
        const uint32_t slot = smem_u32(&s_stats[contrib * L::kRows + row_a_in_tile + 8 * hb]);
        const uint32_t bar = smem_u32(stats_bar);
        const float v1 = hb ? s1b : s1a;
        const float v2 = hb ? s2b : s2a;
        for (uint32_t r = 0; r < cln; ++r) {
          st_cluster_v2_f32(mapa_shared(slot, r), v1, v2);
          mbar_arrive_cluster(mapa_shared(bar, r));
        }
      }
      mbar_wait_cluster(stats_bar, 0);
      float t1a = 0.f, t2a = 0.f, t1b = 0.f, t2b = 0.f;
      for (uint32_t r = 0; r < ncontrib; ++r) {
        const float2 oa = s_stats[r * L::kRows + row_a_in_tile];
        const float2 ob = s_stats[r * L::kRows + row_a_in_tile + 8];
        t1a += oa.x;
        t2a += oa.y;
        t1b += ob.x;
        t2b += ob.y;
      }
      const float inv_n = 1.f / static_cast<float>(p.N);
      const float mean_a = t1a * inv_n;
      const float rstd_a = rsqrtf(fmaxf(fmaf(-mean_a, mean_a, t2a * inv_n), 0.f) + p.eps);
      const float mean_b = t1b * inv_n;
      const float rstd_b = rsqrtf(fmaxf(fmaf(-mean_b, mean_b, t2b * inv_n), 0.f) + p.eps);
      if (contrib == 0 && (lane & 3) < 2) {
        const int hb = lane & 1;
        const long long row = row_a + 8 * hb;
        if (row < p.M) {
          p.mean[row] = hb ? mean_b : mean_a;
          p.rstd[row] = hb ? rstd_b : rstd_a;
        }
      }
      // ------------ pass 2: normalise, gamma / beta, store y (possibly into a peer GPU) ------------
#pragma unroll
      for (int g = 0; g < BLOCK_N / 64; ++g) {
        const int ct = wg_col + g * 64;
        const int col0 = tile_col0 + ct;
        float f[32];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 gm = *reinterpret_cast<const float2*>(s_gamma + ct + j * 8 + c.fc);
          const float2 bt = *reinterpret_cast<const float2*>(s_beta + ct + j * 8 + c.fc);
          f[4 * j] = fmaf((acc[g * 32 + 4 * j] - mean_a) * rstd_a, gm.x, bt.x);
          f[4 * j + 1] = fmaf((acc[g * 32 + 4 * j + 1] - mean_a) * rstd_a, gm.y, bt.y);
          f[4 * j + 2] = fmaf((acc[g * 32 + 4 * j + 2] - mean_b) * rstd_b, gm.x, bt.x);
          f[4 * j + 3] = fmaf((acc[g * 32 + 4 * j + 3] - mean_b) * rstd_b, gm.y, bt.y);
        }
        frag_store_bf16(f, c.stage, lane, reinterpret_cast<__nv_bfloat16*>(p.y), p.ldy, warp_row0,
                        p.M, col0, p.N);
      }
      // publish this CTA's tile of the 128-row panel; the consumer waits for epoch x
      // (N / BLOCK_N) signals per panel
      if (p.signal_flags != nullptr) publish_panel(p.signal_flags, panel128, c.epi_tid);
    }
  }

  __syncwarp();
  cluster_sync_all();   // nobody leaves while a peer may still write its statistics into us
}

template <int BLOCK_N>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_ln_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                     const __grid_constant__ CUtensorMap tmap_b, const GemmLnDev p) {
  gemm_ln_body<BLOCK_N, LnCfg<BLOCK_N>>(&tmap_a, &tmap_b, p);
}

__global__ void __launch_bounds__(kNumThreads, 1)
gemm_ln_pair_kernel(const __grid_constant__ CUtensorMap tmap_a,
                    const __grid_constant__ CUtensorMap tmap_b, const GemmLnDev p) {
  gemm_ln_body<256, LnPairCfg>(&tmap_a, &tmap_b, p);
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e =
        cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  });
  // the encoder is a driver call and needs a current context.  A thread whose first CUDA call
  // this is (autograd's device thread when a backward starts with a GEMM) has none yet:
  // cudaSetDevice makes the device's primary context current, once per thread.
  thread_local bool ctx_current = false;
  if (!ctx_current) {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) ctx_current = true;
  }
  return fn;
}

}  // namespace

// 2D bf16 tensor map: inner (contiguous) extent `inner`, `outer` rows of stride ld elements.
int make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer,
                      uint64_t ld_elems, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return 901;
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 1000 + static_cast<int>(r);
}

// 3D bf16 tensor map (inner, middle, outer) for [outer][middle][inner] data: the attention kernels
// view the [B * S, C] activations as (C, S, B) so that a 128-row box never crosses a sequence.
int make_tmap_bf16_3d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t middle,
                      uint64_t outer, uint64_t ld_middle_elems, uint64_t ld_outer_elems,
                      uint32_t box_inner, uint32_t box_middle) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return 901;
  cuuint64_t gdim[3] = {inner, middle, outer};
  cuuint64_t gstride[2] = {ld_middle_elems * 2, ld_outer_elems * 2};
  cuuint32_t box[3] = {box_inner, box_middle, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 1000 + static_cast<int>(r);
}

int gemm_pick_block_n(int M, int N) {
  // 256-wide tiles halve B re-reads per flop; fall back to 128 when that would leave a third of
  // the 132 SMs idle or N is small.
  const long long tiles256 = static_cast<long long>((M + 127) / 128) * ((N + 255) / 256);
  if (N % 256 != 0 && N <= 128) return 128;
  if (tiles256 < 88) return 128;
  return 256;
}

int gemm_tiles_per_panel(int N, int block_n) { return (N + block_n - 1) / block_n; }

namespace {
// SKY_GEMM_PAIR, SKY_GEMM_QUAD and SKY_GEMM_STREAMK (-1 when unset), read once per process
struct GemmEnv {
  int pair, quad, stream_k;
};
const GemmEnv& gemm_env() {
  static const GemmEnv env = [] {
    auto get = [](const char* name) {
      const char* e = std::getenv(name);
      return e ? std::atoi(e) : -1;
    };
    return GemmEnv{get("SKY_GEMM_PAIR"), get("SKY_GEMM_QUAD"), get("SKY_GEMM_STREAMK")};
  }();
  return env;
}

// 2-CTA clusters (B multicast) and 4-CTA clusters (two pairs, A and B multicast) are opt-in
// (SKY_GEMM_PAIR=1, SKY_GEMM_QUAD=1): not yet measured against independent CTAs on H100.
bool pick_pair(int M) { return gemm_env().pair > 0 && M > 128; }
bool pick_quad() { return gemm_env().quad > 0; }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev_id = 0;
    cudaGetDevice(&dev_id);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev_id);
  }
  return n;
}

// ---- stream-K workspace: one per (device, stream), because GEMMs on different streams overlap ----
constexpr size_t kWsSlotBytes = static_cast<size_t>(BLOCK_M) * 256 * 4;  // one 128 x 256 fp32 tile
constexpr int kWsMaxCtas = 160;                                          // >= SMs of the device (H100: 132)
constexpr int kWsMaxCtaTiles = 8192;
struct StreamKWs {
  float* ws = nullptr;
  uint32_t* counters = nullptr;
};
std::mutex g_ws_mutex;
std::map<std::pair<int, cudaStream_t>, StreamKWs> g_ws;

// nullptr when the workspace does not exist yet and cannot be created (stream is capturing)
const StreamKWs* get_ws(cudaStream_t stream) {
  int dev_id = 0;
  cudaGetDevice(&dev_id);
  std::lock_guard<std::mutex> lock(g_ws_mutex);
  auto key = std::make_pair(dev_id, stream);
  auto it = g_ws.find(key);
  if (it != g_ws.end()) return &it->second;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(stream, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) {
    cudaGetLastError();
    return nullptr;
  }
  StreamKWs w;
  if (cudaMalloc(&w.ws, 2 * kWsMaxCtas * kWsSlotBytes) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (cudaMalloc(&w.counters, 2 * kWsMaxCtaTiles * sizeof(uint32_t)) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(w.ws);
    return nullptr;
  }
  cudaMemset(w.counters, 0, 2 * kWsMaxCtaTiles * sizeof(uint32_t));
  g_ws[key] = w;
  return &g_ws[key];
}

// Stream-K is opt-in (SKY_GEMM_STREAMK=1) and then runs where the classic schedule ends on a
// ragged wave.  The fix-up of split tiles (park + re-read 128 KB per CTA, finisher wait) eats what
// the idle SMs would recover on the BERT shapes.  It pays for fp32 `+=` outputs (weight
// gradients: partials are red.add'ed, no fix-up) with few tiles and a deep K in isolation, but
// inside the training step those weight gradients run on the side stream NEXT TO the dgrad chain,
// where an all-SM stream-K grid takes SMs away from the critical path.
bool want_stream_k(long long tiles, int nk, int units) {
  return gemm_env().stream_k == 1 && tiles > 0 && nk >= 8 && tiles % units != 0;
}

// sets the kernel's dynamic shared memory limit once, then launches `ctas` CTAs in clusters of
// `cluster`
template <auto Kern, class... Args>
int launch(int ctas, int cluster, int smem, cudaStream_t stream, const Args&... args) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr = true;
  }
  cudaError_t le = launch_pdl_cluster(Kern, dim3(ctas), dim3(kNumThreads), smem, stream, cluster,
                                      args...);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

// the parameters both kernels take straight from GemmArgs
GemmCommon common_of(const GemmArgs& a) {
  GemmCommon c;
  c.M = a.M;
  c.N = a.N;
  c.K = a.K;
  c.bias = a.bias;
  c.aux = reinterpret_cast<const __nv_bfloat16*>(a.aux);
  c.ldaux = a.ldaux;
  c.dropout_p = a.dropout_p;
  c.rng_state = a.rng_state;
  c.rng_stream = a.rng_stream;
  c.signal_flags = a.signal_flags;
  c.wait_flags = a.wait_flags;
  c.wait_epoch = a.wait_epoch;
  c.wait_mult = a.wait_mult;
  c.error_flag = a.error_flag;
  return c;
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool OUT_F32, int CL, bool UPD = false>
int launch_inst(const GemmArgs& a, GemmDev d, cudaStream_t stream) {
  constexpr bool PAIR = CL >= 2;
  constexpr bool MC = CL == 4;
  using C = Cfg<BLOCK_N>;
  CUtensorMap tma, tmb;
  int rc;
  if (!A_MN)
    rc = make_tmap_bf16_2d(&tma, a.A, a.K, a.M, a.lda, BLOCK_K, MC ? 64 : BLOCK_M);
  else
    rc = make_tmap_bf16_2d(&tma, a.A, a.M, a.K, a.lda, 64, BLOCK_K);
  if (rc) return rc;
  if (!B_MN)
    rc = make_tmap_bf16_2d(&tmb, a.B, a.K, a.N, a.ldb, BLOCK_K, PAIR ? BLOCK_N / 2 : BLOCK_N);
  else
    rc = make_tmap_bf16_2d(&tmb, a.B, a.N, a.K, a.ldb, 64, BLOCK_K);
  if (rc) return rc;

  // a scheduling unit is one CTA (128 rows) or one CTA pair (256 rows); MC units span two N tiles
  constexpr int UNIT_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  const long long m_units = (a.M + UNIT_M - 1) / UNIT_M;
  const long long n_blks = (a.N + BLOCK_N - 1) / BLOCK_N;
  const long long tiles = m_units * (MC ? n_blks / 2 : n_blks);
  const int sms = num_sms();
  const int max_units = sms / CL;
  int units = max_units;
  if (a.max_ctas > 0 && units > a.max_ctas / CL) units = a.max_ctas / CL;
  if (units < 1) units = 1;
  // stream-K instantiations exist for independent CTAs only (pairs / clusters did not profit), and
  // none with the SGD epilogue
  if constexpr (CL == 1 && !UPD) {
    const int nk = (a.K + BLOCK_K - 1) / BLOCK_K;
    bool sk = a.stream_k < 0 ? want_stream_k(tiles, nk, units) : (a.stream_k != 0);
    // every CTA must own at least 4 k-blocks, the CTA tiles must fit the counter array, a bias
    // must not be added once per partial, and the grid must fit the workspace
    if (tiles * nk < 4LL * units) sk = false;
    if (m_units * n_blks > kWsMaxCtaTiles || sms > kWsMaxCtas) sk = false;
    if (a.accumulate && a.bias != nullptr) sk = false;
    if (sk) {
      if (a.accumulate) {
        d.stream_k = 1;  // partial sums go straight to the fp32 output with red.add
      } else if (const StreamKWs* w = get_ws(stream)) {
        d.stream_k = 1;
        d.ws = w->ws;
        d.counters = w->counters;
      }
    }
  }
  int grid = (tiles < max_units && !d.stream_k) ? static_cast<int>(tiles) : max_units;
  if (a.max_ctas > 0 && grid > a.max_ctas / CL) grid = a.max_ctas / CL;
  if (grid < 1) grid = 1;
  grid *= CL;
  if constexpr (UPD)
    return launch<gemm_wgrad_sgd_kernel<BLOCK_N>>(grid, 1, C::kSmemBytes, stream, tma, tmb, d);
  if constexpr (CL == 1) {
    if (d.stream_k)
      return launch<gemm_wgmma_kernel<BLOCK_N, A_MN, B_MN, OUT_F32, 1, true>>(
          grid, 1, C::kSmemBytes, stream, tma, tmb, d);
  }
  return launch<gemm_wgmma_kernel<BLOCK_N, A_MN, B_MN, OUT_F32, CL, false>>(
      grid, CL, C::kSmemBytes, stream, tma, tmb, d);
}

template <int BLOCK_N, int PAIR>
int dispatch_major(const GemmArgs& a, const GemmDev& dev, cudaStream_t stream) {
  if (!a.a_mn && !a.b_mn)
    return a.out_f32 ? launch_inst<BLOCK_N, false, false, true, PAIR>(a, dev, stream)
                     : launch_inst<BLOCK_N, false, false, false, PAIR>(a, dev, stream);
  if (!a.a_mn && a.b_mn)
    return a.out_f32 ? launch_inst<BLOCK_N, false, true, true, PAIR>(a, dev, stream)
                     : launch_inst<BLOCK_N, false, true, false, PAIR>(a, dev, stream);
  if (a.a_mn && a.b_mn)
    return a.out_f32 ? launch_inst<BLOCK_N, true, true, true, PAIR>(a, dev, stream)
                     : launch_inst<BLOCK_N, true, true, false, PAIR>(a, dev, stream);
  return a.out_f32 ? launch_inst<BLOCK_N, true, false, true, PAIR>(a, dev, stream)
                   : launch_inst<BLOCK_N, true, false, false, PAIR>(a, dev, stream);
}

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; }

// the weight gradient with the SGD update in its epilogue (GemmArgs::sgd_master)
int launch_wgrad_sgd(const GemmArgs& a, GemmDev d, cudaStream_t stream) {
  // an opt-in stream-K or cluster schedule would apply the update once per partial / CTA
  if (!a.out_f32 || !a.a_mn || !a.b_mn || a.stream_k > 0 || a.pair > 0 || a.bias != nullptr ||
      a.aux != nullptr || a.out2 != nullptr || a.act != ACT_NONE || a.dropout_p > 0.f ||
      a.signal_flags != nullptr || a.wait_flags != nullptr)
    return 980;
  if (a.sgd_shadow == nullptr || a.out == nullptr || !aligned16(a.out) ||
      !aligned16(a.sgd_master) || !aligned16(a.sgd_shadow) || (a.ldo % 8) != 0)
    return 981;
  d.sgd_p = a.sgd_master;
  d.sgd_shadow = reinterpret_cast<__nv_bfloat16*>(a.sgd_shadow);
  d.sgd_lr = a.sgd_lr;
  d.sgd_weight_decay = a.sgd_weight_decay;
  d.sgd_grad_scale = a.sgd_grad_scale;
  const int bn = a.block_n ? a.block_n : gemm_pick_block_n(a.M, a.N);
  if (bn == 256) return launch_inst<256, true, true, true, 1, true>(a, d, stream);
  if (bn == 128) return launch_inst<128, true, true, true, 1, true>(a, d, stream);
  return 905;
}
}  // namespace


// ---- GEMM + LayerNorm epilogue: tile width, cluster size ----
int gemm_ln_block_n(int M, int N, bool force) {
  // 0 = do not run the fused kernel for this shape.  The fused kernel is chosen once 256-wide
  // tiles in (N / 256)-CTA clusters fill most of the GPU (>= 96 CTAs, i.e. >= 3072 tokens at
  // N = 1024); with fewer tokens the two-kernel path's 128-wide GEMM tiles use twice as many SMs.
  // `force` (tests, SKY_FUSE_LN=force) accepts every shape the kernel can run.
  if (M <= 0 || N <= 0 || (N % 128) != 0) return 0;
  const long long panels = (M + 127) / 128;
  const bool ok256 = (N % 256) == 0 && N / 256 <= kLnMaxCluster;
  const bool ok128 = N / 128 <= kLnMaxCluster;
  if (ok256 && panels * (N / 256) >= 96) return 256;
  if (!force) return 0;
  if (ok256) return 256;
  return ok128 ? 128 : 0;
}
int gemm_ln_tiles_per_panel(int M, int N, bool force) {
  const int bn = gemm_ln_block_n(M, N, force);
  return bn ? N / bn : 0;
}

namespace {
template <int BLOCK_N>
int launch_ln_inst(const GemmArgs& a, const GemmLnDev& d, cudaStream_t stream) {
  CUtensorMap tma, tmb;
  int rc = make_tmap_bf16_2d(&tma, a.A, a.K, a.M, a.lda, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmb, a.B, a.K, a.N, a.ldb, BLOCK_K, BLOCK_N);
  if (rc) return rc;
  const int cln = a.N / BLOCK_N;
  const int panels = (a.M + BLOCK_M - 1) / BLOCK_M;
  return launch<gemm_ln_wgmma_kernel<BLOCK_N>>(panels * cln, cln, LnCfg<BLOCK_N>::kSmemBytes,
                                               stream, tma, tmb, d);
}

// the pair layout runs N = 1024 with 256-wide warpgroup tiles
bool ln_pair_layout(int N, int block_n) { return block_n == 256 && N == 2 * LnPairCfg::kCols; }

int launch_ln_pair(const GemmArgs& a, const GemmLnDev& d, cudaStream_t stream) {
  using L = LnPairCfg;
  CUtensorMap tma, tmb;
  int rc = make_tmap_bf16_2d(&tma, a.A, a.K, a.M, a.lda, BLOCK_K, L::kRows);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmb, a.B, a.K, a.N, a.ldb, BLOCK_K, L::kCols / 2);
  if (rc) return rc;
  // whole 128-row panels, so that every panel's flag receives its 4 signals even when M is ragged
  // (the rows of a pair past M are loaded as zeros and never stored)
  const int pairs = 2 * ((a.M + BLOCK_M - 1) / BLOCK_M);
  return launch<gemm_ln_pair_kernel>(2 * pairs, 2, L::kSmemBytes, stream, tma, tmb, d);
}
}  // namespace

int launch_gemm_ln(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return 0;
  if (a.a_mn || a.b_mn || a.out_f32 || a.accumulate || a.act != ACT_NONE) return 908;
  if ((a.K % 8) != 0 || (a.lda % 8) != 0 || (a.ldb % 8) != 0) return 902;
  if (a.ln_gamma == nullptr || a.ln_beta == nullptr || a.ln_mean == nullptr ||
      a.ln_rstd == nullptr || a.out == nullptr)
    return 909;
  if (a.dropout_p > 0.f && a.rng_state == nullptr) return 903;
  if (a.aux != nullptr && !a.add_aux) return 908;
  const int bn = a.block_n ? a.block_n : gemm_ln_block_n(a.M, a.N, true);
  if (bn == 0 || (a.N % bn) != 0 || a.N / bn > kLnMaxCluster) return 907;
  GemmLnDev d{common_of(a)};
  d.y = a.out;
  d.ldy = a.ldo;
  d.z = a.out2;
  d.ldz = a.ldo2;
  d.gamma = a.ln_gamma;
  d.beta = a.ln_beta;
  d.mean = a.ln_mean;
  d.rstd = a.ln_rstd;
  d.eps = a.ln_eps;
  d.debug = a.debug;
  if (ln_pair_layout(a.N, bn)) return launch_ln_pair(a, d, stream);
  if (bn == 256) return launch_ln_inst<256>(a, d, stream);
  if (bn == 128) return launch_ln_inst<128>(a, d, stream);
  return 905;
}

namespace {
// clusters of `cluster` CTAs of `kern` with `smem` bytes of dynamic shared memory each that the
// device can hold at once; < 0: minus the CUDA error
template <class Kern>
int max_active_clusters(Kern kern, int smem, int cluster) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return -static_cast<int>(e);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cluster * 64);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = static_cast<unsigned>(cluster);
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
  return e == cudaSuccess ? n : -static_cast<int>(e);
}
}  // namespace

int gemm_ln_max_active_clusters(int N, int block_n, int* cluster) {
  *cluster = 0;
  if ((block_n != 128 && block_n != 256) || N % block_n != 0 || N / block_n > kLnMaxCluster)
    return -907;
  if (ln_pair_layout(N, block_n)) {
    *cluster = 2;
    return max_active_clusters(gemm_ln_pair_kernel, LnPairCfg::kSmemBytes, 2);
  }
  *cluster = N / block_n;
  if (block_n == 256)
    return max_active_clusters(gemm_ln_wgmma_kernel<256>, LnCfg<256>::kSmemBytes, *cluster);
  return max_active_clusters(gemm_ln_wgmma_kernel<128>, LnCfg<128>::kSmemBytes, *cluster);
}

int launch_gemm(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return 0;
  if (a.ln_gamma != nullptr) return launch_gemm_ln(a, stream);
  if ((a.N % 8) != 0 || (a.K % 8) != 0 || (a.lda % 8) != 0 || (a.ldb % 8) != 0) return 902;
  if (a.a_mn && (a.M % 8) != 0) return 902;
  if (a.dropout_p > 0.f && a.rng_state == nullptr) return 903;
  if (a.accumulate && !a.out_f32) return 904;
  GemmDev d{common_of(a)};  // no stream-K until launch_inst picks it
  d.out = a.out;
  d.out2 = a.out2;
  d.ldo = a.ldo;
  d.ldo2 = a.ldo2;
  d.act = a.act;
  d.add_aux = a.add_aux ? 1 : 0;
  d.accumulate = a.accumulate ? 1 : 0;
  d.debug = a.debug;
  if (a.sgd_master != nullptr) return launch_wgrad_sgd(a, d, stream);
  const int bn = a.block_n ? a.block_n : gemm_pick_block_n(a.M, a.N);
  const bool auto_quad = a.pair < 0 && a.block_n == 0 && pick_quad();
  const bool pair = a.pair < 0 ? (auto_quad || pick_pair(a.M)) : (a.pair != 0);
  if (pair) {
    // two pairs + A multicast needs an even number of N tiles
    const bool quad = (a.pair == 2 || auto_quad) &&
                      (((a.N + bn - 1) / bn) % 2 == 0);
    if (quad) {
      if (bn == 256) return dispatch_major<256, 4>(a, d, stream);
      if (bn == 128) return dispatch_major<128, 4>(a, d, stream);
      return 905;
    }
    if (bn == 256) return dispatch_major<256, 2>(a, d, stream);
    if (bn == 128) return dispatch_major<128, 2>(a, d, stream);
    return 905;
  }
  if (bn == 256) return dispatch_major<256, 1>(a, d, stream);
  if (bn == 128) return dispatch_major<128, 1>(a, d, stream);
  return 905;
}

}  // namespace sky
