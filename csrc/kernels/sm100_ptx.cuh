// sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (descriptors / mma_async /
// commit / wait), thread-block clusters and distributed shared memory, system-scope
// release/acquire for cross-GPU flags.
//
// Everything here is hand-written inline PTX for Hopper (H100, compute_90a).  No CUTLASS/CuTe
// types are used; descriptor bit layouts follow the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
namespace sky {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 %%rx;\n"
      ".reg .pred %%px;\n"
      "elect.sync %%rx|%%px, %1;\n"
      "@%%px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Programmatic dependent launch: wait until the previous grid in the stream has completed (and its
// memory is visible); allow the next grid to start launching.  No-ops without the launch attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 2D tiled load global -> shared, completion signalled on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int c_inner, int c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c_inner), "r"(c_outer)
      : "memory");
}

// 3D tiled load (inner, middle, outer coordinates); out-of-range elements are zero-filled, which
// is how the tiled attention kernels read ragged last tiles of a sequence.
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cta address -> shared::cluster address of the same offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr)
               : "memory");
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
// distributed shared memory: store two floats into another CTA of the cluster
__device__ __forceinline__ void st_cluster_v2_f32(uint32_t cluster_addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(cluster_addr), "f"(a), "f"(b)
               : "memory");
}
// wait on a LOCAL mbarrier whose arrivals (and the data they publish) come from other CTAs of the
// cluster: acquire at cluster scope
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
// ----------------------------------------------------------------------------------------------
// wgmma: warpgroup-wide asynchronous MMA, D[64 x N] (fp32 registers) (+)= A[smem] * B[smem]
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, SWIZZLE_128B.  Bit layout (PTX ISA, "wgmma matrix descriptor"):
//   [0,14)  start address >> 4      [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4     [49,52) base offset (0: tiles are 1024B aligned)
//   [62,64) swizzle mode (1 = 128B)
// K-major operand:  8-row atoms 1024 B apart (SBO), LBO unused; a 16-element K step = +32 B
// MN-major operand: 64-element MN chunks LBO apart, 8-k-row groups 1024 B apart (SBO); a 16-row
//                   K step = +2048 B
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// TA / TB = 1: the operand is MN-major in shared memory ("transposed"), 0: K-major
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                                 uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b,
                                                 uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),
        "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b,
                                                 uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),
        "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]),
        "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]),
        "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]),
        "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]),
        "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]),
        "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]),
        "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]),
        "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]),
        "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_k16(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b,
                                          uint32_t scale_d) {
  static_assert(N == 64 || N == 128 || N == 256, "unsupported wgmma width");
  if constexpr (N == 64) wgmma_m64n64k16<TA, TB>(d, desc_a, desc_b, scale_d);
  if constexpr (N == 128) wgmma_m64n128k16<TA, TB>(d, desc_a, desc_b, scale_d);
  if constexpr (N == 256) wgmma_m64n256k16<TA, TB>(d, desc_a, desc_b, scale_d);
}
// Accumulator fragment of one warpgroup thread: warp w of the group owns rows 16w .. 16w+15; lane l
// holds, for every 8-column block j, d[4j], d[4j+1] = (row 16w + l/4, columns 8j + 2(l%4) + {0,1})
// and d[4j+2], d[4j+3] = the same columns of row + 8.

// Register-A wgmma: D[64 x N] (+)= A[64 x 16] (registers) * B (shared memory).  Only B takes a
// transpose bit in this form (TB = 1: B is MN-major).  A thread's A fragment is four bf16x2 words:
//   a[0] = (row fr, k 2(l%4) + {0,1}),     a[1] = (row fr + 8, the same k),
//   a[2] = (row fr, k 8 + 2(l%4) + {0,1}), a[3] = (row fr + 8, the same k),
// with fr = 16 (warp % 4) + l / 4.  That is the accumulator fragment layout above restricted to
// 16 columns, so the accumulator d of columns 16k .. 16k + 15 IS the A fragment of K step k:
//   a[0] = pack(d[8k], d[8k+1]), a[1] = pack(d[8k+2], d[8k+3]),
//   a[2] = pack(d[8k+4], d[8k+5]), a[3] = pack(d[8k+6], d[8k+7])
// (frag_to_a below), and a bf16 probability tile goes from one MMA into the next with no shuffle.
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4],
                                                    uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, %38;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4],
                                                     uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, %70;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),
        "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d), "n"(TB));
}
// Pins an accumulator's registers at this point of the instruction stream.  Zero-initialising an
// accumulator is plain register moves, which the compiler may otherwise sink past an earlier
// wgmma that is still in flight; ptxas then serialises the two MMAs with an injected wait.
template <int NREG>
__device__ __forceinline__ void acc_fence(float (&d)[NREG]) {
#pragma unroll
  for (int i = 0; i < NREG; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N, int TB>
__device__ __forceinline__ void wgmma_rs_k16(float (&d)[N / 2], const uint32_t (&a)[4],
                                             uint64_t desc_b, uint32_t scale_d) {
  static_assert(N == 64 || N == 128, "unsupported register-A wgmma width");
  if constexpr (N == 64) wgmma_m64n64k16_rs<TB>(d, a, desc_b, scale_d);
  if constexpr (N == 128) wgmma_m64n128k16_rs<TB>(d, a, desc_b, scale_d);
}
// TMA load delivered to every CTA of `mask` at the same CTA-relative offsets (data and barrier)
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                               int c_inner, int c_outer, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      ".multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;"
      ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "h"(mask), "r"(c_inner), "r"(c_outer)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// cross-GPU flags (system scope)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void red_release_sys_add(uint32_t* addr, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
// Spin until *addr >= target (monotonic counters). Returns false on timeout (ns budget).
__device__ __forceinline__ bool wait_flag_ge(const uint32_t* addr, uint32_t target,
                                             uint64_t timeout_ns) {
  if (ld_acquire_sys(addr) >= target) return true;
  const uint64_t t0 = globaltimer_ns();
  while (true) {
    if (ld_acquire_sys(addr) >= target) return true;
    if (globaltimer_ns() - t0 > timeout_ns) return false;
    __nanosleep(64);
  }
}

// ----------------------------------------------------------------------------------------------
// small math helpers shared by epilogues
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(h);
}

// erf-form GELU as used by BERT (x * 0.5 * (1 + erf(x / sqrt(2)))).
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
}
// d/dx gelu_erf(x) = Phi(x) + x * phi(x)
__device__ __forceinline__ float dgelu_erf(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// Fast variants for GEMM epilogues (Abramowitz-Stegun 7.1.26 erf, |err| < 1.5e-7 - far below
// bf16 resolution): one MUFU.RCP + one MUFU.EX2 + 6 FMA instead of libdevice erff.
__device__ __forceinline__ float erf_exp_fast(float z_abs, float& e_out) {
  // returns erf(z_abs) for z_abs >= 0 and e_out = exp(-z^2)
  // rcp.approx (one MUFU): __frcp_rn expands to MUFU + Newton steps + a slow-path branch per
  // element, which serialised the whole epilogue (tools/triage_gemm.py: +30 us on FFN1)
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z_abs, 1.0f)));
  float poly = 1.061405429f;
  poly = fmaf(poly, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  e_out = __expf(-z_abs * z_abs);
  return fmaf(-poly, e_out, 1.0f);
}
__device__ __forceinline__ float gelu_fast(float x) {
  float e;
  const float er = erf_exp_fast(fabsf(x) * 0.70710678118654752f, e);
  return 0.5f * x * (1.0f + copysignf(er, x));
}
__device__ __forceinline__ float dgelu_fast(float x) {
  float e;  // exp(-x^2/2)
  const float er = erf_exp_fast(fabsf(x) * 0.70710678118654752f, e);
  const float cdf = 0.5f * (1.0f + copysignf(er, x));
  return fmaf(x * 0.3989422804014327f, e, cdf);
}
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// `bytes` (a multiple of 16) from a 16-byte aligned global address into L2, asynchronously
__device__ __forceinline__ void prefetch_l2_bulk(const void* ptr, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(ptr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void red_add_v2_f32(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// The SGD update of one element, shared by sgd_multi_kernel and the weight-gradient GEMM that
// applies the update in its epilogue: d = g * grad_scale (* clip) + weight_decay * p, then
// p - lr * d.  The roundings are spelled out (one multiply per scale, two FMAs) so that both
// kernels compute the same bits whatever the compiler would contract around the call.
// kScalars: the gradient is also multiplied by the clip coefficient (device OptimScalars).
template <bool kScalars>
__device__ __forceinline__ float sgd_direction(float g, float p, float grad_scale, float clip,
                                               float weight_decay) {
  float s = __fmul_rn(g, grad_scale);
  if constexpr (kScalars) s = __fmul_rn(s, clip);
  return __fmaf_rn(weight_decay, p, s);
}
__device__ __forceinline__ float sgd_apply(float p, float d, float lr) {
  return __fmaf_rn(-lr, d, p);
}

// Counter-based RNG for dropout: splitmix64 of (seed, element-group index) -> 4 x 16-bit lanes.
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// Effective per-step seed: {seed, step} live in device memory so CUDA-graph replays advance it.
__device__ __forceinline__ uint64_t dropout_seed(const uint64_t* rng_state, uint32_t stream) {
  return splitmix64(rng_state[0] + 0x632BE59BD9B4E019ull * (rng_state[1] + 1)) ^
         (static_cast<uint64_t>(stream) << 32);
}
// Dropout parameters of one launch.  The seed is read only when p > 0: rng_state may be null
// otherwise.
struct Dropout {
  bool on;
  uint64_t seed;
  uint32_t thr16;  // p * 65536
  float scale;     // 1 / (1 - p) for kept elements
};
__device__ __forceinline__ Dropout dropout_of(float p, const uint64_t* rng_state, uint32_t stream) {
  Dropout d{p > 0.f, 0, 0, 1.f};
  if (d.on) {
    d.seed = dropout_seed(rng_state, stream);
    d.thr16 = static_cast<uint32_t>(p * 65536.f);
    d.scale = 1.f / (1.f - p);
  }
  return d;
}
// keep-mask for 4 consecutive elements starting at element index `idx4*4`; thr16 = p * 65536.
__device__ __forceinline__ uint32_t dropout_keep4(uint64_t seed, uint64_t idx4, uint32_t thr16) {
  const uint64_t r = splitmix64(seed ^ (idx4 * 0xD1342543DE82EF95ull));
  uint32_t m = 0;
  m |= (static_cast<uint32_t>(r & 0xFFFF) >= thr16) ? 1u : 0u;
  m |= (static_cast<uint32_t>((r >> 16) & 0xFFFF) >= thr16) ? 2u : 0u;
  m |= (static_cast<uint32_t>((r >> 32) & 0xFFFF) >= thr16) ? 4u : 0u;
  m |= (static_cast<uint32_t>((r >> 48) & 0xFFFF) >= thr16) ? 8u : 0u;
  return m;
}

// ----------------------------------------------------------------------------------------------
// epilogues on accumulator fragments (GEMM and attention)
// ----------------------------------------------------------------------------------------------
// A thread holds, of each 64-column group of its warpgroup's 64 x N accumulator, f[4j], f[4j+1] =
// (row fr, columns 8j + fc + {0,1}) and f[4j+2], f[4j+3] = (row fr + 8, the same columns), j =
// 0..7, with fr = lane / 4 and fc = 2 (lane % 4) (see the accumulator fragment layout above).
//
// Per-warp bf16 staging buffer: the warp's 16 fragment rows x 64 columns, rows 144 B apart (128 B +
// 16 B pad).  With that stride both the fragment side (4-byte column pairs, 8 rows x 4 lanes) and
// the global side (16-byte pieces, 8 lanes per row) are bank-conflict free.
constexpr int kStageLd = 144;
constexpr int kWarpStageBytes = 16 * kStageLd;

// f (16 rows x 64 columns, bf16) -> gout rows grow0 .. grow0 + 15, columns col0 .. col0 + 63,
// through the warp's staging buffer `s` so that every global store is a whole 16-byte piece of a
// 128-byte row; rows >= m and 8-column pieces >= n are skipped
__device__ __forceinline__ void frag_store_bf16(const float (&f)[32], uint8_t* s, int lane,
                                                __nv_bfloat16* gout, long long ld, long long grow0,
                                                int m, int col0, int n) {
  uint8_t* mine = s + (lane >> 2) * kStageLd + (lane & 3) * 4;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    *reinterpret_cast<uint32_t*>(mine + j * 16) = pack_bf16x2(f[4 * j], f[4 * j + 1]);
    *reinterpret_cast<uint32_t*>(mine + 8 * kStageLd + j * 16) =
        pack_bf16x2(f[4 * j + 2], f[4 * j + 3]);
  }
  __syncwarp();
  const int piece = lane & 7;
  if (col0 + piece * 8 < n) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = i * 4 + (lane >> 3);
      if (grow0 + r < m) {
        const uint4 val = *reinterpret_cast<const uint4*>(s + r * kStageLd + piece * 16);
        *reinterpret_cast<uint4*>(gout + (grow0 + r) * ld + col0 + piece * 8) = val;
      }
    }
  }
  __syncwarp();
}

// Dropout keep bits of 8-column block j of a fragment group, for the element-wise mask
// dropout_keep4(seed, (row * n + col) >> 2) with row_a = the global row of fragment row fr and
// col0 = the group's first column: bits 0, 1 = (row fr, my two columns), bits 2, 3 = (row fr + 8,
// the same columns).  A 4-column group belongs to lanes l and l ^ 1: the even lane hashes it for
// row fr, the odd lane for row fr + 8, and they swap results.
__device__ __forceinline__ uint32_t frag_keep_bits(uint64_t seed, uint32_t thr16, long long row_a,
                                                   int col0, int n, int lane, int j) {
  const int odd = lane & 1;
  const uint64_t row = static_cast<uint64_t>(row_a + (odd ? 8 : 0));
  const int c4 = col0 + (lane & 2) * 2;  // first column of my 4-column group in block 0
  const uint32_t sh = odd * 2;           // my column pair's bits in the group's mask
  const uint32_t h =
      dropout_keep4(seed, (row * static_cast<uint64_t>(n) + c4 + j * 8) >> 2, thr16);
  const uint32_t o = __shfl_xor_sync(0xffffffffu, h, 1);
  const uint32_t ma = (odd ? o : h) >> sh;
  const uint32_t mb = (odd ? h : o) >> sh;
  return (ma & 3u) | ((mb & 3u) << 2);
}
// dropout on the 64-column fragment groups of f (columns col0, col0 + 64, ...): kept elements are
// multiplied by `scale`, dropped ones become 0
template <int NREG>
__device__ __forceinline__ void frag_dropout(float (&f)[NREG], uint64_t seed, uint32_t thr16,
                                             float scale, long long row_a, int col0, int n,
                                             int lane) {
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    const uint32_t m = frag_keep_bits(seed, thr16, row_a, col0 + (j >> 3) * 64, n, lane, j & 7);
    f[4 * j] = (m & 1u) ? f[4 * j] * scale : 0.f;
    f[4 * j + 1] = (m & 2u) ? f[4 * j + 1] * scale : 0.f;
    f[4 * j + 2] = (m & 4u) ? f[4 * j + 2] * scale : 0.f;
    f[4 * j + 3] = (m & 8u) ? f[4 * j + 3] * scale : 0.f;
  }
}

// accumulator columns 16k .. 16k + 15 -> register A fragment of K step k (see wgmma_m64n64k16_rs)
template <int NREG>
__device__ __forceinline__ void frag_to_a(const float (&d)[NREG], int k, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * k], d[8 * k + 1]);
  a[1] = pack_bf16x2(d[8 * k + 2], d[8 * k + 3]);
  a[2] = pack_bf16x2(d[8 * k + 4], d[8 * k + 5]);
  a[3] = pack_bf16x2(d[8 * k + 6], d[8 * k + 7]);
}

// descriptor of K step k of a K-major [rows x 64 * nblk] bf16 operand kept as 64-wide K blocks
// `blk_bytes` apart (row offset row0, a multiple of 8) / of an MN-major operand
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t base, int k, uint32_t blk_bytes, int row0) {
  return make_smem_desc_sw128(base + (k >> 2) * blk_bytes + (k & 3) * 32 + row0 * 128, 16, 1024);
}
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t base, int k, uint32_t chunk_bytes,
                                                 int chunk) {
  return make_smem_desc_sw128(base + chunk * chunk_bytes + k * 2048, chunk_bytes, 1024);
}

}  // namespace sky
