// cg_tc_ptx.cuh -- inline-PTX wrappers for the sm_90a tensor-core kernels (wgmma / mbarrier / bulk copies).
// Shared by the trunk kernel (cg_trunk_tc.cu) and the fully-connected kernel (cg_linear_tc.cu).
//
// Operand conventions of the wgmma below: D (fp32, registers) = A (registers, or shared memory for wg_ss_*) x B
// (shared memory).
// A and D use the m64nNk16 register fragments of the PTX ISA: warp w of the warpgroup owns rows 16w .. 16w+15;
// with g = lane / 4 and q = lane % 4 a thread holds
//   D: d[4i + e] = (row g, col 8i + 2q + e),  d[4i + 2 + e] = (row g + 8, col 8i + 2q + e)      i < N/8, e < 2
//   A (k-step of 16): r0 = (row g, k 2q..2q+1), r1 = (row g+8, k 2q..), r2 = (row g, k 8+2q..), r3 = (row g+8, k 8+2q..)
// so the D of one layer is the A of the next without any data movement (d_to_a below).
// B (and a shared-memory A) is an [N (M) rows x 64] K-block in the canonical K-major SWIZZLE_128B layout
// (row_chunk_off), 1024-byte aligned.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace cg_ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// the spin loop lives inside the asm: to the compiler the wait is straight-line code, so the wgmma that follow it are
// not in a divergent path (which would make ptxas serialize them)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "CG_MBAR_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra CG_MBAR_WAIT;\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}
// 1-D bulk copy global -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory descriptor, K-major SWIZZLE_128B: start address (>>4), LBO = 1 (unused for swizzled K-major),
// SBO = 1024 B between 8-row groups, layout type 1 = SWIZZLE_128B (bits 62-63).  A K-step of 16 elements inside the
// 128-byte swizzle atom advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Operand fences: an empty asm that reads and writes each of n registers.  The "memory" clobber of the fence / commit /
// wait wrappers above does not order register accesses, so without these the compiler may move a read of an
// accumulator above the wait that completes it, or the write of an A fragment below the fence before its wgmma; ptxas
// then repairs the order by injecting a full warpgroup.wait / warpgroup.arrive (C7517 / C7519) and the pipeline is lost.
// Fence the accumulators before the wgmma.fence of a group and after the wait that completes it, and the A fragments
// after they are written and after the last wgmma that reads them is complete.
template <int N>
__device__ __forceinline__ void wg_fence_regs(float *r) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wg_fence_regs(uint32_t *r) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+r"(r[i])::"memory");
}

#define CG_WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                    "+f"(d[i + 6]), "+f"(d[i + 7])

// D[64 x 64] (+)= A[64 x 16] (registers) . B[64 x 16] (shared, K-major); F16 selects fp16 x fp16, else bf16 x bf16
template <bool F16>
__device__ __forceinline__ void wg_m64n64(float *d, const uint32_t *a, uint64_t bdesc, uint32_t accumulate) {
  if (F16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
}

// D[64 x 128] (+)= A[64 x 16] (registers) . B[128 x 16] (shared, K-major); F16 selects fp16 x fp16, else bf16 x bf16
template <bool F16>
__device__ __forceinline__ void wg_m64n128(float *d, const uint32_t *a, uint64_t bdesc, uint32_t accumulate) {
  if (F16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24), CG_WG_D8(32), CG_WG_D8(40), CG_WG_D8(48), CG_WG_D8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24), CG_WG_D8(32), CG_WG_D8(40), CG_WG_D8(48), CG_WG_D8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
}
// D[64 x 128] (+)= A[64 x 16] (shared, K-major) . B[128 x 16] (shared, K-major); both operands by descriptor
template <bool F16>
__device__ __forceinline__ void wg_ss_m64n128(float *d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if (F16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24), CG_WG_D8(32), CG_WG_D8(40), CG_WG_D8(48), CG_WG_D8(56)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : CG_WG_D8(0), CG_WG_D8(8), CG_WG_D8(16), CG_WG_D8(24), CG_WG_D8(32), CG_WG_D8(40), CG_WG_D8(48), CG_WG_D8(56)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
}
#undef CG_WG_D8

// x = hi + lo in bf16 (hi = bf16(x), lo = bf16(x - hi)); two values per 32-bit word, the first in the low half
__device__ __forceinline__ void split_bf16x2(float x0, float x1, uint32_t &h, uint32_t &l) {
  const __nv_bfloat162 hh = __floats2bfloat162_rn(x0, x1);
  h = *reinterpret_cast<const uint32_t *>(&hh);
  const __nv_bfloat162 ll = __floats2bfloat162_rn(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xffff0000u));
  l = *reinterpret_cast<const uint32_t *>(&ll);
}
// fp16 flavour; inputs are clamped to the fp16 range so that an outlier saturates instead of turning into inf
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t &h, uint32_t &l) {
  x0 = fminf(fmaxf(x0, -65504.f), 65504.f);
  x1 = fminf(fmaxf(x1, -65504.f), 65504.f);
  const __half2 hh = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  h = *reinterpret_cast<const uint32_t *>(&hh);
  l = *reinterpret_cast<const uint32_t *>(&ll);
}

// D fragment (N = 16 * KS columns) -> A fragments of the KS k-steps of the next layer, split into hi / lo
template <int KS, bool F16>
__device__ __forceinline__ void d_to_a(const float *d, uint32_t (*hi)[4], uint32_t (*lo)[4]) {
#pragma unroll
  for (int j = 0; j < KS; j++)
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (F16) split_f16x2(d[8 * j + 2 * r], d[8 * j + 2 * r + 1], hi[j][r], lo[j][r]);
      else split_bf16x2(d[8 * j + 2 * r], d[8 * j + 2 * r + 1], hi[j][r], lo[j][r]);
    }
}

// byte offset of the 16-byte chunk `c16` (8 16-bit elements) of row `row` inside one swizzled [rows x 64] K-block
__host__ __device__ __forceinline__ uint32_t row_chunk_off(int row, int c16) {
  return (uint32_t)(row >> 3) * 1024u + (uint32_t)(row & 7) * 128u + (uint32_t)((c16 ^ (row & 7)) << 4);
}

}  // namespace cg_ptx
