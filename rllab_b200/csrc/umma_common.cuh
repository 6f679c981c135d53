// Warpgroup tensor-core (wgmma, sm_90a) helpers shared by the tensor-core update kernels (update_umma.cu: 64-wide
// gradient and Fisher-vector product; update_umma32.cu: 32-wide passes).  Inline PTX: the shared-memory matrix descriptor
// (K-major, no swizzle), wgmma.mma_async .tf32 with the A operand in registers and the B operand in shared memory, fence /
// commit / wait of the warpgroup's MMA groups.
//
// Fragment layout of one warpgroup's m64nN float32 accumulator (thread = warp w of the warpgroup, lane = 4 g + t):
//   d[i]  row  16 w + g + 8 ((i >> 1) & 1),  column  8 (i >> 2) + 2 t + (i & 1)
// The A operand of an m64n*k8 .tf32 MMA holds, per thread, rows (16 w + g, 16 w + g + 8) at k-slots (t, t + 4).  Feeding
// a layer's output straight back as the next layer's A operand therefore maps k-slot s of each 8-wide k-block to the
// input feature u_kperm^-1(s) (slot t <-> feature 2t, slot t + 4 <-> feature 2t + 1); every weight image stores its K index
// through u_kperm so that the two agree (a permutation of the summation index: the product is unchanged).
#pragma once
#include <stdint.h>

#include "update_common.cuh"

namespace b200rl {

__device__ __forceinline__ uint32_t u_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// hi word of the operand split: the float32 word with its 13 low mantissa bits cleared (exactly representable in TF32);
// lo = x - hi is exact in float32.
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// position of input feature k inside the K-major weight images (see the header comment)
__host__ __device__ constexpr int u_kperm(int k) { return (k & ~7) | ((k & 1) << 2) | ((k >> 1) & 3); }

// row / column of accumulator element i of this thread inside the warpgroup's 64-row block
__device__ __forceinline__ int u_frag_row(int i, int lane) { return (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int u_frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }

// accumulator-ordered values -> A-operand hi / lo words (within each group of four: elements 1 and 2 trade places)
template <int NV>
__device__ __forceinline__ void u_to_operand(const float (&f)[NV], uint32_t (&hi)[NV], uint32_t (&lo)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float v = f[(i & ~3) | ((i & 1) << 1) | ((i >> 1) & 1)];
    const float vh = tf32_hi(v);
    hi[i] = __float_as_uint(vh);
    lo[i] = __float_as_uint(v - vh);
  }
}

// shared-memory matrix descriptor, K-major, no swizzle (layout type 0): start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32.
// LBO: byte distance of adjacent 8x16 B core matrices along K; SBO: along M / N.
__device__ __forceinline__ uint64_t u_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulators across the wait
template <int NV>
__device__ __forceinline__ void wg_fence_operand(float (&d)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A[64 x 8] B[8 x 64]; a: this thread's four A words of the k-step
__device__ __forceinline__ void wg_mma_n64(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                           uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"(accumulate)
      : "memory");
}
// D[64 x 32] (+)= A[64 x 8] B[8 x 32]
__device__ __forceinline__ void wg_mma_n32(float (&d)[16], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                           uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// three-pass split GEMM over KS k-steps of 8 into one warpgroup's accumulator: D (+)= A B with
// a b ~ a_lo b_hi + a_hi b_lo + a_hi b_hi (small terms first), A hi / lo words in registers (u_to_operand), B hi / lo
// images in shared memory, consecutive k-steps `kstep_bytes` apart.  The caller fences before and commits / waits after.
template <int NACC, int NA>
__device__ __forceinline__ void wg_split_gemm(float (&d)[NACC], const uint32_t (&ahi)[NA], const uint32_t (&alo)[NA],
                                              uint64_t b_hi, uint64_t b_lo, uint32_t kstep_bytes, int KS, bool accumulate) {
  static_assert(NACC == 32 || NACC == 16, "m64n64 or m64n32");
#pragma unroll
  for (int ks = 0; ks < NA / 4; ++ks) {
    if (ks < KS) {
      const uint64_t koff = (uint64_t)((ks * kstep_bytes) >> 4);
      const uint32_t acc0 = (accumulate || ks > 0) ? 1u : 0u;
      if constexpr (NACC == 32) {
        wg_mma_n64(d, alo[4 * ks], alo[4 * ks + 1], alo[4 * ks + 2], alo[4 * ks + 3], b_hi + koff, acc0);
        wg_mma_n64(d, ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3], b_lo + koff, 1u);
        wg_mma_n64(d, ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3], b_hi + koff, 1u);
      } else {
        wg_mma_n32(d, alo[4 * ks], alo[4 * ks + 1], alo[4 * ks + 2], alo[4 * ks + 3], b_hi + koff, acc0);
        wg_mma_n32(d, ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3], b_lo + koff, 1u);
        wg_mma_n32(d, ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3], b_hi + koff, 1u);
      }
    }
  }
}

}  // namespace b200rl
