// wgmma helpers of the SH blend kernels (sm_90a, bf16 operands in shared memory, fp32 accumulators in registers,
// no-swizzle canonical layouts).
//
// Shared-memory matrix descriptor (64 bit): start address >> 4 in bits [0,14), leading byte offset >> 4 in
// [16,30), stride byte offset >> 4 in [32,46), base offset 0 in [49,52), layout type 0 (no swizzle) in [62,64).
// For the no-swizzle layouts a "core matrix" is 8 rows x 16 bytes, stored as 128 contiguous bytes:
//   K-major  operand (row = M/N index, 16 B = 8 bf16 along K):  LBO = distance between the two core matrices
//            that one K = 16 instruction spans along K, SBO = distance between groups of 8 rows;
//   MN-major operand (row = K index, 16 B = 8 bf16 along M/N):  LBO = distance between the two groups of 8 K
//            rows of one instruction, SBO = distance between groups of 8 M/N elements.
//
// Accumulator fragment of an m64nN instruction issued by a warpgroup: warp w (of the warpgroup), lane L holds
// d[4 i + 2 r + e] = D[16 w + L / 4 + 8 r][8 i + 2 (L % 4) + e],  i < N / 8, r, e in {0, 1}.
//
// Every .sync.aligned instruction below is preceded by __syncwarp(): after divergent code (a subset of threads
// splitting operands, a spin on an mbarrier) the lanes of a warp are not guaranteed to have reconverged.
#pragma once
#include <cuda_bf16.h>

#include "gs_common.cuh"

namespace gs_tc {

__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  const uint32_t lo = ((addr & 0x3FFFFu) >> 4) | ((lbo >> 4) << 16);
  const uint32_t hi = sbo >> 4;
  return ((uint64_t)hi << 32) | lo;
}

// accumulator registers are written by the asynchronous tensor core: keep the compiler from moving accesses
// across the issue / wait points
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wg_fence() {
  __syncwarp();
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() {
  __syncwarp();
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// generic-proxy shared-memory writes -> visible to the tensor core's (async proxy) operand reads
__device__ __forceinline__ void fence_smem_to_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// D[64 x 24] (+)= A[64 x 16] * B[24 x 16]^T, A and B K-major; issued by the whole warpgroup
__device__ __forceinline__ void mma_n24_kk(float (&d)[12], uint64_t a, uint64_t b, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, %12, %13, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
               : "l"(a), "l"(b), "r"(accumulate)
               : "memory");
}
// D[64 x 32] (+)= A[64 x 16] * B[16 x 32], A and B MN-major; issued by the whole warpgroup
__device__ __forceinline__ void mma_n32_mn(float (&d)[16], uint64_t a, uint64_t b, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b), "r"(accumulate)
               : "memory");
}

// x = hi + lo (+ 2^-17 |x|) with hi, lo in bf16: two values per 32-bit word, the first in the low half
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - __low2float(h), b - __high2float(h));
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

}  // namespace gs_tc
