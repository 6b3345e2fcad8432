// mma_tf32.cuh -- FP32-grade matrix products on the tensor cores (3xTF32), shared by explain_gang.cu and explain_dense.cu.
#pragma once
#include <stdint.h>

namespace {

__device__ __forceinline__ uint32_t tf32_of(float x) { uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return r; }
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_of(x);
  lo = tf32_of(x - __uint_as_float(hi));
}
// c += a b: one mma.sync m16n8k8 (A 16x8 row-major fragment a[4], B 8x8 column fragment (b0, b1), FP32 accumulate)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// 3xTF32: (ahi + alo)(bhi + blo) without the lo*lo term = alo*bhi + ahi*blo (small) + ahi*bhi (big), each an mma_tf32 (see the callers)

}  // namespace
