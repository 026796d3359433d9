// dmma.cuh -- building blocks of the fp64 tensor-core kernels (gramian.cu, project.cu; internal, sm_90a): the exact widening of a
// storage-type element, the cp.async ring primitives and the m16n8k4 fp64 MMA.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace agd {

template <typename T> struct GmElem;
template <> struct GmElem<float> {
  __device__ static double wide(float x) { return (double)x; }
};
template <> struct GmElem<double> {
  __device__ static double wide(double x) { return x; }
};
template <> struct GmElem<__nv_bfloat16> {
  __device__ static double wide(__nv_bfloat16 x) { return (double)__uint_as_float((uint32_t)__bfloat16_as_ushort(x) << 16); }
};

// 16 bytes global -> shared; bytes = 0 reads nothing and fills the 16 bytes with zeros
__device__ __forceinline__ void gm_cp16(uint32_t dst, const void *src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gm_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void gm_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// D (16 x 8) += A (16 x 4, row) B (4 x 8, col), fp64 throughout
__device__ __forceinline__ void gm_dmma(double (&c)[4], const double (&a)[2], double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(b));
}

}  // namespace agd
