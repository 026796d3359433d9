// synth.cu -- K0: counter-based synthetic workload generated in place on each GPU (measurement
// harness; the reference has no benchmark inputs, SURVEY.md 8(d)), plus the load-path row converter.
//
// Spec (integer arithmetic until the final scaling, so any conforming implementation agrees bit
// for bit; tests/ checks this file against an independent CPU statement of the same spec):
//   Philox4x32-10, key = (seed_lo, seed_hi), counter = (c0, c1, c2, stream)
//   X[i][j]   : counter (i_lo, i_hi, j/2, 1) -> r0..r3 ; (r0,r1) for even j, (r2,r3) for odd j
//               t = lo16(a) + hi16(a) + lo16(b) + hi16(b) - 131070 ;  X = (float)t * (float)(sqrt(3)/65536)
//   w_true[j] : counter (j, 0, 0, 2), t from (r0,r1) ;  w = ((double)t * (sqrt(3)/65536)) / sqrt(d)
//   u_i       : counter (i_lo, i_hi, 0, 3) ;  u = ((r0>>5)*2^26 + (r1>>6) + 0.5) * 2^-53
//   e_i       : counter (i_lo, i_hi, 0, 4), t from (r0,r1) ;  e = (double)t * (sqrt(3)/65536)
//   labels    : logistic y = 1[x.w_true + log(u) - log(1-u) > 0] ; least squares y = x.w_true + 0.1 e ;
//               hinge y = 1[x.w_true > 0] flipped when u < 0.05
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"

namespace agd {

namespace {

__device__ __forceinline__ void philox4x32_10(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2,
                                              uint32_t c3, uint32_t (&out)[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ int irwin_hall4(uint32_t a, uint32_t b) {
  return (int)((a & 0xffffu) + (a >> 16) + (b & 0xffffu) + (b >> 16)) - 131070;
}
template <typename T> __device__ __forceinline__ T from_f32(float v) { return (T)v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <typename T> __device__ __forceinline__ double to_f64(T v) { return (double)v; }
template <> __device__ __forceinline__ double to_f64<__nv_bfloat16>(__nv_bfloat16 v) { return (double)__bfloat162float(v); }
template <typename D, typename S> __device__ __forceinline__ D convert_elem(S v) { return (D)v; }
template <> __device__ __forceinline__ __nv_bfloat16 convert_elem<__nv_bfloat16, float>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 convert_elem<__nv_bfloat16, double>(double v) { return __double2bfloat16(v); }

__device__ __forceinline__ float synth_x_scale() { return (float)(1.7320508075688772 / 65536.0); }

template <typename T>
__global__ void __launch_bounds__(256) synth_dense_kernel(T *X, uint64_t seed, long long row0, long long rows, int d,
                                                         int ld) {
  const int pairs = (ld + 1) / 2;  // columns >= d (row padding) are written as zeros
  const long long total = rows * (long long)pairs;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const float scale = synth_x_scale();
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q < total; q += (long long)gridDim.x * 256LL) {
    const long long r = q / pairs;
    const int jp = (int)(q - r * pairs);
    const unsigned long long i = (unsigned long long)(row0 + r);
    uint32_t o[4];
    philox4x32_10(k0, k1, (uint32_t)i, (uint32_t)(i >> 32), (uint32_t)jp, 1u, o);
    const float x0 = __fmul_rn((float)irwin_hall4(o[0], o[1]), scale);
    const float x1 = __fmul_rn((float)irwin_hall4(o[2], o[3]), scale);
    T *row = X + (size_t)r * ld;
    if (2 * jp < ld) row[2 * jp] = from_f32<T>(2 * jp < d ? x0 : 0.f);  // bf16 storage: the fp32 spec value rounded to nearest-even
    if (2 * jp + 1 < ld) row[2 * jp + 1] = from_f32<T>(2 * jp + 1 < d ? x1 : 0.f);
  }
}

__global__ void synth_wtrue_kernel(double *w, uint64_t seed, int d) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d) return;
  uint32_t o[4];
  philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)j, 0u, 0u, 2u, o);
  w[j] = __ddiv_rn(__dmul_rn((double)irwin_hall4(o[0], o[1]), 1.7320508075688772 / 65536.0), sqrt((double)d));
}

// one warp per row: fp64 dot with w_true, then the label rule
template <typename T>
__global__ void __launch_bounds__(256) synth_labels_kernel(const T *X, const double *w_true, double *labels,
                                                          uint64_t seed, int kind, long long row0, long long rows,
                                                          int d, int ld) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * 256LL + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256LL) >> 5;
  for (long long r = warp_global; r < rows; r += nwarps) {
    const T *row = X + (size_t)r * ld;
    double m = 0.0;
    for (int j = lane; j < d; j += 32) m = fma(to_f64<T>(row[j]), w_true[j], m);
    for (int off = 16; off >= 1; off >>= 1) m += __shfl_xor_sync(0xffffffffu, m, off);
    if (lane == 0) {
      const unsigned long long i = (unsigned long long)(row0 + r);
      uint32_t o[4];
      philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)i, (uint32_t)(i >> 32), 0u, 3u, o);
      const double u = ((double)(o[0] >> 5) * 67108864.0 + (double)(o[1] >> 6) + 0.5) * 0x1.0p-53;
      double y;
      if (kind == AGD_GRAD_LOGISTIC) {
        y = (m + log(u) - log(1.0 - u) > 0) ? 1.0 : 0.0;
      } else if (kind == AGD_GRAD_HINGE) {
        y = (m > 0) ? 1.0 : 0.0;
        if (u < 0.05) y = 1.0 - y;
      } else {
        uint32_t e[4];
        philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)i, (uint32_t)(i >> 32), 0u, 4u, e);
        y = m + 0.1 * ((double)irwin_hall4(e[0], e[1]) * (1.7320508075688772 / 65536.0));
      }
      labels[r] = y;
    }
  }
}

// CSR synthetic rows: exactly k stored entries per row, strictly increasing column ids by stratification
//   entry t of row i: counter (i_lo, i_hi, t, 5) -> col = t*(d/k) + r0 % (d/k) ; value = irwin_hall4(r1, r2) * sqrt(3)/65536
template <typename T>
__global__ void __launch_bounds__(256) synth_csr_kernel(long long *rowptr, int *idx, T *val, uint64_t seed,
                                                       long long row0, long long rows, int d, int k) {
  const long long total = rows * (long long)k;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const uint32_t stride = (uint32_t)(d / k);
  const float scale = synth_x_scale();
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q < total; q += (long long)gridDim.x * 256LL) {
    const long long r = q / k;
    const int t = (int)(q - r * k);
    const unsigned long long i = (unsigned long long)(row0 + r);
    uint32_t o[4];
    philox4x32_10(k0, k1, (uint32_t)i, (uint32_t)(i >> 32), (uint32_t)t, 5u, o);
    idx[q] = (int)((uint32_t)t * stride + o[0] % stride);
    val[q] = from_f32<T>(__fmul_rn((float)irwin_hall4(o[1], o[2]), scale));
    if (t == 0) rowptr[r] = r * (long long)k;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) rowptr[rows] = total;
}

// labels for CSR rows (one warp per row)
template <typename T>
__global__ void __launch_bounds__(256) synth_csr_labels_kernel(const long long *rowptr, const int *idx, const T *val,
                                                              const double *w_true, double *labels, uint64_t seed,
                                                              int kind, long long row0, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * 256LL + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256LL) >> 5;
  for (long long r = warp_global; r < rows; r += nwarps) {
    double m = 0.0;
    for (long long q = rowptr[r] + lane; q < rowptr[r + 1]; q += 32) m = fma(to_f64<T>(val[q]), w_true[idx[q]], m);
    for (int off = 16; off >= 1; off >>= 1) m += __shfl_xor_sync(0xffffffffu, m, off);
    if (lane == 0) {
      const unsigned long long i = (unsigned long long)(row0 + r);
      uint32_t o[4];
      philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)i, (uint32_t)(i >> 32), 0u, 3u, o);
      const double u = ((double)(o[0] >> 5) * 67108864.0 + (double)(o[1] >> 6) + 0.5) * 0x1.0p-53;
      double y;
      if (kind == AGD_GRAD_LOGISTIC) y = (m + log(u) - log(1.0 - u) > 0) ? 1.0 : 0.0;
      else if (kind == AGD_GRAD_HINGE) { y = (m > 0) ? 1.0 : 0.0; if (u < 0.05) y = 1.0 - y; }
      else {
        uint32_t e[4];
        philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)i, (uint32_t)(i >> 32), 0u, 4u, e);
        y = m + 0.1 * ((double)irwin_hall4(e[0], e[1]) * (1.7320508075688772 / 65536.0));
      }
      labels[r] = y;
    }
  }
}

// dst (rows x dst_ld, columns >= d zero-filled) <- src (rows x d, leading dimension ld)
template <typename D, typename S>
__global__ void __launch_bounds__(256) convert_rows_kernel(D *dst, const S *src, long long rows, int d, long long ld,
                                                          int dst_ld) {
  const long long total = rows * (long long)dst_ld;
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q < total; q += (long long)gridDim.x * 256LL) {
    const long long r = q / dst_ld;
    const int j = (int)(q - r * dst_ld);
    dst[q] = j < d ? convert_elem<D, S>(src[r * ld + j]) : convert_elem<D, S>((S)0);
  }
}

__global__ void csr_shift_rowptr_kernel(long long *dst, const long long *src, long long n, long long shift) {
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q < n; q += (long long)gridDim.x * 256LL) dst[q] = src[q] + shift;
}

// Validates an appended CSR partition on the device (the host never scans the index stream): rowptr[0..rows] must be
// non-decreasing, start at 0 and stay within nnz; every column id must lie in [0, d).  flag: 0 ok, 1 rowptr, 2 column.
__global__ void csr_validate_kernel(const long long *rowptr, long long rows, const int *idx, long long nnz, int d, int *flag) {
  const long long stride = (long long)gridDim.x * 256LL;
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q <= rows; q += stride) {
    const long long v = rowptr[q];
    if (v < 0 || v > nnz || (q == 0 && v != 0) || (q == rows && v != nnz) || (q < rows && rowptr[q + 1] < v)) atomicMax(flag, 1);
  }
  for (long long q = blockIdx.x * 256LL + threadIdx.x; q < nnz; q += stride)
    if ((unsigned)idx[q] >= (unsigned)d) atomicMax(flag, 2);
}

inline unsigned grid_for(long long total) {
  long long g = (total + 255) / 256;
  if (g > 132LL * 16) g = 132LL * 16;   // 16 CTAs per H100 SM
  if (g < 1) g = 1;
  return (unsigned)g;
}

}  // namespace

cudaError_t synth_dense_launch(void *X, int elem_bytes, uint64_t seed, int64_t row0, int64_t rows, int32_t d, int32_t ld,
                               cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  const long long total = rows * (long long)((ld + 1) / 2);
  if (elem_bytes == 2)
    synth_dense_kernel<__nv_bfloat16><<<grid_for(total), 256, 0, st>>>((__nv_bfloat16 *)X, seed, row0, rows, d, ld);
  else if (elem_bytes == 4)
    synth_dense_kernel<float><<<grid_for(total), 256, 0, st>>>((float *)X, seed, row0, rows, d, ld);
  else
    synth_dense_kernel<double><<<grid_for(total), 256, 0, st>>>((double *)X, seed, row0, rows, d, ld);
  return cudaGetLastError();
}

cudaError_t synth_wtrue_launch(double *w, uint64_t seed, int32_t d, cudaStream_t st) {
  synth_wtrue_kernel<<<(d + 255) / 256, 256, 0, st>>>(w, seed, d);
  return cudaGetLastError();
}

cudaError_t synth_labels_launch(const void *X, int elem_bytes, const double *w_true, double *labels, uint64_t seed,
                                int kind, int64_t row0, int64_t rows, int32_t d, int32_t ld, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  const unsigned grid = grid_for(rows * 32);
  if (elem_bytes == 2)
    synth_labels_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16 *)X, w_true, labels, seed, kind, row0, rows, d, ld);
  else if (elem_bytes == 4)
    synth_labels_kernel<float><<<grid, 256, 0, st>>>((const float *)X, w_true, labels, seed, kind, row0, rows, d, ld);
  else
    synth_labels_kernel<double><<<grid, 256, 0, st>>>((const double *)X, w_true, labels, seed, kind, row0, rows, d, ld);
  return cudaGetLastError();
}

cudaError_t csr_shift_rowptr_launch(int64_t *dst, const int64_t *src, int64_t n, int64_t shift, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  csr_shift_rowptr_kernel<<<grid_for(n), 256, 0, st>>>((long long *)dst, (const long long *)src, n, shift);
  return cudaGetLastError();
}

cudaError_t csr_validate_launch(const int64_t *rowptr_host_order, int64_t rows, const int32_t *idx, int64_t nnz, int32_t d,
                                int *flag, cudaStream_t st) {
  csr_validate_kernel<<<grid_for(nnz > rows ? nnz : rows + 1), 256, 0, st>>>((const long long *)rowptr_host_order, rows, idx,
                                                                              nnz, d, flag);
  return cudaGetLastError();
}

cudaError_t synth_csr_launch(int64_t *rowptr, int32_t *idx, void *val, int elem_bytes, const double *w_true,
                             double *labels, uint64_t seed, int kind, int64_t row0, int64_t rows, int32_t d, int32_t k,
                             cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  const unsigned g1 = grid_for(rows * (long long)k), g2 = grid_for(rows * 32);
  if (elem_bytes == 4) {
    synth_csr_kernel<float><<<g1, 256, 0, st>>>((long long *)rowptr, idx, (float *)val, seed, row0, rows, d, k);
    synth_csr_labels_kernel<float><<<g2, 256, 0, st>>>((const long long *)rowptr, idx, (const float *)val, w_true, labels,
                                                       seed, kind, row0, rows);
  } else {
    synth_csr_kernel<double><<<g1, 256, 0, st>>>((long long *)rowptr, idx, (double *)val, seed, row0, rows, d, k);
    synth_csr_labels_kernel<double><<<g2, 256, 0, st>>>((const long long *)rowptr, idx, (const double *)val, w_true,
                                                        labels, seed, kind, row0, rows);
  }
  return cudaGetLastError();
}

cudaError_t convert_rows_launch(void *dst, int dst_bytes, const void *src, int src_bytes, int64_t rows, int32_t d,
                                int64_t ld, int32_t dst_ld, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  const unsigned grid = grid_for(rows * (long long)dst_ld);
  if (dst_bytes == 2 && src_bytes == 4)
    convert_rows_kernel<__nv_bfloat16, float><<<grid, 256, 0, st>>>((__nv_bfloat16 *)dst, (const float *)src, rows, d, ld, dst_ld);
  else if (dst_bytes == 2 && src_bytes == 8)
    convert_rows_kernel<__nv_bfloat16, double><<<grid, 256, 0, st>>>((__nv_bfloat16 *)dst, (const double *)src, rows, d, ld, dst_ld);
  else if (dst_bytes == 4 && src_bytes == 4)
    convert_rows_kernel<float, float><<<grid, 256, 0, st>>>((float *)dst, (const float *)src, rows, d, ld, dst_ld);
  else if (dst_bytes == 4 && src_bytes == 8)
    convert_rows_kernel<float, double><<<grid, 256, 0, st>>>((float *)dst, (const double *)src, rows, d, ld, dst_ld);
  else if (dst_bytes == 8 && src_bytes == 4)
    convert_rows_kernel<double, float><<<grid, 256, 0, st>>>((double *)dst, (const float *)src, rows, d, ld, dst_ld);
  else
    convert_rows_kernel<double, double><<<grid, 256, 0, st>>>((double *)dst, (const double *)src, rows, d, ld, dst_ld);
  return cudaGetLastError();
}

}  // namespace agd
