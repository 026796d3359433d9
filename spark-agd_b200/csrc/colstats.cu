// colstats.cu -- column statistics of a resident shard (sm_90a): the sweeps behind agd_col_stats
// (Statistics.colStats / MultivariateOnlineSummarizer of mllib 1.3.0).
//
// Two passes over X, each streaming the shard once:
//   * pass 1, per column: sum x, sum x^2, sum |x|, the nonzero count, max and min (and on CSR the stored-entry count), plus
//     the row count of the view;
//   * pass 2, per column: sum (x - mu) and sum (x - mu)^2 with mu = fl(sum x / count) read from pass 1's exchanged sums on
//     the device (no host round trip).  The host derives var = (sum (x-mu)^2 - (sum (x-mu))^2 / n) / (n - 1).
// Dense: a CTA owns a tile of up to 256 16-byte column vectors (or scalar columns) over a contiguous chunk of rows; a thread
// owns the columns of its vector and streams its rows with 128-bit (bf16: 64-bit) streaming loads, several rows in flight.  Compare,
// max / min and the nonzero test run in the storage type (exact); each element is widened to fp64 once for the sums.  The
// CTA adds its row lanes in a fixed order into one slab per CTA; k1_reduce_launch adds the sum slabs and
// colstats_max_reduce the max slabs, both in a fixed order, so dense results are bit-reproducible.
// CSR: one pass over the stored entries, sums scattered with fp64 RED.ADD (reproducible to rounding, as K1's CSR form);
// max / min by atomicMax on the order-preserving 64-bit image of the double (exact); counts exact.
// min travels as max(-x) everywhere, so one NaN-ignoring max serves both (also across ranks, xchg.cu).
// A row outside the view (agd_set_row_filter) is never loaded, as in the evaluation form of score.cu.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

constexpr int kCsThreads = 256;
constexpr int kCsCsrGroup = 8;   // lanes per CSR row

// 16 (or 8) bytes of X, streamed: no L1 allocation, 256-byte L2 prefetch (the load of score.cu)
__device__ __forceinline__ uint4 cs_ld_stream(const uint4 *p) {
  uint4 v;
  asm("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
      : "l"(p));
  return v;
}
__device__ __forceinline__ uint2 cs_ld_stream(const uint2 *p) {
  uint2 v;
  asm("ld.global.nc.L1::no_allocate.L2::256B.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}

__device__ __forceinline__ double cs_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// C = the type compares and max / min run in: the storage type, or fp32 for bf16 (a bf16 is the upper half of an fp32,
// so the widening is exact and free).  A thread's vector is Raw: 16 bytes, or 8 (four columns) for bf16, whose six
// accumulators per column would not fit eight columns in the registers of two CTAs per SM.
template <typename T> struct CsElem;
template <> struct CsElem<float> {
  typedef float C;
  typedef uint4 Raw;
  static constexpr int EPV = 4;
  static constexpr int R = 8;   // rows in flight per thread
  __device__ static C one(const float *p) { return __ldg(p); }
  __device__ static void vec(const uint4 &r, C (&o)[4]) {
    o[0] = __uint_as_float(r.x); o[1] = __uint_as_float(r.y); o[2] = __uint_as_float(r.z); o[3] = __uint_as_float(r.w);
  }
  __device__ static C nan() { return __int_as_float(0x7fc00000); }
};
template <> struct CsElem<double> {
  typedef double C;
  typedef uint4 Raw;
  static constexpr int EPV = 2;
  static constexpr int R = 8;
  __device__ static C one(const double *p) { return __ldg(p); }
  __device__ static void vec(const uint4 &r, C (&o)[2]) {
    o[0] = __hiloint2double((int)r.y, (int)r.x);
    o[1] = __hiloint2double((int)r.w, (int)r.z);
  }
  __device__ static C nan() { return cs_nan(); }
};
template <> struct CsElem<__nv_bfloat16> {
  typedef float C;
  typedef uint2 Raw;
  static constexpr int EPV = 4;
  static constexpr int R = 8;
  __device__ static C one(const __nv_bfloat16 *p) {
    return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short *>(p)) << 16);
  }
  __device__ static void vec(const uint2 &r, C (&o)[4]) {
    o[0] = __uint_as_float(r.x << 16); o[1] = __uint_as_float(r.x & 0xffff0000u);
    o[2] = __uint_as_float(r.y << 16); o[3] = __uint_as_float(r.y & 0xffff0000u);
  }
  __device__ static C nan() { return __int_as_float(0x7fc00000); }
};

__device__ __forceinline__ float cs_max(float a, float b) { return fmaxf(a, b); }     // NaN-ignoring
__device__ __forceinline__ double cs_max(double a, double b) { return fmax(a, b); }
__device__ __forceinline__ float cs_min(float a, float b) { return fminf(a, b); }
__device__ __forceinline__ double cs_min(double a, double b) { return fmin(a, b); }

// One value of a thread's row lane -> the CTA's value for its column unit, adding (or max-ing) the row lanes 0, 1, ... in
// order through shared memory; every thread of the CTA takes part.  Returns the result on row lane 0.
template <bool MAX>
__device__ __forceinline__ double cs_lanes(double v, double *red, int TU, int RL) {
  if (RL == 1) return v;
  red[threadIdx.x] = v;
  __syncthreads();
  double t = v;
  if ((int)threadIdx.x < TU) {
    for (int j = 1; j < RL; ++j) {
      const double o = red[j * TU + threadIdx.x];
      t = MAX ? fmax(t, o) : t + o;
    }
  }
  __syncthreads();
  return t;
}

// PASS 1: sums [SUM | SQ | ABS | NNZ | COUNT] (n_sum = 4 d + 1 per slab), maxima [MAX | -MIN] (2 d per slab)
// PASS 2: sums [DEV | DEV2] (2 d per slab); mu from the world's pass-1 sums (ColStatsArgs::mu_sums)
template <typename T, bool VEC, int PASS>
__global__ void __launch_bounds__(kCsThreads, 2) colstats_dense_kernel(const ColStatsArgs a, const int TU, const long long chunk) {
  __shared__ double red[kCsThreads];
  typedef typename CsElem<T>::C C;
  constexpr int EPV = VEC ? CsElem<T>::EPV : 1;
  constexpr int R = CsElem<T>::R;
  const int RL = kCsThreads / TU;
  const int ul = threadIdx.x % TU, rl = threadIdx.x / TU;
  const int u = blockIdx.y * TU + ul;
  const int d = a.d;
  const int nunit = d / EPV;
  const bool active = u < nunit;
  const long long r0 = (long long)blockIdx.x * chunk;
  long long r1 = r0 + chunk;
  if (r1 > a.rows) r1 = a.rows;
  const T *X = reinterpret_cast<const T *>(a.X);

  double s[EPV], q[EPV], ab[EPV], mu[EPV];
  int nz[EPV];
  C mx[EPV], mn[EPV];
  double cnt = 0.0;
#pragma unroll
  for (int e = 0; e < EPV; ++e) {
    s[e] = 0.0; q[e] = 0.0; ab[e] = 0.0; nz[e] = 0;
    mx[e] = CsElem<T>::nan(); mn[e] = CsElem<T>::nan();
    mu[e] = 0.0;
  }
  if (PASS == 2 && active) {
    const double n = a.mu_sums[4 * (size_t)d];
#pragma unroll
    for (int e = 0; e < EPV; ++e) mu[e] = a.mu_sums[(size_t)u * EPV + e] / n;
  }
  for (long long base = r0 + rl; base < r1; base += (long long)RL * R) {
    bool ok[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long row = base + (long long)r * RL;
      ok[r] = row < r1 && row_in_view(a.filt, a.row_base + row);
      if (PASS == 1 && u == 0 && ok[r]) cnt += 1.0;
    }
    if (!active) continue;
    C xv[R][EPV];
    if (VEC) {
      typedef typename CsElem<T>::Raw Raw;
      Raw raw[R];
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (ok[r]) raw[r] = cs_ld_stream(reinterpret_cast<const Raw *>(X + (size_t)(base + (long long)r * RL) * d + (size_t)u * EPV));
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (ok[r]) {
          C t[CsElem<T>::EPV];
          CsElem<T>::vec(raw[r], t);
#pragma unroll
          for (int e = 0; e < EPV; ++e) xv[r][e] = t[e];
        }
    } else {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (ok[r]) xv[r][0] = CsElem<T>::one(X + (size_t)(base + (long long)r * RL) * d + u);
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (ok[r]) {
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          const C x = xv[r][e];
          const double xd = (double)x;
          if (PASS == 1) {
            s[e] += xd;
            q[e] = fma(xd, xd, q[e]);
            ab[e] += (double)fabs(x);
            nz[e] += x != (C)0 ? 1 : 0;   // a NaN is nonzero
            mx[e] = cs_max(mx[e], x);
            mn[e] = cs_min(mn[e], x);
          } else {
            const double dv = xd - mu[e];
            s[e] += dv;
            q[e] = fma(dv, dv, q[e]);
          }
        }
      }
  }
  // the CTA's row lanes in a fixed order -> one slab per CTA (columns of this CTA's tile only)
  const size_t n_sum = PASS == 1 ? 4 * (size_t)d + 1 : 2 * (size_t)d;
  double *slab = a.slabs + (size_t)blockIdx.x * n_sum;
  double *mslab = a.max_slabs + (size_t)blockIdx.x * 2 * (size_t)d;
  const bool w = active && rl == 0;
#pragma unroll
  for (int e = 0; e < EPV; ++e) {
    const size_t c = (size_t)u * EPV + e;
    double v;
    v = cs_lanes<false>(s[e], red, TU, RL);
    if (w) slab[c] = v;
    v = cs_lanes<false>(q[e], red, TU, RL);
    if (w) slab[d + c] = v;
    if (PASS == 1) {
      v = cs_lanes<false>(ab[e], red, TU, RL);
      if (w) slab[2 * (size_t)d + c] = v;
      v = cs_lanes<false>((double)nz[e], red, TU, RL);
      if (w) slab[3 * (size_t)d + c] = v;
      v = cs_lanes<true>((double)mx[e], red, TU, RL);
      if (w) mslab[c] = v;
      v = cs_lanes<true>(-(double)mn[e], red, TU, RL);
      if (w) mslab[d + c] = v;
    }
  }
  if (PASS == 1) {
    const double v = cs_lanes<false>(cnt, red, TU, RL);
    if (blockIdx.y == 0 && threadIdx.x == 0) slab[4 * (size_t)d] = v;
  }
}

// the order-preserving image of a double as an unsigned 64-bit integer (0 = below every value, decodes to NaN)
__device__ __forceinline__ unsigned long long cs_key(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double cs_unkey(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// PASS 1: out = [SUM | SQ | ABS | NNZ | COUNT | STORED] (5 d + 1, zeroed by the caller), keys [MAX | -MIN] (2 d, zeroed)
// PASS 2: out = [DEV | DEV2] over the stored entries (zeroed), mu from ColStatsArgs::mu; the implicit zeros are added in
// closed form by the host
template <typename T, int PASS>
__global__ void __launch_bounds__(kCsThreads) colstats_csr_kernel(const ColStatsArgs a) {
  __shared__ double red[kCsThreads / 32];
  constexpr int G = kCsCsrGroup, groups = 32 / G;
  const int lane = threadIdx.x & 31, g = lane / G, l = lane & (G - 1);
  const long long warp0 = (long long)blockIdx.x * (kCsThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kCsThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  const size_t d = (size_t)a.d;
  double *out = a.out;
  double cnt = 0.0;
  for (long long base = warp0 * groups; base < a.rows; base += nwarps * groups) {
    const long long row = base + g;
    if (row >= a.rows || !row_in_view(a.filt, a.row_base + row)) continue;
    if (l == 0) cnt += 1.0;
    const long long k0 = __ldg(a.rowptr + row), k1 = __ldg(a.rowptr + row + 1);
    for (long long k = k0 + l; k < k1; k += G) {
      const T x = val[k];
      const size_t c = (size_t)__ldg(a.idx + k);
      const double xd = (double)x;
      if (PASS == 1) {
        atomicAdd(out + c, xd);
        atomicAdd(out + d + c, xd * xd);
        atomicAdd(out + 2 * d + c, fabs(xd));
        if (x != (T)0) atomicAdd(out + 3 * d + c, 1.0);
        atomicAdd(out + 4 * d + 1 + c, 1.0);
        if (!isnan(xd)) {   // the current key is read first: most entries cannot raise it, and then issue no atomic
          const unsigned long long kx = cs_key(xd), kn = cs_key(-xd);
          if (kx > __ldcg(a.keys + c)) atomicMax(a.keys + c, kx);
          if (kn > __ldcg(a.keys + d + c)) atomicMax(a.keys + d + c, kn);
        }
      } else {
        const double dv = xd - a.mu[c];
        atomicAdd(out + c, dv);
        atomicAdd(out + d + c, dv * dv);
      }
    }
  }
  if (PASS == 1) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
    if (lane == 0) red[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int wi = 0; wi < kCsThreads / 32; ++wi) t += red[wi];
      atomicAdd(out + 4 * d, t);   // row counts are small integers: exact in any order
    }
  }
}

// mu[c] = fl(SUM[c] / COUNT) of the world's pass-1 sums (the CSR pass 2 reads it per stored entry)
__global__ void __launch_bounds__(256) colstats_mu_kernel(const double *sums, int d, double *mu) {
  const double n = sums[4 * (size_t)d];
  for (int c = blockIdx.x * 256 + threadIdx.x; c < d; c += gridDim.x * 256) mu[c] = sums[c] / n;
}

__global__ void __launch_bounds__(256) colstats_unkey_kernel(const unsigned long long *keys, int n, double *out) {
  for (int c = blockIdx.x * 256 + threadIdx.x; c < n; c += gridDim.x * 256) out[c] = cs_unkey(keys[c]);
}

// STORED of a dense shard: every row in the view stores every column, so STORED[c] = COUNT
__global__ void __launch_bounds__(256) colstats_fill_stored_kernel(double *sums, int d) {
  const double n = sums[4 * (size_t)d];
  for (int c = blockIdx.x * 256 + threadIdx.x; c < d; c += gridDim.x * 256) sums[4 * (size_t)d + 1 + c] = n;
}

// out[c] = NaN-ignoring max over the slabs of column c, in the fixed tree of k1_reduce_kernel (bit-reproducible)
__global__ void __launch_bounds__(256) colstats_max_reduce_kernel(const double *__restrict__ slabs, int blocks, int n,
                                                                  double *__restrict__ out) {
  __shared__ double part[8][33];
  const int cl = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double s0 = cs_nan(), s1 = cs_nan(), s2 = cs_nan(), s3 = cs_nan();
  if (c < n) {
    int b = grp;
    for (; b + 24 < blocks; b += 32) {
      s0 = fmax(s0, slabs[(size_t)b * n + c]); s1 = fmax(s1, slabs[(size_t)(b + 8) * n + c]);
      s2 = fmax(s2, slabs[(size_t)(b + 16) * n + c]); s3 = fmax(s3, slabs[(size_t)(b + 24) * n + c]);
    }
    for (; b < blocks; b += 8) s0 = fmax(s0, slabs[(size_t)b * n + c]);
  }
  part[grp][cl] = fmax(fmax(s0, s1), fmax(s2, s3));
  __syncthreads();
  if (grp == 0 && c < n) {
    double t = cs_nan();
#pragma unroll
    for (int gi = 0; gi < 8; ++gi) t = fmax(t, part[gi][cl]);
    out[c] = t;
  }
}

template <typename K>
cudaError_t cs_per_sm(K kern, int *per_sm) {
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kern, kCsThreads, 0);
  if (e != cudaSuccess) return e;
  return *per_sm < 1 ? cudaErrorInvalidConfiguration : cudaSuccess;
}

template <typename T, bool VEC, int PASS>
cudaError_t launch_dense(const ColStatsArgs &a, int sm_count, int max_blocks, int *blocks_out) {
  constexpr int EPV = VEC ? CsElem<T>::EPV : 1;
  const int nunit = a.d / EPV;
  int TU = 1;
  while (TU < nunit && TU < kCsThreads) TU <<= 1;
  const int RL = kCsThreads / TU;
  const int ytiles = (nunit + TU - 1) / TU;
  if (ytiles > 65535) return cudaErrorInvalidConfiguration;
  auto kern = colstats_dense_kernel<T, VEC, PASS>;
  int per_sm = 0;
  const cudaError_t e = cs_per_sm(kern, &per_sm);
  if (e != cudaSuccess) return e;
  long long gx = (long long)per_sm * sm_count / ytiles;
  if (gx < 1) gx = 1;
  if (gx > max_blocks) gx = max_blocks;
  const long long step = (long long)RL * CsElem<T>::R;   // rows one CTA covers per step
  const long long need = (a.rows + step - 1) / step;
  if (gx > need) gx = need;
  long long chunk = (a.rows + gx - 1) / gx;
  gx = (a.rows + chunk - 1) / chunk;   // every CTA gets rows
  *blocks_out = (int)gx;
  kern<<<dim3((unsigned)gx, (unsigned)ytiles), kCsThreads, 0, a.stream>>>(a, TU, chunk);
  return cudaGetLastError();
}

template <typename T, int PASS>
cudaError_t launch_dense_t(const ColStatsArgs &a, int sm_count, int max_blocks, int *blocks_out) {
  if (a.d % CsElem<T>::EPV == 0) return launch_dense<T, true, PASS>(a, sm_count, max_blocks, blocks_out);
  return launch_dense<T, false, PASS>(a, sm_count, max_blocks, blocks_out);
}

}  // namespace

int colstats_max_blocks(int sm_count, int32_t d) {
  int b = 2 * sm_count;
  const long long lim = (32LL << 20) / (6LL * d + 1);   // slab memory bounded as K1's generic form bounds it
  if (lim < b) b = lim < 1 ? 1 : (int)lim;
  return b;
}

cudaError_t colstats_dense_launch(const ColStatsArgs &a, int pass, int elem_bytes, int sm_count, int *blocks_out) {
  *blocks_out = 0;
  if (a.rows <= 0) return cudaSuccess;
  const int mb = colstats_max_blocks(sm_count, a.d);
  if (pass == 1) {
    if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16, 1>(a, sm_count, mb, blocks_out);
    if (elem_bytes == 4) return launch_dense_t<float, 1>(a, sm_count, mb, blocks_out);
    if (elem_bytes == 8) return launch_dense_t<double, 1>(a, sm_count, mb, blocks_out);
  } else {
    if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16, 2>(a, sm_count, mb, blocks_out);
    if (elem_bytes == 4) return launch_dense_t<float, 2>(a, sm_count, mb, blocks_out);
    if (elem_bytes == 8) return launch_dense_t<double, 2>(a, sm_count, mb, blocks_out);
  }
  return cudaErrorInvalidValue;
}

cudaError_t colstats_csr_launch(const ColStatsArgs &a, int pass, int elem_bytes, int sm_count) {
  if (a.rows <= 0) return cudaSuccess;
  if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
  auto kern = pass == 1 ? (elem_bytes == 8 ? colstats_csr_kernel<double, 1> : colstats_csr_kernel<float, 1>)
                        : (elem_bytes == 8 ? colstats_csr_kernel<double, 2> : colstats_csr_kernel<float, 2>);
  int per_sm = 0;
  const cudaError_t e = cs_per_sm(kern, &per_sm);
  if (e != cudaSuccess) return e;
  long long grid = (long long)per_sm * sm_count;
  const long long rows_per_cta = (long long)(kCsThreads / 32) * (32 / kCsCsrGroup);
  const long long need = (a.rows + rows_per_cta - 1) / rows_per_cta;
  if (grid > need) grid = need;
  kern<<<(unsigned)grid, kCsThreads, 0, a.stream>>>(a);
  return cudaGetLastError();
}

cudaError_t colstats_unkey_launch(const unsigned long long *keys, int n, double *out, cudaStream_t st) {
  int grid = (n + 255) / 256;
  if (grid > 1024) grid = 1024;
  if (grid < 1) grid = 1;
  colstats_unkey_kernel<<<grid, 256, 0, st>>>(keys, n, out);
  return cudaGetLastError();
}

cudaError_t colstats_mu_launch(const double *sums, int32_t d, double *mu, cudaStream_t st) {
  int grid = (d + 255) / 256;
  if (grid > 1024) grid = 1024;
  colstats_mu_kernel<<<grid, 256, 0, st>>>(sums, d, mu);
  return cudaGetLastError();
}

cudaError_t colstats_fill_stored_launch(double *sums, int32_t d, cudaStream_t st) {
  int grid = (d + 255) / 256;
  if (grid > 1024) grid = 1024;
  colstats_fill_stored_kernel<<<grid, 256, 0, st>>>(sums, d);
  return cudaGetLastError();
}

cudaError_t colstats_max_reduce_launch(const double *slabs, int blocks, int32_t n, double *out, cudaStream_t st) {
  const int grid = (n + 31) / 32;
  colstats_max_reduce_kernel<<<grid, 256, 0, st>>>(slabs, blocks, n, out);
  return cudaGetLastError();
}

}  // namespace agd
