// kmeans.cu -- the kernels behind agd_kmeans_step / _assign / _costs / _sample (KMeans of mllib 1.3.0), sm_90a.
//
// Assignment.  Dense: the projection's row tile (pj_tile.cuh) computes x . B_j on the fp64 tensor cores with B = (s o C)^T; the
// epilogue turns each accumulator into the score ||c_j||^2 - 2 (acc + cb_j) and keeps, per row, the lexicographically smallest
// (score, j) with a NaN score taken as +inf: MLlib's findClosest scan (strict <, from +inf, lowest index on ties, a row no centre
// wins goes to 0), in an order-free form.  A k of more than one 128-column tile writes each tile's best to scratch and a second
// kernel merges the tiles.  CSR: one warp per row, lanes over centres.  The chosen centre depends only on the row and the centres.
// Residuals, sums and sampling run on the CUDA cores in fp64 (see agd_common.cuh for each form's order).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "k1_device.cuh"
#include "pj_tile.cuh"

namespace agd {

namespace {

constexpr int kKmWarpThreads = 256;     // warp-per-row kernels
constexpr int kKmCols = 128;            // columns per CTA of the dense sums
constexpr int kKmCsrCols = 4;           // centres per lane and pass of the CSR assignment
constexpr double kKmInf = __builtin_huge_val();

__device__ __forceinline__ bool km_in_view(const uint32_t *bits, long long r) {
  return !bits || ((bits[r >> 5] >> (r & 31)) & 1u);
}
// (s, j) replaces (bs, bj) iff it is lexicographically smaller; NaN scores arrive as +inf
__device__ __forceinline__ void km_take(double s, int j, double &bs, int &bj) {
  if (s < bs || (s == bs && j < bj)) { bs = s; bj = j; }
}
// kKmDistance: ||c_j||^2 - 2 (acc + cb_j); kKmLinear: -(offset_j + acc + cb_j), the offset in the cn slot (the argmax as an argmin)
template <int MODE> __device__ __forceinline__ double km_score(const KmeansArgs &a, int j, double acc) {
  const double s = MODE == kKmLinear ? -(a.cn[j] + acc + a.cb[j]) : a.cn[j] - 2.0 * (acc + a.cb[j]);
  return s != s ? kKmInf : s;
}
__device__ __forceinline__ void km_warp_min(double &bs, int &bj) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) km_take(__shfl_xor_sync(0xffffffffu, bs, off), __shfl_xor_sync(0xffffffffu, bj, off), bs, bj);
}
__device__ __forceinline__ double km_warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);   // every lane ends with the same bits
  return v;
}

// Feature c of dense row r in the k-means space: s_c x_c (fp64), 1.0 at c == d (the bias)
template <typename T> __device__ __forceinline__ double km_z(const KmeansArgs &a, long long r, int c) {
  if (c >= a.d) return 1.0;
  double x = GmElem<T>::wide(reinterpret_cast<const T *>(a.X)[(size_t)r * a.d + c]);
  if (a.scale) x *= a.scale[c];
  return x;
}

// Row tile rt0 + blockIdx.y (of the range), column tile blockIdx.x
template <typename T, bool VEC, int BN, int MODE>
__global__ void __launch_bounds__(kPjThreads, BN == 128 ? 1 : 2) kmeans_dense_kernel(const KmeansArgs a, const long long rt0) {
  using S = PjShape<BN>;
  extern __shared__ __align__(16) unsigned char pj_smem[];
  long long *orow = pj_orow<T, BN>(pj_smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long l0 = (rt0 + blockIdx.y) * kPjRows;
  const int c0 = (int)blockIdx.x * BN;
  if (tid < kPjRows) {
    const long long l = l0 + tid;
    orow[tid] = l < a.rows && km_in_view(a.view_bits, a.row0 + l) ? l : -1;
  }
  __syncthreads();
  double acc[S::MT][S::NT][4];
  pj_tile_mma<T, VEC, BN>(pj_smem, reinterpret_cast<const T *>(a.X), a.d, a.B, a.kp, a.row0 + l0, c0, acc);

  // the best (score, j) of each of this thread's rows over its columns, then over the 4 lanes that share the rows
  double bs[S::MT][2];
  int bj[S::MT][2];
#pragma unroll
  for (int mt = 0; mt < S::MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      bs[mt][h] = kKmInf;
      bj[mt][h] = 0x7fffffff;
#pragma unroll
      for (int nt = 0; nt < S::NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = c0 + pj_frag_col<BN>(nt, 2 * h + e);
          if (j < a.k) km_take(km_score<MODE>(a, j, acc[mt][nt][2 * h + e]), j, bs[mt][h], bj[mt][h]);
        }
#pragma unroll
      for (int off = 1; off < 4; off <<= 1)
        km_take(__shfl_xor_sync(0xffffffffu, bs[mt][h], off), __shfl_xor_sync(0xffffffffu, bj[mt][h], off), bs[mt][h], bj[mt][h]);
    }
  // ... then over the WN warps that share them, through the fp64 tiles (free once every warp is past its last MMA)
  __syncthreads();
  double *rs = pj_fp64_tiles<T, BN>(pj_smem);
  int *rj = reinterpret_cast<int *>(rs + S::WN * kPjRows);
  if ((lane & 3) == 0)
#pragma unroll
    for (int mt = 0; mt < S::MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = pj_frag_row<BN>(mt, 2 * h);
        rs[(warp % S::WN) * kPjRows + i] = bs[mt][h];
        rj[(warp % S::WN) * kPjRows + i] = bj[mt][h];
      }
  __syncthreads();
  if (tid < kPjRows && l0 + tid < a.rows) {
    double s = rs[tid];
    int j = rj[tid];
    for (int w = 1; w < S::WN; ++w) km_take(rs[w * kPjRows + tid], rj[w * kPjRows + tid], s, j);
    const long long l = l0 + tid;
    if (gridDim.x == 1) {
      a.cluster[l] = orow[tid] < 0 ? -1 : j;
    } else {
      a.tile_score[(size_t)blockIdx.x * a.rows + l] = s;
      a.tile_idx[(size_t)blockIdx.x * a.rows + l] = orow[tid] < 0 ? -1 : j;
    }
  }
}

// The column tiles' bests merged per row (any order gives the same (score, j))
__global__ void kmeans_tiles_kernel(const KmeansArgs a, int tiles) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= a.rows) return;
  double s = a.tile_score[l];
  int j = a.tile_idx[l];
  if (j >= 0)
    for (int t = 1; t < tiles; ++t) km_take(a.tile_score[(size_t)t * a.rows + l], a.tile_idx[(size_t)t * a.rows + l], s, j);
  a.cluster[l] = j;
}

// One warp per row of the range, lanes over centres in passes of 32 kKmCsrCols; every stored entry, in stored order, adds
// x B[col, :] in fp64
template <typename T, int MODE>
__global__ void __launch_bounds__(kKmWarpThreads) kmeans_csr_kernel(const KmeansArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kKmWarpThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kKmWarpThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  for (long long l = warp0; l < a.rows; l += nwarps) {
    const long long r = a.row0 + l;
    if (!km_in_view(a.view_bits, r)) {
      if (lane == 0) a.cluster[l] = -1;
      continue;
    }
    const long long k0 = __ldg(a.rowptr + r), k1 = __ldg(a.rowptr + r + 1);
    double bs = kKmInf;
    int bj = 0x7fffffff;
    for (int j0 = 0; j0 < a.k; j0 += 32 * kKmCsrCols) {
      double acc[kKmCsrCols];
#pragma unroll
      for (int q = 0; q < kKmCsrCols; ++q) acc[q] = 0.0;
      for (long long e = k0; e < k1; ++e) {
        const double x = (double)val[e];
        const double *b = a.B + (size_t)__ldg(a.idx + e) * a.kp;
#pragma unroll
        for (int q = 0; q < kKmCsrCols; ++q) {
          const int j = j0 + q * 32 + lane;
          if (j < a.k) acc[q] = fma(x, __ldg(b + j), acc[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < kKmCsrCols; ++q) {
        const int j = j0 + q * 32 + lane;
        if (j < a.k) km_take(km_score<MODE>(a, j, acc[q]), j, bs, bj);
      }
    }
    km_warp_min(bs, bj);
    if (lane == 0) a.cluster[l] = bj;
  }
}

// Exact residual of row r to centre j, the same bits on every lane of the warp
template <typename T> __device__ __forceinline__ double km_resid_dense(const KmeansArgs &a, long long r, int j, int lane) {
  const double *c = a.C + (size_t)j * a.md;
  double s = 0.0;
  for (int col = lane; col < a.md; col += 32) {
    const double e = km_z<T>(a, r, col) - c[col];
    s = fma(e, e, s);
  }
  return km_warp_sum(s);
}
template <typename T> __device__ __forceinline__ double km_resid_csr(const KmeansArgs &a, long long r, int j, int lane) {
  const double *c = a.C + (size_t)j * a.md;
  const T *val = reinterpret_cast<const T *>(a.val);
  const long long k0 = __ldg(a.rowptr + r), k1 = __ldg(a.rowptr + r + 1);
  double s = 0.0;
  for (long long e = k0 + lane; e < k1; e += 32) {
    const int col = __ldg(a.idx + e);
    double x = (double)val[e];
    if (a.scale) x *= a.scale[col];
    const double cc = c[col], dd = x - cc;
    s += dd * dd - cc * cc;
  }
  s = km_warp_sum(s);
  if (a.bias) {
    const double cc = c[a.d], dd = 1.0 - cc;
    s += dd * dd - cc * cc;
  }
  return a.cn[j] + s;
}
template <typename T> __device__ __forceinline__ double km_resid(const KmeansArgs &a, long long r, int j, int lane) {
  return a.rowptr ? km_resid_csr<T>(a, r, j, lane) : km_resid_dense<T>(a, r, j, lane);
}

template <typename T>
__global__ void __launch_bounds__(kKmWarpThreads) kmeans_dist_kernel(const KmeansArgs a, double *dist, double *delta, int keep,
                                                                      double *slabs) {
  __shared__ double part[kKmWarpThreads / 32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long warp0 = (long long)blockIdx.x * (kKmWarpThreads / 32) + wib;
  const long long nwarps = (long long)gridDim.x * (kKmWarpThreads / 32);
  double sum = 0.0;
  for (long long l = warp0; l < a.rows; l += nwarps) {
    const int j = a.cluster[l];
    if (j < 0) {
      if (dist && lane == 0) dist[l] = __longlong_as_double(0x7ff8000000000000ll);
      continue;
    }
    const double v = km_resid<T>(a, a.row0 + l, j, lane);
    if (lane != 0) continue;
    if (dist) {
      dist[l] = v;
    } else {
      const double n = keep && !(v < delta[l]) ? delta[l] : v;
      delta[l] = n;
      sum += n;
    }
  }
  if (dist) return;
  if (lane == 0) part[wib] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kKmWarpThreads / 32; ++w) s += part[w];
    slabs[blockIdx.x] = s;
  }
}

__global__ void kmeans_keys_kernel(const int32_t *__restrict__ cluster, long long rows, int32_t k, unsigned long long *keys,
                                   uint32_t *vals, unsigned long long *counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const int32_t c = cluster[i];
  const unsigned long long key = c < 0 ? (unsigned long long)k : (unsigned long long)c;
  keys[i] = key;
  vals[i] = (uint32_t)i;
  atomicAdd(counts + key, 1ull);
}

// Piece blockIdx.y, columns blockIdx.x kKmCols + threadIdx.x.  kKmResidual: pres = sum (z - c)^2; kKmNegatives: pres = the
// entries that are not >= 0 (NaN included), and C is not read
template <typename T, int MODE>
__global__ void __launch_bounds__(kKmCols) kmeans_sums_dense_kernel(const KmeansArgs a, const uint32_t *__restrict__ order,
                                                                    const long long *__restrict__ pstart,
                                                                    const int32_t *__restrict__ pcl, double *part, double *pres) {
  __shared__ uint32_t rows[kKmCols];
  const long long p = blockIdx.y;
  const int col = blockIdx.x * kKmCols + threadIdx.x;
  const long long q0 = pstart[p], q1 = pstart[p + 1];
  const double c = MODE == kKmResidual && col < a.md ? a.C[(size_t)pcl[p] * a.md + col] : 0.0;
  double s = 0.0, e2 = 0.0;
  for (long long b = q0; b < q1; b += kKmCols) {
    const int n = q1 - b < kKmCols ? (int)(q1 - b) : kKmCols;
    __syncthreads();
    if (threadIdx.x < n) rows[threadIdx.x] = order[b + threadIdx.x];
    __syncthreads();
    if (col < a.md) {
#pragma unroll 8
      for (int i = 0; i < n; ++i) {
        const double z = km_z<T>(a, a.row0 + rows[i], col);
        s += z;
        if (MODE == kKmNegatives) {
          e2 += z >= 0.0 ? 0.0 : 1.0;
        } else {
          const double e = z - c;
          e2 = fma(e, e, e2);
        }
      }
    }
  }
  if (col < a.md) {
    part[(size_t)p * a.md + col] = s;
    pres[(size_t)p * a.md + col] = e2;
  }
}

// threads over k md sums, then md column residuals (a second kernel adds the columns)
__global__ void kmeans_sums_reduce_kernel(const double *__restrict__ part, const double *__restrict__ pres,
                                          const int32_t *__restrict__ pfirst, long long npieces, int32_t k, int32_t md,
                                          double *out, double *colres) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nsum = (long long)k * md;
  if (t < nsum) {
    const int j = (int)(t / md), c = (int)(t % md);
    double s = 0.0;
    for (int p = pfirst[j]; p < pfirst[j + 1]; ++p) s += part[(size_t)p * md + c];
    out[t] = s;
  } else if (t < nsum + md) {
    const int c = (int)(t - nsum);
    double s = 0.0;
    for (long long p = 0; p < npieces; ++p) s += pres[(size_t)p * md + c];
    colres[c] = s;
  }
}
__global__ void kmeans_cost_kernel(const double *colres, int32_t k, int32_t md, double *out) {
  double s = 0.0;
  for (int c = 0; c < md; ++c) s += colres[c];
  out[(size_t)k * md + k] = s;
}

// kKmResidual: out[k md + k] += each row's residual; kKmNegatives: += the stored entries that are not >= 0 (NaN included)
template <typename T, int MODE>
__global__ void __launch_bounds__(kKmWarpThreads) kmeans_sums_csr_kernel(const KmeansArgs a, double *out) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kKmWarpThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kKmWarpThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  for (long long l = warp0; l < a.rows; l += nwarps) {
    const int j = a.cluster[l];
    if (j < 0) continue;
    const long long r = a.row0 + l;
    const long long k0 = __ldg(a.rowptr + r), k1 = __ldg(a.rowptr + r + 1);
    double *sj = out + (size_t)j * a.md;
    double neg = 0.0;
    for (long long e = k0 + lane; e < k1; e += 32) {
      const int col = __ldg(a.idx + e);
      double x = (double)val[e];
      if (a.scale) x *= a.scale[col];
      atomicAdd(sj + col, x);
      if (MODE == kKmNegatives) neg += x >= 0.0 ? 0.0 : 1.0;
    }
    const double v = MODE == kKmNegatives ? km_warp_sum(neg) : km_resid_csr<T>(a, r, j, lane);
    if (lane == 0) {
      if (a.bias) atomicAdd(sj + a.d, 1.0);
      atomicAdd(out + (size_t)a.k * a.md + a.k, v);
    }
  }
}

__global__ void kmeans_counts_kernel(const unsigned long long *counts, int32_t k, int32_t md, double *out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < k) out[(size_t)k * md + j] = (double)counts[j];
}

__device__ __forceinline__ double km_unit(unsigned long long u) { return (double)(u >> 11) * 0x1.0p-53; }

// one thread per row, a warp per bitmap word
__global__ void kmeans_sample_bits_kernel(const KmeansArgs a, unsigned long long seed, long long row_base, double factor,
                                          const double *delta, uint32_t *bits) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  if (l < a.rows && km_in_view(a.view_bits, l)) {
    const double u = km_unit(row_draw(seed, row_base + l, kKmStream));
    keep = u < (delta ? factor * delta[l] : factor);
  }
  const uint32_t w = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && l < a.rows) bits[l >> 5] = w;
}

template <typename T, bool CSR>
__global__ void __launch_bounds__(kKmWarpThreads) kmeans_sample_rows_kernel(const KmeansArgs a, unsigned long long seed,
                                                                             long long row_base, const uint32_t *bits,
                                                                             const long long *tile_base, double *out) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kKmWarpThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kKmWarpThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  for (long long l = warp0; l < a.rows; l += nwarps) {
    const long long o = view_rank(bits, tile_base, l);
    if (o < 0) continue;
    double *z = out + (size_t)o * (a.md + 1);
    if (CSR) {
      for (int c = lane; c < a.md; c += 32) z[c] = c < a.d ? 0.0 : 1.0;
      __syncwarp();
      if (lane == 0)   // stored order: a repeated column adds up
        for (long long e = a.rowptr[l]; e < a.rowptr[l + 1]; ++e) {
          const int col = a.idx[e];
          double x = (double)val[e];
          if (a.scale) x *= a.scale[col];
          z[col] += x;
        }
    } else {
      for (int c = lane; c < a.md; c += 32) z[c] = km_z<T>(a, l, c);
    }
    if (lane == 0) z[a.md] = km_unit(row_draw(seed, row_base + l, kKmStream));
  }
}

template <typename T, bool VEC, int BN, int MODE>
cudaError_t launch_dense(const KmeansArgs &a) {
  return pj_launch_rows<T, BN>(kmeans_dense_kernel<T, VEC, BN, MODE>, a, a.rows, a.kp / BN, a.stream);
}
template <typename T, int BN, int MODE>
cudaError_t launch_dense_vec(const KmeansArgs &a) {
  if ((size_t)a.d * sizeof(T) % 16 == 0) return launch_dense<T, true, BN, MODE>(a);
  return launch_dense<T, false, BN, MODE>(a);
}
template <typename T, int MODE>
cudaError_t launch_dense_t(const KmeansArgs &a) {
  cudaError_t e;
  switch (project_tile_cols(a.k)) {
    case 16: e = launch_dense_vec<T, 16, MODE>(a); break;
    case 32: e = launch_dense_vec<T, 32, MODE>(a); break;
    case 64: e = launch_dense_vec<T, 64, MODE>(a); break;
    default: e = launch_dense_vec<T, 128, MODE>(a); break;
  }
  if (e != cudaSuccess || a.kp <= 128) return e;
  kmeans_tiles_kernel<<<(unsigned)((a.rows + 255) / 256), 256, 0, a.stream>>>(a, a.kp / 128);
  return cudaGetLastError();
}

template <typename Kern> cudaError_t warp_grid(Kern kern, long long rows, int sm_count, unsigned *grid) {
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kKmWarpThreads, 0);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  long long g = (long long)per_sm * sm_count;
  const long long need = (rows + kKmWarpThreads / 32 - 1) / (kKmWarpThreads / 32);
  if (g > need) g = need;
  *grid = (unsigned)(g > 0 ? g : 1);
  return cudaSuccess;
}

template <int MODE>
cudaError_t assign_launch(const KmeansArgs &a, int elem_bytes, int sm_count) {
  if (a.rows <= 0) return cudaSuccess;
  if (a.rowptr) {
    if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
    auto kern = elem_bytes == 8 ? kmeans_csr_kernel<double, MODE> : kmeans_csr_kernel<float, MODE>;
    unsigned grid = 0;
    cudaError_t e = warp_grid(kern, a.rows, sm_count, &grid);
    if (e != cudaSuccess) return e;
    kern<<<grid, kKmWarpThreads, 0, a.stream>>>(a);
    return cudaGetLastError();
  }
  if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16, MODE>(a);
  if (elem_bytes == 4) return launch_dense_t<float, MODE>(a);
  if (elem_bytes == 8) return launch_dense_t<double, MODE>(a);
  return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t kmeans_assign_launch(const KmeansArgs &a, int elem_bytes, int sm_count, int score_mode) {
  if (score_mode == kKmLinear) return assign_launch<kKmLinear>(a, elem_bytes, sm_count);
  if (score_mode == kKmDistance) return assign_launch<kKmDistance>(a, elem_bytes, sm_count);
  return cudaErrorInvalidValue;
}

// The delta form's grid is fixed by the device alone, so its per-block sums, added in order, repeat bit for bit
int kmeans_dist_blocks(int sm_count) { return 4 * sm_count; }

cudaError_t kmeans_dist_launch(const KmeansArgs &a, int elem_bytes, int sm_count, double *dist, double *delta, int keep,
                               double *slabs, int *blocks_out) {
  *blocks_out = 0;
  if (a.rows <= 0) return cudaSuccess;
  const unsigned grid = (unsigned)kmeans_dist_blocks(sm_count);
  switch (elem_bytes) {
    case 2: kmeans_dist_kernel<__nv_bfloat16><<<grid, kKmWarpThreads, 0, a.stream>>>(a, dist, delta, keep, slabs); break;
    case 4: kmeans_dist_kernel<float><<<grid, kKmWarpThreads, 0, a.stream>>>(a, dist, delta, keep, slabs); break;
    case 8: kmeans_dist_kernel<double><<<grid, kKmWarpThreads, 0, a.stream>>>(a, dist, delta, keep, slabs); break;
    default: return cudaErrorInvalidValue;
  }
  *blocks_out = (int)grid;
  return cudaGetLastError();
}

cudaError_t kmeans_keys_launch(const int32_t *cluster, long long rows, int32_t k, unsigned long long *keys, uint32_t *vals,
                               unsigned long long *counts, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  kmeans_keys_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(cluster, rows, k, keys, vals, counts);
  return cudaGetLastError();
}

cudaError_t kmeans_sums_dense_launch(const KmeansArgs &a, int elem_bytes, const uint32_t *order, const long long *pstart,
                                     const int32_t *pcl, long long npieces, double *part, double *pres, int sums_mode) {
  if (npieces <= 0) return cudaSuccess;
  if (sums_mode != kKmResidual && sums_mode != kKmNegatives) return cudaErrorInvalidValue;
  const bool neg = sums_mode == kKmNegatives;
  const unsigned cx = (unsigned)((a.md + kKmCols - 1) / kKmCols);
  for (long long p0 = 0; p0 < npieces; p0 += kPjMaxGridY) {
    const long long n = npieces - p0 < kPjMaxGridY ? npieces - p0 : kPjMaxGridY;
    const dim3 g(cx, (unsigned)n);
    const long long *ps = pstart + p0;
    const int32_t *pc = pcl + p0;
    double *pa = part + (size_t)p0 * a.md, *pr = pres + (size_t)p0 * a.md;
    switch (elem_bytes) {
      case 2: (neg ? kmeans_sums_dense_kernel<__nv_bfloat16, kKmNegatives> : kmeans_sums_dense_kernel<__nv_bfloat16, kKmResidual>)
                  <<<g, kKmCols, 0, a.stream>>>(a, order, ps, pc, pa, pr); break;
      case 4: (neg ? kmeans_sums_dense_kernel<float, kKmNegatives> : kmeans_sums_dense_kernel<float, kKmResidual>)
                  <<<g, kKmCols, 0, a.stream>>>(a, order, ps, pc, pa, pr); break;
      case 8: (neg ? kmeans_sums_dense_kernel<double, kKmNegatives> : kmeans_sums_dense_kernel<double, kKmResidual>)
                  <<<g, kKmCols, 0, a.stream>>>(a, order, ps, pc, pa, pr); break;
      default: return cudaErrorInvalidValue;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t kmeans_sums_reduce_launch(const double *part, const double *pres, const int32_t *pfirst, long long npieces,
                                      int32_t k, int32_t md, double *out, double *colres, cudaStream_t st) {
  const long long n = (long long)k * md + md;
  kmeans_sums_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, pres, pfirst, npieces, k, md, out, colres);
  kmeans_cost_kernel<<<1, 1, 0, st>>>(colres, k, md, out);
  return cudaGetLastError();
}

cudaError_t kmeans_sums_csr_launch(const KmeansArgs &a, int elem_bytes, int sm_count, double *out, int sums_mode) {
  if (a.rows <= 0) return cudaSuccess;
  if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
  if (sums_mode != kKmResidual && sums_mode != kKmNegatives) return cudaErrorInvalidValue;
  auto kern = sums_mode == kKmNegatives
                  ? (elem_bytes == 8 ? kmeans_sums_csr_kernel<double, kKmNegatives> : kmeans_sums_csr_kernel<float, kKmNegatives>)
                  : (elem_bytes == 8 ? kmeans_sums_csr_kernel<double, kKmResidual> : kmeans_sums_csr_kernel<float, kKmResidual>);
  unsigned grid = 0;
  cudaError_t e = warp_grid(kern, a.rows, sm_count, &grid);
  if (e != cudaSuccess) return e;
  kern<<<grid, kKmWarpThreads, 0, a.stream>>>(a, out);
  return cudaGetLastError();
}

cudaError_t kmeans_counts_launch(const unsigned long long *counts, int32_t k, int32_t md, double *out, cudaStream_t st) {
  kmeans_counts_kernel<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(counts, k, md, out);
  return cudaGetLastError();
}

cudaError_t kmeans_sample_bits_launch(const KmeansArgs &a, unsigned long long seed, long long row_base, double factor,
                                      const double *delta, uint32_t *bits) {
  if (a.rows <= 0) return cudaSuccess;
  kmeans_sample_bits_kernel<<<(unsigned)((a.rows + 255) / 256), 256, 0, a.stream>>>(a, seed, row_base, factor, delta, bits);
  return cudaGetLastError();
}

cudaError_t kmeans_sample_rows_launch(const KmeansArgs &a, int elem_bytes, unsigned long long seed, long long row_base,
                                      const uint32_t *bits, const long long *tile_base, double *out, int sm_count) {
  if (a.rows <= 0) return cudaSuccess;
  auto run = [&](auto kern) {
    unsigned grid = 0;
    cudaError_t e = warp_grid(kern, a.rows, sm_count, &grid);
    if (e != cudaSuccess) return e;
    kern<<<grid, kKmWarpThreads, 0, a.stream>>>(a, seed, row_base, bits, tile_base, out);
    return cudaGetLastError();
  };
  if (a.rowptr) {
    if (elem_bytes == 4) return run(kmeans_sample_rows_kernel<float, true>);
    if (elem_bytes == 8) return run(kmeans_sample_rows_kernel<double, true>);
    return cudaErrorInvalidValue;
  }
  if (elem_bytes == 2) return run(kmeans_sample_rows_kernel<__nv_bfloat16, false>);
  if (elem_bytes == 4) return run(kmeans_sample_rows_kernel<float, false>);
  if (elem_bytes == 8) return run(kmeans_sample_rows_kernel<double, false>);
  return cudaErrorInvalidValue;
}

}  // namespace agd
