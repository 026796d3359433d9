// gramian.cu -- cross-products of a resident shard (sm_90a): the sweeps behind agd_gramian (RowMatrix.computeGramianMatrix /
// computeCovariance of mllib 1.3.0).
//
// The result of one shard is the packed upper triangle of the augmented (d + 1) x (d + 1) matrix
//   [ sum z z^T   sum z ]
//   [ sum z^T     count ]      z = x (uncentered) or x - mu (centered, mu = fl(sum x / count) of the world)
// entry (i, j), i <= j, at gm_packed(i, j, d + 1).
// Dense: an SYRK over the upper block triangle on the fp64 tensor cores (mma.sync m16n8k4 .f64, DMMA).  A CTA owns one pair of
// 128-column blocks I <= J over a contiguous chunk of rows (one row split); the grid is block pairs x row splits.  Rows come
// through a ring of storage-type tiles (cp.async, 16-byte copies; rows whose stride is not a multiple of 16 bytes use plain
// loads), are widened to fp64 and centered once per element into an fp64 tile, and a row outside the view or past the chunk is
// SELECTED to 0 there (never multiplied by a mask: 0 x NaN = NaN), so it leaves no trace.  A diagonal pair (I == J) loads its
// columns once and also sums z of its columns and counts the rows.  Each row split writes one slab of the packed triangle, every
// entry exactly once; k1_reduce_launch adds the slabs in a fixed order, so dense results are bit-reproducible.
// CSR: one warp per row of the view scatters the products of the row's stored-entry pairs with fp64 RED.ADD (reproducible to
// rounding, as colstats_csr_kernel); centered sums are derived from the uncentered ones of the shard (gm_center_kernel).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "dmma.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

constexpr int kGmBlk = 128;        // output block width (columns of X per block)
constexpr int kGmThreads = 256;    // 8 warps, 2 (rows) x 4 (columns) warp tiles of 64 x 32
constexpr int kGmKc = 16;          // rows of X per stage
constexpr int kGmStages = 3;       // ring depth
constexpr int kGmLdz = kGmBlk + 4; // fp64 tile row stride: the fragment reads of a half-warp hit 16 distinct 8-byte banks
constexpr int kGmCsrThreads = 256;

__host__ __device__ inline long long gm_packed(long long i, long long j, long long n) { return i * n - i * (i - 1) / 2 + (j - i); }

// Smem (dynamic): raw ring [kGmStages][2 blocks][kGmKc][kGmBlk] storage elements | z tiles [2 buffers][2 blocks][kGmKc][kGmLdz]
// fp64 | row flags [kGmStages][kGmKc]
template <typename T>
__host__ __device__ constexpr size_t gm_smem_bytes() {
  return (size_t)kGmStages * 2 * kGmKc * kGmBlk * sizeof(T) + 4 * (size_t)kGmKc * kGmLdz * sizeof(double) +
         (size_t)kGmStages * kGmKc * sizeof(int);
}

// VEC: rows are whole 16-byte vectors (d * sizeof(T) % 16 == 0), staged with cp.async; else plain loads.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kGmThreads, 1) gramian_dense_kernel(const GramianArgs a, const long long chunk) {
  extern __shared__ __align__(16) unsigned char gm_smem[];
  T *raw = reinterpret_cast<T *>(gm_smem);
  double *zt = reinterpret_cast<double *>(gm_smem + (size_t)kGmStages * 2 * kGmKc * kGmBlk * sizeof(T));
  int *okf = reinterpret_cast<int *>(zt + 4 * kGmKc * kGmLdz);

  const int d = a.d, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long n1 = (long long)d + 1;
  // block pair of this CTA: the p-th of the upper block triangle, row-major
  const int nb = (d + kGmBlk - 1) / kGmBlk;
  int I = 0, p = blockIdx.x;
  while (p >= nb - I) { p -= nb - I; ++I; }
  const int J = I + p;
  const bool diag = I == J;
  const int nblk = diag ? 1 : 2;
  const int cI = I * kGmBlk, cJ = J * kGmBlk;
  const long long r0 = (long long)blockIdx.y * chunk;
  long long r1 = r0 + chunk;
  if (r1 > a.rows) r1 = a.rows;
  const long long nchunks = r1 > r0 ? (r1 - r0 + kGmKc - 1) / kGmKc : 0;
  const T *X = reinterpret_cast<const T *>(a.X);

  // stage s <- rows [r0 + k kGmKc, + kGmKc) of the CTA's column blocks; a row outside the view or past the chunk is not read
  auto issue = [&](long long k) {
    if (k >= nchunks) return;
    const int s = (int)(k % kGmStages);
    const long long rb = r0 + k * kGmKc;
    if (tid < kGmKc) {
      const long long row = rb + tid;
      bool ok = row < r1;
      if (ok && a.view_bits) ok = (a.view_bits[row >> 5] >> (row & 31)) & 1u;
      okf[s * kGmKc + tid] = ok ? 1 : 0;
    }
    T *dst = raw + (size_t)s * 2 * kGmKc * kGmBlk;
    if (VEC) {
      constexpr int EPV = 16 / sizeof(T), UPR = kGmBlk / EPV;   // 16-byte units per block row
      for (int u = tid; u < nblk * kGmKc * UPR; u += kGmThreads) {
        const int b = u / (kGmKc * UPR), r = (u / UPR) % kGmKc, cu = u % UPR;
        const long long row = rb + r;
        const int col = (b ? cJ : cI) + cu * EPV;
        bool ok = row < r1 && col < d;
        if (ok && a.view_bits) ok = (a.view_bits[row >> 5] >> (row & 31)) & 1u;
        const T *src = ok ? X + (size_t)row * d + col : X;
        const uint32_t sa = (uint32_t)__cvta_generic_to_shared(dst + ((size_t)b * kGmKc + r) * kGmBlk + cu * EPV);
        gm_cp16(sa, src, ok ? 16 : 0);
      }
    } else {
      for (int e = tid; e < nblk * kGmKc * kGmBlk; e += kGmThreads) {
        const int b = e / (kGmKc * kGmBlk), r = (e / kGmBlk) % kGmKc, c = e % kGmBlk;
        const long long row = rb + r;
        const int col = (b ? cJ : cI) + c;
        bool ok = row < r1 && col < d;
        if (ok && a.view_bits) ok = (a.view_bits[row >> 5] >> (row & 31)) & 1u;
        T v;
        if (ok) v = X[(size_t)row * d + col];
        else memset(&v, 0, sizeof v);
        dst[((size_t)b * kGmKc + r) * kGmBlk + c] = v;
      }
    }
  };

  // this thread's conversion column (t % kGmBlk) of each block and its mu
  const int cc = tid % kGmBlk, rh = tid / kGmBlk;   // rows rh, rh + 2, ...
  double muI = 0.0, muJ = 0.0;
  if (a.mu) {
    if (cI + cc < d) muI = a.mu[cI + cc];
    if (cJ + cc < d) muJ = a.mu[cJ + cc];
  }
  double zsum = 0.0, cnt = 0.0;   // diagonal pairs: sum z of column cI + cc over this thread's rows, and their count

  double acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.0;
  const int wm = warp >> 2, wn = warp & 3;

  // chunk k of the ring -> z tile buffer zb: widened, centered, and 0 for a row outside the view or past the chunk
  auto convert = [&](long long k, int zb) {
    const int s = (int)(k % kGmStages);
    const T *src = raw + (size_t)s * 2 * kGmKc * kGmBlk;
    const int *ok = okf + s * kGmKc;
    double *z0 = zt + (size_t)zb * 2 * kGmKc * kGmLdz;
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      if (b == nblk) break;
#pragma unroll
      for (int r = rh; r < kGmKc; r += kGmThreads / kGmBlk) {
        const bool keep = ok[r] != 0;
        const double z = keep ? GmElem<T>::wide(src[((size_t)b * kGmKc + r) * kGmBlk + cc]) - (b ? muJ : muI) : 0.0;
        z0[((size_t)b * kGmKc + r) * kGmLdz + cc] = z;
        if (b == 0) {
          zsum += z;
          cnt += keep ? 1.0 : 0.0;
        }
      }
    }
  };

  // kGmStages chunks in flight; the z tiles are double-buffered, so the conversion of chunk k + 1 overlaps the MMAs of chunk k
  // and one barrier per chunk orders both
  for (int k = 0; k < kGmStages; ++k) {
    issue(k);
    if (VEC) gm_commit();
  }
  if (nchunks > 0) {
    if (VEC) gm_wait<kGmStages - 1>();
    __syncthreads();
    convert(0, 0);
  }
  for (long long k = 0; k < nchunks; ++k) {
    if (VEC) gm_wait<kGmStages - 2>();
    __syncthreads();   // chunk k + 1 landed and chunk k is converted, for every thread; the MMAs of chunk k - 1 are done
    issue(k + kGmStages);   // into the ring stage chunk k was converted from
    if (VEC) gm_commit();
    const int zb = (int)(k & 1);
    const double *As = zt + (size_t)zb * 2 * kGmKc * kGmLdz, *Bs = diag ? As : As + kGmKc * kGmLdz;
#pragma unroll
    for (int ks = 0; ks < kGmKc / 4; ++ks) {
      const int kr = ks * 4 + (lane & 3);
      double af[4][2], bf[4];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        af[mt][0] = As[kr * kGmLdz + wm * 64 + mt * 16 + (lane >> 2)];
        af[mt][1] = As[kr * kGmLdz + wm * 64 + mt * 16 + 8 + (lane >> 2)];
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) bf[nt] = Bs[kr * kGmLdz + wn * 32 + nt * 8 + (lane >> 2)];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) gm_dmma(acc[mt][nt], af[mt], bf[nt]);
    }
    if (k + 1 < nchunks) convert(k + 1, zb ^ 1);
  }

  // this row split's slab: every upper entry of the pair, once
  double *slab = a.slabs + (size_t)blockIdx.y * (size_t)(gm_packed(d, d, n1) + 1);
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = cI + wm * 64 + mt * 16 + (lane >> 2) + (q >> 1) * 8;
        const int j = cJ + wn * 32 + nt * 8 + (lane & 3) * 2 + (q & 1);
        if (i <= j && j < d) slab[gm_packed(i, j, n1)] = acc[mt][nt][q];
      }
  if (diag) {
    // the two row halves of each column in a fixed order (reuses the z tiles: every MMA is done after this barrier)
    __syncthreads();
    double *red = zt;
    red[tid] = zsum;
    red[kGmThreads + tid] = cnt;
    __syncthreads();
    if (rh == 0) {
      const int c = cI + cc;
      if (c < d) slab[gm_packed(c, d, n1)] = red[tid] + red[tid + kGmBlk];
      if (I == 0 && cc == 0) slab[gm_packed(d, d, n1)] = red[kGmThreads + tid] + red[kGmThreads + tid + kGmBlk];
    }
  }
}

// CSR: out (zeroed) += the packed augmented sums of the view's rows, uncentered.  Two stored entries of one row with the same
// column add up, as every other kernel reads them: their pair adds 2 x_a x_b to the diagonal.
template <typename T>
__global__ void __launch_bounds__(kGmCsrThreads) gramian_csr_kernel(const GramianArgs a) {
  __shared__ double red[kGmCsrThreads / 32];
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kGmCsrThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kGmCsrThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  const long long n1 = (long long)a.d + 1;
  double *out = a.out;
  double cnt = 0.0;
  for (long long row = warp0; row < a.rows; row += nwarps) {
    if (!row_in_view(a.filt, a.row_base + row)) continue;
    if (lane == 0) cnt += 1.0;
    const long long k0 = __ldg(a.rowptr + row), k1 = __ldg(a.rowptr + row + 1);
    for (long long ka = k0; ka < k1; ++ka) {
      const int ia = __ldg(a.idx + ka);
      const double xa = (double)val[ka];
      for (long long kb = ka + lane; kb < k1; kb += 32) {
        const int ib = __ldg(a.idx + kb);
        const double xb = (double)val[kb];
        const int i = ia < ib ? ia : ib, j = ia < ib ? ib : ia;
        const double v = (kb != ka && ia == ib) ? 2.0 * (xa * xb) : xa * xb;
        atomicAdd(out + gm_packed(i, j, n1), v);
      }
    }
    for (long long k = k0 + lane; k < k1; k += 32) atomicAdd(out + gm_packed(__ldg(a.idx + k), a.d, n1), (double)val[k]);
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
  if (lane == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kGmCsrThreads / 32; ++w) t += red[w];
    atomicAdd(out + gm_packed(a.d, a.d, n1), t);   // row counts are small integers: exact in any order
  }
}

// out = the centered sums from the uncentered ones u of the same rows (packed, n = u[d][d] of them) and mu:
//   sum z_i z_j = u_ij - mu_i u_jd - mu_j u_id + n mu_i mu_j,  sum z_i = u_id - n mu_i,  count = n
__global__ void __launch_bounds__(256) gramian_center_kernel(const double *__restrict__ u, const double *__restrict__ mu, int d,
                                                            double *__restrict__ out) {
  const long long n1 = (long long)d + 1;
  const int i = blockIdx.x;
  const double n = u[gm_packed(d, d, n1)];
  if (i == d) {
    if (threadIdx.x == 0) out[gm_packed(d, d, n1)] = n;
    return;
  }
  const double mi = mu[i], si = u[gm_packed(i, d, n1)];
  for (int j = i + threadIdx.x; j <= d; j += 256) {
    const long long p = gm_packed(i, j, n1);
    if (j == d) out[p] = si - n * mi;
    else {
      const double mj = mu[j], sj = u[gm_packed(j, d, n1)];
      out[p] = ((u[p] - mi * sj) - mj * si) + n * (mi * mj);
    }
  }
}

template <typename T, bool VEC>
cudaError_t launch_dense(const GramianArgs &a, int sm_count, int splits, long long chunk) {
  auto kern = gramian_dense_kernel<T, VEC>;
  constexpr size_t smem = gm_smem_bytes<T>();
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int nb = (a.d + kGmBlk - 1) / kGmBlk;
  kern<<<dim3((unsigned)(nb * (nb + 1) / 2), (unsigned)splits), kGmThreads, smem, a.stream>>>(a, chunk);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_dense_t(const GramianArgs &a, int sm_count, int splits, long long chunk) {
  if ((size_t)a.d * sizeof(T) % 16 == 0) return launch_dense<T, true>(a, sm_count, splits, chunk);
  return launch_dense<T, false>(a, sm_count, splits, chunk);
}

}  // namespace

size_t gramian_packed_n(int32_t d) { return (size_t)gm_packed(d, d, (long long)d + 1) + 1; }

int gramian_splits(int sm_count, int32_t d, int64_t rows) {
  const long long nb = (d + kGmBlk - 1) / kGmBlk, pairs = nb * (nb + 1) / 2;
  // one resident CTA per SM; the split count that finishes the fewest full waves per unit of work, the smallest on a tie,
  // with each split's slab bounded (1 GiB of slabs in all) and at least 8 stages of rows per split
  long long smax = (1LL << 27) / (long long)gramian_packed_n(d);
  const long long by_rows = rows / (8LL * kGmKc);
  if (smax > by_rows) smax = by_rows;
  if (smax > 64) smax = 64;
  if (smax < 1) smax = 1;
  int best = 1;
  double best_cost = 1e300;
  for (long long s = 1; s <= smax; ++s) {
    const long long waves = (pairs * s + sm_count - 1) / sm_count;
    const double cost = (double)waves / (double)s;
    if (cost < best_cost * (1.0 - 1e-12)) { best_cost = cost; best = (int)s; }
  }
  return best;
}

cudaError_t gramian_dense_launch(const GramianArgs &a, int elem_bytes, int sm_count, int splits) {
  long long chunk = (a.rows + splits - 1) / splits;
  chunk = (chunk + kGmKc - 1) / kGmKc * kGmKc;
  if (chunk < kGmKc) chunk = kGmKc;
  if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16>(a, sm_count, splits, chunk);
  if (elem_bytes == 4) return launch_dense_t<float>(a, sm_count, splits, chunk);
  if (elem_bytes == 8) return launch_dense_t<double>(a, sm_count, splits, chunk);
  return cudaErrorInvalidValue;
}

cudaError_t gramian_csr_launch(const GramianArgs &a, int elem_bytes, int sm_count) {
  if (a.rows <= 0) return cudaSuccess;
  if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
  auto kern = elem_bytes == 8 ? gramian_csr_kernel<double> : gramian_csr_kernel<float>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kGmCsrThreads, 0);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  long long grid = (long long)per_sm * sm_count;
  const long long need = (a.rows + kGmCsrThreads / 32 - 1) / (kGmCsrThreads / 32);
  if (grid > need) grid = need;
  kern<<<(unsigned)grid, kGmCsrThreads, 0, a.stream>>>(a);
  return cudaGetLastError();
}

cudaError_t gramian_center_launch(const double *u, const double *mu, int32_t d, double *out, cudaStream_t st) {
  gramian_center_kernel<<<(unsigned)d + 1, 256, 0, st>>>(u, mu, d, out);
  return cudaGetLastError();
}

}  // namespace agd
