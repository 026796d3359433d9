// project.cu -- Y = X B + c of the rows of a view of a resident shard, into another handle's shard (sm_90a): the kernels behind
// agd_project (RowMatrix.multiply of mllib 1.3.0).
//
// Dense: a GEMM on the fp64 tensor cores (mma.sync m16n8k4 .f64, DMMA).  A CTA owns kPjRows rows of X and one tile of BN <= 128
// output columns; it streams its rows through a ring of storage-type tiles in chunks of kPjKc columns (cp.async 16-byte copies;
// rows whose stride is not a multiple of 16 bytes use plain loads), widens every element once into a double-buffered fp64 tile,
// and takes the matching kPjKc x BN chunk of B (zero-padded) through the same ring.  Every output element is one accumulator
// carried over the chunks in column order, with the same MMA sequence for every row of every tile, so its bits depend only on
// the row, B and c: not on where the row sits, which tile it lands in, the device, the rank or the view.  c_j is added last and
// the sum rounded once to the destination's storage type.  A row outside the view is never read (0-byte copies fill it with
// zeros) and never written; the kept rows are compacted in physical order through an exclusive scan of the view bitmap.
// CSR: one warp per row of the view, lanes over output columns; every stored entry, in stored order, adds x B[col, :] in fp64.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "dmma.cuh"

namespace agd {

namespace {

constexpr int kPjThreads = 256;         // 8 warps
constexpr int kPjKc = 16;               // columns of X (rows of B) per stage
constexpr int kPjStages = 4;            // ring depth: two chunks in flight while one is multiplied and the next widened
constexpr int kPjLda = kPjKc + 4;       // fp64 tile row stride: the fragment reads of a half-warp hit 16 distinct 8-byte banks
constexpr int kPjScanThreads = 1024;
constexpr int kPjCsrThreads = 256;
constexpr int kPjCsrCols = 4;           // output columns per lane and pass of the CSR kernel
constexpr long long kPjMaxGridY = 65535;

// Warp layout of a BN-column tile: WM x WN warps, each owning MT 16-row by NT 8-column MMA tiles.  LDB = BN + 4 keeps the B
// fragment reads of a half-warp on distinct banks.
template <int BN> struct PjShape {
  static constexpr int WN = BN >= 32 ? BN / 32 : 1;
  static constexpr int WM = 8 / WN;
  static constexpr int MT = kPjRows / (16 * WM);
  static constexpr int NT = BN / (8 * WN);
  static constexpr int LDB = BN + 4;
};

// Smem (dynamic): B ring [kPjStages][kPjKc][LDB] fp64 | X ring [kPjStages][kPjRows][kPjKc] storage elements | fp64 tiles
// [2][kPjRows][kPjLda] | output row of each tile row [kPjRows]
template <typename T, int BN>
__host__ __device__ constexpr size_t pj_smem_bytes() {
  return (size_t)kPjStages * kPjKc * PjShape<BN>::LDB * sizeof(double) + (size_t)kPjStages * kPjRows * kPjKc * sizeof(T) +
         2 * (size_t)kPjRows * kPjLda * sizeof(double) + (size_t)kPjRows * sizeof(long long);
}

__device__ __forceinline__ void pj_store(void *Y, int out_bytes, long long at, double y) {
  if (out_bytes == 8) reinterpret_cast<double *>(Y)[at] = y;
  else if (out_bytes == 4) reinterpret_cast<float *>(Y)[at] = __double2float_rn(y);
  else reinterpret_cast<__nv_bfloat16 *>(Y)[at] = __double2bfloat16(y);
}

// Destination row of physical row `row` (-1: outside the view): its rank among the kept rows, from the kept rows before its
// tile (tile_base) and the bitmap words of the tile up to it.
__device__ __forceinline__ long long pj_out_row(const ProjectArgs &a, long long row) {
  if (!a.view_bits) return row;
  const uint32_t w = a.view_bits[row >> 5];
  if (!((w >> (row & 31)) & 1u)) return -1;
  const long long t = row / kPjRows;
  long long o = a.tile_base[t];
  for (long long q = t * (kPjRows / 32); q < (row >> 5); ++q) o += __popc(a.view_bits[q]);
  return o + __popc(w & ((1u << (row & 31)) - 1u));
}

// tile_base[t] = kept rows in tiles 0 .. t - 1, *total = kept rows of the shard (one CTA; each thread a contiguous run of tiles)
__global__ void __launch_bounds__(kPjScanThreads) project_scan_kernel(const uint32_t *__restrict__ bits, long long rows,
                                                                      long long *__restrict__ tile_base,
                                                                      long long *__restrict__ total) {
  __shared__ long long part[kPjScanThreads];
  const int tid = threadIdx.x;
  const long long tiles = (rows + kPjRows - 1) / kPjRows, words = (rows + 31) / 32;
  const long long per = (tiles + kPjScanThreads - 1) / kPjScanThreads;
  const long long t0 = tid * per, t1 = t0 + per < tiles ? t0 + per : tiles;
  auto tile_count = [&](long long t) {
    long long s = 0;
    for (long long w = t * (kPjRows / 32); w < (t + 1) * (kPjRows / 32) && w < words; ++w) s += __popc(bits[w]);
    return s;
  };
  long long mine = 0;
  for (long long t = t0; t < t1; ++t) mine += tile_count(t);
  part[tid] = mine;
  __syncthreads();
  for (int off = 1; off < kPjScanThreads; off <<= 1) {
    const long long v = tid >= off ? part[tid - off] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  long long base = part[tid] - mine;
  for (long long t = t0; t < t1; ++t) {
    tile_base[t] = base;
    base += tile_count(t);
  }
  if (tid == kPjScanThreads - 1) *total = part[tid];
}

// VEC: rows are whole 16-byte vectors (d * sizeof(T) % 16 == 0), staged with cp.async; else plain loads.  Row tile rt0 +
// blockIdx.y, column tile blockIdx.x (the column tiles of one row tile run side by side and share its rows through L2).
template <typename T, bool VEC, int BN>
__global__ void __launch_bounds__(kPjThreads, BN == 128 ? 1 : 2) project_dense_kernel(const ProjectArgs a, const long long rt0) {
  using S = PjShape<BN>;
  extern __shared__ __align__(16) unsigned char pj_smem[];
  double *bring = reinterpret_cast<double *>(pj_smem);
  T *xring = reinterpret_cast<T *>(bring + (size_t)kPjStages * kPjKc * S::LDB);
  double *at = reinterpret_cast<double *>(xring + (size_t)kPjStages * kPjRows * kPjKc);
  long long *orow = reinterpret_cast<long long *>(at + 2 * kPjRows * kPjLda);

  const int d = a.d, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long r0 = (rt0 + blockIdx.y) * kPjRows;
  const int c0 = (int)blockIdx.x * BN;
  const T *X = reinterpret_cast<const T *>(a.X);
  if (tid < kPjRows) orow[tid] = r0 + tid < a.rows ? pj_out_row(a, r0 + tid) : -1;
  __syncthreads();

  const int nch = (d + kPjKc - 1) / kPjKc;
  // stage kc % kPjStages <- columns [kc kPjKc, + kPjKc) of the tile's rows and the same rows of B's column tile; a row outside the
  // view or past the shard, and columns past d, are not read (zeros)
  auto issue = [&](int kc) {
    if (kc >= nch) return;
    const int s = kc % kPjStages, col0 = kc * kPjKc;
    double *bs = bring + (size_t)s * kPjKc * S::LDB;
    for (int u = tid; u < kPjKc * (BN / 2); u += kPjThreads) {
      const int r = u / (BN / 2), cu = u % (BN / 2);
      gm_cp16((uint32_t)__cvta_generic_to_shared(bs + r * S::LDB + cu * 2), a.B + (size_t)(col0 + r) * a.kp + c0 + cu * 2, 16);
    }
    T *xs = xring + (size_t)s * kPjRows * kPjKc;
    if (VEC) {
      constexpr int EPV = 16 / sizeof(T), UPR = kPjKc / EPV;   // 16-byte units per row of a chunk
      for (int u = tid; u < kPjRows * UPR; u += kPjThreads) {
        const int r = u / UPR, col = col0 + (u % UPR) * EPV;
        const bool ok = orow[r] >= 0 && col < d;
        const T *src = ok ? X + (size_t)(r0 + r) * d + col : X;
        gm_cp16((uint32_t)__cvta_generic_to_shared(xs + r * kPjKc + (u % UPR) * EPV), src, ok ? 16 : 0);
      }
    } else {
      for (int e = tid; e < kPjRows * kPjKc; e += kPjThreads) {
        const int r = e / kPjKc, col = col0 + e % kPjKc;
        T v;
        if (orow[r] >= 0 && col < d) v = X[(size_t)(r0 + r) * d + col];
        else memset(&v, 0, sizeof v);
        xs[e] = v;
      }
    }
  };
  // chunk kc of the X ring -> fp64 tile zb, every element widened once
  auto convert = [&](int kc, int zb) {
    const T *xs = xring + (size_t)(kc % kPjStages) * kPjRows * kPjKc;
    double *z = at + (size_t)zb * kPjRows * kPjLda;
#pragma unroll
    for (int e = tid; e < kPjRows * kPjKc; e += kPjThreads) z[(e / kPjKc) * kPjLda + e % kPjKc] = GmElem<T>::wide(xs[e]);
  };

  double acc[S::MT][S::NT][4];
#pragma unroll
  for (int i = 0; i < S::MT; ++i)
#pragma unroll
    for (int j = 0; j < S::NT; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.0;
  const int wm = warp / S::WN, wn = warp % S::WN;

  for (int q = 0; q < kPjStages - 1; ++q) {
    issue(q);
    gm_commit();
  }
  if (nch > 0) {
    gm_wait<kPjStages - 2>();
    __syncthreads();
    convert(0, 0);
  }
  for (int kc = 0; kc < nch; ++kc) {
    gm_wait<kPjStages - 3>();
    __syncthreads();   // chunk kc + 1 landed and chunk kc is widened, for every thread; the MMAs of chunk kc - 1 are done
    issue(kc + kPjStages - 1);   // into the stage of chunk kc - 1
    gm_commit();
    const double *As = at + (size_t)(kc & 1) * kPjRows * kPjLda;
    const double *Bs = bring + (size_t)(kc % kPjStages) * kPjKc * S::LDB;
#pragma unroll
    for (int ks = 0; ks < kPjKc / 4; ++ks) {
      const int kr = ks * 4 + (lane & 3);
      double af[S::MT][2], bf[S::NT];
#pragma unroll
      for (int mt = 0; mt < S::MT; ++mt) {
        const int m = wm * S::MT * 16 + mt * 16 + (lane >> 2);
        af[mt][0] = As[m * kPjLda + kr];
        af[mt][1] = As[(m + 8) * kPjLda + kr];
      }
#pragma unroll
      for (int nt = 0; nt < S::NT; ++nt) bf[nt] = Bs[kr * S::LDB + wn * S::NT * 8 + nt * 8 + (lane >> 2)];
#pragma unroll
      for (int mt = 0; mt < S::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < S::NT; ++nt) gm_dmma(acc[mt][nt], af[mt], bf[nt]);
    }
    if (kc + 1 < nch) convert(kc + 1, (kc + 1) & 1);
  }

  // y = acc + c_j, rounded once; the destination's padded columns k .. ldy - 1 are written as 0
#pragma unroll
  for (int mt = 0; mt < S::MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < S::NT; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = wm * S::MT * 16 + mt * 16 + (lane >> 2) + (q >> 1) * 8;
        const int j = c0 + wn * S::NT * 8 + nt * 8 + (lane & 3) * 2 + (q & 1);
        const long long o = orow[i];
        if (o >= 0 && j < a.ldy) pj_store(a.Y, a.out_bytes, o * a.ldy + j, j < a.k ? acc[mt][nt][q] + a.c[j] : 0.0);
      }
  if (blockIdx.x == 0 && tid < kPjRows && orow[tid] >= 0) a.Ylabels[orow[tid]] = a.labels[r0 + tid];
}

template <typename T>
__global__ void __launch_bounds__(kPjCsrThreads) project_csr_kernel(const ProjectArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kPjCsrThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kPjCsrThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  for (long long row = warp0; row < a.rows; row += nwarps) {
    const long long o = pj_out_row(a, row);
    if (o < 0) continue;
    const long long k0 = __ldg(a.rowptr + row), k1 = __ldg(a.rowptr + row + 1);
    for (int j0 = 0; j0 < a.ldy; j0 += 32 * kPjCsrCols) {
      double acc[kPjCsrCols];
#pragma unroll
      for (int q = 0; q < kPjCsrCols; ++q) acc[q] = 0.0;
      for (long long e = k0; e < k1; ++e) {
        const double x = (double)val[e];
        const double *b = a.B + (size_t)__ldg(a.idx + e) * a.kp;
#pragma unroll
        for (int q = 0; q < kPjCsrCols; ++q) {
          const int j = j0 + q * 32 + lane;
          if (j < a.ldy) acc[q] = fma(x, __ldg(b + j), acc[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < kPjCsrCols; ++q) {
        const int j = j0 + q * 32 + lane;
        if (j < a.ldy) pj_store(a.Y, a.out_bytes, o * a.ldy + j, j < a.k ? acc[q] + a.c[j] : 0.0);
      }
    }
    if (lane == 0) a.Ylabels[o] = a.labels[row];
  }
}

template <int BN> constexpr bool pj_bn_ok = BN == 16 || BN == 32 || BN == 64 || BN == 128;

template <typename T, bool VEC, int BN>
cudaError_t launch_dense(const ProjectArgs &a) {
  static_assert(pj_bn_ok<BN>, "column tile");
  auto kern = project_dense_kernel<T, VEC, BN>;
  constexpr size_t smem = pj_smem_bytes<T, BN>();
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long tiles = (a.rows + kPjRows - 1) / kPjRows;
  for (long long rt0 = 0; rt0 < tiles; rt0 += kPjMaxGridY) {
    const long long n = tiles - rt0 < kPjMaxGridY ? tiles - rt0 : kPjMaxGridY;
    kern<<<dim3((unsigned)(a.kp / BN), (unsigned)n), kPjThreads, smem, a.stream>>>(a, rt0);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

template <typename T, int BN>
cudaError_t launch_dense_vec(const ProjectArgs &a) {
  if ((size_t)a.d * sizeof(T) % 16 == 0) return launch_dense<T, true, BN>(a);
  return launch_dense<T, false, BN>(a);
}

template <typename T>
cudaError_t launch_dense_t(const ProjectArgs &a) {
  switch (project_tile_cols(a.k)) {
    case 16: return launch_dense_vec<T, 16>(a);
    case 32: return launch_dense_vec<T, 32>(a);
    case 64: return launch_dense_vec<T, 64>(a);
    default: return launch_dense_vec<T, 128>(a);
  }
}

}  // namespace

int project_tile_cols(int32_t k) { return k <= 16 ? 16 : (k <= 32 ? 32 : (k <= 64 ? 64 : 128)); }

cudaError_t project_scan_launch(const uint32_t *bits, int64_t rows, long long *tile_base, long long *total, cudaStream_t st) {
  project_scan_kernel<<<1, kPjScanThreads, 0, st>>>(bits, rows, tile_base, total);
  return cudaGetLastError();
}

cudaError_t project_dense_launch(const ProjectArgs &a, int elem_bytes) {
  if (a.rows <= 0) return cudaSuccess;
  if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16>(a);
  if (elem_bytes == 4) return launch_dense_t<float>(a);
  if (elem_bytes == 8) return launch_dense_t<double>(a);
  return cudaErrorInvalidValue;
}

cudaError_t project_csr_launch(const ProjectArgs &a, int elem_bytes, int sm_count) {
  if (a.rows <= 0) return cudaSuccess;
  if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
  auto kern = elem_bytes == 8 ? project_csr_kernel<double> : project_csr_kernel<float>;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kPjCsrThreads, 0);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  long long grid = (long long)per_sm * sm_count;
  const long long need = (a.rows + kPjCsrThreads / 32 - 1) / (kPjCsrThreads / 32);
  if (grid > need) grid = need;
  kern<<<(unsigned)grid, kPjCsrThreads, 0, a.stream>>>(a);
  return cudaGetLastError();
}

}  // namespace agd
