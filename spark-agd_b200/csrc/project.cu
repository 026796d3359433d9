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
#include "pj_tile.cuh"

namespace agd {

namespace {

constexpr int kPjScanThreads = 1024;
constexpr int kPjCsrThreads = 256;
constexpr int kPjCsrCols = 4;           // output columns per lane and pass of the CSR kernel

__device__ __forceinline__ void pj_store(void *Y, int out_bytes, long long at, double y) {
  if (out_bytes == 8) reinterpret_cast<double *>(Y)[at] = y;
  else if (out_bytes == 4) reinterpret_cast<float *>(Y)[at] = __double2float_rn(y);
  else reinterpret_cast<__nv_bfloat16 *>(Y)[at] = __double2bfloat16(y);
}

// Destination row of physical row `row` (-1: outside the view)
__device__ __forceinline__ long long pj_out_row(const ProjectArgs &a, long long row) {
  if (!a.view_bits) return row;
  return view_rank(a.view_bits, a.tile_base, row);
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
// blockIdx.y, column tile blockIdx.x.
template <typename T, bool VEC, int BN>
__global__ void __launch_bounds__(kPjThreads, BN == 128 ? 1 : 2) project_dense_kernel(const ProjectArgs a, const long long rt0) {
  using S = PjShape<BN>;
  extern __shared__ __align__(16) unsigned char pj_smem[];
  long long *orow = pj_orow<T, BN>(pj_smem);
  const int tid = threadIdx.x;
  const long long r0 = (rt0 + blockIdx.y) * kPjRows;
  const int c0 = (int)blockIdx.x * BN;
  if (tid < kPjRows) orow[tid] = r0 + tid < a.rows ? pj_out_row(a, r0 + tid) : -1;
  __syncthreads();
  double acc[S::MT][S::NT][4];
  pj_tile_mma<T, VEC, BN>(pj_smem, reinterpret_cast<const T *>(a.X), a.d, a.B, a.kp, r0, c0, acc);

  // y = acc + c_j, rounded once; the destination's padded columns k .. ldy - 1 are written as 0
#pragma unroll
  for (int mt = 0; mt < S::MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < S::NT; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = pj_frag_row<BN>(mt, q);
        const int j = c0 + pj_frag_col<BN>(nt, q);
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

template <typename T, bool VEC, int BN>
cudaError_t launch_dense(const ProjectArgs &a) {
  return pj_launch_rows<T, BN>(project_dense_kernel<T, VEC, BN>, a, a.rows, a.kp / BN, a.stream);
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
