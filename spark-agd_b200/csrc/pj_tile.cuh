// pj_tile.cuh -- the row tile of the fp64 tensor-core GEMM X B (internal, sm_90a), shared by the projection (project.cu) and
// the k-means assignment (kmeans.cu), which differ only in what they do with the accumulators.
//
// A CTA of kPjThreads owns kPjRows rows of X and one tile of BN <= 128 columns of B; it streams its rows through a ring of
// storage-type tiles in chunks of kPjKc columns (cp.async 16-byte copies; rows whose stride is not a multiple of 16 bytes use
// plain loads), widens every element once into a double-buffered fp64 tile, and takes the matching kPjKc x BN chunk of B
// (zero-padded) through the same ring.  Every accumulator is carried over the chunks in column order, with the same MMA
// sequence for every row of every tile, so its bits depend only on the row and B.  A row whose orow entry is negative is
// never read (0-byte copies fill it with zeros).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>

#include "agd_common.cuh"
#include "dmma.cuh"

namespace agd {

constexpr int kPjThreads = 256;         // 8 warps
constexpr int kPjKc = 16;               // columns of X (rows of B) per stage
constexpr int kPjStages = 4;            // ring depth: two chunks in flight while one is multiplied and the next widened
constexpr int kPjLda = kPjKc + 4;       // fp64 tile row stride: the fragment reads of a half-warp hit 16 distinct 8-byte banks
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
// [2][kPjRows][kPjLda] | a long long per tile row (orow)
template <typename T, int BN>
__host__ __device__ constexpr size_t pj_smem_bytes() {
  return (size_t)kPjStages * kPjKc * PjShape<BN>::LDB * sizeof(double) + (size_t)kPjStages * kPjRows * kPjKc * sizeof(T) +
         2 * (size_t)kPjRows * kPjLda * sizeof(double) + (size_t)kPjRows * sizeof(long long);
}
template <typename T, int BN> __device__ __forceinline__ long long *pj_orow(unsigned char *smem) {
  return reinterpret_cast<long long *>(smem + pj_smem_bytes<T, BN>() - (size_t)kPjRows * sizeof(long long));
}
// the fp64 tiles, free for an epilogue once pj_tile_mma has returned and the CTA has synchronised
template <typename T, int BN> __device__ __forceinline__ double *pj_fp64_tiles(unsigned char *smem) {
  return reinterpret_cast<double *>(smem + (size_t)kPjStages * kPjKc * PjShape<BN>::LDB * sizeof(double) +
                                    (size_t)kPjStages * kPjRows * kPjKc * sizeof(T));
}

// Rank of physical row `row` among the rows of a view (-1: outside it), from the kept rows before its tile of kPjRows rows
// (tile_base, project_scan_launch) and the bitmap words of the tile up to it.
__device__ __forceinline__ long long view_rank(const uint32_t *bits, const long long *tile_base, long long row) {
  const uint32_t w = bits[row >> 5];
  if (!((w >> (row & 31)) & 1u)) return -1;
  const long long t = row / kPjRows;
  long long o = tile_base[t];
  for (long long q = t * (kPjRows / 32); q < (row >> 5); ++q) o += __popc(bits[q]);
  return o + __popc(w & ((1u << (row & 31)) - 1u));
}

// acc[mt][nt][q] = sum over l < d of x[r0 + i][l] B[l][c0 + j] for the fragment element (i, j) of this thread (see the
// epilogues), rows i with orow[i] < 0 contributing zeros.  orow (kPjRows entries in smem) must be written and synchronised
// by the caller.  B is [round_up(d, kPjKc)][kp] doubles.
template <typename T, bool VEC, int BN>
__device__ __forceinline__ void pj_tile_mma(unsigned char *smem, const T *__restrict__ X, int d, const double *__restrict__ B,
                                            int kp, long long r0, int c0, double (&acc)[PjShape<BN>::MT][PjShape<BN>::NT][4]) {
  using S = PjShape<BN>;
  double *bring = reinterpret_cast<double *>(smem);
  T *xring = reinterpret_cast<T *>(bring + (size_t)kPjStages * kPjKc * S::LDB);
  double *at = reinterpret_cast<double *>(xring + (size_t)kPjStages * kPjRows * kPjKc);
  const long long *orow = reinterpret_cast<const long long *>(at + 2 * kPjRows * kPjLda);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  const int nch = (d + kPjKc - 1) / kPjKc;
  // stage kc % kPjStages <- columns [kc kPjKc, + kPjKc) of the tile's rows and the same rows of B's column tile; a row outside the
  // view or past the shard, and columns past d, are not read (zeros)
  auto issue = [&](int kc) {
    if (kc >= nch) return;
    const int s = kc % kPjStages, col0 = kc * kPjKc;
    double *bs = bring + (size_t)s * kPjKc * S::LDB;
    for (int u = tid; u < kPjKc * (BN / 2); u += kPjThreads) {
      const int r = u / (BN / 2), cu = u % (BN / 2);
      gm_cp16((uint32_t)__cvta_generic_to_shared(bs + r * S::LDB + cu * 2), B + (size_t)(col0 + r) * kp + c0 + cu * 2, 16);
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
}

// Tile row and column of fragment element (mt, nt, q) of this thread's accumulators
template <int BN> __device__ __forceinline__ int pj_frag_row(int mt, int q) {
  using S = PjShape<BN>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp / S::WN) * S::MT * 16 + mt * 16 + (lane >> 2) + (q >> 1) * 8;
}
template <int BN> __device__ __forceinline__ int pj_frag_col(int nt, int q) {
  using S = PjShape<BN>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp % S::WN) * S::NT * 8 + nt * 8 + (lane & 3) * 2 + (q & 1);
}

template <int BN> constexpr bool pj_bn_ok = BN == 16 || BN == 32 || BN == 64 || BN == 128;

// Row tiles rt0 + blockIdx.y of every launch: grids of at most kPjMaxGridY row tiles, each with `col_tiles` column tiles side
// by side (they share their rows through L2).  kern(args, rt0).
template <typename T, int BN, typename Kern, typename Args>
cudaError_t pj_launch_rows(Kern kern, const Args &a, long long rows, int col_tiles, cudaStream_t st) {
  static_assert(pj_bn_ok<BN>, "column tile");
  constexpr size_t smem = pj_smem_bytes<T, BN>();
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long tiles = (rows + kPjRows - 1) / kPjRows;
  for (long long rt0 = 0; rt0 < tiles; rt0 += kPjMaxGridY) {
    const long long n = tiles - rt0 < kPjMaxGridY ? tiles - rt0 : kPjMaxGridY;
    kern<<<dim3((unsigned)col_tiles, (unsigned)n), kPjThreads, smem, st>>>(a, rt0);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace agd
