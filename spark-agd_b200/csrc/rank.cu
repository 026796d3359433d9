// rank.cu -- ranking metrics of a view (agd_binary_curve, sm_90a): a stable LSD radix sort of (margin key, value) pairs, the
// run-length reduce of the sorted pairs into the curve of cumulative counts, the concatenation of the world's lists, and the
// trapezoid areas under ROC and PR.
//   * sort: 8-bit digits, tiles of kTile pairs.  One pass over the keys counts all eight digits first; a digit that is the
//     same in every key (the exponent bytes of margins often are) costs no pass.  A pass counts each tile's digits, scans the
//     counts per digit in tile order (digit-major, so digit starts come from the histogram) and scatters stably: a tile is
//     taken 256 pairs at a time in index order, a warp ranks equal digits with match.any, the warps before it add their counts.
//   * runs: heads (first pair of a key) and the two class counts are scanned over the sorted pairs (per-tile sums, one scan of
//     the tile sums, per-tile scans); the last pair of a key writes {key, cumulative positives, cumulative negatives}.
//     Counts are integers, so the curve is exact and does not depend on the order of equal keys.
//   * areas: one trapezoid per segment, each block sums its segments in index order (per thread, then a fixed xor butterfly,
//     then the warps in order), and one block adds the block sums the same way: the bits depend on the curve only.
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"

namespace agd {

namespace {

constexpr int kThreads = 256, kItems = 8, kTile = kThreads * kItems;

long long tiles_of(long long n) { return (n + kTile - 1) / kTile; }

// exclusive scan of one value per thread over the block; *total = the block's sum.  Every thread of the block calls it.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T *total) {
  __shared__ T warp_tot[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, inc, off);
    if (lane >= off) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  T base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    if (w < warp) base += warp_tot[w];
    tot += warp_tot[w];
  }
  __syncthreads();   // warp_tot is reused by the next call
  *total = tot;
  return base + inc - v;
}

// fixed-order block sum of one double per thread (xor butterfly per warp, then the warps in index order); valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double red[kThreads / 32];
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
  __syncthreads();
  return t;
}

// ---- sort
__global__ void __launch_bounds__(kThreads) bin_hist8_kernel(const unsigned long long *keys, long long n, unsigned *hist) {
  __shared__ unsigned h[8 * 256];
  for (int i = threadIdx.x; i < 8 * 256; i += kThreads) h[i] = 0;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    const unsigned long long k = keys[i];
#pragma unroll
    for (int p = 0; p < 8; ++p) atomicAdd(&h[p * 256 + (unsigned)((k >> (8 * p)) & 255u)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * 256; i += kThreads)
    if (h[i]) atomicAdd(hist + i, h[i]);
}

// counts[digit * tiles + tile] = pairs of the tile with that digit
__global__ void __launch_bounds__(kThreads) bin_count_kernel(const unsigned long long *keys, long long n, int shift,
                                                             unsigned *counts, long long tiles) {
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * kTile;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const long long i = t0 + j * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(unsigned)(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  counts[threadIdx.x * tiles + blockIdx.x] = h[threadIdx.x];
}

// one block per digit: counts -> the tile's first output position for that digit (digit start + earlier tiles' counts)
__global__ void __launch_bounds__(kThreads) bin_offsets_kernel(unsigned *counts, long long tiles, const unsigned *hist_pass) {
  __shared__ unsigned start;
  const int dg = blockIdx.x;
  if (threadIdx.x == 0) {
    unsigned s = 0;
    for (int e = 0; e < dg; ++e) s += hist_pass[e];
    start = s;
  }
  __syncthreads();
  unsigned run = start;
  unsigned *c = counts + (long long)dg * tiles;
  for (long long t0 = 0; t0 < tiles; t0 += kThreads) {
    const long long t = t0 + threadIdx.x;
    const unsigned v = t < tiles ? c[t] : 0u;
    unsigned tot;
    const unsigned ex = block_exclusive_scan(v, &tot);
    if (t < tiles) c[t] = run + ex;
    run += tot;
  }
}

template <typename V>
__global__ void __launch_bounds__(kThreads) bin_scatter_kernel(const unsigned long long *keys, const V *vals,
                                                               unsigned long long *keys_out, V *vals_out, long long n, int shift,
                                                               const unsigned *offs, long long tiles) {
  __shared__ unsigned base[256];                  // next output position of each digit
  __shared__ unsigned wcnt[kThreads / 32][256];   // this round's pairs per warp and digit
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  base[threadIdx.x] = offs[threadIdx.x * tiles + blockIdx.x];
  for (int w = 0; w < kThreads / 32; ++w) wcnt[w][threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * kTile;
  for (int j = 0; j < kItems; ++j) {
    if (t0 + (long long)j * kThreads >= n) break;   // uniform over the block
    const long long i = t0 + (long long)j * kThreads + threadIdx.x;
    const bool ok = i < n;
    const unsigned long long k = ok ? keys[i] : 0ull;
    const unsigned dg = ok ? ((unsigned)(k >> shift) & 255u) : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, dg);
    const unsigned before = __popc(peers & ((1u << lane) - 1u));
    if (ok && before == 0) wcnt[warp][dg] = __popc(peers);
    __syncthreads();
    if (ok) {
      unsigned pos = base[dg] + before;
      for (int w = 0; w < warp; ++w) pos += wcnt[w][dg];
      keys_out[pos] = k;
      vals_out[pos] = vals[i];
    }
    __syncthreads();
    unsigned add = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      add += wcnt[w][threadIdx.x];
      wcnt[w][threadIdx.x] = 0;
    }
    base[threadIdx.x] += add;
    __syncthreads();
  }
}

// ---- runs
struct ClassVals {   // local pairs: the value is the class
  const uint8_t *v;
  __device__ void get(long long i, long long &pos, long long &neg) const {
    pos = v[i];
    neg = 1 - pos;
  }
};
struct IndexVals {   // the world's lists: the value indexes a record's own counts
  const uint32_t *v;
  const long long *upos, *uneg;
  __device__ void get(long long i, long long &pos, long long &neg) const {
    const uint32_t j = v[i];
    pos = upos[j];
    neg = uneg[j];
  }
};

// this thread's kItems consecutive pairs of the tile: sums of the two counts and of the heads
template <typename G>
__device__ __forceinline__ void run_sums(const unsigned long long *keys, const G &g, long long n, long long first, long long &p,
                                         long long &q, long long &hd) {
  p = q = hd = 0;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const long long i = first + j;
    if (i < n) {
      long long a, b;
      g.get(i, a, b);
      p += a;
      q += b;
      hd += (i == 0 || keys[i - 1] != keys[i]) ? 1 : 0;
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(kThreads) bin_runs_tile_kernel(const unsigned long long *keys, const G g, long long n,
                                                                 long long *tile_sums) {
  long long p, q, hd, tp, tq, th;
  run_sums(keys, g, n, (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems, p, q, hd);
  block_exclusive_scan(p, &tp);
  block_exclusive_scan(q, &tq);
  block_exclusive_scan(hd, &th);
  if (threadIdx.x == 0) {
    tile_sums[3 * (long long)blockIdx.x] = tp;
    tile_sums[3 * (long long)blockIdx.x + 1] = tq;
    tile_sums[3 * (long long)blockIdx.x + 2] = th;
  }
}

// one block: the tile sums -> their exclusive prefix sums, in place
__global__ void __launch_bounds__(kThreads) bin_runs_scan_kernel(long long *tile_sums, long long tiles) {
  long long run[3] = {0, 0, 0};
  for (long long t0 = 0; t0 < tiles; t0 += kThreads) {
    const long long t = t0 + threadIdx.x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long v = t < tiles ? tile_sums[3 * t + c] : 0;
      long long tot;
      const long long ex = block_exclusive_scan(v, &tot);
      if (t < tiles) tile_sums[3 * t + c] = run[c] + ex;
      run[c] += tot;
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(kThreads) bin_runs_write_kernel(const unsigned long long *keys, const G g, long long n,
                                                                  const long long *tile_sums, BinRec *out, long long *n_out) {
  const long long first = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems;
  long long p, q, hd, tp, tq, th;
  run_sums(keys, g, n, first, p, q, hd);
  long long cp = block_exclusive_scan(p, &tp) + tile_sums[3 * (long long)blockIdx.x];
  long long cq = block_exclusive_scan(q, &tq) + tile_sums[3 * (long long)blockIdx.x + 1];
  long long ch = block_exclusive_scan(hd, &th) + tile_sums[3 * (long long)blockIdx.x + 2];
  for (int j = 0; j < kItems; ++j) {
    const long long i = first + j;
    if (i >= n) break;
    long long a, b;
    g.get(i, a, b);
    const unsigned long long k = keys[i];
    cp += a;
    cq += b;
    if (i == 0 || keys[i - 1] != k) ch += 1;
    if (i == n - 1 || keys[i + 1] != k) {   // the key's last pair: its point of the curve
      BinRec r;
      r.key = k;
      r.tp = cp;
      r.fp = cq;
      out[ch - 1] = r;
      if (i == n - 1) *n_out = ch;
    }
  }
}

template <typename G>
cudaError_t runs(const unsigned long long *keys, const G &g, long long n, long long *tile_sums, BinRec *out, long long *n_out,
                 cudaStream_t st) {
  const long long T = tiles_of(n);
  bin_runs_tile_kernel<G><<<(unsigned)T, kThreads, 0, st>>>(keys, g, n, tile_sums);
  bin_runs_scan_kernel<<<1, kThreads, 0, st>>>(tile_sums, T);
  bin_runs_write_kernel<G><<<(unsigned)T, kThreads, 0, st>>>(keys, g, n, tile_sums, out, n_out);
  return cudaGetLastError();
}

// ---- the world's lists, concatenated in rank order
__global__ void __launch_bounds__(kThreads) bin_union_prep_kernel(const BinRec *blocks, long long stride, const long long *off,
                                                                  int world, long long total, unsigned long long *keys,
                                                                  uint32_t *idx, long long *upos, long long *uneg) {
  for (long long j = (long long)blockIdx.x * kThreads + threadIdx.x; j < total; j += (long long)gridDim.x * kThreads) {
    int lo = 0, hi = world - 1;   // the rank r with off[r] <= j < off[r + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= j) lo = mid;
      else hi = mid - 1;
    }
    const long long l = j - off[lo];
    const BinRec *b = blocks + (long long)lo * stride;
    const BinRec c = b[l];
    long long pp = 0, pq = 0;
    if (l > 0) {
      pp = b[l - 1].tp;
      pq = b[l - 1].fp;
    }
    keys[j] = c.key;
    idx[j] = (uint32_t)j;
    upos[j] = c.tp - pp;
    uneg[j] = c.fp - pq;
  }
}

// ---- areas
// ROC segment s in [0, K]: from point s - 1 to point s, with point -1 = (0, 0) and point K = (1, 1);
// PR segment s in [0, K): from point s - 1 to point s, with point -1 = (0, 1)
__device__ __forceinline__ void roc_point(const BinRec *c, long long K, long long k, double P, double N, double &x, double &y) {
  if (k < 0) { x = 0.0; y = 0.0; }
  else if (k >= K) { x = 1.0; y = 1.0; }
  else { x = (double)c[k].fp / N; y = (double)c[k].tp / P; }
}
__device__ __forceinline__ void pr_point(const BinRec *c, long long k, double P, double &x, double &y) {
  if (k < 0) { x = 0.0; y = 1.0; return; }
  const double tp = (double)c[k].tp;
  x = tp / P;
  y = tp / (tp + (double)c[k].fp);
}

__global__ void __launch_bounds__(kThreads) bin_area_kernel(const BinRec *c, long long K, double *partials) {
  const double P = (double)c[K - 1].tp, N = (double)c[K - 1].fp;
  const long long s0 = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems;
  double roc = 0.0, pr = 0.0;
  for (int j = 0; j < kItems; ++j) {
    const long long s = s0 + j;
    if (s <= K) {
      double x0, y0, x1, y1;
      roc_point(c, K, s - 1, P, N, x0, y0);
      roc_point(c, K, s, P, N, x1, y1);
      roc += (x1 - x0) * (y1 + y0) / 2.0;
    }
    if (s < K) {
      double x0, y0, x1, y1;
      pr_point(c, s - 1, P, x0, y0);
      pr_point(c, s, P, x1, y1);
      pr += (x1 - x0) * (y1 + y0) / 2.0;
    }
  }
  roc = block_sum(roc);
  pr = block_sum(pr);
  if (threadIdx.x == 0) {
    partials[2 * (long long)blockIdx.x] = roc;
    partials[2 * (long long)blockIdx.x + 1] = pr;
  }
}

__global__ void __launch_bounds__(kThreads) bin_area_final_kernel(const double *partials, int blocks, double *out) {
  const int per = (blocks + kThreads - 1) / kThreads;
  double roc = 0.0, pr = 0.0;
  for (int b = threadIdx.x * per; b < (threadIdx.x + 1) * per && b < blocks; ++b) {
    roc += partials[2 * b];
    pr += partials[2 * b + 1];
  }
  roc = block_sum(roc);
  pr = block_sum(pr);
  if (threadIdx.x == 0) {
    out[0] = roc;
    out[1] = pr;
  }
}

}  // namespace

size_t bin_sort_tile_words(long long n) { return 256 * (size_t)tiles_of(n); }
size_t bin_runs_tile_words(long long n) { return 3 * (size_t)tiles_of(n); }
int bin_area_blocks(long long K) { return (int)((K + 1 + kTile - 1) / kTile); }

cudaError_t bin_sort_pairs(unsigned long long *keys[2], void *vals[2], int val_bytes, long long n, unsigned *hist,
                           unsigned *tiles, int *which, int *passes, cudaStream_t st) {
  *which = 0;
  *passes = 0;
  if (val_bytes != 1 && val_bytes != 4) return cudaErrorInvalidValue;
  if (n <= 1) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(hist, 0, 8 * 256 * sizeof(unsigned), st);
  if (e != cudaSuccess) return e;
  long long g = (n + kThreads - 1) / kThreads;
  if (g > 1024) g = 1024;
  bin_hist8_kernel<<<(unsigned)g, kThreads, 0, st>>>(keys[0], n, hist);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  unsigned h[8 * 256];
  if ((e = cudaMemcpyAsync(h, hist, sizeof h, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
  const long long T = tiles_of(n);
  int cur = 0;
  for (int p = 0; p < 8; ++p) {
    bool constant = false;
    for (int b = 0; b < 256 && !constant; ++b) constant = h[p * 256 + b] == (unsigned)n;
    if (constant) continue;   // the identity permutation
    const int shift = 8 * p;
    bin_count_kernel<<<(unsigned)T, kThreads, 0, st>>>(keys[cur], n, shift, tiles, T);
    bin_offsets_kernel<<<256, kThreads, 0, st>>>(tiles, T, hist + p * 256);
    if (val_bytes == 1)
      bin_scatter_kernel<uint8_t><<<(unsigned)T, kThreads, 0, st>>>(keys[cur], (const uint8_t *)vals[cur], keys[cur ^ 1],
                                                                    (uint8_t *)vals[cur ^ 1], n, shift, tiles, T);
    else
      bin_scatter_kernel<uint32_t><<<(unsigned)T, kThreads, 0, st>>>(keys[cur], (const uint32_t *)vals[cur], keys[cur ^ 1],
                                                                     (uint32_t *)vals[cur ^ 1], n, shift, tiles, T);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    cur ^= 1;
    ++*passes;
  }
  *which = cur;
  return cudaSuccess;
}

cudaError_t bin_runs_launch(const unsigned long long *keys, const void *vals, int val_bytes, const long long *upos,
                            const long long *uneg, long long n, long long *tile_sums, BinRec *out, long long *n_out,
                            cudaStream_t st) {
  if (n <= 0) return cudaMemsetAsync(n_out, 0, sizeof(long long), st);
  if (val_bytes == 1) return runs(keys, ClassVals{(const uint8_t *)vals}, n, tile_sums, out, n_out, st);
  if (val_bytes == 4) return runs(keys, IndexVals{(const uint32_t *)vals, upos, uneg}, n, tile_sums, out, n_out, st);
  return cudaErrorInvalidValue;
}

cudaError_t bin_union_prep_launch(const BinRec *blocks, long long stride, const long long *off, int world, long long total,
                                  unsigned long long *keys, uint32_t *idx, long long *upos, long long *uneg, cudaStream_t st) {
  if (total <= 0) return cudaSuccess;
  long long g = (total + kThreads - 1) / kThreads;
  if (g > 4096) g = 4096;
  bin_union_prep_kernel<<<(unsigned)g, kThreads, 0, st>>>(blocks, stride, off, world, total, keys, idx, upos, uneg);
  return cudaGetLastError();
}

cudaError_t bin_areas_launch(const BinRec *recs, long long K, double *partials, double *out, cudaStream_t st) {
  if (K <= 0) return cudaErrorInvalidValue;
  const int nb = bin_area_blocks(K);
  bin_area_kernel<<<nb, kThreads, 0, st>>>(recs, K, partials);
  bin_area_final_kernel<<<1, kThreads, 0, st>>>(partials, nb, out);
  return cudaGetLastError();
}

}  // namespace agd
