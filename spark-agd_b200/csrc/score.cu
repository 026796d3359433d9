// score.cu -- scoring sweeps over a resident shard (sm_90a): the margins m_i = x_i . w + b of a row range, and the
// AGD_EVAL_* sums of one shard (count, loss, confusion counts, error and label moments).
//
// A second, simpler read of the shards K1 sweeps: no gradient, so X is streamed once with no reuse and nothing is written
// back but one margin per row or one slab of AGD_EVAL_N sums per CTA.
//   * dense: a group of G lanes owns a row (G = the smallest power of two >= the 16-byte vectors of a row, at most 32, so
//     narrow rows put several rows in one warp); lane l of the group takes vectors l, l + G, ... with 128-bit streaming
//     loads, widens every element to fp64 and accumulates x * w with DFMA in column order, then the group adds its lanes
//     with a fixed xor butterfly.  G depends on d only, so a margin depends on the row, w, b and d -- never on where the
//     row sits, which range was asked for, or how many devices / ranks hold the matrix.  w lives in shared memory when it
//     fits (generic loads then hit shared memory), otherwise it is read through L1 / L2.
//   * CSR: a group of 8 lanes owns a row; lane l takes the row's stored entries l, l + 8, ... (the row's own entries, in
//     storage order, as mllib's sparse dot does), gathers w[idx] through the read-only path, and the same butterfly adds.
//   * the evaluation form accumulates the AGD_EVAL_N sums per thread, adds them over the CTA in a fixed order and writes
//     one slab per CTA; k1_reduce_launch then adds the slabs in a fixed order, so repeated calls return identical bits
//     (also on CSR shards, where K1 scatters with RED.ADD).
// Non-finite features follow IEEE arithmetic: nothing is skipped (0 * inf = NaN, as ddot gives).
//   * the key form (agd_binary_curve) writes, for every row of the view whose margin is not NaN, the 64-bit descending-order
//     key of the margin (margin_key, agd_common.cuh) and the row's class (label > 0.5), compacted by one atomic per warp and
//     step; NaN margins are only counted.  The margin is the G-lane margin above, so a key carries agd_margins' bits.
// On a view (agd_set_row_filter) the evaluation and key forms treat a row outside it as past the end of the shard: its loads are
// never issued, so it leaves no trace in the sums, and a held-out view reads only its own rows' lines of X.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

constexpr int kScoreThreads = 256;
enum { kScoreMargins = 0, kScoreEval = 1, kScoreKeys = 2 };   // the three forms of the scoring sweeps
constexpr int kCsrGroup = 8;                 // lanes per CSR row
// w (fp64) lives in dynamic shared memory when it fits beside the evaluation form's static reduction array within the
// 48 KB a block gets without an opt-in: up to d = 6056
constexpr int kEvalRedBytes = (kScoreThreads / 32) * AGD_EVAL_N * (int)sizeof(double);
constexpr int kScoreWSmemMax = (48 * 1024 - kEvalRedBytes) / (int)sizeof(double);

// 16 bytes of X, streamed: no L1 allocation, 256-byte L2 prefetch
__device__ __forceinline__ uint4 ld_stream(const void *p) {
  uint4 v;
  asm("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
      : "l"(p));
  return v;
}

template <typename T> struct ScoreElem;
template <> struct ScoreElem<float> {
  static constexpr int EPV = 4;
  __device__ static double one(const float *p) { return (double)*p; }
  __device__ static void vec(const uint4 &r, double (&o)[4]) {
    o[0] = (double)__uint_as_float(r.x); o[1] = (double)__uint_as_float(r.y);
    o[2] = (double)__uint_as_float(r.z); o[3] = (double)__uint_as_float(r.w);
  }
};
template <> struct ScoreElem<double> {
  static constexpr int EPV = 2;
  __device__ static double one(const double *p) { return *p; }
  __device__ static void vec(const uint4 &r, double (&o)[2]) {
    o[0] = __hiloint2double((int)r.y, (int)r.x);
    o[1] = __hiloint2double((int)r.w, (int)r.z);
  }
};
template <> struct ScoreElem<__nv_bfloat16> {
  static constexpr int EPV = 8;
  __device__ static double one(const __nv_bfloat16 *p) { return (double)__bfloat162float(*p); }
  __device__ static void vec(const uint4 &r, double (&o)[8]) {   // a bf16 is the upper half of an fp32
    const uint32_t wds[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      o[2 * i] = (double)__uint_as_float(wds[i] << 16);
      o[2 * i + 1] = (double)__uint_as_float(wds[i] & 0xffff0000u);
    }
  }
};

// one row's contribution to the AGD_EVAL_* sums; the loss is K1's own loss_eval, with the intercept inside m
__device__ __forceinline__ void eval_row(double (&s)[AGD_EVAL_N], int kind, double thr, double m, double y) {
  double mult, loss;
  loss_eval(kind, m, y, mult, loss);
  s[AGD_EVAL_COUNT] += 1.0;
  s[AGD_EVAL_LOSS] += loss;
  // binary predictPoint of LogisticRegressionModel / SVMModel (mllib 1.3.0), on rows labelled exactly 0 or 1
  if ((kind == AGD_GRAD_LOGISTIC || kind == AGD_GRAD_HINGE) && (y == 0.0 || y == 1.0)) {
    const bool pos = kind == AGD_GRAD_LOGISTIC ? (1.0 / (1.0 + exp(-m)) > thr) : (m > thr);
    const bool one = y == 1.0;
    s[AGD_EVAL_TP] += (pos && one) ? 1.0 : 0.0;
    s[AGD_EVAL_FP] += (pos && !one) ? 1.0 : 0.0;
    s[AGD_EVAL_TN] += (!pos && !one) ? 1.0 : 0.0;
    s[AGD_EVAL_FN] += (!pos && one) ? 1.0 : 0.0;
  }
  const double e = m - y;
  s[AGD_EVAL_SUM_ERR] += e;
  s[AGD_EVAL_SUM_ERR2] += e * e;
  s[AGD_EVAL_SUM_ABS_ERR] += fabs(e);
  s[AGD_EVAL_SUM_Y] += y;
  s[AGD_EVAL_SUM_Y2] += y * y;
}

// the CTA's sums -> slab[blockIdx.x] in a fixed order (xor butterfly per warp, then the warps in index order)
__device__ __forceinline__ void eval_flush(double (&s)[AGD_EVAL_N], double *slabs) {
  __shared__ double red[kScoreThreads / 32][AGD_EVAL_N];
  static_assert(sizeof(red) == kEvalRedBytes, "kScoreWSmemMax leaves room for this array");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < AGD_EVAL_N; ++k) {
    double v = s[k];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < AGD_EVAL_N) {
    double t = 0.0;
#pragma unroll
    for (int wi = 0; wi < kScoreThreads / 32; ++wi) t += red[wi][threadIdx.x];
    slabs[(size_t)blockIdx.x * AGD_EVAL_N + threadIdx.x] = t;
  }
}

// group butterfly over the G lanes of a row group (G a power of two; every lane of the warp takes part)
__device__ __forceinline__ double group_sum(double v, int G) {
  for (int off = G >> 1; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// R rows per row group and step: one load of w serves R rows, and R rows of loads are in flight per lane
template <typename T> struct ScoreRows { static constexpr int R = 4; };

// key form: every lane of the warp calls it (the row loops are warp-uniform); `ok` rows with a non-NaN margin are appended
// to keys / classes, NaN margins are counted
__device__ __forceinline__ void key_emit(const ScoreArgs &a, bool ok, double m, double y) {
  const bool nan = ok && m != m, emit = ok && !nan;
  const unsigned em = __ballot_sync(0xffffffffu, emit), nm = __ballot_sync(0xffffffffu, nan);
  const int lane = threadIdx.x & 31;
  unsigned base = 0;
  if (lane == 0 && em) base = atomicAdd(a.counters, (unsigned)__popc(em));
  if (lane == 0 && nm) atomicAdd(a.counters + 1, (unsigned)__popc(nm));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (emit) {
    const unsigned i = base + __popc(em & ((1u << lane) - 1u));
    a.keys[i] = margin_key(m);
    a.classes[i] = y > 0.5 ? 1 : 0;
  }
}

template <typename T, bool VEC, int MODE>
__global__ void __launch_bounds__(kScoreThreads, 2) score_dense_kernel(const ScoreArgs a, const int G, const int w_smem) {
  extern __shared__ __align__(16) double w_sh[];
  constexpr int EPV = VEC ? ScoreElem<T>::EPV : 1;
  constexpr int R = ScoreRows<T>::R;
  constexpr bool EVAL = MODE == kScoreEval, VIEWED = MODE != kScoreMargins;
  const int lane = threadIdx.x & 31;
  const double *w = a.w;
  if (w_smem) {
    for (int c = threadIdx.x; c < a.d; c += kScoreThreads) w_sh[c] = a.w[c];
    __syncthreads();
    w = w_sh;
  }
  const int g = lane / G, l = lane & (G - 1);
  const int groups = 32 / G;
  const long long step_rows = (long long)groups * R;   // rows one warp covers per step
  const long long warp0 = (long long)blockIdx.x * (kScoreThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kScoreThreads / 32);
  const int nunit = a.d / EPV;
  const T *X = reinterpret_cast<const T *>(a.X);
  double s[AGD_EVAL_N];
#pragma unroll
  for (int k = 0; k < AGD_EVAL_N; ++k) s[k] = 0.0;
  for (long long base = warp0 * step_rows; base < a.rows; base += nwarps * step_rows) {
    long long row[R];
    bool ok[R];
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      row[r] = base + (long long)r * groups + g;
      ok[r] = row[r] < a.rows && (!VIEWED || row_in_view(a.filt, a.row_base + a.row0 + row[r]));
      acc[r] = 0.0;
    }
    const T *xr[R];
    double yv[R];   // labels fetched ahead of the row tails
#pragma unroll
    for (int r = 0; r < R; ++r) {
      xr[r] = X + (size_t)(a.row0 + (ok[r] ? row[r] : 0)) * a.d;
      yv[r] = (VIEWED && ok[r]) ? __ldg(a.labels + a.row0 + row[r]) : 0.0;
    }
#pragma unroll 2
    for (int u = l; u < nunit; u += G) {
      if (VEC) {
        uint4 raw[R];
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ok[r]) raw[r] = ld_stream(xr[r] + (size_t)u * EPV);
        double wv[EPV];
#pragma unroll
        for (int e = 0; e < EPV; e += 2) {
          const double2 p = *reinterpret_cast<const double2 *>(w + (size_t)u * EPV + e);
          wv[e] = p.x;
          wv[e + 1] = p.y;
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ok[r]) {
            double xv[ScoreElem<T>::EPV];
            ScoreElem<T>::vec(raw[r], xv);
#pragma unroll
            for (int e = 0; e < EPV; ++e) acc[r] = fma(xv[e], wv[e], acc[r]);
          }
      } else {
        const double wc = w[u];
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ok[r]) acc[r] = fma(ScoreElem<T>::one(xr[r] + u), wc, acc[r]);
      }
    }
    double m[R];
#pragma unroll
    for (int r = 0; r < R; ++r) m[r] = group_sum(acc[r], G) + a.b;
    if (G >= R) {  // lane r of the group finishes row r: the R row tails (loss, exp) run side by side
      double mm = m[0], y = yv[0];
      long long rr = row[0];
      bool o = ok[0];
#pragma unroll
      for (int r = 1; r < R; ++r)
        if (l == r) { mm = m[r]; y = yv[r]; rr = row[r]; o = ok[r]; }
      if constexpr (MODE == kScoreKeys) {
        key_emit(a, l < R && o, mm, y);
      } else {
        if (l < R && o) {
          if (EVAL) eval_row(s, a.kind, a.threshold, mm, y);
          else a.margins[rr] = mm;
        }
      }
    } else {
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if constexpr (MODE == kScoreKeys) {
          key_emit(a, ok[r] && l == 0, m[r], yv[r]);
        } else {
          if (ok[r] && l == 0) {
            if (EVAL) eval_row(s, a.kind, a.threshold, m[r], yv[r]);
            else a.margins[row[r]] = m[r];
          }
        }
      }
    }
  }
  if (EVAL) eval_flush(s, a.slabs);
}

template <typename T, int MODE>
__global__ void __launch_bounds__(kScoreThreads) score_csr_kernel(const ScoreArgs a) {
  constexpr int G = kCsrGroup, groups = 32 / G;
  constexpr bool EVAL = MODE == kScoreEval, VIEWED = MODE != kScoreMargins;
  const int lane = threadIdx.x & 31, g = lane / G, l = lane & (G - 1);
  const long long warp0 = (long long)blockIdx.x * (kScoreThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kScoreThreads / 32);
  const T *val = reinterpret_cast<const T *>(a.val);
  double s[AGD_EVAL_N];
#pragma unroll
  for (int k = 0; k < AGD_EVAL_N; ++k) s[k] = 0.0;
  for (long long base = warp0 * groups; base < a.rows; base += nwarps * groups) {
    const long long row = base + g;
    const bool ok = row < a.rows && (!VIEWED || row_in_view(a.filt, a.row_base + a.row0 + row));
    double acc = 0.0;
    if (ok) {
      const long long r = a.row0 + row;
      const long long k0 = __ldg(a.rowptr + r), k1 = __ldg(a.rowptr + r + 1);
#pragma unroll 4
      for (long long k = k0 + l; k < k1; k += G) acc = fma(ScoreElem<T>::one(val + k), __ldg(a.w + __ldg(a.idx + k)), acc);
    }
    const double m = group_sum(acc, G) + a.b;
    if constexpr (MODE == kScoreKeys) key_emit(a, ok && l == 0, m, (ok && l == 0) ? a.labels[a.row0 + row] : 0.0);
    else if (ok && l == 0) {
      if (EVAL) eval_row(s, a.kind, a.threshold, m, a.labels[a.row0 + row]);
      else a.margins[row] = m;
    }
  }
  if (EVAL) eval_flush(s, a.slabs);
}

// occupancy-sized grid; a configuration that cannot run even one block per SM is an error, not a smaller grid
template <typename K>
cudaError_t persistent_grid(K kern, int smem, int sm_count, long long rows, long long rows_per_cta, int *grid_out) {
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kScoreThreads, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  long long grid = (long long)per_sm * sm_count;
  if (grid > score_max_blocks(sm_count)) grid = score_max_blocks(sm_count);
  const long long need = (rows + rows_per_cta - 1) / rows_per_cta;
  if (grid > need) grid = need;
  *grid_out = (int)grid;
  return cudaSuccess;
}

template <typename T, bool VEC, int MODE>
cudaError_t launch_dense(const ScoreArgs &a, int sm_count, int *blocks_out) {
  constexpr int EPV = VEC ? ScoreElem<T>::EPV : 1;
  const int nunit = a.d / EPV;
  int G = 1;
  while (G < nunit && G < 32) G <<= 1;
  const int w_smem = a.d <= kScoreWSmemMax ? 1 : 0;
  const int smem = w_smem ? a.d * (int)sizeof(double) : 0;
  auto kern = score_dense_kernel<T, VEC, MODE>;
  int grid = 0;
  const cudaError_t e =
      persistent_grid(kern, smem, sm_count, a.rows, (long long)(kScoreThreads / 32) * (32 / G) * ScoreRows<T>::R, &grid);
  if (e != cudaSuccess) return e;
  *blocks_out = grid;
  kern<<<grid, kScoreThreads, smem, a.stream>>>(a, G, w_smem);
  return cudaGetLastError();
}

template <typename T, int MODE>
cudaError_t launch_dense_t(const ScoreArgs &a, int sm_count, int *blocks_out) {
  if ((a.d * sizeof(T)) % 16 == 0) return launch_dense<T, true, MODE>(a, sm_count, blocks_out);
  return launch_dense<T, false, MODE>(a, sm_count, blocks_out);
}

template <int MODE>
cudaError_t launch_any(const ScoreArgs &a, int elem_bytes, int sm_count, int *blocks_out) {
  *blocks_out = 0;
  if (a.rows <= 0) return cudaSuccess;
  if (a.rowptr) {
    if (elem_bytes != 4 && elem_bytes != 8) return cudaErrorInvalidValue;
    auto kern = elem_bytes == 8 ? score_csr_kernel<double, MODE> : score_csr_kernel<float, MODE>;
    int grid = 0;
    const cudaError_t e = persistent_grid(kern, 0, sm_count, a.rows, (long long)(kScoreThreads / 32) * (32 / kCsrGroup), &grid);
    if (e != cudaSuccess) return e;
    *blocks_out = grid;
    kern<<<grid, kScoreThreads, 0, a.stream>>>(a);
    return cudaGetLastError();
  }
  if (elem_bytes == 2) return launch_dense_t<__nv_bfloat16, MODE>(a, sm_count, blocks_out);
  if (elem_bytes == 4) return launch_dense_t<float, MODE>(a, sm_count, blocks_out);
  if (elem_bytes == 8) return launch_dense_t<double, MODE>(a, sm_count, blocks_out);
  return cudaErrorInvalidValue;
}

// which rows of a range pass a view: the predicate the K1 and evaluation sweeps apply, one row per thread
__global__ void __launch_bounds__(kScoreThreads) row_filter_mask_kernel(const RowFilter *f, long long row_base, int64_t rows,
                                                                       uint8_t *out) {
  for (long long i = blockIdx.x * (long long)kScoreThreads + threadIdx.x; i < rows; i += (long long)gridDim.x * kScoreThreads)
    out[i] = row_in_view(f, row_base + i) ? 1 : 0;
}

// the same predicate packed 32 rows to a word: one row per thread, a warp's ballot is one word
__global__ void __launch_bounds__(kScoreThreads) row_filter_bits_kernel(const RowFilter *f, long long row_base, int64_t rows,
                                                                       uint32_t *bits) {
  const long long stride = (long long)gridDim.x * kScoreThreads;
  for (long long i = blockIdx.x * (long long)kScoreThreads + threadIdx.x; i - (threadIdx.x & 31) < rows; i += stride) {
    const uint32_t word = __ballot_sync(0xffffffffu, i < rows && row_in_view(f, row_base + i));
    if ((threadIdx.x & 31) == 0) bits[i >> 5] = word;
  }
}

}  // namespace

cudaError_t row_filter_bits_launch(const RowFilter *f, long long row_base, int64_t rows, uint32_t *bits, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  long long grid = (rows + kScoreThreads - 1) / kScoreThreads;
  if (grid > 4096) grid = 4096;
  row_filter_bits_kernel<<<(unsigned)grid, kScoreThreads, 0, st>>>(f, row_base, rows, bits);
  return cudaGetLastError();
}

cudaError_t row_filter_mask_launch(const RowFilter *f, long long row_base, int64_t rows, uint8_t *out, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  long long grid = (rows + kScoreThreads - 1) / kScoreThreads;
  if (grid > 4096) grid = 4096;
  row_filter_mask_kernel<<<(unsigned)grid, kScoreThreads, 0, st>>>(f, row_base, rows, out);
  return cudaGetLastError();
}

int score_max_blocks(int sm_count) { return 8 * sm_count; }

cudaError_t score_margins_launch(const ScoreArgs &a, int elem_bytes, int sm_count) {
  int blocks = 0;
  return launch_any<kScoreMargins>(a, elem_bytes, sm_count, &blocks);
}

cudaError_t score_eval_launch(const ScoreArgs &a, int elem_bytes, int sm_count, int *blocks_out) {
  return launch_any<kScoreEval>(a, elem_bytes, sm_count, blocks_out);
}

cudaError_t score_keys_launch(const ScoreArgs &a, int elem_bytes, int sm_count) {
  int blocks = 0;
  return launch_any<kScoreKeys>(a, elem_bytes, sm_count, &blocks);
}

}  // namespace agd
