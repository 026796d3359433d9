// k1_dense.cu -- K1: fused row-block gradient kernel for dense shards (sm_90a).
//
// One launch = the seqOp fold of applySmooth (AGD.scala:197-200) over one GPU's shard:
//   m_i = x_i . w            (BLAS.dot inside Gradient.compute [mllib-1.3.0], call site AGD.scala:198)
//   (mult_i, loss_i) = loss'(m_i, y_i)   (LogisticGradient / LeastSquaresGradient / HingeGradient)
//   g += mult_i * x_i        (BLAS.axpy into cumGradient),  loss += loss_i
// with X read from HBM exactly once.  X is stored fp32 or fp64; every product and every sum is fp64
// (the driver loop branches on catastrophically cancelling fp64 quantities, AGD.scala:273-281,327).
//
// k1_ring_kernel (hot path, d*sizeof(T) a multiple of 16 and d <= 1024 vectors/row):
//   * 32 KB row tiles stream HBM -> shared memory with TMA bulk copies (cp.async.bulk + mbarrier
//     complete_tx) through an S-stage ring, labels ride along; a stage is refilled right behind the
//     CTA barrier that follows its last read;
//   * w is staged once per CTA with the same TMA path, then lives in registers;
//   * 256 consumer threads: thread t of a row group owns 128-bit column vectors {t, t+TPR, ...};
//     it pulls its R x V vectors of the tile out of shared memory (LDS.128), converts once to fp64,
//     forms R partial dots, warp-shuffle transpose-reduces them, one rotating "scalar" warp finishes
//     the margins and evaluates loss', and the retained fp64 tile is then accumulated into the
//     thread's private column sums (no atomics);
//   * per-CTA column sums go to a slab; k1_reduce_kernel adds the slabs in fixed order.
// k1_generic_kernel: any (rows, d), scalar loads, slab accumulators in global memory (L2-resident).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "agd_common.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

constexpr int kConsumers = 256;
constexpr int kMaxTileRows = 32;

template <typename T> struct Elem;
template <> struct Elem<float> { static constexpr int EPV = 4; };
template <> struct Elem<double> { static constexpr int EPV = 2; };
template <> struct Elem<__nv_bfloat16> { static constexpr int EPV = 8; };

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

template <typename T, int EPV>
__device__ __forceinline__ void cvt_vec(const uint4 &raw, double (&out)[EPV]);
template <>
__device__ __forceinline__ void cvt_vec<float, 4>(const uint4 &raw, double (&out)[4]) {
  out[0] = (double)__uint_as_float(raw.x);
  out[1] = (double)__uint_as_float(raw.y);
  out[2] = (double)__uint_as_float(raw.z);
  out[3] = (double)__uint_as_float(raw.w);
}
template <>
__device__ __forceinline__ void cvt_vec<double, 2>(const uint4 &raw, double (&out)[2]) {
  out[0] = __hiloint2double((int)raw.y, (int)raw.x);
  out[1] = __hiloint2double((int)raw.w, (int)raw.z);
}

template <>
__device__ __forceinline__ void cvt_vec<__nv_bfloat16, 8>(const uint4 &raw, double (&out)[8]) {
  // a bf16 is the upper half of an fp32: widen with a shift / mask, then F2F to fp64
  const uint32_t wds[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    out[2 * i] = (double)__uint_as_float(wds[i] << 16);
    out[2 * i + 1] = (double)__uint_as_float(wds[i] & 0xffff0000u);
  }
}

__host__ __device__ inline uint32_t round_up_u32(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

// shared-memory carve-up (identical on host and device)
struct RingLayout {
  uint32_t stage_stride, aux_off, partial_off, partial2_off, mult_off, mult2_off, red_off, cnt_off, skip_off, bars_off, total;
};
// mode: 0 = one point; 1 = the launch also evaluates the LOSS at a second point w2 (pass fusion of the history evaluation);
// 2 = loss AND gradient at w2 (the speculative sweep of the memoised pass structure).  aux holds w (and w2) in the
// conflict-free plane layout described at the kernel.
__host__ __device__ inline RingLayout ring_layout(uint32_t tile_bytes, uint32_t aux_bytes, int stages, int mode) {
  RingLayout L;
  L.stage_stride = round_up_u32(tile_bytes, 128);
  L.aux_off = L.stage_stride * stages;
  L.partial_off = L.aux_off + round_up_u32(aux_bytes, 128);
  L.partial2_off = L.partial_off + kMaxTileRows * 8 * 8;
  L.mult_off = L.partial2_off + (mode ? kMaxTileRows * 8 * 8 : 0);
  L.mult2_off = L.mult_off + kMaxTileRows * 8;
  L.red_off = L.mult2_off + (mode == 2 ? kMaxTileRows * 8 : 0);
  L.cnt_off = L.red_off + 32 * 8;
  L.skip_off = L.cnt_off + round_up_u32(stages * 4, 8);
  L.bars_off = L.skip_off + 8;
  L.total = L.bars_off + (stages + 1) * 8;
  return L;
}

// Row permutation that makes the warp transpose-reduce select-free: register r of a lane holds tile row r ^ row_perm<R>(lane).
// Level (bit, width) of warp_rows_reduce_perm pairs lane L with L ^ bit and folds registers i and i + width; because the
// partner's permutation differs exactly in `width`, its register i + width holds the SAME row as this lane's register i,
// so every level is "p[i] += shfl_xor(p[i + width])" with no lane-dependent selects (4 FSEL per pair before).
template <int R>
__device__ __forceinline__ int row_perm(int lane) {
  int m = 0, bit = 16;
#pragma unroll
  for (int width = R / 2; width >= 1; width >>= 1, bit >>= 1) m |= (lane & bit) ? width : 0;
  return m;
}
// afterwards every lane holds the warp total of row row_perm<R>(lane); the pairings -- and therefore the bits -- are those of
// warp_rows_reduce (k1_device.cuh)
template <int R>
__device__ __forceinline__ double warp_rows_reduce_perm(double (&p)[R]) {
  int bit = 16;
#pragma unroll
  for (int width = R / 2; width >= 1; width >>= 1, bit >>= 1) {
#pragma unroll
    for (int i = 0; i < width; ++i) p[i] = p[i] + __shfl_xor_sync(0xffffffffu, p[i + width], bit);
  }
  double tot = p[0];
  for (; bit >= 1; bit >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, bit);
  return tot;
}

// ---------------------------------------------------------------- the hot kernel
template <typename T, int NT, int TPR, int V, int R, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB)
k1_ring_kernel(const K1Args a, const int nvec, const long long ntiles, const uint32_t aux_bytes) {
  constexpr int EPV = Elem<T>::EPV;
  constexpr int NG = NT / TPR;          // row groups per CTA
  constexpr int WPG = TPR / 32;         // warps per row group
  constexpr int TR = NG * R;            // rows per tile
  constexpr int NW = NT / 32;
  constexpr bool DUAL = MODE != 0;      // a second point rides along (its loss; with MODE == 2 its gradient too)
  constexpr int NP = DUAL ? 2 : 1;      // points per sweep
  constexpr int NCH = EPV / 2;          // 16-byte chunks per fp64-widened vector
  static_assert(TR <= kMaxTileRows && TR % 2 == 0 && (NW & (NW - 1)) == 0, "tile rows / warps");
  // DUAL: lanes 0-15 of the scalar warp evaluate the rows at w, lanes 16-31 the same rows at w2
  static_assert(!DUAL || TR <= 16, "pass fusion needs the tile's rows twice in one warp");
  // One accumulator set per point in every mode, so a point's sums do not depend on which sweep form evaluated it (the
  // fused / memoised / plain pass structures agree bit for bit).  Round 1 kept two sets (even / odd rows) for narrow threads;
  // measured on the headline shard (tools/k1_modes.py, same box): one-point 7.11 -> 7.27 ms without them, two-point equal,
  // and the two-gradient sweep 10.05 -> 9.15 ms because its four sets spilled.
  extern __shared__ __align__(128) unsigned char smem[];

  const int S = a.stages;
  const uint32_t row_bytes = (uint32_t)a.d * (uint32_t)sizeof(T);
  const RingLayout L = ring_layout(TR * row_bytes + kMaxTileRows * 8, aux_bytes, S, MODE);  // rows, then their labels
  unsigned char *aux = smem + L.aux_off;                               // w [and w2] planes; reused for the row-group reduce
  double *partial = reinterpret_cast<double *>(smem + L.partial_off);  // [TR][8]
  double *partial2 = reinterpret_cast<double *>(smem + L.partial2_off);  // [TR][8] at w2 (DUAL)
  double *mult_s = reinterpret_cast<double *>(smem + L.mult_off);      // [TR]
  double *mult2_s = reinterpret_cast<double *>(smem + L.mult2_off);    // [TR] at w2 (MODE 2)
  double *red = reinterpret_cast<double *>(smem + L.red_off);
  unsigned int *cnt = reinterpret_cast<unsigned int *>(smem + L.cnt_off);  // [S] warps done with the stage (diagnostic modes)
  uint32_t *skip_s = reinterpret_cast<uint32_t *>(smem + L.skip_off);      // the tile's rows that must add nothing (below)
  const uint32_t bars = smem_u32(smem + L.bars_off);                   // full[s] = bars + 8*s ; wbar = bars + 8*S
  const uint32_t wbar = bars + 8u * S;
  const unsigned char *Xb = reinterpret_cast<const unsigned char *>(a.X);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // TMA fill of ring slot (kk % S) with this CTA's kk-th tile
  auto fill = [&](long long kk, int s) {
    const long long tile = blockIdx.x + kk * (long long)gridDim.x;
    if (tile >= ntiles) return;
    const long long row0 = tile * TR;
    const long long left = a.rows - row0;
    const uint32_t rv = left < TR ? (uint32_t)left : (uint32_t)TR;
    const uint32_t full = bars + 8u * s;
    const uint32_t lbytes = round_up_u32(rv * 8u, 16u);  // label arrays are padded, row0 is even
    mbar_expect_tx(full, rv * row_bytes + lbytes);
    tma_bulk_g2s(smem_u32(smem + (size_t)s * L.stage_stride), Xb + (size_t)row0 * row_bytes, rv * row_bytes, full);
    tma_bulk_g2s(smem_u32(smem + (size_t)s * L.stage_stride + TR * row_bytes), a.labels + row0, lbytes, full);
  };
  // one point's share of the w staging area: TPR * V vectors of EPV doubles (>= d doubles: columns past d are zero weights)
  constexpr uint32_t kPointBytes = (uint32_t)TPR * V * EPV * 8u;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bars + 8u * s, 1);
      cnt[s] = 0u;
    }
    mbar_init(wbar, 1);
    mbar_fence_init();
    mbar_expect_tx(wbar, (uint32_t)a.d * 8u * NP);
    tma_bulk_g2s(smem_u32(aux), a.w, (uint32_t)a.d * 8u, wbar);  // w: TMA-staged once per CTA
    if (DUAL) tma_bulk_g2s(smem_u32(aux + kPointBytes), a.w2, (uint32_t)a.d * 8u, wbar);
    for (int s = 0; s < S; ++s) fill(s, s);
  }
  __syncthreads();

  const int g = tid / TPR, t = tid % TPR, wig = t >> 5;
  const bool full_row = nvec == V * TPR && a.tune_full == 0;
  const int rperm = row_perm<R>(lane);   // register r of this lane holds tile row g * R + (r ^ rperm)
  mbar_wait(wbar, 0);
  // Re-lay w (and w2) out once per CTA, in place through registers, from the linear order TMA delivered into PLANES: chunk c
  // (16 bytes = 2 doubles) of vector v of point q for thread t sits at ((v * NCH + c) * NP + q) * TPR + t.  The per-tile
  // re-read (w is not kept live across phase 2) is then one conflict-free LDS.128 per chunk -- in the linear order a thread's
  // 32-byte stride made every such read a 2-way bank conflict -- and columns past d read as exact zeros without predicates.
  {
    double wtmp[NP][V][EPV];
    if (tid < TPR) {
#pragma unroll
      for (int q = 0; q < NP; ++q)
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const int vec = v * TPR + t;
#pragma unroll
          for (int e = 0; e < EPV; ++e)
            wtmp[q][v][e] = vec < nvec ? reinterpret_cast<const double *>(aux + q * kPointBytes)[vec * EPV + e] : 0.0;
        }
    }
    __syncthreads();
    if (tid < TPR) {
#pragma unroll
      for (int q = 0; q < NP; ++q)
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
          for (int c = 0; c < NCH; ++c)
            *reinterpret_cast<double2 *>(aux + ((size_t)((v * NCH + c) * NP + q) * TPR + t) * 16) =
                make_double2(wtmp[q][v][2 * c], wtmp[q][v][2 * c + 1]);
    }
    __syncthreads();
  }
  double acc[V][EPV], accB[MODE == 2 ? V : 1][MODE == 2 ? EPV : 1];   // gradient at w; at w2 (MODE 2)
#pragma unroll
  for (int v = 0; v < V; ++v)
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      acc[v][e] = 0.0;
      if (MODE == 2) accB[MODE == 2 ? v : 0][MODE == 2 ? e : 0] = 0.0;
    }
  double lossacc = 0.0, cntacc = 0.0;
  const int rv_last = (int)(a.rows - (ntiles - 1) * TR);

  int k = 0, s = -1;
  uint32_t par = 1;
  const int ntiles32 = (int)ntiles, last_tile = ntiles32 - 1, tile_step = (int)gridDim.x;  // the launch keeps ntiles < 2^31
  for (int tile = blockIdx.x; tile < ntiles32; tile += tile_step, ++k) {
    if (++s == S) s = 0;          // ring slot and its mbarrier phase, kept incrementally
    if (s == 0) par ^= 1u;
    const int rv = (tile == last_tile) ? rv_last : TR;  // only the shard's last tile can be ragged
    const int sw = k & (NW - 1);  // this tile's scalar warp
    mbar_wait(bars + 8u * s, par);
    // labels ride in the stage: no warp ever waits on a global load inside the loop
    const int srow = DUAL ? (lane & 15) : lane;   // the tile row this lane of the scalar warp evaluates
    // every lane of the scalar warp runs the evaluation (the label / partial-dot arrays have kMaxTileRows entries, lanes
    // without a row read stale values and are masked by row_ok), so nothing needs initialising on the other warps
    const bool sactive = warp == sw;
    double ylab = 0.0;
    if (sactive)
      ylab = *reinterpret_cast<const double *>(smem + (size_t)s * L.stage_stride + TR * row_bytes + srow * 8);

    // pull this thread's R x V vectors out of the stage and widen them to fp64 once
    double xd[R][V][EPV];
    const unsigned char *stage = smem + (size_t)s * L.stage_stride;
    if (full_row) {  // every thread owns V whole vectors of the row (d = 1024 fp32 ...): no predicates, no zero fill
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const uint4 raw = *reinterpret_cast<const uint4 *>(stage + (size_t)(g * R + (r ^ rperm)) * row_bytes + (size_t)(v * TPR + t) * 16);
          cvt_vec<T, EPV>(raw, xd[r][v]);
        }
    } else {
#pragma unroll
      for (int r = 0; r < R; ++r) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const int vec = v * TPR + t;
          uint4 raw = make_uint4(0u, 0u, 0u, 0u);
          if (vec < nvec) raw = *reinterpret_cast<const uint4 *>(stage + (size_t)(g * R + (r ^ rperm)) * row_bytes + (size_t)vec * 16);
          cvt_vec<T, EPV>(raw, xd[r][v]);
        }
      }
    }
    if (rv < TR) {  // ragged last tile: rows past the shard hold stale bytes
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (g * R + (r ^ rperm) >= rv) {
#pragma unroll
          for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < EPV; ++e) xd[r][v][e] = 0.0;
        }
    }
    // this tile's weights out of the planes (conflict-free LDS.128).  Threads that own few columns (V * EPV <= 4) fetch them
    // up front; wide threads fetch each 16-byte chunk right where phase 1 consumes it (kJit), which keeps them spill-free.
    auto wplane = [&](int q, int v, int c) {
      return *reinterpret_cast<const double2 *>(aux + ((size_t)((v * NCH + c) * NP + q) * TPR + t) * 16);
    };
    constexpr bool kJit = V * EPV > 4;
    double wreg[NP][kJit ? 1 : V][kJit ? 1 : EPV];
    if (!kJit) {
#pragma unroll
      for (int q = 0; q < NP; ++q)
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const double2 wv = wplane(q, v, c);
            wreg[q][kJit ? 0 : v][kJit ? 0 : 2 * c] = wv.x;
            wreg[q][kJit ? 0 : v][kJit ? 0 : 2 * c + 1] = wv.y;
          }
    }
    if (a.kind == 100 || a.kind == 101) {  // diagnostics (option k1_diag): 100 = stream + widen only, 101 = + phase 1, no barriers
      __syncwarp();
      if (lane == 0) {  // no CTA barrier in these modes: the last warp to leave the stage refills it
        const unsigned int done = atomicAdd(&cnt[s], 1u);
        if (done == NW - 1) {
          cnt[s] = 0u;
          fill((long long)k + S, s);
        }
      }
      double sacc = 0.0;
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const double we = kJit ? (e & 1 ? wplane(0, v, e / 2).y : wplane(0, v, e / 2).x) : wreg[0][kJit ? 0 : v][kJit ? 0 : e];
            sacc = (a.kind == 100) ? sacc + xd[r][v][e] : fma(xd[r][v][e], we, sacc);
          }
      acc[0][0] += sacc;
      continue;
    }

    // phase 1: R partial dots over this thread's columns (against w, and against w2 on the same retained tile).  Either way
    // every p[r] is the same (v, e)-ascending FMA chain, so the two forms (and the one- and two-point kernels) agree bit for bit.
    if (kJit) {
      double p[R], p2[DUAL ? R : 1];
#pragma unroll
      for (int r = 0; r < R; ++r) { p[r] = 0.0; if (DUAL) p2[DUAL ? r : 0] = 0.0; }
#pragma unroll
      for (int v = 0; v < V; ++v)
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const double2 wa = wplane(0, v, c);
          const double2 wb = DUAL ? wplane(NP - 1, v, c) : wa;
#pragma unroll
          for (int r = 0; r < R; ++r) {
            p[r] = fma(xd[r][v][2 * c + 1], wa.y, fma(xd[r][v][2 * c], wa.x, p[r]));
            if (DUAL) p2[DUAL ? r : 0] = fma(xd[r][v][2 * c + 1], wb.y, fma(xd[r][v][2 * c], wb.x, p2[DUAL ? r : 0]));
          }
        }
      const double tot = warp_rows_reduce_perm<R>(p);
      if ((lane % (32 / R)) == 0) partial[(g * R + rperm) * 8 + wig] = tot;
      if (DUAL) {
        double (&pr)[R] = reinterpret_cast<double (&)[R]>(p2);
        const double tot2 = warp_rows_reduce_perm<R>(pr);
        if ((lane % (32 / R)) == 0) partial2[(g * R + rperm) * 8 + wig] = tot2;
      }
    } else {
#pragma unroll
      for (int q = 0; q < NP; ++q) {
        double p[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          double sacc = 0.0;
#pragma unroll
          for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < EPV; ++e) sacc = fma(xd[r][v][e], wreg[q][kJit ? 0 : v][kJit ? 0 : e], sacc);
          p[r] = sacc;
        }
        const double tot = warp_rows_reduce_perm<R>(p);
        if ((lane % (32 / R)) == 0) (q ? partial2 : partial)[(g * R + rperm) * 8 + wig] = tot;
      }
    }
    __syncthreads();
    // every warp holds its part of the tile in registers: the stage is free.  One lane of a warp that is not this tile's
    // scalar warp re-arms the mbarrier and issues the TMA refill (no producer warp, no counters).
    if (warp == ((sw + NW / 2) & (NW - 1)) && lane == 0) fill((long long)k + S, s);

    // scalar section: only the multiplier is needed by phase 2, so for logistic only the exp + reciprocal part of
    // the evaluation sits between the barriers; the log part follows, interleaved with this warp's phase-2 FMAs
    LogisticMid mid;   // written and read by the scalar warp only
    bool row_ok = false;
    if (sactive) {
      const long long row0 = (long long)tile * TR;
      const double *pp = (DUAL && lane >= 16) ? partial2 : partial;
      double pw[8];
#pragma unroll
      for (int wi = 0; wi < 8; ++wi) pw[wi] = (wi < WPG) ? pp[srow * 8 + wi] : 0.0;
      const double m = ((pw[0] + pw[1]) + (pw[2] + pw[3])) + ((pw[4] + pw[5]) + (pw[6] + pw[7]));
      row_ok = srow < rv && row_selected(a.sample_seed, a.sample_thresh, a.row_base + row0 + srow);
      double mult, loss = 0.0;
      if (a.kind == AGD_GRAD_LOGISTIC) mult = logistic_head(m, ylab, mid);
      else loss_eval(a.kind, m, ylab, mult, loss);
      const double mw = row_ok ? mult : 0.0;
      if (DUAL ? lane < 16 : srow < TR) mult_s[srow] = mw;
      if (MODE == 2 && lane >= 16) mult2_s[srow] = mw;
      if (a.kind != AGD_GRAD_LOGISTIC) lossacc += row_ok ? loss : 0.0;
      cntacc += row_ok ? 1.0 : 0.0;
      // A row whose multiplier is exactly 0 adds nothing (netlib DAXPY returns when DA == 0), but 0 * inf is NaN.  Flag the
      // rows where that can happen: a finite margin means every feature of the row is finite (padded columns are zero).
      // Bit = tile row; with a second gradient (MODE 2), bits 16 + row are the rows at w2.
      const bool poison = srow < rv && (!DUAL || MODE == 2 || lane < 16) && mw == 0.0 && !isfinite(m);
      const uint32_t flagged_rows = __ballot_sync(0xffffffffu, poison);
      if (lane == 0) *skip_s = flagged_rows;
    }
    __syncthreads();

    // phase 2: g += mult_i * x_i on the retained fp64 tile.  Flagged rows (rare: non-finite features) must leave the sums as
    // they are.  With one gradient their retained x is zeroed, which only turns +-0 or NaN terms into +0; with two, the FMAs
    // are select-guarded, one guard per point.
    const uint32_t skip = *skip_s;
    auto fold = [&](const double *ms, double (&av)[V][EPV], uint32_t flagged) {
      double mu[R];
#pragma unroll
      for (int r = 0; r < R; ++r) mu[r] = ms[g * R + (r ^ rperm)];
      if (MODE != 2 || flagged == 0u) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < EPV; ++e) av[v][e] = fma(mu[r], xd[r][v][e], av[v][e]);
      } else {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const bool keep = ((flagged >> (g * R + (r ^ rperm))) & 1u) == 0u;
#pragma unroll
          for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < EPV; ++e) av[v][e] = keep ? fma(mu[r], xd[r][v][e], av[v][e]) : av[v][e];
        }
      }
    };
    if (MODE != 2 && skip != 0u) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if ((skip >> (g * R + (r ^ rperm))) & 1u) {
#pragma unroll
          for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < EPV; ++e) xd[r][v][e] = 0.0;
        }
    }
    auto phase2 = [&]() {
      fold(mult_s, acc, MODE == 2 ? (skip & 0xffffu) : skip);
      if (MODE == 2)   // the gradient at w2 from the same retained tile
        fold(mult2_s, reinterpret_cast<double (&)[V][EPV]>(accB), skip >> 16);
    };
    if (a.kind == AGD_GRAD_LOGISTIC && warp == sw) {
      // warp-uniform branch: the log chain of the loss (all 32 lanes, lanes >= TR carry don't-care values) is
      // independent of the FMAs, so the scheduler interleaves the two instead of serialising them
      const double loss = logistic_tail(mid, ylab);
      phase2();
      lossacc += row_ok ? loss : 0.0;
    } else {
      phase2();
    }
  }

  // ---------------- per-CTA slab: column sums (row groups added in fixed order) and loss sum.  MODE 2: a second block of
  // d + 4 doubles [gradient at w2 | loss sum | count | 0 | 0] follows the first.
  double *slab = a.slabs + (size_t)blockIdx.x * a.slab_stride;
  auto write_columns = [&](double (&av)[V][EPV], double *dst) {
    if (NG > 1) {
      __syncthreads();  // aux (w staging) is free for reuse: every thread is past the tile loop
      double *ax = reinterpret_cast<double *>(aux);
#pragma unroll
      for (int v = 0; v < V; ++v)
#pragma unroll
        for (int e = 0; e < EPV; ++e) ax[(size_t)g * (TPR * V * EPV) + (v * TPR + t) * EPV + e] = av[v][e];
      __syncthreads();
      if (g == 0) {
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            double sacc = 0.0;
            for (int gg = 0; gg < NG; ++gg) sacc += ax[(size_t)gg * (TPR * V * EPV) + (v * TPR + t) * EPV + e];
            av[v][e] = sacc;
          }
      }
    }
    if (g == 0) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int vec = v * TPR + t;
        if (vec < nvec) {
#pragma unroll
          for (int e = 0; e < EPV; ++e) dst[vec * EPV + e] = av[v][e];
        }
      }
    }
  };
  write_columns(acc, slab);
  if (MODE == 2) write_columns(reinterpret_cast<double (&)[V][EPV]>(accB), slab + a.d + 4);
  // DUAL: lanes 16-31 hold the sums at w2.  Skipping the xor-16 step leaves the lane-0 total bit-identical to the
  // single-point kernel's, whose lanes >= 16 only ever contribute exact zeros.
  for (int off = DUAL ? 8 : 16; off >= 1; off >>= 1) {
    lossacc += __shfl_xor_sync(0xffffffffu, lossacc, off);
    cntacc += __shfl_xor_sync(0xffffffffu, cntacc, off);
  }
  if (lane == 0) { red[warp] = lossacc; red[8 + warp] = cntacc; }
  if (DUAL && lane == 16) { red[16 + warp] = lossacc; red[24 + warp] = cntacc; }
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0, cacc = 0.0, sacc2 = 0.0, cacc2 = 0.0;
    for (int wi = 0; wi < NW; ++wi) { sacc += red[wi]; cacc += red[8 + wi]; }
    if (DUAL)
      for (int wi = 0; wi < NW; ++wi) { sacc2 += red[16 + wi]; cacc2 += red[24 + wi]; }
    slab[a.d] = sacc;
    slab[a.d + 1] = cacc;
    slab[a.d + 2] = sacc2;   // loss sum and row count at w2 (zero when the launch has no second point)
    slab[a.d + 3] = cacc2;
    if (MODE == 2) {
      double *slab2 = slab + a.d + 4;
      slab2[a.d] = sacc2;
      slab2[a.d + 1] = cacc2;
      slab2[a.d + 2] = 0.0;
      slab2[a.d + 3] = 0.0;
    }
  }
}

template <typename T> __device__ __forceinline__ double load_elem(const T *p) { return (double)*p; }
template <> __device__ __forceinline__ double load_elem<__nv_bfloat16>(const __nv_bfloat16 *p) {
  return (double)__bfloat162float(*p);
}

// ---------------------------------------------------------------- generic shapes
// a.w2 != nullptr: the loss (not the gradient) is also evaluated at w2 in the same sweep -- threads 32..32+R-1 play the
// part of threads 0..R-1 for it, so its sum is formed exactly as a launch of its own would form it.
template <typename T>
__global__ void __launch_bounds__(256) k1_generic_kernel(const K1Args a, const long long ntiles) {
  constexpr int R = 8;
  __shared__ double part[2][R][8];
  __shared__ double mult_s[R];
  __shared__ double red[32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool dual = a.w2 != nullptr;
  const T *X = reinterpret_cast<const T *>(a.X);
  double *slab = a.slabs + (size_t)blockIdx.x * a.slab_stride;
  for (int c = tid; c <= a.d; c += 256) slab[c] = 0.0;
  double lossacc = 0.0, cntacc = 0.0;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long row0 = tile * R;
    const long long left = a.rows - row0;
    const int rv = left < R ? (int)left : R;
    double p[R], p2[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { p[r] = 0.0; p2[r] = 0.0; }
    if (!dual) {
      for (int c = tid; c < a.d; c += 256) {
        const double wc = a.w[c];
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (r < rv) p[r] = fma(load_elem<T>(&X[(size_t)(row0 + r) * a.d + c]), wc, p[r]);
      }
    } else {
      for (int c = tid; c < a.d; c += 256) {
        const double wc = a.w[c], wc2 = a.w2[c];
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (r < rv) {
            const double xv = load_elem<T>(&X[(size_t)(row0 + r) * a.d + c]);
            p[r] = fma(xv, wc, p[r]);
            p2[r] = fma(xv, wc2, p2[r]);
          }
      }
    }
    const double tot = warp_rows_reduce<R>(p, lane);
    if ((lane & 3) == 0) part[0][lane >> 2][warp] = tot;
    if (dual) {
      const double tot2 = warp_rows_reduce<R>(p2, lane);
      if ((lane & 3) == 0) part[1][lane >> 2][warp] = tot2;
    }
    __syncthreads();
    const int which = tid >> 5, srow = tid & 31;
    if (srow < R && (which == 0 || (dual && which == 1))) {
      double m = 0.0;
#pragma unroll
      for (int wi = 0; wi < 8; ++wi) m += part[which][srow][wi];
      double mult = 0.0, loss = 0.0;
      if (srow < rv && row_selected(a.sample_seed, a.sample_thresh, a.row_base + row0 + srow)) {
        loss_eval(a.kind, m, a.labels[row0 + srow], mult, loss);
        cntacc += 1.0;
      }
      if (which == 0) mult_s[srow] = mult;
      lossacc += loss;
    }
    __syncthreads();
    // a row whose multiplier is exactly 0 adds nothing, whatever its features (netlib DAXPY returns when DA == 0): the test
    // is uniform over the CTA, and on finite rows it drops only +-0 terms
    double mu[R];
#pragma unroll
    for (int r = 0; r < R; ++r) mu[r] = mult_s[r];
    for (int c = tid; c < a.d; c += 256) {
      double sacc = slab[c];
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (r < rv && mu[r] != 0.0) sacc = fma(mu[r], load_elem<T>(&X[(size_t)(row0 + r) * a.d + c]), sacc);
      slab[c] = sacc;
    }
  }
  for (int off = 16; off >= 1; off >>= 1) {
    lossacc += __shfl_xor_sync(0xffffffffu, lossacc, off);
    cntacc += __shfl_xor_sync(0xffffffffu, cntacc, off);
  }
  if (lane == 0) { red[warp] = lossacc; red[8 + warp] = cntacc; }
  __syncthreads();
  if (tid == 0) {
    // warp 0 carries the sums at w, warp 1 those at w2 (all other entries are exact zeros)
    double sacc = 0.0, cacc = 0.0, sacc2 = 0.0, cacc2 = 0.0;
    for (int wi = 0; wi < 8; ++wi) {
      if (dual && wi == 1) { sacc2 = red[wi]; cacc2 = red[8 + wi]; continue; }
      sacc += red[wi];
      cacc += red[8 + wi];
    }
    slab[a.d] = sacc;
    slab[a.d + 1] = cacc;
    slab[a.d + 2] = sacc2;
    slab[a.d + 3] = cacc2;
  }
}

// ---------------------------------------------------------------- slab reduction (combOp, AGD.scala:201-204)
// out[c] = sum over slabs of column c, c < n (gradient, loss sum, row count, then the same pair at the second point of a
// fused sweep; after a two-gradient sweep a second such block).  32 columns per block; 8 slab groups per block sum
// strided subsets (slab b -> group b % 8) with 4 loads in flight, then group 0 adds the 8 group sums in
// order: the summation tree is fixed, so the result is bit-reproducible.
template <bool PUB>
__global__ void __launch_bounds__(256) k1_reduce_kernel(const double *__restrict__ slabs, int blocks, int n,
                                                        double *__restrict__ out, const XchgPub pub) {
  __shared__ double part[8][33];
  __shared__ bool last;
  const int cl = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const size_t stride = (size_t)n;   // n = d + 4 columns per evaluation point held by the slabs (2 (d + 4) after a two-gradient sweep)
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
  if (c < n) {
    int b = grp;
    for (; b + 24 < blocks; b += 32) {
      const double v0 = slabs[(size_t)b * stride + c], v1 = slabs[(size_t)(b + 8) * stride + c],
                   v2 = slabs[(size_t)(b + 16) * stride + c], v3 = slabs[(size_t)(b + 24) * stride + c];
      s0 += v0; s1 += v1; s2 += v2; s3 += v3;
    }
    for (; b < blocks; b += 8) s0 += slabs[(size_t)b * stride + c];
  }
  part[grp][cl] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (grp == 0 && c < n) {
    double t = 0.0;
#pragma unroll
    for (int gi = 0; gi < 8; ++gi) t += part[gi][cl];
    out[c] = t;
    if (PUB) {  // compute + collective in one kernel: the result goes straight into every peer's HBM over NVLink
      const size_t off = ((size_t)pub.buf * pub.world + pub.my_rank) * pub.slot_stride + c;
      for (int p = 0; p < pub.world; ++p) pub.peers.slot[p][off] = t;
    }
  }
  if (PUB) {
    // Release: the CTA barrier orders every thread's peer stores before thread 0, whose system-scope fence is cumulative over
    // them (one fence per block instead of one per thread: a MEMBAR.SC.SYS waits for NVLink acknowledgements).  The block that
    // takes the last ticket has therefore observed all blocks' stores as performed and raises the epoch flag on every peer.
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      last = (atomicAdd(pub.ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
      if (threadIdx.x < pub.world) {
        __threadfence_system();
        *reinterpret_cast<volatile unsigned long long *>(&pub.peers.flag[threadIdx.x][pub.buf * pub.world + pub.my_rank]) = pub.epoch;
      }
      if (threadIdx.x == 0) *pub.ticket = 0u;
    }
  }
}

struct RingShape { int tpr, v, r; };
inline bool ring_shape(int32_t d, int elem_bytes, RingShape &sh, int &nvec) {
  const int epv = 16 / elem_bytes;
  if (d <= 0 || d % epv != 0) return false;
  nvec = d / epv;
  if (elem_bytes == 2) {  // bf16: 8 elements per vector, so at most 4 vectors per thread and tile
    if (nvec <= 256) {
      int tpr = 32;
      while (tpr < nvec) tpr <<= 1;
      sh = {tpr, 1, 4};
      return true;
    }
    if (nvec <= 512) { sh = {256, 2, 2}; return true; }
    return false;
  }
  if (nvec <= 256) {
    int tpr = 32;
    while (tpr < nvec) tpr <<= 1;
    const int ng = 256 / tpr;
    int r = 8;
    if (ng * r > kMaxTileRows) r = kMaxTileRows / ng;
    sh = {tpr, 1, r};
    return true;
  }
  if (nvec <= 512) { sh = {256, 2, 4}; return true; }
  if (nvec <= 1024) { sh = {256, 4, 2}; return true; }
  return false;
}

template <typename T, int NT, int TPR, int V, int R, int MINB, int MODE = 0>
cudaError_t launch_ring_inst(const K1Args &a_in, int nvec, int sm_count, int *blocks_out, cudaStream_t st) {
  constexpr int EPV = Elem<T>::EPV;
  constexpr int NG = NT / TPR;
  constexpr int TR = NG * R;
  K1Args a = a_in;
  const uint32_t row_bytes = (uint32_t)a.d * sizeof(T);
  const uint32_t tile_bytes = TR * row_bytes + kMaxTileRows * 8;  // rows + their labels
  // w staging: one plane set of TPR * V vectors per point; the same area later holds NG row-group partial sums
  uint32_t aux_bytes = (uint32_t)(MODE ? 2 : 1) * TPR * V * EPV * 8u;
  if (NG > 1) {
    const uint32_t need = (uint32_t)NG * TPR * V * EPV * 8u;
    if (need > aux_bytes) aux_bytes = need;
  }
  const uint32_t budget = (227u * 1024u - MINB * 1024u) / MINB;
  int stages = a.stages > 0 ? a.stages : 4;
  while (stages > 1 && ring_layout(tile_bytes, aux_bytes, stages, MODE).total > budget) --stages;
  a.stages = stages;
  a.slab_stride = (MODE == 2 ? 2 : 1) * (a.d + 4);
  const RingLayout L = ring_layout(tile_bytes, aux_bytes, stages, MODE);
  auto kern = k1_ring_kernel<T, NT, TPR, V, R, MINB, MODE>;
  // the opt-in shared-memory size is a per-device property of the function: set it when it changes, not on every launch
  static int smem_set[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || smem_set[dev] != (int)L.total) {
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) smem_set[dev] = (int)L.total;
  }
  const long long ntiles = (a.rows + TR - 1) / TR;
  long long grid = (long long)MINB * sm_count;
  if (grid > ntiles) grid = ntiles;
  if (grid < 1) grid = 1;
  *blocks_out = (int)grid;
  kern<<<(unsigned)grid, NT, L.total, st>>>(a, nvec, ntiles, aux_bytes);
  return cudaGetLastError();
}

cudaError_t launch_ring_bf16(const K1Args &a, const RingShape &sh, int nvec, int sm_count, int *blocks_out,
                             cudaStream_t st) {
  using T = __nv_bfloat16;
  if (a.w2 && a.dual_full) return cudaErrorInvalidValue;  // the two-gradient sweep exists for fp32 / fp64 storage
  if (a.w2) {  // fused sweep: tiles of at most 16 rows
    if (sh.v == 2) return launch_ring_inst<T, 256, 256, 2, 2, 2, 1>(a, nvec, sm_count, blocks_out, st);
    switch (sh.tpr) {
      case 64: return launch_ring_inst<T, 256, 64, 1, 4, 2, 1>(a, nvec, sm_count, blocks_out, st);
      case 128: return launch_ring_inst<T, 256, 128, 1, 4, 2, 1>(a, nvec, sm_count, blocks_out, st);
      case 256: return launch_ring_inst<T, 256, 256, 1, 4, 2, 1>(a, nvec, sm_count, blocks_out, st);
      default: return cudaErrorInvalidValue;
    }
  }
  if (sh.v == 2) return launch_ring_inst<T, 256, 256, 2, 2, 2>(a, nvec, sm_count, blocks_out, st);
  switch (sh.tpr) {
    case 32: return launch_ring_inst<T, 256, 32, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
    case 64: return launch_ring_inst<T, 256, 64, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
    case 128: return launch_ring_inst<T, 256, 128, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
    default: return launch_ring_inst<T, 256, 256, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
  }
}

template <typename T>
cudaError_t launch_ring_t(const K1Args &a, const RingShape &sh, int nvec, int sm_count, int *blocks_out,
                          cudaStream_t st) {
  if (a.w2 && a.dual_full) {  // two full evaluations per sweep (speculative sweep of the memoised pass structure)
    if (sh.v == 4) return cudaErrorInvalidValue;   // four vectors per thread: no registers for a second gradient
    if (sh.v == 2) return launch_ring_inst<T, 256, 256, 2, 4, 2, 2>(a, nvec, sm_count, blocks_out, st);
    if (sh.tpr == 128) return launch_ring_inst<T, 256, 128, 1, 8, 2, 2>(a, nvec, sm_count, blocks_out, st);
    if (sh.tpr == 256) return launch_ring_inst<T, 256, 256, 1, 8, 2, 2>(a, nvec, sm_count, blocks_out, st);
    return cudaErrorInvalidValue;
  }
  if (a.w2) {  // fused sweep: tiles of at most 16 rows
    if (sh.v == 4) return launch_ring_inst<T, 256, 256, 4, 2, 2, 1>(a, nvec, sm_count, blocks_out, st);
    if (sh.v == 2) return launch_ring_inst<T, 256, 256, 2, 4, 2, 1>(a, nvec, sm_count, blocks_out, st);
    if (sh.tpr == 128) return launch_ring_inst<T, 256, 128, 1, 8, 2, 1>(a, nvec, sm_count, blocks_out, st);
    if (sh.tpr == 256) return launch_ring_inst<T, 256, 256, 1, 8, 2, 1>(a, nvec, sm_count, blocks_out, st);
    return cudaErrorInvalidValue;
  }
  if (sh.v == 1) {
    switch (sh.tpr) {
      case 32: return launch_ring_inst<T, 256, 32, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
      case 64: return launch_ring_inst<T, 256, 64, 1, 8, 2>(a, nvec, sm_count, blocks_out, st);
      case 128: return launch_ring_inst<T, 256, 128, 1, 8, 2>(a, nvec, sm_count, blocks_out, st);
      default: {
        // tuning variants of the headline shape: (threads per CTA) x (rows per tile) x (resident CTAs per SM)
        const int key = a.tune_rows * 10 + a.tune_ctas;
        switch (key) {
          case 81: return launch_ring_inst<T, 256, 256, 1, 8, 1>(a, nvec, sm_count, blocks_out, st);
          case 42: return launch_ring_inst<T, 256, 256, 1, 4, 2>(a, nvec, sm_count, blocks_out, st);
          case 43: return launch_ring_inst<T, 256, 256, 1, 4, 3>(a, nvec, sm_count, blocks_out, st);
          case 44: return launch_ring_inst<T, 128, 128, 2, 4, 4>(a, nvec, sm_count, blocks_out, st);  // 128-thread CTAs
          case 45: return launch_ring_inst<T, 128, 128, 2, 4, 3>(a, nvec, sm_count, blocks_out, st);
          case 46: return launch_ring_inst<T, 256, 128, 2, 4, 2>(a, nvec, sm_count, blocks_out, st);  // 2 row groups x 2 vectors
          default: return launch_ring_inst<T, 256, 256, 1, 8, 2>(a, nvec, sm_count, blocks_out, st);
        }
      }
    }
  }
  if (sh.v == 2) return launch_ring_inst<T, 256, 256, 2, 4, 2>(a, nvec, sm_count, blocks_out, st);
  return launch_ring_inst<T, 256, 256, 4, 2, 2>(a, nvec, sm_count, blocks_out, st);
}


}  // namespace

int k1_max_blocks(int sm_count) { return 4 * sm_count; }

int k1_ring_supported(int32_t d, int elem_bytes) {
  RingShape sh;
  int nvec;
  return ring_shape(d, elem_bytes, sh, nvec) ? 1 : 0;
}

// the fused (two-point) sweep exists for ring shapes whose tile has at most 16 rows
int k1_ring_dual_supported(int32_t d, int elem_bytes) {
  RingShape sh;
  int nvec;
  if (!ring_shape(d, elem_bytes, sh, nvec)) return 0;
  return (256 / sh.tpr) * sh.r <= 16 ? 1 : 0;
}

// ... and the two-gradient sweep for the fp32 / fp64 instantiations of those shapes
int k1_ring_dual_full_supported(int32_t d, int elem_bytes) {
  RingShape sh;
  int nvec;
  if ((elem_bytes != 4 && elem_bytes != 8) || !ring_shape(d, elem_bytes, sh, nvec)) return 0;
  if (sh.v == 2) return 1;                                          // two vectors per thread: d <= 2048 (fp32) / 1024 (fp64)
  return sh.v == 1 && (sh.tpr == 128 || sh.tpr == 256) ? 1 : 0;   // one vector per thread: d <= 1024 (fp32) / 512 (fp64)
}

cudaError_t k1_ring_launch(const K1Args &a, int elem_bytes, int sm_count, int *blocks_out, cudaStream_t st) {
  RingShape sh;
  int nvec = 0;
  if (!ring_shape(a.d, elem_bytes, sh, nvec)) return cudaErrorInvalidValue;
  if (a.rows <= 0) { *blocks_out = 0; return cudaSuccess; }
  if (elem_bytes == 2) return launch_ring_bf16(a, sh, nvec, sm_count, blocks_out, st);
  if (elem_bytes == 4) return launch_ring_t<float>(a, sh, nvec, sm_count, blocks_out, st);
  return launch_ring_t<double>(a, sh, nvec, sm_count, blocks_out, st);
}

cudaError_t k1_generic_launch(const K1Args &a, int elem_bytes, int sm_count, int max_blocks, int *blocks_out,
                              cudaStream_t st) {
  if (a.rows <= 0) { *blocks_out = 0; return cudaSuccess; }
  const long long ntiles = (a.rows + 7) / 8;
  long long grid = k1_max_blocks(sm_count);
  if (grid > max_blocks) grid = max_blocks;
  if (grid > ntiles) grid = ntiles;
  if (grid < 1) grid = 1;
  *blocks_out = (int)grid;
  if (elem_bytes == 2) k1_generic_kernel<__nv_bfloat16><<<(unsigned)grid, 256, 0, st>>>(a, ntiles);
  else if (elem_bytes == 4) k1_generic_kernel<float><<<(unsigned)grid, 256, 0, st>>>(a, ntiles);
  else k1_generic_kernel<double><<<(unsigned)grid, 256, 0, st>>>(a, ntiles);
  return cudaGetLastError();
}

cudaError_t k1_reduce_launch(const double *slabs, int blocks, int32_t n, double *out, const XchgPub *pub, cudaStream_t st) {
  const int grid = (n + 31) / 32;
  if (pub) k1_reduce_kernel<true><<<grid, 256, 0, st>>>(slabs, blocks, n, out, *pub);
  else k1_reduce_kernel<false><<<grid, 256, 0, st>>>(slabs, blocks, n, out, XchgPub());
  return cudaGetLastError();
}

}  // namespace agd
