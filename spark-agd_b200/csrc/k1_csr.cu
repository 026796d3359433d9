// k1_csr.cu -- K1 for SparseVector rows stored as CSR (sm_90a).
//
// Same contract as the dense kernel (seqOp fold of AGD.scala:197-200 with the sparse branches of
// BLAS.dot / BLAS.axpy [mllib-1.3.0]): one warp per row, lanes stride the row's stored entries
// (coalesced idx/val reads), w is gathered from the L2-resident fp64 vector, the margin is
// warp-shuffle reduced, loss' is evaluated once per row, and mult * val is scattered into the
// L2-resident fp64 gradient with RED.ADD.F64.  HBM traffic per pass = nnz*(4 + elem) + rows*16.
// The scatter order is not fixed, so the gradient is reproducible only to fp64 rounding (~1e-16).
// DUAL: the loss is also evaluated at a second point w2 in the same sweep (one more gather per stored entry).
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

// Which rows reach the scatter.  The sparse BLAS.axpy [mllib-1.3.0] is a plain loop with no zero test, so a row the sample
// keeps adds mult * x even when mult is exactly 0 (0 * inf = NaN must show); only a hinge row outside the margin, for which
// HingeGradient never calls axpy, adds nothing.  A hinge row inside the margin has mult = -+1, never 0.
__device__ __forceinline__ bool csr_row_folds(int kind, bool sel, double mult) {
  return sel && (mult != 0.0 || kind != AGD_GRAD_HINGE);
}

// BIAS: the model has an intercept: w[d] (w2[d]) joins every margin, the multipliers sum into gacc[d], scalars from d + 1
template <typename T, bool DUAL, bool VIEW, bool BIAS>
__global__ void __launch_bounds__(256) k1_csr_kernel(const K1CsrArgs a) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warp_global = (blockIdx.x * 256LL + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256LL) >> 5;
  const T *val = reinterpret_cast<const T *>(a.val);
  double lossacc = 0.0, cntacc = 0.0, lossacc2 = 0.0, multacc = 0.0;
  for (long long r = warp_global; r < a.rows; r += nwarps) {
    const long long lo = a.rowptr[r], hi = a.rowptr[r + 1];
    double m = 0.0, m2 = 0.0;
    for (long long k = lo + lane; k < hi; k += 32) {
      const double xv = (double)val[k];
      const int c = a.idx[k];
      m = fma(xv, a.w[c], m);
      if (DUAL) m2 = fma(xv, a.w2[c], m2);
    }
    for (int off = 16; off >= 1; off >>= 1) {
      m += __shfl_xor_sync(0xffffffffu, m, off);
      if (DUAL) m2 += __shfl_xor_sync(0xffffffffu, m2, off);
    }
    if (BIAS) { m += a.w[a.d]; if (DUAL) m2 += a.w2[a.d]; }
    double mult, loss;
    const double ylab = a.labels[r];
    loss_eval(a.kind, m, ylab, mult, loss);
    const bool sel = row_kept(a.sample_seed, a.sample_thresh, VIEW ? a.filt : nullptr, a.row_base + r);
    if (!sel) { mult = 0.0; loss = 0.0; }
    else if (lane == 0) cntacc += 1.0;
    if (lane == 0) lossacc += loss;
    if (BIAS && lane == 0) multacc += mult;
    if (DUAL && sel && lane == 0) {
      double mult2, loss2;
      loss_eval(a.kind, m2, ylab, mult2, loss2);
      lossacc2 += loss2;
    }
    if (csr_row_folds(a.kind, sel, mult)) {
      for (long long k = lo + lane; k < hi; k += 32) atomicAdd(&a.gacc[a.idx[k]], mult * (double)val[k]);
    }
  }
  for (int off = 16; off >= 1; off >>= 1) {
    lossacc += __shfl_xor_sync(0xffffffffu, lossacc, off);
    cntacc += __shfl_xor_sync(0xffffffffu, cntacc, off);
    if (DUAL) lossacc2 += __shfl_xor_sync(0xffffffffu, lossacc2, off);
    if (BIAS) multacc += __shfl_xor_sync(0xffffffffu, multacc, off);
  }
  if (lane == 0) { red[warp] = lossacc; red[8 + warp] = cntacc; red[16 + warp] = lossacc2; if (BIAS) red[24 + warp] = multacc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int DB = a.d + (BIAS ? 1 : 0);
    double s = 0.0, c = 0.0, s2 = 0.0, mc = 0.0;
    for (int w = 0; w < 8; ++w) { s += red[w]; c += red[8 + w]; s2 += red[16 + w]; if (BIAS) mc += red[24 + w]; }
    if (BIAS) atomicAdd(&a.gacc[a.d], mc);
    atomicAdd(&a.gacc[DB], s);
    atomicAdd(&a.gacc[DB + 1], c);   // counts are small integers: exact in any order
    if (DUAL) {
      atomicAdd(&a.gacc[DB + 2], s2);
      atomicAdd(&a.gacc[DB + 3], c);  // the same rows are selected at both points
    }
  }
}

// The same fold with more loads in flight (selected by default; option ring_rows=1 keeps the simple loop above): the kernel is
// bound by the latency of dependent loads, rowptr -> idx/val -> w gather (ncu: 74 % long-scoreboard stalls, L2 at 65 % of peak).
template <typename T, bool DUAL, bool VIEW, bool BIAS>
__global__ void __launch_bounds__(256) k1_csr_pipelined_kernel(const K1CsrArgs a) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warp_global = (blockIdx.x * 256LL + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256LL) >> 5;
  const T *val = reinterpret_cast<const T *>(a.val);
  double lossacc = 0.0, cntacc = 0.0, lossacc2 = 0.0, multacc = 0.0;
  // The kernel is bound by the latency of dependent loads (rowptr -> idx/val -> w gather; ncu: 74 % long-scoreboard stalls), so
  // the next row's extent is fetched one row ahead, a lane's first two entries are loaded together (rows of up to 64 entries:
  // both gathers in flight at once) and kept in registers for the scatter instead of being read again.
  long long lo = 0, hi = 0;
  if (warp_global < a.rows) { lo = a.rowptr[warp_global]; hi = a.rowptr[warp_global + 1]; }
  for (long long r = warp_global; r < a.rows; r += nwarps) {
    const long long rn = r + nwarps;
    long long lo_n = 0, hi_n = 0;
    if (rn < a.rows) { lo_n = a.rowptr[rn]; hi_n = a.rowptr[rn + 1]; }
    const double ylab = a.labels[r];
    double m = 0.0, m2 = 0.0;
    const long long k0 = lo + lane, k1 = k0 + 32;
    const bool h0 = k0 < hi, h1 = k1 < hi;
    int c0 = 0, c1 = 0;
    double x0 = 0.0, x1 = 0.0;
    if (h0) { c0 = a.idx[k0]; x0 = (double)val[k0]; }
    if (h1) { c1 = a.idx[k1]; x1 = (double)val[k1]; }
    if (h0) {
      const double w0 = a.w[c0];
      const double w1 = h1 ? a.w[c1] : 0.0;
      m = fma(x0, w0, m);
      if (h1) m = fma(x1, w1, m);
      if (DUAL) {
        const double v0 = a.w2[c0];
        const double v1 = h1 ? a.w2[c1] : 0.0;
        m2 = fma(x0, v0, m2);
        if (h1) m2 = fma(x1, v1, m2);
      }
    }
    for (long long k = k1 + 32; k < hi; k += 32) {   // longer rows: the remaining entries, one per lane and round
      const double xv = (double)val[k];
      const int c = a.idx[k];
      m = fma(xv, a.w[c], m);
      if (DUAL) m2 = fma(xv, a.w2[c], m2);
    }
    for (int off = 16; off >= 1; off >>= 1) {
      m += __shfl_xor_sync(0xffffffffu, m, off);
      if (DUAL) m2 += __shfl_xor_sync(0xffffffffu, m2, off);
    }
    if (BIAS) { m += a.w[a.d]; if (DUAL) m2 += a.w2[a.d]; }
    double mult, loss;
    loss_eval(a.kind, m, ylab, mult, loss);
    const bool sel = row_kept(a.sample_seed, a.sample_thresh, VIEW ? a.filt : nullptr, a.row_base + r);
    if (!sel) { mult = 0.0; loss = 0.0; }
    else if (lane == 0) cntacc += 1.0;
    if (lane == 0) lossacc += loss;
    if (BIAS && lane == 0) multacc += mult;
    if (DUAL && sel && lane == 0) {
      double mult2, loss2;
      loss_eval(a.kind, m2, ylab, mult2, loss2);
      lossacc2 += loss2;
    }
    if (csr_row_folds(a.kind, sel, mult)) {
      if (h0) atomicAdd(&a.gacc[c0], mult * x0);
      if (h1) atomicAdd(&a.gacc[c1], mult * x1);
      for (long long k = k1 + 32; k < hi; k += 32) atomicAdd(&a.gacc[a.idx[k]], mult * (double)val[k]);
    }
    lo = lo_n; hi = hi_n;
  }
  for (int off = 16; off >= 1; off >>= 1) {
    lossacc += __shfl_xor_sync(0xffffffffu, lossacc, off);
    cntacc += __shfl_xor_sync(0xffffffffu, cntacc, off);
    if (DUAL) lossacc2 += __shfl_xor_sync(0xffffffffu, lossacc2, off);
    if (BIAS) multacc += __shfl_xor_sync(0xffffffffu, multacc, off);
  }
  if (lane == 0) { red[warp] = lossacc; red[8 + warp] = cntacc; red[16 + warp] = lossacc2; if (BIAS) red[24 + warp] = multacc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int DB = a.d + (BIAS ? 1 : 0);
    double s = 0.0, c = 0.0, s2 = 0.0, mc = 0.0;
    for (int w = 0; w < 8; ++w) { s += red[w]; c += red[8 + w]; s2 += red[16 + w]; if (BIAS) mc += red[24 + w]; }
    if (BIAS) atomicAdd(&a.gacc[a.d], mc);
    atomicAdd(&a.gacc[DB], s);
    atomicAdd(&a.gacc[DB + 1], c);   // counts are small integers: exact in any order
    if (DUAL) {
      atomicAdd(&a.gacc[DB + 2], s2);
      atomicAdd(&a.gacc[DB + 3], c);  // the same rows are selected at both points
    }
  }
}

}  // namespace

// VIEW: a launch on a view (a.filt != nullptr).  A launch without one takes the instantiation that has no view code, whose
// registers and instructions are those of a plain sweep.
template <bool VIEW, bool BIAS>
static void k1_csr_launch_t(const K1CsrArgs &a, int elem_bytes, unsigned grid, cudaStream_t st) {
  const bool simple = a.tune == 1;
  if (elem_bytes == 4) {
    if (simple) {
      if (a.w2) k1_csr_kernel<float, true, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
      else k1_csr_kernel<float, false, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
    } else {
      if (a.w2) k1_csr_pipelined_kernel<float, true, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
      else k1_csr_pipelined_kernel<float, false, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
    }
  } else {
    if (simple) {
      if (a.w2) k1_csr_kernel<double, true, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
      else k1_csr_kernel<double, false, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
    } else {
      if (a.w2) k1_csr_pipelined_kernel<double, true, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
      else k1_csr_pipelined_kernel<double, false, VIEW, BIAS><<<grid, 256, 0, st>>>(a);
    }
  }
}

cudaError_t k1_csr_launch(const K1CsrArgs &a, int bias, int elem_bytes, int sm_count, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(a.gacc, 0, ((size_t)a.d + (bias ? 1 : 0) + 4) * sizeof(double), st);
  if (e != cudaSuccess) return e;
  long long grid = (a.rows + 7) / 8;
  if (grid > 8LL * sm_count) grid = 8LL * sm_count;
  if (grid < 1) grid = 1;
  if (bias) {
    if (a.filt) k1_csr_launch_t<true, true>(a, elem_bytes, (unsigned)grid, st);
    else k1_csr_launch_t<false, true>(a, elem_bytes, (unsigned)grid, st);
  } else {
    if (a.filt) k1_csr_launch_t<true, false>(a, elem_bytes, (unsigned)grid, st);
    else k1_csr_launch_t<false, false>(a, elem_bytes, (unsigned)grid, st);
  }
  return cudaGetLastError();
}

}  // namespace agd
