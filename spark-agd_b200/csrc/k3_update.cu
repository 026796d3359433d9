// k3_update.cu -- K3: fused O(d) vector kernels of the driver loop (sm_90a).
//
// Replaces, on the device and in one launch per applySmooth result:
//   grad / count                                  AGD.scala:207
//   z = applyProjector(z_old, g_y, step)._2       AGD.scala:254  -> Updater.compute [mllib-1.3.0] (:215)
//   x = x_old * (1 - theta) + z * theta           AGD.scala:255
//   xy = x - y, norm(xy)^2, xy.dot(g_y)           AGD.scala:263-264,273
//   (x - y).dot(g_x - g_y)                        AGD.scala:278
//   norm(x), norm(x - x_old), g_y.dot(x - x_old)  AGD.scala:315-316,327
//   the regulariser value of applyProjector(x, g_x, 0.0)._1   AGD.scala:305
// Element-wise arithmetic keeps the reference's roundings (JVM: no FMA contraction), so the
// vectors agree with the oracle bit for bit given the same gradient; only the reductions differ in
// summation order.  Reductions are deterministic: per-block partials, then a last-block fixed-order sum.
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"

namespace agd {

namespace {

constexpr int kK3Threads = 256;
constexpr int kK3MaxBlocks = 128;

// Updater.compute(w, g, step, iter = 1, reg) element [mllib-1.3.0]
__device__ __forceinline__ double prox_elem(int updater, double w, double g, double step, double reg) {
  if (updater == AGD_UPD_SIMPLE) {
    return __dadd_rn(w, __dmul_rn(-step, g));
  } else if (updater == AGD_UPD_SQUARED_L2) {
    const double shrink = __dsub_rn(1.0, __dmul_rn(step, reg));
    return __dadd_rn(__dmul_rn(w, shrink), __dmul_rn(-step, g));
  } else {  // L1: step, then soft-threshold by reg*step
    const double u = __dadd_rn(w, __dmul_rn(-step, g));
    const double shrinkage = __dmul_rn(reg, step);
    const double sg = (u > 0.0) ? 1.0 : ((u < 0.0) ? -1.0 : u);
    double mag = __dsub_rn(fabs(u), shrinkage);
    if (!(mag != mag)) mag = (mag > 0.0) ? mag : 0.0;  // Java Math.max(0.0, .) propagates NaN
    return __dmul_rn(sg, mag);
  }
}

// block reduce NS values, write partials, last block sums partials in block order -> scalars
// ---- gather half of the peer-memory exchange, inlined into its consumer (see XchgGather)
__device__ __forceinline__ void xg_wait(const XchgGather &xg) {
  if (xg.world) {
    if (threadIdx.x < xg.world) {
      const volatile unsigned long long *f = xg.flags + xg.buf * xg.world + threadIdx.x;   // flags already points at the right set
      while (*f < xg.epoch) __nanosleep(20);
      __threadfence_system();   // acquire: the slots this flag guards are read after the CTA barrier
    }
    __syncthreads();
  }
}
__device__ __forceinline__ double xg_load(const XchgGather &xg, const double *acc, int j) {
  if (!xg.world) return acc[j];
  if (xg.rs) return __ldcg(xg.xbuf + (size_t)xg.buf * xg.slot_stride + j);   // reduce-scatter form: the finished sum
  double s = 0.0;
  for (int r = 0; r < xg.world; ++r) s += __ldcg(xg.xbuf + ((size_t)xg.buf * xg.world + r) * xg.slot_stride + j);  // rank order
  return s;
}
// entries d .. n-1 (loss sums, counts, the second block of a two-gradient sweep) for later readers of acc
__device__ __forceinline__ void xg_materialize_tail(const XchgGather &xg, double *acc_w, int d) {
  if (!xg.world) return;
  for (int c = d + blockIdx.x * kK3Threads + threadIdx.x; c < xg.n; c += gridDim.x * kK3Threads) acc_w[c] = xg_load(xg, acc_w, c);
}

// block reduce NS values, write partials, last block sums partials in block order -> scalars (mapped pinned host memory).
// tail != nullptr: scalars[6..7] = tail[0..1] (loss sum, count of the evaluation the kernel consumed).
// seq_out != nullptr: ONE thread stores every scalar, fences at system scope once, then stores the sequence number of this
// launch behind them -- the host waits for it by polling that word instead of synchronising the stream.
template <int NS>
__device__ __forceinline__ void finish_reduce(double (&v)[NS], double *partials, unsigned int *ticket,
                                              double *scalars, const int (&slot)[NS], const double *tail = nullptr,
                                              unsigned long long *seq_out = nullptr, unsigned long long seq = 0ull,
                                              const double *tail_vals = nullptr) {
  __shared__ double sh[NS][kK3Threads / 32];
  __shared__ double fin[NS];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NS; ++i) {
    double x = v[i];
    for (int off = 16; off >= 1; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    if (lane == 0) sh[i][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x < NS) {
    double s = 0.0;
    for (int w = 0; w < kK3Threads / 32; ++w) s += sh[threadIdx.x][w];
    partials[(size_t)blockIdx.x * NS + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(ticket, 1u);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    if (threadIdx.x < NS) {
      double s = 0.0;
      for (unsigned int b = 0; b < gridDim.x; ++b) s += partials[(size_t)b * NS + threadIdx.x];
      fin[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int i = 0; i < NS; ++i) scalars[slot[i]] = fin[i];
      if (tail_vals) { scalars[6] = tail_vals[0]; scalars[7] = tail_vals[1]; }
      else if (tail) { scalars[6] = tail[0]; scalars[7] = tail[1]; }
      *ticket = 0u;
      if (seq_out) {
        __threadfence_system();
        *reinterpret_cast<volatile unsigned long long *>(seq_out) = seq;
      }
    }
  }
}

__global__ void __launch_bounds__(kK3Threads) k3_step_kernel(const K3StepArgs a) {
  xg_wait(a.xg);
  const double count = xg_load(a.xg, a.acc, a.d + 1);
  __shared__ double tailv[2];
  if (threadIdx.x == 0) { tailv[0] = xg_load(a.xg, a.acc, a.d); tailv[1] = count; }
  if (a.hist_out && blockIdx.x == 0 && threadIdx.x == 1) {   // the history evaluation that rode along (:304): straight to the host
    a.hist_out[0] = xg_load(a.xg, a.acc, a.d + 2);
    a.hist_out[1] = xg_load(a.xg, a.acc, a.d + 3);
  }
  double v[6] = {0, 0, 0, 0, 0, 0};
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < a.d; j += gridDim.x * kK3Threads) {
    const double aj = xg_load(a.xg, a.acc, j);
    if (a.xg.world) a.acc_w[j] = aj;
    const double g = __ddiv_rn(aj, count);                                                // :207
    const double xo = a.x_old[j];
    const double z = prox_elem(a.updater, a.z_old[j], g, a.step, a.reg);                  // :254
    const double x = __dadd_rn(__dmul_rn(xo, a.one_minus_theta), __dmul_rn(z, a.theta));  // :255
    a.g_y[j] = g;
    a.z[j] = z;
    a.x[j] = x;
    // the guessed y of the NEXT iteration (:249 with its theta), formed exactly as k3_begin / k3_combine form it
    if (a.y_spec) a.y_spec[j] = __dadd_rn(__dmul_rn(x, a.spec_ca), __dmul_rn(z, a.spec_cb));
    const double xy = __dsub_rn(x, a.y[j]);                                               // :263
    const double dx = __dsub_rn(x, xo);
    v[0] = fma(xy, xy, v[0]);
    v[1] = fma(xy, g, v[1]);
    v[2] = fma(x, x, v[2]);
    v[3] = fma(dx, dx, v[3]);
    v[4] = fma(g, dx, v[4]);
    v[5] += fabs(x);
  }
  xg_materialize_tail(a.xg, a.acc_w, a.d);
  const int slot[6] = {0, 1, 2, 3, 4, 5};
  finish_reduce<6>(v, a.partials, a.ticket, a.scalars, slot, a.acc + a.d, a.seq_out, a.seq, tailv);
}

__global__ void __launch_bounds__(kK3Threads) k3_gx_kernel(const K3GxArgs a) {
  xg_wait(a.xg);
  const double count = xg_load(a.xg, a.acc, a.d + 1);
  __shared__ double tailv[2];
  if (threadIdx.x == 0) { tailv[0] = xg_load(a.xg, a.acc, a.d); tailv[1] = count; }
  double v[1] = {0};
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < a.d; j += gridDim.x * kK3Threads) {
    const double aj = xg_load(a.xg, a.acc, j);
    if (a.xg.world) a.acc_w[j] = aj;
    const double g = __ddiv_rn(aj, count);
    a.g_x[j] = g;
    const double xy = __dsub_rn(a.x[j], a.y[j]);
    const double dg = __dsub_rn(g, a.g_y[j]);
    v[0] = fma(xy, dg, v[0]);                                                             // :278
  }
  xg_materialize_tail(a.xg, a.acc_w, a.d);
  const int slot[1] = {0};
  finish_reduce<1>(v, a.partials, a.ticket, a.scalars, slot, a.acc + a.d, a.seq_out, a.seq, tailv);
}

__global__ void __launch_bounds__(kK3Threads) k3_prox_kernel(const K3ProxArgs a) {
  double v[2] = {0, 0};
  const bool norm = a.acc_tail != nullptr;
  const double count = norm ? a.acc_tail[1] : 1.0;
  const bool skip = norm && !(count > 0.0);  // empty mini-batch: runMiniBatchSGD skips the update
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < a.d; j += gridDim.x * kK3Threads) {
    double g = a.g[j];
    if (norm) g = __ddiv_rn(g, count);
    const double w = skip ? a.w[j] : prox_elem(a.updater, a.w[j], g, a.step, a.reg);
    a.w_out[j] = w;
    v[0] = fma(w, w, v[0]);
    v[1] += fabs(w);
  }
  // scalars[2] = sum w'^2, scalars[5] = sum |w'| (same slots as k3_step)
  const int slot[2] = {2, 5};
  finish_reduce<2>(v, a.partials, a.ticket, a.scalars, slot, norm ? a.acc_tail : nullptr);
}

__global__ void __launch_bounds__(kK3Threads) k3_combine_kernel(double *out, const double *a, double ca,
                                                               const double *b, double cb, int d) {
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < d; j += gridDim.x * kK3Threads)
    out[j] = __dadd_rn(__dmul_rn(a[j], ca), __dmul_rn(b[j], cb));                          // :249
}

// first inner round of an outer iteration: (x_old, z_old) = (x, z) (AGD.scala:241) fused with y (:249)
__global__ void __launch_bounds__(kK3Threads) k3_begin_kernel(double *x_old, double *z_old, double *y, const double *x,
                                                             const double *z, double ca, double cb, int d) {
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < d; j += gridDim.x * kK3Threads) {
    const double xv = x[j], zv = z[j];
    x_old[j] = xv;
    z_old[j] = zv;
    y[j] = __dadd_rn(__dmul_rn(xv, ca), __dmul_rn(zv, cb));
  }
}

__global__ void __launch_bounds__(kK3Threads) k3_copy2_kernel(double *d0, const double *s0, double *d1,
                                                             const double *s1, int d) {
  for (int j = blockIdx.x * kK3Threads + threadIdx.x; j < d; j += gridDim.x * kK3Threads) {
    if (d0) d0[j] = s0[j];
    if (d1) d1[j] = s1[j];
  }
}

}  // namespace

int k3_blocks(int32_t d) {
  int b = (d + kK3Threads * 4 - 1) / (kK3Threads * 4);
  if (b < 1) b = 1;
  if (b > kK3MaxBlocks) b = kK3MaxBlocks;
  return b;
}

cudaError_t k3_step_launch(const K3StepArgs &a, cudaStream_t st) {
  k3_step_kernel<<<k3_blocks(a.d), kK3Threads, 0, st>>>(a);
  return cudaGetLastError();
}
cudaError_t k3_gx_launch(const K3GxArgs &a, cudaStream_t st) {
  k3_gx_kernel<<<k3_blocks(a.d), kK3Threads, 0, st>>>(a);
  return cudaGetLastError();
}
cudaError_t k3_prox_launch(const K3ProxArgs &a, cudaStream_t st) {
  k3_prox_kernel<<<k3_blocks(a.d), kK3Threads, 0, st>>>(a);
  return cudaGetLastError();
}
cudaError_t k3_combine_launch(double *out, const double *a, double ca, const double *b, double cb, int32_t d,
                              cudaStream_t st) {
  k3_combine_kernel<<<k3_blocks(d), kK3Threads, 0, st>>>(out, a, ca, b, cb, d);
  return cudaGetLastError();
}
cudaError_t k3_begin_launch(double *x_old, double *z_old, double *y, const double *x, const double *z, double ca,
                            double cb, int32_t d, cudaStream_t st) {
  k3_begin_kernel<<<k3_blocks(d), kK3Threads, 0, st>>>(x_old, z_old, y, x, z, ca, cb, d);
  return cudaGetLastError();
}
cudaError_t k3_copy2_launch(double *dst0, const double *src0, double *dst1, const double *src1, int32_t d,
                            cudaStream_t st) {
  k3_copy2_kernel<<<k3_blocks(d), kK3Threads, 0, st>>>(dst0, src0, dst1, src1, d);
  return cudaGetLastError();
}

}  // namespace agd
