// xchg.cu -- K2': the one-shot all-reduce over NVLink peer memory (see agd_common.cuh for the protocol).
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"

namespace agd {

namespace {

// the gather's reduction over the W slots (kXchgSum / kXchgMax, agd_common.cuh), applied in rank order
template <int OP> struct XchgOp;
template <> struct XchgOp<kXchgSum> {
  __device__ static double init() { return 0.0; }
  __device__ static double apply(double s, double v) { return s + v; }
};
template <> struct XchgOp<kXchgMax> {
  __device__ static double init() { return __longlong_as_double(0x7ff8000000000000LL); }   // NaN: fmax ignores it
  __device__ static double apply(double s, double v) { return fmax(s, v); }
};

// standalone publish (the CSR path has no slab reduction to fuse it into)
__global__ void __launch_bounds__(256) xchg_publish_kernel(const double *__restrict__ acc, const XchgPub pub) {
  __shared__ bool last;
  const size_t base = ((size_t)pub.buf * pub.world + pub.my_rank) * pub.slot_stride;
  for (int c = blockIdx.x * 256 + threadIdx.x; c < pub.n; c += gridDim.x * 256) {
    const double v = acc[c];
    for (int p = 0; p < pub.world; ++p) pub.peers.slot[p][base + c] = v;
  }
  __syncthreads();   // one cumulative system-scope fence per block (see k1_reduce_kernel)
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

// wait for the W flags of this epoch, then add (or max) the W slots in rank order (identical bits on every rank)
template <int OP>
__global__ void __launch_bounds__(256) xchg_gather_kernel(const XchgGather g, double *acc_out) {
  if (threadIdx.x < g.world) {
    const volatile unsigned long long *f = g.flags + g.buf * g.world + threadIdx.x;
    while (*f < g.epoch) __nanosleep(20);
    __threadfence_system();   // acquire: the slot data this flag guards is read (ld.cg, from L2) after the CTA barrier
  }
  __syncthreads();
  for (int c = blockIdx.x * 256 + threadIdx.x; c < g.n; c += gridDim.x * 256) {
    double s = XchgOp<OP>::init();
    for (int r = 0; r < g.world; ++r) s = XchgOp<OP>::apply(s, __ldcg(g.xbuf + ((size_t)g.buf * g.world + r) * g.slot_stride + c));  // written remotely: bypass L1
    acc_out[c] = s;
  }
}

// kXchgCopy: wait for the W flags of this epoch, then concatenate the W slots in rank order (plain moves: the bits travel)
__global__ void __launch_bounds__(256) xchg_gather_copy_kernel(const XchgGather g, double *out, size_t out_stride) {
  if (threadIdx.x < g.world) {
    const volatile unsigned long long *f = g.flags + g.buf * g.world + threadIdx.x;
    while (*f < g.epoch) __nanosleep(20);
    __threadfence_system();
  }
  __syncthreads();
  for (int c = blockIdx.x * 256 + threadIdx.x; c < g.n; c += gridDim.x * 256)
    for (int r = 0; r < g.world; ++r) out[(size_t)r * out_stride + c] = __ldcg(g.xbuf + ((size_t)g.buf * g.world + r) * g.slot_stride + c);
}

// ---- reduce-scatter + all-gather for large payloads (see agd_common.cuh)
// step 1: slice p of this rank's partial sums -> slot my_rank of rank p's rs area; then the "arrived" flag on every peer
__global__ void __launch_bounds__(256) xchg_rs_publish_kernel(const double *__restrict__ acc, const XchgPub x) {
  __shared__ bool last;
  const int W = x.world, S = x.slot_stride;
  const size_t L = xchg_rs_slice(S, W);                          // slot capacity
  const int l = (x.n + W - 1) / W;                               // slice length of this sweep
  const size_t off_rs = xchg_off_rs(S, W);
  for (int c = blockIdx.x * 256 + threadIdx.x; c < x.n; c += gridDim.x * 256) {
    const int p = c / l;
    x.peers.slot[p][off_rs + ((size_t)x.buf * W + x.my_rank) * L + (size_t)(c - p * l)] = acc[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    last = (atomicAdd(x.ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    if (threadIdx.x < W) {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned long long *>(&x.peers.flag[threadIdx.x][xchg_flags_rs(W) + x.buf * W + x.my_rank]) = x.epoch;
    }
    if (threadIdx.x == 0) *x.ticket = 0u;
  }
}

// step 2: wait for the W contributions to MY slice, add (or max) them in rank order, store the finished slice into every rank's res area
template <int OP>
__global__ void __launch_bounds__(256) xchg_rs_reduce_bcast_kernel(const double *xbuf, const unsigned long long *flags, const XchgPub x) {
  __shared__ bool last;
  const int W = x.world, S = x.slot_stride;
  const size_t L = xchg_rs_slice(S, W);
  const int l = (x.n + W - 1) / W;
  const size_t off_rs = xchg_off_rs(S, W), off_res = xchg_off_res(S, W);
  if (threadIdx.x < W) {
    const volatile unsigned long long *f = flags + xchg_flags_rs(W) + x.buf * W + threadIdx.x;
    while (*f < x.epoch) __nanosleep(20);
    __threadfence_system();
  }
  __syncthreads();
  const int c0 = x.my_rank * l;
  int len = x.n - c0;
  if (len > l) len = l;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < len; i += gridDim.x * 256) {
    double s = XchgOp<OP>::init();
    for (int r = 0; r < W; ++r) s = XchgOp<OP>::apply(s, __ldcg(xbuf + off_rs + ((size_t)x.buf * W + r) * L + i));   // rank order: identical bits everywhere
    const size_t dst = off_res + (size_t)x.buf * S + (size_t)(c0 + i);
    for (int q = 0; q < W; ++q) x.peers.slot[q][dst] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    last = (atomicAdd(x.ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    if (threadIdx.x < W) {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned long long *>(&x.peers.flag[threadIdx.x][xchg_flags_res(W) + x.buf * W + x.my_rank]) = x.epoch;
    }
    if (threadIdx.x == 0) *x.ticket = 0u;
  }
}

// step 3 (stand-alone form; K3 kernels inline it): wait for the W finished slices, copy them out.  g points at the res area
// and at the "finished slice arrived" flags.
__global__ void __launch_bounds__(256) xchg_rs_gather_kernel(const XchgGather g, double *acc_out) {
  if (threadIdx.x < g.world) {
    const volatile unsigned long long *f = g.flags + g.buf * g.world + threadIdx.x;
    while (*f < g.epoch) __nanosleep(20);
    __threadfence_system();
  }
  __syncthreads();
  const double *res = g.xbuf + (size_t)g.buf * g.slot_stride;
  for (int c = blockIdx.x * 256 + threadIdx.x; c < g.n; c += gridDim.x * 256) acc_out[c] = __ldcg(res + c);
}

}  // namespace

cudaError_t xchg_publish_launch(const double *acc, const XchgPub &pub, cudaStream_t st) {
  int grid = (pub.n + 255) / 256;
  if (grid > 64) grid = 64;
  xchg_publish_kernel<<<grid, 256, 0, st>>>(acc, pub);
  return cudaGetLastError();
}

cudaError_t xchg_rs_publish_launch(const double *acc, const XchgPub &x, cudaStream_t st) {
  int grid = (x.n + 255) / 256;
  if (grid > 264) grid = 264;
  xchg_rs_publish_kernel<<<grid, 256, 0, st>>>(acc, x);
  return cudaGetLastError();
}

cudaError_t xchg_rs_reduce_bcast_launch(const double *xbuf_local, const unsigned long long *flags_local, const XchgPub &x, cudaStream_t st,
                                        int op) {
  const int l = (x.n + x.world - 1) / x.world;
  int grid = (l + 255) / 256;
  if (grid > 132) grid = 132;   // one CTA per H100 SM
  if (grid < 1) grid = 1;
  if (op == kXchgMax) xchg_rs_reduce_bcast_kernel<kXchgMax><<<grid, 256, 0, st>>>(xbuf_local, flags_local, x);
  else xchg_rs_reduce_bcast_kernel<kXchgSum><<<grid, 256, 0, st>>>(xbuf_local, flags_local, x);
  return cudaGetLastError();
}

cudaError_t xchg_gather_launch(const XchgGather &g, double *out, size_t out_stride, int op, cudaStream_t st) {
  int grid = (g.n + 255) / 256;
  if (op == kXchgCopy) {
    if (grid > 64) grid = 64;
    if (grid < 1) grid = 1;
    xchg_gather_copy_kernel<<<grid, 256, 0, st>>>(g, out, out_stride);
  } else if (g.rs) {
    if (grid > 264) grid = 264;
    xchg_rs_gather_kernel<<<grid, 256, 0, st>>>(g, out);
  } else {
    if (grid > 64) grid = 64;
    if (op == kXchgMax) xchg_gather_kernel<kXchgMax><<<grid, 256, 0, st>>>(g, out);
    else xchg_gather_kernel<kXchgSum><<<grid, 256, 0, st>>>(g, out);
  }
  return cudaGetLastError();
}

}  // namespace agd
