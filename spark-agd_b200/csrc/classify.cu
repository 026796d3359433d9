// classify.cu -- the small kernels of NaiveBayes and MulticlassMetrics (mllib 1.3.0) on the resident shards, sm_90a.
//
// Everything else they need is the k-means machinery: the radix sort and run-length reduce of rank.cu turn label_keys' keys into
// the distinct labels and their counts; the k-means sums (kmeans.cu, kKmNegatives) add each class's rows; the k-means assignment
// (kmeans.cu, kKmLinear) scores every class of a linear model at once.  These kernels only read labels and class indices:
//   * label_keys: the view's non-NaN labels as ascending 64-bit keys, compacted by one atomic per warp and step (score.cu's key
//     form); NaN labels are only counted;
//   * label_class: each row's class by binary search over the ascending class labels;
//   * label_confusion: exact (label index, predicted class) counts in shared-memory histograms.  The L x C counters are cut into
//     slices of whole label rows that fit in 48 KB; blockIdx.y is the slice, and its CTAs count only the rows whose label falls
//     in it (every slice reads the labels and classes once more, which costs far less than global atomics on the few
//     addresses a good model's diagonal takes).  Counts are integers, so the result does not depend on the order.
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"

namespace agd {

namespace {

constexpr int kClsThreads = 256;
constexpr int kClsSmemCounters = 48 * 1024 / (int)sizeof(unsigned);

__device__ __forceinline__ bool cls_in_view(const uint32_t *bits, long long r) {
  return !bits || ((bits[r >> 5] >> (r & 31)) & 1u);
}

// the index of y in the C ascending classes, -1 when it is none of them (a NaN y compares false everywhere)
__device__ __forceinline__ int cls_find(const double *classes, int C, double y) {
  int lo = 0, hi = C;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (classes[mid] < y) lo = mid + 1;
    else hi = mid;
  }
  return lo < C && classes[lo] == y ? lo : -1;
}

unsigned cls_grid(long long rows, long long cap) {
  long long g = (rows + kClsThreads - 1) / kClsThreads;
  if (g > cap) g = cap;
  return (unsigned)(g > 0 ? g : 1);
}

// warp-uniform loop: every lane of a warp takes part in each step's ballots
__global__ void __launch_bounds__(kClsThreads) label_keys_kernel(const double *__restrict__ labels, const uint32_t *view_bits,
                                                                 long long rows, unsigned long long *keys, uint8_t *ones,
                                                                 unsigned *counters) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * kClsThreads;
  for (long long i0 = (long long)blockIdx.x * kClsThreads + (threadIdx.x & ~31); i0 < rows; i0 += stride) {
    const long long i = i0 + lane;
    const bool in = i < rows && cls_in_view(view_bits, i);
    const double y = in ? labels[i] : 0.0;
    const bool nan = in && y != y, emit = in && !nan;
    const unsigned em = __ballot_sync(0xffffffffu, emit), nm = __ballot_sync(0xffffffffu, nan);
    unsigned base = 0;
    if (lane == 0 && em) base = atomicAdd(counters, (unsigned)__popc(em));
    if (lane == 0 && nm) atomicAdd(counters + 1, (unsigned)__popc(nm));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (emit) {
      const unsigned o = base + __popc(em & ((1u << lane) - 1u));
      keys[o] = label_key(y);
      ones[o] = 1;
    }
  }
}

__global__ void __launch_bounds__(kClsThreads) label_class_kernel(const double *__restrict__ labels, const uint32_t *view_bits,
                                                                  long long rows, const double *__restrict__ classes, int C,
                                                                  int32_t *cls) {
  const long long stride = (long long)gridDim.x * kClsThreads;
  for (long long i = (long long)blockIdx.x * kClsThreads + threadIdx.x; i < rows; i += stride)
    cls[i] = cls_in_view(view_bits, i) ? cls_find(classes, C, labels[i]) : -1;
}

// label rows l0 .. l0 + lps - 1 (slice blockIdx.y) of the counts
__global__ void __launch_bounds__(kClsThreads) label_confusion_kernel(const double *__restrict__ labels,
                                                                      const int32_t *__restrict__ pred, long long rows,
                                                                      const double *__restrict__ classes, int L, int C, int lps,
                                                                      unsigned long long *counts) {
  extern __shared__ unsigned cnt_sh[];
  const int l0 = (int)blockIdx.y * lps, l1 = l0 + lps < L ? l0 + lps : L;
  const int n = (l1 - l0) * C;
  for (int q = threadIdx.x; q < n; q += kClsThreads) cnt_sh[q] = 0;
  __syncthreads();
  const long long stride = (long long)gridDim.x * kClsThreads;
  for (long long i = (long long)blockIdx.x * kClsThreads + threadIdx.x; i < rows; i += stride) {
    const int c = pred[i];
    if (c < 0) continue;
    const int l = cls_find(classes, L, labels[i]);
    if (l >= l0 && l < l1) atomicAdd(cnt_sh + (l - l0) * C + c, 1u);
  }
  __syncthreads();
  unsigned long long *out = counts + (size_t)l0 * C;
  for (int q = threadIdx.x; q < n; q += kClsThreads)
    if (cnt_sh[q]) atomicAdd(out + q, (unsigned long long)cnt_sh[q]);
}

}  // namespace

cudaError_t label_keys_launch(const double *labels, const uint32_t *view_bits, long long rows, unsigned long long *keys,
                              uint8_t *ones, unsigned *counters, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  label_keys_kernel<<<cls_grid(rows, 4096), kClsThreads, 0, st>>>(labels, view_bits, rows, keys, ones, counters);
  return cudaGetLastError();
}

cudaError_t label_class_launch(const double *labels, const uint32_t *view_bits, long long rows, const double *classes,
                               int32_t C, int32_t *cls, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  label_class_kernel<<<cls_grid(rows, 4096), kClsThreads, 0, st>>>(labels, view_bits, rows, classes, C, cls);
  return cudaGetLastError();
}

cudaError_t label_confusion_launch(const double *labels, const int32_t *pred, long long rows, const double *classes, int32_t L,
                                   int32_t C, unsigned long long *counts, int sm_count, cudaStream_t st) {
  if (rows <= 0) return cudaSuccess;
  if (L < 1 || C < 1 || C > kClsSmemCounters) return cudaErrorInvalidValue;
  const int lps = L < kClsSmemCounters / C ? L : kClsSmemCounters / C;   // label rows per slice
  const unsigned slices = (unsigned)((L + lps - 1) / lps);
  // a few CTAs per SM and slice: each zeroes and flushes its counters once, so the grid stays small
  const dim3 grid(cls_grid(rows, 4 * (long long)sm_count), slices);
  label_confusion_kernel<<<grid, kClsThreads, (size_t)lps * C * sizeof(unsigned), st>>>(labels, pred, rows, classes, L, C, lps,
                                                                                       counts);
  return cudaGetLastError();
}

}  // namespace agd
