// agd_api.cu -- the C-ABI of include/agd_b200.h: handle, shard loading, the collective, and the
// AcceleratedGradientDescent.run driver loop (AGD.scala:177-338) executed natively around the
// K1 / all-reduce / K3 kernels.  No CPU fallback: every compute entry point needs an sm_90 GPU.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only; the library is dlopen'ed (torch ships its own libnccl.so.2)
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <functional>
#include <limits>
#include <mutex>
#include <string>
#include <vector>

#include "agd_common.cuh"

using namespace agd;

// ---------------------------------------------------------------- NCCL through dlopen
namespace {

struct NcclApi {
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool ok = false;
  std::string why;
};

NcclApi &nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) { api.why = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return; }
#define AGD_NCCL_SYM(name)                                                   \
  api.name = reinterpret_cast<decltype(api.name)>(dlsym(lib, "nccl" #name)); \
  if (!api.name) { api.why = "missing symbol nccl" #name; return; }
    AGD_NCCL_SYM(GetUniqueId)
    AGD_NCCL_SYM(CommInitRank)
    AGD_NCCL_SYM(AllReduce)
    AGD_NCCL_SYM(AllGather)
    AGD_NCCL_SYM(GroupStart)
    AGD_NCCL_SYM(GroupEnd)
    AGD_NCCL_SYM(CommDestroy)
    AGD_NCCL_SYM(GetErrorString)
#undef AGD_NCCL_SYM
    api.ok = true;
  });
  return api;
}

std::string g_create_error;
std::mutex g_create_mu;

struct Shard {
  void *X = nullptr;          // dense, row-major, ld == d
  double *labels = nullptr;   // cap + pad
  int64_t rows = 0, cap = 0;
  int elem_bytes = 0;         // 4 (fp32) or 8 (fp64) storage
  bool csr = false;
  int64_t *rowptr = nullptr;
  int32_t *idx = nullptr;
  void *val = nullptr;
  int64_t nnz = 0, nnz_cap = 0;
};

// agd_binary_curve's scratch buffers on a device
enum BinBuf {
  kBinKeys0, kBinKeys1,   // keys of a sort (ping-pong): the view's rows, then on device 0 the world's concatenated lists
  kBinVals0, kBinVals1,   // their values: classes (1 byte), then indices (4 bytes)
  kBinMisc,               // [8 x 256 digit counts | counters (2 u32) | runs (i64) | areas (2) | own {len, nan} (2) | world's {len, nan} | offsets]
  kBinTiles,              // per-tile digit counts / sums of the scans / area partials
  kBinList,               // this device's curve: BinRec per distinct key
  kBinUnion,              // the world's lists, rank r's at r * (longest list)
  kBinCounts,             // each concatenated record's own counts: pos [T] | neg [T]
  kBinCurve,              // the world's curve
  kBinBufs
};
// agd_kmeans_* scratch buffers on a device
enum KmBuf {
  kKmCluster,             // each row's centre (int32), or each sampled row's bit
  kKmDelta,               // agd_kmeans_costs' per-row cost
  kKmCentres,             // the centres as the kernels read them: B | cb | cn | C
  kKmTiles,               // per column tile: best score (double) of each row | its index (int32)
  kKmKeys0, kKmKeys1,     // the stable sort of (centre, row)
  kKmVals0, kKmVals1,
  kKmSortTiles,           // the sort's per-tile digit counts
  kKmMisc,                // [8 x 256 digit counts | counts (k + 1) u64] / sampling: [tile_base | total] | lengths
  kKmPieces,              // pstart | pcl | pfirst of the dense sums
  kKmPart,                // per-piece sums | per-piece residuals | column residuals
  kKmPayload,             // [sums k x md | counts k | cost], exchanged over the world
  kKmRows,                // sampled rows, this device's at its rank's block of the world's
  kKmClasses,             // agd_class_sums / agd_linear_confusion: the class labels (doubles) | confusion counts (u64)
  kKmBufs
};
constexpr size_t kBinMiscCounters = 8 * 256 * sizeof(unsigned), kBinMiscRuns = kBinMiscCounters + 8,
                 kBinMiscAreas = kBinMiscRuns + 8, kBinMiscOwn = kBinMiscAreas + 16, kBinMiscAll = kBinMiscOwn + 16;

struct Dev {
  int ordinal = -1;
  int sm_count = 0;
  cudaStream_t st = nullptr;
  Shard sh;
  // d-vectors of the driver loop (AGD.scala:224-230,241,249) + packed pass result
  double *x = nullptr, *z = nullptr, *x_old = nullptr, *z_old = nullptr, *y = nullptr, *g_y = nullptr,
         *g_x = nullptr, *wtmp = nullptr, *acc = nullptr, *y_spec = nullptr;
  int32_t vec_d = 0;
  double *slabs = nullptr;
  size_t slabs_doubles = 0;
  double *eval = nullptr;          // AGD_EVAL_N sums of agd_evaluate (this shard's, then the world's)
  double *cs = nullptr;            // agd_col_stats: pass-1 sums, maxima, pass-2 sums, CSR max keys (see colstats_layout)
  size_t cs_doubles = 0;
  double *gm = nullptr;            // agd_gramian: packed result, mu, pass-1 sums, CSR keys, slabs (see gramian_layout)
  size_t gm_doubles = 0;
  void *bin[kBinBufs] = {};        // agd_binary_curve scratch (see BinBuf), grown on demand, freed by agd_clear / agd_destroy
  size_t bin_bytes[kBinBufs] = {};
  void *km[kKmBufs] = {};          // agd_kmeans_* scratch (see KmBuf), grown on demand, freed by agd_clear / agd_destroy
  size_t km_bytes[kKmBufs] = {};
  int64_t km_delta_rows = -1;      // rows kKmDelta describes (-1: no agd_kmeans_costs since the last load or clear)
  double *partials = nullptr;
  unsigned int *ticket = nullptr;
  double *scalars_dev = nullptr;   // device alias of scalars_host: K3 writes its scalars straight to the host
  double *scalars_host = nullptr;  // pinned + mapped, 2*K3_NS
  void *stage_dev = nullptr;
  size_t stage_bytes = 0;
  ncclComm_t comm = nullptr;
  std::vector<cudaEvent_t> ev;     // K1 start/stop pairs (device 0 only)
  size_t ev_used = 0;
  std::vector<cudaEvent_t> ev_ar;  // all-reduce start/stop pairs
  size_t ev_ar_used = 0;
  std::mutex *mu = nullptr;
  long long row_base = 0;          // global index of this shard's first row (for the sampling mask)
  RowFilter *filt_dev = nullptr;   // device copy of the handle's row filter (agd_set_row_filter)
  uint32_t *view_bits = nullptr;   // the filter as a bitmap of this shard's rows (the ring kernel reads it), see ensure_view_bits
  size_t view_bits_words = 0;      // capacity
  int64_t view_bits_rows = -1;     // rows the bitmap describes (-1: none) ...
  long long view_bits_base = 0;    // ... numbered from this row_base ...
  RowFilter view_bits_filt;        // ... under this filter
  double *tf_scale = nullptr;      // the feature scaling of agd_set_feature_transform: d doubles (zero on padded columns) ...
  double *weff = nullptr, *weff2 = nullptr;   // ... and the points K1 evaluates under it, (s o v, b) at w and at w2
  int32_t tf_cap = 0;              // capacity of the three, in doubles
  double *hist_host = nullptr;            // pinned + mapped: [2k] = loss sum, [2k+1] = count of the history pass of iteration k
  double *hist_dev = nullptr;             // device alias of hist_host (k3_step stores the pair that rode along with a fused sweep)
  size_t hist_cap = 0;
  // K2' peer-memory exchange (xchg.cu)
  double *xbuf = nullptr;                 // [2][W][xchg_slot_stride(d)] (+ reduce-scatter areas), written by every rank over NVLink
  unsigned long long *xflags = nullptr;   // [2][W] epochs
  unsigned int *xticket = nullptr;
  XchgPeers xpeers;                       // every rank's xbuf / xflags as mapped into this device
  std::vector<void *> xopened;            // cudaIpcOpenMemHandle mappings to close
};

// One epoch of the cross-rank exchange (open_epoch and the helpers around it)
struct Epoch {
  unsigned long long e = 0;   // 0: none (one rank, NCCL, or no exchange pending)
  int n = 0;                  // doubles per rank
  bool rs = false;            // reduce-scatter form (n >= kXchgRsMin)
  bool bulk = false;          // through the bulk area, kXchgBulk doubles per slot
};

}  // namespace

struct agd_handle {
  std::vector<Dev> devs;
  int32_t d = 0;       // INTERNAL dimension: d_user padded with zero columns so that rows are whole 16-byte vectors
  int32_t d_user = 0;  // the caller's feature count (what agd_dim reports)
  int world = 1, first_rank = 0;
  bool comm_ready = false;
  bool comm_auto = false;   // the world is this process's own GPUs (agd_create): NCCL is only built if it is ever needed
  bool ipc_only = false;    // agd_comm_init_ipc: no NCCL at all, the host ships the CUDA IPC handles (agd_xchg_export/import)
  int k1_variant = 0;  // 0 auto, 1 ring, 2 generic, 4 wgmma (bf16)
  int ring_stages = 0;
  int tune_rows = 0, tune_ctas = 0, tune_full = 0;
  int k1_diag = 0;
  int tc_margins_f64 = 0;    // wgmma kernel: fp64-exact margins instead of the fp32 phase 1
  unsigned long long sample_seed = 0, sample_thresh = 0;  // mini-batch row mask of the current pass (0 = every row)
  RowFilter filt;            // the view every collective sweep runs on (agd_set_row_filter; n = 0: every row) ...
  const RowFilter *filt_of(const Dev &D) const { return filt.n ? D.filt_dev : nullptr; }   // ... as the kernels get it
  // The feature transform of agd_set_feature_transform: the model is (v, b) on appendBias(s o x).  Only K1's row loop runs in
  // the stored width d; every vector of the solver, the payload and its offsets use the MODEL dimension model_d() = d + bias,
  // in which the intercept is the last weight (index d internally, d_user for the caller).
  bool tf_scale = false;
  int32_t tf_bias = 0;
  std::vector<double> tf_scale_host;   // the scale factors, d_user of them (k-means folds them into its centres on the host)
  int32_t model_d() const { return d + tf_bias; }
  const double *scale_of(const Dev &D) const { return tf_scale ? D.tf_scale : nullptr; }
  int collective = 0;        // 0 = auto (peer memory if every pair of ranks can map each other, else NCCL), 1 = nccl, 2 = p2p
  int32_t x_d = 0;           // dimension the exchange buffers were built for (0 = not built)
  bool x_p2p = false;        // exchange buffers are live
  unsigned long long x_epoch = 0;
  Epoch pending;             // a sweep whose gather was left to the K3 kernel that consumes it (smooth_device(..., defer_gather))
  std::string err;
  std::mutex mu;
  unsigned long long seq_base = 0;   // last round sequence number handed out (wait_scalars)
  // AGD_TRACE=1 (diagnostics): an event after every launch on device 0; agd_run prints per-kernel totals (gap + run time) to stderr
  int trace = -1;
  std::vector<std::pair<const char *, cudaEvent_t>> tr;
  std::vector<cudaEvent_t> tr_pool;
  int64_t launches = 0;  // per device, current call
  int64_t collectives = 0;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
};

namespace {

int fail(agd_handle *h, const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  else {
    std::lock_guard<std::mutex> g(g_create_mu);
    g_create_error = buf;
  }
  return 1;
}

#define CK(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) return fail(h, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)
#define CKN(call)                                                                                        \
  do {                                                                                                   \
    ncclResult_t r_ = (call);                                                                            \
    if (r_ != ncclSuccess) return fail(h, "%s failed: %s (%s:%d)", #call, nccl_api().GetErrorString(r_), __FILE__, __LINE__); \
  } while (0)

// Java Math.max / Math.min (NaN-propagating), used at AGD.scala:274,275,286,292,322
double jmax(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return std::signbit(a) ? b : a;
  return a > b ? a : b;
}
double jmin(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return std::signbit(a) ? a : b;
  return a < b ? a : b;
}

int dtype_bytes(int dt) { return dt == AGD_F64 ? 8 : (dt == AGD_F32 ? 4 : (dt == AGD_BF16 ? 2 : 0)); }
int bytes_dtype(int eb) { return eb == 8 ? AGD_F64 : (eb == 4 ? AGD_F32 : AGD_BF16); }

int free_shard(agd_handle *h, Dev &D) {
  CK(cudaSetDevice(D.ordinal));
  Shard &s = D.sh;
  if (s.X) cudaFree(s.X);
  if (s.labels) cudaFree(s.labels);
  if (s.rowptr) cudaFree(s.rowptr);
  if (s.idx) cudaFree(s.idx);
  if (s.val) cudaFree(s.val);
  s = Shard();
  return 0;
}

int ensure_vectors(agd_handle *h, Dev &D, int32_t d) {
  if (D.vec_d >= d) return 0;   // a model with an intercept is one longer: switching a transform on and off reallocates nothing
  CK(cudaSetDevice(D.ordinal));
  double **v[] = {&D.x, &D.z, &D.x_old, &D.z_old, &D.y, &D.g_y, &D.g_x, &D.wtmp, &D.y_spec};
  for (double **p : v) {
    if (*p) cudaFree(*p);
    *p = nullptr;
    CK(cudaMalloc(p, ((size_t)d + 4) * sizeof(double)));
    CK(cudaMemsetAsync(*p, 0, ((size_t)d + 4) * sizeof(double), D.st));
  }
  if (D.acc) cudaFree(D.acc);
  // [grad(d) | loss | count | loss at w2 | count at w2], and after a two-gradient sweep a second block [grad at w2 | loss | count | 0 | 0]
  CK(cudaMalloc(&D.acc, 2 * ((size_t)d + 4) * sizeof(double)));
  if (D.partials) cudaFree(D.partials);
  CK(cudaMalloc(&D.partials, (size_t)k3_blocks(d) * K3_NS * sizeof(double)));
  D.vec_d = d;
  return 0;
}

// A point of the model (d_user + bias doubles from the caller) -> dst (model_d() doubles on the device): the features, zero
// weights on the padded columns, the intercept last.  And back.
int put_point(agd_handle *h, Dev &D, double *dst, const double *w) {
  CK(cudaMemsetAsync(dst, 0, ((size_t)h->model_d() + 2) * sizeof(double), D.st));
  CK(cudaMemcpyAsync(dst, w, (size_t)h->d_user * sizeof(double), cudaMemcpyHostToDevice, D.st));
  if (h->tf_bias) CK(cudaMemcpyAsync(dst + h->d, w + h->d_user, sizeof(double), cudaMemcpyHostToDevice, D.st));
  return 0;
}
int get_point(agd_handle *h, Dev &D, double *w_out, const double *src) {
  CK(cudaMemcpyAsync(w_out, src, (size_t)h->d_user * sizeof(double), cudaMemcpyDeviceToHost, D.st));
  if (h->tf_bias) CK(cudaMemcpyAsync(w_out + h->d_user, src + h->d, sizeof(double), cudaMemcpyDeviceToHost, D.st));
  return 0;
}
// the same on host memory: the caller's d_user + bias values of a model_d() vector, divided by `div`
void model_values(const agd_handle *h, const double *src, double div, double *out) {
  for (int32_t j = 0; j < h->d_user; ++j) out[j] = src[j] / div;
  if (h->tf_bias) out[h->d_user] = src[h->d] / div;
}

int ensure_slabs(agd_handle *h, Dev &D, int blocks, int32_t n) {
  const size_t need = (size_t)blocks * (size_t)n;
  if (need <= D.slabs_doubles) return 0;
  CK(cudaSetDevice(D.ordinal));
  if (D.slabs) cudaFree(D.slabs);
  D.slabs = nullptr;
  CK(cudaMalloc(&D.slabs, need * sizeof(double)));
  D.slabs_doubles = need;
  return 0;
}

// elem_bytes > 0: dense storage -- rows are padded with zero columns to whole 16-byte vectors when that puts the
// shard on the TMA-ring / wgmma kernels.  The solver then runs in the padded dimension, which is bit-identical:
// the extra gradient entries are exactly 0, so the extra weights stay exactly 0 under every updater.
int set_dim(agd_handle *h, int32_t d, int elem_bytes = 0) {
  std::lock_guard<std::mutex> g(h->mu);
  if (d <= 0) return fail(h, "feature dimension must be positive (got %d)", d);
  if (h->d_user == 0) {
    h->d_user = d;
    h->d = d;
    if (elem_bytes > 0) {
      const int epv = 16 / elem_bytes;
      const int padded = (d + epv - 1) / epv * epv;
      if (padded != d && k1_ring_supported(padded, elem_bytes)) h->d = padded;
    }
  } else if (h->d_user != d) {
    return fail(h, "feature dimension mismatch: shard has d=%d, call passed d=%d", h->d_user, d);
  }
  return 0;
}

int reserve_locked(agd_handle *h, Dev &D, int64_t cap, int32_t d, int store_dtype) {
  const int eb = dtype_bytes(store_dtype);
  if (!eb) return fail(h, "store_dtype must be AGD_F64, AGD_F32 or AGD_BF16");
  if (cap < 0) return fail(h, "negative capacity");
  CK(cudaSetDevice(D.ordinal));
  Shard &s = D.sh;
  if (s.csr) return fail(h, "device already holds a CSR shard");
  if (s.cap > 0 && s.elem_bytes != eb) return fail(h, "storage dtype mismatch with the resident shard");
  if (cap <= s.cap) {
    if (!s.elem_bytes) s.elem_bytes = eb;  // an empty shard still records its storage type
    return 0;
  }
  void *nx = nullptr;
  double *nl = nullptr;
  const size_t xbytes = (size_t)cap * d * eb + 64;
  CK(cudaMalloc(&nx, xbytes));
  CK(cudaMalloc(&nl, ((size_t)cap + 64) * sizeof(double)));
  CK(cudaMemsetAsync(nl, 0, ((size_t)cap + 64) * sizeof(double), D.st));
  if (s.rows > 0) {
    CK(cudaMemcpyAsync(nx, s.X, (size_t)s.rows * d * eb, cudaMemcpyDeviceToDevice, D.st));
    CK(cudaMemcpyAsync(nl, s.labels, (size_t)s.rows * sizeof(double), cudaMemcpyDeviceToDevice, D.st));
  }
  CK(cudaStreamSynchronize(D.st));
  if (s.X) cudaFree(s.X);
  if (s.labels) cudaFree(s.labels);
  s.X = nx;
  s.labels = nl;
  s.cap = cap;
  s.elem_bytes = eb;
  return 0;
}

int ensure_stage(agd_handle *h, Dev &D, size_t bytes) {
  if (D.stage_bytes >= bytes) return 0;
  if (D.stage_dev) cudaFree(D.stage_dev);
  D.stage_dev = nullptr;
  CK(cudaMalloc(&D.stage_dev, bytes));
  D.stage_bytes = bytes;
  return 0;
}

int ensure_bin(agd_handle *h, Dev &D, int which, size_t bytes) {
  if (D.bin_bytes[which] >= bytes) return 0;
  if (D.bin[which]) cudaFree(D.bin[which]);
  D.bin[which] = nullptr;
  D.bin_bytes[which] = 0;
  if (cudaMalloc(&D.bin[which], bytes) != cudaSuccess) {
    cudaGetLastError();
    return fail(h, "agd_binary_curve: cannot allocate %zu bytes of scratch on device %d", bytes, D.ordinal);
  }
  D.bin_bytes[which] = bytes;
  return 0;
}
void free_bin(Dev &D) {
  for (int i = 0; i < kBinBufs; ++i) {
    if (D.bin[i]) cudaFree(D.bin[i]);
    D.bin[i] = nullptr;
    D.bin_bytes[i] = 0;
  }
}
void free_km(Dev &D) {
  for (int i = 0; i < kKmBufs; ++i) {
    if (D.km[i]) cudaFree(D.km[i]);
    D.km[i] = nullptr;
    D.km_bytes[i] = 0;
  }
  D.km_delta_rows = -1;
}

int ensure_km(agd_handle *h, Dev &D, int which, size_t bytes) {
  if (D.km_bytes[which] >= bytes) return 0;
  if (D.km[which]) cudaFree(D.km[which]);
  D.km[which] = nullptr;
  D.km_bytes[which] = 0;
  if (which == kKmDelta) D.km_delta_rows = -1;
  if (cudaMalloc(&D.km[which], bytes) != cudaSuccess) {
    cudaGetLastError();
    return fail(h, "agd_kmeans: cannot allocate %zu bytes of scratch on device %d", bytes, D.ordinal);
  }
  D.km_bytes[which] = bytes;
  return 0;
}

// The current filter as a bitmap of D's rows, drawn by the kernels' own row_in_view() (one launch, one Philox per row and
// predicate): rebuilt when the filter, the shard's row count or its row numbering changed since the last build, so a run of
// many sweeps on one view draws its rows once.  One bit per row (rows / 8 bytes next to the shard).
int ensure_view_bits(agd_handle *h, Dev &D) {
  if (h->filt.n == 0) return 0;
  const int64_t rows = D.sh.rows;
  const RowFilter &f = h->filt;
  bool same = D.view_bits_rows == rows && D.view_bits_base == D.row_base && D.view_bits_filt.n == f.n;
  for (int i = 0; same && i < f.n; ++i)
    same = D.view_bits_filt.seed[i] == f.seed[i] && D.view_bits_filt.lo[i] == f.lo[i] && D.view_bits_filt.hi[i] == f.hi[i] &&
           D.view_bits_filt.flags[i] == f.flags[i];
  if (same) return 0;
  const size_t words = (size_t)((rows + 31) / 32) + 1;
  if (D.view_bits_words < words) {
    if (D.view_bits) cudaFree(D.view_bits);
    D.view_bits = nullptr;
    D.view_bits_words = 0;
    CK(cudaMalloc(&D.view_bits, words * sizeof(uint32_t)));
    D.view_bits_words = words;
  }
  CK(row_filter_bits_launch(D.filt_dev, D.row_base, rows, D.view_bits, D.st));
  if (&D == &h->devs[0]) h->launches += 1;
  D.view_bits_rows = rows;
  D.view_bits_base = D.row_base;
  D.view_bits_filt = f;
  return 0;
}

cudaEvent_t next_event(std::vector<cudaEvent_t> &pool, size_t &used) {
  if (used == pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    pool.push_back(e);
  }
  return pool[used++];
}


void free_xchg(agd_handle *h) {
  for (Dev &D : h->devs) {
    cudaSetDevice(D.ordinal);
    for (void *p : D.xopened) cudaIpcCloseMemHandle(p);
    D.xopened.clear();
    if (D.xbuf) cudaFree(D.xbuf);
    if (D.xflags) cudaFree(D.xflags);
    if (D.xticket) cudaFree(D.xticket);
    D.xbuf = nullptr; D.xflags = nullptr; D.xticket = nullptr;
  }
  h->x_d = 0;
  h->x_p2p = false;
}

// What one rank tells the others about its exchange buffers (AGD_XCHG_HANDLE_BYTES on the wire).
struct XHandles {
  cudaIpcMemHandle_t buf, flags;
  int32_t can_peer, d, rank, pad;
  unsigned char reserve[AGD_XCHG_HANDLE_BYTES - 2 * sizeof(cudaIpcMemHandle_t) - 16];
};
static_assert(sizeof(XHandles) == AGD_XCHG_HANDLE_BYTES, "exchange handle blob size is part of the ABI");

void destroy_comms(agd_handle *h) {
  for (Dev &D : h->devs) {
    if (D.comm && nccl_api().ok) { cudaSetDevice(D.ordinal); nccl_api().CommDestroy(D.comm); }
    D.comm = nullptr;
  }
}

// NCCL communicator of a single-process world, built on first need (fallback / collective=nccl)
int ensure_nccl(agd_handle *h) {
  if (h->world <= 1) return 0;
  bool have = true;
  for (Dev &D : h->devs) have = have && D.comm != nullptr;
  if (have) return 0;
  if (h->ipc_only) return fail(h, "this world was set up with agd_comm_init_ipc: there is no NCCL communicator to fall back to");
  if (!h->comm_auto) return fail(h, "world_ranks=%d but agd_comm_init was not called", h->world);
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(h, "NCCL unavailable: %s", N.why.c_str());
  ncclUniqueId id;
  CKN(N.GetUniqueId(&id));
  const int nd = (int)h->devs.size();
  CKN(N.GroupStart());
  for (int i = 0; i < nd; ++i) {
    CK(cudaSetDevice(h->devs[i].ordinal));
    CKN(N.CommInitRank(&h->devs[i].comm, nd, id, i));
  }
  CKN(N.GroupEnd());
  return 0;
}

// step 1 of the exchange setup: allocate this process's buffers for the current dimension and describe them
int xchg_alloc(agd_handle *h, std::vector<XHandles> &mine) {
  const int W = h->world, nd = (int)h->devs.size();
  const int S = xchg_slot_stride(h->d);      // slot stride: room for a two-gradient sweep or an evaluation
  const size_t total = xchg_alloc_doubles(S, W), nflags = 6 * (size_t)W;   // one-shot, reduce-scatter and bulk areas (agd_common.cuh)
  mine.assign((size_t)nd, XHandles());
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    CK(cudaMalloc(&D.xbuf, total * sizeof(double)));
    CK(cudaMalloc(&D.xflags, nflags * sizeof(unsigned long long)));
    CK(cudaMalloc(&D.xticket, sizeof(unsigned int)));
    CK(cudaMemset(D.xbuf, 0, total * sizeof(double)));
    CK(cudaMemset(D.xflags, 0, nflags * sizeof(unsigned long long)));
    CK(cudaMemset(D.xticket, 0, sizeof(unsigned int)));
    memset(&mine[i], 0, sizeof(XHandles));
    mine[i].can_peer = 1;
    mine[i].d = h->d;
    mine[i].rank = h->first_rank + i;
    for (int j = 0; j < nd; ++j) {
      if (j == i) continue;
      int can = 0;
      CK(cudaDeviceCanAccessPeer(&can, D.ordinal, h->devs[j].ordinal));
      if (!can) mine[i].can_peer = 0;
      else { cudaError_t e = cudaDeviceEnablePeerAccess(h->devs[j].ordinal, 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) mine[i].can_peer = 0; cudaGetLastError(); }
    }
    if (nd < W) {  // buffers of other processes are reached through CUDA IPC
      if (cudaIpcGetMemHandle(&mine[i].buf, D.xbuf) != cudaSuccess || cudaIpcGetMemHandle(&mine[i].flags, D.xflags) != cudaSuccess) {
        mine[i].can_peer = 0;
        cudaGetLastError();
      }
    }
  }
  return 0;
}

// step 3: map every rank's buffers into every local device; *ok_out = false when some pair cannot be mapped
int xchg_map(agd_handle *h, const std::vector<XHandles> &all, bool *ok_out) {
  const int W = h->world, nd = (int)h->devs.size();
  bool ok = true;
  for (int r = 0; r < W; ++r) ok = ok && all[(size_t)r].can_peer && all[(size_t)r].d == h->d && all[(size_t)r].rank == r;
  for (int i = 0; i < nd && ok; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    for (int r = 0; r < W; ++r) {
      const int lj = r - h->first_rank;
      if (lj >= 0 && lj < nd) {  // same process: direct pointers (peer access enabled above)
        D.xpeers.slot[r] = h->devs[lj].xbuf;
        D.xpeers.flag[r] = h->devs[lj].xflags;
        continue;
      }
      void *pb = nullptr, *pf = nullptr;
      if (cudaIpcOpenMemHandle(&pb, all[(size_t)r].buf, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess ||
          cudaIpcOpenMemHandle(&pf, all[(size_t)r].flags, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        ok = false;
        break;
      }
      D.xopened.push_back(pb);
      D.xopened.push_back(pf);
      D.xpeers.slot[r] = (double *)pb;
      D.xpeers.flag[r] = (unsigned long long *)pf;
    }
  }
  *ok_out = ok;
  return 0;
}

// Builds the peer-memory exchange for the current dimension.  Three transports for the setup (never for the data):
//  * every rank is a GPU of this process: nothing travels (direct peer pointers), NCCL is not touched;
//  * agd_comm_init worlds: the CUDA IPC handles travel once through an NCCL all-gather, the yes/no decision through a
//    one-int all-reduce; if some pair of ranks cannot map each other NCCL carries the all-reduce instead;
//  * agd_comm_init_ipc worlds: the host ships the handles (agd_xchg_export / agd_xchg_import) -- no NCCL anywhere.
// Collective: every rank calls it from the same entry point.
int ensure_xchg(agd_handle *h) {
  if (h->world <= 1) return 0;
  if (h->collective == 1) return ensure_nccl(h);
  if (h->x_d == h->d) return h->x_p2p ? 0 : ensure_nccl(h);
  if (h->ipc_only)
    return fail(h, "peer-memory exchange not established for d=%d: call agd_xchg_export / agd_xchg_import after loading the shards", h->d);
  free_xchg(h);
  h->x_d = h->d;
  const int W = h->world, nd = (int)h->devs.size();
  if (W > kMaxRanks) { if (h->collective == 2) return fail(h, "peer exchange supports at most %d ranks", kMaxRanks); return ensure_nccl(h); }
  std::vector<XHandles> mine, all((size_t)W);
  if (xchg_alloc(h, mine)) return 1;
  bool ok = true;
  if (nd == W) {
    all = mine;
    if (xchg_map(h, all, &ok)) return 1;
  } else {
    if (ensure_nccl(h)) return 1;
    NcclApi &N = nccl_api();
    // all-gather the handles (device staging through NCCL; setup only)
    std::vector<void *> stage(nd);
    for (int i = 0; i < nd; ++i) {
      Dev &D = h->devs[i];
      CK(cudaSetDevice(D.ordinal));
      CK(cudaMalloc(&stage[i], (size_t)W * sizeof(XHandles)));
      CK(cudaMemcpyAsync((char *)stage[i] + (size_t)(h->first_rank + i) * sizeof(XHandles), &mine[i], sizeof(XHandles), cudaMemcpyHostToDevice, D.st));
    }
    CKN(N.GroupStart());
    for (int i = 0; i < nd; ++i) {
      Dev &D = h->devs[i];
      CKN(N.AllGather((char *)stage[i] + (size_t)(h->first_rank + i) * sizeof(XHandles), stage[i], sizeof(XHandles), ncclChar, D.comm, D.st));
    }
    CKN(N.GroupEnd());
    CK(cudaSetDevice(h->devs[0].ordinal));
    CK(cudaMemcpyAsync(all.data(), stage[0], (size_t)W * sizeof(XHandles), cudaMemcpyDeviceToHost, h->devs[0].st));
    for (int i = 0; i < nd; ++i) { CK(cudaSetDevice(h->devs[i].ordinal)); CK(cudaStreamSynchronize(h->devs[i].st)); }
    for (int i = 0; i < nd; ++i) { cudaSetDevice(h->devs[i].ordinal); cudaFree(stage[i]); }
    if (xchg_map(h, all, &ok)) return 1;
    // every rank must take the same decision: agree through one more (tiny) all-reduce of the ok flag
    int v = ok ? 1 : 0;
    std::vector<int *> fl(nd);
    for (int i = 0; i < nd; ++i) {
      CK(cudaSetDevice(h->devs[i].ordinal));
      CK(cudaMalloc(&fl[i], sizeof(int)));
      CK(cudaMemcpyAsync(fl[i], &v, sizeof(int), cudaMemcpyHostToDevice, h->devs[i].st));
    }
    CKN(N.GroupStart());
    for (int i = 0; i < nd; ++i) CKN(N.AllReduce(fl[i], fl[i], 1, ncclInt, ncclMin, h->devs[i].comm, h->devs[i].st));
    CKN(N.GroupEnd());
    CK(cudaSetDevice(h->devs[0].ordinal));
    CK(cudaMemcpyAsync(&v, fl[0], sizeof(int), cudaMemcpyDeviceToHost, h->devs[0].st));
    for (int i = 0; i < nd; ++i) { CK(cudaSetDevice(h->devs[i].ordinal)); CK(cudaStreamSynchronize(h->devs[i].st)); cudaFree(fl[i]); }
    ok = v == 1;
  }
  if (!ok) {
    if (h->collective == 2) return fail(h, "peer-memory exchange unavailable (no P2P / IPC mapping between every pair of ranks)");
    const int32_t keep = h->x_d;
    free_xchg(h);
    h->x_d = keep;  // do not retry every pass; NCCL carries the all-reduce
    return ensure_nccl(h);
  }
  h->x_p2p = true;
  h->x_epoch = 0;
  return 0;
}

// ---------------------------------------------------------------- the cross-rank exchange
// Every payload that crosses ranks goes through the helpers below.  On the peer-memory exchange an epoch is one payload of at
// most one slot (or one bulk chunk) per rank: every local device publishes, then every local device gathers, each in stream
// order.  So a rank publishes epoch e + 2 only after its own gather of e + 1, which needed every rank's publish of e + 1, which
// each rank enqueued after its gather of e: the parity buffer of e is free again when e + 2 writes into it.  (struct Epoch
// is declared above agd_handle, which keeps the pending one.)
// a buffer on local device i
using DevBuf = std::function<double *(size_t i)>;

Epoch open_epoch(agd_handle *h, int n, bool bulk = false) {
  Epoch x;
  if (h->world <= 1 || !h->x_p2p) return x;
  x.e = ++h->x_epoch;
  x.n = n;
  x.rs = !bulk && n >= kXchgRsMin;
  x.bulk = bulk;
  return x;
}

// what local device i publishes in epoch x
XchgPub publisher(const agd_handle *h, size_t i, const Epoch &x) {
  const Dev &D = h->devs[i];
  const int S = xchg_slot_stride(h->d), W = h->world;
  XchgPub p;
  p.peers = D.xpeers;
  if (x.bulk)
    for (int r = 0; r < W; ++r) p.peers.slot[r] += xchg_off_bulk(S, W);
  p.world = W; p.my_rank = h->first_rank + (int)i; p.buf = (int)(x.e & 1ull); p.n = x.n;
  p.slot_stride = x.bulk ? kXchgBulk : S;
  p.epoch = x.e; p.ticket = D.xticket;
  return p;
}

// what D gathers of epoch x: the slots (one-shot, bulk) or the finished sums (rs), and the flags that guard them; world == 0
// when x is none
XchgGather gatherer(const agd_handle *h, const Dev &D, const Epoch &x) {
  XchgGather g;
  if (!x.e) return g;
  const int S = xchg_slot_stride(h->d), W = h->world;
  g.xbuf = D.xbuf + (x.rs ? xchg_off_res(S, W) : x.bulk ? xchg_off_bulk(S, W) : 0);
  g.flags = D.xflags + (x.rs ? xchg_flags_res(W) : xchg_flags_oneshot(W));
  g.world = W; g.buf = (int)(x.e & 1ull); g.n = x.n;
  g.slot_stride = x.bulk ? kXchgBulk : S;
  g.rs = x.rs ? 1 : 0;
  g.epoch = x.e;
  return g;
}

// stand-alone publish of local device i's n doubles at src (the caller has made device i current): one-shot, or the rs publish
// and the reduce-bcast of this rank's slice by op
int publish(agd_handle *h, size_t i, const Epoch &x, const double *src, int op) {
  const Dev &D = h->devs[i];
  const XchgPub p = publisher(h, i, x);
  if (x.rs) {
    CK(xchg_rs_publish_launch(src, p, D.st));
    CK(xchg_rs_reduce_bcast_launch(D.xbuf, D.xflags, p, D.st, op));
  } else {
    CK(xchg_publish_launch(src, p, D.st));
  }
  return 0;
}

// stand-alone gather of epoch x into dst(i) on every local device (see xchg_gather_launch)
int gather(agd_handle *h, const Epoch &x, const DevBuf &dst, size_t out_stride, int op) {
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    CK(xchg_gather_launch(gatherer(h, D, x), dst(i), out_stride, op, D.st));
  }
  return 0;
}

// The NCCL form of an exchange (collective=nccl, or ranks that cannot map each other's memory): kXchgSum / kXchgMax all-reduce
// the n doubles at buf(i) in place; kXchgCopy all-gathers rank r's n doubles at buf(i) into [W][n] at dst(i).
int nccl_exchange(agd_handle *h, const DevBuf &buf, size_t n, int op, const DevBuf &dst = nullptr) {
  if (!h->comm_ready || !h->devs[0].comm) return fail(h, "world_ranks=%d but there is no communicator (agd_comm_init)", h->world);
  NcclApi &N = nccl_api();
  CKN(N.GroupStart());
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    if (op == kXchgCopy) CKN(N.AllGather(buf(i), dst(i), n, ncclDouble, D.comm, D.st));   // moves bytes: no arithmetic
    else CKN(N.AllReduce(buf(i), buf(i), n, ncclDouble, op == kXchgMax ? ncclMax : ncclSum, D.comm, D.st));
  }
  CKN(N.GroupEnd());
  return 0;
}

// The all-reduce (sum, or NaN-ignoring max) of the n doubles at buf(i) on every local device: epochs of at most one slot
// stride each (one-shot or reduce-scatter form by the epoch's size), or one NCCL all-reduce.
int world_reduce(agd_handle *h, const DevBuf &buf, size_t n, int op) {
  if (h->world <= 1 || n == 0) return 0;
  if (!h->x_p2p) return nccl_exchange(h, buf, n, op);
  const size_t S = (size_t)xchg_slot_stride(h->d);
  for (size_t c0 = 0; c0 < n; c0 += S) {
    const Epoch x = open_epoch(h, (int)std::min(S, n - c0));
    for (size_t i = 0; i < h->devs.size(); ++i) {
      CK(cudaSetDevice(h->devs[i].ordinal));
      if (publish(h, i, x, buf(i) + c0, op)) return 1;
    }
    if (gather(h, x, [&](size_t i) { return buf(i) + c0; }, 0, op)) return 1;
  }
  return 0;
}

// Every rank's n doubles at src(i), concatenated in rank order into [W][n] at dst(i) on every local device: copy epochs
// through the bulk area (one per kXchgBulk doubles), or one NCCL all-gather.
int world_concat(agd_handle *h, const DevBuf &src, size_t n, const DevBuf &dst) {
  if (!h->x_p2p) return nccl_exchange(h, src, n, kXchgCopy, dst);
  for (size_t c0 = 0; c0 < n; c0 += kXchgBulk) {
    const Epoch x = open_epoch(h, (int)std::min((size_t)kXchgBulk, n - c0), true);
    for (size_t i = 0; i < h->devs.size(); ++i) {
      CK(cudaSetDevice(h->devs[i].ordinal));
      if (publish(h, i, x, src(i) + c0, kXchgCopy)) return 1;
    }
    if (gather(h, x, [&](size_t i) { return dst(i) + c0; }, n, kXchgCopy)) return 1;
  }
  return 0;
}

// drains every local stream
int sync_all(agd_handle *h) {
  for (Dev &D : h->devs) {
    CK(cudaSetDevice(D.ordinal));
    CK(cudaStreamSynchronize(D.st));
  }
  return 0;
}

void trace_mark(agd_handle *h, const char *tag) {
  if (h->trace < 0) { const char *e = getenv("AGD_TRACE"); h->trace = (e && *e && *e != '0') ? 1 : 0; }
  if (!h->trace) return;
  Dev &D = h->devs[0];
  cudaSetDevice(D.ordinal);
  cudaEvent_t ev;
  if (h->tr.size() < h->tr_pool.size()) ev = h->tr_pool[h->tr.size()];
  else { cudaEventCreate(&ev); h->tr_pool.push_back(ev); }
  cudaEventRecord(ev, D.st);
  h->tr.push_back({tag, ev});
}

void trace_report(agd_handle *h, const char *what) {
  if (h->trace != 1 || h->tr.size() < 2) { h->tr.clear(); return; }
  struct Acc { double ms = 0; int n = 0; };
  std::vector<std::pair<std::string, Acc>> sums;
  double total = 0;
  for (size_t i = 1; i < h->tr.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->tr[i - 1].second, h->tr[i].second);
    total += ms;
    bool found = false;
    for (auto &kv : sums) if (kv.first == h->tr[i].first) { kv.second.ms += ms; kv.second.n++; found = true; break; }
    if (!found) { Acc a; a.ms = ms; a.n = 1; sums.push_back({h->tr[i].first, a}); }
  }
  fprintf(stderr, "[AGD_TRACE %s rank %d] total %.3f ms:", what, h->first_rank, total);
  for (auto &kv : sums) fprintf(stderr, " %s %.3f ms / %d = %.1f us;", kv.first.c_str(), kv.second.ms, kv.second.n, kv.second.ms / kv.second.n * 1e3);
  fprintf(stderr, "\n");
  h->tr.clear();
}

typedef const double *(*WSel)(Dev &);

// which K1 kernel a dense shard of this handle runs on (0 generic, 1 ring, 3 wgmma)
int dense_kernel_of(const agd_handle *h, int eb) {
  bool ring = k1_ring_supported(h->d, eb) != 0;
  if (h->k1_variant == 2) ring = false;
  if (k1_tc_supported(h->d, eb) && (h->k1_variant == 0 || h->k1_variant == 4)) return 3;
  return ring ? 1 : 0;
}

// can one sweep evaluate the loss at a second point as well (pass fusion)?
bool dual_supported(const agd_handle *h) {
  for (const Dev &D : h->devs) {
    const Shard &s = D.sh;
    if (s.csr) continue;
    const int eb = s.elem_bytes ? s.elem_bytes : 4;
    const int k = dense_kernel_of(h, eb);
    if (k == 3 && (h->tune_rows != 0 || h->tc_margins_f64)) return false;   // wgmma: the default (fp32-margin) mapping has one
    if (k == 1 && !k1_ring_dual_supported(h->d, eb)) return false;
  }
  return h->k1_diag == 0;
}

// ... and the gradient there too (the speculative sweep of the memoised pass structure)?
bool dual_full_supported(const agd_handle *h) {
  for (const Dev &D : h->devs) {
    const Shard &s = D.sh;
    if (s.csr) return false;
    const int eb = s.elem_bytes ? s.elem_bytes : 4;
    const int k = dense_kernel_of(h, eb);
    if (k == 3) { if (h->tune_rows != 0 || h->tc_margins_f64) return false; continue; }   // wgmma: default mapping has one
    if (k != 1 || !k1_ring_dual_full_supported(h->d, eb)) return false;
  }
  return h->k1_diag == 0;
}

// One applySmooth (AGD.scala:192-208) at the device-resident point `w_of(dev)`: K1 over every local
// shard, slab reduction, one all-reduce of [grad | loss | count | loss2 | count2].  Result: Dev::acc on every device.
// w2_of != nullptr: the same sweep also evaluates the loss (not the gradient) at `w2_of(dev)` -> acc[D+2], acc[D+3];
// with dual_full also the gradient there -> a second block acc[D+4 .. 2D+7] = [grad | loss | count | 0 | 0].
// D = h->model_d(): under a feature transform the points and the gradient are those of the model on appendBias(s o x);
// K1 runs on the stored x at w_eff = (s o v, b) and the gradient columns are scaled by s before the exchange.
// defer_gather: on the peer-memory path the gather is left to the next K3 kernel (h->pending; see XchgGather) -- one launch
// fewer per sweep; the caller must hand the pending exchange to a k3_step / k3_gx launch before anything else reads acc.
int smooth_device(agd_handle *h, int kind, WSel w_of, bool timed, WSel w2_of = nullptr, bool dual_full = false,
                  bool defer_gather = false) {
  if (h->pending.e) return fail(h, "internal: an exchange is still waiting for its consumer");
  const int32_t d = h->d, md = h->model_d();
  const int32_t n = (dual_full ? 2 : 1) * (md + 4);   // doubles this sweep produces and exchanges
  const Epoch ep = open_epoch(h, n);   // large payloads: reduce-scatter + all-gather instead of the one-shot exchange
  const bool p2p = ep.e != 0, rs = ep.rs;
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    const Shard &s = D.sh;
    const bool t0 = timed && i == 0;
    const double *w = w_of(D), *w2 = w2_of ? w2_of(D) : nullptr;
    const double *scale = h->scale_of(D);
    if (scale) {   // the points on the stored features: (s o v, b)
      CK(transform_point_launch(D.weff, w, w2 ? D.weff2 : nullptr, w2, scale, d, md, D.st));
      w = D.weff;
      if (w2) w2 = D.weff2;
      if (i == 0) h->launches += 1;
    }
    if (s.csr) {
      if (dual_full) return fail(h, "internal: two-gradient sweep requested on a CSR shard");
      K1CsrArgs a;
      a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; a.labels = s.labels; a.w = w;
      a.w2 = w2;
      a.gacc = D.acc; a.rows = s.rows; a.d = d; a.kind = kind;
      a.sample_seed = h->sample_seed; a.sample_thresh = h->sample_thresh; a.row_base = D.row_base; a.filt = h->filt_of(D); a.tune = h->tune_rows;
      if (t0) CK(cudaEventRecord(next_event(D.ev, D.ev_used), D.st));
      CK(k1_csr_launch(a, h->tf_bias, s.elem_bytes, D.sm_count, D.st));
      if (t0) CK(cudaEventRecord(next_event(D.ev, D.ev_used), D.st));
      if (scale) {   // K1 summed the gradient straight into acc: scale it before the exchange
        CK(scale_columns_launch(D.acc, scale, d, D.st));
        if (i == 0) h->launches += 1;
      }
      if (p2p && publish(h, i, ep, D.acc, kXchgSum)) return 1;
      h->launches += (i == 0) ? (rs ? 4 : (p2p ? 3 : 2)) : 0;
      continue;
    }
    if (ensure_view_bits(h, D)) return 1;
    K1Args a;
    a.X = s.X; a.labels = s.labels; a.w = w; a.w2 = w2; a.dual_full = dual_full ? 1 : 0;
    a.rows = s.rows; a.d = d; a.kind = h->k1_diag ? h->k1_diag : kind;
    a.stages = h->ring_stages; a.slab_stride = n;
    a.sample_seed = h->sample_seed; a.sample_thresh = h->sample_thresh; a.row_base = D.row_base; a.filt = h->filt_of(D); a.view_bits = a.filt ? D.view_bits : nullptr; a.tune_rows = h->tune_rows; a.tune_ctas = h->tune_ctas; a.tune_full = h->tune_full;
    a.tc_margins_f64 = h->tc_margins_f64;
    const int eb = s.elem_bytes ? s.elem_bytes : 4;
    bool ring = k1_ring_supported(d, eb) != 0;
    if (h->k1_variant == 2) ring = false;
    const bool tc = k1_tc_supported(d, eb) && (h->k1_variant == 0 || h->k1_variant == 4);
    if (h->k1_variant == 4 && !tc) return fail(h, "wgmma kernel needs bf16 storage with d %% 128 == 0 and d <= 4096 (d=%d)", d);
    if (h->k1_variant == 1 && !ring) return fail(h, "ring kernel does not support d=%d with %d-byte elements", d, eb);
    if (a.w2 && ((tc && (h->tune_rows != 0 || h->tc_margins_f64)) || (!tc && ring && !k1_ring_dual_supported(d, eb))))
      return fail(h, "internal: two-point sweep requested on a kernel without one");
    if (dual_full && ((tc && (h->tune_rows != 0 || h->tc_margins_f64)) || (!tc && (!ring || !k1_ring_dual_full_supported(d, eb)))))
      return fail(h, "internal: two-gradient sweep requested on a kernel without one");
    int max_blocks = k1_max_blocks(D.sm_count);
    if (!ring) {  // generic: bound the slab memory for very wide rows
      const long long lim = (32LL << 20) / ((long long)d + 4);
      if (lim < max_blocks) max_blocks = lim < 1 ? 1 : (int)lim;
    }
    if (ensure_slabs(h, D, max_blocks, n)) return 1;
    a.slabs = D.slabs;
    int blocks = 0;
    if (t0) CK(cudaEventRecord(next_event(D.ev, D.ev_used), D.st));
    if (tc) CK(k1_tc_launch(a, h->tf_bias, D.sm_count, &blocks, D.st));
    else if (ring) CK(k1_ring_launch(a, h->tf_bias, eb, D.sm_count, &blocks, D.st));
    else CK(k1_generic_launch(a, h->tf_bias, eb, D.sm_count, max_blocks, &blocks, D.st));
    if (t0) CK(cudaEventRecord(next_event(D.ev, D.ev_used), D.st));
    if (i == 0) trace_mark(h, dual_full ? "K1x2" : (w2_of ? "K1+loss" : "K1"));
    if (p2p && !rs) { const XchgPub pub = publisher(h, i, ep); CK(k1_reduce_launch(D.slabs, blocks, n, D.acc, &pub, D.st, scale, d, md + 4)); }
    else CK(k1_reduce_launch(D.slabs, blocks, n, D.acc, nullptr, D.st, scale, d, md + 4));
    if (rs) {
      if (publish(h, i, ep, D.acc, kXchgSum)) return 1;
      if (i == 0) h->launches += 2;
    }
    if (i == 0) trace_mark(h, p2p ? "reduce+publish" : "reduce");
    if (i == 0) h->launches += (s.rows > 0 ? 2 : 1);
  }
  const DevBuf acc = [h](size_t i) { return h->devs[i].acc; };
  Dev &D0 = h->devs[0];
  if (p2p && defer_gather) {
    h->pending = ep;
    h->collectives += 1;
  } else if (p2p) {  // K2': every rank already holds every rank's partial sums; add them in rank order
    if (timed) { CK(cudaSetDevice(D0.ordinal)); CK(cudaEventRecord(next_event(D0.ev_ar, D0.ev_ar_used), D0.st)); }
    if (gather(h, ep, acc, 0, kXchgSum)) return 1;
    if (timed) { CK(cudaSetDevice(D0.ordinal)); CK(cudaEventRecord(next_event(D0.ev_ar, D0.ev_ar_used), D0.st)); }
    trace_mark(h, "gather");
    h->launches += 1;
    h->collectives += 1;
  } else if (h->world > 1) {
    if (timed) { CK(cudaSetDevice(D0.ordinal)); CK(cudaEventRecord(next_event(D0.ev_ar, D0.ev_ar_used), D0.st)); }
    if (nccl_exchange(h, acc, (size_t)n, kXchgSum)) return 1;
    if (timed) { CK(cudaSetDevice(D0.ordinal)); CK(cudaEventRecord(next_event(D0.ev_ar, D0.ev_ar_used), D0.st)); }
    h->collectives += 1;
  }
  return 0;
}

int read_scalars(agd_handle *h, double *out) {
  Dev &D = h->devs[0];
  CK(cudaSetDevice(D.ordinal));
  CK(cudaStreamSynchronize(D.st));  // the kernel's zero-copy stores are visible once the stream has drained
  memcpy(out, D.scalars_host, K3_NS * sizeof(double));
  return 0;
}

// The same without draining the stream: the last K3 kernel of a round stores `seq` behind its scalars in mapped pinned memory
// (after a system-scope fence); the host polls that word.  No driver call sits between the kernel's last store and the host
// loop continuing, and the stream may already hold later work.  A stream query every few thousand polls catches errors.
int wait_scalars(agd_handle *h, unsigned long long seq, double *out) {
  Dev &D = h->devs[0];
  volatile unsigned long long *flag = reinterpret_cast<volatile unsigned long long *>(D.scalars_host + 2 * K3_NS);
  unsigned int spins = 0;
  while (*flag != seq) {
    if ((++spins & 0x3fffu) == 0) {
      CK(cudaSetDevice(D.ordinal));
      const cudaError_t q = cudaStreamQuery(D.st);
      if (q == cudaSuccess) { if (*flag != seq) return fail(h, "internal: the round's scalars never arrived"); break; }
      if (q != cudaErrorNotReady) return fail(h, "stream failed while waiting for a round: %s", cudaGetErrorString(q));
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  memcpy(out, D.scalars_host, K3_NS * sizeof(double));
  return 0;
}

int sum_events(agd_handle *h, std::vector<cudaEvent_t> &pool, size_t used, double *ms_out) {
  double ms = 0.0;
  for (size_t i = 0; i + 1 < used; i += 2) {
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, pool[i], pool[i + 1]));
    ms += t;
  }
  *ms_out = ms;
  return 0;
}

int check_ready(agd_handle *h) {
  if (!h) return 1;
  h->pending = Epoch();   // a call that failed half-way may have left one behind
  if (h->d <= 0) return fail(h, "no shard loaded (call agd_load_dense / agd_load_csr / agd_generate first)");
  for (Dev &D : h->devs)
    if (ensure_vectors(h, D, h->model_d())) return 1;
  if (h->world > 1 && !h->comm_ready) return fail(h, "world_ranks=%d but agd_comm_init was not called", h->world);
  return ensure_xchg(h);
}

int call_begin(agd_handle *h) {
  Dev &D = h->devs[0];
  CK(cudaSetDevice(D.ordinal));
  if (!h->ev_begin) { CK(cudaEventCreate(&h->ev_begin)); CK(cudaEventCreate(&h->ev_end)); }
  h->launches = 0;
  h->collectives = 0;
  D.ev_used = D.ev_ar_used = 0;
  CK(cudaEventRecord(h->ev_begin, D.st));
  return 0;
}

// all devices drained; fills the timing part of the stats
int call_end(agd_handle *h, agd_stats &s, std::chrono::steady_clock::time_point t_begin) {
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  CK(cudaEventRecord(h->ev_end, D0.st));
  if (sync_all(h)) return 1;
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, h->ev_begin, h->ev_end));
  s.device_ms_total = ms;
  if (sum_events(h, D0.ev, D0.ev_used, &s.k1_ms_total)) return 1;
  if (sum_events(h, D0.ev_ar, D0.ev_ar_used, &s.allreduce_ms_total)) return 1;
  s.k1_launches = (int64_t)(D0.ev_used / 2);
  s.gpu_launches = h->launches;
  s.collective_calls = h->collectives;
  s.collective_kind = h->x_p2p ? 1 : 0;
  s.seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  return 0;
}

double reg_value(int updater, double reg, double sum_sq, double sum_abs) {
  if (updater == AGD_UPD_SQUARED_L2) {
    const double nrm = std::sqrt(sum_sq);  // brzNorm(w, 2.0)
    return 0.5 * reg * nrm * nrm;
  }
  if (updater == AGD_UPD_L1) return sum_abs * reg;
  return 0.0;
}

}  // namespace

namespace agd {
void set_last_error(agd_handle *h, const char *msg) { fail(h, "%s", msg); }
}  // namespace agd

// ================================================================ C-ABI
extern "C" {

int agd_abi_version(void) { return AGD_B200_ABI_VERSION; }
int agd_sizeof_params(void) { return (int)sizeof(agd_params); }
int agd_sizeof_stats(void) { return (int)sizeof(agd_stats); }

void agd_default_params(agd_params *p) {  // AGD.scala:44-51
  memset(p, 0, sizeof *p);
  p->convergence_tol = 1e-4;
  p->num_iterations = 100;
  p->reg_param = 0.0;
  p->L0 = 1.0;
  p->Lexact = std::numeric_limits<double>::infinity();
  p->beta = 0.5;
  p->alpha = 0.9;
  p->may_restart = 1;
  p->gradient = AGD_GRAD_LOGISTIC;
  p->updater = AGD_UPD_SIMPLE;
  p->flags = 0;
}

const char *agd_last_error(const agd_handle *h) {
  if (h) return h->err.c_str();
  return g_create_error.c_str();
}

int agd_create(const int32_t *device_ids, int32_t n_dev, agd_handle **out) {
  agd_handle *h = nullptr;  // errors before the handle exists go to the global slot
  if (!out) return fail(h, "out is NULL");
  *out = nullptr;
  if (n_dev < 1 || !device_ids) return fail(h, "need at least one device");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(h, "no CUDA device available (%s); this library has no CPU fallback",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  agd_handle *nh = new agd_handle();
  nh->devs.resize(n_dev);
  for (int i = 0; i < n_dev; ++i) {
    Dev &D = nh->devs[i];
    D.ordinal = device_ids[i];
    D.mu = new std::mutex();
    if (D.ordinal < 0 || D.ordinal >= count) { fail(h, "device ordinal %d out of range (0..%d)", D.ordinal, count - 1); agd_destroy(nh); return 1; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, D.ordinal) != cudaSuccess || prop.major != 9) {
      fail(h, "device %d is not an sm_90 (Hopper H100) GPU; kernels are built for sm_90a only", D.ordinal);
      agd_destroy(nh);
      return 1;
    }
    D.sm_count = prop.multiProcessorCount;
    if (cudaSetDevice(D.ordinal) != cudaSuccess || cudaStreamCreateWithFlags(&D.st, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMalloc(&D.ticket, sizeof(unsigned int)) != cudaSuccess ||
        cudaMemset(D.ticket, 0, sizeof(unsigned int)) != cudaSuccess ||
        cudaHostAlloc(&D.scalars_host, (2 * K3_NS + 2) * sizeof(double), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
        cudaHostGetDevicePointer((void **)&D.scalars_dev, D.scalars_host, 0) != cudaSuccess) {
      fail(h, "device %d setup failed: %s", D.ordinal, cudaGetErrorString(cudaGetLastError()));
      agd_destroy(nh);
      return 1;
    }
    memset(D.scalars_host, 0, (2 * K3_NS + 2) * sizeof(double));   // the sequence word behind the scalars starts at 0
  }
  nh->world = n_dev;
  nh->first_rank = 0;
  for (int i = 0; i < n_dev; ++i) nh->devs[i].row_base = (long long)i << 40;  // loaded shards: one mask stream per rank
  *out = nh;
  // A single-process owner of several GPUs is a complete world of its own: ranks 0..n_dev-1 exchange through direct peer
  // pointers, and NCCL is built only if it is ever needed (ensure_nccl).  agd_comm_init / agd_comm_init_ipc replace this
  // default when the process is part of a larger world.
  nh->comm_auto = true;
  nh->comm_ready = true;
  return 0;
}

int agd_destroy(agd_handle *h) {
  if (!h) return 0;
  free_xchg(h);
  for (Dev &D : h->devs) {
    cudaSetDevice(D.ordinal);
    cudaStreamSynchronize(D.st);
    if (D.comm && nccl_api().ok) nccl_api().CommDestroy(D.comm);
    D.comm = nullptr;
    free_shard(h, D);
    double *v[] = {D.x, D.z, D.x_old, D.z_old, D.y, D.g_y, D.g_x, D.wtmp, D.y_spec, D.acc, D.slabs, D.partials, D.eval, D.cs,
                   D.gm, D.tf_scale, D.weff, D.weff2};
    for (double *p : v)
      if (p) cudaFree(p);
    if (D.ticket) cudaFree(D.ticket);
    if (D.scalars_host) cudaFreeHost(D.scalars_host);
    if (D.hist_host) cudaFreeHost(D.hist_host);
    if (D.stage_dev) cudaFree(D.stage_dev);
    if (D.filt_dev) cudaFree(D.filt_dev);
    if (D.view_bits) cudaFree(D.view_bits);
    free_bin(D);
    free_km(D);
    for (cudaEvent_t e : D.ev) cudaEventDestroy(e);
    for (cudaEvent_t e : D.ev_ar) cudaEventDestroy(e);
    if (&D == &h->devs[0] && h->ev_begin) { cudaEventDestroy(h->ev_begin); cudaEventDestroy(h->ev_end); }
    if (D.st) cudaStreamDestroy(D.st);
    delete D.mu;
  }
  delete h;
  return 0;
}

int agd_comm_unique_id(void *out128) {
  agd_handle *h = nullptr;
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(h, "NCCL unavailable: %s", N.why.c_str());
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  ncclUniqueId id;
  ncclResult_t r = N.GetUniqueId(&id);
  if (r != ncclSuccess) return fail(h, "ncclGetUniqueId failed: %s", N.GetErrorString(r));
  memcpy(out128, &id, 128);
  return 0;
}

int agd_comm_init(agd_handle *h, const void *id128, int32_t world_ranks, int32_t first_rank) {
  if (!h) return 1;
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(h, "NCCL unavailable: %s", N.why.c_str());
  const int nd = (int)h->devs.size();
  if (world_ranks < nd || first_rank < 0 || first_rank + nd > world_ranks)
    return fail(h, "bad rank layout: world=%d first=%d local=%d", world_ranks, first_rank, nd);
  if (h->comm_ready && !h->comm_auto) return fail(h, "communicator already initialised");
  // replaces the default single-process world of agd_create (its NCCL communicator, if one was ever built, and its exchange)
  free_xchg(h);
  destroy_comms(h);
  h->comm_auto = false;
  h->ipc_only = false;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  if (world_ranks > 1) {
    CKN(N.GroupStart());
    for (int i = 0; i < nd; ++i) {
      CK(cudaSetDevice(h->devs[i].ordinal));
      CKN(N.CommInitRank(&h->devs[i].comm, world_ranks, id, first_rank + i));
    }
    CKN(N.GroupEnd());
  }
  h->world = world_ranks;
  h->first_rank = first_rank;
  h->comm_ready = true;
  for (int i = 0; i < nd; ++i) h->devs[i].row_base = (long long)(first_rank + i) << 40;
  return 0;
}

// ---- the same world without NCCL: the host language ships the CUDA IPC handles of the exchange buffers
int agd_comm_init_ipc(agd_handle *h, int32_t world_ranks, int32_t first_rank) {
  if (!h) return 1;
  const int nd = (int)h->devs.size();
  if (world_ranks < nd || first_rank < 0 || first_rank + nd > world_ranks)
    return fail(h, "bad rank layout: world=%d first=%d local=%d", world_ranks, first_rank, nd);
  if (world_ranks > kMaxRanks) return fail(h, "the peer-memory exchange supports at most %d ranks", kMaxRanks);
  if (h->comm_ready && !h->comm_auto) return fail(h, "communicator already initialised");
  free_xchg(h);
  destroy_comms(h);
  h->comm_auto = false;
  h->ipc_only = world_ranks > nd;   // a world of local GPUs only needs no handles at all
  if (!h->ipc_only) h->comm_auto = true;
  h->world = world_ranks;
  h->first_rank = first_rank;
  h->comm_ready = true;
  for (int i = 0; i < nd; ++i) h->devs[i].row_base = (long long)(first_rank + i) << 40;
  return 0;
}

int agd_xchg_export(agd_handle *h, void *out, int64_t capacity_bytes, int64_t *bytes_written) {
  if (!h || !out || !bytes_written) return 1;
  if (!h->ipc_only) return fail(h, "agd_xchg_export needs a world set up with agd_comm_init_ipc");
  if (h->d <= 0) return fail(h, "load the shards first: the exchange buffers are sized by the feature dimension");
  const int nd = (int)h->devs.size();
  if (capacity_bytes < (int64_t)nd * AGD_XCHG_HANDLE_BYTES) return fail(h, "capacity too small: need %d bytes", nd * AGD_XCHG_HANDLE_BYTES);
  free_xchg(h);
  std::vector<XHandles> mine;
  if (xchg_alloc(h, mine)) return 1;
  for (Dev &D : h->devs) { CK(cudaSetDevice(D.ordinal)); CK(cudaDeviceSynchronize()); }  // the zeroed buffers are visible before any peer maps them
  memcpy(out, mine.data(), (size_t)nd * sizeof(XHandles));
  *bytes_written = (int64_t)nd * AGD_XCHG_HANDLE_BYTES;
  return 0;
}

int agd_xchg_import(agd_handle *h, const void *all_ranks, int64_t bytes) {
  if (!h || !all_ranks) return 1;
  if (!h->ipc_only) return fail(h, "agd_xchg_import needs a world set up with agd_comm_init_ipc");
  if (!h->devs[0].xbuf) return fail(h, "call agd_xchg_export first");
  if (bytes != (int64_t)h->world * AGD_XCHG_HANDLE_BYTES) return fail(h, "expected %d handle blobs (%d bytes)", h->world, h->world * AGD_XCHG_HANDLE_BYTES);
  std::vector<XHandles> all((size_t)h->world);
  memcpy(all.data(), all_ranks, (size_t)bytes);
  bool ok = true;
  if (xchg_map(h, all, &ok)) return 1;
  if (!ok) {
    free_xchg(h);
    return fail(h, "peer-memory exchange unavailable: some pair of ranks cannot map each other's buffers (or the blobs are not in rank order / of another dimension)");
  }
  h->x_d = h->d;
  h->x_p2p = true;
  h->x_epoch = 0;
  return 0;
}

int agd_reserve(agd_handle *h, int32_t dev, int64_t rows_capacity, int32_t d, int32_t store_dtype) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  if (set_dim(h, d, dtype_bytes(store_dtype))) return 1;
  Dev &D = h->devs[dev];
  std::lock_guard<std::mutex> g(*D.mu);
  return reserve_locked(h, D, rows_capacity, h->d, store_dtype);
}

int agd_load_dense(agd_handle *h, int32_t dev, const void *X, int32_t src_dtype, const double *labels,
                   int64_t rows, int32_t d, int64_t ld, int32_t store_dtype) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  const int sb = dtype_bytes(src_dtype);
  if (sb != 4 && sb != 8) return fail(h, "src_dtype must be AGD_F32 or AGD_F64");
  if (rows < 0 || ld < d) return fail(h, "bad geometry rows=%lld d=%d ld=%lld", (long long)rows, d, (long long)ld);
  if (rows > 0 && (!X || !labels)) return fail(h, "NULL data pointer");
  if (set_dim(h, d, dtype_bytes(store_dtype))) return 1;
  const int32_t di = h->d;  // stored row length (>= d, zero-padded)
  Dev &D = h->devs[dev];
  std::lock_guard<std::mutex> g(*D.mu);
  Shard &s = D.sh;
  const int64_t need = s.rows + rows;
  if (s.cap == 0 || need > s.cap) {
    const int64_t cap = s.cap == 0 ? need : (need > 2 * s.cap ? need : 2 * s.cap);
    if (reserve_locked(h, D, cap, di, s.cap ? bytes_dtype(s.elem_bytes) : store_dtype)) return 1;
  }
  const int eb = s.elem_bytes;
  if (dtype_bytes(store_dtype) != eb) return fail(h, "storage dtype mismatch with the resident shard");
  CK(cudaSetDevice(D.ordinal));
  unsigned char *dst = (unsigned char *)s.X + (size_t)s.rows * di * eb;
  const unsigned char *src = (const unsigned char *)X;
  if (rows > 0) {
    if (sb == eb && ld == d && di == d) {
      CK(cudaMemcpyAsync(dst, src, (size_t)rows * d * eb, cudaMemcpyHostToDevice, D.st));
    } else {
      int64_t chunk = (int64_t)((64u << 20) / ((size_t)ld * sb));
      if (chunk < 1) chunk = 1;
      if (chunk > rows) chunk = rows;
      if (ensure_stage(h, D, (size_t)chunk * ld * sb)) return 1;
      for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
        const int64_t rc = rows - r0 < chunk ? rows - r0 : chunk;
        CK(cudaMemcpyAsync(D.stage_dev, src + (size_t)r0 * ld * sb, (size_t)rc * ld * sb, cudaMemcpyHostToDevice, D.st));
        CK(convert_rows_launch(dst + (size_t)r0 * di * eb, eb, D.stage_dev, sb, rc, d, ld, di, D.st));
        CK(cudaStreamSynchronize(D.st));  // the staging buffer is reused
      }
    }
    CK(cudaMemcpyAsync(s.labels + s.rows, labels, (size_t)rows * sizeof(double), cudaMemcpyHostToDevice, D.st));
  }
  CK(cudaStreamSynchronize(D.st));
  s.rows += rows;
  return 0;
}

// grows the CSR arrays of a device to hold `rows_cap` rows and `nnz_cap` entries (contents preserved)
static int csr_reserve_locked(agd_handle *h, Dev &D, int64_t rows_cap, int64_t nnz_cap, int eb) {
  Shard &s = D.sh;
  CK(cudaSetDevice(D.ordinal));
  if (!s.csr && (s.cap > 0 || s.rows > 0)) return fail(h, "device already holds a dense shard");
  if (s.csr && s.elem_bytes != eb) return fail(h, "storage dtype mismatch with the resident shard");
  if (rows_cap > s.cap || !s.rowptr) {
    int64_t *nr = nullptr;
    double *nl = nullptr;
    CK(cudaMalloc(&nr, ((size_t)rows_cap + 1) * sizeof(int64_t)));
    CK(cudaMalloc(&nl, ((size_t)rows_cap + 64) * sizeof(double)));
    if (s.rowptr) {
      CK(cudaMemcpyAsync(nr, s.rowptr, ((size_t)s.rows + 1) * sizeof(int64_t), cudaMemcpyDeviceToDevice, D.st));
      CK(cudaMemcpyAsync(nl, s.labels, (size_t)s.rows * sizeof(double), cudaMemcpyDeviceToDevice, D.st));
    } else {
      CK(cudaMemsetAsync(nr, 0, sizeof(int64_t), D.st));
    }
    CK(cudaStreamSynchronize(D.st));
    if (s.rowptr) cudaFree(s.rowptr);
    if (s.labels) cudaFree(s.labels);
    s.rowptr = nr; s.labels = nl; s.cap = rows_cap;
  }
  if (nnz_cap > s.nnz_cap || !s.idx) {
    int32_t *ni = nullptr;
    void *nv = nullptr;
    CK(cudaMalloc(&ni, ((size_t)nnz_cap + 4) * sizeof(int32_t)));
    CK(cudaMalloc(&nv, ((size_t)nnz_cap + 4) * eb));
    if (s.idx && s.nnz > 0) {
      CK(cudaMemcpyAsync(ni, s.idx, (size_t)s.nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice, D.st));
      CK(cudaMemcpyAsync(nv, s.val, (size_t)s.nnz * eb, cudaMemcpyDeviceToDevice, D.st));
    }
    CK(cudaStreamSynchronize(D.st));
    if (s.idx) cudaFree(s.idx);
    if (s.val) cudaFree(s.val);
    s.idx = ni; s.val = nv; s.nnz_cap = nnz_cap;
  }
  s.csr = true;
  s.elem_bytes = eb;
  return 0;
}

int agd_load_csr(agd_handle *h, int32_t dev, const int64_t *rowptr, const int32_t *idx, const void *val,
                 int32_t src_dtype, const double *labels, int64_t rows, int32_t d, int32_t store_dtype) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  const int sb = dtype_bytes(src_dtype), eb = dtype_bytes(store_dtype);
  if ((sb != 4 && sb != 8) || (eb != 4 && eb != 8)) return fail(h, "CSR dtypes must be AGD_F32 or AGD_F64");
  if (rows < 0 || (rows > 0 && (!rowptr || !labels))) return fail(h, "bad CSR arguments");
  if (set_dim(h, d)) return 1;
  Dev &D = h->devs[dev];
  std::lock_guard<std::mutex> g(*D.mu);
  Shard &s = D.sh;
  if (rows > 0 && rowptr[0] != 0) return fail(h, "rowptr[0] must be 0");
  const int64_t nnz = rows > 0 ? rowptr[rows] : 0;
  if (nnz < 0) return fail(h, "rowptr[rows] = %lld is negative", (long long)nnz);
  if (nnz > 0 && (!idx || !val)) return fail(h, "NULL index / value pointer");
  // APPENDS rows (Spark hands partitions over one at a time); arrays grow geometrically
  const int64_t need_rows = s.rows + rows, need_nnz = s.nnz + nnz;
  const int64_t rows_cap = need_rows > s.cap ? (need_rows > 2 * s.cap ? need_rows : 2 * s.cap) : s.cap;
  const int64_t nnz_cap = need_nnz > s.nnz_cap ? (need_nnz > 2 * s.nnz_cap ? need_nnz : 2 * s.nnz_cap) : s.nnz_cap;
  if (csr_reserve_locked(h, D, rows_cap, nnz_cap, eb)) return 1;
  if (rows > 0) {
    // device rowptr entries for the new rows = host rowptr[1..rows] + resident nnz
    if (ensure_stage(h, D, ((size_t)rows + 1) * sizeof(int64_t) + (size_t)nnz * sb + 64)) return 1;
    CK(cudaMemcpyAsync(D.stage_dev, rowptr, ((size_t)rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, D.st));
    CK(csr_shift_rowptr_launch(s.rowptr + s.rows, (const int64_t *)D.stage_dev, rows + 1, s.nnz, D.st));
    CK(cudaMemcpyAsync(s.labels + s.rows, labels, (size_t)rows * sizeof(double), cudaMemcpyHostToDevice, D.st));
  }
  if (nnz > 0) {
    CK(cudaMemcpyAsync(s.idx + s.nnz, idx, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, D.st));
    if (sb == eb) {
      CK(cudaMemcpyAsync((unsigned char *)s.val + (size_t)s.nnz * eb, val, (size_t)nnz * eb, cudaMemcpyHostToDevice, D.st));
    } else {
      unsigned char *stage_vals = (unsigned char *)D.stage_dev + (((size_t)rows + 1) * sizeof(int64_t) + 63) / 64 * 64;
      CK(cudaMemcpyAsync(stage_vals, val, (size_t)nnz * sb, cudaMemcpyHostToDevice, D.st));
      CK(convert_rows_launch((unsigned char *)s.val + (size_t)s.nnz * eb, eb, stage_vals, sb, nnz, 1, 1, 1, D.st));
    }
  }
  // Validate on the device before the partition becomes part of the shard: the gradient kernel gathers w[idx] and
  // scatters into g[idx] with these raw indices, so one bad column id would be an out-of-bounds device write.
  if (rows > 0) {
    int *flag = nullptr, host_flag = 0;   // D.stage_dev still holds the caller's rowptr
    CK(cudaMalloc(&flag, sizeof(int)));
    CK(cudaMemsetAsync(flag, 0, sizeof(int), D.st));
    CK(csr_validate_launch((const int64_t *)D.stage_dev, rows, s.idx + s.nnz, nnz, d, flag, D.st));
    CK(cudaMemcpyAsync(&host_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));
    cudaFree(flag);
    if (host_flag == 1) return fail(h, "bad CSR partition: rowptr must be non-decreasing from 0 to nnz=%lld", (long long)nnz);
    if (host_flag == 2) return fail(h, "bad CSR partition: a column index lies outside [0, %d) (SparseVector size differs from the weights?)", d);
  }
  CK(cudaStreamSynchronize(D.st));
  s.rows = need_rows;
  s.nnz = need_nnz;
  return 0;
}

int agd_generate_csr(agd_handle *h, int64_t total_rows, int32_t d, int32_t nnz_per_row, int32_t store_dtype,
                     uint64_t seed, int32_t gradient) {
  if (!h) return 1;
  const int eb = dtype_bytes(store_dtype);
  if (eb != 4 && eb != 8) return fail(h, "CSR store_dtype must be AGD_F32 or AGD_F64");
  if (total_rows < 0 || nnz_per_row < 1 || nnz_per_row > d) return fail(h, "bad CSR geometry");
  if (agd_clear(h)) return 1;
  if (set_dim(h, d)) return 1;
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    std::lock_guard<std::mutex> g(*D.mu);
    const long long rank = h->first_rank + (long long)i, W = h->world;
    const int64_t lo = (int64_t)(((__int128)rank * total_rows) / W), hi = (int64_t)(((__int128)(rank + 1) * total_rows) / W);
    if (csr_reserve_locked(h, D, hi - lo, (hi - lo) * nnz_per_row, eb)) return 1;
    if (ensure_vectors(h, D, d)) return 1;
    CK(cudaSetDevice(D.ordinal));
    D.row_base = lo;
    CK(synth_wtrue_launch(D.wtmp, seed, d, D.st));
    CK(synth_csr_launch(D.sh.rowptr, D.sh.idx, D.sh.val, eb, D.wtmp, D.sh.labels, seed, gradient, lo, hi - lo, d,
                        nnz_per_row, D.st));
    D.sh.rows = hi - lo;
    D.sh.nnz = (hi - lo) * nnz_per_row;
  }
  if (sync_all(h)) return 1;
  return 0;
}

int agd_get_csr_rows(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, int64_t *rowptr_out, int32_t *idx_out,
                     void *val_out, int64_t nnz_capacity, double *labels_out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  Dev &D = h->devs[dev];
  const Shard &s = D.sh;
  if (!s.csr) return fail(h, "agd_get_csr_rows serves CSR shards only");
  if (row0 < 0 || rows < 0 || row0 + rows > s.rows) return fail(h, "row range out of bounds");
  CK(cudaSetDevice(D.ordinal));
  CK(cudaMemcpyAsync(rowptr_out, s.rowptr + row0, ((size_t)rows + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  const int64_t a = rowptr_out[0], b = rowptr_out[rows];
  if (b - a > nnz_capacity) return fail(h, "nnz_capacity too small: need %lld", (long long)(b - a));
  if (b > a) {
    CK(cudaMemcpyAsync(idx_out, s.idx + a, (size_t)(b - a) * sizeof(int32_t), cudaMemcpyDeviceToHost, D.st));
    CK(cudaMemcpyAsync(val_out, (const unsigned char *)s.val + (size_t)a * s.elem_bytes, (size_t)(b - a) * s.elem_bytes,
                       cudaMemcpyDeviceToHost, D.st));
  }
  if (labels_out && rows) CK(cudaMemcpyAsync(labels_out, s.labels + row0, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  for (int64_t i = rows; i >= 0; --i) rowptr_out[i] -= a;
  return 0;
}

int agd_clear(agd_handle *h) {
  if (!h) return 1;
  for (Dev &D : h->devs) {
    std::lock_guard<std::mutex> g(*D.mu);
    CK(cudaSetDevice(D.ordinal));
    CK(cudaStreamSynchronize(D.st));
    if (free_shard(h, D)) return 1;
    free_bin(D);
    free_km(D);
    if (D.gm) cudaFree(D.gm);
    D.gm = nullptr;
    D.gm_doubles = 0;
  }
  h->d = 0;
  h->d_user = 0;
  h->filt = RowFilter();
  h->tf_scale = false;
  h->tf_bias = 0;
  return 0;
}

int64_t agd_rows(const agd_handle *h, int32_t dev) {
  if (!h || dev < 0 || dev >= (int)h->devs.size()) return -1;
  return h->devs[dev].sh.rows;
}
int32_t agd_dim(const agd_handle *h) { return h ? h->d_user : 0; }

int agd_generate(agd_handle *h, int64_t total_rows, int32_t d, int32_t store_dtype, uint64_t seed, int32_t gradient) {
  if (!h) return 1;
  const int eb = dtype_bytes(store_dtype);
  if (!eb) return fail(h, "store_dtype must be AGD_F64, AGD_F32 or AGD_BF16");
  if (total_rows < 0) return fail(h, "negative row count");
  if (agd_clear(h)) return 1;
  if (set_dim(h, d, eb)) return 1;
  const int32_t di = h->d;
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    std::lock_guard<std::mutex> g(*D.mu);
    const long long rank = h->first_rank + (long long)i, W = h->world;
    const int64_t lo = (int64_t)(((__int128)rank * total_rows) / W), hi = (int64_t)(((__int128)(rank + 1) * total_rows) / W);
    if (reserve_locked(h, D, hi - lo, di, store_dtype)) return 1;
    if (ensure_vectors(h, D, di)) return 1;
    CK(cudaSetDevice(D.ordinal));
    D.row_base = lo;
    CK(synth_dense_launch(D.sh.X, eb, seed, lo, hi - lo, d, di, D.st));
    CK(synth_wtrue_launch(D.wtmp, seed, d, D.st));
    CK(synth_labels_launch(D.sh.X, eb, D.wtmp, D.sh.labels, seed, gradient, lo, hi - lo, d, di, D.st));
    CK(cudaMemsetAsync(D.wtmp, 0, ((size_t)di + 2) * sizeof(double), D.st));
    D.sh.rows = hi - lo;
  }
  if (sync_all(h)) return 1;
  return 0;
}

int agd_get_rows(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, void *X_out, double *labels_out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  Dev &D = h->devs[dev];
  const Shard &s = D.sh;
  if (s.csr) return fail(h, "agd_get_rows serves dense shards only");
  if (row0 < 0 || rows < 0 || row0 + rows > s.rows) return fail(h, "row range out of bounds");
  CK(cudaSetDevice(D.ordinal));
  const size_t rb = (size_t)h->d * s.elem_bytes, ub = (size_t)h->d_user * s.elem_bytes;  // stored / user row bytes
  if (X_out && rows) CK(cudaMemcpy2DAsync(X_out, ub, (const unsigned char *)s.X + (size_t)row0 * rb, rb, ub, (size_t)rows, cudaMemcpyDeviceToHost, D.st));
  if (labels_out && rows) CK(cudaMemcpyAsync(labels_out, s.labels + row0, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  return 0;
}

int agd_synth_wtrue(agd_handle *h, uint64_t seed, int32_t d, double *w_out) {
  if (!h) return 1;
  Dev &D = h->devs[0];
  CK(cudaSetDevice(D.ordinal));
  double *tmp = nullptr;
  CK(cudaMalloc(&tmp, (size_t)d * sizeof(double)));
  CK(synth_wtrue_launch(tmp, seed, d, D.st));
  CK(cudaMemcpyAsync(w_out, tmp, (size_t)d * sizeof(double), cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  cudaFree(tmp);
  return 0;
}

const char *agd_kernel_name(const agd_handle *h, int32_t dev) {
  if (!h || dev < 0 || dev >= (int)h->devs.size() || h->d <= 0) return "";
  const Shard &s = h->devs[dev].sh;
  if (s.csr) return s.elem_bytes == 8 ? "k1_csr_pipelined_kernel<double>" : "k1_csr_pipelined_kernel<float>";
  const int eb = s.elem_bytes ? s.elem_bytes : 4;
  const char *t = eb == 8 ? "double" : (eb == 4 ? "float" : "__nv_bfloat16");
  static thread_local char buf[96];
  switch (dense_kernel_of(h, eb)) {
    case 3: return "k1_tc_kernel (wgmma, bf16 storage)";
    case 1: snprintf(buf, sizeof buf, "k1_ring_kernel<%s,...>", t); return buf;
    default: snprintf(buf, sizeof buf, "k1_generic_kernel<%s>", t); return buf;
  }
}

int agd_set_option(agd_handle *h, const char *key, const char *value) {
  if (!h || !key || !value) return 1;
  if (!strcmp(key, "k1_variant")) {
    if (!strcmp(value, "auto")) h->k1_variant = 0;
    else if (!strcmp(value, "ring")) h->k1_variant = 1;
    else if (!strcmp(value, "generic")) h->k1_variant = 2;
    else if (!strcmp(value, "tc")) h->k1_variant = 4;
    else return fail(h, "k1_variant must be auto|ring|generic|tc");
    return 0;
  }
  if (!strcmp(key, "ring_stages")) { h->ring_stages = atoi(value); return 0; }
  if (!strcmp(key, "collective")) {
    if (!strcmp(value, "auto")) h->collective = 0;
    else if (!strcmp(value, "nccl")) h->collective = 1;
    else if (!strcmp(value, "p2p")) h->collective = 2;
    else return fail(h, "collective must be auto|nccl|p2p");
    free_xchg(h);
    return 0;
  }
  if (!strcmp(key, "k1_diag")) { h->k1_diag = atoi(value); return 0; }
  if (!strcmp(key, "tc_margins")) {
    if (!strcmp(value, "f32")) h->tc_margins_f64 = 0;
    else if (!strcmp(value, "f64")) h->tc_margins_f64 = 1;
    else return fail(h, "tc_margins must be f32|f64");
    return 0;
  }
  if (!strcmp(key, "ring_rows")) { h->tune_rows = atoi(value); return 0; }
  if (!strcmp(key, "ring_ctas")) { h->tune_ctas = atoi(value); return 0; }
  if (!strcmp(key, "ring_predicated")) { h->tune_full = atoi(value); return 0; }
  return fail(h, "unknown option %s", key);
}

// ---------------------------------------------------------------- applySmooth with host buffers
static int smooth_host(agd_handle *h, int32_t gradient, const double *w, const double *w2, double *loss, double *grad,
                       int64_t *count, double *loss2, double *grad2 = nullptr) {
  if (check_ready(h)) return 1;
  if (gradient < 0 || gradient > AGD_GRAD_LEAST_SQUARES_HALF) return fail(h, "unknown gradient %d", gradient);
  if (!w || !loss || !grad) return fail(h, "NULL argument");
  if (w2 && !dual_supported(h)) return fail(h, "this shard's gradient kernel has no two-point form (use two agd_smooth calls)");
  if (grad2 && !dual_full_supported(h)) return fail(h, "this shard's gradient kernel has no two-gradient form (use two agd_smooth calls)");
  const int32_t d = h->model_d();
  for (Dev &D : h->devs) {
    CK(cudaSetDevice(D.ordinal));
    if (put_point(h, D, D.wtmp, w)) return 1;                  // = broadcast, AGD.scala:193
    if (w2 && put_point(h, D, D.g_x, w2)) return 1;            // g_x doubles as the staging vector of w2
  }
  h->devs[0].ev_used = h->devs[0].ev_ar_used = 0;
  h->launches = h->collectives = 0;
  if (smooth_device(h, gradient, [](Dev &D) { return (const double *)D.wtmp; }, false,
                    w2 ? (WSel)[](Dev &D) { return (const double *)D.g_x; } : (WSel) nullptr, grad2 != nullptr))
    return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> host(2 * ((size_t)d + 4));
  CK(cudaMemcpyAsync(host.data(), D0.acc, (grad2 ? 2 : 1) * ((size_t)d + 4) * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  const double cnt = host[(size_t)d + 1];
  *loss = host[d] / cnt;                                    // AGD.scala:207
  model_values(h, host.data(), cnt, grad);
  if (count) *count = (int64_t)cnt;
  if (w2 && loss2) *loss2 = host[(size_t)d + 2] / host[(size_t)d + 3];
  if (grad2) {  // second block: [grad at w2 | loss | count | 0 | 0]
    const double *b2 = host.data() + (size_t)d + 4;
    model_values(h, b2, b2[(size_t)d + 1], grad2);
  }
  return 0;
}

int agd_smooth(agd_handle *h, int32_t gradient, const double *w, double *loss, double *grad, int64_t *count) {
  return smooth_host(h, gradient, w, nullptr, loss, grad, count, nullptr);
}

int agd_smooth_pair(agd_handle *h, int32_t gradient, const double *w, const double *w2, double *loss, double *grad,
                    int64_t *count, double *loss2) {
  if (h && (!w2 || !loss2)) return fail(h, "NULL argument");
  return smooth_host(h, gradient, w, w2, loss, grad, count, loss2);
}

int agd_smooth_two(agd_handle *h, int32_t gradient, const double *w, const double *w2, double *loss, double *grad,
                   int64_t *count, double *loss2, double *grad2) {
  if (h && (!w2 || !loss2 || !grad2)) return fail(h, "NULL argument");
  return smooth_host(h, gradient, w, w2, loss, grad, count, loss2, grad2);
}

// ---------------------------------------------------------------- scoring (score.cu)
// w (d_user doubles) -> D.wtmp, zero on the padded columns
static int stage_weights(agd_handle *h, Dev &D, const double *w) {
  CK(cudaMemsetAsync(D.wtmp, 0, ((size_t)h->d + 2) * sizeof(double), D.st));
  CK(cudaMemcpyAsync(D.wtmp, w, (size_t)h->d_user * sizeof(double), cudaMemcpyHostToDevice, D.st));
  return 0;
}

static ScoreArgs score_args(const agd_handle *h, const Dev &D, double intercept) {
  const Shard &s = D.sh;
  ScoreArgs a;
  if (s.csr) { a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; }
  else a.X = s.X;
  a.labels = s.labels; a.w = D.wtmp; a.b = intercept; a.d = h->d; a.stream = D.st;
  return a;
}

int agd_margins(agd_handle *h, int32_t dev, const double *w, double intercept, int64_t row0, int64_t rows, double *out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  if (h->d <= 0) return fail(h, "no shard loaded (call agd_load_dense / agd_load_csr / agd_generate first)");
  Dev &D = h->devs[dev];
  const Shard &s = D.sh;
  if (row0 < 0 || rows < 0 || rows > s.rows - row0)
    return fail(h, "row range [%lld, %lld + %lld) lies outside the %lld rows of device %d", (long long)row0, (long long)row0,
                (long long)rows, (long long)s.rows, dev);
  if (!w || (rows > 0 && !out)) return fail(h, "NULL argument");
  if (rows == 0) return 0;
  if (ensure_vectors(h, D, h->model_d())) return 1;
  CK(cudaSetDevice(D.ordinal));
  if (stage_weights(h, D, w)) return 1;
  // margins depend on the row only, so the range is scored in chunks through the staging buffer
  const int64_t chunk = rows < (int64_t)(1 << 22) ? rows : (int64_t)(1 << 22);
  if (ensure_stage(h, D, (size_t)chunk * sizeof(double))) return 1;
  ScoreArgs a = score_args(h, D, intercept);
  a.margins = (double *)D.stage_dev;
  for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
    a.row0 = row0 + r0;
    a.rows = rows - r0 < chunk ? rows - r0 : chunk;
    CK(score_margins_launch(a, s.elem_bytes, D.sm_count));
    CK(cudaMemcpyAsync(out + r0, D.stage_dev, (size_t)a.rows * sizeof(double), cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));   // the staging buffer is reused
  }
  return 0;
}

// Collective: one evaluation sweep per local shard, the fixed-order slab reduce, and the same exchange a sweep of agd_smooth
// uses (one epoch of the peer-memory exchange with an AGD_EVAL_N-double payload, or an NCCL all-reduce).
int agd_evaluate(agd_handle *h, int32_t gradient, const double *w, double intercept, double threshold, double *out) {
  if (check_ready(h)) return 1;
  if (gradient < 0 || gradient > AGD_GRAD_LEAST_SQUARES_HALF) return fail(h, "unknown gradient %d", gradient);
  if (!w || !out) return fail(h, "NULL argument");
  const int32_t n = AGD_EVAL_N;
  const Epoch ep = open_epoch(h, n);
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    if (!D.eval) CK(cudaMalloc(&D.eval, (size_t)n * sizeof(double)));
    if (ensure_slabs(h, D, score_max_blocks(D.sm_count), n)) return 1;
    if (stage_weights(h, D, w)) return 1;
    ScoreArgs a = score_args(h, D, intercept);
    a.rows = D.sh.rows; a.kind = gradient; a.threshold = threshold; a.slabs = D.slabs;
    a.row_base = D.row_base; a.filt = h->filt_of(D);
    int blocks = 0;
    CK(score_eval_launch(a, D.sh.elem_bytes, D.sm_count, &blocks));
    if (ep.e) {
      const XchgPub pub = publisher(h, i, ep);
      CK(k1_reduce_launch(D.slabs, blocks, n, D.eval, &pub, D.st));
    } else {
      CK(k1_reduce_launch(D.slabs, blocks, n, D.eval, nullptr, D.st));
    }
  }
  const DevBuf eval = [h](size_t i) { return h->devs[i].eval; };
  if (ep.e) {
    if (gather(h, ep, eval, 0, kXchgSum)) return 1;
  } else if (h->world > 1) {
    if (nccl_exchange(h, eval, (size_t)n, kXchgSum)) return 1;
  }
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  CK(cudaMemcpyAsync(out, D0.eval, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  return 0;
}

// ---------------------------------------------------------------- column statistics (colstats.cu)
// D.cs, in doubles: [pass-1 sums col_sum_n(d) | maxima 2 d | pass-2 sums 2 d | CSR max keys 2 d]
struct ColStatsLayout {
  size_t sums, max, dev, keys, total;
};
static ColStatsLayout colstats_layout(int32_t d) {
  ColStatsLayout L;
  L.sums = 0;
  L.max = col_sum_n(d);
  L.dev = L.max + 2 * (size_t)d;
  L.keys = L.dev + 2 * (size_t)d;
  L.total = L.keys + 2 * (size_t)d;
  return L;
}

// Collective: pass 1 on every local shard, the exchange of its sums and maxima, pass 2 (mu from the exchanged sums, on the
// device), the exchange of its sums; the host then adds a CSR column's implicit zeros in closed form.
int agd_col_stats(agd_handle *h, double *count, double *out) {
  if (check_ready(h)) return 1;
  if (!count || !out) return fail(h, "NULL argument");
  const int32_t d = h->d, du = h->d_user;
  const ColStatsLayout L = colstats_layout(d);
  const size_t nsum1 = 4 * (size_t)d + 1;   // what a dense sweep's slabs carry of the pass-1 sums (STORED is filled after)
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    if (D.cs_doubles < L.total) {
      if (D.cs) cudaFree(D.cs);
      D.cs = nullptr;
      D.cs_doubles = 0;
      CK(cudaMalloc(&D.cs, L.total * sizeof(double)));
      D.cs_doubles = L.total;
    }
    const Shard &s = D.sh;
    ColStatsArgs a;
    a.rows = s.rows; a.d = d; a.row_base = D.row_base; a.filt = h->filt_of(D); a.stream = D.st;
    if (s.csr) {
      a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val;
      a.out = D.cs + L.sums; a.keys = reinterpret_cast<unsigned long long *>(D.cs + L.keys);
      CK(cudaMemsetAsync(D.cs + L.sums, 0, L.max * sizeof(double), D.st));
      CK(cudaMemsetAsync(D.cs + L.keys, 0, 2 * (size_t)d * sizeof(double), D.st));
      CK(colstats_csr_launch(a, 1, s.elem_bytes, D.sm_count));
      CK(colstats_unkey_launch(a.keys, 2 * d, D.cs + L.max, D.st));
    } else {
      const int mb = colstats_max_blocks(D.sm_count, d);
      if (ensure_slabs(h, D, mb, (int32_t)(nsum1 + 2 * (size_t)d))) return 1;
      a.X = s.X; a.slabs = D.slabs; a.max_slabs = D.slabs + (size_t)mb * nsum1;
      int blocks = 0;
      CK(colstats_dense_launch(a, 1, s.elem_bytes, D.sm_count, &blocks));
      CK(k1_reduce_launch(a.slabs, blocks, (int32_t)nsum1, D.cs + L.sums, nullptr, D.st));
      CK(colstats_max_reduce_launch(a.max_slabs, blocks, 2 * d, D.cs + L.max, D.st));
      CK(colstats_fill_stored_launch(D.cs + L.sums, d, D.st));
    }
  }
  if (world_reduce(h, [&](size_t i) { return h->devs[i].cs + L.sums; }, col_sum_n(d), kXchgSum)) return 1;
  if (world_reduce(h, [&](size_t i) { return h->devs[i].cs + L.max; }, 2 * (size_t)d, kXchgMax)) return 1;
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    const Shard &s = D.sh;
    ColStatsArgs a;
    a.rows = s.rows; a.d = d; a.row_base = D.row_base; a.filt = h->filt_of(D); a.stream = D.st; a.mu_sums = D.cs + L.sums;
    if (s.csr) {
      a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; a.out = D.cs + L.dev; a.mu = D.cs + L.keys;   // the keys are spent
      CK(colstats_mu_launch(D.cs + L.sums, d, D.cs + L.keys, D.st));
      CK(cudaMemsetAsync(D.cs + L.dev, 0, 2 * (size_t)d * sizeof(double), D.st));
      CK(colstats_csr_launch(a, 2, s.elem_bytes, D.sm_count));
    } else {
      a.X = s.X; a.slabs = D.slabs;
      int blocks = 0;
      CK(colstats_dense_launch(a, 2, s.elem_bytes, D.sm_count, &blocks));
      CK(k1_reduce_launch(a.slabs, blocks, 2 * d, D.cs + L.dev, nullptr, D.st));
    }
  }
  if (world_reduce(h, [&](size_t i) { return h->devs[i].cs + L.dev; }, 2 * (size_t)d, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> r(L.keys);
  CK(cudaMemcpyAsync(r.data(), D0.cs, L.keys * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  const double n = r[4 * (size_t)d];
  *count = n;
  for (int32_t c = 0; c < du; ++c) {
    const double sum = r[c], implicit = n - r[4 * (size_t)d + 1 + c];
    double dev = r[L.dev + c], dev2 = r[L.dev + d + c], mx = r[L.max + c], nmn = r[L.max + d + c];
    if (implicit > 0.0) {   // CSR: the column's zeros that are not stored, each x - mu = -mu
      const double mu = sum / n;   // the mu of pass 2
      dev += implicit * -mu;
      dev2 += implicit * (mu * mu);
      mx = std::fmax(mx, 0.0);
      nmn = std::fmax(nmn, 0.0);
    }
    const double v[AGD_COLSTAT_N] = {sum, r[d + c], r[2 * (size_t)d + c], r[3 * (size_t)d + c], dev, dev2, mx, -nmn};
    for (int k = 0; k < AGD_COLSTAT_N; ++k) out[(size_t)k * du + c] = v[k];
  }
  return 0;
}

// ---------------------------------------------------------------- cross-products (gramian.cu)
// D.gm, in doubles: [packed result P | mu d | pass-1 sums col_sum_n(d) | CSR max keys 2 d | work], P = gramian_packed_n(d); work =
// the dense sweep's slabs (splits x P), or a CSR shard's uncentered sums (P) when they are centered after
struct GramianLayout {
  size_t out, mu, sums, keys, work, total;
};
static GramianLayout gramian_layout(int32_t d, size_t work) {
  GramianLayout L;
  L.out = 0;
  L.mu = gramian_packed_n(d);
  L.sums = L.mu + (size_t)d;
  L.keys = L.sums + col_sum_n(d);
  L.work = L.keys + 2 * (size_t)d;
  L.total = L.work + work;
  return L;
}

// Collective.  Centered: colStats pass 1 on every local shard and the exchange of its sums (4 d + 1, the same payload on dense
// and CSR shards), mu on the device; then the cross-product sweep of every local shard, its packed sums exchanged over the world
// in epochs of one slot stride.  The host mirrors the packed triangle into the full matrix.
int agd_gramian(agd_handle *h, int32_t centered, double *count, double *out) {
  if (check_ready(h)) return 1;
  if (h->d_user > AGD_GRAMIAN_MAX_DIM)
    return fail(h, "agd_gramian: d = %d features; the d x d result is limited to d <= %d", h->d_user, AGD_GRAMIAN_MAX_DIM);
  if (!count || !out) return fail(h, "NULL argument");
  const int32_t d = h->d, du = h->d_user;
  const size_t P = gramian_packed_n(d), nsum1 = 4 * (size_t)d + 1;
  std::vector<int> splits(h->devs.size(), 0);
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    const Shard &s = D.sh;
    if (!s.csr) splits[i] = gramian_splits(D.sm_count, d, s.rows);
    const GramianLayout L = gramian_layout(d, s.csr ? (centered ? P : 0) : (size_t)splits[i] * P);
    if (D.gm_doubles < L.total) {
      if (D.gm) cudaFree(D.gm);
      D.gm = nullptr;
      D.gm_doubles = 0;
      if (cudaMalloc(&D.gm, L.total * sizeof(double)) != cudaSuccess) {
        cudaGetLastError();
        return fail(h, "agd_gramian: cannot allocate %zu bytes of scratch on device %d", L.total * sizeof(double), D.ordinal);
      }
      D.gm_doubles = L.total;
    }
    if (!centered) continue;
    ColStatsArgs a;
    a.rows = s.rows; a.d = d; a.row_base = D.row_base; a.filt = h->filt_of(D); a.stream = D.st;
    if (s.csr) {
      a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val;
      a.out = D.gm + L.sums; a.keys = reinterpret_cast<unsigned long long *>(D.gm + L.keys);
      CK(cudaMemsetAsync(D.gm + L.sums, 0, (col_sum_n(d) + 2 * (size_t)d) * sizeof(double), D.st));
      CK(colstats_csr_launch(a, 1, s.elem_bytes, D.sm_count));
    } else {
      const int mb = colstats_max_blocks(D.sm_count, d);
      if (ensure_slabs(h, D, mb, (int32_t)(nsum1 + 2 * (size_t)d))) return 1;
      a.X = s.X; a.slabs = D.slabs; a.max_slabs = D.slabs + (size_t)mb * nsum1;
      int blocks = 0;
      CK(colstats_dense_launch(a, 1, s.elem_bytes, D.sm_count, &blocks));
      CK(k1_reduce_launch(a.slabs, blocks, (int32_t)nsum1, D.gm + L.sums, nullptr, D.st));
    }
  }
  const GramianLayout L = gramian_layout(d, 0);   // every offset below the work area is the same on every device
  if (centered) {
    if (world_reduce(h, [&](size_t i) { return h->devs[i].gm + L.sums; }, nsum1, kXchgSum)) return 1;
    for (Dev &D : h->devs) {
      CK(cudaSetDevice(D.ordinal));
      CK(colstats_mu_launch(D.gm + L.sums, d, D.gm + L.mu, D.st));
    }
  }
  for (size_t i = 0; i < h->devs.size(); ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    const Shard &s = D.sh;
    GramianArgs a;
    a.rows = s.rows; a.d = d; a.stream = D.st;
    if (s.csr) {
      a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; a.row_base = D.row_base; a.filt = h->filt_of(D);
      a.out = D.gm + (centered ? L.work : L.out);
      CK(cudaMemsetAsync(a.out, 0, P * sizeof(double), D.st));
      CK(gramian_csr_launch(a, s.elem_bytes, D.sm_count));
      if (centered) CK(gramian_center_launch(a.out, D.gm + L.mu, d, D.gm + L.out, D.st));
    } else {
      if (ensure_view_bits(h, D)) return 1;
      a.X = s.X; a.view_bits = h->filt.n ? D.view_bits : nullptr; a.mu = centered ? D.gm + L.mu : nullptr;
      a.slabs = D.gm + L.work;
      CK(gramian_dense_launch(a, s.elem_bytes, D.sm_count, splits[i]));
      CK(k1_reduce_launch(a.slabs, splits[i], (int32_t)P, D.gm + L.out, nullptr, D.st));
    }
  }
  if (world_reduce(h, [&](size_t i) { return h->devs[i].gm + L.out; }, P, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> r(P);
  CK(cudaMemcpyAsync(r.data(), D0.gm + L.out, P * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  // internal index k (d = the augmented one) -> the caller's (du); padded columns du .. d - 1 are dropped
  const size_t n1 = (size_t)du + 1;
  auto ext = [&](int32_t k) { return k == d ? du : k; };
  size_t p = 0;
  for (int32_t i = 0; i <= d; ++i)
    for (int32_t j = i; j <= d; ++j, ++p) {
      if ((i >= du && i < d) || (j >= du && j < d)) continue;
      const size_t a = (size_t)ext(i), b = (size_t)ext(j);
      out[a * n1 + b] = r[p];
      out[b * n1 + a] = r[p];
    }
  *count = r[P - 1];
  return 0;
}

// ---------------------------------------------------------------- projection (project.cu)
// Rank-local.  Per local device: the view's bitmap and the exclusive scan of its tile counts (the kept rows, read back), the
// destination shard reserved as a load of that many rows would reserve it, B and c padded into the source device's staging
// buffer, and one launch on the source's stream.  Any failure after the checks clears dst.
static int project_device(agd_handle *h, Dev &D, const std::vector<double> &Bp, const std::vector<double> &cp, int32_t k,
                          int32_t kp, agd_handle *dst, Dev &E, int32_t store_dtype) {
  const Shard &s = D.sh;
  const bool filtered = h->filt.n > 0;
  const size_t tiles = (size_t)((s.rows + kPjRows - 1) / kPjRows);
  const size_t bytes = (Bp.size() + cp.size() + tiles + 1) * sizeof(double);
  CK(cudaSetDevice(D.ordinal));
  if (D.stage_bytes < bytes) {
    if (D.stage_dev) cudaFree(D.stage_dev);
    D.stage_dev = nullptr;
    D.stage_bytes = 0;
    if (cudaMalloc(&D.stage_dev, bytes) != cudaSuccess) {
      cudaGetLastError();
      return fail(h, "agd_project: cannot allocate %zu bytes of scratch on device %d", bytes, D.ordinal);
    }
    D.stage_bytes = bytes;
  }
  double *Bd = (double *)D.stage_dev, *cd = Bd + Bp.size();
  long long *tile_base = (long long *)(cd + cp.size()), *total_d = tile_base + tiles;
  CK(cudaMemcpyAsync(Bd, Bp.data(), Bp.size() * sizeof(double), cudaMemcpyHostToDevice, D.st));
  CK(cudaMemcpyAsync(cd, cp.data(), cp.size() * sizeof(double), cudaMemcpyHostToDevice, D.st));
  long long kept = s.rows;
  if (filtered && s.rows > 0) {
    if (ensure_view_bits(h, D)) return 1;
    CK(project_scan_launch(D.view_bits, s.rows, tile_base, total_d, D.st));
    CK(cudaMemcpyAsync(&kept, total_d, sizeof kept, cudaMemcpyDeviceToHost, D.st));
  }
  CK(cudaStreamSynchronize(D.st));
  {
    std::lock_guard<std::mutex> g(*E.mu);
    if (reserve_locked(dst, E, kept, dst->d, store_dtype)) {
      const std::string why = dst->err;
      return fail(h, "agd_project: cannot reserve %zu bytes for %lld rows x %d features on device %d (%s)",
                  (size_t)kept * dst->d * dtype_bytes(store_dtype) + ((size_t)kept + 64) * sizeof(double), kept, dst->d,
                  E.ordinal, why.c_str());
    }
  }
  ProjectArgs a;
  if (s.csr) { a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; }
  else a.X = s.X;
  a.labels = s.labels; a.rows = s.rows; a.d = h->d; a.stream = D.st;
  a.view_bits = filtered ? D.view_bits : nullptr; a.tile_base = filtered ? tile_base : nullptr;
  a.B = Bd; a.c = cd; a.k = k; a.kp = kp;
  a.Y = E.sh.X; a.Ylabels = E.sh.labels; a.ldy = dst->d; a.out_bytes = dtype_bytes(store_dtype);
  if (kept > 0) {
    if (s.csr) CK(project_csr_launch(a, s.elem_bytes, D.sm_count));
    else CK(project_dense_launch(a, s.elem_bytes));
  }
  CK(cudaStreamSynchronize(D.st));   // dst's own stream never races the rows written on this one
  E.sh.rows = kept;
  if (!filtered) E.row_base = D.row_base;   // the same rows, numbered as the source numbers them
  return 0;
}

int agd_project(agd_handle *h, const double *B, int32_t k, const double *offset, agd_handle *dst, int32_t store_dtype) {
  if (!h) return 1;
  if (!dst || dst == h) return fail(h, "agd_project: dst must be another handle");
  if (h->d <= 0) return fail(h, "no shard loaded (call agd_load_dense / agd_load_csr / agd_generate first)");
  bool empty = dst->d == 0;
  for (const Dev &E : dst->devs) empty = empty && E.sh.rows == 0 && E.sh.cap == 0;
  if (!empty) return fail(h, "agd_project: the destination handle is not empty (agd_clear it or open a new one)");
  bool same = dst->devs.size() == h->devs.size() && dst->world == h->world && dst->first_rank == h->first_rank;
  for (size_t i = 0; same && i < h->devs.size(); ++i) same = dst->devs[i].ordinal == h->devs[i].ordinal;
  if (!same) return fail(h, "agd_project: dst must be opened on the same local devices in the same world position as the source");
  if (k < 1) return fail(h, "agd_project: k = %d columns (at least 1)", k);
  if (!dtype_bytes(store_dtype)) return fail(h, "store_dtype must be AGD_F64, AGD_F32 or AGD_BF16");
  if (!B) return fail(h, "NULL argument");
  const int32_t du = h->d_user;
  for (size_t q = 0; q < (size_t)du * k; ++q)
    if (!std::isfinite(B[q])) return fail(h, "agd_project: B[%zu][%zu] = %g is not finite", q / k, q % k, B[q]);
  if (offset)
    for (int32_t j = 0; j < k; ++j)
      if (!std::isfinite(offset[j])) return fail(h, "agd_project: offset[%d] = %g is not finite", j, offset[j]);
  for (const Dev &D : h->devs)
    if (D.sh.rows >= (int64_t)1 << 31)
      return fail(h, "agd_project: %lld rows on device %d (at most 2^31 - 1)", (long long)D.sh.rows, D.ordinal);
  // B as the kernels read it: [bd][kp], rows padded to whole 16-row chunks and columns to whole column tiles, zeros elsewhere
  const int32_t bd = (h->d + 15) / 16 * 16, tc = project_tile_cols(k), kp = (k + tc - 1) / tc * tc;
  std::vector<double> Bp((size_t)bd * kp, 0.0), cp((size_t)kp, 0.0);
  for (int32_t l = 0; l < du; ++l) memcpy(&Bp[(size_t)l * kp], B + (size_t)l * k, (size_t)k * sizeof(double));
  if (offset) memcpy(cp.data(), offset, (size_t)k * sizeof(double));
  if (set_dim(dst, k, dtype_bytes(store_dtype))) return fail(h, "agd_project: %s", dst->err.c_str());
  for (size_t i = 0; i < h->devs.size(); ++i)
    if (project_device(h, h->devs[i], Bp, cp, k, kp, dst, dst->devs[i], store_dtype)) {
      agd_clear(dst);
      return 1;
    }
  return 0;
}

// ---------------------------------------------------------------- ranking metrics (rank.cu)
static int bin_list(agd_handle *h, Dev &D, long long n, int64_t *len);
// One shard: the key form of the scoring sweep (rows of the view, non-NaN margins), the radix sort and the run-length reduce
// into this device's curve (D.bin[kBinList], *len records); *nan = rows of the view whose margin is NaN.
static int bin_local(agd_handle *h, Dev &D, double intercept, int64_t *len, int64_t *nan) {
  const int64_t rows = D.sh.rows;
  if (rows >= (int64_t)1 << 31) return fail(h, "agd_binary_curve: %lld rows on device %d (at most 2^31 - 1)", (long long)rows, D.ordinal);
  const size_t r1 = rows > 0 ? (size_t)rows : 1;
  if (ensure_bin(h, D, kBinMisc, kBinMiscAll + 16 * (size_t)h->world + 8 * ((size_t)h->world + 1)) ||
      ensure_bin(h, D, kBinKeys0, 8 * r1) || ensure_bin(h, D, kBinKeys1, 8 * r1) || ensure_bin(h, D, kBinVals0, r1) ||
      ensure_bin(h, D, kBinVals1, r1))
    return 1;
  char *misc = (char *)D.bin[kBinMisc];
  unsigned *counters = (unsigned *)(misc + kBinMiscCounters);
  CK(cudaMemsetAsync(counters, 0, 2 * sizeof(unsigned), D.st));
  ScoreArgs a = score_args(h, D, intercept);
  a.rows = rows; a.row_base = D.row_base; a.filt = h->filt_of(D);
  a.keys = (unsigned long long *)D.bin[kBinKeys0]; a.classes = (uint8_t *)D.bin[kBinVals0]; a.counters = counters;
  CK(score_keys_launch(a, D.sh.elem_bytes, D.sm_count));
  unsigned cnt[2];
  CK(cudaMemcpyAsync(cnt, counters, sizeof cnt, cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  *nan = cnt[1];
  return bin_list(h, D, cnt[0], len);
}

// The n keys and 1-byte values in D.bin[kBinKeys0] / [kBinVals0] sorted and reduced into this device's list (D.bin[kBinList],
// *len records)
static int bin_list(agd_handle *h, Dev &D, long long n, int64_t *len) {
  char *misc = (char *)D.bin[kBinMisc];
  if (ensure_bin(h, D, kBinTiles, std::max(bin_sort_tile_words(n) * sizeof(unsigned), bin_runs_tile_words(n) * sizeof(long long))) ||
      ensure_bin(h, D, kBinList, (n > 0 ? (size_t)n : 1) * sizeof(BinRec)))
    return 1;
  unsigned long long *keys[2] = {(unsigned long long *)D.bin[kBinKeys0], (unsigned long long *)D.bin[kBinKeys1]};
  void *vals[2] = {D.bin[kBinVals0], D.bin[kBinVals1]};
  int which = 0, passes = 0;
  CK(bin_sort_pairs(keys, vals, 1, n, (unsigned *)misc, (unsigned *)D.bin[kBinTiles], &which, &passes, D.st));
  long long *runs = (long long *)(misc + kBinMiscRuns);
  CK(bin_runs_launch(keys[which], vals[which], 1, nullptr, nullptr, n, (long long *)D.bin[kBinTiles], (BinRec *)D.bin[kBinList],
                     runs, D.st));
  long long k = 0;
  CK(cudaMemcpyAsync(&k, runs, sizeof k, cudaMemcpyDeviceToHost, D.st));
  CK(cudaStreamSynchronize(D.st));
  *len = k;
  return 0;
}

// Every rank's list -> the world's curve on device 0 (*curve, *K records), identical on every rank: the lengths travel first,
// then the lists (rank r's at r * Lmax in kBinUnion), each by world_concat; device 0 concatenates them in rank order, sorts and
// reduces again.
static int bin_world(agd_handle *h, const std::vector<int64_t> &len, const std::vector<int64_t> &nan, BinRec **curve,
                     int64_t *K, int64_t *nan_total) {
  const int W = h->world, nd = (int)h->devs.size();
  // 1. {list length, NaN count} of every rank
  auto misc_at = [h](size_t i, size_t off) { return (double *)((char *)h->devs[i].bin[kBinMisc] + off); };
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    const double v[2] = {(double)len[i], (double)nan[i]};
    CK(cudaMemcpyAsync(misc_at(i, kBinMiscOwn), v, sizeof v, cudaMemcpyHostToDevice, D.st));
    CK(cudaStreamSynchronize(D.st));   // v is on this stack frame
  }
  if (world_concat(h, [&](size_t i) { return misc_at(i, kBinMiscOwn); }, 2, [&](size_t i) { return misc_at(i, kBinMiscAll); })) return 1;
  std::vector<double> all((size_t)2 * W);
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  CK(cudaMemcpyAsync(all.data(), misc_at(0, kBinMiscAll), all.size() * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  std::vector<long long> off((size_t)W + 1, 0);
  long long lmax = 0, nans = 0;
  for (int r = 0; r < W; ++r) {
    const long long l = (long long)all[2 * (size_t)r];
    off[(size_t)r + 1] = off[(size_t)r] + l;
    lmax = std::max(lmax, l);
    nans += (long long)all[2 * (size_t)r + 1];
  }
  const long long T = off[(size_t)W];
  *nan_total = nans;
  *K = 0;
  if (T == 0) return 0;
  if (T >= (long long)1 << 31) return fail(h, "agd_binary_curve: %lld distinct scores over the world (at most 2^31 - 1)", T);
  // 2. the lists
  const size_t ld = 3 * (size_t)lmax;   // doubles of one rank's block
  auto uni = [h](size_t i) { return (double *)h->devs[i].bin[kBinUnion]; };
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    if (ensure_bin(h, D, kBinUnion, (size_t)W * ld * sizeof(double))) return 1;
    if (len[i] > 0) CK(cudaMemcpyAsync(uni(i) + (size_t)(h->first_rank + i) * ld, D.bin[kBinList], (size_t)len[i] * sizeof(BinRec),
                                       cudaMemcpyDeviceToDevice, D.st));
  }
  if (world_concat(h, [&](size_t i) { return uni(i) + (size_t)(h->first_rank + (int)i) * ld; }, ld, uni)) return 1;
  // 3. device 0: the concatenation in rank order, sorted and reduced
  CK(cudaSetDevice(D0.ordinal));
  const size_t t1 = (size_t)T;
  if (ensure_bin(h, D0, kBinKeys0, 8 * t1) || ensure_bin(h, D0, kBinKeys1, 8 * t1) || ensure_bin(h, D0, kBinVals0, 4 * t1) ||
      ensure_bin(h, D0, kBinVals1, 4 * t1) || ensure_bin(h, D0, kBinCounts, 16 * t1) ||
      ensure_bin(h, D0, kBinCurve, t1 * sizeof(BinRec)) ||
      ensure_bin(h, D0, kBinTiles, std::max(bin_sort_tile_words(T) * sizeof(unsigned), bin_runs_tile_words(T) * sizeof(long long))))
    return 1;
  char *misc = (char *)D0.bin[kBinMisc];
  long long *off_dev = (long long *)(misc + kBinMiscAll + 16 * (size_t)W);
  CK(cudaMemcpyAsync(off_dev, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice, D0.st));
  long long *upos = (long long *)D0.bin[kBinCounts], *uneg = upos + T;
  unsigned long long *keys[2] = {(unsigned long long *)D0.bin[kBinKeys0], (unsigned long long *)D0.bin[kBinKeys1]};
  void *vals[2] = {D0.bin[kBinVals0], D0.bin[kBinVals1]};
  CK(bin_union_prep_launch((const BinRec *)D0.bin[kBinUnion], lmax, off_dev, W, T, keys[0], (uint32_t *)vals[0], upos, uneg, D0.st));
  int which = 0, passes = 0;
  CK(bin_sort_pairs(keys, vals, 4, T, (unsigned *)misc, (unsigned *)D0.bin[kBinTiles], &which, &passes, D0.st));   // synchronises
  long long *runs = (long long *)(misc + kBinMiscRuns);
  CK(bin_runs_launch(keys[which], vals[which], 4, upos, uneg, T, (long long *)D0.bin[kBinTiles], (BinRec *)D0.bin[kBinCurve], runs,
                     D0.st));
  long long k = 0;
  CK(cudaMemcpyAsync(&k, runs, sizeof k, cudaMemcpyDeviceToHost, D0.st));
  CK(cudaStreamSynchronize(D0.st));
  *curve = (BinRec *)D0.bin[kBinCurve];
  *K = k;
  return 0;
}

// Collective: the local curves, their union over the world, the areas on device 0; the curve is copied out only on request.
int agd_binary_curve(agd_handle *h, const double *w, double intercept, int64_t capacity, double *margin_out, int64_t *tp_out,
                     int64_t *fp_out, int64_t *n_points, double *out) {
  if (check_ready(h)) return 1;
  if (!w || !n_points || !out) return fail(h, "NULL argument");
  if (capacity < 0) return fail(h, "capacity must be >= 0 (got %lld)", (long long)capacity);
  if (capacity > 0 && (!margin_out || !tp_out || !fp_out)) return fail(h, "NULL argument");
  const int nd = (int)h->devs.size();
  std::vector<int64_t> len((size_t)nd), nan((size_t)nd);
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    if (stage_weights(h, D, w)) return 1;
    if (bin_local(h, D, intercept, &len[(size_t)i], &nan[(size_t)i])) return 1;
  }
  Dev &D0 = h->devs[0];
  BinRec *curve = (BinRec *)D0.bin[kBinList];
  int64_t K = len[0], nans = nan[0];
  if (h->world > 1 && bin_world(h, len, nan, &curve, &K, &nans)) return 1;
  CK(cudaSetDevice(D0.ordinal));
  double areas[2] = {0.0, 0.0};
  BinRec last = {0ull, 0, 0};
  std::vector<BinRec> host;
  if (K > 0) {
    if (ensure_bin(h, D0, kBinTiles, 2 * (size_t)bin_area_blocks(K) * sizeof(double))) return 1;
    double *dev_areas = (double *)((char *)D0.bin[kBinMisc] + kBinMiscAreas);
    CK(bin_areas_launch(curve, K, (double *)D0.bin[kBinTiles], dev_areas, D0.st));
    CK(cudaMemcpyAsync(areas, dev_areas, sizeof areas, cudaMemcpyDeviceToHost, D0.st));
    CK(cudaMemcpyAsync(&last, curve + (K - 1), sizeof last, cudaMemcpyDeviceToHost, D0.st));
    if (capacity >= K) {
      host.resize((size_t)K);
      CK(cudaMemcpyAsync(host.data(), curve, (size_t)K * sizeof(BinRec), cudaMemcpyDeviceToHost, D0.st));
    }
  }
  if (sync_all(h)) return 1;
  const double nan_v = std::numeric_limits<double>::quiet_NaN();
  const int64_t P = last.tp, Nn = last.fp;
  out[AGD_BIN_POS] = (double)P;
  out[AGD_BIN_NEG] = (double)Nn;
  out[AGD_BIN_NAN] = (double)nans;
  out[AGD_BIN_AUROC] = (P > 0 && Nn > 0) ? areas[0] : nan_v;
  out[AGD_BIN_AUPR] = P > 0 ? areas[1] : nan_v;
  *n_points = K;
  for (size_t k = 0; k < host.size(); ++k) {
    margin_out[k] = margin_of_key(host[k].key);
    tp_out[k] = host[k].tp;
    fp_out[k] = host[k].fp;
  }
  return 0;
}

// ---------------------------------------------------------------- clustering (kmeans.cu)
// The centres as the kernels read them, built once on the host for every device: C [k][md] in the internal width md = d + bias
// (zeros on padded columns), B [round_up(d, 16)][kp] = (s o C)^T zero-padded, cb = the bias entries, cn = ||c_j||^2 added over
// the columns in order.  With an offset (agd_linear_*: the rows of W as centres, kKmLinear scores) cn = the offset and C is
// not built.
struct KmCentres {
  int32_t k = 0, kp = 0, md = 0;
  std::vector<double> buf;   // B | cb | cn | C
  size_t nB = 0;
};
static int km_centres(agd_handle *h, const char *what, const double *centers, int32_t k, KmCentres &c,
                      const double *offset = nullptr) {
  if (h->d <= 0) return fail(h, "no shard loaded (call agd_load_dense / agd_load_csr / agd_generate first)");
  const bool linear = offset != nullptr;
  if (k < 1) return fail(h, linear ? "%s: C = %d classes (at least 1)" : "%s: k = %d centres (at least 1)", what, k);
  if (!centers) return fail(h, "NULL argument");
  for (const Dev &D : h->devs)
    if (D.sh.rows >= (int64_t)1 << 31) return fail(h, "%s: %lld rows on device %d (at most 2^31 - 1)", what, (long long)D.sh.rows, D.ordinal);
  const int32_t du = h->d_user, d = h->d, b = h->tf_bias, Dx = du + b;
  for (size_t q = 0; q < (size_t)k * Dx; ++q)
    if (!std::isfinite(centers[q]))
      return fail(h, linear ? "%s: W[%zu][%zu] = %g is not finite" : "%s: centre %zu, feature %zu = %g is not finite", what, q / Dx,
                  q % Dx, centers[q]);
  if (linear)
    for (int32_t j = 0; j < k; ++j)
      if (!std::isfinite(offset[j])) return fail(h, "%s: offset[%d] = %g is not finite", what, j, offset[j]);
  const int32_t tc = project_tile_cols(k), bd = (d + 15) / 16 * 16;
  c.k = k; c.kp = (k + tc - 1) / tc * tc; c.md = d + b;
  c.nB = (size_t)bd * c.kp;
  c.buf.assign(c.nB + 2 * (size_t)c.kp + (linear ? 0 : (size_t)k * c.md), 0.0);
  double *B = c.buf.data(), *cb = B + c.nB, *cn = cb + c.kp, *C = cn + c.kp;
  for (int32_t j = 0; j < k; ++j) {
    const double *src = centers + (size_t)j * Dx;
    for (int32_t l = 0; l < du; ++l) B[(size_t)l * c.kp + j] = h->tf_scale ? h->tf_scale_host[(size_t)l] * src[l] : src[l];
    if (b) cb[j] = src[du];
    if (linear) {
      cn[j] = offset[j];
      continue;
    }
    double *cj = C + (size_t)j * c.md;
    for (int32_t l = 0; l < du; ++l) cj[l] = src[l];
    if (b) cj[d] = src[du];
    double n = 0.0;
    for (int32_t l = 0; l < c.md; ++l) n += cj[l] * cj[l];
    cn[j] = n;
  }
  return 0;
}

// D's arguments for the rows [0, rows) of its shard in the view's feature space (no centres)
static int km_data(agd_handle *h, Dev &D, KmeansArgs &a) {
  const Shard &s = D.sh;
  CK(cudaSetDevice(D.ordinal));
  if (h->filt.n && ensure_view_bits(h, D)) return 1;
  a = KmeansArgs();
  if (s.csr) { a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; }
  else a.X = s.X;
  a.rows = s.rows; a.d = h->d; a.md = h->d + h->tf_bias; a.bias = h->tf_bias; a.scale = h->scale_of(D);
  a.view_bits = h->filt.n ? D.view_bits : nullptr;
  a.stream = D.st;
  return 0;
}

// ... and the centres uploaded
static int km_args(agd_handle *h, Dev &D, const KmCentres &c, KmeansArgs &a) {
  if (km_data(h, D, a)) return 1;
  if (ensure_km(h, D, kKmCentres, c.buf.size() * sizeof(double))) return 1;
  double *dev = (double *)D.km[kKmCentres];
  CK(cudaMemcpyAsync(dev, c.buf.data(), c.buf.size() * sizeof(double), cudaMemcpyHostToDevice, D.st));
  a.k = c.k; a.kp = c.kp;
  a.B = dev; a.cb = dev + c.nB; a.cn = a.cb + c.kp; a.C = a.cn + c.kp;
  return 0;
}

// centres (kKmLinear: argmax classes) of rows [a.row0, a.row0 + a.rows) into D.km[kKmCluster]
static int km_assign(agd_handle *h, Dev &D, KmeansArgs &a, int score_mode = kKmDistance) {
  const size_t r1 = a.rows > 0 ? (size_t)a.rows : 1;
  if (ensure_km(h, D, kKmCluster, r1 * sizeof(int32_t))) return 1;
  a.cluster = (int32_t *)D.km[kKmCluster];
  if (!a.rowptr && a.kp > 128) {
    const size_t tiles = (size_t)a.kp / 128;
    if (ensure_km(h, D, kKmTiles, tiles * r1 * (sizeof(double) + sizeof(int32_t)))) return 1;
    a.tile_score = (double *)D.km[kKmTiles];
    a.tile_idx = (int32_t *)(a.tile_score + tiles * r1);
  }
  CK(kmeans_assign_launch(a, D.sh.elem_bytes, D.sm_count, score_mode));
  return 0;
}

// One device's sums over the rows a.cluster assigns to a.k groups (-1: none): the payload [sums k x md | counts k | cost] in
// D.km[kKmPayload], cost = the residuals to the centres (kKmResidual) or the count of entries not >= 0 (kKmNegatives)
static int km_sums_device(agd_handle *h, Dev &D, const KmeansArgs &a, int sums_mode) {
  const Shard &s = D.sh;
  const int32_t k = a.k, md = a.md;
  const size_t P = (size_t)k * md + k + 1, r1 = s.rows > 0 ? (size_t)s.rows : 1;
  if (ensure_km(h, D, kKmPayload, P * sizeof(double)) || ensure_km(h, D, kKmMisc, 8 * 256 * sizeof(unsigned) + ((size_t)k + 1) * 8) ||
      ensure_km(h, D, kKmKeys0, 8 * r1) || ensure_km(h, D, kKmVals0, 4 * r1))
    return 1;
  double *pay = (double *)D.km[kKmPayload];
  unsigned *hist = (unsigned *)D.km[kKmMisc];
  unsigned long long *counts = (unsigned long long *)(hist + 8 * 256);
  unsigned long long *keys[2] = {(unsigned long long *)D.km[kKmKeys0], nullptr};
  void *vals[2] = {D.km[kKmVals0], nullptr};
  CK(cudaMemsetAsync(pay, 0, P * sizeof(double), D.st));
  CK(cudaMemsetAsync(counts, 0, ((size_t)k + 1) * 8, D.st));
  CK(kmeans_keys_launch(a.cluster, s.rows, k, keys[0], (uint32_t *)vals[0], counts, D.st));
  if (s.csr) {
    CK(kmeans_sums_csr_launch(a, s.elem_bytes, D.sm_count, pay, sums_mode));
  } else if (s.rows > 0) {
    // rows sorted stably by centre, then each centre's rows in pieces of kKmPiece, every piece's columns added in sorted order
    if (ensure_km(h, D, kKmKeys1, 8 * r1) || ensure_km(h, D, kKmVals1, 4 * r1) ||
        ensure_km(h, D, kKmSortTiles, bin_sort_tile_words(s.rows) * sizeof(unsigned)))
      return 1;
    keys[1] = (unsigned long long *)D.km[kKmKeys1];
    vals[1] = D.km[kKmVals1];
    int which = 0, passes = 0;
    CK(bin_sort_pairs(keys, vals, 4, s.rows, hist, (unsigned *)D.km[kKmSortTiles], &which, &passes, D.st));   // synchronises
    std::vector<unsigned long long> cnt((size_t)k);
    CK(cudaMemcpyAsync(cnt.data(), counts, (size_t)k * 8, cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));
    std::vector<long long> pstart;
    std::vector<int32_t> pcl, pfirst((size_t)k + 1);
    long long off = 0;
    for (int32_t j = 0; j < k; ++j) {
      pfirst[(size_t)j] = (int32_t)pcl.size();
      for (long long q = 0; q < (long long)cnt[(size_t)j]; q += kKmPiece) {
        pstart.push_back(off + q);
        pcl.push_back(j);
      }
      off += (long long)cnt[(size_t)j];
    }
    pfirst[(size_t)k] = (int32_t)pcl.size();
    pstart.push_back(off);
    const long long np = (long long)pcl.size();
    const size_t pbytes = pstart.size() * 8 + (pcl.size() + pfirst.size()) * 4;
    if (ensure_km(h, D, kKmPieces, pbytes) || ensure_km(h, D, kKmPart, (2 * (size_t)np + 1) * md * sizeof(double))) return 1;
    long long *ps = (long long *)D.km[kKmPieces];
    int32_t *pc = (int32_t *)(ps + pstart.size()), *pf = pc + pcl.size();
    CK(cudaMemcpyAsync(ps, pstart.data(), pstart.size() * 8, cudaMemcpyHostToDevice, D.st));
    if (np) CK(cudaMemcpyAsync(pc, pcl.data(), pcl.size() * 4, cudaMemcpyHostToDevice, D.st));
    CK(cudaMemcpyAsync(pf, pfirst.data(), pfirst.size() * 4, cudaMemcpyHostToDevice, D.st));
    double *part = (double *)D.km[kKmPart], *pres = part + (size_t)np * md, *colres = pres + (size_t)np * md;
    CK(kmeans_sums_dense_launch(a, s.elem_bytes, (const uint32_t *)vals[which], ps, pc, np, part, pres, sums_mode));
    CK(kmeans_sums_reduce_launch(part, pres, pf, np, k, md, pay, colres, D.st));
    CK(cudaStreamSynchronize(D.st));   // pstart / pcl / pfirst live on this stack frame until the copies ran
  }
  CK(kmeans_counts_launch(counts, k, md, pay, D.st));
  return 0;
}

// One device's share of a step: every row of the view assigned to its centre, then the sums
static int km_step_device(agd_handle *h, Dev &D, const KmCentres &c) {
  KmeansArgs a;
  return km_args(h, D, c, a) || km_assign(h, D, a) || km_sums_device(h, D, a, kKmResidual);
}

int agd_kmeans_step(agd_handle *h, const double *centers, int32_t k, double *sums_out, double *counts_out, double *cost_out) {
  KmCentres c;
  if (check_ready(h) || km_centres(h, "agd_kmeans_step", centers, k, c)) return 1;
  if (!counts_out || !cost_out) return fail(h, "NULL argument");
  for (Dev &D : h->devs)
    if (km_step_device(h, D, c)) return 1;
  const size_t P = (size_t)k * c.md + k + 1;
  if (world_reduce(h, [&](size_t i) { return (double *)h->devs[i].km[kKmPayload]; }, P, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> r(P);
  CK(cudaMemcpyAsync(r.data(), D0.km[kKmPayload], P * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  const int32_t du = h->d_user, Dx = du + h->tf_bias;
  for (int32_t j = 0; j < k; ++j) {
    if (sums_out) model_values(h, &r[(size_t)j * c.md], 1.0, sums_out + (size_t)j * Dx);
    counts_out[j] = r[(size_t)k * c.md + j];
  }
  *cost_out = r[P - 1];
  return 0;
}

int agd_kmeans_assign(agd_handle *h, int32_t dev, const double *centers, int32_t k, int64_t row0, int64_t rows,
                      int32_t *cluster_out, double *dist_out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  KmCentres c;
  if (km_centres(h, "agd_kmeans_assign", centers, k, c)) return 1;
  Dev &D = h->devs[dev];
  if (row0 < 0 || rows < 0 || rows > D.sh.rows - row0)
    return fail(h, "row range [%lld, %lld + %lld) lies outside the %lld rows of device %d", (long long)row0, (long long)row0,
                (long long)rows, (long long)D.sh.rows, dev);
  if (rows > 0 && !cluster_out) return fail(h, "NULL argument");
  if (rows == 0) return 0;
  KmeansArgs a;
  if (km_args(h, D, c, a)) return 1;
  // a row's centre depends on the row only, so the range is assigned in chunks through the staging buffer
  const int64_t chunk = rows < (int64_t)(1 << 22) ? rows : (int64_t)(1 << 22);
  if (dist_out && ensure_stage(h, D, (size_t)chunk * sizeof(double))) return 1;
  for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
    a.row0 = row0 + r0;
    a.rows = rows - r0 < chunk ? rows - r0 : chunk;
    if (km_assign(h, D, a)) return 1;
    CK(cudaMemcpyAsync(cluster_out + r0, a.cluster, (size_t)a.rows * sizeof(int32_t), cudaMemcpyDeviceToHost, D.st));
    if (dist_out) {
      int blocks = 0;
      CK(kmeans_dist_launch(a, D.sh.elem_bytes, D.sm_count, (double *)D.stage_dev, nullptr, 0, nullptr, &blocks));
      CK(cudaMemcpyAsync(dist_out + r0, D.stage_dev, (size_t)a.rows * sizeof(double), cudaMemcpyDeviceToHost, D.st));
    }
    CK(cudaStreamSynchronize(D.st));   // the buffers are reused
  }
  return 0;
}

int agd_kmeans_costs(agd_handle *h, const double *centers, int32_t m, int32_t keep, double *sum_out) {
  KmCentres c;
  if (check_ready(h) || km_centres(h, "agd_kmeans_costs", centers, m, c)) return 1;
  if (!sum_out) return fail(h, "NULL argument");
  if (keep != 0 && keep != 1) return fail(h, "agd_kmeans_costs: keep must be 0 or 1 (got %d)", keep);
  if (keep)
    for (const Dev &D : h->devs)
      if (D.km_delta_rows != D.sh.rows)
        return fail(h, "agd_kmeans_costs: keep = 1 needs a previous agd_kmeans_costs on the same rows of device %d", D.ordinal);
  for (Dev &D : h->devs) {
    KmeansArgs a;
    if (km_args(h, D, c, a) || km_assign(h, D, a)) return 1;
    const size_t r1 = D.sh.rows > 0 ? (size_t)D.sh.rows : 1;
    if (D.km_bytes[kKmDelta] < r1 * sizeof(double) && ensure_km(h, D, kKmDelta, r1 * sizeof(double))) return 1;
    if (ensure_km(h, D, kKmPayload, sizeof(double))) return 1;
    const int mb = kmeans_dist_blocks(D.sm_count);
    if (ensure_slabs(h, D, mb, 1)) return 1;
    int blocks = 0;
    CK(kmeans_dist_launch(a, D.sh.elem_bytes, D.sm_count, nullptr, (double *)D.km[kKmDelta], keep, D.slabs, &blocks));
    CK(k1_reduce_launch(D.slabs, blocks, 1, (double *)D.km[kKmPayload], nullptr, D.st));
    D.km_delta_rows = D.sh.rows;
  }
  if (world_reduce(h, [&](size_t i) { return (double *)h->devs[i].km[kKmPayload]; }, 1, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  CK(cudaMemcpyAsync(sum_out, D0.km[kKmPayload], sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  return 0;
}

int agd_kmeans_sample(agd_handle *h, uint64_t seed, double factor, int32_t weighted, int64_t capacity, double *rows_out,
                      double *draws_out, int64_t *n_out) {
  if (check_ready(h)) return 1;
  if (!n_out) return fail(h, "NULL argument");
  if (!(factor >= 0.0) || !std::isfinite(factor)) return fail(h, "agd_kmeans_sample: factor must be finite and >= 0 (got %g)", factor);
  if (weighted != 0 && weighted != 1) return fail(h, "agd_kmeans_sample: weighted must be 0 or 1 (got %d)", weighted);
  if (capacity < 0) return fail(h, "capacity must be >= 0 (got %lld)", (long long)capacity);
  if (capacity > 0 && !rows_out) return fail(h, "NULL argument");
  for (const Dev &D : h->devs) {
    if (D.sh.rows >= (int64_t)1 << 31)
      return fail(h, "agd_kmeans_sample: %lld rows on device %d (at most 2^31 - 1)", (long long)D.sh.rows, D.ordinal);
    if (weighted && D.km_delta_rows != D.sh.rows)
      return fail(h, "agd_kmeans_sample: weighted = 1 needs a previous agd_kmeans_costs on the same rows of device %d", D.ordinal);
  }
  const int W = h->world, nd = (int)h->devs.size();
  const int32_t md = h->d + h->tf_bias, du = h->d_user, Dx = du + h->tf_bias;
  const size_t ld1 = (size_t)md + 1;   // a sampled row and its draw
  std::vector<long long> len((size_t)nd);
  std::vector<KmeansArgs> args((size_t)nd);
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    const Shard &s = D.sh;
    CK(cudaSetDevice(D.ordinal));
    if (h->filt.n && ensure_view_bits(h, D)) return 1;
    const size_t words = (size_t)((s.rows + 31) / 32) + 1, tiles = (size_t)((s.rows + kPjRows - 1) / kPjRows);
    if (ensure_km(h, D, kKmCluster, words * 4) || ensure_km(h, D, kKmMisc, (tiles + 2) * 8 + 16 * ((size_t)W + 1))) return 1;
    KmeansArgs &a = args[(size_t)i];
    if (s.csr) { a.rowptr = s.rowptr; a.idx = s.idx; a.val = s.val; }
    else a.X = s.X;
    a.rows = s.rows; a.d = h->d; a.md = md; a.bias = h->tf_bias; a.scale = h->scale_of(D);
    a.view_bits = h->filt.n ? D.view_bits : nullptr; a.stream = D.st;
    uint32_t *bits = (uint32_t *)D.km[kKmCluster];
    long long *tile_base = (long long *)D.km[kKmMisc], *total = tile_base + tiles;
    long long n = 0;
    if (s.rows > 0) {
      CK(kmeans_sample_bits_launch(a, seed, D.row_base, factor, weighted ? (const double *)D.km[kKmDelta] : nullptr, bits));
      CK(project_scan_launch(bits, s.rows, tile_base, total, D.st));
      CK(cudaMemcpyAsync(&n, total, sizeof n, cudaMemcpyDeviceToHost, D.st));
      CK(cudaStreamSynchronize(D.st));
    }
    len[(size_t)i] = n;
  }
  // every rank's count, then every rank's rows at rank r's block of lmax rows
  std::vector<long long> all(len);
  if (W > 1) {
    auto lens = [&](size_t i) {
      const Dev &D = h->devs[i];
      const size_t tiles = (size_t)((D.sh.rows + kPjRows - 1) / kPjRows);
      return (double *)D.km[kKmMisc] + tiles + 2;
    };
    for (int i = 0; i < nd; ++i) {
      Dev &D = h->devs[i];
      CK(cudaSetDevice(D.ordinal));
      const double v = (double)len[(size_t)i];
      CK(cudaMemcpyAsync(lens(i), &v, sizeof v, cudaMemcpyHostToDevice, D.st));
      CK(cudaStreamSynchronize(D.st));   // v is on this stack frame
    }
    if (world_concat(h, lens, 1, [&](size_t i) { return lens(i) + 1; })) return 1;
    std::vector<double> got((size_t)W);
    Dev &D0 = h->devs[0];
    CK(cudaSetDevice(D0.ordinal));
    CK(cudaMemcpyAsync(got.data(), lens(0) + 1, (size_t)W * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
    if (sync_all(h)) return 1;
    all.assign((size_t)W, 0);
    for (int r = 0; r < W; ++r) all[(size_t)r] = (long long)got[(size_t)r];
  }
  long long total = 0, lmax = 0;
  for (long long n : all) { total += n; lmax = std::max(lmax, n); }
  *n_out = total;
  if (total == 0 || capacity < total) return 0;
  const size_t blk = (size_t)lmax * ld1;
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    CK(cudaSetDevice(D.ordinal));
    if (ensure_km(h, D, kKmRows, (W > 1 ? (size_t)W : 1) * (blk > 0 ? blk : 1) * sizeof(double))) return 1;
    double *out = (double *)D.km[kKmRows] + (W > 1 ? (size_t)(h->first_rank + i) * blk : 0);
    if (len[(size_t)i] > 0)
      CK(kmeans_sample_rows_launch(args[(size_t)i], D.sh.elem_bytes, seed, D.row_base, (const uint32_t *)D.km[kKmCluster],
                                   (const long long *)D.km[kKmMisc], out, D.sm_count));
  }
  auto rows_of = [h](size_t i) { return (double *)h->devs[i].km[kKmRows]; };
  if (W > 1 && world_concat(h, [&](size_t i) { return rows_of(i) + (size_t)(h->first_rank + (int)i) * blk; }, blk, rows_of)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> host((W > 1 ? (size_t)W : 1) * blk);
  CK(cudaMemcpyAsync(host.data(), D0.km[kKmRows], host.size() * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  size_t o = 0;
  for (size_t r = 0; r < all.size(); ++r)
    for (long long q = 0; q < all[r]; ++q, ++o) {
      const double *z = host.data() + r * blk + (size_t)q * ld1;
      model_values(h, z, 1.0, rows_out + o * Dx);
      if (draws_out) draws_out[o] = z[md];
    }
  return 0;
}

// ---------------------------------------------------------------- classification (classify.cu, and the k-means kernels)
int agd_label_classes(agd_handle *h, int64_t capacity, double *labels_out, int64_t *counts_out, int64_t *n_out,
                      int64_t *nan_out) {
  if (check_ready(h)) return 1;
  if (!n_out || !nan_out) return fail(h, "NULL argument");
  if (capacity < 0) return fail(h, "capacity must be >= 0 (got %lld)", (long long)capacity);
  if (capacity > 0 && (!labels_out || !counts_out)) return fail(h, "NULL argument");
  const int nd = (int)h->devs.size();
  std::vector<int64_t> len((size_t)nd), nan((size_t)nd);
  for (int i = 0; i < nd; ++i) {
    Dev &D = h->devs[i];
    const int64_t rows = D.sh.rows;
    CK(cudaSetDevice(D.ordinal));
    if (rows >= (int64_t)1 << 31) return fail(h, "agd_label_classes: %lld rows on device %d (at most 2^31 - 1)", (long long)rows, D.ordinal);
    const size_t r1 = rows > 0 ? (size_t)rows : 1;
    if (ensure_bin(h, D, kBinMisc, kBinMiscAll + 16 * (size_t)h->world + 8 * ((size_t)h->world + 1)) ||
        ensure_bin(h, D, kBinKeys0, 8 * r1) || ensure_bin(h, D, kBinKeys1, 8 * r1) || ensure_bin(h, D, kBinVals0, r1) ||
        ensure_bin(h, D, kBinVals1, r1))
      return 1;
    if (h->filt.n && ensure_view_bits(h, D)) return 1;
    unsigned *counters = (unsigned *)((char *)D.bin[kBinMisc] + kBinMiscCounters);
    CK(cudaMemsetAsync(counters, 0, 2 * sizeof(unsigned), D.st));
    CK(label_keys_launch(D.sh.labels, h->filt.n ? D.view_bits : nullptr, rows, (unsigned long long *)D.bin[kBinKeys0],
                         (uint8_t *)D.bin[kBinVals0], counters, D.st));
    unsigned cnt[2];
    CK(cudaMemcpyAsync(cnt, counters, sizeof cnt, cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));
    nan[(size_t)i] = cnt[1];
    if (bin_list(h, D, cnt[0], &len[(size_t)i])) return 1;
  }
  Dev &D0 = h->devs[0];
  BinRec *list = (BinRec *)D0.bin[kBinList];
  int64_t K = len[0], nans = nan[0];
  if (h->world > 1 && bin_world(h, len, nan, &list, &K, &nans)) return 1;
  CK(cudaSetDevice(D0.ordinal));
  std::vector<BinRec> host;
  if (K > 0 && capacity >= K) {
    host.resize((size_t)K);
    CK(cudaMemcpyAsync(host.data(), list, (size_t)K * sizeof(BinRec), cudaMemcpyDeviceToHost, D0.st));
  }
  if (sync_all(h)) return 1;
  *n_out = K;
  *nan_out = nans;
  for (size_t k = 0; k < host.size(); ++k) {   // tp holds the cumulative count: every key came with the value 1
    labels_out[k] = label_of_key(host[k].key);
    counts_out[k] = host[k].tp - (k > 0 ? host[k - 1].tp : 0);
  }
  return 0;
}

// The C class labels uploaded to D.km[kKmClasses], extra_bytes more behind them
static int cls_upload(agd_handle *h, Dev &D, const double *labels, int32_t C, size_t extra_bytes) {
  if (ensure_km(h, D, kKmClasses, (size_t)C * sizeof(double) + extra_bytes)) return 1;
  CK(cudaMemcpyAsync(D.km[kKmClasses], labels, (size_t)C * sizeof(double), cudaMemcpyHostToDevice, D.st));
  return 0;
}
// C ascending, distinct, non-NaN class labels, at most AGD_MAX_CLASSES
static int cls_check(agd_handle *h, const char *what, const double *labels, int32_t C) {
  if (C < 1 || C > AGD_MAX_CLASSES) return fail(h, "%s: %d classes (1 to %d)", what, C, (int)AGD_MAX_CLASSES);
  if (!labels) return fail(h, "NULL argument");
  for (int32_t c = 0; c < C; ++c) {
    if (labels[c] != labels[c]) return fail(h, "%s: labels[%d] is NaN", what, c);
    if (c > 0 && !(labels[c - 1] < labels[c]))
      return fail(h, "%s: labels must ascend strictly (labels[%d] = %g, labels[%d] = %g)", what, c - 1, labels[c - 1], c, labels[c]);
  }
  return 0;
}

int agd_class_sums(agd_handle *h, const double *labels, int32_t C, double *sums_out, double *counts_out, double *negative_out) {
  if (check_ready(h) || cls_check(h, "agd_class_sums", labels, C)) return 1;
  if (!sums_out || !counts_out || !negative_out) return fail(h, "NULL argument");
  for (const Dev &D : h->devs)
    if (D.sh.rows >= (int64_t)1 << 31)
      return fail(h, "agd_class_sums: %lld rows on device %d (at most 2^31 - 1)", (long long)D.sh.rows, D.ordinal);
  for (Dev &D : h->devs) {
    KmeansArgs a;
    if (km_data(h, D, a) || cls_upload(h, D, labels, C, 0)) return 1;
    const size_t r1 = D.sh.rows > 0 ? (size_t)D.sh.rows : 1;
    if (ensure_km(h, D, kKmCluster, r1 * sizeof(int32_t))) return 1;
    a.k = C;
    a.cluster = (int32_t *)D.km[kKmCluster];
    CK(label_class_launch(D.sh.labels, a.view_bits, D.sh.rows, (const double *)D.km[kKmClasses], C, a.cluster, D.st));
    if (km_sums_device(h, D, a, kKmNegatives)) return 1;
  }
  const int32_t md = h->d + h->tf_bias;
  const size_t P = (size_t)C * md + C + 1;
  if (world_reduce(h, [&](size_t i) { return (double *)h->devs[i].km[kKmPayload]; }, P, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  std::vector<double> r(P);
  CK(cudaMemcpyAsync(r.data(), D0.km[kKmPayload], P * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  const int32_t Dx = h->d_user + h->tf_bias;
  for (int32_t c = 0; c < C; ++c) {
    model_values(h, &r[(size_t)c * md], 1.0, sums_out + (size_t)c * Dx);
    counts_out[c] = r[(size_t)C * md + c];
  }
  *negative_out = r[P - 1];
  return 0;
}

int agd_linear_argmax(agd_handle *h, int32_t dev, const double *W, int32_t C, const double *offset, int64_t row0, int64_t rows,
                      int32_t *class_out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  if (!offset) return fail(h, "NULL argument");
  KmCentres c;
  if (km_centres(h, "agd_linear_argmax", W, C, c, offset)) return 1;
  Dev &D = h->devs[dev];
  if (row0 < 0 || rows < 0 || rows > D.sh.rows - row0)
    return fail(h, "row range [%lld, %lld + %lld) lies outside the %lld rows of device %d", (long long)row0, (long long)row0,
                (long long)rows, (long long)D.sh.rows, dev);
  if (rows > 0 && !class_out) return fail(h, "NULL argument");
  if (rows == 0) return 0;
  KmeansArgs a;
  if (km_args(h, D, c, a)) return 1;
  // a row's class depends on the row only, so the range is scored in chunks
  const int64_t chunk = rows < (int64_t)(1 << 22) ? rows : (int64_t)(1 << 22);
  for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
    a.row0 = row0 + r0;
    a.rows = rows - r0 < chunk ? rows - r0 : chunk;
    if (km_assign(h, D, a, kKmLinear)) return 1;
    CK(cudaMemcpyAsync(class_out + r0, a.cluster, (size_t)a.rows * sizeof(int32_t), cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));   // the buffer is reused
  }
  return 0;
}

int agd_linear_confusion(agd_handle *h, const double *W, int32_t C, const double *offset, const double *labels, int32_t L,
                         double *counts_out) {
  if (check_ready(h) || cls_check(h, "agd_linear_confusion", labels, L)) return 1;
  if (!offset || !counts_out) return fail(h, "NULL argument");
  if (C > AGD_MAX_CLASSES) return fail(h, "agd_linear_confusion: C = %d classes (at most %d)", C, (int)AGD_MAX_CLASSES);
  KmCentres c;
  if (km_centres(h, "agd_linear_confusion", W, C, c, offset)) return 1;
  const size_t n = (size_t)L * C;
  for (Dev &D : h->devs) {
    KmeansArgs a;
    if (km_args(h, D, c, a) || km_assign(h, D, a, kKmLinear)) return 1;
    const size_t lb = ((size_t)L * sizeof(double) + 15) / 16 * 16;
    if (cls_upload(h, D, labels, L, lb - (size_t)L * sizeof(double) + n * 8) ||
        ensure_km(h, D, kKmPayload, n * sizeof(double)))
      return 1;
    unsigned long long *cnt = (unsigned long long *)((char *)D.km[kKmClasses] + lb);
    CK(cudaMemsetAsync(cnt, 0, n * 8, D.st));
    CK(label_confusion_launch(D.sh.labels, a.cluster, D.sh.rows, (const double *)D.km[kKmClasses], L, C, cnt, D.sm_count, D.st));
    // the counts as doubles: kmeans_counts_launch with k = L C and md = 0 writes out[j] = counts[j]
    CK(kmeans_counts_launch(cnt, (int32_t)n, 0, (double *)D.km[kKmPayload], D.st));
  }
  if (world_reduce(h, [&](size_t i) { return (double *)h->devs[i].km[kKmPayload]; }, n, kXchgSum)) return 1;
  Dev &D0 = h->devs[0];
  CK(cudaSetDevice(D0.ordinal));
  CK(cudaMemcpyAsync(counts_out, D0.km[kKmPayload], n * sizeof(double), cudaMemcpyDeviceToHost, D0.st));
  if (sync_all(h)) return 1;
  return 0;
}

// ---------------------------------------------------------------- views (row filters)
int agd_set_row_filter(agd_handle *h, int32_t n, const uint64_t *seeds, const double *lo, const double *hi,
                       const int32_t *complement) {
  if (!h) return 1;
  if (n < 0 || n > kMaxRowPredicates) return fail(h, "a row filter holds 0 to %d predicates (got %d)", kMaxRowPredicates, n);
  if (n > 0 && (!seeds || !lo || !hi || !complement)) return fail(h, "NULL argument");
  RowFilter f;
  f.n = n;
  for (int i = 0; i < n; ++i) {
    if (!(lo[i] >= 0.0 && lo[i] <= hi[i] && hi[i] <= 1.0))   // also refuses NaN
      return fail(h, "predicate %d: bounds must satisfy 0 <= lo <= hi <= 1 (lo=%.17g, hi=%.17g)", i, lo[i], hi[i]);
    if (complement[i] != 0 && complement[i] != 1) return fail(h, "predicate %d: complement must be 0 or 1 (got %d)", i, complement[i]);
    // b = floor(c 2^64): exact for c < 1 (ldexp is exact and the result is below 2^64); c = 1 is "to the end"
    f.seed[i] = seeds[i];
    f.lo[i] = lo[i] < 1.0 ? (unsigned long long)std::ldexp(lo[i], 64) : 0ull;
    f.hi[i] = hi[i] < 1.0 ? (unsigned long long)std::ldexp(hi[i], 64) : 0ull;
    f.flags[i] = (complement[i] ? kRowPredComplement : 0u) | (lo[i] < 1.0 ? 0u : kRowPredLoEnd) | (hi[i] < 1.0 ? 0u : kRowPredHiEnd);
  }
  // Until every device holds the new filter the handle runs without one: a failure part-way leaves no device on a filter the
  // handle does not describe (the call then fails and the handle has no filter).
  h->filt = RowFilter();
  auto upload = [&]() -> int {
    for (Dev &D : h->devs) {   // stream-ordered after every sweep that still reads the previous filter
      CK(cudaSetDevice(D.ordinal));
      if (!D.filt_dev) CK(cudaMalloc(&D.filt_dev, sizeof(RowFilter)));
      CK(cudaMemcpyAsync(D.filt_dev, &f, sizeof(RowFilter), cudaMemcpyHostToDevice, D.st));
      CK(cudaStreamSynchronize(D.st));
    }
    return 0;
  };
  if (upload()) return 1;
  h->filt = f;
  return 0;
}

int agd_row_filter_mask(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, uint8_t *out) {
  if (!h) return 1;
  if (dev < 0 || dev >= (int)h->devs.size()) return fail(h, "bad local device index %d", dev);
  Dev &D = h->devs[dev];
  if (row0 < 0 || rows < 0 || rows > D.sh.rows - row0)
    return fail(h, "row range [%lld, %lld + %lld) lies outside the %lld rows of device %d", (long long)row0, (long long)row0,
                (long long)rows, (long long)D.sh.rows, dev);
  if (rows > 0 && !out) return fail(h, "NULL argument");
  if (rows == 0) return 0;
  CK(cudaSetDevice(D.ordinal));
  const int64_t chunk = rows < (int64_t)(1 << 24) ? rows : (int64_t)(1 << 24);
  if (ensure_stage(h, D, (size_t)chunk)) return 1;
  for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
    const int64_t m = rows - r0 < chunk ? rows - r0 : chunk;
    CK(row_filter_mask_launch(h->filt_of(D), D.row_base + row0 + r0, m, (uint8_t *)D.stage_dev, D.st));
    CK(cudaMemcpyAsync(out + r0, D.stage_dev, (size_t)m, cudaMemcpyDeviceToHost, D.st));
    CK(cudaStreamSynchronize(D.st));   // the staging buffer is reused
  }
  return 0;
}

// ---------------------------------------------------------------- feature transforms (scaling, intercept)
int agd_set_feature_transform(agd_handle *h, const double *scale, int32_t append_bias) {
  if (!h) return 1;
  if (append_bias != 0 && append_bias != 1) return fail(h, "append_bias must be 0 or 1 (got %d)", append_bias);
  // Until every device holds the new transform the handle runs without one: a failure part-way leaves none installed.
  h->tf_scale = false;
  h->tf_bias = 0;
  if (!scale && !append_bias) return 0;
  if (h->d <= 0) return fail(h, "no shard loaded: a feature transform is sized by the feature dimension");
  std::vector<double> s((size_t)h->d, 0.0);   // zero on the padded columns
  if (scale)
    for (int32_t j = 0; j < h->d_user; ++j) {
      if (!std::isfinite(scale[j])) return fail(h, "scale[%d] = %g is not finite", j, scale[j]);
      s[(size_t)j] = scale[j];
    }
  const int32_t cap = h->d + 5;   // model_d() + 4 with an intercept
  for (Dev &D : h->devs) {   // stream-ordered after every sweep that still reads the previous transform
    CK(cudaSetDevice(D.ordinal));
    if (D.tf_cap < cap) {
      CK(cudaStreamSynchronize(D.st));
      double **bufs[] = {&D.tf_scale, &D.weff, &D.weff2};
      for (double **b : bufs) {
        if (*b) cudaFree(*b);
        *b = nullptr;
      }
      D.tf_cap = 0;
      for (double **b : bufs) CK(cudaMalloc(b, (size_t)cap * sizeof(double)));
      D.tf_cap = cap;
    }
    if (scale) CK(cudaMemcpyAsync(D.tf_scale, s.data(), s.size() * sizeof(double), cudaMemcpyHostToDevice, D.st));
    CK(cudaStreamSynchronize(D.st));
  }
  h->tf_scale_host.assign(s.begin(), s.begin() + h->d_user);
  h->tf_scale = scale != nullptr;
  h->tf_bias = append_bias;
  return 0;
}

// ---------------------------------------------------------------- applyProjector with host buffers
int agd_prox(agd_handle *h, int32_t updater, const double *w, const double *g, double step, double reg,
             int32_t d, double *w_out, double *reg_val) {
  if (!h) return 1;
  if (updater < 0 || updater > AGD_UPD_L1) return fail(h, "unknown updater %d", updater);
  if (d <= 0) return fail(h, "bad dimension");
  Dev &D = h->devs[0];
  CK(cudaSetDevice(D.ordinal));
  double *buf = nullptr, *partials = nullptr;
  CK(cudaMalloc(&buf, 3 * (size_t)d * sizeof(double)));
  CK(cudaMalloc(&partials, (size_t)k3_blocks(d) * K3_NS * sizeof(double)));
  CK(cudaMemcpyAsync(buf, w, (size_t)d * sizeof(double), cudaMemcpyHostToDevice, D.st));
  CK(cudaMemcpyAsync(buf + d, g, (size_t)d * sizeof(double), cudaMemcpyHostToDevice, D.st));
  K3ProxArgs a;
  a.w = buf; a.g = buf + d; a.w_out = buf + 2 * (size_t)d; a.partials = partials; a.ticket = D.ticket;
  a.scalars = D.scalars_dev; a.step = step; a.reg = reg; a.acc_tail = nullptr; a.d = d; a.updater = updater;
  CK(k3_prox_launch(a, D.st));
  CK(cudaMemcpyAsync(w_out, buf + 2 * (size_t)d, (size_t)d * sizeof(double), cudaMemcpyDeviceToHost, D.st));
  double sc[K3_NS];
  if (read_scalars(h, sc)) return 1;
  if (reg_val) *reg_val = reg_value(updater, reg, sc[2], sc[5]);
  cudaFree(buf);
  cudaFree(partials);
  return 0;
}

// ---------------------------------------------------------------- AcceleratedGradientDescent.run
int agd_run(agd_handle *h, const agd_params *p, const double *w0, double *w_out, double *loss_hist,
            int32_t *n_hist, agd_stats *stats) {
  if (check_ready(h)) return 1;
  if (!p || !w0 || !w_out || !loss_hist || !n_hist) return fail(h, "NULL argument");
  if (p->gradient < 0 || p->gradient > AGD_GRAD_LEAST_SQUARES_HALF) return fail(h, "unknown gradient %d", p->gradient);
  if (p->updater < 0 || p->updater > AGD_UPD_L1) return fail(h, "unknown updater %d", p->updater);
  const auto t_begin = std::chrono::steady_clock::now();
  const int32_t d = h->model_d();
  const double INF = std::numeric_limits<double>::infinity();
  agd_stats s;
  memset(&s, 0, sizeof s);
  if (call_begin(h)) return 1;
  const bool memoize = (p->flags & AGD_FLAG_MEMOIZE_FX) != 0;
  // Pass fusion: the history evaluation applySmooth(x) (:304) of iteration k and applySmooth(y) (:250) of iteration k+1
  // (first backtracking round) do not depend on each other, so ONE sweep over X evaluates both.
  const bool fuse = (p->flags & AGD_FLAG_NO_FUSE) == 0 && dual_supported(h);
  bool y_ready = false;   // acc already holds applySmooth(y) for the first round of the coming iteration
  // Speculative sweep of the memoised pass structure: applySmooth(x) of the backtracking test (:269) and applySmooth(y) of the
  // NEXT iteration (:250) -- y_{k+1} = x_k (1 - theta') + z_k theta' with theta' from L alpha, i.e. assuming the test accepts and
  // the gradient test does not restart -- are evaluated by ONE two-gradient sweep over X.  An accepted iteration then reads X
  // once.  Every evaluation is the arithmetic a sweep of its own would do (same kernel code path), so weights and history
  // stay bit-identical; a rejected guess only wastes the extra FMAs.  On a restart y_{k+1} = x_k exactly, and the memoised
  // (f_x, g_x) are reused without any evaluation at all.
  const bool reuse_fx = memoize && (p->flags & AGD_FLAG_NO_FUSE) == 0 && p->beta < 1.0;   // restart: applySmooth(y_{k+1}) = (f_x, g_x)
  const bool speculate_y = reuse_fx && dual_full_supported(h);
  size_t acc_off = 0;     // where applySmooth(y) of the current round lives inside Dev::acc (0, or d + 4 after a good guess)

  for (Dev &D : h->devs) {                                                 // :224-225  x = w0 ; z = x
    CK(cudaSetDevice(D.ordinal));
    if (put_point(h, D, D.x, w0)) return 1;  // padded columns carry zero weights throughout
    CK(k3_copy2_launch(D.z, D.x, nullptr, nullptr, d, D.st));
  }
  h->launches += 1;
  double theta = INF;                                                      // :226
  int nh = 0;                                                              // :227
  double f_y = 0.0;                                                        // :229
  double L = p->L0;                                                        // :232
  bool backtrack_simple = true;                                            // :234
  const double backtrack_tol = 1e-10;                                      // :235
  const double Lexact = p->Lexact, beta = p->beta;
  double sc[K3_NS] = {0}, sg[K3_NS] = {0};
  unsigned long long &round_seq = h->seq_base;  // every round of every call gets a fresh sequence number

  auto launch_all = [&](auto fn) -> int {
    for (Dev &D : h->devs) {
      CK(cudaSetDevice(D.ordinal));
      CK(fn(D));
    }
    trace_mark(h, "k3");
    h->launches += 1;
    return 0;
  };
  trace_mark(h, "start");

  // Host round trips: the host needs device scalars once per backtracking round.  Pass 2 (applySmooth(x), :269) is
  // enqueued speculatively right behind pass 1 -- it is wasted only when ||x - y||^2 == 0 (:265) -- and the f_x of the
  // history pass (:304) is copied to pinned memory asynchronously and read after the loop, so the GPU runs
  // pass 3(k) -> pass 1(k+1) -> pass 2(k+1) back to back with a single synchronisation per round.
  Dev &H0 = h->devs[0];
  if (H0.hist_cap < 2 * (size_t)(p->num_iterations > 0 ? p->num_iterations : 1)) {
    CK(cudaSetDevice(H0.ordinal));
    if (H0.hist_host) cudaFreeHost(H0.hist_host);
    H0.hist_cap = 2 * (size_t)(p->num_iterations > 0 ? p->num_iterations : 1);
    CK(cudaHostAlloc(&H0.hist_host, H0.hist_cap * sizeof(double), cudaHostAllocMapped | cudaHostAllocPortable));
    CK(cudaHostGetDevicePointer((void **)&H0.hist_dev, H0.hist_host, 0));
  }
  long long pending_hist = -1;        // slot of H0.hist_host the next k3_step fills from the fused sweep it consumes
  std::vector<double> cx_of;          // c_x per iteration (:305)
  std::vector<char> fx_deferred;      // f_x of iteration k still sits in H0.hist_host[2k..2k+1]
  for (int nIter = 1; nIter <= p->num_iterations; ++nIter) {              // :237
    const double L_old = L;                                                // :242
    L = L * p->alpha;                                                      // :243
    const double theta_old = theta;                                        // :244
    bool nonterminating = false, have_fx = false, first_round = true;
    bool guess_live = false;     // acc[d+4 ..] holds applySmooth at y_spec, sharing its sweep with this round's applySmooth(x)
    double guess_theta = 0.0;
    double f_x = 0.0;
    for (;;) {                                                             // :246
      theta = 2.0 / (1.0 + std::sqrt(1.0 + 4.0 * (L / L_old) / (theta_old * theta_old)));  // :248
      const double omt = 1.0 - theta;
      if (first_round) {  // (x_old, z_old) = (x, z) :241 fused with y = x_old*(1-theta) + z_old*theta :249
        if (!y_ready && launch_all([&](Dev &D) { return k3_begin_launch(D.x_old, D.z_old, D.y, D.x, D.z, omt, theta, d, D.st); })) return 1;
        first_round = false;
      } else if (launch_all([&](Dev &D) { return k3_combine_launch(D.y, D.x_old, omt, D.z_old, theta, d, D.st); })) return 1;  // :249
      if (!y_ready) {
        if (smooth_device(h, p->gradient, [](Dev &D) { return (const double *)D.y; }, true, nullptr, false, true)) return 1;  // :250
        acc_off = 0;
      }
      y_ready = false;
      s.passes++;
      const double step = 1.0 / (theta * L);                               // :253
      const bool speculate = beta < 1.0;                                   // :257 is known up front
      // this round's applySmooth(x) sweep also carries a guess of y_{k+1} (formed inside k3_step from the new x and z)
      const bool guessed = speculate && speculate_y && nIter < p->num_iterations;
      double theta_guess = 0.0;
      if (guessed) {
        const double L_n = L * p->alpha;                                   // :243-248 of iteration nIter + 1 if this round accepts
        theta_guess = 2.0 / (1.0 + std::sqrt(1.0 + 4.0 * (L_n / L) / (theta * theta)));
      }
      if (launch_all([&](Dev &D) {                                         // :254-255,263-264 fused
            K3StepArgs a;
            a.y_spec = guessed ? D.y_spec : nullptr; a.spec_ca = 1.0 - theta_guess; a.spec_cb = theta_guess;
            a.acc = D.acc + acc_off; a.x_old = D.x_old; a.z_old = D.z_old; a.y = D.y; a.g_y = D.g_y; a.z = D.z; a.x = D.x;
            a.partials = D.partials; a.ticket = D.ticket; a.scalars = D.scalars_dev;
            a.theta = theta; a.one_minus_theta = omt; a.step = step; a.reg = p->reg_param; a.d = d; a.updater = p->updater;
            if (!speculate) { a.seq_out = reinterpret_cast<unsigned long long *>(D.scalars_dev + 2 * K3_NS); a.seq = round_seq + 1; }
            a.xg = gatherer(h, D, h->pending); a.acc_w = D.acc;   // the K3 kernel gathers the sweep it consumes
            a.hist_out = (pending_hist >= 0 && &D == &h->devs[0]) ? D.hist_dev + pending_hist : nullptr;
            return k3_step_launch(a, D.st);
          })) return 1;
      h->pending = Epoch();
      pending_hist = -1;
      if (speculate) {                                                     // :269, enqueued before :265 is known
        if (guessed) {
          if (smooth_device(h, p->gradient, [](Dev &D) { return (const double *)D.x; }, true,
                            [](Dev &D) { return (const double *)D.y_spec; }, true, true))
            return 1;
        } else if (smooth_device(h, p->gradient, [](Dev &D) { return (const double *)D.x; }, true, nullptr, false, true)) return 1;
        if (launch_all([&](Dev &D) {
              K3GxArgs a;
              a.acc = D.acc; a.x = D.x; a.y = D.y; a.g_y = D.g_y; a.g_x = D.g_x; a.partials = D.partials;
              a.ticket = D.ticket; a.scalars = D.scalars_dev + K3_NS; a.d = d;
              a.seq_out = reinterpret_cast<unsigned long long *>(D.scalars_dev + 2 * K3_NS); a.seq = round_seq + 1;
              a.xg = gatherer(h, D, h->pending); a.acc_w = D.acc;
              return k3_gx_launch(a, D.st);
            })) return 1;
        h->pending = Epoch();
      }
      if (wait_scalars(h, ++round_seq, sc)) return 1;                      // the one host wait of this round (no stream drain)
      trace_mark(h, "host-gap");
      memcpy(sg, H0.scalars_host + K3_NS, K3_NS * sizeof(double));
      f_y = sc[6] / sc[7];                                                 // :207
      have_fx = false;
      if (beta >= 1.0) break;                                              // :257
      const double nxy = std::sqrt(sc[0]);
      const double xy_sq = nxy * nxy;                                      // :264  math.pow(norm(xy), 2)
      if (xy_sq == 0) { s.wasted_passes++; guess_live = false; break; }    // :265  (the speculative pass is discarded)
      s.passes++;
      f_x = sg[6] / sg[7];
      have_fx = true;
      guess_live = guessed;                                                // valid only if this round is the accepted one
      guess_theta = theta_guess;
      double localL;
      if (backtrack_simple) {                                              // :272
        const double q_x = f_y + sc[1] + 0.5 * L * xy_sq;                  // :273
        localL = L + 2.0 * jmax(f_x - q_x, 0.0) / xy_sq;                   // :274
        backtrack_simple = (std::fabs(f_y - f_x) >= backtrack_tol * jmax(std::fabs(f_x), std::fabs(f_y)));  // :275
      } else {
        localL = 2.0 * sg[0] / xy_sq;                                      // :278
      }
      if (localL <= L || L >= Lexact) break;                               // :281
      if (!std::isinf(localL)) L = jmin(Lexact, localL);                   // :285-287
      else localL = L;                                                     // :288-290
      L = jmin(Lexact, jmax(localL, L / beta));                            // :292
      s.backtracks++;
      if (guess_live) { s.wasted_passes++; guess_live = false; }   // rejected: y_{k+1} was guessed from an L that did not survive
      if (L != L) { nonterminating = true; break; }  // the reference never leaves :246-293 once L is NaN
    }
    const double c_x = reg_value(p->updater, p->reg_param, sc[2], sc[5]);  // :305  applyProjector(x, g_x, 0.0)._1
    cx_of.push_back(c_x);
    s.iterations = nIter;
    // The exits of :309-324 and the restart of :327-331 depend on nothing the history evaluation (:304) produces, so they
    // are decided first: when another iteration follows, that evaluation shares its sweep with the next applySmooth(y).
    bool stop = false;
    if (nonterminating) { s.stopped_nan = 1; s.nonterminating = 1; stop = true; }
    else if (std::isnan(f_y) || std::isinf(f_y)) { s.stopped_nan = 1; stop = true; }  // :309-312
    else {
      const double norm_x = std::sqrt(sc[2]);                              // :315
      const double norm_dx = std::sqrt(sc[3]);                             // :316
      if (norm_dx == 0.0 && nIter > 1) { s.converged = 1; stop = true; }   // :317-321
      else if (norm_dx < p->convergence_tol * jmax(norm_x, 1)) { s.converged = 1; stop = true; }  // :322-324
    }
    const bool restart = !stop && p->may_restart && sc[4] > 0.0;           // :327
    const bool need_hist = !(memoize && have_fx);
    const bool fuse_now = need_hist && fuse && !stop && nIter < p->num_iterations;
    if (need_hist && !fuse_now) {                                          // :304  (f_x, g_x) = applySmooth(x)
      if (smooth_device(h, p->gradient, [](Dev &D) { return (const double *)D.x; }, true)) return 1;
      s.passes++;
      CK(cudaSetDevice(H0.ordinal));
      CK(cudaMemcpyAsync(H0.hist_host + 2 * (size_t)nh, H0.acc + d, 2 * sizeof(double), cudaMemcpyDeviceToHost, H0.st));
      fx_deferred.push_back(1);                                            // read after the loop
      loss_hist[nh++] = 0.0;
    } else if (!need_hist) {
      fx_deferred.push_back(0);
      loss_hist[nh++] = f_x + c_x;                                         // :306
    }
    if (restart) {
      if (launch_all([&](Dev &D) { return k3_copy2_launch(D.z, D.x, nullptr, nullptr, d, D.st); })) return 1;  // :328
      theta = INF;                                                         // :329
      backtrack_simple = true;                                             // :330
      s.restarts++;
    }
    if (reuse_fx && have_fx && !stop && nIter < p->num_iterations && (guess_live || restart)) {
      // The coming iteration's first round is already evaluated.  (x_old, z_old) = (x, z) and y (:241,:249) are formed as the
      // loop head would form them -- the same kernel, the same doubles -- and pass 1 is skipped (y_ready):
      //   * no restart: y_{k+1} is the guess; its sums are the second block of acc;
      //   * restart: theta' = 1, so y_{k+1} = x_k * 0 + z * 1 with z = x_k (:328) = x_k exactly; applySmooth(x_k) is the first block.
      const double L_n = L * p->alpha;
      const double theta_n = 2.0 / (1.0 + std::sqrt(1.0 + 4.0 * (L_n / L) / (theta * theta)));
      if (restart || theta_n == guess_theta) {
        const double omt_n = 1.0 - theta_n;
        if (launch_all([&](Dev &D) { return k3_begin_launch(D.x_old, D.z_old, D.y, D.x, D.z, omt_n, theta_n, d, D.st); })) return 1;
        acc_off = restart ? 0 : (size_t)d + 4;
        if (restart && guess_live) s.wasted_passes++;
        if (!restart) s.fused_passes++;      // pass 1 of iteration nIter + 1 shared its sweep with pass 2 of this one
        y_ready = true;
      } else if (guess_live) s.wasted_passes++;
    } else if (guess_live) s.wasted_passes++;
    if (fuse_now) {
      // :243-249 of iteration nIter + 1, first round (the loop head recomputes the same doubles), then one sweep:
      // acc[0..d+1] = applySmooth(y) sums, acc[d+2..d+3] = loss sum / count at x
      const double L_n = L * p->alpha;
      const double theta_n = 2.0 / (1.0 + std::sqrt(1.0 + 4.0 * (L_n / L) / (theta * theta)));
      const double omt_n = 1.0 - theta_n;
      if (launch_all([&](Dev &D) { return k3_begin_launch(D.x_old, D.z_old, D.y, D.x, D.z, omt_n, theta_n, d, D.st); })) return 1;
      if (smooth_device(h, p->gradient, [](Dev &D) { return (const double *)D.y; }, true,
                        [](Dev &D) { return (const double *)D.x; }, false, true))
        return 1;
      s.passes++;          // the history evaluation; the applySmooth(y) half is counted by the next iteration
      s.fused_passes++;
      y_ready = true;
      pending_hist = 2 * (long long)nh;   // the k3_step that consumes this sweep stores {loss sum, count} at x into the history slot
      fx_deferred.push_back(1);
      loss_hist[nh++] = 0.0;
    }
    if (stop) break;
  }
  {
    Dev &D = h->devs[0];
    CK(cudaSetDevice(D.ordinal));
    if (get_point(h, D, w_out, D.x)) return 1;                             // :337
  }
  if (h->pending.e || pending_hist >= 0) return fail(h, "internal: a sweep was left without its consumer");
  if (call_end(h, s, t_begin)) return 1;
  trace_report(h, memoize ? "agd_run memoised" : (fuse ? "agd_run" : "agd_run unfused"));
  for (int k = 0; k < nh; ++k)                                             // :306 for the deferred f_x values
    if (fx_deferred[(size_t)k]) loss_hist[k] = H0.hist_host[2 * (size_t)k] / H0.hist_host[2 * (size_t)k + 1] + cx_of[(size_t)k];
  *n_hist = nh;
  s.final_L = L;
  s.final_theta = theta;
  if (stats) *stats = s;
  return 0;
}

// ---------------------------------------------------------------- GradientDescent.runMiniBatchSGD (fraction 1.0)
int agd_gd_run(agd_handle *h, int32_t gradient, int32_t updater, double step_size, int32_t num_iterations,
               double reg_param, const double *w0, double *w_out, double *loss_hist, int32_t *n_hist,
               agd_stats *stats) {
  return agd_gd_run_minibatch(h, gradient, updater, step_size, num_iterations, reg_param, 1.0, w0, w_out, loss_hist,
                              n_hist, stats);
}

int agd_gd_run_minibatch(agd_handle *h, int32_t gradient, int32_t updater, double step_size, int32_t num_iterations,
                         double reg_param, double mini_batch_fraction, const double *w0, double *w_out,
                         double *loss_hist, int32_t *n_hist, agd_stats *stats) {
  if (check_ready(h)) return 1;
  if (!(mini_batch_fraction > 0.0)) return fail(h, "miniBatchFraction must be positive");
  if (gradient < 0 || gradient > AGD_GRAD_LEAST_SQUARES_HALF) return fail(h, "unknown gradient %d", gradient);
  if (updater < 0 || updater > AGD_UPD_L1) return fail(h, "unknown updater %d", updater);
  const auto t_begin = std::chrono::steady_clock::now();
  const int32_t d = h->model_d();
  const size_t vb = (size_t)d * sizeof(double);
  agd_stats s;
  memset(&s, 0, sizeof s);
  if (call_begin(h)) return 1;
  double sc[K3_NS];
  int64_t total_rows_local = 0;
  for (Dev &D : h->devs) total_rows_local += D.sh.rows;
  auto prox_all = [&](const double *acc_tail_sel, double step, bool from_acc) -> int {
    for (Dev &D : h->devs) {
      CK(cudaSetDevice(D.ordinal));
      K3ProxArgs a;
      a.w = D.x; a.g = from_acc ? D.acc : D.g_x; a.w_out = D.z; a.partials = D.partials; a.ticket = D.ticket;
      a.scalars = D.scalars_dev; a.step = step; a.reg = reg_param; a.acc_tail = from_acc ? D.acc + d : nullptr;
      a.d = d; a.updater = updater;
      CK(k3_prox_launch(a, D.st));
      CK(k3_copy2_launch(D.x, D.z, nullptr, nullptr, d, D.st));
    }
    (void)acc_tail_sel;
    h->launches += 2;
    return 0;
  };
  for (Dev &D : h->devs) {
    CK(cudaSetDevice(D.ordinal));
    if (put_point(h, D, D.x, w0)) return 1;  // padded columns carry zero weights throughout
    CK(cudaMemsetAsync(D.g_x, 0, vb, D.st));
  }
  // regVal = updater.compute(weights, zeros, 0, 1, regParam)._2
  if (prox_all(nullptr, 0.0, false)) return 1;
  if (read_scalars(h, sc)) return 1;
  double reg_val = reg_value(updater, reg_param, sc[2], sc[5]);
  int nh = 0;
  for (int i = 1; i <= num_iterations; ++i) {
    // data.sample(false, miniBatchFraction, 42 + i): Bernoulli row mask keyed by the iteration
    h->sample_seed = 42ull + (unsigned long long)i;
    h->sample_thresh = mini_batch_fraction >= 1.0 ? 0ull : (unsigned long long)std::ldexp(mini_batch_fraction, 64);
    const int rc_smooth = smooth_device(h, gradient, [](Dev &D) { return (const double *)D.x; }, true);
    h->sample_thresh = 0ull;
    if (rc_smooth) return 1;
    s.passes++;
    const double this_step = step_size / std::sqrt((double)i);
    if (prox_all(nullptr, this_step, true)) return 1;
    if (read_scalars(h, sc)) return 1;
    if (!(sc[7] > 0)) continue;  // miniBatchSize == 0: the reference logs a warning and skips the update
    loss_hist[nh++] = sc[6] / sc[7] + reg_val;
    reg_val = reg_value(updater, reg_param, sc[2], sc[5]);
    s.iterations = i;
  }
  {
    Dev &D = h->devs[0];
    CK(cudaSetDevice(D.ordinal));
    if (get_point(h, D, w_out, D.x)) return 1;
  }
  if (call_end(h, s, t_begin)) return 1;
  *n_hist = nh;
  if (stats) *stats = s;
  return 0;
}

}  // extern "C"
