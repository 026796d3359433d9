// agd_common.cuh -- shared declarations of the sm_90a hot-path kernels (internal, not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/agd_b200.h"

namespace agd {

// ---------------------------------------------------------------- views of the resident shards (agd_set_row_filter)
// A conjunction of up to kMaxRowPredicates predicates on the row's own 64-bit draw u(seed, grow) (row_in_view(),
// k1_device.cuh).  Predicate i holds iff lo_i <= u < hi_i, negated under kRowPredComplement; a bound of exactly 2^64 (c = 1)
// is carried as a flag, since it does not fit the integer.  The kernels read it from device memory through a pointer in their
// arguments; a null pointer means every row, and they test that first, uniformly.
constexpr int kMaxRowPredicates = 4;
enum { kRowPredComplement = 1, kRowPredLoEnd = 2, kRowPredHiEnd = 4 };
struct RowFilter {
  int32_t n = 0;
  uint32_t flags[kMaxRowPredicates] = {};
  unsigned long long seed[kMaxRowPredicates] = {}, lo[kMaxRowPredicates] = {}, hi[kMaxRowPredicates] = {};
};

// ---------------------------------------------------------------- K1: fused row-block gradient
// Replaces the seqOp fold of AGD.scala:197-200 + Gradient.compute [mllib-1.3.0] over one shard.
struct K1Args {
  const void *X;          // shard, row-major, ld == d, element type float or double
  const double *labels;   // rows (+ padding)
  const double *w;        // d doubles (device)
  const double *w2;       // optional second point of a fused sweep (AGD.scala:304 riding along with :250): loss only ...
  int32_t dual_full;      // ... unless dual_full: loss AND gradient at w2 (second slab block of d + 4 doubles; ring kernel, fp32/fp64)
  double *slabs;          // [grid][d + 4]: per-block column sums of loss' * x, the loss sum, the row count at w; loss sum, count at w2
  int64_t rows;           // rows in the shard
  int32_t d;
  int32_t kind;           // AGD_GRAD_*
  int32_t stages;         // smem ring depth
  int32_t slab_stride;    // d + 4
  unsigned long long sample_seed, sample_thresh;  // Bernoulli row mask (thresh 0 = every row), see row_selected()
  long long row_base;     // global index of the shard's first row
  const RowFilter *filt;  // the view a collective call runs on (device copy; nullptr: every row), see row_in_view()
  const uint32_t *view_bits;  // with filt: bit r % 32 of word r / 32 = row_in_view() of local row r, drawn when the filter
                              // was set (the ring and wgmma kernels read these: no Philox between their barriers)
  int32_t tune_rows;      // 0 = default; rows per tile of the headline ring shape (4|8)
  int32_t tune_ctas;      // 0 = default; resident CTAs per SM (1|2|3)
  int32_t tune_full;      // 0 = default; 1 = keep the column predicates even when every thread owns whole vectors
  int32_t tc_margins_f64; // wgmma kernel: 1 = fp64-exact margins on the CUDA cores (option tc_margins=f64), 0 = fp32 (default)
};

// launch helpers (k1_dense.cu); return the number of blocks that wrote a slab.
// bias = 1: the model has an intercept, w[d] (and w2[d]), and every payload block is [grad (d) | sum of the multipliers | loss |
// count | loss2 | count2], D + 4 doubles with D = d + 1 (slab_stride and the slabs sized for it).  It is an argument of the
// launch, not a field of K1Args: the kernels without an intercept keep the parent's parameter block, registers and bits.
int k1_ring_supported(int32_t d, int elem_bytes);
int k1_ring_dual_supported(int32_t d, int elem_bytes);
cudaError_t k1_ring_launch(const K1Args &a, int bias, int elem_bytes, int sm_count, int *blocks_out, cudaStream_t st);
int k1_ring_dual_full_supported(int32_t d, int elem_bytes);
cudaError_t k1_generic_launch(const K1Args &a, int bias, int elem_bytes, int sm_count, int max_blocks, int *blocks_out,
                              cudaStream_t st);
int k1_max_blocks(int sm_count);
// bf16 shards: margins on CUDA cores, X^T r on wgmma (k1_tc.cu); d % 128 == 0, d <= 4096
int k1_tc_supported(int32_t d, int elem_bytes);
cudaError_t k1_tc_launch(const K1Args &a, int bias, int sm_count, int *blocks_out, cudaStream_t st);
// ---------------------------------------------------------------- K2': one-shot all-reduce over NVLink peer memory
// Every rank owns an exchange buffer xbuf[2][W][n] (+ flags[2][W]) that all peers can store into (P2P / CUDA IPC).
// publish: rank r stores its n = d+4 partial sums into slot r of EVERY rank's buffer, fences, then raises the flag
// (epoch) -- fused into the tail of k1_reduce_kernel, or standalone for the CSR path.  gather: each rank waits for the
// W flags of the epoch and adds the W slots in rank order, so every rank gets the same bits (replaces combOp +
// treeAggregate + broadcast, AGD.scala:193-204, without a library call in the loop).  Buffers alternate by epoch parity.
constexpr int kMaxRanks = 16;
struct XchgPeers {
  double *slot[kMaxRanks];               // base of rank p's xbuf as mapped into THIS device
  unsigned long long *flag[kMaxRanks];   // base of rank p's flags
};
// The publish half of one epoch on one rank, in the one-shot or the reduce-scatter form (below).
struct XchgPub {
  XchgPeers peers;
  int world, my_rank, buf, n;
  int slot_stride;          // doubles between two ranks' slots: xchg_slot_stride(d) (kXchgBulk in the bulk area), the capacity, NOT this
                            // sweep's n: sweeps of different payloads -- d + 4, 2 (d + 4) or AGD_EVAL_N -- must not move the
                            // slots of the other parity buffer
  unsigned long long epoch;
  unsigned int *ticket;
};
// The gather half of the exchange, for kernels that consume the all-reduced sums right away (K3): instead of a launch of its own,
// the consumer waits for the W flags, adds the W slots in rank order where it needs a value, and writes every one of the n sums
// to `acc` for later readers.  world == 0: nothing pending, read `acc` as usual.
struct XchgGather {
  const double *xbuf = nullptr;               // this device's [2][W][slot_stride] slots (one-shot or bulk area) or its result area (rs)
  const unsigned long long *flags = nullptr;  // [2][W] of the flag set to wait on
  int world = 0, buf = 0, n = 0, slot_stride = 0;
  int rs = 0;                                 // 1: reduce-scatter form -- the finished sums sit at xbuf[buf * slot_stride + j]
  unsigned long long epoch = 0;
};
// ---- large payloads (n >= kXchgRsMin doubles, e.g. d = 10^6): reduce-scatter + all-gather over the same peer memory.
// Rank r stores slice p of its partial sums into rank p's `rs` area (slot r), rank p adds the W slots of ITS slice in rank order
// and stores the finished slice into every rank's `res` area; 2 n / W doubles leave each rank per sweep instead of n W.
// Layout of one device's exchange allocation (doubles): [one-shot: 2 W S][rs: 2 W L][res: 2 S], S = xchg_slot_stride(d) (below), L = ceil(S / W);
// flags (u64): [one-shot 2 W][rs arrived 2 W][res arrived 2 W].  The helpers below are the only place this layout is written.
constexpr int kXchgRsMin = 32768;
__host__ __device__ inline size_t xchg_rs_slice(int S, int W) { return ((size_t)S + W - 1) / W; }
__host__ __device__ inline size_t xchg_off_rs(int S, int W) { return 2 * (size_t)W * S; }
__host__ __device__ inline size_t xchg_off_res(int S, int W) { return xchg_off_rs(S, W) + 2 * (size_t)W * xchg_rs_slice(S, W); }
__host__ __device__ inline size_t xchg_total_doubles(int S, int W) { return xchg_off_res(S, W) + 2 * (size_t)S; }
__host__ __device__ inline int xchg_flags_oneshot(int) { return 0; }         // raised by a one-shot (or bulk) publish
__host__ __device__ inline int xchg_flags_rs(int W) { return 2 * W; }        // a rank's slices arrived in the rs area
__host__ __device__ inline int xchg_flags_res(int W) { return 4 * W; }       // a finished slice arrived in the res area
// Bulk area behind the areas above, [2][W][kXchgBulk] doubles, for payloads that do not fit a slot (agd_binary_curve's lists):
// the same publish kernel and flags with the peers' bases moved to xchg_off_bulk and a slot stride of kXchgBulk, one epoch per
// chunk of at most kXchgBulk doubles.  It only extends the one allocation each rank exports, so no offset of the areas above
// and no handle format changes.
constexpr int kXchgBulk = 65536;
__host__ __device__ inline size_t xchg_off_bulk(int S, int W) { return xchg_total_doubles(S, W); }
__host__ __device__ inline size_t xchg_alloc_doubles(int S, int W) { return xchg_off_bulk(S, W) + 2 * (size_t)W * kXchgBulk; }
// The reduction the gather kernels apply to the W slots, in rank order: a sum, or a NaN-ignoring max (column maxima; a minimum
// travels as the max of -x).  Either way every rank gets identical bits.  kXchgCopy is the concatenation of the W slots: no
// arithmetic touches the payload, so bit-cast keys and counts travel unchanged.
enum { kXchgSum = 0, kXchgMax = 1, kXchgCopy = 2 };
cudaError_t xchg_publish_launch(const double *acc, const XchgPub &pub, cudaStream_t st);
cudaError_t xchg_rs_publish_launch(const double *acc, const XchgPub &x, cudaStream_t st);
cudaError_t xchg_rs_reduce_bcast_launch(const double *xbuf_local, const unsigned long long *flags_local, const XchgPub &x, cudaStream_t st,
                                        int op);
// The stand-alone gather (K3 kernels inline it): waits for the W flags of g's epoch, then
//   op == kXchgCopy: out[r * out_stride + c] = slot r [c], c < n;
//   g.rs:            out[c] = the finished sum c;
//   otherwise:       out[c] = the W slots reduced by op in rank order.
cudaError_t xchg_gather_launch(const XchgGather &g, double *out, size_t out_stride, int op, cudaStream_t st);

// out[c] = sum_b slabs[b][c] for c < n, n = D + 4 or 2 (D + 4) (gradient sums, loss sum, row count, loss sum and count at w2; fixed order =>
// deterministic);
// with pub != nullptr the sums are also stored into every peer's exchange slot and the epoch flag is raised;
// with scale != nullptr column c % blk < scale_d is multiplied by scale[c % blk] first (feature scaling, blk = D + 4)
cudaError_t k1_reduce_launch(const double *slabs, int blocks, int32_t n, double *out, const XchgPub *pub, cudaStream_t st,
                             const double *scale = nullptr, int32_t scale_d = 0, int32_t blk = 1);
// Feature scaling around K1 (agd_set_feature_transform).  out[c] = s[c] w[c] for c < d, w[c] for d <= c < n (the intercept);
// the same from w2 into out2 unless out2 is null
cudaError_t transform_point_launch(double *out, const double *w, double *out2, const double *w2, const double *s, int32_t d,
                                   int32_t n, cudaStream_t st);
// acc[c] *= s[c], c < d (the CSR gradient, which K1 sums straight into acc)
cudaError_t scale_columns_launch(double *acc, const double *s, int32_t d, cudaStream_t st);

// CSR variant (k1_csr.cu)
struct K1CsrArgs {
  const int64_t *rowptr;
  const int32_t *idx;
  const void *val;        // float or double
  const double *labels;
  const double *w;
  const double *w2;       // optional second point (loss only), as in K1Args
  double *gacc;           // d + 4 doubles (d + 5 with bias), zeroed by the launch: gradient sum, loss sum, count; loss sum, count at w2
  int64_t rows;
  int32_t d;
  int32_t kind;
  unsigned long long sample_seed, sample_thresh;
  long long row_base;
  const RowFilter *filt;  // as in K1Args
  int32_t tune;           // option ring_rows: 1 = the simple (unpipelined) loop
};
cudaError_t k1_csr_launch(const K1CsrArgs &a, int bias, int elem_bytes, int sm_count, cudaStream_t st);

// Slot stride of the peer-memory exchange (doubles per rank's slot): the largest payload any sweep on a handle of this
// dimension publishes -- 2 (d + 5) for a two-gradient sweep with an intercept, AGD_EVAL_N for an evaluation.  ONE stride per
// handle, whether or not a transform is installed: sweeps of different payloads must not move the slots of the other parity
// buffer, and the host-shipped (ipc) exchange is built once per dimension.
inline int xchg_slot_stride(int32_t d) { return 2 * (d + 5) > AGD_EVAL_N ? 2 * (d + 5) : AGD_EVAL_N; }

// ---------------------------------------------------------------- scoring sweeps (score.cu)
// Margins m_i = x_i . w + b of rows [row0, row0 + rows) of one shard, or the AGD_EVAL_* sums over them (one slab of
// AGD_EVAL_N doubles per CTA, added in fixed order by k1_reduce_launch).  Dense (rowptr == nullptr) or CSR.
struct ScoreArgs {
  const void *X = nullptr;          // dense shard, row-major, ld == d (fp32 / fp64 / bf16)
  const int64_t *rowptr = nullptr;  // CSR shard (fp32 / fp64 values)
  const int32_t *idx = nullptr;
  const void *val = nullptr;
  const double *labels = nullptr;
  const double *w = nullptr;        // d doubles (device), zero on padded columns
  double b = 0.0;                   // intercept
  int64_t row0 = 0, rows = 0;
  int32_t d = 0;                    // stored row length (the handle's internal dimension)
  int32_t kind = 0;                 // AGD_GRAD_* (evaluation)
  // The key form's outputs share the words of fields it does not use, so the kernels' parameter block keeps its size (and the
  // margins and evaluation forms their register allocation).
  union {
    double threshold = 0.0;         // evaluation: confusion-count threshold
    unsigned int *counters;         // key form: [0] = keys written, [1] = NaN margins (zeroed by the caller)
  };
  union {
    double *margins = nullptr;      // margins form: rows doubles
    unsigned long long *keys;       // key form: margin_key of the kept rows' non-NaN margins, compacted, ...
  };
  union {
    double *slabs = nullptr;        // evaluation form: [score_max_blocks][AGD_EVAL_N]
    uint8_t *classes;               // key form: ... and their classes (1: label > 0.5)
  };
  long long row_base = 0;           // evaluation and key forms: global index of the shard's first row ...
  const RowFilter *filt = nullptr;  // ... and the view whose rows are summed (rows outside it are not even read)
  cudaStream_t stream = nullptr;
};
int score_max_blocks(int sm_count);
cudaError_t score_margins_launch(const ScoreArgs &a, int elem_bytes, int sm_count);
// *blocks_out = slabs written (0 for an empty range)
cudaError_t score_eval_launch(const ScoreArgs &a, int elem_bytes, int sm_count, int *blocks_out);
cudaError_t score_keys_launch(const ScoreArgs &a, int elem_bytes, int sm_count);

// ---------------------------------------------------------------- ranking metrics (rank.cu, agd_binary_curve)
// The descending-order key of a non-NaN margin: the fp64 bits (-0 taken as +0) mapped to an unsigned integer whose ascending
// order is the DESCENDING order of the margins (so a key sort puts the highest score first).  margin_of_key inverts it.
__host__ __device__ inline unsigned long long margin_key(double m) {
  if (m == 0.0) m = 0.0;
  unsigned long long u;
  memcpy(&u, &m, sizeof u);
  const unsigned long long asc = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
  return ~asc;
}
__host__ __device__ inline double margin_of_key(unsigned long long k) {
  const unsigned long long asc = ~k;
  const unsigned long long u = (asc >> 63) ? (asc & 0x7fffffffffffffffull) : ~asc;
  double m;
  memcpy(&m, &u, sizeof m);
  return m;
}
// One point of the curve: a distinct key and the cumulative counts of positives / negatives down to it (inclusive).
struct BinRec {
  unsigned long long key;
  long long tp, fp;
};
// Stable LSD radix sort of (key, value) pairs, 8-bit digits, value 1 byte (a class) or 4 bytes (an index).  keys[0] / vals[0]
// hold the input; *which = the buffer pair holding the result.  One histogram of all eight digits decides the passes first:
// a pass whose digit is the same in every key is skipped.  hist: 8 x 256 counters; tiles: bin_sort_tile_words(n) words.
// Synchronises the stream once (the histogram decides the passes on the host).
size_t bin_sort_tile_words(long long n);
cudaError_t bin_sort_pairs(unsigned long long *keys[2], void *vals[2], int val_bytes, long long n, unsigned *hist,
                           unsigned *tiles, int *which, int *passes, cudaStream_t st);
// Run-length reduce of sorted pairs into the curve: out[r] = {key, cumulative positives, cumulative negatives} of the r-th
// distinct key, *n_out = distinct keys.  val_bytes 1: vals are classes; 4: vals index (pos, neg) in upos / uneg.
// tile_sums: bin_runs_tile_words(n) long longs.
size_t bin_runs_tile_words(long long n);
cudaError_t bin_runs_launch(const unsigned long long *keys, const void *vals, int val_bytes, const long long *upos,
                            const long long *uneg, long long n, long long *tile_sums, BinRec *out, long long *n_out,
                            cudaStream_t st);
// The world's lists (rank r's records off[r + 1] - off[r] of them, at blocks + r * stride) concatenated in rank order: key,
// index, and each record's own counts (the difference of consecutive cumulative counts within its list).  off: world + 1
// offsets in device memory.
cudaError_t bin_union_prep_launch(const BinRec *blocks, long long stride, const long long *off, int world, long long total,
                                  unsigned long long *keys, uint32_t *idx, long long *upos, long long *uneg, cudaStream_t st);
// Trapezoid areas under ROC and PR of the K-point curve (K >= 1): out[0] = AUROC, out[1] = AUPR, summed in a fixed order
// (per block in index order, then the blocks in order).  partials: bin_area_blocks(K) x 2 doubles.
int bin_area_blocks(long long K);
cudaError_t bin_areas_launch(const BinRec *recs, long long K, double *partials, double *out, cudaStream_t st);
// ---------------------------------------------------------------- column statistics (colstats.cu, agd_col_stats)
// Pass 1 sums, per device and after the exchange: [SUM d | SQ d | ABS d | NNZ d | COUNT 1 | STORED d] (col_sum_n(d) doubles);
// maxima [MAX d | -MIN d]; pass 2 sums [DEV d | DEV2 d].  STORED is the stored-entry count of a CSR column (= COUNT on
// dense shards), so the host adds the implicit zeros of a column, COUNT - STORED of them, in closed form.
inline size_t col_sum_n(int32_t d) { return 5 * (size_t)d + 1; }
struct ColStatsArgs {
  const void *X = nullptr;          // dense shard (fp32 / fp64 / bf16), row-major, ld == d
  const int64_t *rowptr = nullptr;  // CSR shard (fp32 / fp64 values)
  const int32_t *idx = nullptr;
  const void *val = nullptr;
  int64_t rows = 0;
  int32_t d = 0;
  long long row_base = 0;           // global index of the shard's first row ...
  const RowFilter *filt = nullptr;  // ... and the view whose rows are summarised (rows outside it are not read)
  const double *mu_sums = nullptr;  // dense pass 2: the world's pass-1 sums; mu = fl(SUM / COUNT) on the device
  const double *mu = nullptr;       // CSR pass 2: d values of mu (colstats_mu_launch)
  double *slabs = nullptr;          // dense: [blocks][4 d + 1] (pass 1) or [blocks][2 d] (pass 2) ...
  double *max_slabs = nullptr;      // ... and [blocks][2 d] maxima (pass 1)
  double *out = nullptr;            // CSR: pass-1 sums (zeroed) or pass-2 sums (zeroed), scattered with RED.ADD
  unsigned long long *keys = nullptr;   // CSR pass 1: [2 d] order-preserving images of MAX / -MIN (zeroed = none)
  cudaStream_t stream = nullptr;
};
// slabs a dense sweep writes at most (its slab memory is bounded for wide rows)
int colstats_max_blocks(int sm_count, int32_t d);
cudaError_t colstats_dense_launch(const ColStatsArgs &a, int pass, int elem_bytes, int sm_count, int *blocks_out);
cudaError_t colstats_csr_launch(const ColStatsArgs &a, int pass, int elem_bytes, int sm_count);
cudaError_t colstats_unkey_launch(const unsigned long long *keys, int n, double *out, cudaStream_t st);
cudaError_t colstats_fill_stored_launch(double *sums, int32_t d, cudaStream_t st);
cudaError_t colstats_mu_launch(const double *sums, int32_t d, double *mu, cudaStream_t st);
// out[c] = NaN-ignoring max over the slabs of column c < n, fixed order
cudaError_t colstats_max_reduce_launch(const double *slabs, int blocks, int32_t n, double *out, cudaStream_t st);

// ---------------------------------------------------------------- cross-products (gramian.cu, agd_gramian)
// The packed upper triangle of the augmented (d + 1) x (d + 1) matrix [sum z z^T, sum z; sum z^T, count], entry (i, j), i <= j,
// at i (d + 1) - i (i - 1) / 2 + (j - i): gramian_packed_n(d) doubles.
struct GramianArgs {
  const void *X = nullptr;          // dense shard (fp32 / fp64 / bf16), row-major, ld == d
  const int64_t *rowptr = nullptr;  // CSR shard (fp32 / fp64 values)
  const int32_t *idx = nullptr;
  const void *val = nullptr;
  int64_t rows = 0;
  int32_t d = 0;
  long long row_base = 0;           // CSR: global index of the shard's first row ...
  const RowFilter *filt = nullptr;  // ... and the view (rows outside it are not read)
  const uint32_t *view_bits = nullptr;   // dense: the view as a bitmap of the shard's rows (nullptr: every row)
  const double *mu = nullptr;       // dense: d values subtracted from every kept element (nullptr: uncentered)
  double *slabs = nullptr;          // dense: [splits][gramian_packed_n(d)], every entry written
  double *out = nullptr;            // CSR: gramian_packed_n(d) doubles (zeroed), scattered with RED.ADD
  cudaStream_t stream = nullptr;
};
size_t gramian_packed_n(int32_t d);
// row splits of a dense sweep (slabs it writes)
int gramian_splits(int sm_count, int32_t d, int64_t rows);
cudaError_t gramian_dense_launch(const GramianArgs &a, int elem_bytes, int sm_count, int splits);
cudaError_t gramian_csr_launch(const GramianArgs &a, int elem_bytes, int sm_count);
// out = the centered packed sums derived from the uncentered ones u (the same rows) and the world's mu
cudaError_t gramian_center_launch(const double *u, const double *mu, int32_t d, double *out, cudaStream_t st);

// ---------------------------------------------------------------- projection (project.cu, agd_project)
// Y = X B + c over the rows of a view, compacted in physical order into another handle's dense shard.  B is [bd][kp] doubles,
// bd = d rounded up to 16 and kp = k rounded up to project_tile_cols(k), zero-padded; c is kp doubles, zero beyond k.
constexpr int kPjRows = 128;        // rows of X per dense CTA, and the rows per entry of tile_base
struct ProjectArgs {
  const void *X = nullptr;          // dense source (fp32 / fp64 / bf16), row-major, ld == d
  const int64_t *rowptr = nullptr;  // CSR source (fp32 / fp64 values)
  const int32_t *idx = nullptr;
  const void *val = nullptr;
  const double *labels = nullptr;
  int64_t rows = 0;
  int32_t d = 0;                    // the source's stored row length
  const uint32_t *view_bits = nullptr;   // the view as a bitmap of the shard's rows (nullptr: every row) ...
  const long long *tile_base = nullptr;  // ... and the kept rows before each tile of kPjRows rows (project_scan_launch)
  const double *B = nullptr;
  const double *c = nullptr;
  int32_t k = 0, kp = 0;
  void *Y = nullptr;                // destination rows, ld == ldy (k, padded as a load pads it), storage out_bytes
  double *Ylabels = nullptr;
  int32_t ldy = 0, out_bytes = 8;
  cudaStream_t stream = nullptr;
};
int project_tile_cols(int32_t k);
cudaError_t project_scan_launch(const uint32_t *bits, int64_t rows, long long *tile_base, long long *total, cudaStream_t st);
cudaError_t project_dense_launch(const ProjectArgs &a, int elem_bytes);
cudaError_t project_csr_launch(const ProjectArgs &a, int elem_bytes, int sm_count);

// ---------------------------------------------------------------- k-means (kmeans.cu, agd_kmeans_*)
// Rows [row0, row0 + rows) of one shard in the feature space z = appendBias(s o x) of md = d + bias columns, against k centres.
// A row's centre is the lowest index j minimising the score ||c_j||^2 - 2 (x . B_j + cb_j) with B_lj = s_l c_jl: the cross term
// is the projection's fp64 sum (pj_tile.cuh, or a CSR row's stored entries in stored order); a NaN score never wins.
constexpr int kKmPiece = 4096;      // sorted rows per piece of the dense sums
// Compile-time modes of the k-means kernels.  Score: kKmDistance is k-means' own; kKmLinear scores class j as
// -(offset_j + x . B_j + cb_j) with the offset in the cn slot, so the lowest (score, j) is the linear model's argmax (agd_linear_*).
// Sums: kKmResidual adds the residuals to the centres; kKmNegatives counts the entries that are not >= 0 (agd_class_sums).
enum { kKmDistance = 0, kKmLinear = 1 };
enum { kKmResidual = 0, kKmNegatives = 1 };
struct KmeansArgs {
  const void *X = nullptr;          // dense shard (fp32 / fp64 / bf16), row-major, ld == d
  const int64_t *rowptr = nullptr;  // CSR shard (fp32 / fp64 values)
  const int32_t *idx = nullptr;
  const void *val = nullptr;
  long long row0 = 0, rows = 0;
  int32_t d = 0;                    // stored row length
  int32_t md = 0;                   // d + bias: columns of C
  int32_t bias = 0;                 // 1: z_d = 1.0
  const double *scale = nullptr;    // d factors s (nullptr: s = 1)
  const uint32_t *view_bits = nullptr;   // the view as a bitmap of the shard's rows (nullptr: every row)
  int32_t k = 0, kp = 0;            // centres, and k rounded up to whole column tiles (project_tile_cols)
  const double *B = nullptr;        // [round_up(d, 16)][kp], zero-padded
  const double *cb = nullptr;       // kp: each centre's bias entry (0 without one)
  const double *cn = nullptr;       // kp: ||c_j||^2
  const double *C = nullptr;        // [k][md]: the centres
  int32_t *cluster = nullptr;       // rows: the row's centre, -1 outside the view
  double *tile_score = nullptr;     // [kp / 128][rows] and ...
  int32_t *tile_idx = nullptr;      // ... the best of each 128-column tile, when kp > 128
  cudaStream_t stream = nullptr;
};
cudaError_t kmeans_assign_launch(const KmeansArgs &a, int elem_bytes, int sm_count, int score_mode = kKmDistance);
// Exact residual sum_l (z_l - c_l)^2 of each row of the range to its cluster's centre (CSR: ||c||^2 + sum over the stored
// entries of (z_l - c_l)^2 - c_l^2, the bias column counted as stored).  dist != nullptr: dist[i] (NaN outside the view).
// Else delta[i] = the residual, or with keep the smaller of it and delta[i] (a NaN residual never replaces delta[i]), and the
// view's sum of delta per block into slabs (*blocks_out of them, added in order by k1_reduce_launch).
int kmeans_dist_blocks(int sm_count);
cudaError_t kmeans_dist_launch(const KmeansArgs &a, int elem_bytes, int sm_count, double *dist, double *delta, int keep,
                               double *slabs, int *blocks_out);
// keys[i] = cluster[i] (k outside the view), vals[i] = i, counts[keys[i]] += 1 (counts: k + 1 zeroed words)
cudaError_t kmeans_keys_launch(const int32_t *cluster, long long rows, int32_t k, unsigned long long *keys, uint32_t *vals,
                               unsigned long long *counts, cudaStream_t st);
// Dense sums over pieces of the rows sorted by cluster: piece p is sorted positions [pstart[p], pstart[p + 1]) of cluster
// pcl[p]; part[p][c] = sum z_c, pres[p][c] = sum (z_c - C[pcl[p]][c])^2 (kKmNegatives: the count of z_c not >= 0), each a
// sequential fp64 sum in sorted order.
cudaError_t kmeans_sums_dense_launch(const KmeansArgs &a, int elem_bytes, const uint32_t *order, const long long *pstart,
                                     const int32_t *pcl, long long npieces, double *part, double *pres,
                                     int sums_mode = kKmResidual);
// out[j][c] = the pieces pfirst[j] .. pfirst[j + 1] - 1 of part added in order; out[k md + k] = the cost, pres added over the
// pieces in order per column, then over the columns in order
cudaError_t kmeans_sums_reduce_launch(const double *part, const double *pres, const int32_t *pfirst, long long npieces,
                                      int32_t k, int32_t md, double *out, double *colres, cudaStream_t st);
// CSR: out[j][c] += z_c and out[k md + k] += the row's residual (kKmNegatives: its stored z_c not >= 0), by fp64 RED.ADD (out
// zeroed by the caller)
cudaError_t kmeans_sums_csr_launch(const KmeansArgs &a, int elem_bytes, int sm_count, double *out, int sums_mode = kKmResidual);
// out[k md + j] = counts[j], j < k
cudaError_t kmeans_counts_launch(const unsigned long long *counts, int32_t k, int32_t md, double *out, cudaStream_t st);
// k-means sampling: row r of the view is kept iff u < factor delta[r] (delta = 1 when delta == nullptr), u = the row's draw of
// stream kKmStream under seed as a double in [0, 1) (the top 53 bits); bit r % 32 of bits[r / 32]
constexpr uint32_t kKmStream = 8;
cudaError_t kmeans_sample_bits_launch(const KmeansArgs &a, unsigned long long seed, long long row_base, double factor,
                                      const double *delta, uint32_t *bits);
// the kept rows, compacted through tile_base (project_scan_launch of bits): out[o] = [z (md doubles) | u]
cudaError_t kmeans_sample_rows_launch(const KmeansArgs &a, int elem_bytes, unsigned long long seed, long long row_base,
                                      const uint32_t *bits, const long long *tile_base, double *out, int sm_count);

// ---------------------------------------------------------------- classification (classify.cu, agd_label_classes / agd_class_sums /
// agd_linear_confusion).  Labels are compared by value (-0.0 == 0.0); `classes` are C ascending non-NaN doubles.
// The label key of a row: ascending in the label, -0.0 keyed as 0.0 (label_of_key inverts it, giving +0.0)
__host__ __device__ inline unsigned long long label_key(double y) { return margin_key(-y); }
__host__ __device__ inline double label_of_key(unsigned long long k) { return 0.0 - margin_of_key(k); }
// For every row of [0, rows) in the view (view_bits, nullptr: every row): a non-NaN label appends (label_key, 1) to keys / ones
// (compacted, counters[0] = their number); a NaN label adds 1 to counters[1].  counters zeroed by the caller.
cudaError_t label_keys_launch(const double *labels, const uint32_t *view_bits, long long rows, unsigned long long *keys,
                              uint8_t *ones, unsigned *counters, cudaStream_t st);
// cls[i] = the index of labels[i] in classes, -1 for a label that is none of them (NaN included) or a row outside the view
cudaError_t label_class_launch(const double *labels, const uint32_t *view_bits, long long rows, const double *classes,
                               int32_t C, int32_t *cls, cudaStream_t st);
// counts[l][c] += the rows with labels[i] == classes[l] and pred[i] == c >= 0 (counts: L x C zeroed u64; C <= 12,288)
cudaError_t label_confusion_launch(const double *labels, const int32_t *pred, long long rows, const double *classes, int32_t L,
                                   int32_t C, unsigned long long *counts, int sm_count, cudaStream_t st);

// out[i] = 1 if row row_base + i passes the filter, else 0 (agd_row_filter_mask; the kernels' own row_in_view())
cudaError_t row_filter_mask_launch(const RowFilter *f, long long row_base, int64_t rows, uint8_t *out, cudaStream_t st);
// the same predicate as a bitmap: bit i % 32 of bits[i / 32] for rows [0, rows) (ceil(rows / 32) words)
cudaError_t row_filter_bits_launch(const RowFilter *f, long long row_base, int64_t rows, uint32_t *bits, cudaStream_t st);


// ---------------------------------------------------------------- K3: fused O(d) driver-side vector work
// Replaces the breeze d-vector ops of AGD.scala:249,255,263-264,273,278,315-316,327, the
// normalisation of :207 and Updater.compute [mllib-1.3.0] behind applyProjector (:214-222).
enum { K3_NS = 8 };  // scalars produced per call
struct K3StepArgs {
  const double *acc;      // packed [grad_sum(d) | loss_sum | count] after the all-reduce
  const double *x_old, *z_old, *y;
  double *g_y, *z, *x;
  double *partials;       // [blocks][K3_NS]
  unsigned int *ticket;
  double *scalars;        // [K3_NS]: S(x-y)^2, (x-y).g_y, S x^2, S (x-x_old)^2, g_y.(x-x_old), S|x|, loss_sum, count
  double theta, one_minus_theta, step, reg;
  int32_t d, updater;
  double *y_spec;         // optional: y_spec = x * spec_ca + z * spec_cb, the guessed y of the next iteration (speculative sweep)
  double spec_ca, spec_cb;
  unsigned long long *seq_out = nullptr;   // optional: launch sequence number stored behind the scalars (host polls it)
  unsigned long long seq = 0;
  XchgGather xg;          // pending exchange whose sums this kernel gathers itself (then `acc` is written, not only read)
  double *acc_w = nullptr;
  double *hist_out = nullptr;   // optional (mapped host memory): {loss sum, count} at the second point of the sweep just consumed (AGD.scala:304)
};
cudaError_t k3_step_launch(const K3StepArgs &a, cudaStream_t st);
struct K3GxArgs {
  const double *acc;
  const double *x, *y, *g_y;
  double *g_x;
  double *partials;
  unsigned int *ticket;
  double *scalars;        // [0] = (x-y).(g_x-g_y), [6] = loss_sum, [7] = count
  int32_t d;
  unsigned long long *seq_out = nullptr;
  unsigned long long seq = 0;
  XchgGather xg;          // as in K3StepArgs
  double *acc_w = nullptr;
};
cudaError_t k3_gx_launch(const K3GxArgs &a, cudaStream_t st);
// out = a*ca + b*cb (separate roundings, as breeze does at AGD.scala:249)
cudaError_t k3_combine_launch(double *out, const double *a, double ca, const double *b, double cb, int32_t d,
                              cudaStream_t st);
// x_old = x ; z_old = z ; y = x*ca + z*cb  (AGD.scala:241 + :249 in one launch)
cudaError_t k3_begin_launch(double *x_old, double *z_old, double *y, const double *x, const double *z, double ca,
                            double cb, int32_t d, cudaStream_t st);
// dst0 = src0 ; dst1 = src1 (either pair may be null)
cudaError_t k3_copy2_launch(double *dst0, const double *src0, double *dst1, const double *src1, int32_t d,
                            cudaStream_t st);
// plain prox for agd_prox / the GD comparator: w_out = Updater.compute(w, g[/count], step, reg); scalars[2]=S w'^2, [5]=S|w'|
struct K3ProxArgs {
  const double *w, *g;
  double *w_out;
  double *partials;
  unsigned int *ticket;
  double *scalars;
  double step, reg;
  const double *acc_tail;   // optional {loss_sum, count} on the device: g is divided by count first
                            // (count == 0 leaves w unchanged); scalars[6..7] receive the pair
  int32_t d, updater;
};
cudaError_t k3_prox_launch(const K3ProxArgs &a, cudaStream_t st);
int k3_blocks(int32_t d);

// ---------------------------------------------------------------- K0: synthetic workload (harness)
cudaError_t synth_dense_launch(void *X, int elem_bytes, uint64_t seed, int64_t row0, int64_t rows, int32_t d, int32_t ld,
                               cudaStream_t st);
cudaError_t synth_wtrue_launch(double *w, uint64_t seed, int32_t d, cudaStream_t st);
cudaError_t synth_labels_launch(const void *X, int elem_bytes, const double *w_true, double *labels, uint64_t seed,
                                int kind, int64_t row0, int64_t rows, int32_t d, int32_t ld, cudaStream_t st);

cudaError_t synth_csr_launch(int64_t *rowptr, int32_t *idx, void *val, int elem_bytes, const double *w_true,
                             double *labels, uint64_t seed, int kind, int64_t row0, int64_t rows, int32_t d, int32_t k,
                             cudaStream_t st);

// dst[i] = src[i] + shift (rebasing an appended partition's rowptr onto the resident CSR shard)
cudaError_t csr_shift_rowptr_launch(int64_t *dst, const int64_t *src, int64_t n, int64_t shift, cudaStream_t st);

// rowptr (as the caller passed it: rows + 1 entries from 0) and idx of an appended CSR partition, checked on the device:
// *flag = 0 ok, 1 = rowptr not monotone / not ending at nnz, 2 = a column id outside [0, d)
cudaError_t csr_validate_launch(const int64_t *rowptr_host_order, int64_t rows, const int32_t *idx, int64_t nnz, int32_t d,
                                int *flag, cudaStream_t st);

// records `msg` as the handle's agd_last_error (for translation units other than agd_api.cu)
void set_last_error(agd_handle *h, const char *msg);

// ---------------------------------------------------------------- load path
// dst (store dtype, rows x dst_ld, columns >= d zero) <- src (src dtype, leading dimension ld), rows x d
cudaError_t convert_rows_launch(void *dst, int dst_bytes, const void *src, int src_bytes, int64_t rows, int32_t d,
                                int64_t ld, int32_t dst_ld, cudaStream_t st);

}  // namespace agd
