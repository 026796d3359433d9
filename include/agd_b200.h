/*
 * agd_b200.h -- C-ABI of the H100-native accelerated-gradient-descent hot path.
 *
 * This is the drop-in boundary a JVM binding (JNI) for staple/spark-agd would bind: plain
 * pointers and sizes, no C++/torch types.  Reference paths are relative to /root/reference:
 *   AGD.scala   = src/main/scala/org/apache/spark/mllib/optimization/AcceleratedGradientDescent.scala
 *   Suite.scala = src/test/scala/org/apache/spark/mllib/optimization/AcceleratedGradientDescentSuite.scala
 *
 * Model: one agd_handle per process owns one or more local H100s.  Each GPU pins one row-shard of
 * the (n x d) design matrix in HBM (the analogue of `dataRDD.cache()`, Suite.scala:51).  A "pass" is
 * one applySmooth (AGD.scala:192-208): fused row-block gradient kernel over the shard, one
 * all-reduce of the packed [grad(d) | loss | count] fp64 buffer, and the fused O(d) update kernel.
 * All entry points return 0 on success, nonzero on error (see agd_last_error).  There is no CPU
 * fallback anywhere: without a usable sm_90 GPU every compute entry point fails.
 *
 * Threading: agd_reserve / agd_load_* may be called concurrently for DIFFERENT local devices (Spark
 * task threads); everything else is single-caller, like the driver thread of AGD.scala:177.
 * Ownership: the caller owns every host buffer; the library owns device memory until agd_destroy.
 */
#ifndef AGD_B200_H
#define AGD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AGD_B200_ABI_VERSION 2

typedef struct agd_handle agd_handle;

/* Closed enum of the Gradient plug-ins the reference can be given (AGD.scala:41,198):
 * LogisticGradient (binary), LeastSquaresGradient, HingeGradient of spark-mllib 1.3.0.
 * AGD_GRAD_LEAST_SQUARES_HALF is the Spark >= 1.4 definition (loss diff^2/2, gradient diff*x). */
enum { AGD_GRAD_LOGISTIC = 0, AGD_GRAD_LEAST_SQUARES = 1, AGD_GRAD_HINGE = 2, AGD_GRAD_LEAST_SQUARES_HALF = 3 };
/* Closed enum of the Updater plug-ins (AGD.scala:41,215): SimpleUpdater, SquaredL2Updater, L1Updater. */
enum { AGD_UPD_SIMPLE = 0, AGD_UPD_SQUARED_L2 = 1, AGD_UPD_L1 = 2 };
/* Element types: host source type and HBM storage type of the design matrix. */
enum { AGD_F64 = 0, AGD_F32 = 1, AGD_BF16 = 2 };
/* agd_params.flags */
enum {
  AGD_FLAG_MEMOIZE_FX = 1, /* reuse (f_x, g_x) of AGD.scala:269 for the history pass at :304 when x is
                              unchanged (bit-identical result, 3 -> 2 passes per iteration).  Where the shard's kernel has a
                              two-gradient form, applySmooth(x) then shares its sweep with applySmooth(y) of the NEXT
                              iteration (y guessed from "accepted, no restart"; a wrong guess is discarded, a restart reuses
                              (f_x, g_x) because then y = x): an accepted iteration reads X once. */
  AGD_FLAG_NO_FUSE = 2,    /* by default the history evaluation applySmooth(x) of AGD.scala:304 rides along with
                              applySmooth(y) of the NEXT iteration (AGD.scala:250) in one sweep over the shards: the same
                              evaluations and the same results bit for bit (dense shards), one read of X fewer per iteration.
                              This flag runs every evaluation as a sweep of its own. */
};

/* The constructor arguments + eight hyper-parameters of AGD.scala:41-51 (defaults: agd_default_params). */
typedef struct {
  double convergence_tol; /* AGD.scala:44  default 1e-4 */
  int32_t num_iterations; /* AGD.scala:45  default 100  */
  double reg_param;       /* AGD.scala:46  default 0.0  */
  double L0;              /* AGD.scala:47  default 1.0  */
  double Lexact;          /* AGD.scala:48  default +inf */
  double beta;            /* AGD.scala:49  default 0.5  */
  double alpha;           /* AGD.scala:50  default 0.9  */
  int32_t may_restart;    /* AGD.scala:51  default 1    */
  int32_t gradient;       /* AGD_GRAD_*  (the `gradient` delegate, AGD.scala:41) */
  int32_t updater;        /* AGD_UPD_*   (the `updater` delegate,  AGD.scala:41) */
  int32_t flags;          /* AGD_FLAG_*; 0 reproduces the reference's pass structure exactly */
} agd_params;

/* What `run` learned; the reference only logs (AGD.scala:310,334). */
typedef struct {
  int32_t iterations;     /* = length of the loss history */
  int32_t passes;         /* applySmooth evaluations executed */
  int32_t backtracks;     /* times AGD.scala:292 raised L */
  int32_t restarts;       /* times AGD.scala:327-331 fired */
  int32_t converged;      /* left through AGD.scala:319 or :323 */
  int32_t stopped_nan;    /* left through AGD.scala:309-312 */
  int32_t nonterminating; /* L became NaN: the reference would spin forever in :246-293; we stop */
  int32_t collective_kind; /* 0 = none / NCCL all-reduce, 1 = one-shot exchange over NVLink peer memory */
  double final_L;
  double final_theta;
  double seconds_total;   /* host wall time inside agd_run */
  double k1_ms_total;     /* CUDA-event time of the gradient kernel (device 0), all passes */
  int64_t k1_launches;    /* launches of the gradient kernel per device */
  int64_t gpu_launches;   /* this library's own kernel launches issued by the call, per device */
  double allreduce_ms_total; /* CUDA-event time of the all-reduce (0 when world == 1) */
  double device_ms_total;    /* CUDA events on device 0's stream around the whole call */
  int64_t collective_calls;  /* all-reduces enqueued per device */
  int32_t wasted_passes;     /* speculative applySmooth(x) passes discarded because ||x-y||^2 == 0 (AGD.scala:265) */
  int32_t fused_passes;      /* applySmooth evaluations that shared a sweep over X with another one (sweeps = passes - fused_passes) */
} agd_stats;

/* ---- lifecycle ---- */
int agd_abi_version(void);
/* sizeof(agd_params) / sizeof(agd_stats) as compiled, so a foreign binding can verify its struct layout */
int agd_sizeof_params(void);
int agd_sizeof_stats(void);
void agd_default_params(agd_params *p);
/* Opens n_dev local GPUs (device ordinals in device_ids).  Fails when a device is not sm_90. */
int agd_create(const int32_t *device_ids, int32_t n_dev, agd_handle **out);
int agd_destroy(agd_handle *h);
/* Message of the last failure on this handle (h may be NULL: last agd_create failure). */
const char *agd_last_error(const agd_handle *h);

/* ---- the collective (replaces treeAggregate + broadcast, AGD.scala:193,196-204) ----
 * One rank per GPU.  With a single process owning all GPUs nothing needs to be called (the local GPUs
 * are a complete world: direct peer pointers, NCCL only as a fallback); calling agd_comm_init on such a
 * handle replaces that default, e.g. two processes with two GPUs each = world 4.  With one process per GPU (torchrun / one executor per GPU): rank 0
 * calls agd_comm_unique_id, ships the 128 bytes to every process, and every process calls
 * agd_comm_init(h, id, world_ranks, first_rank) where its local GPUs take ranks
 * first_rank .. first_rank + n_dev - 1. */
int agd_comm_unique_id(void *out128);
int agd_comm_init(agd_handle *h, const void *id128, int32_t world_ranks, int32_t first_rank);
/* The same world WITHOUT NCCL.  The per-pass exchange never uses a library (P2P stores + epoch flags into peer HBM,
 * csrc/xchg.cu); only its setup needs every rank to learn every other rank's CUDA IPC handles, and the host language can
 * ship those itself (a Spark driver collecting one small blob per executor; torch.distributed / gloo in the tests):
 *   1. every process:          agd_comm_init_ipc(h, world_ranks, first_rank)
 *   2. after loading its shards (the feature dimension sizes the buffers):
 *                              agd_xchg_export(h, blob, capacity, &n)   -> n = local GPUs * AGD_XCHG_HANDLE_BYTES
 *   3. host: concatenate every process's blob in rank order, hand the whole to every process:
 *                              agd_xchg_import(h, all, world_ranks * AGD_XCHG_HANDLE_BYTES)
 * Works between processes on different GPUs (NVLink / PCIe P2P) and between processes sharing ONE GPU (CUDA IPC on the
 * same device), which is how the 1-GPU test box exercises this path.  There is no fallback in such a world: if a pair
 * of ranks cannot map each other, agd_xchg_import fails.  Steps 2-3 are repeated after agd_clear + a load with another d. */
#define AGD_XCHG_HANDLE_BYTES 192
int agd_comm_init_ipc(agd_handle *h, int32_t world_ranks, int32_t first_rank);
int agd_xchg_export(agd_handle *h, void *out, int64_t capacity_bytes, int64_t *bytes_written);
int agd_xchg_import(agd_handle *h, const void *all_ranks, int64_t bytes);

/* ---- shard loading (replaces RDD[(Double, Vector)] partitions cached on executors, AGD.scala:178) ----
 * agd_reserve fixes the shard geometry of local device `dev` and allocates HBM for `rows_capacity`
 * rows stored as `store_dtype` (AGD_F64, AGD_F32 or AGD_BF16; values are rounded to nearest-even).  agd_load_dense APPENDS `rows` rows (row-major,
 * leading dimension ld elements, element type src_dtype AGD_F64|AGD_F32) and their labels.  If the
 * device was not reserved, the first load reserves exactly `rows`. */
int agd_reserve(agd_handle *h, int32_t dev, int64_t rows_capacity, int32_t d, int32_t store_dtype);
int agd_load_dense(agd_handle *h, int32_t dev, const void *X, int32_t src_dtype, const double *labels,
                   int64_t rows, int32_t d, int64_t ld, int32_t store_dtype);
/* SparseVector rows as CSR (values src_dtype AGD_F64|AGD_F32, stored as store_dtype AGD_F64|AGD_F32).
 * APPENDS `rows` rows: rowptr has rows+1 entries starting at 0 and is rebased onto the resident shard. */
int agd_load_csr(agd_handle *h, int32_t dev, const int64_t *rowptr, const int32_t *idx, const void *val,
                 int32_t src_dtype, const double *labels, int64_t rows, int32_t d, int32_t store_dtype);
/* LIBSVM text ingest (MLUtils.loadLibSVMFile of spark-mllib 1.3.0, the usual producer of the RDD handed to optimize):
 * `label index:value ...` per line, one-based ascending indices, '#' comment lines and blank lines skipped,
 * num_features <= 0 infers the dimension.  agd_libsvm_read parses on the host (no GPU needed) into an opaque
 * object with accessors; agd_load_libsvm parses and appends the rows as CSR, split over the local GPUs. */
typedef struct agd_libsvm agd_libsvm;
int agd_libsvm_read(const char *path, int32_t num_features, agd_libsvm **out);
int64_t agd_libsvm_rows(const agd_libsvm *L);
int32_t agd_libsvm_dim(const agd_libsvm *L);
int64_t agd_libsvm_nnz(const agd_libsvm *L);
const int64_t *agd_libsvm_rowptr(const agd_libsvm *L);
const int32_t *agd_libsvm_indices(const agd_libsvm *L);
const double *agd_libsvm_values(const agd_libsvm *L);
const double *agd_libsvm_labels(const agd_libsvm *L);
const char *agd_libsvm_error(const agd_libsvm *L);
void agd_libsvm_free(agd_libsvm *L);
int agd_load_libsvm(agd_handle *h, const char *path, int32_t num_features, int32_t store_dtype);
/* Drops every shard (all local devices). */
int agd_clear(agd_handle *h);
/* Rows currently resident on local device `dev`; feature count (0 when empty). */
int64_t agd_rows(const agd_handle *h, int32_t dev);
int32_t agd_dim(const agd_handle *h);

/* ---- measurement harness (not in the reference): synthetic workload generated in place ----
 * Every GPU rank r of the world fills its shard with global rows [r*total_rows/W, (r+1)*total_rows/W)
 * of the counter-based synthetic design matrix (spec: spark-agd_b200/csrc/synth.cu) and labels for
 * `gradient`.  agd_get_rows downloads rows (as the storage dtype) and labels for checking. */
int agd_generate(agd_handle *h, int64_t total_rows, int32_t d, int32_t store_dtype, uint64_t seed,
                 int32_t gradient);
int agd_get_rows(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, void *X_out, double *labels_out);
int agd_synth_wtrue(agd_handle *h, uint64_t seed, int32_t d, double *w_out);
/* CSR flavour of the synthetic workload: exactly nnz_per_row stored entries per row, strictly increasing
 * column ids (stratified), same label rules.  agd_get_csr_rows downloads a row range (rowptr rebased to 0). */
int agd_generate_csr(agd_handle *h, int64_t total_rows, int32_t d, int32_t nnz_per_row, int32_t store_dtype,
                     uint64_t seed, int32_t gradient);
int agd_get_csr_rows(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, int64_t *rowptr_out, int32_t *idx_out,
                     void *val_out, int64_t nnz_capacity, double *labels_out);

/* ---- plug-in granularity entry points (host buffers in and out) ----
 * agd_smooth = applySmooth (AGD.scala:192-208): loss/count and grad/count over ALL shards of the
 * world; w, grad are d doubles on the host.  Every rank must call it. */
int agd_smooth(agd_handle *h, int32_t gradient, const double *w, double *loss, double *grad, int64_t *count);
/* agd_smooth at w plus the loss (no gradient) at a second point w2, both from ONE sweep over the shards -- the fused form of
 * applySmooth(y) (AGD.scala:250) and the history evaluation applySmooth(x) (:304) that agd_run uses.  On dense shards every
 * output equals, bit for bit, what two agd_smooth calls return.  Fails on shards whose kernel has no two-point form
 * (wgmma bf16 path, d below one 16-row tile); agd_run then simply does not fuse. */
int agd_smooth_pair(agd_handle *h, int32_t gradient, const double *w, const double *w2, double *loss, double *grad,
                    int64_t *count, double *loss2);
/* Two complete applySmooth evaluations (loss and gradient at w AND at w2) from ONE sweep over the shards -- what agd_run's
 * memoised pass structure uses to evaluate applySmooth(x) of the backtracking test (AGD.scala:269) together with
 * applySmooth(y) of the next iteration (:250).  Bit for bit what two agd_smooth calls return.  Dense fp32 / fp64 shards with
 * at most 512 16-byte vectors per row (d <= 2048 fp32, <= 1024 fp64) and bf16 shards on the wgmma kernel; fails elsewhere. */
int agd_smooth_two(agd_handle *h, int32_t gradient, const double *w, const double *w2, double *loss, double *grad,
                   int64_t *count, double *loss2, double *grad2);
/* ---- scoring the resident shards (GeneralizedLinearModel.predict and model evaluation without a host copy of X) ----
 * Both compute the margin m_i = x_i . w + b in fp64 (every element widened, products and sums by DFMA); w is d doubles.
 * A margin depends only on the row, w, b and d: not on the row's position, the range asked for, the devices or the rank.
 * Padded columns take zero weight, CSR margins sum exactly the row's stored entries, non-finite features follow IEEE
 * arithmetic (an inf feature under a zero weight gives a NaN margin). */
/* Margins of rows [row0, row0 + rows) of the shard on local device dev into out (rank-local, not collective). */
int agd_margins(agd_handle *h, int32_t dev, const double *w, double intercept, int64_t row0, int64_t rows, double *out);
/* The AGD_EVAL_* sums over ALL shards of the world (collective, like agd_smooth); identical bits on every rank and on
 * every repeated call.  LOSS is the `gradient` loss of m_i (intercept included).  TP/FP/TN/FN count rows labelled exactly
 * 0 or 1 whose predicted class is 1 when sigmoid(m) > threshold (logistic) or m > threshold (hinge); they stay 0 for the
 * least-squares gradients.  SUM_ERR* are over e = m_i - y_i, SUM_Y* over the labels. */
enum { AGD_EVAL_COUNT = 0, AGD_EVAL_LOSS, AGD_EVAL_TP, AGD_EVAL_FP, AGD_EVAL_TN, AGD_EVAL_FN,
       AGD_EVAL_SUM_ERR, AGD_EVAL_SUM_ERR2, AGD_EVAL_SUM_ABS_ERR, AGD_EVAL_SUM_Y, AGD_EVAL_SUM_Y2, AGD_EVAL_N };
int agd_evaluate(agd_handle *h, int32_t gradient, const double *w, double intercept, double threshold, double *out);
/* Column statistics over ALL shards of the world (Statistics.colStats; collective, like agd_evaluate): *count = rows in the
 * view, out = AGD_COLSTAT_N x agd_dim(h) doubles, statistic-major (out[k * agd_dim(h) + j]).  Zeros count as values
 * (explicit zeros, a CSR row's implicit zeros, zeros of dense rows); padded columns are not reported.  SUM = sum x,
 * SUM_SQ = sum x^2, SUM_ABS = sum |x|, NNZ = entries with x != 0 (a NaN is nonzero), DEV / DEV2 = sum (x - mu) and
 * sum (x - mu)^2 with mu = fl(SUM / count) (the unbiased variance is (DEV2 - DEV^2 / count) / (count - 1)), MAX / MIN over
 * every value, NaN ignored (NaN when every value is NaN).  Two reads of X; sums follow IEEE arithmetic.  Identical bits on
 * every rank; dense shards also on every repeated call (CSR sums are scattered: equal to rounding). */
enum { AGD_COLSTAT_SUM = 0, AGD_COLSTAT_SUM_SQ, AGD_COLSTAT_SUM_ABS, AGD_COLSTAT_NNZ,
       AGD_COLSTAT_DEV, AGD_COLSTAT_DEV2, AGD_COLSTAT_MAX, AGD_COLSTAT_MIN, AGD_COLSTAT_N };
int agd_col_stats(agd_handle *h, double *count, double *out);
/* Cross-products over ALL shards of the world (RowMatrix.computeGramianMatrix / computeCovariance; collective, like
 * agd_col_stats; agd_set_row_filter applies, agd_set_feature_transform does not).  *count = rows in the view; out =
 * (agd_dim(h) + 1)^2 doubles, row-major and exactly symmetric: out[i][j] = sum z_i z_j, out[i][d] = out[d][i] = sum z_i,
 * out[d][d] = count, with z = x (centered = 0) or z = x - mu, mu = fl(sum x / count) (centered = 1; CSR shards derive the
 * centered sums from the uncentered ones).  Zeros count as values; a row outside the view leaves no trace; sums follow IEEE
 * arithmetic.  Identical bits on every rank; dense shards also on every repeated call (CSR sums are scattered: equal to
 * rounding).  agd_dim(h) <= AGD_GRAMIAN_MAX_DIM. */
enum { AGD_GRAMIAN_MAX_DIM = 8192 };
int agd_gramian(agd_handle *h, int32_t centered, double *count, double *out);
/* RowMatrix.multiply: the rows of h's current view times B (agd_dim(h) x k, row-major, finite fp64) plus offset (k doubles,
 * NULL = 0), into the EMPTY handle dst opened on the same local device ordinals in the same world position (rank-local, not
 * collective; agd_set_row_filter of h applies, agd_set_feature_transform does not: fold a transform into B and offset).
 * On every local device i, dst's shard i then holds the view's rows of h's shard i in physical order, as k features stored as
 * store_dtype (AGD_F64, AGD_F32 or AGD_BF16), each with its label: exactly the shard a load of those rows would give (the same
 * padding, kernel and solver).  Every y_ij is an fp64 sum of x_il b_lj over the row's features (a CSR row's stored entries in
 * stored order, a repeated column adding up) in an order that depends only on agd_dim(h) and k, then + offset_j, rounded
 * once to nearest-even: the bits of a projected row depend only on that row, B and offset.  Non-finite features follow IEEE
 * arithmetic; a row outside the view is never read.  Without a row filter dst's rows keep h's numbering (a view of dst selects
 * the rows the same view of h selects); with one, dst numbers them as a loaded shard.  Fails on a non-empty dst (left as it
 * is), other devices or world position, k < 1, a non-finite entry of B or offset, or a shard of 2^31 rows or more; a failure
 * after these checks (e.g. an allocation) leaves dst cleared. */
int agd_project(agd_handle *h, const double *B, int32_t k, const double *offset, agd_handle *dst, int32_t store_dtype);
/* Ranking metrics over ALL shards of the world (BinaryClassificationMetrics of mllib 1.3.0; collective, like agd_evaluate).
 * Rows: every row of the current view (agd_set_row_filter applies; agd_set_feature_transform does not: score a transformed
 * model with weights s o v and intercept b, as for agd_evaluate); a row outside the view leaves no trace.  A row is positive
 * iff label > 0.5.  Its score is the fp64 margin m = x . w + intercept with exactly the bits agd_margins returns, -0 taken as
 * +0; a row whose margin is NaN is only counted (AGD_BIN_NAN) and left out of the curve.
 * The curve has one point per distinct score, in descending order, with the cumulative counts TP_k / FP_k of the rows scoring
 * at least that much.  With P positives and N negatives, ROC = (0, 0), (FP_k / N, TP_k / P) ..., (1, 1) and PR = (0, 1),
 * (TP_k / P, TP_k / (TP_k + FP_k)) ...; the areas are trapezoid sums over those points, fp64 in a fixed order (the bits depend
 * on the curve only: identical on every rank, every repeated call, every partitioning of the same rows, dense or CSR).
 * AUROC is NaN when P = 0 or N = 0, AUPR when P = 0.  Counts are exact.
 * w: agd_dim(h) doubles; out: AGD_BIN_N doubles; *n_points = points of the curve.  The curve (margin_out descending, tp_out,
 * fp_out cumulative) is written only when capacity >= *n_points; capacity 0 asks for the areas only.  Scratch memory (about
 * 18 bytes per local row, and 48 bytes per distinct score of the world on the first local device) stays on the handle until
 * agd_clear / agd_destroy. */
enum { AGD_BIN_POS = 0, AGD_BIN_NEG, AGD_BIN_NAN, AGD_BIN_AUROC, AGD_BIN_AUPR, AGD_BIN_N };
int agd_binary_curve(agd_handle *h, const double *w, double intercept, int64_t capacity, double *margin_out, int64_t *tp_out,
                     int64_t *fp_out, int64_t *n_points, double *out);

/* ---- clustering the resident shards (KMeans of mllib 1.3.0) ----
 * Every call works on the rows of the current view in its feature space: agd_set_row_filter applies (a row outside the view is
 * never read, so a non-finite feature in one leaves no trace) and so does agd_set_feature_transform, so a row is
 * z = appendBias(s o x), D = agd_dim(h) + append_bias features, s o x formed in fp64.  Centres are k x D finite doubles,
 * row-major; sums and sampled rows have D entries per row.
 * A row's centre is the lowest index j minimising the score ||c_j||^2 - 2 z . c_j, with z . c_j the fp64 sum agd_project forms
 * (x . (s o c_j), plus the bias entry of c_j; dense shards: DMMA in an order that depends only on agd_dim(h) and k; CSR: the
 * stored entries in stored order).  A NaN score never wins; a row no centre wins goes to centre 0.  The centre therefore
 * depends only on the row and the centres, and differs from the exact argmin only where the two best exact distances lie
 * within the cross term's rounding.  Distances and costs are exact residuals sum_l (z_l - c_l)^2 in fp64 (a CSR row:
 * ||c||^2 + the sum over its stored entries, and the bias, of (z_l - c_l)^2 - c_l^2).  Shards of 2^31 rows or more are refused.
 * Scratch (about 40 bytes per local row, 12 more per 128 centres beyond the first 128, and 8 for agd_kmeans_costs' per-row
 * cost) stays on the handle until agd_clear / agd_destroy. */
/* One Lloyd step over ALL shards of the world (collective): every row of the view assigned to its centre; sums_out (k x D, NULL =
 * not returned) = the sum of each centre's rows, counts_out (k) = their number, *cost_out = the sum of every row's residual to
 * its centre.  One exchange of k (D + 1) + 1 doubles.  Dense sums are fp64 in a fixed order (the rows sorted stably by centre,
 * pieces of 4096 rows added in order): identical bits on every rank and every repeated call.  CSR sums and cost are scattered
 * with fp64 RED.ADD: equal to rounding.  Counts are exact. */
int agd_kmeans_step(agd_handle *h, const double *centers, int32_t k, double *sums_out, double *counts_out, double *cost_out);
/* Centres of physical rows [row0, row0 + rows) of the shard on local device dev (rank-local, not collective, like agd_margins):
 * cluster_out[i] = the row's centre, or -1 for a row outside the view; dist_out (NULL = not returned) = its residual (NaN
 * outside the view). */
int agd_kmeans_assign(agd_handle *h, int32_t dev, const double *centers, int32_t k, int64_t row0, int64_t rows,
                      int32_t *cluster_out, double *dist_out);
/* The cost update of k-means|| (collective): every row of the view gets delta = its residual to the centre among these m
 * candidates that it is assigned to, or with keep the smaller of that and its previous delta (a NaN residual never replaces
 * it); *sum_out = the sum of delta over the world, added in a fixed order (identical bits on every rank and repeated call).
 * delta stays on the handle (8 bytes per local row) for agd_kmeans_sample.  keep needs a previous call on the same rows. */
int agd_kmeans_costs(agd_handle *h, const double *centers, int32_t m, int32_t keep, double *sum_out);
/* The rows of the view kept by the k-means draw (collective): row r is kept iff u < factor * delta_r (weighted = 1, delta of
 * the last agd_kmeans_costs) or u < factor (weighted = 0), u = the top 53 bits of the row's Philox draw u(seed, grow) of
 * stream 8 (see agd_set_row_filter) as a double in [0, 1).  *n_out = rows kept over the world; when capacity >= *n_out,
 * rows_out (n x D) holds them as fp64 features of the view's space and draws_out (NULL = not returned) their u, in rank order
 * and physical order within a rank.  capacity 0 asks for the count only.  factor must be finite and >= 0. */
int agd_kmeans_sample(agd_handle *h, uint64_t seed, double factor, int32_t weighted, int64_t capacity, double *rows_out,
                      double *draws_out, int64_t *n_out);

/* ---- classifying the resident shards (NaiveBayes and MulticlassMetrics of mllib 1.3.0) ----
 * Labels are compared by value (-0.0 is 0.0).  Like the clustering calls, these work on the rows of the current view
 * (agd_set_row_filter applies; a row outside the view is never read) in its feature space (agd_set_feature_transform applies:
 * z = appendBias(s o x), D = agd_dim(h) + append_bias features).  Class labels passed in ascend strictly and are not NaN, at
 * most AGD_MAX_CLASSES of them.  Shards of 2^31 rows or more are refused.  Scratch stays on the handle until agd_clear /
 * agd_destroy.  The JNI shim does not bind these calls. */
enum { AGD_MAX_CLASSES = 1024 };
/* The distinct labels of the view over ALL shards of the world (collective; the distinct values of MLlib's labels), ascending,
 * with exact counts; *nan_out = rows of the view whose label is NaN (not among the labels).  *n_out = distinct labels; they and
 * counts_out are written only when capacity >= *n_out (capacity 0 asks for the counts only, as agd_binary_curve does).  The
 * sort and reduce are agd_binary_curve's, over a key that orders labels ascending. */
int agd_label_classes(agd_handle *h, int64_t capacity, double *labels_out, int64_t *counts_out, int64_t *n_out,
                      int64_t *nan_out);
/* Per class over ALL shards of the world (collective; the aggregate of NaiveBayes.run): the rows of the view whose label equals
 * labels[c] give counts_out[c] = their number and sums_out[c] (C x D, row-major) = the sum of their features; *negative_out =
 * the entries of those rows that are not >= 0 (NaN included; a CSR row's stored entries only).  One exchange of C (D + 1) + 1
 * doubles.  The sums are agd_kmeans_step's: dense shards add each class's rows in a fixed order (identical bits on every rank
 * and repeated call), CSR shards scatter with fp64 RED.ADD (equal to rounding).  Counts are exact. */
int agd_class_sums(agd_handle *h, const double *labels, int32_t C, double *sums_out, double *counts_out, double *negative_out);
/* The linear model's class of physical rows [row0, row0 + rows) of the shard on local device dev (rank-local, not collective,
 * like agd_kmeans_assign; NaiveBayesModel.predict): class_out[i] = the lowest c maximising offset_c + z . W_c, or -1 for a row
 * outside the view.  W is C x D finite doubles, row-major, offset C finite doubles; z . W_c is the fp64 sum agd_kmeans_assign
 * forms.  A NaN score never wins; a row no class wins goes to class 0. */
int agd_linear_argmax(agd_handle *h, int32_t dev, const double *W, int32_t C, const double *offset, int64_t row0, int64_t rows,
                      int32_t *class_out);
/* counts_out (L x C doubles, row-major) = the rows of the view over ALL shards of the world (collective) whose label equals
 * labels[l] and whose agd_linear_argmax class is c; exact.  C is at most AGD_MAX_CLASSES too. */
int agd_linear_confusion(agd_handle *h, const double *W, int32_t C, const double *offset, const double *labels, int32_t L,
                         double *counts_out);

/* ---- views of the resident shards (RDD.randomSplit / sample / MLUtils.kFold without copying a row) ----
 * Every row has a 64-bit draw u = Philox4x32-10 keyed by `seed`, counter (grow lo, grow hi, 0, 7), words 0 and 1, where grow
 * = the shard's first global row + local row (the numbering of the mini-batch mask: a generated shard's global row, or
 * rank << 40 + row on loaded shards, so views of loaded shards depend on the partitioning).  Predicate i holds iff
 * floor(lo[i] 2^64) <= u < floor(hi[i] 2^64), with hi = 1 meaning "to the end"; complement[i] = 1 negates it.  A row is in
 * the view iff all n predicates hold (n <= 4).  agd_set_row_filter installs the view; it applies to agd_smooth,
 * agd_smooth_pair, agd_smooth_two, agd_run, agd_gd_run, agd_gd_run_minibatch (a row must then also pass the mini-batch
 * mask), agd_evaluate, agd_col_stats, agd_gramian, agd_project, agd_binary_curve, agd_kmeans_step, agd_kmeans_assign, agd_kmeans_costs,
 * agd_kmeans_sample, agd_label_classes, agd_class_sums, agd_linear_argmax and agd_linear_confusion, and not to agd_margins, agd_get_rows or the loads, which address physical rows.  Rows outside the
 * view are never touched: a non-finite feature in one leaves no trace.  The filter stays until it is replaced, cleared
 * (n = 0) or dropped by agd_clear; every rank must set the same filter before a collective call.  Bounds must satisfy
 * 0 <= lo <= hi <= 1 and complement must be 0 or 1.  A view still streams the whole shard through the gradient kernels. */
int agd_set_row_filter(agd_handle *h, int32_t n, const uint64_t *seeds, const double *lo, const double *hi,
                       const int32_t *complement);
/* out[i] = 1 if physical row row0 + i of the shard on local device dev is in the current view, else 0 (rank-local, not
 * collective; the kernels' own predicate, so a host never restates the draw). */
int agd_row_filter_mask(agd_handle *h, int32_t dev, int64_t row0, int64_t rows, uint8_t *out);

/* ---- feature transforms: train on appendBias(s o x) without materialising it ----
 * Installs the transform MLlib's GeneralizedLinearAlgorithm applies before its optimizer: each stored feature x_j is multiplied by
 * scale[j] (StandardScaler, withMean = false: scale = 1 / sigma, or 0 where sigma = 0), and with append_bias a constant 1.0 is
 * appended as the last feature (MLUtils.appendBias): the intercept is the last weight, regularised like every other.
 * scale: NULL (no scaling) or agd_dim(h) finite doubles; append_bias: 0 or 1.  (NULL, 0) clears the transform.
 * It applies to agd_smooth, agd_smooth_pair, agd_smooth_two, agd_run, agd_gd_run and agd_gd_run_minibatch: their weights and
 * gradients then have agd_dim(h) + append_bias doubles, the intercept last.  It applies to agd_kmeans_step, agd_kmeans_assign,
 * agd_kmeans_costs and agd_kmeans_sample too: their centres, sums and rows have agd_dim(h) + append_bias entries; and to
 * agd_class_sums, agd_linear_argmax and agd_linear_confusion: their sums and W rows have agd_dim(h) + append_bias entries.  (agd_prox takes its dimension as an argument.)
 * It does not apply to agd_margins, agd_evaluate, agd_col_stats, agd_gramian, agd_project, the loads or the row accessors, which address the stored
 * features: score a transformed model there with weights s o v and intercept b.
 * The rows are never rewritten: the gradient kernels add b to every margin and sum the multipliers for the intercept's
 * gradient, the point is scaled (w_eff = s o v) before each sweep and the gradient columns after it, so a scaled value is never
 * rounded to the storage type.  Like agd_set_row_filter, the transform stays until it is replaced, cleared or dropped by
 * agd_clear, a failed install leaves none, and every rank must install the same one before a collective call. */
int agd_set_feature_transform(agd_handle *h, const double *scale, int32_t append_bias);

/* agd_prox = applyProjector (AGD.scala:214-222): Updater.compute(w, g, step, iter = 1, reg). */
int agd_prox(agd_handle *h, int32_t updater, const double *w, const double *g, double step, double reg,
             int32_t d, double *w_out, double *reg_val);

/* ---- the whole loop, natively: AcceleratedGradientDescent.run (AGD.scala:177-338) ----
 * w0, w_out: d doubles.  loss_hist: capacity >= max(num_iterations, 1); *n_hist receives its length.
 * Every rank must call it with identical arguments; every rank receives identical results. */
int agd_run(agd_handle *h, const agd_params *p, const double *w0, double *w_out, double *loss_hist,
            int32_t *n_hist, agd_stats *stats);

/* GradientDescent.runMiniBatchSGD of spark-mllib 1.3.0 with miniBatchFraction = 1.0 (the comparator
 * the reference's tests run beside AGD, Suite.scala:78,118,225), on the same kernels. */
int agd_gd_run(agd_handle *h, int32_t gradient, int32_t updater, double step_size, int32_t num_iterations,
               double reg_param, const double *w0, double *w_out, double *loss_hist, int32_t *n_hist,
               agd_stats *stats);

/* The mini-batch form: iteration i uses the rows kept by `data.sample(false, miniBatchFraction, 42 + i)`, realised as a
 * counter-based Bernoulli mask (Philox keyed by 42 + i and the global row index; Spark's own sampler is seeded per
 * partition and is not reproducible across partitionings either).  fraction >= 1 is the full batch. */
int agd_gd_run_minibatch(agd_handle *h, int32_t gradient, int32_t updater, double step_size, int32_t num_iterations,
                         double reg_param, double mini_batch_fraction, const double *w0, double *w_out,
                         double *loss_hist, int32_t *n_hist, agd_stats *stats);

/* Name of the gradient kernel the shard on local device `dev` dispatches to (for reports), "" when empty. */
const char *agd_kernel_name(const agd_handle *h, int32_t dev);

/* Options: "k1_variant" = auto|ring|generic|tc, "collective" = auto|nccl|p2p, ring tuning knobs. */
int agd_set_option(agd_handle *h, const char *key, const char *value);

#ifdef __cplusplus
}
#endif
#endif /* AGD_B200_H */
