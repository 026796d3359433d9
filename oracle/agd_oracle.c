/*
 * agd_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C, fp64 restatement of the reference's accelerated-gradient-descent
 * hot path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may link or call this file; the product
 * (spark-agd_b200/, include/) never does.
 *
 * What it follows (paths relative to /root/reference):
 *   AGD.scala = src/main/scala/org/apache/spark/mllib/optimization/AcceleratedGradientDescent.scala
 *   Suite.scala = src/test/scala/org/apache/spark/mllib/optimization/AcceleratedGradientDescentSuite.scala
 *
 *   oracle_smooth      <- applySmooth            AGD.scala:192-208 (seqOp :197-200, combOp :201-204)
 *   oracle_prox        <- applyProjector         AGD.scala:214-222
 *   oracle_agd_run     <- AcceleratedGradientDescent.run  AGD.scala:177-338
 *   oracle_gd_run      <- GradientDescent.runMiniBatchSGD (comparator in Suite.scala:78,118,225)
 *   oracle_generate_gd_input <- GradientDescentSuite.generateGDInput (Suite.scala:46)
 *
 * The per-example arithmetic is NOT in /root/reference: it lives in the un-vendored
 * dependency org.apache.spark:spark-mllib_2.10:1.3.0 (build.sbt:7) -- Gradient.scala
 * (LogisticGradient / LeastSquaresGradient / HingeGradient), Updater.scala (SimpleUpdater /
 * L1Updater / SquaredL2Updater), MLUtils.log1pExp, BLAS.dot/axpy (netlib F2J ddot/daxpy,
 * i.e. a single sequential accumulator), breeze norm/dot (sequential) -- and is restated
 * here from the published 1.3.0 algorithm.
 *
 * PARITY PIN STATUS: the reference ships NO golden vectors for this path and cannot be
 * executed in this image (no JVM).  This oracle is pinned against every test the
 * reference's own suite holds (Suite.scala T1-T4 relational assertions, T5 plumbing) in
 * tests/test_oracle_reference_suite.py; bit-level results of Gradient/Updater are
 * "parity unpinned" by the reference itself.
 *
 * Arithmetic rules kept on purpose (JVM semantics): no FMA contraction (compile with
 * -ffp-contract=off), sequential single-accumulator dot/norm, elementwise a*s + b*t with
 * separate roundings, Java Math.min/max NaN propagation, xy_sq = pow(norm(xy), 2).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#ifdef __linux__
#include <sched.h> /* sched_setaffinity: the Makefile passes -D_GNU_SOURCE */
#endif

#include "agd_oracle.h"

/* ---------- Java Math.min / Math.max (NaN-propagating; AGD.scala:274,286,292,322) ---------- */
static double jmax(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return signbit(a) ? b : a; /* max(-0.0, 0.0) = 0.0 */
  return a > b ? a : b;
}
static double jmin(double a, double b) {
  if (a != a) return a;
  if (b != b) return b;
  if (a == 0.0 && b == 0.0) return signbit(a) ? a : b;
  return a < b ? a : b;
}

/* ---------- MLUtils.log1pExp [mllib-1.3.0] ---------- */
static double log1p_exp(double x) {
  if (x > 0) return x + log1p(exp(-x));
  return log1p(exp(x));
}

/* ---------- row access: dense f64 / dense f32 (upcast) / CSR ---------- */
static inline double row_dot(const oracle_data *D, int64_t i, const double *w) {
  double s = 0.0; /* netlib ddot: one sequential accumulator */
  if (D->storage == ORACLE_DENSE_F64) {
    const double *x = D->Xd + i * D->ld;
    for (int32_t j = 0; j < D->d; ++j) s += x[j] * w[j];
  } else if (D->storage == ORACLE_DENSE_F32) {
    const float *x = D->Xf + i * D->ld;
    for (int32_t j = 0; j < D->d; ++j) s += (double)x[j] * w[j];
  } else { /* SparseVector dot: iterate stored entries in index order */
    for (int64_t k = D->rowptr[i]; k < D->rowptr[i + 1]; ++k) {
      double v = D->csr_val_f32 ? (double)D->csr_val_f32[k] : D->csr_val[k];
      s += v * w[D->csr_idx[k]];
    }
  }
  return s;
}
/* Dense axpy is netlib DAXPY (through F2J), which starts with IF (DA.EQ.0) RETURN: a dense row with multiplier exactly 0 adds
   nothing, whatever its features.  The sparse axpy of BLAS.scala is a plain loop with no such test, so 0 * inf = NaN shows.
   On finite rows the return only drops +-0 terms, and a sum that starts at +0 never becomes -0: the bits are the same. */
static inline void row_axpy(const oracle_data *D, int64_t i, double a, double *g) {
  if (D->storage != ORACLE_CSR && a == 0.0) return;
  if (D->storage == ORACLE_DENSE_F64) {
    const double *x = D->Xd + i * D->ld;
    for (int32_t j = 0; j < D->d; ++j) g[j] += a * x[j];
  } else if (D->storage == ORACLE_DENSE_F32) {
    const float *x = D->Xf + i * D->ld;
    for (int32_t j = 0; j < D->d; ++j) g[j] += a * (double)x[j];
  } else {
    for (int64_t k = D->rowptr[i]; k < D->rowptr[i + 1]; ++k) {
      double v = D->csr_val_f32 ? (double)D->csr_val_f32[k] : D->csr_val[k];
      g[D->csr_idx[k]] += a * v;
    }
  }
}

/* ---------- Gradient.compute(data, label, weights, cumGradient) [mllib-1.3.0], called at AGD.scala:198 ---------- */
static double gradient_compute(const oracle_data *D, int kind, int64_t i, const double *w, double *cum) {
  const double label = D->labels[i];
  switch (kind) {
  case ORACLE_GRAD_LOGISTIC: { /* LogisticGradient, binary branch */
    double margin = -1.0 * row_dot(D, i, w);
    double multiplier = (1.0 / (1.0 + exp(margin))) - label;
    row_axpy(D, i, multiplier, cum);
    if (label > 0) return log1p_exp(margin);
    return log1p_exp(margin) - margin;
  }
  case ORACLE_GRAD_LEAST_SQUARES: { /* 1.3.0: loss diff^2, gradient 2*diff*x (no 1/2) */
    double diff = row_dot(D, i, w) - label;
    row_axpy(D, i, 2.0 * diff, cum);
    return diff * diff;
  }
  case ORACLE_GRAD_LEAST_SQUARES_HALF: { /* Spark >= 1.4 variant, kept behind a switch */
    double diff = row_dot(D, i, w) - label;
    row_axpy(D, i, diff, cum);
    return diff * diff / 2.0;
  }
  case ORACLE_GRAD_HINGE: {
    double dotp = row_dot(D, i, w);
    double label_scaled = 2 * label - 1.0;
    if (1.0 > label_scaled * dotp) {
      row_axpy(D, i, -label_scaled, cum);
      return 1.0 - label_scaled * dotp;
    }
    return 0.0;
  }
  }
  return NAN;
}

/* ---------- applySmooth, AGD.scala:192-208, in treeAggregate shape ---------- */
int oracle_smooth(const oracle_data *D, int grad_kind, const double *w, int partitions, int threads,
                  double *loss_out, double *grad_out, int64_t *count_out) {
  const int32_t d = D->d;
  int P = partitions < 1 ? 1 : partitions;
  double *pg = (double *)calloc((size_t)P * (size_t)d, sizeof(double));
  double *pl = (double *)calloc((size_t)P, sizeof(double));
  int64_t *pc = (int64_t *)calloc((size_t)P, sizeof(int64_t));
  if (!pg || !pl || !pc) { free(pg); free(pl); free(pc); return -1; }
  (void)threads;
  /* per-partition sequential fold (seqOp AGD.scala:197-200); partition p owns the
     ParallelCollectionRDD slice [p*n/P, (p+1)*n/P).  Partition p always runs on thread p % threads (the result does
     not depend on the mapping -- the combine below is ordered -- but the CPU timing on a NUMA host does). */
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(threads > 0 ? threads : 1)
#endif
  for (int p = 0; p < P; ++p) {
    int64_t lo = (int64_t)(((__int128)p * D->n) / P), hi = (int64_t)(((__int128)(p + 1) * D->n) / P);
    double *g = pg + (size_t)p * d;
    double l = 0.0;
    int64_t c = 0;
    for (int64_t i = lo; i < hi; ++i) {
      if (D->sample_thresh && !oracle_row_selected(D->sample_seed, D->sample_thresh, i)) continue; /* data.sample(...) */
      l = l + gradient_compute(D, grad_kind, i, w, g);
      c = c + 1;
    }
    pl[p] = l; pc[p] = c;
  }
  /* combOp AGD.scala:201-204, ordered left fold over partitions 0..P-1 */
  double loss = pl[0];
  int64_t count = pc[0];
  double *grad = pg;
  for (int p = 1; p < P; ++p) {
    loss = loss + pl[p];
    count = count + pc[p];
    const double *g2 = pg + (size_t)p * d;
    for (int32_t j = 0; j < d; ++j) grad[j] += g2[j];
  }
  /* AGD.scala:207 (loss / count, grad / (count: Double)) */
  *loss_out = loss / (double)count;
  for (int32_t j = 0; j < d; ++j) grad_out[j] = grad[j] / (double)count;
  if (count_out) *count_out = count;
  free(pg); free(pl); free(pc);
  return 0;
}

/* ---------- Updater.compute(weightsOld, gradient, stepSize, iter, regParam) [mllib-1.3.0] ---------- */
static double updater_compute(int kind, const double *w_old, const double *g, double step_size, int iter,
                              double reg, int32_t d, double *w_new) {
  const double this_step = step_size / sqrt((double)iter);
  switch (kind) {
  case ORACLE_UPD_SIMPLE:
    for (int32_t j = 0; j < d; ++j) w_new[j] = w_old[j] + (-this_step) * g[j];
    return 0.0;
  case ORACLE_UPD_L1: {
    const double shrink = reg * this_step;
    double n1 = 0.0;
    for (int32_t j = 0; j < d; ++j) {
      double wi = w_old[j] + (-this_step) * g[j];
      double sg = (wi > 0.0) ? 1.0 : ((wi < 0.0) ? -1.0 : wi); /* scala signum */
      double v = sg * jmax(0.0, fabs(wi) - shrink);
      w_new[j] = v;
    }
    for (int32_t j = 0; j < d; ++j) n1 += fabs(w_new[j]);
    return n1 * reg;
  }
  case ORACLE_UPD_SQUARED_L2: {
    const double shrink = 1.0 - this_step * reg;
    double ss = 0.0;
    for (int32_t j = 0; j < d; ++j) {
      double wi = w_old[j] * shrink;
      wi = wi + (-this_step) * g[j];
      w_new[j] = wi;
    }
    for (int32_t j = 0; j < d; ++j) ss += w_new[j] * w_new[j];
    double nrm = sqrt(ss);
    return 0.5 * reg * nrm * nrm;
  }
  }
  return NAN;
}

/* applyProjector AGD.scala:214-222: iter = 1 neutralises the 1/sqrt(iter) decay. */
int oracle_prox(int upd_kind, const double *w, const double *g, double step, double reg, int32_t d,
                double *w_out, double *reg_val) {
  double r = updater_compute(upd_kind, w, g, step, 1, reg, d, w_out);
  if (reg_val) *reg_val = r;
  return 0;
}

/* breeze helpers (sequential) */
static double v_dot(const double *a, const double *b, int32_t d) {
  double s = 0.0;
  for (int32_t j = 0; j < d; ++j) s += a[j] * b[j];
  return s;
}
static double v_norm(const double *a, int32_t d) {
  double s = 0.0;
  for (int32_t j = 0; j < d; ++j) s += a[j] * a[j];
  return sqrt(s);
}

void oracle_default_params(oracle_params *p) { /* AGD.scala:44-51 */
  p->convergence_tol = 1e-4;
  p->num_iterations = 100;
  p->reg_param = 0.0;
  p->L0 = 1.0;
  p->Lexact = INFINITY;
  p->beta = 0.5;
  p->alpha = 0.9;
  p->may_restart = 1;
  p->partitions = 2;
  p->threads = 1;
}

/* ---------- AcceleratedGradientDescent.run, AGD.scala:177-338 ---------- */
int oracle_agd_run(const oracle_data *D, int grad_kind, int upd_kind, const oracle_params *p,
                   const double *w0, double *w_out, double *loss_hist, int32_t *n_hist,
                   oracle_stats *st) {
  const int32_t d = D->d;
  const size_t bytes = (size_t)d * sizeof(double);
  double *x = malloc(bytes), *z = malloc(bytes), *x_old = malloc(bytes), *z_old = malloc(bytes);
  double *y = malloc(bytes), *g_y = malloc(bytes), *g_x = malloc(bytes), *tmp = malloc(bytes);
  double *xy = malloc(bytes);
  if (!x || !z || !x_old || !z_old || !y || !g_y || !g_x || !tmp || !xy) return -1;
  oracle_stats s; memset(&s, 0, sizeof s);

  memcpy(x, w0, bytes);              /* :224 */
  memcpy(z, x, bytes);               /* :225 */
  double theta = INFINITY;           /* :226 */
  int nh = 0;                        /* :227 */
  double f_y = 0.0;                  /* :229 */
  memset(g_y, 0, bytes);             /* :230 */
  double L = p->L0;                  /* :232 */
  int backtrack_simple = 1;          /* :234 */
  const double backtrack_tol = 1e-10;/* :235 */
  const double Lexact = p->Lexact, beta = p->beta;

  for (int nIter = 1; nIter <= p->num_iterations; ++nIter) { /* :237 */
    memcpy(x_old, x, bytes); memcpy(z_old, z, bytes);        /* :241 */
    const double L_old = L;                                  /* :242 */
    L = L * p->alpha;                                        /* :243 */
    const double theta_old = theta;                          /* :244 */
    int nonterminating = 0;
    for (;;) {                                               /* :246 */
      theta = 2.0 / (1.0 + sqrt(1.0 + 4.0 * (L / L_old) / (theta_old * theta_old))); /* :248 */
      for (int32_t j = 0; j < d; ++j) y[j] = x_old[j] * (1.0 - theta) + z_old[j] * theta; /* :249 */
      oracle_smooth(D, grad_kind, y, p->partitions, p->threads, &f_y, g_y, NULL);        /* :250 */
      s.passes++;
      const double step = 1.0 / (theta * L);                                              /* :253 */
      updater_compute(upd_kind, z_old, g_y, step, 1, p->reg_param, d, z);                 /* :254 */
      for (int32_t j = 0; j < d; ++j) x[j] = x_old[j] * (1.0 - theta) + z[j] * theta;     /* :255 */
      if (beta >= 1.0) break;                                                             /* :257 */
      for (int32_t j = 0; j < d; ++j) xy[j] = x[j] - y[j];                                /* :263 */
      const double nxy = v_norm(xy, d);
      const double xy_sq = nxy * nxy; /* math.pow(norm(xy), 2) :264 */
      if (xy_sq == 0) break;                                                              /* :265 */
      double f_x;
      oracle_smooth(D, grad_kind, x, p->partitions, p->threads, &f_x, g_x, NULL);         /* :269 */
      s.passes++;
      double localL;
      if (backtrack_simple) {                                                             /* :272 */
        const double q_x = f_y + v_dot(xy, g_y, d) + 0.5 * L * xy_sq;                     /* :273 */
        localL = L + 2.0 * jmax(f_x - q_x, 0.0) / xy_sq;                                  /* :274 */
        backtrack_simple = (fabs(f_y - f_x) >= backtrack_tol * jmax(fabs(f_x), fabs(f_y))); /* :275 */
      } else {
        for (int32_t j = 0; j < d; ++j) tmp[j] = g_x[j] - g_y[j];
        localL = 2.0 * v_dot(xy, tmp, d) / xy_sq;                                         /* :278 */
      }
      if (localL <= L || L >= Lexact) break;                                              /* :281 */
      if (!isinf(localL)) L = jmin(Lexact, localL);                                       /* :285-287 */
      else localL = L;                                                                    /* :288-290 */
      L = jmin(Lexact, jmax(localL, L / beta));                                           /* :292 */
      s.backtracks++;
      if (L != L) { nonterminating = 1; break; } /* the reference would spin forever here (NaN never
                                                    satisfies :281); we stop and flag it. */
    }
    {                                                                                     /* :302-307 */
      double f_x, c_x;
      oracle_smooth(D, grad_kind, x, p->partitions, p->threads, &f_x, g_x, NULL);
      s.passes++;
      c_x = updater_compute(upd_kind, x, g_x, 0.0, 1, p->reg_param, d, tmp);
      loss_hist[nh++] = f_x + c_x;
    }
    s.iterations = nIter;
    if (nonterminating) { s.stopped_nan = 1; s.nonterminating = 1; break; }
    if (isnan(f_y) || isinf(f_y)) { s.stopped_nan = 1; break; }                           /* :309-312 */
    const double norm_x = v_norm(x, d);                                                   /* :315 */
    for (int32_t j = 0; j < d; ++j) tmp[j] = x[j] - x_old[j];
    const double norm_dx = v_norm(tmp, d);                                                /* :316 */
    if (norm_dx == 0.0) { if (nIter > 1) { s.converged = 1; break; } }                    /* :317-321 */
    if (norm_dx < p->convergence_tol * jmax(norm_x, 1)) { s.converged = 1; break; }       /* :322-324 */
    if (p->may_restart && v_dot(g_y, tmp, d) > 0.0) {                                     /* :327 */
      memcpy(z, x, bytes); theta = INFINITY; backtrack_simple = 1;                        /* :328-330 */
      s.restarts++;
    }
  }
  memcpy(w_out, x, bytes);                                                                /* :337 */
  *n_hist = nh;
  s.final_L = L; s.final_theta = theta;
  if (st) *st = s;
  free(x); free(z); free(x_old); free(z_old); free(y); free(g_y); free(g_x); free(tmp); free(xy);
  return 0;
}

/* ---------- GradientDescent.runMiniBatchSGD [mllib-1.3.0], miniBatchFraction = 1.0 only ----------
 * (BernoulliSampler with fraction 1.0 keeps every row, so sample(false, 1.0, 42+i) is the identity.) */
int oracle_gd_run(const oracle_data *D, int grad_kind, int upd_kind, double step_size, int num_iterations,
                  double reg_param, int partitions, int threads, const double *w0, double *w_out,
                  double *loss_hist, int32_t *n_hist) {
  const int32_t d = D->d;
  const size_t bytes = (size_t)d * sizeof(double);
  double *w = malloc(bytes), *g = malloc(bytes), *wn = malloc(bytes), *zero = calloc((size_t)d, sizeof(double));
  if (!w || !g || !wn || !zero) return -1;
  memcpy(w, w0, bytes);
  int nh = 0;
  if (D->n == 0) { memcpy(w_out, w0, bytes); *n_hist = 0; free(w); free(g); free(wn); free(zero); return 0; }
  double reg_val = updater_compute(upd_kind, w, zero, 0.0, 1, reg_param, d, wn);
  for (int i = 1; i <= num_iterations; ++i) {
    double mean_loss; int64_t cnt;
    /* gradientSum / miniBatchSize and lossSum / miniBatchSize: oracle_smooth performs the same divisions */
    oracle_smooth(D, grad_kind, w, partitions, threads, &mean_loss, g, &cnt);
    loss_hist[nh++] = mean_loss + reg_val;
    reg_val = updater_compute(upd_kind, w, g, step_size, i, reg_param, d, wn);
    memcpy(w, wn, bytes);
  }
  memcpy(w_out, w, bytes);
  *n_hist = nh;
  free(w); free(g); free(wn); free(zero);
  return 0;
}


/* StrictMath.log == fdlibm __ieee754_log (java.util.Random.nextGaussian is specified in terms of
 * StrictMath, so the fixture needs fdlibm's rounding, not glibc's).  Restated from the published
 * algorithm: argument reduction x = 2^k (1+f), s = f/(2+f), minimax polynomial in s^2. */
static double fdlibm_log(double x) {
  static const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10,
                      two54 = 1.80143985094819840000e+16, Lg1 = 6.666666666666735130e-01,
                      Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
                      Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01,
                      Lg6 = 1.531383769920937332e-01, Lg7 = 1.479819860511658591e-01;
  union { double d; uint64_t u; } b; b.d = x;
  int32_t hx = (int32_t)(b.u >> 32); uint32_t lx = (uint32_t)b.u;
  int32_t k = 0, i, j;
  if (hx < 0x00100000) {
    if (((hx & 0x7fffffff) | lx) == 0) return -two54 / 0.0;
    if (hx < 0) return (x - x) / 0.0;
    k -= 54; x *= two54; b.d = x; hx = (int32_t)(b.u >> 32);
  }
  if (hx >= 0x7ff00000) return x + x;
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  i = (hx + 0x95f64) & 0x100000;
  b.d = x; b.u = (b.u & 0xffffffffULL) | ((uint64_t)(uint32_t)(hx | (i ^ 0x3ff00000)) << 32); x = b.d;
  k += (i >> 20);
  double f = x - 1.0, dk, R, s, z, w, t1, t2, hfsq;
  if ((0x000fffff & (2 + hx)) < 3) {
    if (f == 0.0) { if (k == 0) return 0.0; dk = (double)k; return dk * ln2_hi + dk * ln2_lo; }
    R = f * f * (0.5 - 0.33333333333333333 * f);
    if (k == 0) return f - R;
    dk = (double)k; return dk * ln2_hi - ((R - dk * ln2_lo) - f);
  }
  s = f / (2.0 + f); dk = (double)k; z = s * s;
  i = hx - 0x6147a; w = z * z; j = 0x6b851 - hx;
  t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  i |= j; R = t2 + t1;
  if (i > 0) {
    hfsq = 0.5 * f * f;
    if (k == 0) return f - (hfsq - s * (hfsq + R));
    return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
  }
  if (k == 0) return f - s * (f - R);
  return dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f);
}

/* runMiniBatchSGD with miniBatchFraction < 1: iteration i folds the rows of data.sample(false, fraction, 42 + i),
 * realised as the counter-based Bernoulli mask of oracle_row_selected; an empty sample skips the update. */
int oracle_gd_run_minibatch(oracle_data *D, int grad_kind, int upd_kind, double step_size, int num_iterations,
                            double reg_param, double fraction, int partitions, int threads, const double *w0,
                            double *w_out, double *loss_hist, int32_t *n_hist) {
  const int32_t d = D->d;
  const size_t bytes = (size_t)d * sizeof(double);
  double *w = malloc(bytes), *g = malloc(bytes), *wn = malloc(bytes), *zero = calloc((size_t)d, sizeof(double));
  if (!w || !g || !wn || !zero) return -1;
  memcpy(w, w0, bytes);
  int nh = 0;
  double reg_val = updater_compute(upd_kind, w, zero, 0.0, 1, reg_param, d, wn);
  for (int i = 1; i <= num_iterations && D->n > 0; ++i) {
    double mean_loss; int64_t cnt;
    D->sample_seed = 42ull + (uint64_t)i;
    D->sample_thresh = fraction >= 1.0 ? 0ull : (uint64_t)ldexp(fraction, 64);
    oracle_smooth(D, grad_kind, w, partitions, threads, &mean_loss, g, &cnt);
    D->sample_thresh = 0;
    if (cnt <= 0) continue;
    loss_hist[nh++] = mean_loss + reg_val;
    reg_val = updater_compute(upd_kind, w, g, step_size, i, reg_param, d, wn);
    memcpy(w, wn, bytes);
  }
  memcpy(w_out, w, bytes);
  *n_hist = nh;
  free(w); free(g); free(wn); free(zero);
  return 0;
}

/* ---------- java.util.Random (48-bit LCG) ---------- */
void oracle_jrandom_seed(oracle_jrandom *r, int64_t seed) {
  r->seed = ((uint64_t)seed ^ 0x5DEECE66DULL) & ((1ULL << 48) - 1);
  r->have_next = 0; r->next_gaussian = 0.0;
}
static int32_t jr_next(oracle_jrandom *r, int bits) {
  r->seed = (r->seed * 0x5DEECE66DULL + 0xBULL) & ((1ULL << 48) - 1);
  return (int32_t)((int64_t)r->seed >> (48 - bits));
}
double oracle_jrandom_next_double(oracle_jrandom *r) {
  int64_t hi = (int64_t)jr_next(r, 26), lo = (int64_t)jr_next(r, 27);
  return (double)((hi << 27) + lo) * 0x1.0p-53;
}
double oracle_jrandom_next_gaussian(oracle_jrandom *r) {
  if (r->have_next) { r->have_next = 0; return r->next_gaussian; }
  double v1, v2, s;
  do {
    v1 = 2 * oracle_jrandom_next_double(r) - 1;
    v2 = 2 * oracle_jrandom_next_double(r) - 1;
    s = v1 * v1 + v2 * v2;
  } while (s >= 1 || s == 0);
  double mul = sqrt(-2 * fdlibm_log(s) / s); /* StrictMath.sqrt(-2 * StrictMath.log(s) / s) */
  r->next_gaussian = v2 * mul; r->have_next = 1;
  return v1 * mul;
}
void oracle_jrandom_fill_double(int64_t seed, int64_t n, double *out) {
  oracle_jrandom r; oracle_jrandom_seed(&r, seed);
  for (int64_t i = 0; i < n; ++i) out[i] = oracle_jrandom_next_double(&r);
}
int oracle_jrandom_continue_fill_double(oracle_jrandom *r, int64_t n, double *out) {
  for (int64_t i = 0; i < n; ++i) out[i] = oracle_jrandom_next_double(r);
  return 0;
}

/* GradientDescentSuite.generateGDInput(offset, scale, nPoints, seed) [mllib-1.3.0 tests];
 * the uniform stream's seed 45 is hard-coded upstream.  Called at Suite.scala:46. */
void oracle_generate_gd_input(double offset, double scale, int32_t n_points, int32_t seed, double *x1,
                              double *y) {
  oracle_jrandom rnd, unif;
  oracle_jrandom_seed(&rnd, seed);
  for (int32_t i = 0; i < n_points; ++i) x1[i] = oracle_jrandom_next_gaussian(&rnd);
  oracle_jrandom_seed(&unif, 45);
  for (int32_t i = 0; i < n_points; ++i) {
    double u = oracle_jrandom_next_double(&unif);
    double r_logis = log(u) - log(1.0 - u);
    double y_val = offset + scale * x1[i] + r_logis;
    y[i] = (y_val > 0) ? 1.0 : 0.0;
  }
}

/* ---------- CPU-timing hygiene (bench.py's reference arm): thread pinning and first-touch placement ---------- */
/* Pins OpenMP thread t of a `threads`-wide team to the t-th CPU of the process's affinity mask (the master too, until
 * oracle_unbind_threads).  libgomp keeps its pool between regions of the same width, so the folds that follow run on
 * the same cores that first-touched their partitions.  Returns the number of CPUs in the mask. */
#ifdef __linux__
static cpu_set_t g_saved_mask;
static int g_have_saved_mask = 0;
#endif
int oracle_bind_threads(int threads) {
#if defined(__linux__) && defined(_OPENMP)
  cpu_set_t mask;
  if (sched_getaffinity(0, sizeof mask, &mask) != 0) return -1;
  if (!g_have_saved_mask) { g_saved_mask = mask; g_have_saved_mask = 1; }
  else mask = g_saved_mask;
  int cpus[CPU_SETSIZE], nc = 0;
  for (int c = 0; c < CPU_SETSIZE; ++c)
    if (CPU_ISSET(c, &mask)) cpus[nc++] = c;
  if (nc == 0) return -1;
#pragma omp parallel num_threads(threads > 0 ? threads : 1)
  {
    cpu_set_t one;
    CPU_ZERO(&one);
    CPU_SET(cpus[omp_get_thread_num() % nc], &one);
    sched_setaffinity(0, sizeof one, &one);
  }
  return nc;
#else
  (void)threads;
  return 0;
#endif
}
void oracle_unbind_threads(void) { /* gives the calling (master) thread its original mask back */
#if defined(__linux__) && defined(_OPENMP)
  if (g_have_saved_mask) sched_setaffinity(0, sizeof g_saved_mask, &g_saved_mask);
#endif
}
/* Zero-fills rows*row_bytes at `base` partition by partition in oracle_smooth's thread mapping (first touch). */
void oracle_first_touch(void *base, int64_t rows, int64_t row_bytes, int partitions, int threads) {
  const int P = partitions < 1 ? 1 : partitions;
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(threads > 0 ? threads : 1)
#endif
  for (int p = 0; p < P; ++p) {
    const int64_t lo = (int64_t)(((__int128)p * rows) / P), hi = (int64_t)(((__int128)(p + 1) * rows) / P);
    memset((char *)base + lo * row_bytes, 0, (size_t)((hi - lo) * row_bytes));
  }
}
void oracle_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

int oracle_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
