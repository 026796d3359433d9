// k1_device.cuh -- device helpers shared by the K1 gradient kernels (dense ring, generic, CSR).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/agd_b200.h"
#include "agd_common.cuh"

namespace agd {

// MLUtils.log1pExp [mllib-1.3.0] through libm (kept for the non-logistic callers and as documentation)
__device__ __forceinline__ double log1p_exp(double x) { return x > 0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

// ---- short-dependency-chain fp64 sigmoid / softplus -------------------------------------------
// LogisticGradient needs, per row, 1/(1+exp(margin)) and log1pExp(margin).  Through libm that is
// exp -> (division | exp -> log1p): ~1300 dependent cycles that sit between the two CTA barriers of
// the gradient kernel.  Here both come from ONE e = exp(-|margin|) in (0,1]:
//     u = 1 + e,  q = 1/u,  sigmoid = margin <= 0 ? q : e*q,  log1p(e) = log(u) + (e - (u-1))*q
// with  exp: 32-entry 2^(j/32) table + degree-7 polynomial (Estrin), Cody-Waite reduction;
//       1/u: rcp.approx seed + 2 Newton steps;  log(u): fdlibm's s = f/(2+f) series, Estrin form.
// The q and log chains are independent, so one lane overlaps them.  Accuracy ~2 ulp (4e-16 relative
// on both outputs against a long-double evaluation; libm: 2.6e-16) -- see tests/test_gpu_parity.py; e is right
// into the subnormals (|margin| up to 745.13, then 0), checked row by row in tests/test_k1_exact.py.
static __device__ const double kExp2Tab[32] = {
    1.0, 1.0218971486541166, 1.0442737824274138, 1.0671404006768237, 1.0905077326652577, 1.1143867425958924,
    1.1387886347566916, 1.1637248587775775, 1.189207115002721, 1.215247359980469, 1.2418578120734840,
    1.2690509571917332, 1.2968395546510096, 1.3252366431597413, 1.3542555469368927, 1.3839098819638320,
    1.4142135623730951, 1.4451808069770467, 1.4768261459394993, 1.5091644275934228, 1.5422108254079407,
    1.5759808451078865, 1.6104903319492543, 1.6457554781539650, 1.6817928305074290, 1.7186192981224779,
    1.7562521603732995, 1.7947090750031072, 1.8340080864093424, 1.8741676341103000, 1.9152065613971474,
    1.9571441241754002};

__device__ __forceinline__ double rcp_1to4(double u) {  // u in [1, 4)
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(u));  // ~20 good bits
  double e = fma(-u, y, 1.0);
  y = fma(y, e, y);
  e = fma(-u, y, 1.0);
  return fma(y, e, y);
}

// The evaluation is split so that a kernel can put only what phase 2 needs (the multiplier) between its barriers:
//   logistic_head: e = exp(-|margin|), u = 1 + e, q = 1/u  ->  mult = sigmoid - y        (exp chain + reciprocal)
//   logistic_tail: log1p(e) = log(u) + (e - (u - 1)) * q   ->  loss                      (log chain, off the critical path)
struct LogisticMid { double margin, e, u, q; };

__device__ __forceinline__ double logistic_head(double m, double y, LogisticMid &mid) {
  const double margin = -1.0 * m;
  const double a = fabs(m);
  // e = exp(-a): -a = (32*me + j) * ln2/32 + r
  const double kMagic = 6755399441055744.0, kInv = 46.16624130844683;
  const double kChi = 0.021660849390173098, kClo = 2.325192846878874e-12;  // ln2/32 split, kChi has 33 bits
  const double t = fma(-a, kInv, kMagic);
  const double nf = t - kMagic;
  const int n = __double2loint(t);
  double r = fma(nf, -kChi, -a);
  r = fma(nf, -kClo, r);
  const double r2 = r * r, r4 = r2 * r2;
  const double A = fma(r, 1.0 / 6.0, 0.5), B = fma(r, 1.0 / 120.0, 1.0 / 24.0), Cc = fma(r, 1.0 / 5040.0, 1.0 / 720.0);
  const double S = fma(r4, Cc, fma(r2, B, A));
  const double em1 = fma(r2, S, r);
  const double T = kExp2Tab[n & 31];
  double e = fma(T, em1, T);
  // 2^(n >> 5) in two exact steps: one factor would leave the normal range below a ~ 708.4, while the product rounds once,
  // into the subnormals, down to the underflow point a ~ 745.13 (above 746 the reduction itself is out of range)
  const int k1 = (n >> 5) >> 1, k2 = (n >> 5) - k1;
  e *= __longlong_as_double((long long)(k1 + 1023) << 52);
  e *= __longlong_as_double((long long)(k2 + 1023) << 52);
  if (a > 746.0) e = 0.0;
  if (a != a) e = a;  // NaN margin propagates, as it does through Math.exp
  const double u = 1.0 + e;
  const double q = rcp_1to4(u);
  mid.margin = margin; mid.e = e; mid.u = u; mid.q = q;
  const double sig = (margin > 0) ? e * q : q;
  return sig - y;
}

__device__ __forceinline__ double logistic_tail(const LogisticMid &mid, double y) {
  const double e = mid.e, u = mid.u, q = mid.q, margin = mid.margin;
  const double c = e - (u - 1.0);
  const bool big = u > 1.4142135623730951;
  const double f = (big ? u * 0.5 : u) - 1.0;
  const double d2 = 2.0 + f;
  const double rd = rcp_1to4(d2);
  double s = f * rd;
  s = fma(fma(-d2, s, f), rd, s);
  const double z = s * s, w = z * z;
  const double t1 = w * fma(w, fma(w, 1.531383769920937332e-01, 2.222219843214978396e-01), 3.999999999940941908e-01);
  const double t2 = z * fma(w, fma(w, fma(w, 1.479819860511658591e-01, 1.818357216161805012e-01), 2.857142874366239149e-01),
                            6.666666666666735130e-01);
  const double R = t1 + t2;
  const double hfsq = 0.5 * f * f;
  const double kf = big ? 1.0 : 0.0;
  const double logu = kf * 6.93147180369123816490e-01 - ((hfsq - (s * (hfsq + R) + kf * 1.90821492927058770002e-10)) - f);
  const double L = fma(c, q, logu);  // log1p(e)
  const double l1 = (margin > 0) ? margin + L : L;
  return (y > 0) ? l1 : l1 - margin;
}

// mult = 1/(1+exp(margin)) - y ; loss = y > 0 ? log1pExp(margin) : log1pExp(margin) - margin, margin = -m
__device__ __forceinline__ void logistic_eval(double m, double y, double &mult, double &loss) {
  LogisticMid mid;
  mult = logistic_head(m, y, mid);
  loss = logistic_tail(mid, y);
}

// loss'(margin) and loss for one example; `m` = x.w.  Formulas: Gradient.scala of spark-mllib 1.3.0.
__device__ __forceinline__ void loss_eval(int kind, double m, double y, double &mult, double &loss) {
  if (kind == AGD_GRAD_LOGISTIC) {
    logistic_eval(m, y, mult, loss);
  } else if (kind == AGD_GRAD_LEAST_SQUARES) {
    const double diff = m - y;
    mult = 2.0 * diff;
    loss = diff * diff;
  } else if (kind == AGD_GRAD_LEAST_SQUARES_HALF) {
    const double diff = m - y;
    mult = diff;
    loss = diff * diff / 2.0;
  } else {  // hinge
    const double s = 2 * y - 1.0;
    if (1.0 > s * m) {
      mult = -s;
      loss = 1.0 - s * m;
    } else {
      mult = 0.0;
      loss = 0.0;
    }
  }
}

// The 64-bit per-row draw: Philox4x32-10 keyed by `seed`, counter (grow lo, grow hi, 0, stream), output words 0 and 1.
// Streams 1-5 belong to the synthetic generator (synth.cu), 6 to the mini-batch mask, 7 to views.
__device__ __forceinline__ unsigned long long row_draw(unsigned long long seed, long long grow, uint32_t stream) {
  uint32_t c0 = (uint32_t)grow, c1 = (uint32_t)((unsigned long long)grow >> 32), c2 = 0u, c3 = stream;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return ((unsigned long long)c0 << 32) | c1;
}

// Bernoulli row mask of the mini-batch form of runMiniBatchSGD (`data.sample(false, fraction, 42 + i)`):
// row `grow` (global index) is kept iff its stream-6 draw is below `thresh` (= fraction * 2^64; thresh == 0 means
// "no sampling").  Counter-based, so the mask does not depend on how rows are sharded over GPUs.  (Spark's own
// sampler is seeded per partition and is not reproducible either.)
__device__ __forceinline__ bool row_selected(unsigned long long seed, unsigned long long thresh, long long grow) {
  if (thresh == 0ull) return true;
  return row_draw(seed, grow, 6u) < thresh;
}

// Whether row `grow` belongs to the view `f` (agd_set_row_filter): every predicate i must hold on the row's stream-7
// draw u = row_draw(seed_i, grow, 7), i.e. lo_i <= u < hi_i, negated when complemented.  f == nullptr returns before any
// arithmetic, so a call without a view runs the instructions it ran before views existed.  The predicates are read from
// device memory inside the row loop (one rolled loop, L1 hits) rather than held in registers: the callers' register
// budgets stay what they were.
__device__ __forceinline__ bool row_in_view(const RowFilter *f, long long grow) {
  if (f == nullptr) return true;
  const int n = f->n;
  bool keep = true;
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const unsigned long long u = row_draw(f->seed[i], grow, 7u);
    const uint32_t fl = f->flags[i];
    const bool in = ((fl & kRowPredLoEnd) == 0u && u >= f->lo[i]) && ((fl & kRowPredHiEnd) != 0u || u < f->hi[i]);
    keep = keep && (in != ((fl & kRowPredComplement) != 0u));
  }
  return keep;
}

// The row rule of every gradient sweep: inside the view, and kept by the mini-batch mask
__device__ __forceinline__ bool row_kept(unsigned long long seed, unsigned long long thresh, const RowFilter *f,
                                         long long grow) {
  return row_selected(seed, thresh, grow) && row_in_view(f, grow);
}

// A load the compiler may not hoist out of a loop: the intercept of a model, read where a margin needs it (an L1 hit) instead
// of taking a register for the whole row loop of a kernel that has none to spare
__device__ __forceinline__ double ld_volatile_f64(const double *p) {
  double v;
  asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

// Transpose-reduce R per-lane partials across a warp: afterwards every lane holds the warp total of
// row (lane / (32/R)).  R/2 + R/4 + ... + 1 + log2(32/R) 64-bit shuffles instead of 5R.
template <int R>
__device__ __forceinline__ double warp_rows_reduce(double (&p)[R], int lane) {
  int bit = 16;
#pragma unroll
  for (int width = R / 2; width >= 1; width >>= 1, bit >>= 1) {
    const bool up = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < width; ++i) {
      const double send = up ? p[i] : p[i + width];
      const double keep = up ? p[i + width] : p[i];
      p[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
    }
  }
  double tot = p[0];
  for (; bit >= 1; bit >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, bit);
  return tot;
}


}  // namespace agd
