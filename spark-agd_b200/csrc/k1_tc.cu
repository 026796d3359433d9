// k1_tc.cu -- K1 for bf16-stored dense shards: margins on the CUDA cores, X^T r on wgmma (sm_90a).
//
// north_star's split for the bf16 configuration: the row tile is brought in ONCE by TMA tensor copies
// (128B swizzle) and used twice without ever being widened into registers:
//   phase 1 (CUDA cores): m_i = x_i . w  -- the consumer threads stream the 16-row tile out of shared
//           memory, widen bf16 on the fly and FMA into row accumulators; nothing is retained, so the loop
//           runs at streaming speed;
//   scalar  (1 dedicated warp): margins -> loss', loss (k1_device.cuh); r_i = loss'_i is split into three
//           bf16 pieces (hi / mid / lo, 24 mantissa bits) that form the B operand [K=16 rows x N columns];
//   phase 2 (wgmma, fp32 in registers): D (64 features x N) = A (X^T block, MN-major view of the SAME swizzled
//           tile) * B, two wgmma.m64nNk16 per 128 features, issued by one warpgroup; each result (a sum over
//           the tile's 16 rows) is added into fp64 registers right away.
// The pieces are replicated across B's columns so that every lane of the accumulator fragment holds hi, mid
// and lo of its own two features (column 2j: hi, 2j+1: mid, 8+2j: lo for lane j of a quad): no shuffles.
// Roles: warps 0-15 consumers, warp 16 TMA producer, warp 18 scalar, warps 20-23 the MMA warpgroup that owns
// the fp64 gradient; setmaxnreg moves registers from the consumers/aux warps to the MMA warpgroup.  Shared-memory
// ring of groups of gb blocks of [16 rows][64 features] (gb = the largest even divisor of d / 64 that is <= 8, so a tile is
// a whole number of groups for every role); a group is released once the wgmmas reading it
// have completed in all four MMA warps.
// Accuracy (per element; DESIGN.md section 4, tests/k1_reference.py): |dg_j| <= [sum_i |x_ij| (lambda eps_i + 2^-20 |r_i|)] / n
// (+ rows at the hinge kink), eps_i = 2^-20 sum_j |x_ij w_j| with fp32 margins.  r of each tile is scaled by a power of two
// before the split, so this holds for every finite r while |x| <= 2^100; fp32 margins need |x_ij w_j| and their partial
// sums inside fp32's exponent range.  Measured on an H100 80GB HBM3 at 400 W: at most 0.064 of the gradient bound.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agd_common.cuh"
#include "k1_device.cuh"

namespace agd {

namespace {

constexpr int kKR = 16;            // rows per tile = K of one MMA
// RPT = rows per consumer thread.  RPT = 2: 512 consumers (+ 256 aux/MMA threads, setmaxnreg 64/56/168 out of the 80 at
// launch).  RPT = 4: 256 consumers, each w value fetched from shared memory serves four rows instead of two -- the kernel is
// bound by shared-memory bandwidth (TMA writes + MMA operand reads + x reads + w reads), and w is the largest reader.
// MMA warpgroup: 80 at launch + everything released by 512 consumers (16 each) and 128 aux threads (24 each)
constexpr int kRegsConsumer = 64, kRegsAux = 56, kRegsMma = 168;
constexpr int kBlockBytes = kKR * 128;     // one [16 rows][64 features] swizzled block
constexpr int kBBytes = 1024;              // one B operand buffer: [N <= 24 columns][16 rows] bf16, K-major, no swizzle
constexpr int kScaleOff = 768;             // ... followed by the tile's scale factor 2^s per point (2 doubles), which no MMA reads

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
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
__device__ __forceinline__ void named_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_tile_2d(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_tile_3d(uint32_t dst, const CUtensorMap *map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
               "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
               : "memory");
}
// sm_90 shared-memory matrix descriptor: start, leading / stride byte offsets (16-byte units), layout type in bits 62-63
__device__ __forceinline__ uint64_t gmma_desc(uint32_t addr, uint32_t lbo, uint32_t sbo, uint64_t layout) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32) | (layout << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N] = A[64 x 16] * B[16 x N], bf16 in, fp32 out (scale-d = 0: nothing is accumulated); A MN-major (transposed)
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);
template <>
__device__ __forceinline__ void wgmma_bf16<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, 0, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 1, 0; }"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(adesc), "l"(bdesc)
               : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<24>(float (&d)[12], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, 0, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, %12, %13, p, 1, 1, 1, 0; }"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
               : "l"(adesc), "l"(bdesc)
               : "memory");
}

// MMA warpgroup: adds the owned feature's hi + mid + lo (and hi2 + mid2 + lo2) of a 128-feature pair into fp64, undoing the
// tile's power-of-two scaling of r (sc[0] = 2^s; sc[1] at the second point).  Fragment index for row-half 0
// (row-half 1: + 2): hi 0, mid 1, lo 4, hi2 5, mid2 8, lo2 9.
template <int N, bool TWO>
__device__ __forceinline__ void mma_accumulate(const float (&e)[2][N / 2], int hb, int hs, const double (&sc)[2], double &g,
                                               double *g2) {
  float v[6];
#pragma unroll
  for (int t = 0; t < (TWO ? 6 : 3); ++t) {
    const int i = t == 0 ? 0 : t == 1 ? 1 : t == 2 ? 4 : t == 3 ? 5 : t == 4 ? 8 : 9;
    const float x0 = hs ? e[0][i + 2] : e[0][i], x1 = hs ? e[1][i + 2] : e[1][i];
    v[t] = hb ? x1 : x0;
  }
  g += (((double)v[0] + (double)v[1]) + (double)v[2]) * sc[0];
  if (TWO) *g2 += (((double)v[3] + (double)v[4]) + (double)v[5]) * sc[1];
}
// 2^k for -1022 <= k <= 1023
__device__ __forceinline__ double pow2i(int k) { return __longlong_as_double((long long)(k + 1023) << 52); }
// the ring group may be refilled once all four MMA warps are done with it
__device__ __forceinline__ void mma_release(uint32_t empty_bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(empty_bar);
}

struct TcLayout {
  uint32_t ring_off, w_off, b2_off, partial_off, bars_off, g2_off, total;
};
// g2: the fp64 gradient at the second point of the two-gradient form (one owner thread per entry)
__host__ __device__ inline TcLayout tc_layout(int ring_groups, int group_bytes, int d, bool two_gradient) {
  TcLayout L;
  L.ring_off = 0;
  L.w_off = (uint32_t)ring_groups * group_bytes;
  L.b2_off = L.w_off + (uint32_t)d * 8;
  L.partial_off = L.b2_off + 2 * kBBytes;
  L.bars_off = L.partial_off + 2 * kKR * 16 * 8;
  L.g2_off = L.bars_off + (2 * (uint32_t)ring_groups + 8) * 8;
  L.total = L.g2_off + (two_gradient ? (uint32_t)d * 8 : 0u);
  return L;
}

struct TcArgs {
  const double *labels;
  const double *w;
  const double *w2;  // optional second point (loss only): pass fusion on the bf16 path (fp32-margin mapping)
  double *slabs;
  long long rows;
  int d, kind, slab_stride;
  unsigned long long sample_seed, sample_thresh;
  long long row_base;
  int gb;           // 64-feature blocks per ring group: the largest even divisor of d / 64 that is <= 8
  int ngt;          // groups per tile = d / (64 * gb)
  int ring_groups;  // ring capacity in groups
  int one_copy;     // 1: a ring group arrives as ONE 3-D TMA copy [gb blocks][16 rows][64 features] instead of gb 2-D copies
  int diag;         // option k1_diag: 100 = consumers skip the arithmetic, 101 = the MMAs are not issued (timing bisection only)
};

// RPT = 0 selects the row-per-lane consumer mapping: a warp covers all 16 rows of the tile for two adjacent 8-feature chunks,
// so its w reads are broadcasts (one shared-memory wavefront instead of four) and each lane owns one row's partial dot.
__host__ __device__ constexpr int tc_consumers(int rpt) { return rpt == 4 ? 256 : 512; }
// fp32 FMA on a packed pair: d.{x,y} = a.{x,y} * b.{x,y} + c.{x,y}, two round-to-nearest FMAs
__device__ __forceinline__ unsigned long long ffma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  const float x = __fmaf_rn(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)c));
  const float y = __fmaf_rn(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)),
                            __uint_as_float((uint32_t)(c >> 32)));
  return ((unsigned long long)__float_as_uint(y) << 32) | __float_as_uint(x);
}
__device__ __forceinline__ unsigned long long pack2(uint32_t lo, uint32_t hi) {
  unsigned long long d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}

// F32: phase 1 in fp32 (option tc_margins=f32, the default): a bf16 is the upper half of an fp32, so widening is one ALU op
// and there is no fp64 conversion per element; products are accumulated by fp32 FMAs on packed pairs over at most 8 terms per
// accumulator and then added into the fp64 row sums.  Margins carry ~2^-23 relative to sum |x_i w_i| (w rounded to fp32) --
// the same class as the gradient of this kernel (bf16 x 3 split, fp32 tensor-core sums).  F32 = false keeps fp64-exact margins.
// DUAL (F32 mapping only): the loss is also evaluated at a second point w2 from the same tile -- one more packed FMA per
// feature pair in phase 1, lanes 16-31 of the scalar warp -- with bits identical to a launch of its own at w2.
// DUAL == 2: the GRADIENT at w2 as well (two-gradient sweep): r at w2 takes columns 2j+9, 16+2j and 17+2j of a 24-column B
// operand (hi2, mid2, lo2 for lane j of a quad), so the second X^T r costs no extra MMA instruction; its fp64 gradient
// lives in shared memory (g2), each entry owned by the one MMA thread that updates it.
template <int RPT, bool F32, int DUAL = 0>
__global__ void __launch_bounds__(tc_consumers(RPT) + 256, 1)
k1_tc_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap3, const TcArgs a,
             const long long ntiles) {
  constexpr int kConsumers = tc_consumers(RPT);   // RPT > 0: 64 threads (one 16-byte vector each) per group row
  constexpr int kThreads = kConsumers + 256;   // + warpgroup (producer, idle, scalar, idle) + MMA warpgroup
  constexpr int kN = DUAL == 2 ? 24 : 16;      // B columns: (hi, mid) x 4, (lo, hi2) x 4 [, (mid2, lo2) x 4]
  constexpr int kCW = kConsumers / 32;         // consumer warps; the aux warps follow
  constexpr bool kRepartition = RPT != 4;      // 768 threads start with 80 registers: move some to the flush warpgroup
  extern __shared__ __align__(1024) unsigned char smem[];
  const int group_bytes = a.gb * kBlockBytes;
  const TcLayout L = tc_layout(a.ring_groups, group_bytes, a.d, DUAL == 2);
  double *w_s = reinterpret_cast<double *>(smem + L.w_off);
  unsigned char *b2 = smem + L.b2_off;                                       // [2][kBBytes]
  double *partial = reinterpret_cast<double *>(smem + L.partial_off);         // [2][16 rows][2] (RPT > 0) or [2][16 rows][16 warps]
  const uint32_t bars = smem_u32(smem + L.bars_off);
  const int RG = a.ring_groups;
  // full[g] = bars + 8g ; empty[g] = bars + 8(RG+g) ; then wbar, b2_full[2], b2_empty[2]
  const uint32_t wbar = bars + 16u * RG, b2_full = wbar + 8, b2_empty = b2_full + 16;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long my_tiles = (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const int npairs = a.d / 128;   // 128-feature pairs of 64-feature blocks
  double *slab = a.slabs + (size_t)blockIdx.x * a.slab_stride;

  if (tid == 0) {
    for (int g = 0; g < RG; ++g) {
      mbar_init(bars + 8u * g, 1);
      mbar_init(bars + 8u * (RG + g), 4);   // one arrival per MMA warp
    }
    mbar_init(wbar, 1);
    mbar_init(b2_full, 1); mbar_init(b2_full + 8, 1);
    mbar_init(b2_empty, 4); mbar_init(b2_empty + 8, 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // B operand columns nobody writes (2j+9 without a second gradient) stay zero for the whole kernel
  for (int i = tid; i < 2 * kBBytes / 4; i += kThreads) reinterpret_cast<uint32_t *>(b2)[i] = 0u;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  if (warp >= kCW && warp < kCW + 4) {
   if (kRepartition) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsAux));
   if (warp == kCW) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(wbar, (uint32_t)a.d * 8u);
      tma_bulk_g2s(smem_u32(w_s), a.w, (uint32_t)a.d * 8u, wbar);
      int slot = -1;
      uint32_t epar = 0;   // parity of the PREVIOUS use of a slot's empty barrier
      bool wrapped = false;
      for (long long k = 0; k < my_tiles; ++k) {
        const long long row0 = (blockIdx.x + k * (long long)gridDim.x) * kKR;
        for (int gi = 0; gi < a.ngt; ++gi) {
          if (++slot == RG) { slot = 0; if (wrapped) epar ^= 1u; wrapped = true; }
          if (wrapped) mbar_wait(bars + 8u * (RG + slot), epar);
          const uint32_t full = bars + 8u * slot;
          mbar_expect_tx(full, (uint32_t)group_bytes);  // rows past the shard are zero-filled by TMA
          if (a.one_copy) {
            tma_tile_3d(smem_u32(smem + (size_t)slot * group_bytes), &tmap3, 0, (int)row0, gi * a.gb, full);
          } else {
            for (int b = 0; b < a.gb; ++b)
              tma_tile_2d(smem_u32(smem + (size_t)slot * group_bytes + b * kBlockBytes), &tmap, (gi * a.gb + b) * 64, (int)row0, full);
          }
        }
      }
    }
   } else if (warp == kCW + 2) {
    // ===================== scalar warp =====================
    // lanes 0-15: the tile's rows at w (loss', loss); DUAL: lanes 16-31 the same rows at w2 (loss only)
    double lossacc = 0.0, cntacc = 0.0;
    double ynext = 0.0;
    const int srow = lane & 15;
    const bool second = DUAL && lane >= kKR;
    if (lane < kKR || DUAL) {
      const long long r = (long long)blockIdx.x * kKR + srow;
      if (r < a.rows) ynext = a.labels[r];
    }
    const double *partial2 = partial + 2 * kKR * 2;   // [2][16 rows][2] at w2 (RPT = 2 layout)
    for (long long k = 0; k < my_tiles; ++k) {
      const int bb = (int)(k & 1);
      const long long tile = blockIdx.x + k * (long long)gridDim.x;
      const long long left = a.rows - tile * kKR;
      const int rv = left < kKR ? (int)left : kKR;
      const double ylab = ynext;
      if (lane < kKR || DUAL) {
        const long long r = (tile + gridDim.x) * kKR + srow;
        if (r < a.rows) ynext = a.labels[r];
      }
      named_sync(1 + bb, kConsumers + 32);                     // partial dots of tile k are in shared memory
      double mult = 0.0;
      bool nonfinite = false;   // a non-finite margin at a point whose gradient this launch forms
      if (lane < kKR || second) {
        double m;
        if (RPT) {
          const double *pp = second ? partial2 : partial;
          m = pp[(bb * kKR + srow) * 2] + pp[(bb * kKR + srow) * 2 + 1];
        } else {  // one partial per consumer warp, fixed tree
          const double *pp = partial + (bb * kKR + lane) * 16;
          m = (((pp[0] + pp[1]) + (pp[2] + pp[3])) + ((pp[4] + pp[5]) + (pp[6] + pp[7]))) +
              (((pp[8] + pp[9]) + (pp[10] + pp[11])) + ((pp[12] + pp[13]) + (pp[14] + pp[15])));
        }
        nonfinite = (lane < kKR || DUAL == 2) && srow < rv && !isfinite(m);
        double mu, loss;
        loss_eval(a.kind, m, ylab, mu, loss);
        if (srow < rv && row_selected(a.sample_seed, a.sample_thresh, a.row_base + tile * kKR + srow)) {
          mult = mu; lossacc += loss; cntacc += 1.0;
        }
      }
      named_arrive(3 + bb, kConsumers + 32);                   // partial[bb] may be overwritten
      // r of the tile is split after scaling by 2^-s, s = the exponent of max |r| over its 16 rows (per point): the pieces
      // and the fp32 sums then stay in range for every finite r as long as |x| <= 2^100 (16 x 2^100 < 2^127).  Scaling by a
      // power of two is exact, so in-range tiles give the bits of the unscaled split.
      // The largest exponent field of the tile (high word of |r|, one warp reduction per point) gives s with
      // max |r| 2^-s in [0.5, 1): s = E - 1022; a subnormal maximum takes s = -1022, inf / NaN s = 0.
      // A row whose multiplier is exactly 0 adds nothing (netlib DAXPY returns when DA == 0), but the MMA would form 0 * inf =
      // NaN from it.  A finite margin means every feature of the row is finite, so only rows with a non-finite margin and
      // multiplier 0 are flagged, and their 128-byte lines in every group of tile k are zeroed before the MMAs read the tile.
      // All groups of tile k are still resident: the MMA warps release a group only after reading it, which waits for b2_full.
      // With a second gradient the tile is shared by both points: only rows flagged at both are zeroed (DESIGN.md section 4).
      // A non-finite margin rides in bit 31 of the exponent reduction, so tiles without one run no extra warp-wide operation.
      const uint32_t hw = (uint32_t)__double2hiint(mult) & 0x7fffffffu;
      const uint32_t hwf = hw | (nonfinite ? 0x80000000u : 0u);
      uint32_t top = __reduce_max_sync(0xffffffffu, lane < kKR ? hwf : 0u), top2 = 0u;
      if (DUAL == 2) top2 = __reduce_max_sync(0xffffffffu, lane < kKR ? 0u : hwf);
      if ((top | top2) >> 31) {   // rare: the exponents again without the flag, then the rows to zero
        top = __reduce_max_sync(0xffffffffu, lane < kKR ? hw : 0u);
        if (DUAL == 2) top2 = __reduce_max_sync(0xffffffffu, lane < kKR ? 0u : hw);
        const uint32_t fl = __ballot_sync(0xffffffffu, nonfinite && mult == 0.0);
        const uint32_t zero_rows = DUAL == 2 ? (fl & (fl >> 16) & 0xffffu) : fl;
        // every role walks the ring in the same order: tile k's groups sit in slots (k ngt + gi) mod RG.  Lane = (block of the
        // group, 16-byte chunk): the 128B swizzle only permutes the chunks within a row's line.  Rolled loops keep this rare
        // path from taking registers from the scalar warp's loop (an out-of-line call cost 0.3% of K1 time at d = 1024, H100
        // 80GB HBM3 at 700 W).
        const int slot0 = (int)((k * a.ngt) % RG);
#pragma unroll 1
        for (uint32_t rows = zero_rows; rows; rows &= rows - 1u) {
          const int zr = __ffs(rows) - 1;
          int sl = slot0;
#pragma unroll 1
          for (int gi = 0; gi < a.ngt; ++gi) {
#pragma unroll 1
            for (int c = lane; c < a.gb * 8; c += 32)
              *reinterpret_cast<uint4 *>(smem + sl * group_bytes + (c >> 3) * kBlockBytes + zr * 128 + (c & 7) * 16) =
                  make_uint4(0u, 0u, 0u, 0u);
            if (++sl == RG) sl = 0;
          }
        }
      }
      uint32_t E = top >> 20;
      if (DUAL == 2 && second) E = top2 >> 20;
      // (s = 1024 is taken as 1023, max |r| 2^-s in [1, 2): then 2^s is a normal double and one DMUL undoes it)
      const int s = E == 0x7ffu ? 0 : E == 0u ? -1022 : E == 0x7feu ? 1023 : (int)E - 1022;
      const int ns = -s;
      const double ms = (mult * pow2i(ns >> 1)) * pow2i(ns - (ns >> 1));
      if (k >= 2) mbar_wait(b2_empty + 8u * bb, (uint32_t)(((k >> 1) - 1) & 1));  // MMAs of tile k-2 have read b2[bb]
      if (srow == 0 && (lane < kKR || (DUAL == 2 && second))) {
        reinterpret_cast<double *>(b2 + bb * kBBytes + kScaleOff)[second ? 1 : 0] = pow2i(s);
      }
      if (lane < kKR || (DUAL == 2 && second)) {
        // r_i 2^-s -> three bf16 pieces, each written to four columns of the K-major B operand: element (n, row) sits at
        // (n / 8) * 256 + (row / 8) * 128 + (n % 8) * 16 + (row % 8) * 2.  At w: hi -> 2t, mid -> 2t+1, lo -> 8+2t;
        // at w2: hi2 -> 9+2t, mid2 -> 16+2t, lo2 -> 17+2t (t = 0..3)
        const __nv_bfloat16 hi = __double2bfloat16(ms);
        const double r1 = ms - (double)__bfloat162float(hi);
        const __nv_bfloat16 mid = __double2bfloat16(r1);
        const double r2 = r1 - (double)__bfloat162float(mid);
        const __nv_bfloat16 lo = __double2bfloat16(r2);
        const int n0 = second ? 9 : 0, n1 = second ? 16 : 1, n2 = second ? 17 : 8;
        unsigned char *base = b2 + bb * kBBytes + (srow / 8) * 128 + (srow % 8) * 2;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int c0 = n0 + 2 * t, c1 = n1 + 2 * t, c2 = n2 + 2 * t;
          *reinterpret_cast<__nv_bfloat16 *>(base + (c0 / 8) * 256 + (c0 % 8) * 16) = hi;
          *reinterpret_cast<__nv_bfloat16 *>(base + (c1 / 8) * 256 + (c1 % 8) * 16) = mid;
          *reinterpret_cast<__nv_bfloat16 *>(base + (c2 / 8) * 256 + (c2 % 8) * 16) = lo;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(b2_full + 8u * bb);
    }
    // DUAL: skipping the xor-16 step keeps the lane-0 / lane-16 totals bit-identical to a one-point launch at either point
    // (whose lanes >= 16 only ever contribute exact zeros)
    for (int off = DUAL ? 8 : 16; off >= 1; off >>= 1) {
      lossacc += __shfl_xor_sync(0xffffffffu, lossacc, off);
      cntacc += __shfl_xor_sync(0xffffffffu, cntacc, off);
    }
    if (lane == 0) { slab[a.d] = lossacc; slab[a.d + 1] = cntacc; if (!DUAL) { slab[a.d + 2] = 0.0; slab[a.d + 3] = 0.0; } }
    if (DUAL && lane == kKR) {
      slab[a.d + 2] = lossacc; slab[a.d + 3] = cntacc;
      if (DUAL == 2) {   // second block: [gradient at w2 | loss sum | count | 0 | 0]
        double *slab2 = slab + a.d + 4;
        slab2[a.d] = lossacc; slab2[a.d + 1] = cntacc; slab2[a.d + 2] = 0.0; slab2[a.d + 3] = 0.0;
      }
    }
   }
  } else if (warp >= kCW + 4) {
    // ===================== MMA warpgroup: X^T r on wgmma, owns the fp64 gradient(s) =====================
    if (kRepartition) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegsMma));
    const int mw = warp - (kCW + 4);   // warp of the warpgroup (kCW + 4 is a multiple of 4)
    const int q = lane >> 2, j = lane & 3;
    // accumulator fragment of wgmma.m64nNk16: lane (q, j) of warp mw holds rows 16 mw + q and 16 mw + q + 8 (features of the
    // 64-feature block), columns {2j, 2j+1} + 8i.  Within a 128-feature pair, this thread owns block (j >> 1), row-half (j & 1).
    const int hb = j >> 1, hs = j & 1;
    const int fo = 64 * hb + 16 * mw + q + 8 * hs;
    double gacc[32];                // feature 128 p + fo, p < d / 128
#pragma unroll
    for (int p = 0; p < 32; ++p) gacc[p] = 0.0;
    double *g2 = reinterpret_cast<double *>(smem + L.g2_off);   // DUAL == 2: the gradient at w2
    if (DUAL == 2)
      for (int p = 0; p < npairs; ++p) g2[128 * p + fo] = 0.0;
    const int hp = a.gb / 2;        // pairs per ring group
    int slot = -1;
    uint32_t par = 1;
    float acc[2][kN / 2];           // [block of the pair][fragment]
    for (long long k = 0; k < my_tiles; ++k) {
      const int bb = (int)(k & 1);
      mbar_wait(b2_full + 8u * bb, (uint32_t)((k >> 1) & 1));
      const uint64_t bdesc = gmma_desc(smem_u32(b2 + bb * kBBytes), 128, 256, 0);   // K-major, no swizzle
      const double *scs = reinterpret_cast<const double *>(b2 + bb * kBBytes + kScaleOff);
      const double sc[2] = {scs[0], DUAL == 2 ? scs[1] : 1.0};
#pragma unroll
      for (int p = 0; p < 32; ++p) {
        if (p < npairs) {
          const int pg = p % hp;
          if (pg == 0) {
            if (++slot == RG) slot = 0;
            if (slot == 0) par ^= 1u;
            mbar_wait(bars + 8u * slot, par);
          }
          const uint32_t a0 = smem_u32(smem + (size_t)slot * group_bytes + (2 * pg) * kBlockBytes);
          wgmma_fence();
          if (a.diag != 101) {
            // A: [64 features][16 rows] MN-major, 128B swizzle, 8-row groups 1024 B apart
            wgmma_bf16<kN>(acc[0], gmma_desc(a0, kBlockBytes, 1024, 1), bdesc);
            wgmma_bf16<kN>(acc[1], gmma_desc(a0 + kBlockBytes, kBlockBytes, 1024, 1), bdesc);
          }
          wgmma_commit();
          wgmma_wait<0>();
          mma_accumulate<kN, DUAL == 2>(acc, hb, hs, sc, gacc[p], g2 + 128 * p + fo);
          if (pg == hp - 1) mma_release(bars + 8u * (RG + slot), lane);   // last pair of the group
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(b2_empty + 8u * bb);   // B[bb] may be rewritten (tile k + 2)
    }
#pragma unroll
    for (int p = 0; p < 32; ++p)
      if (p < npairs) {
        slab[128 * p + fo] = gacc[p];
        if (DUAL == 2) slab[a.d + 4 + 128 * p + fo] = g2[128 * p + fo];
      }
  } else {
    // ===================== consumers: phase 1 in fp64, straight out of the swizzled tile =====================
    if (kRepartition) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsConsumer));
    if constexpr (RPT == 0) {
      const int r = lane & 15, hsel = lane >> 4;
      mbar_wait(wbar, 0);
      int slot = -1;
      uint32_t par = 1;
      const int npairs = a.gb * 4;                       // pairs of adjacent 8-feature chunks per ring group
      // this lane's chunk in task j: c = 2 * (warp + 16 j) + hsel; block c >> 3, 16-byte position (c & 7) ^ (row & 7)
      uint32_t x_off[2];
      int w_off[2];
      bool act[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = 2 * (warp + 16 * j) + hsel;
        act[j] = warp + 16 * j < npairs;
        x_off[j] = (uint32_t)((c >> 3) * kBlockBytes + r * 128 + (((c & 7) ^ (r & 7)) << 4));
        w_off[j] = c * 8;
      }
      for (long long k = 0; k < my_tiles; ++k) {
        const int bb = (int)(k & 1);
        double pa[2] = {0.0, 0.0}, pb[2] = {0.0, 0.0};
        const double *wp = w_s;
        for (int gi = 0; gi < a.ngt; ++gi) {
          if (++slot == RG) slot = 0;
          if (slot == 0) par ^= 1u;
          mbar_wait(bars + 8u * slot, par);
          if (a.diag != 100) {
            const unsigned char *gbase = smem + (uint32_t)slot * (uint32_t)group_bytes;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              if (act[j]) {
                const uint4 xr = *reinterpret_cast<const uint4 *>(gbase + x_off[j]);
                const double2 *wv = reinterpret_cast<const double2 *>(wp + w_off[j]);   // the same address on 16 lanes
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const double2 wq = wv[q];
                  const uint32_t xw = q == 0 ? xr.x : q == 1 ? xr.y : q == 2 ? xr.z : xr.w;
                  pa[j] = fma((double)__uint_as_float(xw << 16), wq.x, pa[j]);
                  pb[j] = fma((double)__uint_as_float(xw & 0xffff0000u), wq.y, pb[j]);
                }
              }
            }
          }
          wp += a.gb * 64;
        }
        double p = (pa[0] + pb[0]) + (pa[1] + pb[1]);
        p += __shfl_xor_sync(0xffffffffu, p, 16);              // the two chunk columns of the warp
        if (k >= 2) named_sync(3 + bb, kConsumers + 32);         // scalar warp is done with partial[bb] of tile k-2
        if (lane < 16) partial[(bb * kKR + r) * 16 + warp] = p;
        named_arrive(1 + bb, kConsumers + 32);
      }
    } else {
    constexpr int kSlots = kKR / (RPT ? RPT : 1);   // thread (rq, vv) handles rows rq, rq + kSlots, ... of every tile
    const int rq = tid >> 6;
    const int vv = tid & 63;        // 16-byte vector within the group row
    mbar_wait(wbar, 0);
    int slot = -1;
    uint32_t par = 1;               // ring slot and its mbarrier phase, kept incrementally
    const int blk = vv >> 3, ch = vv & 7;
    const bool active = vv < a.gb * 8;
    uint32_t x_off[RPT];            // row rq + j * kSlots of a block: 128-byte rows, 16-byte chunks XOR-swizzled by (row & 7)
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int row = rq + j * kSlots;
      x_off[j] = (uint32_t)(blk * kBlockBytes + row * 128 + ((ch ^ (row & 7)) << 4));
    }
    if constexpr (F32) {
      // one-time re-layout of w, in place through registers: fp64 (as TMA delivered it) -> fp32 PLANES.  Chunk c (8 features)
      // keeps features 0-3 at plane0[c] and 4-7 at plane1[c] (16 bytes each), so both per-group reads of a warp are
      // contiguous LDS.128s.  The fp64 copy is dead afterwards (the planes overwrite its first half).
      const int nchunks = a.d / 8;
      float4 lo4[2], hi4[2], lo4b[2], hi4b[2];   // d <= 4096: at most 2 chunks per consumer thread
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = tid + i * kConsumers;
        if (c < nchunks) {
          const double *src = w_s + (size_t)c * 8;
          lo4[i] = make_float4((float)src[0], (float)src[1], (float)src[2], (float)src[3]);
          hi4[i] = make_float4((float)src[4], (float)src[5], (float)src[6], (float)src[7]);
          if (DUAL) {   // w2 comes straight from global memory (L2): once per CTA
            const double *s2 = a.w2 + (size_t)c * 8;
            lo4b[i] = make_float4((float)s2[0], (float)s2[1], (float)s2[2], (float)s2[3]);
            hi4b[i] = make_float4((float)s2[4], (float)s2[5], (float)s2[6], (float)s2[7]);
          }
        }
      }
      named_sync(5, kConsumers);
      // planes of w in the first half of the staging area, of w2 in the second half (the fp64 copy of w is dead by now)
      float4 *plane0 = reinterpret_cast<float4 *>(w_s), *plane1 = plane0 + nchunks;
      float4 *plane0b = plane1 + nchunks, *plane1b = plane0b + nchunks;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = tid + i * kConsumers;
        if (c < nchunks) {
          plane0[c] = lo4[i]; plane1[c] = hi4[i];
          if (DUAL) { plane0b[c] = lo4b[i]; plane1b[c] = hi4b[i]; }
        }
      }
      named_sync(5, kConsumers);
      double *partial2 = partial + 2 * kKR * 2;
      for (long long k = 0; k < my_tiles; ++k) {
        const int bb = (int)(k & 1);
        double pd[RPT], pd2[RPT];
        unsigned long long acc[RPT], acc2[RPT];     // packed fp32 pair: even / odd features of this thread's chunk
#pragma unroll
        for (int j = 0; j < RPT; ++j) { pd[j] = 0.0; acc[j] = 0ull; pd2[j] = 0.0; acc2[j] = 0ull; }
        const ulonglong2 *wp0 = reinterpret_cast<const ulonglong2 *>(plane0) + vv;
        const ulonglong2 *wp1 = reinterpret_cast<const ulonglong2 *>(plane1) + vv;
        const ulonglong2 *wq0 = reinterpret_cast<const ulonglong2 *>(plane0b) + vv;
        const ulonglong2 *wq1 = reinterpret_cast<const ulonglong2 *>(plane1b) + vv;
        for (int gi = 0; gi < a.ngt; ++gi) {
          if (++slot == RG) slot = 0;
          if (slot == 0) par ^= 1u;
          mbar_wait(bars + 8u * slot, par);
          if (active && a.diag != 100) {
            const unsigned char *gbase = smem + (uint32_t)slot * (uint32_t)group_bytes;
            uint4 xr[RPT];
#pragma unroll
            for (int j = 0; j < RPT; ++j) xr[j] = *reinterpret_cast<const uint4 *>(gbase + x_off[j]);
            const ulonglong2 wa = *wp0, wb = *wp1;   // (w0,w1),(w2,w3) and (w4,w5),(w6,w7) as packed fp32 pairs
            ulonglong2 va = wa, vb = wb;
            if (DUAL) { va = *wq0; vb = *wq1; }
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
              const unsigned long long x0 = pack2(xr[j].x << 16, xr[j].x & 0xffff0000u), x1 = pack2(xr[j].y << 16, xr[j].y & 0xffff0000u),
                                       x2 = pack2(xr[j].z << 16, xr[j].z & 0xffff0000u), x3 = pack2(xr[j].w << 16, xr[j].w & 0xffff0000u);
              acc[j] = ffma2(x0, wa.x, acc[j]);
              acc[j] = ffma2(x1, wa.y, acc[j]);
              acc[j] = ffma2(x2, wb.x, acc[j]);
              acc[j] = ffma2(x3, wb.y, acc[j]);
              if (DUAL) {
                acc2[j] = ffma2(x0, va.x, acc2[j]);
                acc2[j] = ffma2(x1, va.y, acc2[j]);
                acc2[j] = ffma2(x2, vb.x, acc2[j]);
                acc2[j] = ffma2(x3, vb.y, acc2[j]);
              }
            }
          }
          wp0 += a.gb * 8;
          wp1 += a.gb * 8;
          wq0 += a.gb * 8;
          wq1 += a.gb * 8;
          if ((gi & 1) || gi + 1 == a.ngt) {   // at most 8 products per fp32 accumulator, then exact fp64
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
              pd[j] += (double)(__uint_as_float((uint32_t)acc[j]) + __uint_as_float((uint32_t)(acc[j] >> 32)));
              acc[j] = 0ull;
              if (DUAL) {
                pd2[j] += (double)(__uint_as_float((uint32_t)acc2[j]) + __uint_as_float((uint32_t)(acc2[j] >> 32)));
                acc2[j] = 0ull;
              }
            }
          }
        }
        const double tot = warp_rows_reduce<RPT>(pd, lane);
        double tot2 = 0.0;
        if (DUAL) tot2 = warp_rows_reduce<RPT>(pd2, lane);
        if (k >= 2) named_sync(3 + bb, kConsumers + 32);         // scalar warp is done with partial[bb] of tile k-2
        if ((lane & (32 / RPT - 1)) == 0) {
          partial[(bb * kKR + rq + kSlots * (lane / (32 / RPT))) * 2 + (warp & 1)] = tot;
          if (DUAL) partial2[(bb * kKR + rq + kSlots * (lane / (32 / RPT))) * 2 + (warp & 1)] = tot2;
        }
        named_arrive(1 + bb, kConsumers + 32);
      }
    } else {
    // one-time re-layout of w: within each 64-byte chunk c (8 features) swap the four 16-byte pairs j -> j ^ ((c>>1)&3)
    for (int c = tid; c < a.d / 8; c += kConsumers) {
      const int f = (c >> 1) & 3;
      if (f) {
        double2 *blk = reinterpret_cast<double2 *>(w_s + (size_t)c * 8);
        const double2 t0 = blk[0], t1 = blk[1], t2 = blk[2], t3 = blk[3];
        const double2 v[4] = {t0, t1, t2, t3};
        blk[0 ^ f] = v[0]; blk[1 ^ f] = v[1]; blk[2 ^ f] = v[2]; blk[3 ^ f] = v[3];
      }
    }
    named_sync(5, kConsumers);
    const int sw = (lane >> 1) & 3;
    for (long long k = 0; k < my_tiles; ++k) {
      const int bb = (int)(k & 1);
      double pa[RPT], pb[RPT];
#pragma unroll
      for (int j = 0; j < RPT; ++j) { pa[j] = 0.0; pb[j] = 0.0; }
      const double *wp = w_s + (blk * 64 + ch * 8);
      for (int gi = 0; gi < a.ngt; ++gi) {
        if (++slot == RG) slot = 0;
        if (slot == 0) par ^= 1u;
        mbar_wait(bars + 8u * slot, par);
        if (active && a.diag != 100) {
          const unsigned char *gbase = smem + (uint32_t)slot * (uint32_t)group_bytes;
          uint4 xr[RPT];
#pragma unroll
          for (int j = 0; j < RPT; ++j) xr[j] = *reinterpret_cast<const uint4 *>(gbase + x_off[j]);
          // w was re-laid out once per CTA (above): the 16-byte pair j of chunk c sits at position j ^ ((c >> 1) & 3), so
          // the 8 lanes of a quarter-warp touch 8 different bank groups with no per-element shuffling of the x words
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const double2 wq = *reinterpret_cast<const double2 *>(wp + 2 * (q ^ sw));  // features 2q, 2q+1 of this chunk
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
              const uint32_t xw = q == 0 ? xr[j].x : q == 1 ? xr[j].y : q == 2 ? xr[j].z : xr[j].w;
              pa[j] = fma((double)__uint_as_float(xw << 16), wq.x, pa[j]);
              pb[j] = fma((double)__uint_as_float(xw & 0xffff0000u), wq.y, pb[j]);
            }
          }
        }
        wp += a.gb * 64;
      }
      double p[RPT];
#pragma unroll
      for (int j = 0; j < RPT; ++j) p[j] = pa[j] + pb[j];
      // afterwards the lanes of eighth/half-warp j hold the warp total of row rq + j * kSlots
      const double tot = warp_rows_reduce<RPT>(p, lane);
      if (k >= 2) named_sync(3 + bb, kConsumers + 32);         // scalar warp is done with partial[bb] of tile k-2
      if ((lane & (32 / RPT - 1)) == 0) partial[(bb * kKR + rq + kSlots * (lane / (32 / RPT))) * 2 + (warp & 1)] = tot;
      named_arrive(1 + bb, kConsumers + 32);
    }
    }  // fp64 margins
    }  // column-slice mapping
  }
}

// the opt-in shared-memory size is a per-device property of a function: set it when it changes, not on every launch
// (one static table per call site, i.e. per kernel instantiation)
template <int SITE, typename K>
cudaError_t set_smem_once(K kern, int bytes) {
  static int cur[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && cur[dev] == bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev >= 0 && dev < 64) cur[dev] = bytes;
  return e;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

int k1_tc_supported(int32_t d, int elem_bytes) { return elem_bytes == 2 && d >= 128 && d <= 4096 && d % 128 == 0; }

cudaError_t k1_tc_launch(const K1Args &a, int sm_count, int *blocks_out, cudaStream_t st) {
  if (!k1_tc_supported(a.d, 2)) return cudaErrorInvalidValue;
  if (a.rows <= 0) { *blocks_out = 0; return cudaSuccess; }
  static EncodeTiledFn encode = nullptr;
  if (!encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || !fn) return e != cudaSuccess ? e : cudaErrorUnknown;
    encode = (EncodeTiledFn)fn;
  }
  CUtensorMap tmap;
  const cuuint64_t gdim[2] = {(cuuint64_t)a.d, (cuuint64_t)a.rows};
  const cuuint64_t gstr[1] = {(cuuint64_t)a.d * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)kKR};
  const cuuint32_t estr[2] = {1, 1};
  if (encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(a.X), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorInvalidValue;
  // a tile is a whole number of ring groups, and a group a whole number of 128-feature pairs (d / 64 is even): every role
  // (TMA producer, consumers, MMA warpgroup) then walks the same groups
  const int nblk = a.d / 64;
  int gb = 8;
  while (nblk % gb) gb -= 2;
  CUtensorMap tmap3;
  {
    const cuuint64_t gdim3[3] = {64, (cuuint64_t)a.rows, (cuuint64_t)nblk};
    const cuuint64_t gstr3[2] = {(cuuint64_t)a.d * 2, 128};
    const cuuint32_t box3[3] = {64, (cuuint32_t)kKR, (cuuint32_t)gb};
    const cuuint32_t estr3[3] = {1, 1, 1};
    if (encode(&tmap3, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(a.X), gdim3, gstr3, box3, estr3,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return cudaErrorInvalidValue;
  }
  TcArgs t;
  t.one_copy = a.tune_ctas == 2 ? 0 : 1;   // option ring_ctas=2: one 2-D copy per 64-feature block (slower: 8x the TMA operations)
  t.diag = (a.kind == 100 || a.kind == 101) ? a.kind : 0;
  if (a.w2 && (a.tune_rows != 0 || a.tc_margins_f64)) return cudaErrorInvalidValue;   // two-point form: default mapping only
  t.labels = a.labels; t.w = a.w; t.w2 = a.w2; t.slabs = a.slabs; t.rows = a.rows; t.d = a.d; t.kind = a.kind;
  t.slab_stride = a.slab_stride;
  t.sample_seed = a.sample_seed; t.sample_thresh = a.sample_thresh; t.row_base = a.row_base;
  t.gb = gb;
  t.ngt = nblk / gb;
  const int group_bytes = t.gb * kBlockBytes;
  int ring = a.stages > 0 ? a.stages : 16;
  const bool two_gradient = a.w2 && a.dual_full;
  const uint32_t budget = 227u * 1024u - 2048u;   // H100: 227 KB of shared memory per block
  while (ring > 2 && tc_layout(ring, group_bytes, a.d, two_gradient).total + 1024 > budget) --ring;
  if (ring < t.ngt + 1) ring = t.ngt + 1;  // at least one tile and a bit
  t.ring_groups = ring;
  const TcLayout L = tc_layout(ring, group_bytes, a.d, two_gradient);
  if (L.total + 1024 > budget) return cudaErrorInvalidValue;
  const long long ntiles = (a.rows + kKR - 1) / kKR;
  long long grid = sm_count;
  if (grid > ntiles) grid = ntiles;
  *blocks_out = (int)grid;
  const int smem_bytes = (int)L.total + 1024;
  cudaError_t e;
  if (a.tune_rows == 1) {  // option ring_rows=1: row-per-lane consumers (broadcast w reads; measured slower)
    e = set_smem_once<1>(k1_tc_kernel<0, false, 0>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<0, false, 0><<<(unsigned)grid, 768, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  } else if (a.tune_rows == 4) {  // option ring_rows=4: 256 consumers with four rows each (measured slower)
    e = set_smem_once<2>(k1_tc_kernel<4, false, 0>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<4, false, 0><<<(unsigned)grid, 512, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  } else if (a.tc_margins_f64) {  // option tc_margins=f64: 512 consumers, two rows per thread, fp64-exact margins
    e = set_smem_once<3>(k1_tc_kernel<2, false, 0>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<2, false, 0><<<(unsigned)grid, 768, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  } else if (a.w2 && a.dual_full) {  // the default mapping + loss AND gradient at a second point (speculative sweep)
    e = set_smem_once<6>(k1_tc_kernel<2, true, 2>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<2, true, 2><<<(unsigned)grid, 768, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  } else if (a.w2) {  // the default mapping + the loss at a second point (pass fusion)
    e = set_smem_once<4>(k1_tc_kernel<2, true, 1>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<2, true, 1><<<(unsigned)grid, 768, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  } else {  // default: the same mapping with fp32 phase-1 arithmetic (fp32 FMAs on packed pairs, no fp64 conversion per element)
    e = set_smem_once<5>(k1_tc_kernel<2, true, 0>, smem_bytes);
    if (e != cudaSuccess) return e;
    k1_tc_kernel<2, true, 0><<<(unsigned)grid, 768, smem_bytes, st>>>(tmap, tmap3, t, ntiles);
  }
  return cudaGetLastError();
}

}  // namespace agd
