// Scoring kernels for the linear predictor  X . W^T + b -> argmax   (sm_90a).
//
// Replaces the numeric body of sklearn's LinearClassifierMixin.predict (sklearn/linear_model/_base.py:366-427), which
// is what the reference's canonical predictor runs (unionml:README.md:87-92).
//
//  * linear_argmax_tma_kernel<C, EXACT, QUEUE, SCHED>: persistent, warp-specialised.  One producer warp streams X
//    through a 16 KiB-per-stage shared-memory ring with TMA + mbarriers: 128-row x 32-feature boxes (128B-swizzled), or
//    at 33 <= F <= 64 (kWhole) stages of 64 complete rows, or (kHalf) 32 KiB stages of 256 complete rows from the
//    batch's compact fp16 copy; eight consumer warps (four in kHalf) each own one tile at a time (4, 2 or 8
//    rows per lane), read X with conflict-free LDS.128, W as warp-uniform broadcast
//    LDS.128 from a transposed copy in shared memory, keep C (+1) fp32 accumulators per row in registers, and fuse
//    bias, argmax (first maximum wins, like np.argmax) and the label store.  In EXACT mode one extra accumulator
//    carries A = max|b| + sum_f |x_f| * max_c |w_cf|; rows whose top-2 margin is not provably larger than the fp32
//    rounding error (2 (F+4) 2^-24 A) are appended to a list and re-scored in fp64 by rescore_f64_kernel.
//  * rescore_f64_kernel: warp per row, lanes over features, fp64 FMA + shuffle reduction; serves the flagged rows of
//    EXACT mode and is the generic (any F, any C) path when the tile kernel's shape limits do not hold.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "uml_common.cuh"
#include "label_store.cuh"
#include "tma_ring.cuh"
#include "rescore_util.cuh"
#include "wgmma.cuh"

#ifndef UML_RESCORE_QUEUE_DEFAULT
#define UML_RESCORE_QUEUE_DEFAULT 1  // one launch per step; the few flagged rows (0.02 % on digits) cost the queue little
#endif


namespace uml {

struct RowScore {
  int idx;
  bool bad;        // NaN/Inf in the row
  bool ambiguous;  // fp64 top-2 margin inside the fp64 rounding bound: a true tie, decided by the first-index rule
};

// float64 scores of one row by one warp, first maximum wins like np.argmax.  Lanes split the features; classes are
// scored CB at a time (at most sixteen: 2 CB independent fp64 chains per lane), the sums are reduced with warp_reduce16
// and the arg-max / runner-up found by a butterfly over the lanes.  LOAD(f) yields feature f of the row as double.
// Callers that know the class count at compile time pass CB = C, KNOWN_C and C itself: one round, whose accumulators
// ptxas keeps in registers (warp_reduce16<true>); the generic callers take CB = 16 and loop over the rounds.  For
// C <= 16 both do the same operations in the same order.
// w64 is feature-major, w64[f * S + c]: a lane fetches the classes of its feature with 16-byte loads off ONE address
// (immediate offsets) - the class-major table this replaces cost a 64-bit multiply-add per weight, half of the kernel's
// instructions at F = 784.  b64 holds 2C doubles: the biases, then each class's bias magnitude for the bound (|b_c|, or
// |b_c| + sum_f |shift_f w'_cf| for a folded affine map); fold_rel is the bound's extra relative term of a folded map
// (0 otherwise) and `binary` selects sklearn's `score > 0` rule for the expanded binary layout [0, s] (DESIGN.md 3.2).
template <int CB = 16, bool KNOWN_C = false, typename LOAD>
__device__ __forceinline__ RowScore score_row_f64(LOAD load, const double* __restrict__ w64, int S,
                                                  const double* __restrict__ b64, int F, int C, double fold_rel,
                                                  bool binary, int lane) {
  const double u = 1.1102230246251565e-16;  // 2^-53
  const double q64 = 4.9406564584124654e-324;  // 2^-1074: the spacing of float64 subnormals
  bool bad = false;
  double best = 0.0, second = -INFINITY, amax = 0.0;
  int idx = 0;
  static_assert(KNOWN_C ? CB >= 1 && CB <= 16 : CB == 16, "rounds of sixteen classes, or one round of the known C");
  for (int c0 = 0; c0 < (KNOWN_C ? CB : C); c0 += CB) {
    const int pairs = KNOWN_C ? (CB + 1) / 2 : min((CB + 1) / 2, (C - c0 + 1) / 2);  // 16-byte loads per feature this round (an odd C ends in a zero pad)
    double s[16], a[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) s[q] = a[q] = 0.0;
    // the row's features come from global memory (or, on the online path, over PCIe): four loads are issued before the
    // first is used, otherwise every 32-feature step of a wide model (F = 784: 25 steps) waits a full round trip
    constexpr int XB = 4;
    for (int f0 = lane; f0 < F; f0 += 32 * XB) {
      double xb[XB];
#pragma unroll
      for (int k = 0; k < XB; ++k) xb[k] = f0 + 32 * k < F ? load(f0 + 32 * k) : 0.0;
#pragma unroll
      for (int k = 0; k < XB; ++k) {
        const int f = f0 + 32 * k;
        if (f < F) {
          const double xv = xb[k];
          if (!isfinite(xv)) bad = true;
          const double ax = fabs(xv);
          const double2* wp = reinterpret_cast<const double2*>(w64 + static_cast<size_t>(f) * S + c0);
#pragma unroll
          for (int q2 = 0; q2 < 8; ++q2) {
            if (q2 < pairs) {
              const double2 w = wp[q2];
              s[2 * q2] = fma(xv, w.x, s[2 * q2]);
              a[2 * q2] = fma(ax, fabs(w.x), a[2 * q2]);
              s[2 * q2 + 1] = fma(xv, w.y, s[2 * q2 + 1]);
              a[2 * q2 + 1] = fma(ax, fabs(w.y), a[2 * q2 + 1]);
            }
          }
        }
      }
    }
    const double sv = warp_reduce16<KNOWN_C>(s, lane), av = warp_reduce16<KNOWN_C>(a, lane);
    const int cl = c0 + (lane >> 1);  // the class this lane pair now holds
    const bool valid = cl < C;
    Top2 t;
    t.best = valid ? sv + b64[cl] : -INFINITY;
    t.second = -INFINITY;
    t.idx = cl;
    top2_butterfly(t, 2);
    amax = fmax(amax, warp_max(valid ? av + b64[C + cl] : 0.0, 2));
    if (c0 == 0) {
      best = t.best;
      second = t.second;
      idx = t.idx;
    } else if (isnan(t.best) ? !isnan(best) : t.best > best) {  // strict: a tie keeps the earlier (lower) class; the
      second = fmax(best, t.second);                             // first NaN wins, as in np.argmax
      best = t.best;
      idx = t.idx;
    } else {
      second = fmax(second, t.best);
    }
  }
  if (idx >= C) idx = 0;  // padding classes score -inf and lose every tie, so this is a guard only
  if (binary && isnan(best)) idx = 0;  // sklearn's binary rule: `NaN > 0` is False
  RowScore r;
  r.idx = idx;
  r.bad = __any_sync(0xffffffffu, bad);
  // fp64 error of each score: at most F/32 + 7 roundings (<= 32-way split FMA chains + 5 shuffle adds + bias add),
  // each <= u |result| or, in the subnormals, <= 2^-1075 absolute.  A folded affine map adds fold_rel a.
  const double n_ops = static_cast<double>(F) / 32.0 + 8.0;
  const double err = (n_ops * u + fold_rel) * amax + n_ops * q64;
  r.ambiguous = !((best - second) > 2.0 * err);
  return r;
}

// ---------------------------------------------------------------------------------------------------------------
// TMA fp32 tile kernel
// ---------------------------------------------------------------------------------------------------------------
struct TmaKernelParams {
  const float* wt;    // [f_pad][CP]
  const float* bias;  // [CP]
  LabelTargets targets;
  long long n_rows;
  long long num_tiles;
  int f_pad;
  int kc;          // 32-feature chunks per tile
  int num_stages;  // ring depth
  float thr;       // relative margin threshold 2 (F+4) 2^-24 (1 + slack)
  int* flag_count;
  int32_t* flag_rows;
  int flag_cap;
  // QUEUE kernels (EXACT): flagged rows are re-scored in fp64 by a dedicated warp of the same launch - no flag list in
  // global memory, no second kernel behind every step
  const float* x;
  const double* x64;
  SrcView src;
  long long ld, ld64;
  const double* w64;  // [F][w64_stride], feature-major
  const double* b64;
  int w64_stride;
  int n_classes, n_features;
  double fold_rel;  // score_row_f64's extra relative bound term (LinearDeviceModel)
  int binary;
  unsigned long long* counters;
#ifdef UML_PROBE_WAIT_CLOCKS
  unsigned long long* probe_clocks;  // [12], see the diagnostic builds below
#endif
#ifdef UML_PROBE_TIMELINE
  unsigned long long* probe_timeline;  // [gridDim.x][kProbeStamps], see the diagnostic builds below
#endif
  const void* tc_ops;  // tensor-core schedules: LinearDeviceModel::tc_ops
  float tc_kappa;
};

// fp64 scores of one row by the whole warp (kept out of line so the hot loop's register allocation is untouched)
__device__ __noinline__ int rescore_row_inline(const TmaKernelParams& p, long long row, int lane) {
  RowScore r;
  if (p.src.base) {
    const SrcView v = p.src;
    r = score_row_f64([&](int f) { return load_src(v, row, f); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, p.fold_rel, p.binary != 0, lane);
  } else if (p.x64) {
    const double* xr64 = p.x64 + row * p.ld64;
    r = score_row_f64([&](int f) { return xr64[f]; }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, p.fold_rel, p.binary != 0, lane);
  } else {
    const float* xr = p.x + row * p.ld;
    r = score_row_f64([&](int f) { return static_cast<double>(xr[f]); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, p.fold_rel, p.binary != 0, lane);
  }
  if (lane == 0) count_rescored_row(p, r.bad, r.ambiguous);
  return r.idx;
}

// The tensor-core schedules' fp64 scores of one row, from the batch's float64 copy when it keeps one (its fp32 rows are
// not the caller's values) and from the fp32 rows otherwise; no source view reaches these schedules (launch_linear_tma's
// dispatch).  C is known, so this is one copy of score_row_f64 with its 2 C accumulators in registers, instead of
// rescore_row_inline's three copies with sixteen of each in local memory.
template <int C>
__device__ __noinline__ int rescore_row_tc(const TmaKernelParams& p, long long row, int lane) {
  const float* xr = p.x + row * p.ld;
  const double* xr64 = p.x64 ? p.x64 + row * p.ld64 : nullptr;
  const RowScore r = score_row_f64<C, true>([&](int f) { return xr64 ? xr64[f] : static_cast<double>(xr[f]); }, p.w64,
                                            p.w64_stride, p.b64, p.n_features, C, p.fold_rel, p.binary != 0, lane);
  if (lane == 0) count_rescored_row(p, r.bad, r.ambiguous);
  return r.idx;
}

constexpr int kTileSentinel = -1;        // claimed schedules: ring item that ends a scoring warp's loop
constexpr int kQueueCap = 2048;           // flagged-row queue of the QUEUE kernels (power of two)
constexpr int kQueueHeadroom = 1024;      // a warp publishes only while this many slots are free (8 warps x 128 rows)

// Diagnostic builds of this file (tools/linear_probe.cu defines these; the library defines neither):
//  UML_PROBE_FEED_ONLY    the scoring warps hand each stage back as soon as it has landed, without the math: what the
//                         ring (producer, order, barriers) delivers on its own
//  UML_PROBE_WAIT_CLOCKS  clock64() totals added into p.probe_clocks: [0] the producer's `empty` waits, [1] its whole
//                         loop, [2] the scoring warps' waits for their data, [3] their whole loops, [4] the time they
//                         hold a landed stage (from the return of the `full` wait to the `empty` arrive); QUEUE
//                         kernels also [5] the re-score warp's time on rows it took from the queue (replay and fp64
//                         re-score), [6] its whole loop, [10] the fp64 part of [5] and [11] the rows every warp took
//                         from the queue; kByteMma also [7] the MMA warps' waits for a free score slot, [8] the
//                         epilogue warps' waits for a full one and [9] their whole loops ([2]-[4] count the MMA warps
//                         only)
//  UML_PROBE_TIMELINE     %globaltimer per CTA into p.probe_timeline[blockIdx.x][kProbeStamps]: [0] entry, [1] the
//                         producer's first issue, [2] the first stage landed (warp 0), [3] the last `empty` arrive,
//                         [4] exit; tensor-core schedules also [5] the first drain warp to see every publisher done,
//                         [6] the last batch claimed, [7] the last replay finished, [8] the last fp64 row finished
//  UML_PROBE_NO_W         kHalf only, wrong scores: every feature's W^T row is one set of registers loaded once per warp,
//                         so the scoring loop issues no W loads
//  UML_PROBE_NO_X         kHalf only, wrong scores: every feature of a row is one register set once per warp, so the
//                         scoring loop issues no x loads and no fp16 conversions (both defines: the FMAs alone)
//  UML_PROBE_NO_EPILOGUE  kByteMma only, no labels: the epilogue warps hand every score slot back unread, and skip the
//                         top-2, the label stores and the queue hand-off (the MMA warpgroups and the slots as they are)
//  UML_PROBE_NO_HANDOFF   kByteMma only, wrong labels for near-ties: tier 1's verdict is forced to "certified", so no
//                         row goes through the queue
constexpr int kProbeStamps = 9;  // UML_PROBE_TIMELINE's stamps per CTA
#ifdef UML_PROBE_NO_EPILOGUE
constexpr bool kProbeNoEpilogue = true;
#else
constexpr bool kProbeNoEpilogue = false;
#endif
#ifdef UML_PROBE_NO_HANDOFF
constexpr bool kProbeNoHandoff = true;
#else
constexpr bool kProbeNoHandoff = false;
#endif
#ifdef UML_PROBE_NO_W
constexpr bool kProbeNoW = true;
#else
constexpr bool kProbeNoW = false;
#endif
#ifdef UML_PROBE_NO_X
constexpr bool kProbeNoX = true;
#else
constexpr bool kProbeNoX = false;
#endif
#ifdef UML_PROBE_FEED_ONLY
constexpr bool kFeedOnly = true;
#else
constexpr bool kFeedOnly = false;
#endif
#ifdef UML_PROBE_WAIT_CLOCKS
#define UML_PROBE_TIMED(total, ...)     \
  do {                                  \
    const long long t0_ = clock64();    \
    __VA_ARGS__;                        \
    (total) += clock64() - t0_;         \
  } while (0)
#define UML_PROBE_CLOCK(t) const long long t = clock64()
#define UML_PROBE_SINCE(total, t) (total) += clock64() - (t)
#else
#define UML_PROBE_TIMED(total, ...) __VA_ARGS__
#define UML_PROBE_CLOCK(t)
#define UML_PROBE_SINCE(total, t)
#endif
#ifdef UML_PROBE_TIMELINE
__device__ __forceinline__ unsigned long long probe_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define UML_PROBE_STAMP(slot) (p.probe_timeline[blockIdx.x * kProbeStamps + (slot)] = probe_globaltimer())
#define UML_PROBE_STAMP_MIN(slot) atomicMin(&p.probe_timeline[blockIdx.x * kProbeStamps + (slot)], probe_globaltimer())
#define UML_PROBE_STAMP_MAX(slot) atomicMax(&p.probe_timeline[blockIdx.x * kProbeStamps + (slot)], probe_globaltimer())
#define UML_PROBE_LANDED(first) \
  if ((first) && warp == 0 && lane == 0) UML_PROBE_STAMP(2)
#define UML_PROBE_RELEASED() probe_last_release = probe_globaltimer()
#else
#define UML_PROBE_STAMP(slot)
#define UML_PROBE_STAMP_MIN(slot)
#define UML_PROBE_STAMP_MAX(slot)
#define UML_PROBE_LANDED(first)
#define UML_PROBE_RELEASED()
#endif

// How the ring is fed (the schedule):
//  kChunked  one stage is a 128-row x 32-feature fp32 box, a tile takes f_pad / 32 stages (4 rows per lane) and the
//            CTA scores tiles blockIdx.x, blockIdx.x + gridDim.x, ...
//  kWhole    (f_pad == 64, linear_whole_rows) one stage is one 64-row tile with all its features, loaded as two
//            {32 features, 64 rows} fp32 boxes onto one barrier (2 rows per lane)
//  kHalf     (f_pad <= 64, the batch has a compact fp16 copy) one stage is one 256-row tile with all its features, two
//            {64 features, 128 rows} fp16 boxes onto one barrier (8 rows per lane)
//  kHalfMma  (EXACT + QUEUE, the same stages, every fp16 value >= 0, the model has tc_ops) two warpgroups score the
//            stages on the tensor cores (wgmma, f16 x f16 -> fp32, W^T as scaled hi | lo pieces); ring item n goes to
//            warpgroup n % 2.  Rows the tensor-core guard does not certify go through the queue, where the re-score warp
//            first replays the fp32 route on them (DESIGN.md 3.1, 3.2)
//  kByteMma  (kHalfMma's conditions, the batch has a byte copy) kHalfMma on 16 KiB stages of one {64 bytes, 256 rows}
//            box of the byte copy: a thread loads its A fragments of each m64 block with two LDS.128, widens the
//            bytes to the same f16 values kHalfMma reads and issues wgmma with A from registers; epilogue warps of their
//            own score the rows
// kWhole, kHalf and the tensor-core schedules claim their tiles in groups of NCU (the units that take ring items: the
// scoring warps, or the two warpgroups) from a global counter; ring item n goes to unit n % NCU.
enum class LinearSched { kChunked, kWhole, kHalf, kHalfMma, kByteMma };
__host__ __device__ constexpr bool linear_tc_sched(LinearSched s) { return s == LinearSched::kHalfMma || s == LinearSched::kByteMma; }

// scoring warps of a schedule; the producer is warp NCW and the QUEUE kernels' re-score warp NCW + 1
// kByteMma: two MMA warpgroups (warps 0-7) and a pair of epilogue warps per warpgroup (8-11).  Its feed takes half of
// kHalfMma's time, so the time per item outside the tensor cores is the limit: the epilogue warps take the per-row tail
// (top-2, tier 1, label stores, queue hand-off) off the warpgroups, which then keep up with the feed in two.  Two
// epilogue warps for three warpgroups (16 warps) could not: 0.349 against 0.280 ms (DESIGN.md 5.1).
constexpr int kByteWarpgroups = 2;
constexpr int kByteEpiWarps = 2 * kByteWarpgroups;
__host__ __device__ constexpr int linear_consumer_warps(LinearSched s) {
  return s == LinearSched::kHalf ? kHalfConsumerWarps : s == LinearSched::kByteMma ? 4 * kByteWarpgroups + kByteEpiWarps : kConsumerWarps;
}
// units that take ring items (and the ring's floor): warps, or the tensor-core schedules' warpgroups
__host__ __device__ constexpr int linear_ring_units(LinearSched s) {
  return s == LinearSched::kByteMma ? kByteWarpgroups : linear_tc_sched(s) ? linear_consumer_warps(s) / 4 : linear_consumer_warps(s);
}
__host__ __device__ constexpr int linear_threads(LinearSched s, bool queue) { return (linear_consumer_warps(s) + (queue ? 2 : 1)) * 32; }
// bytes of one ring stage: in kHalf and kHalfMma two 16 KiB fp16 boxes
__host__ __device__ constexpr int linear_stage_bytes(LinearSched s) {
  return s == LinearSched::kHalf || s == LinearSched::kHalfMma ? 2 * kStageBytes : kStageBytes;
}
// tensor-core schedules: bytes of the B operand in shared memory (rounded up to the 1 KiB that keeps what follows aligned)
__host__ __device__ constexpr int linear_tc_b_bytes(int C) { return (linear_tc_cols(C) * 128 + 1023) / 1024 * 1024; }
// kByteMma: the score slots between the MMA warpgroups and the epilogue warps, kEpiSlots per warpgroup.  A slot holds
// one item: per MMA warp the C + 1 folded columns (classes, bound) of its 64 rows, column-major with a pitch of
// kEpiPitch floats (the bank argument is at the write-out in the kernel).  In front of the slots: their `full` and
// `empty` mbarriers and tile indices (kEpiCtlBytes).
constexpr int kEpiPitch = 68;
constexpr int kEpiSlots = 2;
constexpr int kEpiCtlBytes = 128;
__host__ __device__ constexpr int linear_epi_bytes(LinearSched s, int C) {
  return s == LinearSched::kByteMma ? kEpiCtlBytes + kByteWarpgroups * kEpiSlots * 4 * (C + 1) * kEpiPitch * 4 : 0;
}

// The tensor-core schedules' tier 2 (DESIGN.md 3.2): the fp32 route's scores of up to 32 queued rows, one row per lane
// (row < 0: the lane has none), replayed bit for bit: columns c < C run their FMA chains in feature order from bias_s[c]
// over the lane's fp32 row (zeros past F up to f_pad, as the fp32 route's boxes hold), column C (the bound) on |x|; then
// finish_rows' sequential best / second loop and the same p.thr comparison.  A lane whose row that route certifies
// stores its label and returns true; the caller sends the others to fp64.  W^T rows are read as warp-uniform LDS.128
// (broadcast; CP % 4 == 0).  Out of line, so that the MMA and epilogue loops keep their register allocation, and small:
// it runs a few times per CTA per launch, from a cold instruction cache, so the FMAs of one 32-feature half are
// unrolled and the two halves are one rolled loop (the second half's values move down between the passes).
template <int C>
__device__ __noinline__ bool replay_fp32_rows(const TmaKernelParams& p, const float* wt_s, const float* bias_s,
                                              long long row) {
  constexpr int CP = (C + 1 + 3) / 4 * 4;
  const int F = p.n_features;
  const bool has = row >= 0;
  const float* xr = p.x + (has ? row : 0) * p.ld;
  float acc[C + 1];
#pragma unroll
  for (int c = 0; c <= C; ++c) acc[c] = bias_s[c];
  // one feature x with its W^T row wf: every column's next FMA, in the fp32 route's order
  auto fma_feature = [&](float x, const float* wf) {
#pragma unroll
    for (int m = 0; m < CP / 4; ++m) {
      const float4 w = *reinterpret_cast<const float4*>(wf + 4 * m);
      const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 4 * m + e;
        if (c < C) acc[c] = fmaf(x, wv[e], acc[c]);
        if (c == C) acc[C] = fmaf(fabsf(x), wv[e], acc[C]);
      }
    }
  };
  if (((reinterpret_cast<uintptr_t>(p.x) | static_cast<uintptr_t>(p.ld) * 4u) & 15u) == 0) {
    // 16-byte loads of the whole row (f_pad <= 64) before the first FMA: one round trip to memory per batch.  ld is a
    // multiple of 4 >= F, so the last group's load stays inside the row; its values past F are replaced by zeros.
    float xv[64];
#pragma unroll
    for (int g = 0; g < 16; ++g) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (has && 4 * g < F) v = __ldg(reinterpret_cast<const float4*>(xr + 4 * g));
      xv[4 * g] = v.x;
      xv[4 * g + 1] = 4 * g + 1 < F ? v.y : 0.f;
      xv[4 * g + 2] = 4 * g + 2 < F ? v.z : 0.f;
      xv[4 * g + 3] = 4 * g + 3 < F ? v.w : 0.f;
    }
#pragma unroll 1
    for (int f0 = 0; f0 < p.f_pad; f0 += 32) {
#pragma unroll
      for (int k = 0; k < 32; ++k) fma_feature(xv[k], wt_s + (f0 + k) * CP);
#pragma unroll
      for (int k = 0; k < 32; ++k) xv[k] = xv[32 + k];
    }
  } else {
#pragma unroll 1
    for (int f = 0; f < p.f_pad; ++f) fma_feature(has && f < F ? __ldg(xr + f) : 0.f, wt_s + f * CP);
  }
  float best = acc[0], second = -INFINITY;
  int bi = 0;
#pragma unroll
  for (int c = 1; c < C; ++c) {
    if (acc[c] > best) {
      second = best;
      best = acc[c];
      bi = c;
    } else {
      second = fmaxf(second, acc[c]);
    }
  }
  const bool certified = has && (best - second) > p.thr * acc[C];
  if (certified) store_label(p.targets, row, bi);
  return certified;
}

// kHalf: rows per lane scored in one pass over a 256-row stage (NPASS = 8 / this passes).  All 8 rows of a lane at
// once for every class count: their 8 NCOL accumulators and the operands in flight fit in 255 registers without a
// spill up to C = 16 in FAST, EXACT and EXACT + QUEUE (ptxas -v, DESIGN.md 5.1).  The diagnostic builds' two passes
// of 4 rows separate the W reuse of 8 rows from the warp count.
#ifdef UML_PROBE_HALF_PASS_ROWS
constexpr int kHalfPassRows = UML_PROBE_HALF_PASS_ROWS;
#else
constexpr int kHalfPassRows = 8;
#endif

template <int C, bool EXACT, bool QUEUE, LinearSched SCHED>
__global__ void __launch_bounds__(linear_threads(SCHED, true), 1)
linear_argmax_tma_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ TmaKernelParams p) {
  constexpr int NCOL = C + (EXACT ? 1 : 0);  // accumulators per row (classes + error-bound column)
  constexpr int CP = (C + 1 + 3) / 4 * 4;    // padded columns of wt in shared memory (layout shared by both modes)
  constexpr int NW4 = (NCOL + 3) / 4;        // float4 loads of W per feature
  constexpr bool WHOLE = SCHED == LinearSched::kWhole;
  constexpr bool HALF = SCHED == LinearSched::kHalf;
  constexpr bool MMA = linear_tc_sched(SCHED);               // kHalfMma or kByteMma
  constexpr bool BYTES = SCHED == LinearSched::kByteMma;    // 256-row stages of the byte rows, one box
  constexpr bool F16 = HALF || SCHED == LinearSched::kHalfMma;  // 256-row stages of the compact fp16 rows, two boxes
  constexpr bool CLAIMED = WHOLE || F16 || BYTES;            // tiles claimed from kCounterTileClaim, one tile per stage
  constexpr int NCW = linear_consumer_warps(SCHED);
  constexpr int NCU = linear_ring_units(SCHED);
  static_assert(!MMA || (EXACT && QUEUE), "the tensor-core schedule certifies rows through the queue's replay");
  constexpr int TILE = F16 || BYTES ? kHalfTileRows : WHOLE ? kWholeTileRows : kTileRows;  // rows per tile = per ring stage
  // warps that publish to the queue (kByteMma: the epilogue warps, warps NMW .. NCW - 1)
  constexpr int NMW = BYTES ? 4 * kByteWarpgroups : NCW;
  constexpr int NPUB = BYTES ? kByteEpiWarps : NCW;
  static_assert(!BYTES || NMW + NPUB == NCW, "warps NMW .. NCW - 1 are the epilogue warps");
  // free queue slots a publishing warp wants before it publishes: every one may publish all its rows of a tile at once
  // (kHalfMma: the 64 rows of the tile a warp stores; kByteMma: an epilogue warp's 128, half a tile)
  constexpr int HEADROOM = HALF ? NCW * TILE : BYTES ? NPUB * TILE / 2 : MMA ? NCW * 64 : kQueueHeadroom;
  static_assert(HEADROOM <= kQueueCap, "the queue holds one tile of every scoring warp");
  // rows per lane held in registers at once (kHalf: one pass, NPASS passes per tile)
  constexpr int R = HALF ? kHalfPassRows : TILE / 32;
  constexpr int NPASS = TILE / 32 / R;
  static_assert(NPASS * R * 32 == TILE && (!HALF || R % 4 == 0), "a pass is whole 128-row boxes");
  // one box: 8 KiB (two per kWhole stage) or 16 KiB (two per kHalf stage, one per kByteMma stage)
  constexpr int BOX_BYTES = BYTES ? kHalfTileRows * kByteRowBytes : (F16 ? kTileRows : TILE) * kChunkF * 4;
  constexpr int STAGE_BYTES = linear_stage_bytes(SCHED);
  static_assert(!F16 || (BOX_BYTES == kTileRows * kHalfBoxF * 2 && STAGE_BYTES == 2 * BOX_BYTES),
                "an fp16 stage is two boxes");
  static_assert(!BYTES || STAGE_BYTES == BOX_BYTES, "a byte stage is one box");
  // fp32x2 accumulator pairs (see the accumulator comment below).  Not in the fp16 schedule: fma2 is two fmaf, so the
  // scores are the same bits, and without the 64-bit register pairs ptxas schedules its 128 registers better
  // (0.534 -> 0.523 ms at cfg 2, DESIGN.md 5.1)
  constexpr bool USE_F2 = EXACT && !HALF;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // SWIZZLE_128B wants 1 KiB alignment

  const int S = p.num_stages;
  // tensor-core schedules: the B operand (1 KiB aligned, as SWIZZLE_128B wants) between the ring and W^T
  float* wt_s = reinterpret_cast<float*>(smem + static_cast<size_t>(S) * STAGE_BYTES + (MMA ? linear_tc_b_bytes(C) : 0));
  float* bias_s = wt_s + p.f_pad * CP;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + CP);
  uint64_t* empty_bar = full_bar + S;
  // QUEUE kernels: rows flagged by the scoring warps travel through this shared-memory queue to the re-score warp
  // (slot value = row + 1, 0 = empty); ctl[0] = tail (reserved), ctl[1] = head (tickets claimed), ctl[2] = publishing
  // warps done (NPUB), ctl[3] = slots consumed
  int* q_slots = reinterpret_cast<int*>(empty_bar + S);
  int* q_ctl = q_slots + kQueueCap;
  // CLAIMED: the tile each stage holds, written by the producer before the stage's `full` arrive (whose release makes it
  // visible to the waiters); kTileSentinel ends a scoring warp's loop
  int* tile_slot = q_ctl + 4;
  // kByteMma: the score slots (linear_epi_bytes), behind the 64 tile slots the host reserves; slot s of warpgroup g is
  // epi_full / epi_empty / epi_tile [g * kEpiSlots + s] and its MMA warp w's rows at epi_buf + ((g * kEpiSlots + s) * 4
  // + w % 4) * (C + 1) * kEpiPitch
  [[maybe_unused]] uint64_t* epi_full = reinterpret_cast<uint64_t*>(tile_slot + 64);
  [[maybe_unused]] uint64_t* epi_empty = epi_full + kByteWarpgroups * kEpiSlots;
  [[maybe_unused]] int* epi_tile = reinterpret_cast<int*>(epi_empty + kByteWarpgroups * kEpiSlots);
  static_assert(2 * kByteWarpgroups * kEpiSlots * 8 + kByteWarpgroups * kEpiSlots * 4 <= kEpiCtlBytes, "slot control");
  [[maybe_unused]] float* epi_buf = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(epi_full) + kEpiCtlBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) UML_PROBE_STAMP(0);

  // stage W^T (with its wmax column) and the bias once per CTA; they stay resident for every tile this CTA scores
  {
    const float4* src = reinterpret_cast<const float4*>(p.wt);
    float4* dst = reinterpret_cast<float4*>(wt_s);
    const int n4 = p.f_pad * CP / 4;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = __ldg(src + i);
    if (threadIdx.x < CP) bias_s[threadIdx.x] = __ldg(p.bias + threadIdx.x);
    if constexpr (MMA) {
      const uint4* bsrc = static_cast<const uint4*>(p.tc_ops);
      uint4* bdst = reinterpret_cast<uint4*>(smem + static_cast<size_t>(S) * STAGE_BYTES);
      for (int i = threadIdx.x; i < linear_tc_cols(C) * 8; i += blockDim.x) bdst[i] = __ldg(bsrc + i);
      fence_proxy_async_smem();  // st.shared -> visible to the wgmma reads
    }
    if constexpr (QUEUE) {
      for (int i = threadIdx.x; i < kQueueCap + 4; i += blockDim.x) q_slots[i] = 0;
    }
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], MMA ? 4 : 1);  // tensor cores: every warp of the warpgroup hands the stage back
    }
    if constexpr (BYTES) {
      for (int s = 0; s < kByteWarpgroups * kEpiSlots; ++s) {
        mbar_init(&epi_full[s], 4);   // the four warps of the warpgroup post the item
        mbar_init(&epi_empty[s], 2);  // both epilogue warps of the warpgroup hand the slot back
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  pdl_launch_dependents();  // the re-score kernel behind this launch may be scheduled now; it waits for this grid to finish
  const long long G = gridDim.x;
  const long long num_tiles = p.num_tiles;
  const int KC = p.kc;
#ifdef UML_PROBE_WAIT_CLOCKS
  long long probe_wait = 0;
  const long long probe_start = clock64();
#endif

  if (warp == NCW) {
    // ===================== TMA producer (one elected lane) =====================
    if (elect_one_sync()) {
      tma_prefetch_desc(&xmap);
#ifdef UML_PROBE_TIMELINE
      bool probe_first_issue = true;
#endif
      const uint64_t policy = make_evict_first_policy();  // X is read exactly once
      int stage = 0;
      uint32_t phase = 0;
      auto next_stage = [&] {
        if (++stage == S) {
          stage = 0;
          phase ^= 1u;
        }
      };
      if constexpr (CLAIMED) {
        // Tiles are claimed, NCW at a time, from a counter shared by the grid: with a static split, CTAs
        // with equal tile counts finished up to ~0.24 ms apart (SMs draw unequal shares of HBM bandwidth), and the
        // launch lasted as long as the slowest one.  Ring item n is one tile with both halves of its rows and goes to
        // warp n % NCW; a group claimed past the end hands every warp kTileSentinel.  The next group is
        // claimed while this one is issued, so the atomic's round trip stays off the ring.
        unsigned long long* claim = &p.counters[kCounterTileClaim];
        unsigned long long* claim_done = &p.counters[kCounterTileClaimDone];
        long long base = static_cast<long long>(atomicAdd(claim, static_cast<unsigned long long>(NCU)));
        for (;;) {
          const long long next =
              base < num_tiles ? static_cast<long long>(atomicAdd(claim, static_cast<unsigned long long>(NCU))) : base;
          for (int w = 0; w < NCU; ++w) {
            const long long tile = base + w;
            UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u));
            tile_slot[stage] = base < num_tiles ? static_cast<int>(tile) : kTileSentinel;
            if (tile < num_tiles) {
              if constexpr (F16) {
                // rows 128-255 of the last tile may all lie past the batch: that box is not loaded (its rows are
                // scored from stale shared memory and never stored)
                uint8_t* dst = smem + static_cast<size_t>(stage) * STAGE_BYTES;
                const int row = static_cast<int>(tile * TILE);
                const bool second = row + kTileRows < p.n_rows;
                mbar_arrive_expect_tx(&full_bar[stage], second ? STAGE_BYTES : BOX_BYTES);
                tma_load_2d(dst, &xmap, &full_bar[stage], 0, row, policy);
                if (second) tma_load_2d(dst + BOX_BYTES, &xmap, &full_bar[stage], 0, row + kTileRows, policy);
              } else {
                // (kByteMma: one {64, 256} box; rows past the batch are filled with zeros and never stored)
                mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
                uint8_t* dst = smem + static_cast<size_t>(stage) * kStageBytes;
                const int row = static_cast<int>(tile * TILE);
                tma_load_2d(dst, &xmap, &full_bar[stage], 0, row, policy);
                if constexpr (WHOLE) tma_load_2d(dst + BOX_BYTES, &xmap, &full_bar[stage], kChunkF, row, policy);
              }
#ifdef UML_PROBE_TIMELINE
              if (probe_first_issue) UML_PROBE_STAMP(1);
              probe_first_issue = false;
#endif
            } else {
              mbar_arrive(&full_bar[stage]);  // past the last tile: nothing to load, the warp skips or stops
            }
            next_stage();
          }
          if (base >= num_tiles) break;
          base = next;
        }
        // this CTA claims no more; the last CTA to get here hands the counter back at 0 for the next launch on the
        // stream (no memset between steps, and correct under CUDA-graph replay)
        __threadfence();
        if (atomicAdd(claim_done, 1ull) == static_cast<unsigned long long>(gridDim.x) - 1ull) {
          *claim = 0ull;
          *claim_done = 0ull;
          __threadfence();
        }
      } else {
        // Work items in ring order: for each round (kConsumerWarps tiles), for each 32-feature chunk k, for each
        // active warp w: (tile = first + w*G, chunk k).  Producer and consumers derive the same sequence numbers.
        for (long long first = blockIdx.x; first < num_tiles; first += G * kConsumerWarps) {
          const int nv = static_cast<int>(min(static_cast<long long>(kConsumerWarps), (num_tiles - first + G - 1) / G));
          for (int k = 0; k < KC; ++k) {
            for (int w = 0; w < nv; ++w) {
              UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u));
              mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
              tma_load_2d(smem + static_cast<size_t>(stage) * kStageBytes, &xmap, &full_bar[stage], k * kChunkF,
                          static_cast<int>((first + w * G) * TILE), policy);
#ifdef UML_PROBE_TIMELINE
              if (first == blockIdx.x && k == 0 && w == 0) UML_PROBE_STAMP(1);
#endif
              next_stage();
            }
          }
        }
      }
#ifdef UML_PROBE_WAIT_CLOCKS
      atomicAdd(&p.probe_clocks[0], static_cast<unsigned long long>(probe_wait));
      atomicAdd(&p.probe_clocks[1], static_cast<unsigned long long>(clock64() - probe_start));
#endif
    }
  } else {
    // ===================== consumers: one tile per warp at a time (warp 9 of the QUEUE kernels: re-score) ==========
    const bool scoring_warp = warp < NMW;  // (kByteMma: the MMA warps)
    // lane l owns rows l, l+32, ... of the tile.  In every box row r sits at byte r*128 with its 16-byte chunks
    // XOR-swizzled by (r & 7); r & 7 == l & 7 for all of a lane's rows, so one swizzle term serves them all and the
    // eight lanes of every LDS.128 phase (lanes 8i..8i+7: l & 7 = 0..7) hit eight distinct bank groups.  The whole-row
    // stage is two such boxes (features 0-31, then 32-63 at +8 KiB), so the same holds in both halves; an fp16 row is
    // 64 halves in the same 128 bytes, so the same addresses serve it, and the fp16 stage's second box (rows 128-255
    // at +16 KiB) puts every one of its 256 rows at r*128.
    const uint32_t lanebase = static_cast<uint32_t>(lane) * 128u + static_cast<uint32_t>(lane & 7) * 16u;
#ifdef UML_PROBE_WAIT_CLOCKS
    long long probe_hold = 0;
#endif
#ifdef UML_PROBE_TIMELINE
    unsigned long long probe_last_release = 0;
#endif

    // USE_F2 (EXACT kernels): class accumulators as fp32x2 pairs (classes 2i, 2i+1 -> one fma2); an odd last class
    // and the error-bound column (|x| is a free operand modifier on scalar FFMA) stay scalar.
    constexpr int NPAIR = C / 2;
    constexpr bool ODD = (C & 1) != 0;
    uint64_t acc2[R][NPAIR > 0 ? NPAIR : 1];
    float acc_last[R], acc_bound[R];
    float acc[R][C + 1];
    auto init_acc = [&] {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if constexpr (USE_F2) {
#pragma unroll
          for (int i = 0; i < NPAIR; ++i) acc2[j][i] = pack2(bias_s[2 * i], bias_s[2 * i + 1]);
          acc_last[j] = ODD ? bias_s[C - 1] : 0.f;
          acc_bound[j] = EXACT ? bias_s[C] : 0.f;
        } else {
#pragma unroll
          for (int c = 0; c < NCOL; ++c) acc[j][c] = bias_s[c];
        }
      }
    };
    // one feature x of row j with wv = its W^T row: every class accumulator and the bound column
    auto fma_feature = [&](int j, float x, const float* wv) {
      if constexpr (USE_F2) {
        const uint64_t xx = pack2(x, x);
#pragma unroll
        for (int i = 0; i < NPAIR; ++i) acc2[j][i] = fma2(xx, pack2(wv[2 * i], wv[2 * i + 1]), acc2[j][i]);
        if (ODD) acc_last[j] = fmaf(x, wv[C - 1], acc_last[j]);
        if (EXACT) acc_bound[j] = fmaf(fabsf(x), wv[C], acc_bound[j]);
      } else {
#pragma unroll
        for (int c = 0; c < C; ++c) acc[j][c] = fmaf(x, wv[c], acc[j][c]);
        if (EXACT) acc[j][C] = fmaf(fabsf(x), wv[C], acc[j][C]);
      }
    };
    // features kChunkF*k .. +31 of the lane's rows from box xs, with wk = the W^T rows of those features; every row's
    // FMAs run in feature order, so scores do not depend on the schedule
    auto fma_box = [&](const uint8_t* xs, const float* wk) {
      if constexpr (kFeedOnly) return;
#pragma unroll
      for (int q = 0; q < kChunkF / 4; ++q) {
        float4 xv[R];
        const uint32_t off = lanebase ^ static_cast<uint32_t>(q * 16);
#pragma unroll
        for (int j = 0; j < R; ++j) xv[j] = *reinterpret_cast<const float4*>(xs + off + j * 32 * 128);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float wv[NW4 * 4];
#pragma unroll
          for (int m = 0; m < NW4; ++m) {
            const float4 t = *reinterpret_cast<const float4*>(wk + (q * 4 + e) * CP + m * 4);
            wv[m * 4 + 0] = t.x;
            wv[m * 4 + 1] = t.y;
            wv[m * 4 + 2] = t.z;
            wv[m * 4 + 3] = t.w;
          }
#pragma unroll
          for (int j = 0; j < R; ++j) fma_feature(j, e == 0 ? xv[j].x : e == 1 ? xv[j].y : e == 2 ? xv[j].z : xv[j].w, wv);
        }
      }
    };

    // kHalf: features 0 .. f_pad - 1 of the lane's rows from an fp16 stage, eight features (one 16-byte chunk of each
    // row) per iteration.  cvt.f32.f16 is exact, so every FMA gets the operands the fp32 route gives it, in the same
    // order (fma2 pairs there, plain fmaf here: the same IEEE operations): scores, flags and labels are those of the
    // fp32 rows bit for bit.  The loop over the chunks stays rolled: unrolled over 64 features, 8 rows of 11 columns
    // are ~7 000 instructions (112 KB of SASS), no other warp on the scheduler covers their instruction fetches, and
    // the kernel ran 3.7x slower (2x unrolled by 2, DESIGN.md 5.1).  The next chunk's x is loaded while this one is
    // scored.
    [[maybe_unused]] float probe_w[NW4 * 4], probe_x[R];  // UML_PROBE_NO_W / UML_PROBE_NO_X
    if constexpr (kProbeNoW) {
#pragma unroll
      for (int c = 0; c < NW4 * 4; ++c) probe_w[c] = wt_s[c];
    }
    if constexpr (kProbeNoX) {
#pragma unroll
      for (int j = 0; j < R; ++j) probe_x[j] = p.thr * static_cast<float>(lane + 32 * j + 1);
    }
    auto load_chunk = [&](uint4* hv, const uint8_t* xs, int k) {
      if constexpr (!kProbeNoX) {
        const uint32_t off = lanebase ^ static_cast<uint32_t>(k * 16);
#pragma unroll
        for (int j = 0; j < R; ++j) hv[j] = *reinterpret_cast<const uint4*>(xs + off + j * 32 * 128);
      }
    };
    auto fma_half = [&](const uint8_t* xs) {
      if constexpr (kFeedOnly) return;
      const int nk = p.f_pad / 8;  // f_pad 32: the box's zero columns 32-63 are not scored
      [[maybe_unused]] uint4 hv[R], hn[R];
      load_chunk(hv, xs, 0);
#pragma unroll 1
      for (int k = 0; k < nk; ++k) {
        load_chunk(hn, xs, k + 1 < nk ? k + 1 : k);
        const float* wk = wt_s + k * 8 * CP;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float wv[NW4 * 4];
#pragma unroll
          for (int m = 0; m < NW4; ++m) {
            if constexpr (kProbeNoW) {
#pragma unroll
              for (int i = 0; i < 4; ++i) wv[m * 4 + i] = probe_w[m * 4 + i];
            } else {
              const float4 t = *reinterpret_cast<const float4*>(wk + e * CP + m * 4);
              wv[m * 4 + 0] = t.x;
              wv[m * 4 + 1] = t.y;
              wv[m * 4 + 2] = t.z;
              wv[m * 4 + 3] = t.w;
            }
          }
#pragma unroll
          for (int j = 0; j < R; ++j) {
            if constexpr (kProbeNoX) {
              fma_feature(j, probe_x[j], wv);
            } else {
              const uint32_t word = e < 2 ? hv[j].x : e < 4 ? hv[j].y : e < 6 ? hv[j].z : hv[j].w;
              fma_feature(j, __half2float(__ushort_as_half(static_cast<unsigned short>((e & 1) ? word >> 16 : word & 0xffffu))), wv);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < R; ++j) hv[j] = hn[j];
      }
    };

    // ---- fused epilogue of the rows row0 + lane + 32 j, j < R: argmax (first maximum wins), margin guard, label store
    // (+ peer stores) ----
    auto finish_rows = [&](long long row0) {
      if constexpr (USE_F2) {
#pragma unroll
        for (int j = 0; j < R; ++j) {
#pragma unroll
          for (int i = 0; i < NPAIR; ++i) unpack2(acc2[j][i], acc[j][2 * i], acc[j][2 * i + 1]);
          if (ODD) acc[j][C - 1] = acc_last[j];
          acc[j][C] = acc_bound[j];
        }
      }
      int idxs[R];
      bool flag[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const long long row = row0 + lane + 32 * j;
        float best = acc[j][0];
        float second = -INFINITY;
        int idx = 0;
#pragma unroll
        for (int c = 1; c < C; ++c) {
          const float v = acc[j][c];
          if (v > best) {
            second = best;
            best = v;
            idx = c;
          } else {
            second = fmaxf(second, v);
          }
        }
        idxs[j] = idx;
        // certain iff margin > 2 * err, err <= (F+4) 2^-24 A; NaN/Inf anywhere makes the comparison false
        flag[j] = EXACT && row < p.n_rows && !((best - second) > p.thr * acc[j][C]);
      }
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const long long row = row0 + lane + 32 * j;
        if (row < p.n_rows) store_label_i32(p.targets, row, idxs[j]);
        if constexpr (EXACT && !QUEUE) flag_rows_warp(flag[j], row, p, lane);
      }
      if (p.targets.wire_u8 && p.targets.n_peers > 0) {
        // byte labels: transpose through shuffles so lane l < GR/4 holds rows 4l..4l+3 of a group of GR = 32 RG rows
        // and the group leaves as ONE coalesced GR-byte store per target (instead of RG int32 stores).  Row 4l+t sits
        // in byte (4l+t)/32 = l/8 of lane (4l+t) % 32's packed word.  One group per pass, except kHalf's 8 rows per
        // lane: two 128-row groups.
        constexpr int NG = HALF ? R / 4 : 1;
        constexpr int RG = R / NG;
#pragma unroll
        for (int g = 0; g < NG; ++g) {
          uint32_t packed = 0, word = 0;
#pragma unroll
          for (int j = 0; j < RG; ++j) packed |= static_cast<uint32_t>(idxs[g * RG + j]) << (8 * j);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const uint32_t w = __shfl_sync(0xffffffffu, packed, (4 * lane + t) & 31);
            word |= ((w >> (8 * (lane >> 3))) & 0xffu) << (8 * t);
          }
          store_label_word_u8(p, row0 + g * 32 * RG + 4 * lane, word, 4 * lane < 32 * RG);
        }
      }
      if constexpr (EXACT && QUEUE) {
        // hand the (rare) flagged rows to the re-score warp: the labels above are provisional for them
        unsigned masks[R];
        int total = 0;
#pragma unroll
        for (int j = 0; j < R; ++j) {
          masks[j] = __ballot_sync(0xffffffffu, flag[j]);
          total += __popc(masks[j]);
        }
        if (total > 0) {
          __threadfence();  // the provisional labels are visible before the re-score warp may overwrite them
          int base = -1;
          if (lane == 0) {
            const int tail = atomicAdd(&q_ctl[0], 0);
            const int consumed = atomicAdd(&q_ctl[3], 0);
            if (tail - consumed <= kQueueCap - HEADROOM) base = atomicAdd(&q_ctl[0], total);
          }
          base = __shfl_sync(0xffffffffu, base, 0);
          if (base >= 0) {
            int off = base;
#pragma unroll
            for (int j = 0; j < R; ++j) {
              if (flag[j]) {
                const int slot = (off + __popc(masks[j] & ((1u << lane) - 1u))) & (kQueueCap - 1);
                // (atomics, not plain volatile accesses: the queue is a lock-free hand-off between warps and the
                // race checker should see it as one)
                while (atomicAdd(&q_slots[slot], 0) != 0) {  // only if the slot's previous ticket is claimed but not read yet
                }
                atomicExch(&q_slots[slot], static_cast<int>(row0 + lane + 32 * j) + 1);
              }
              off += __popc(masks[j]);
            }
          } else {
            // the queue is backed up (most rows of the batch are near-ties): this warp re-scores its own rows, which
            // keeps the worst case at "every warp does fp64" instead of "every warp waits for one"
#pragma unroll
            for (int j = 0; j < R; ++j) {
              unsigned mask = masks[j];
              while (mask != 0u) {
                const int l = __ffs(static_cast<int>(mask)) - 1;
                mask &= mask - 1u;
                const long long row = row0 + l + 32 * j;
                const int idx64 = rescore_row_inline(p, row, lane);
                if (lane == 0) store_label(p.targets, row, idx64);
              }
            }
            if (lane == 0) atomicAdd(&p.counters[kCounterFlagged], static_cast<unsigned long long>(total));
          }
        }
      }
    };

    if constexpr (MMA) {
      // ===== kHalfMma, kByteMma: warpgroup wg = warp / 4 takes ring items wg, wg + NCU, ...; per item four m64 blocks of
      // 64 rows x NT columns, f_pad / 16 k16 steps each.  Fragment (WgmmaTf32's layout): thread (warp w, lane l) holds
      // fragment rows 16 (w % 4) + l / 4 and the row 8 below of each block, columns 8 i + 2 (l % 4) + {0, 1}: class c's
      // hi piece at c, its lo piece at NH + c, the bound column at C - all of a row in one quad ----
      constexpr int NH = linear_tc_hi_cols(C), NT = linear_tc_cols(C), NL = NT - NH;
      const int q = lane & 3;
      const float* tcb = reinterpret_cast<const float*>(static_cast<const uint8_t*>(p.tc_ops) + NT * 128);
      float bz[NH / 8][2];
#pragma unroll
      for (int i = 0; i < NH / 8; ++i) {
        bz[i][0] = __ldg(tcb + 8 * i + 2 * q);
        bz[i][1] = __ldg(tcb + 8 * i + 2 * q + 1);
      }
      const uint32_t b_base = smem_u32(smem + static_cast<size_t>(S) * STAGE_BYTES);
      const int nk = p.f_pad / 16;
      const float kappa = p.tc_kappa;
      if constexpr (BYTES) {
        // ----- kByteMma.  A comes from registers, so the kernel picks the tile row of each fragment row: warp w's
        // fragment rows of block b are tile rows 64 (w % 4) + 16 b + {l / 4, l / 4 + 8}, and every warp owns 64
        // consecutive rows of the tile.  Per block (one commit group) a thread loads its two fragment rows with one
        // LDS.128 each (the eight lanes of a phase read two whole 64-byte rows: conflict-free), widens the bytes to the
        // f16 values kHalfMma reads and issues the block's wgmma.  The stage goes back as soon as the last block's A
        // fragments are in registers (B lives outside the ring).  Once a block's group is done its scores are folded
        // as finish_mma folds them, (hi + lo) + bz, into the warp's part of a score slot, which frees the accumulators.
        // The warpgroup then posts the item and takes its next stage.  Its two epilogue warps score the posted rows
        // with the fp32 route's sequential top-2: the same values and comparisons as finish_mma's quad merge, so labels
        // and tier-1 verdicts are the same bit for bit.
        // Slots: warpgroup g's k-th item goes to slot (g, k % kEpiSlots), and g's epilogue warps walk the same
        // sequence.  Every item is posted; an unscored one (past the batch, or the sentinel) carries only its tile
        // index, and the sentinel ends both sides' loops.
        static_assert(kEpiPitch % 32 == 4 && kEpiPitch >= 64, "conflict-free write-out and reads");
        constexpr int WARP_FLOATS = (C + 1) * kEpiPitch;  // one MMA warp's part of a slot
        if (warp < NMW) {
          const int g = warp >> 2;
          // Bank of the write of (block b, half h, column 8 i + 2 q + e) by lane l = 4 t + q: (8 i + 2 q + e) * 68 + 16 b
          // + 8 h + t = 8 q + t + (32 i + 4 e + 16 b + 8 h) mod 32, so the warp's 32 lanes (t < 8, q < 4) hit 32 banks.
          auto write_out = [&](float* eb, float (&db)[NT / 2], int b) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int i = 0; i < NH / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int c = 8 * i + 2 * q + e;
                  const float lo = i < NL / 8 ? db[4 * (NH / 8 + i) + 2 * h + e] : 0.f;
                  if (c <= C) eb[c * kEpiPitch + 16 * b + 8 * h + (lane >> 2)] = (db[4 * i + 2 * h + e] + lo) + bz[i][e];
                }
          };
          // (at NT = 40, C = 16, two blocks' fragments beside 80 accumulators made ptxas serialize the wgmma chain)
          constexpr int INFLIGHT = NT >= 40 ? 1 : 2;
          uint32_t stage = static_cast<uint32_t>(g), phase = 0;
          int slot = 0;
          uint32_t slot_phase = 0;
#ifdef UML_PROBE_WAIT_CLOCKS
          long long probe_slot_wait = 0;
#endif
          for (bool first = true;; first = false) {
            UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u); mbar_wait(&full_bar[stage], phase));
            UML_PROBE_CLOCK(probe_landed);
            UML_PROBE_LANDED(first);
            const int tile = tile_slot[stage];
            const bool scored = !kFeedOnly && tile >= 0 && tile < num_tiles;
            const int es = g * kEpiSlots + slot;
            auto release = [&] {
              __syncwarp();
              if (lane == 0) mbar_arrive(&empty_bar[stage]);  // the fourth warp's arrive hands the stage back
              UML_PROBE_SINCE(probe_hold, probe_landed);
              UML_PROBE_RELEASED();
            };
            // both epilogue warps have read the slot's previous item
            auto wait_slot = [&] { UML_PROBE_TIMED(probe_slot_wait, mbar_wait(&epi_empty[es], slot_phase ^ 1u)); };
            if (scored) {
              float* eb = epi_buf + (es * 4 + (warp & 3)) * WARP_FLOATS;  // column c of the warp's row r at eb[c * kEpiPitch + r]
              float d[4][NT / 2];
              uint32_t a[4][kHalfBoxF / 16][4];
#pragma unroll
              for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int r = 0; r < NT / 2; ++r) {
                  d[b][r] = 0.f;
                  wgmma_fence_operand(d[b][r]);
                }
              const uint8_t* xs = smem + static_cast<size_t>(stage) * STAGE_BYTES + (64 * (warp & 3) + (lane >> 2)) * kByteRowBytes + 16 * q;
              // block b's group is done: its A registers may be reused, its scores go to the slot
              auto retire = [&](int b) {
#pragma unroll
                for (int k = 0; k < kHalfBoxF / 16; ++k)
#pragma unroll
                  for (int i = 0; i < 4; ++i) wgmma_fence_operand(a[b][k][i]);
#pragma unroll
                for (int r = 0; r < NT / 2; ++r) wgmma_fence_operand(d[b][r]);
                write_out(eb, d[b], b);
              };
#pragma unroll
              for (int b = 0; b < 4; ++b) {
                if (b >= INFLIGHT) {
                  wgmma_wait<INFLIGHT - 1>();
                  if (b == INFLIGHT) wait_slot();  // (under the wgmma of the blocks in flight)
                  retire(b - INFLIGHT);
                }
                const uint4 x0 = *reinterpret_cast<const uint4*>(xs + 16 * b * kByteRowBytes);
                const uint4 x1 = *reinterpret_cast<const uint4*>(xs + (16 * b + 8) * kByteRowBytes);
#pragma unroll
                for (int k = 0; k < kHalfBoxF / 16; ++k) {
                  const uint32_t w0 = k == 0 ? x0.x : k == 1 ? x0.y : k == 2 ? x0.z : x0.w;
                  const uint32_t w1 = k == 0 ? x1.x : k == 1 ? x1.y : k == 2 ? x1.z : x1.w;
                  a[b][k][0] = bytes_to_half2(w0, 0);
                  a[b][k][1] = bytes_to_half2(w1, 0);
                  a[b][k][2] = bytes_to_half2(w0, 1);
                  a[b][k][3] = bytes_to_half2(w1, 1);
                }
                if (b == 3) release();
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kHalfBoxF / 16; ++k) {
                  if (k < nk) WgmmaF16<NT>::mma_ra(d[b], a[b][k], wgmma_desc_k_sw128(b_base + 32 * k), k != 0 ? 1u : 0u);
                }
                wgmma_commit();
              }
              wgmma_wait<0>();
#pragma unroll
              for (int b = 4 - INFLIGHT; b < 4; ++b) retire(b);
            } else {
              release();
              wait_slot();
            }
            // post the item: warp 0 of the group writes the tile index, and the slot is full once all four warps'
            // scores are in (each warp's __syncwarp orders its lanes' writes before its arrive)
            if ((warp & 3) == 0 && lane == 0) epi_tile[es] = tile;
            __syncwarp();
            if (lane == 0) mbar_arrive(&epi_full[es]);
            if (tile == kTileSentinel) break;
            stage += NCU;
            if (stage >= static_cast<uint32_t>(S)) {
              stage -= S;
              phase ^= 1u;
            }
            if (++slot == kEpiSlots) {
              slot = 0;
              slot_phase ^= 1u;
            }
          }
#ifdef UML_PROBE_WAIT_CLOCKS
          if (lane == 0) atomicAdd(&p.probe_clocks[7], static_cast<unsigned long long>(probe_slot_wait));
#endif
        } else if (warp < NCW) {
          // ===== epilogue warp e = warp - NMW serves warpgroup e / 2: rows 128 h .. 128 h + 127 (h = e % 2) of each of
          // its items, lane l rows 128 h + 32 j + l (j < 4) from the parts of MMA warps 2 h (j < 2) and 2 h + 1; the reads
          // of column c are 32 consecutive words.
          // Every row has one writer: certified rows are stored here, queued rows only by the drain (which stores
          // every target of a row it takes).  So a queued row carries no provisional label that the drain's
          // store must be ordered after, and publication needs no device-scope fence: the slot's shared-memory atomic
          // carries the row index, and nothing this warp wrote to global memory is read or overwritten by the drain.
          // The byte words of peers leave out queued rows' bytes (store_label_word_u8's `keep`), so a peer's byte has
          // one writer as well.
          static_assert(C <= 16, "a label takes 4 bits of the byte-word gather");
          const int g = (warp - NMW) >> 1, h = (warp - NMW) & 1;
#ifdef UML_PROBE_WAIT_CLOCKS
          long long probe_epi_wait = 0;
#endif
          auto score_rows = [&](int es, long long row0) {
            auto hand_back = [&] {
              __syncwarp();  // every lane has read the slot
              if (lane == 0) mbar_arrive(&epi_empty[es]);
            };
            if constexpr (kProbeNoEpilogue) {
              hand_back();
              return;
            }
            const float* eb = epi_buf + (es * 4 + 2 * h) * WARP_FLOATS + lane;
            int lab[4];
            bool flg[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float* col = eb + (j >> 1) * WARP_FLOATS + 32 * (j & 1);
              float best = col[0], second = -INFINITY;
              int bi = 0;
#pragma unroll
              for (int c = 1; c < C; ++c) {
                const float v = col[c * kEpiPitch];
                if (v > best) {
                  second = best;
                  best = v;
                  bi = c;
                } else {
                  second = fmaxf(second, v);
                }
              }
              const float a = col[C * kEpiPitch];
              lab[j] = bi;
              // tier 1: certain iff margin > kappa A; NaN / Inf anywhere makes the comparison false
              flg[j] = !kProbeNoHandoff && row0 + 32 * j + lane < p.n_rows && !((best - second) > kappa * a);
            }
            hand_back();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const long long row = row0 + 32 * j + lane;
              if (row < p.n_rows && !flg[j]) store_label_i32(p.targets, row, lab[j]);
            }
            if (p.targets.wire_u8 && p.targets.n_peers > 0) {
              // lane l gathers rows 4 l .. 4 l + 3 (row 4 l + t sits in lane (4 l + t) % 32, j = l / 8) into one word,
              // and the bits of the queued ones into `keep`
              uint32_t packed = 0;
#pragma unroll
              for (int j = 0; j < 4; ++j) packed |= static_cast<uint32_t>(lab[j]) << (4 * j) | (flg[j] ? 1u << (16 + j) : 0u);
              uint32_t word = 0;
              unsigned keep = 0;
#pragma unroll
              for (int t = 0; t < 4; ++t) {
                const uint32_t w = __shfl_sync(0xffffffffu, packed, (4 * lane + t) & 31);
                word |= ((w >> (4 * (lane >> 3))) & 0xfu) << (8 * t);
                keep |= ((w >> (16 + (lane >> 3))) & 1u) ? 0u : 1u << t;
              }
              store_label_word_u8(p, row0 + 4 * lane, word, true, keep);
            }
            unsigned masks[4];
            int total = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              masks[j] = __ballot_sync(0xffffffffu, flg[j]);
              total += __popc(masks[j]);
            }
            if (total == 0) return;
            // When the queue is backed up (most rows near-ties) the warp waits for room: the drain never waits for an
            // epilogue warp, so the wait ends
            int base = -1;
            if (lane == 0) {
              for (;;) {
                const int tail = atomicAdd(&q_ctl[0], 0);
                const int consumed = atomicAdd(&q_ctl[3], 0);
                if (tail - consumed <= kQueueCap - HEADROOM) break;
                __nanosleep(500);
              }
              base = atomicAdd(&q_ctl[0], total);
            }
            int off = __shfl_sync(0xffffffffu, base, 0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (flg[j]) {
                const int slot = (off + __popc(masks[j] & ((1u << lane) - 1u))) & (kQueueCap - 1);
                while (atomicAdd(&q_slots[slot], 0) != 0) {  // only if the slot's previous ticket is claimed but not read yet
                }
                atomicExch(&q_slots[slot], static_cast<int>(row0 + 32 * j + lane) + 1);
              }
              off += __popc(masks[j]);
            }
          };
          int slot = 0;
          uint32_t slot_phase = 0;
          for (;;) {
            const int es = g * kEpiSlots + slot;
            UML_PROBE_TIMED(probe_epi_wait, mbar_wait(&epi_full[es], slot_phase));
            const int tile = epi_tile[es];
            if (tile == kTileSentinel) break;
            if (!kFeedOnly && tile < num_tiles) {
              score_rows(es, static_cast<long long>(tile) * TILE + 128 * h);
            } else {
              __syncwarp();
              if (lane == 0) mbar_arrive(&epi_empty[es]);
            }
            if (++slot == kEpiSlots) {
              slot = 0;
              slot_phase ^= 1u;
            }
          }
#ifdef UML_PROBE_WAIT_CLOCKS
          if (lane == 0) {
            atomicAdd(&p.probe_clocks[8], static_cast<unsigned long long>(probe_epi_wait));
            atomicAdd(&p.probe_clocks[9], static_cast<unsigned long long>(clock64() - probe_start));
          }
#endif
        }
      } else {
        // ----- kHalfMma: one commit group per item; the stage goes back after the wait, the epilogue runs from registers
        const long long row_in = 16 * (warp & 3) + (lane >> 2);  // row of fragment row-half 0 in block 0
        // scores, top-2 and the tier-1 guard of the 8 rows whose columns this thread's quad holds; quad lane q then stores
        // and (if not certified) publishes the two rows of block q, so every row leaves once
        auto finish_mma = [&](float (&d)[4][NT / 2], long long row0) {
          int lab[4][2];
          bool flg[4][2];
#pragma unroll
          for (int b = 0; b < 4; ++b) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float best = -INFINITY, second = -INFINITY, bound = 0.f;
              int bi = C;  // a thread without classes loses every tie
#pragma unroll
              for (int i = 0; i < NH / 8; ++i) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int c = 8 * i + 2 * q + e;
                  const float lo = i < NL / 8 ? d[b][4 * (NH / 8 + i) + 2 * h + e] : 0.f;
                  const float v = (d[b][4 * i + 2 * h + e] + lo) + bz[i][e];
                  if (c < C) {
                    if (v > best) {
                      second = best;
                      best = v;
                      bi = c;
                    } else {
                      second = fmaxf(second, v);
                    }
                  } else if (c == C) {
                    bound = v;
                  }
                }
              }
              // merge over the quad: the larger score wins, the lower class on a tie (first maximum, like np.argmax)
#pragma unroll
              for (int off = 1; off <= 2; off <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, off);
                const float os = __shfl_xor_sync(0xffffffffu, second, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                if (ob > best || (ob == best && oi < bi)) {
                  second = fmaxf(best, os);
                  best = ob;
                  bi = oi;
                } else {
                  second = fmaxf(second, ob);
                }
              }
              const float a = __shfl_sync(0xffffffffu, bound, (lane & ~3) | ((C % 8) / 2));
              const long long row = row0 + b * 64 + row_in + 8 * h;
              lab[b][h] = bi;
              // tier 1: certain iff margin > kappa A; NaN / Inf anywhere makes the comparison false
              flg[b][h] = row < p.n_rows && !((best - second) > kappa * a);
            }
          }
          unsigned masks[2];
          int total = 0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int idx = q == 0 ? lab[0][h] : q == 1 ? lab[1][h] : q == 2 ? lab[2][h] : lab[3][h];
            const bool flag = q == 0 ? flg[0][h] : q == 1 ? flg[1][h] : q == 2 ? flg[2][h] : flg[3][h];
            const long long row = row0 + q * 64 + row_in + 8 * h;
            if (row < p.n_rows) store_label(p.targets, row, idx);
            masks[h] = __ballot_sync(0xffffffffu, flag);
            total += __popc(masks[h]);
          }
          if (total == 0) return;
          // the (few) uncertified rows go to the re-score warp, as in finish_rows: the labels above are provisional.  When
          // the queue is backed up (most rows near-ties) the warp waits for room instead of settling its rows itself: a
          // call from this loop made ptxas save the loop's live registers around it, spill stores and loads in the hot
          // path at every class count (-Xptxas -v).  The drain never waits for a scoring warp, so the wait ends.
          auto row_of = [&](int l, int h) { return row0 + (l & 3) * 64 + 16 * (warp & 3) + (l >> 2) + 8 * h; };
          __threadfence();
          int base = -1;
          if (lane == 0) {
            for (;;) {
              const int tail = atomicAdd(&q_ctl[0], 0);
              const int consumed = atomicAdd(&q_ctl[3], 0);
              if (tail - consumed <= kQueueCap - HEADROOM) break;
              __nanosleep(500);
            }
            base = atomicAdd(&q_ctl[0], total);
          }
          base = __shfl_sync(0xffffffffu, base, 0);
          int off = base;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if ((masks[h] >> lane) & 1u) {
              const int slot = (off + __popc(masks[h] & ((1u << lane) - 1u))) & (kQueueCap - 1);
              while (atomicAdd(&q_slots[slot], 0) != 0) {
              }
              atomicExch(&q_slots[slot], static_cast<int>(row_of(lane, h)) + 1);
            }
            off += __popc(masks[h]);
          }
        };
        uint32_t stage = static_cast<uint32_t>(warp >> 2), phase = 0;
        for (bool first = true; scoring_warp; first = false) {
          UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u); mbar_wait(&full_bar[stage], phase));
          UML_PROBE_CLOCK(probe_landed);
          UML_PROBE_LANDED(first);
          const int tile = tile_slot[stage];
          const bool scored = !kFeedOnly && tile >= 0 && tile < num_tiles;
          float d[4][NT / 2];
          if (scored) {
            [[maybe_unused]] const uint32_t a_base = smem_u32(smem + static_cast<size_t>(stage) * STAGE_BYTES);
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
              for (int r = 0; r < NT / 2; ++r) {
                d[b][r] = 0.f;
                wgmma_fence_operand(d[b][r]);
              }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kHalfBoxF / 16; ++k) {
              if (k < nk) {  // f_pad 32: the box's zero columns 32-63 are not multiplied
                const uint64_t bd = wgmma_desc_k_sw128(b_base + 32 * k);
#pragma unroll
                for (int b = 0; b < 4; ++b)
                  WgmmaF16<NT>::mma(d[b], wgmma_desc_k_sw128(a_base + b * 64 * 128 + 32 * k), bd, k != 0 ? 1u : 0u);
              }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
              for (int r = 0; r < NT / 2; ++r) wgmma_fence_operand(d[b][r]);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);  // the fourth warp's arrive hands the stage back
          UML_PROBE_SINCE(probe_hold, probe_landed);
          UML_PROBE_RELEASED();
          if (tile == kTileSentinel) break;
          stage += NCU;
          if (stage >= static_cast<uint32_t>(S)) {
            stage -= S;
            phase ^= 1u;
          }
          if (scored) finish_mma(d, static_cast<long long>(tile) * TILE);
        }
      }
    } else if constexpr (CLAIMED) {
      // this warp's ring items are n = warp, warp + NCW, ... (stage n % S, phase (n / S) & 1); S >= NCW lets stage and
      // phase advance without a division.  Both waits keep the invariant argued below: the next item is n + NCW <= n + S.
      uint32_t stage = static_cast<uint32_t>(warp), phase = 0;
      for (bool first = true; scoring_warp; first = false) {
        init_acc();
        UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u); mbar_wait(&full_bar[stage], phase));
        UML_PROBE_CLOCK(probe_landed);
        UML_PROBE_LANDED(first);
        const int tile = tile_slot[stage];
        const bool scored = tile >= 0 && tile < num_tiles;
        if (scored) {
          const uint8_t* xs = smem + static_cast<size_t>(stage) * STAGE_BYTES;
          if constexpr (HALF) {
            // NPASS > 1: every pass but the last is finished while the stage is held, the last one after its release
#pragma unroll
            for (int pass = 0; pass < NPASS; ++pass) {
              if (pass > 0) {
                finish_rows(static_cast<long long>(tile) * TILE + (pass - 1) * 32 * R);
                init_acc();
              }
              fma_half(xs + pass * 32 * R * 128);
            }
          } else {
            fma_box(xs, wt_s);
            fma_box(xs + BOX_BYTES, wt_s + kChunkF * CP);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);  // hand the stage back to the producer
        UML_PROBE_SINCE(probe_hold, probe_landed);
        UML_PROBE_RELEASED();
        if (tile == kTileSentinel) break;
        stage += NCW;
        if (stage >= static_cast<uint32_t>(S)) {
          stage -= S;
          phase ^= 1u;
        }
        if (scored) finish_rows(static_cast<long long>(tile) * TILE + (NPASS - 1) * 32 * R);
      }
    } else {
      uint32_t seq_base = 0;
      for (long long first = blockIdx.x; scoring_warp && first < num_tiles; first += G * kConsumerWarps) {
        const int nv = static_cast<int>(min(static_cast<long long>(kConsumerWarps), (num_tiles - first + G - 1) / G));
        if (warp < nv) {
          const long long tile = first + warp * G;
          init_acc();
          for (int k = 0; k < KC; ++k) {
            const uint32_t seq = seq_base + static_cast<uint32_t>(k * nv + warp);
            const uint32_t stage = seq % static_cast<uint32_t>(S);
            const uint32_t phase = (seq / static_cast<uint32_t>(S)) & 1u;
            // A parity wait can only tell the current phase from the one before it.  Several warps share this ring
            // and TMA completions are unordered, so the previous occupant of the stage (item seq - S, another warp's)
            // may still be in flight or unread when this warp gets here; waiting on `full` right away would then
            // match the *older* phase and read another tile's half-landed box.  First wait until that occupant has
            // been released (empty phase seq/S - 1), then for our own data.  Both waits are at most one phase ahead
            // of their barrier because a warp's next item is seq + nv <= seq + kConsumerWarps and the ring has
            // S >= kConsumerWarps stages: the producer could only issue item seq after item seq - S was released, so
            // item seq + nv - 2S was too.
            UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u); mbar_wait(&full_bar[stage], phase));
            UML_PROBE_CLOCK(probe_landed);
            UML_PROBE_LANDED(seq == 0);
            fma_box(smem + static_cast<size_t>(stage) * kStageBytes, wt_s + k * kChunkF * CP);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);  // hand the stage back to the producer
            UML_PROBE_SINCE(probe_hold, probe_landed);
            UML_PROBE_RELEASED();
          }
          finish_rows(tile * TILE);
        }
        seq_base += static_cast<uint32_t>(KC * nv);
      }
    }
#ifdef UML_PROBE_TIMELINE
    if (scoring_warp && lane == 0 && probe_last_release != 0) atomicMax(&p.probe_timeline[blockIdx.x * kProbeStamps + 3], probe_last_release);
#endif
#ifdef UML_PROBE_WAIT_CLOCKS
    if (scoring_warp && lane == 0) {
      atomicAdd(&p.probe_clocks[2], static_cast<unsigned long long>(probe_wait));
      atomicAdd(&p.probe_clocks[3], static_cast<unsigned long long>(clock64() - probe_start));
      atomicAdd(&p.probe_clocks[4], static_cast<unsigned long long>(probe_hold));
    }
#endif
    if constexpr (EXACT && QUEUE) {
      if (BYTES ? warp >= NMW && warp < NCW : warp < NCW) {
        __syncwarp();
        if (lane == 0) {
          __threadfence_block();
          atomicAdd(&q_ctl[2], 1);  // this warp has published everything it will ever publish
        }
      }
      // ===================== fp64 re-score: warp 9 drains the queue while the scoring warps stream; a scoring warp
      // that has finished its tiles joins in, so a long tail of flagged rows (wide rows, many near-ties) is shared
      // by all ten warps instead of waiting for one =====================
      int n_done = 0;
#ifdef UML_PROBE_WAIT_CLOCKS
      long long probe_busy = 0, probe_f64 = 0, probe_rows = 0;
#endif
      if constexpr (MMA) {
        // tier 2 in batches of 32 rows, one per lane.  While publishers are still running a batch starts only when 32
        // tickets are reserved (at about one row every few thousand cycles, smaller batches would mostly hold one row);
        // once all have published, what is left is split evenly over the NCW + 1 warps that drain, so that the float64
        // rows of the CTA's last batch do not run one after another in one warp.  Labels are due at the end of the grid
        // only, and the queue holds 2048 rows against ~100 per CTA, so the wait costs nothing.  Tickets are claimed
        // with a CAS on the head, so every claimed ticket is reserved and its row is being published.
#ifdef UML_PROBE_TIMELINE
        bool probe_saw_done = false;
#endif
        for (;;) {
          int t0 = 0, n = 0;
          if (lane == 0) {
            for (;;) {
              const bool done = atomicAdd(&q_ctl[2], 0) == NPUB;
              __threadfence_block();  // the tail read below is final once `done` is seen
#ifdef UML_PROBE_TIMELINE
              if (done && !probe_saw_done) UML_PROBE_STAMP_MIN(5);
              probe_saw_done = done;
#endif
              const int head = atomicAdd(&q_ctl[1], 0);
              const int avail = atomicAdd(&q_ctl[0], 0) - head;
              if (done && avail <= 0) break;
              if (done || avail >= 32) {
                n = done ? min((avail + NCW) / (NCW + 1), 32) : 32;
                if (atomicCAS(&q_ctl[1], head, head + n) == head) {
                  t0 = head;
                  UML_PROBE_STAMP_MAX(6);
                  break;
                }
                n = 0;
                continue;
              }
              __nanosleep(200);
            }
          }
          n = __shfl_sync(0xffffffffu, n, 0);
          t0 = __shfl_sync(0xffffffffu, t0, 0);
          if (n == 0) break;
          UML_PROBE_CLOCK(probe_batch);
          // lane i takes ticket t0 + i: its publisher has reserved it, so the slot is written soon
          long long row = -1;
          if (lane < n) {
            int* slot = &q_slots[(t0 + lane) & (kQueueCap - 1)];
            int v;
            while ((v = atomicAdd(slot, 0)) == 0) {
            }
            atomicExch(slot, 0);
            row = static_cast<long long>(v) - 1;
          }
          __syncwarp();
          if (lane == 0) atomicAdd(&q_ctl[3], n);
          const bool certified = replay_fp32_rows<C>(p, wt_s, bias_s, row);
          if (lane == 0) UML_PROBE_STAMP_MAX(7);
          // the rows the fp32 route would flag go to fp64 one at a time, by the whole warp (they count in n_flagged)
          UML_PROBE_CLOCK(probe_f64_start);
          for (unsigned todo = __ballot_sync(0xffffffffu, row >= 0 && !certified); todo != 0; todo &= todo - 1) {
            const long long r = __shfl_sync(0xffffffffu, row, __ffs(todo) - 1);
            const int idx64 = rescore_row_tc<C>(p, r, lane);
            if (lane == 0) {
              store_label(p.targets, r, idx64);
              UML_PROBE_STAMP_MAX(8);
            }
            ++n_done;
          }
          UML_PROBE_SINCE(probe_f64, probe_f64_start);
          UML_PROBE_SINCE(probe_busy, probe_batch);
#ifdef UML_PROBE_WAIT_CLOCKS
          probe_rows += n;
#endif
        }
      } else {
        for (;;) {
          // claim the next ticket, then wait until its slot is published (lane 0 polls and broadcasts: the lanes of a
          // warp need not run in lockstep)
          int t = 0;
          if (lane == 0) t = atomicAdd(&q_ctl[1], 1);
          t = __shfl_sync(0xffffffffu, t, 0);
          int v = 0;
          for (;;) {
            int state = 0;  // 1: nothing will ever be published for this ticket
            if (lane == 0) {
              v = atomicAdd(&q_slots[t & (kQueueCap - 1)], 0);
              if (v == 0 && atomicAdd(&q_ctl[2], 0) == NPUB) {
                __threadfence_block();
                if (t >= atomicAdd(&q_ctl[0], 0)) state = 1;
              }
            }
            v = __shfl_sync(0xffffffffu, v, 0);
            state = __shfl_sync(0xffffffffu, state, 0);
            if (v != 0 || state == 1) break;
            __nanosleep(200);
          }
          if (v == 0) break;
          if (lane == 0) {
            atomicExch(&q_slots[t & (kQueueCap - 1)], 0);
            atomicAdd(&q_ctl[3], 1);
          }
          const long long row = static_cast<long long>(v) - 1;
          UML_PROBE_CLOCK(probe_row);
          const int idx64 = rescore_row_inline(p, row, lane);
          if (lane == 0) store_label(p.targets, row, idx64);
          ++n_done;
          UML_PROBE_SINCE(probe_busy, probe_row);
#ifdef UML_PROBE_WAIT_CLOCKS
          ++probe_rows;
#endif
        }
      }
#ifdef UML_PROBE_WAIT_CLOCKS
      if (warp == NCW + 1 && lane == 0) {
        atomicAdd(&p.probe_clocks[5], static_cast<unsigned long long>(probe_busy));
        atomicAdd(&p.probe_clocks[6], static_cast<unsigned long long>(clock64() - probe_start));
        atomicAdd(&p.probe_clocks[10], static_cast<unsigned long long>(MMA ? probe_f64 : probe_busy));
      }
      if (lane == 0 && probe_rows > 0) atomicAdd(&p.probe_clocks[11], static_cast<unsigned long long>(probe_rows));
#endif
      if (lane == 0 && n_done > 0) atomicAdd(&p.counters[kCounterFlagged], static_cast<unsigned long long>(n_done));
    }
  }
#ifdef UML_PROBE_TIMELINE
  if (lane == 0) atomicMax(&p.probe_timeline[blockIdx.x * kProbeStamps + 4], probe_globaltimer());
#endif
}

// ---------------------------------------------------------------------------------------------------------------
// fp64 re-score / generic kernel: warp per row, lanes over features
// ---------------------------------------------------------------------------------------------------------------
struct RescoreParams {
  const float* x;
  const double* x64;
  SrcView src;
  long long ld, ld64;
  long long n_rows;
  const double* w64;  // [F][w64_stride], feature-major
  const double* b64;
  int w64_stride;
  int n_classes, n_features;
  const int* flag_count;
  const int32_t* flag_rows;
  int flag_cap;
  int all_rows;
  LabelTargets targets;
  unsigned long long* counters;
  int smem_weights;              // W, b staged in dynamic shared memory ((C F + 2 C) doubles)
  double fold_rel;
  int binary;
};


// rows [warp_global, n) step warps_total of the flag list (or of the batch), one warp per row
template <typename WPTR>
__device__ __forceinline__ void rescore_rows(const RescoreParams& p, WPTR w64, WPTR b64, long long n, int lane,
                                             long long warp_global, long long warps_total) {
  const int F = p.n_features, C = p.n_classes, S = p.w64_stride;
  for (long long i = warp_global; i < n; i += warps_total) {
    const long long row = p.all_rows ? i : static_cast<long long>(p.flag_rows[i]);
    RowScore r;
    if (p.src.base) {
      const SrcView v = p.src;
      r = score_row_f64([&](int f) { return load_src(v, row, f); }, w64, S, b64, F, C, p.fold_rel, p.binary != 0, lane);
    } else if (p.x64) {
      const double* xr64 = p.x64 + row * p.ld64;
      r = score_row_f64([&](int f) { return xr64[f]; }, w64, S, b64, F, C, p.fold_rel, p.binary != 0, lane);
    } else {
      const float* xr = p.x + row * p.ld;
      r = score_row_f64([&](int f) { return static_cast<double>(xr[f]); }, w64, S, b64, F, C, p.fold_rel, p.binary != 0, lane);
    }
    if (lane == 0) {
      store_label(p.targets, row, r.idx);
      count_rescored_row(p, r.bad, r.ambiguous);
    }
  }
}

__global__ void __launch_bounds__(256) rescore_f64_kernel(const RescoreParams p) {
  // W (fp64, feature-major [F][S]) and b are staged in shared memory when they fit (p.smem_weights): a wide model
  // (784 x 10 = 62 KB) would otherwise be re-read from L2 for every re-scored row.  Two copies of the row loop so that
  // the shared-memory one compiles to LDS.128 (a pointer chosen at run time would make every weight load generic).
  extern __shared__ __align__(16) double rs_w[];
  const int nw = p.n_features * p.w64_stride;
  if (p.smem_weights) {
    const double2* src = reinterpret_cast<const double2*>(p.w64);
    double2* dst = reinterpret_cast<double2*>(rs_w);
    for (int i = threadIdx.x; i < nw / 2; i += blockDim.x) dst[i] = src[i];
    for (int i = threadIdx.x; i < 2 * p.n_classes; i += blockDim.x) rs_w[nw + i] = p.b64[i];  // biases + magnitudes
    __syncthreads();
  }
  pdl_wait_for_predecessor();  // the flag list is written by the scoring kernel this launch depends on
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long n = flag_list_rows(p);
  if (p.smem_weights) {
    const double* ws = rs_w;
    rescore_rows(p, ws, ws + nw, n, lane, warp_global, warps_total);
  } else {
    rescore_rows(p, p.w64, p.b64, n, lane, warp_global, warps_total);
  }
  flag_list_hand_back(p);
}

// ---------------------------------------------------------------------------------------------------------------
// small-batch kernel of the online path (fastapi.py:50-64, B <= 64 rows): one warp per row, float64 scores straight
// from the request's raw feature block (any dtype / order) - no staging pass, no guard, exact by construction
// ---------------------------------------------------------------------------------------------------------------
struct SmallParams {
  SrcView src;
  const double* w64;  // [F][w64_stride], feature-major
  const double* b64;
  int w64_stride;
  int n_classes, n_features, n_rows;
  double fold_rel;
  int binary;
  SmallResult* out;
};

__global__ void __launch_bounds__(256) linear_small_kernel(const SmallParams p) {
  const int lane = threadIdx.x & 31;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= p.n_rows) return;
  const SrcView v = p.src;
  const RowScore r = score_row_f64([&](int f) { return load_src(v, row, f); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, p.fold_rel, p.binary != 0, lane);
  if (lane == 0) {
    p.out[row].label = r.idx;
    p.out[row].status = (r.bad ? 1 : 0) | (r.ambiguous ? 2 : 0);
  }
}

cudaError_t launch_linear_small(const LinearDeviceModel& m, const SrcView& src, int n_rows, SmallResult* out,
                                cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  SmallParams p{};
  p.src = src;
  p.w64 = m.w64;
  p.w64_stride = m.w64_stride;
  p.b64 = m.b64;
  p.n_classes = m.n_classes;
  p.n_features = m.n_features;
  p.n_rows = n_rows;
  p.fold_rel = m.fold_rel;
  p.binary = m.binary;
  p.out = out;
  linear_small_kernel<<<(n_rows + 7) / 8, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// class probabilities: softmax of the fp32 scores (sigmoid for the binary layout, which the model stores expanded as
// scores [0, s]: softmax([0, s]) = [1 - sigmoid(s), sigmoid(s)], sklearn/linear_model/_logistic.py predict_proba)
// ---------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) linear_proba_kernel(const float* __restrict__ x, long long ld, long long n_rows,
                                                           const float* __restrict__ wt, const float* __restrict__ bias,
                                                           int F, int cp, float* __restrict__ proba) {
  extern __shared__ float proba_smem[];
  float* wt_s = proba_smem;  // [F][cp]
  for (int i = threadIdx.x; i < F * cp; i += blockDim.x) wt_s[i] = __ldg(wt + i);
  __syncthreads();
  for (long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; row < n_rows;
       row += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* xr = x + row * ld;
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = __ldg(bias + c);
    int f = 0;
    for (; f + 4 <= F; f += 4) {  // rows are 16-byte aligned (ld % 4 == 0)
      const float4 v = *reinterpret_cast<const float4*>(xr + f);
      const float xs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float* wrow = wt_s + (f + e) * cp;
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] = fmaf(xs[e], wrow[c], acc[c]);
      }
    }
    for (; f < F; ++f) {
      const float xv = xr[f];
      const float* wrow = wt_s + f * cp;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] = fmaf(xv, wrow[c], acc[c]);
    }
    float mx = acc[0];
#pragma unroll
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, acc[c]);
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      acc[c] = expf(acc[c] - mx);
      sum += acc[c];
    }
    const float inv = 1.0f / sum;
    float* out = proba + row * C;
#pragma unroll
    for (int c = 0; c < C; ++c) out[c] = acc[c] * inv;
  }
}

// any number of classes: scores go through the output row (used as scratch), then max / exp / normalise in place
__global__ void __launch_bounds__(256) linear_proba_generic_kernel(const float* __restrict__ x, long long ld,
                                                                   long long n_rows, const float* __restrict__ wt,
                                                                   const float* __restrict__ bias, int F, int C, int cp,
                                                                   float* __restrict__ proba) {
  for (long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; row < n_rows;
       row += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* xr = x + row * ld;
    float* out = proba + row * C;
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) {
      float s = __ldg(bias + c);
      for (int f = 0; f < F; ++f) s = fmaf(xr[f], __ldg(wt + static_cast<long long>(f) * cp + c), s);
      out[c] = s;
      mx = fmaxf(mx, s);
    }
    float sum = 0.f;
    for (int c = 0; c < C; ++c) {
      const float e = expf(out[c] - mx);
      out[c] = e;
      sum += e;
    }
    const float inv = 1.0f / sum;
    for (int c = 0; c < C; ++c) out[c] *= inv;
  }
}

cudaError_t launch_linear_proba(const LinearDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, float* proba,
                                int sm_count, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  const long long want = (n_rows + 255) / 256;
  const int grid = static_cast<int>(std::min<long long>(want, static_cast<long long>(sm_count) * 8));
  const size_t smem = static_cast<size_t>(m.n_features) * m.cp * 4;
  const int F = m.n_features, cp = m.cp;
  if (m.n_classes <= kMaxClassesTma && smem <= 160 * 1024) {
    switch (m.n_classes) {
#define UML_PCASE(N)                                                                                              \
  case N: {                                                                                                       \
    auto kern = linear_proba_kernel<N>;                                                                           \
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)); \
    if (err != cudaSuccess) return err;                                                                           \
    kern<<<grid, 256, smem, stream>>>(x, ld, n_rows, m.wt, m.bias, F, cp, proba);                                 \
    return cudaGetLastError();                                                                                    \
  }
      UML_PCASE(2) UML_PCASE(3) UML_PCASE(4) UML_PCASE(5) UML_PCASE(6) UML_PCASE(7) UML_PCASE(8) UML_PCASE(9)
      UML_PCASE(10) UML_PCASE(11) UML_PCASE(12) UML_PCASE(13) UML_PCASE(14) UML_PCASE(15) UML_PCASE(16)
#undef UML_PCASE
      default:
        break;
    }
  }
  linear_proba_generic_kernel<<<grid, 256, 0, stream>>>(x, ld, n_rows, m.wt, m.bias, F, m.n_classes, cp, proba);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// ---- tensor-core operands of the linear tile kernel (DESIGN.md 3.1, 3.2) ----
// the fp16 value nearest to v (ties to even; up: the smallest fp16 value >= v), for |v| below 2^16
static double f16_round(double v, bool up = false) {
  if (v == 0.0) return v;
  int e = 0;
  std::frexp(std::fabs(v), &e);  // |v| in [2^(e-1), 2^e): 11 significant bits, or the subnormal spacing 2^-24
  const int q = std::max(e - 11, -24);
  const double m = std::ldexp(v, -q);
  return std::ldexp(up ? std::ceil(m) : std::nearbyint(m), q);
}
// bit pattern of an fp16 value held exactly in v
static uint16_t f16_bits(double v) {
  const uint16_t sign = std::signbit(v) ? 0x8000u : 0u;
  const double a = std::fabs(v);
  if (a < 0x1p-14) return sign | (uint16_t)std::ldexp(a, 24);
  int e = 0;
  const double m = std::frexp(a, &e);  // a = m 2^e, m in [0.5, 1)
  return sign | (uint16_t)((e + 14) << 10) | (uint16_t)std::ldexp(m * 2.0 - 1.0, 10);
}
// per-k16-step budget of the f16 wgmma accumulation, in u = 2^-24 of the running |.| sum (DESIGN.md 3.2): above the
// 36u of a truncating aligner without guard bits over 16 products and the accumulator ((2 x 17 + 2) u, the model of
// 3.3), and at least 4x the worst that tests/test_gpu_wgmma_f16_accum.py measures on the hardware
constexpr double kTcStepBudget = 64.0;
// The B operand image of LinearDeviceModel::tc_ops and the certification factor, or false when the model does not take
// the tensor-core schedule: a folded affine map (its score error is bounded in the fp64 terms only), non-finite weights,
// or magnitudes at which the scaled A of DESIGN.md 3.2 could leave the normal fp32 range.  wt / bias are the fp32
// route's operands (its bound column and bias bound are what tier 1 must dominate).
bool build_tc_operands(const std::vector<double>& w, const std::vector<double>& b, const std::vector<float>& wt,
                              const std::vector<float>& bias, int C, int F, int f_pad, int cp, double fold_rel,
                              std::vector<uint8_t>* image, float* kappa) {
  if (f_pad > uml::kHalfBoxF || fold_rel != 0.0) return false;
  double wabs = 0.0;
  for (double v : w) {
    if (!std::isfinite(v)) return false;
    wabs = std::max(wabs, std::fabs(v));
  }
  for (int c = 0; c < C; ++c)
    if (!std::isfinite(b[c])) return false;
  int ex = 0;
  if (wabs > 0.0) std::frexp(wabs, &ex);  // wabs < 2^ex
  const int sigma = 15 - ex;               // max |w| 2^sigma in [2^14, 2^15): every hi piece is a normal fp16 value
  double wsum = 0.0;
  for (int f = 0; f < F; ++f) wsum += wt[(size_t)f * cp + C];
  const double a32 = (double)bias[C] + 65504.0 * wsum;  // the fp32 route's A of the largest fp16 row
  if (!(std::ldexp(a32, std::max(sigma, 0)) < 0x1p100) || !(std::ldexp((double)bias[C], sigma) > 0x1p-100)) return false;
  const int NH = uml::linear_tc_hi_cols(C), N = uml::linear_tc_cols(C);
  std::vector<uint16_t> bt((size_t)N * uml::kHalfBoxF, 0);
  // column n's 128-byte row, its 16-byte chunks XOR-swizzled by (n & 7): the SWIZZLE_128B K-major layout
  auto put = [&](int n, int f, double v) { bt[(size_t)n * 64 + (((f / 8) ^ (n & 7)) * 8) + f % 8] = f16_bits(v); };
  for (int f = 0; f < F; ++f) {
    double wmax = std::ldexp((double)wt[(size_t)f * cp + C], sigma);
    for (int c = 0; c < C; ++c) {
      const double v = std::ldexp(w[(size_t)c * F + f], sigma);
      const double hi = f16_round(v);
      put(c, f, hi);
      put(NH + c, f, f16_round(v - hi));
      wmax = std::max(wmax, std::fabs(v));
    }
    // floored at 2^-3 so that 2^-22 of it covers the 2^-25 a subnormal piece errs by (hi + lo errs by <= 2^-21 of it).
    // The fp32 route's FLT_MIN floor can scale past fp16 when every weight is below 2^-127: no route then.
    const double wb = f16_round(std::max(wmax, 0.125), true);
    if (!(wb <= 65504.0)) return false;
    put(C, f, wb);
  }
  std::vector<float> tb(NH, 0.f);
  for (int c = 0; c < C; ++c) tb[c] = (float)std::ldexp(b[c], sigma);
  tb[C] = (float)std::ldexp((double)bias[C], sigma);  // exact: a power-of-two multiple of an fp32 value in range
  image->assign((size_t)N * 128 + tb.size() * 4, 0);
  std::memcpy(image->data(), bt.data(), (size_t)N * 128);
  std::memcpy(image->data() + (size_t)N * 128, tb.data(), tb.size() * 4);
  // tier 1 certifies iff margin > 2 Etc + 2.5 thr A32+ (DESIGN.md 3.2): Etc <= e_rel A, A <= Ahat / (1 - step)
  const double u = uml::kU;
  const double step = kTcStepBudget * u * (f_pad / 16);
  const double e_rel = (0x1p-21 + step * (1.0 + 0x1p-10) + 4.0 * u) * (1.0 + 0x1p-10);
  const double thr = uml::linear_margin_thr(F);
  *kappa = (float)((2.0 * e_rel + 2.5 * thr * (1.0 + (F + 2.0) * u)) / (1.0 - step) * (1.0 + 0x1p-10));
  return true;
}


static size_t tma_fixed_smem(const LinearDeviceModel& m, bool claimed = false) {
  // alignment slack + W^T + bias + barriers (64 stages max) + the flagged-row queue of the QUEUE kernels (+ the tile
  // index of each stage, claimed schedules)
  return 1024 + static_cast<size_t>(m.f_pad) * m.cp * 4 + static_cast<size_t>(m.cp) * 4 + 2 * 64 * 8 + (kQueueCap + 4) * 4 +
         (claimed || linear_whole_rows(m.f_pad) ? 64 * 4 : 0);
}

bool linear_tma_supported(const LinearDeviceModel& m, std::string* why) {
  if (m.n_classes < 2 || m.n_classes > kMaxClassesTma) {
    if (why) *why = "n_classes outside [2,16] for the register-tiled kernel";
    return false;
  }
  // the ring protocol needs at least as many stages as consumer warps (see the comment at the consumers' waits)
  if (tma_fixed_smem(m) + kConsumerWarps * static_cast<size_t>(kStageBytes) > static_cast<size_t>(kMaxSmemBytes)) {
    if (why) *why = "W^T does not fit in shared memory next to an 8-stage ring";
    return false;
  }
  return true;
}

template <int C, bool EXACT, bool QUEUE, LinearSched SCHED>
static cudaError_t launch_one(const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                              cudaStream_t stream) {
  auto kern = linear_argmax_tma_kernel<C, EXACT, QUEUE, SCHED>;
  static size_t configured = 0;  // per instantiation (one device per process): set the attribute once, not per launch
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  kern<<<grid, linear_threads(SCHED, QUEUE), smem, stream>>>(xmap, p);
  return cudaGetLastError();
}

template <bool EXACT, bool QUEUE, LinearSched SCHED>
static cudaError_t dispatch_classes(int C, const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                                    cudaStream_t stream) {
  switch (C) {
#define UML_CASE(N) \
  case N:           \
    return launch_one<N, EXACT, QUEUE, SCHED>(xmap, p, grid, smem, stream);
#ifdef UML_PROBE_CLASSES  // diagnostic builds compile only the class count they launch
    UML_CASE(UML_PROBE_CLASSES)
#else
    UML_CASE(2) UML_CASE(3) UML_CASE(4) UML_CASE(5) UML_CASE(6) UML_CASE(7) UML_CASE(8) UML_CASE(9) UML_CASE(10)
    UML_CASE(11) UML_CASE(12) UML_CASE(13) UML_CASE(14) UML_CASE(15) UML_CASE(16)
#endif
#undef UML_CASE
    default:
      return cudaErrorInvalidValue;
  }
}

bool linear_queue_rescore() {
  // UML_B200_RESCORE_MODE=queue: flagged rows go through a shared-memory queue to a tenth warp of the tile kernel that
  // re-scores them in fp64 while the other warps keep streaming (one launch per step); =kernel: flag list in global
  // memory + rescore_f64_kernel behind the tile kernel (two launches).  Default below.
  static const int mode = [] {
    const char* env = getenv("UML_B200_RESCORE_MODE");
    if (env && env[0] == 'q') return 1;
    if (env && env[0] == 'k') return 0;
    return UML_RESCORE_QUEUE_DEFAULT;
  }();
  return mode == 1;
}

cudaError_t launch_linear_tma(const CUtensorMap& xmap, const CUtensorMap* half_map, const CUtensorMap* byte_map,
                              const LinearDeviceModel& m, const LinearLaunch& l, bool exact, const FlagList& flags,
                              int sm_count, cudaStream_t stream, std::string* err, bool* rescore_kernel_needed,
                              bool half_nonneg, int* x_elem_bytes, int* x_read_bytes) {
  // the in-kernel queue re-scores rows with W in global memory / L2: fine for a 5 KB model, not for 62 KB of fp64
  // weights per row (cfg 3) - wide models take the re-score kernel, which stages W in shared memory
  const bool small_model = static_cast<size_t>(m.w64_stride) * m.n_features * sizeof(double) <= 16 * 1024;
  const bool inline_rescore = exact && small_model && linear_queue_rescore();
  if (rescore_kernel_needed) *rescore_kernel_needed = exact && !inline_rescore;
  if (!linear_tma_supported(m, err)) return cudaErrorInvalidValue;
  if (l.n_rows <= 0) return cudaSuccess;
  TmaKernelParams p{};
  p.wt = m.wt;
  p.bias = m.bias;
  p.targets = l.targets;
  p.n_rows = l.n_rows;
  // (at f_pad <= 64 the fp16 schedule's shortest ring always fits beside the largest W^T, 16 classes)
  static_assert(1024 + (kHalfBoxF + 1) * 20 * 4 + 2 * 64 * 8 + (kQueueCap + 4) * 4 + 64 * 4 +
                        kHalfConsumerWarps * linear_stage_bytes(LinearSched::kHalf) <= kMaxSmemBytes,
                "kHalfConsumerWarps stages do not fit");
  const bool half = half_map != nullptr && linear_half_rows_ok(m.f_pad);
  // the tensor-core schedule: EXACT with the queue (its uncertified rows are replayed there), a model with tc_ops, an
  // fp16 copy without negative values (its bound column is a product with x, not |x|), and no source view (its drain
  // re-scores in fp64 from the float64 copy or the fp32 rows only, rescore_row_tc; resident batches, the only ones with
  // an fp16 copy, have no view).  UML_B200_LINEAR_TC=0 (read per call) keeps such a batch on kHalf: a test and A/B hook.
  const char* tc_env = getenv("UML_B200_LINEAR_TC");
  const bool tc = half && half_nonneg && inline_rescore && m.tc_ops != nullptr && l.x != nullptr && l.src.base == nullptr &&
                  !(tc_env && tc_env[0] == '0');
  // UML_B200_LINEAR_TC=1: the call fails unless it takes the tensor-core schedule (tests assert the dispatch with it)
  if (tc_env && tc_env[0] == '1' && !tc) {
    if (err) *err = "UML_B200_LINEAR_TC=1, but the batch or the model does not take the tensor-core schedule";
    return cudaErrorInvalidValue;
  }
  // a batch with a byte copy reads it on the tensor cores (a quarter of the fp32 rows' bytes)
  const bool bytes = tc && byte_map != nullptr;
  const LinearSched sched = bytes  ? LinearSched::kByteMma
                            : tc   ? LinearSched::kHalfMma
                            : half ? LinearSched::kHalf
                            : linear_whole_rows(m.f_pad) ? LinearSched::kWhole
                                                         : LinearSched::kChunked;
  const int tile_rows = half ? kHalfTileRows : linear_box_rows(m.f_pad);
  p.num_tiles = (l.n_rows + tile_rows - 1) / tile_rows;
  p.f_pad = m.f_pad;
  p.kc = m.f_pad / kChunkF;
  p.tc_ops = m.tc_ops;
  p.tc_kappa = m.tc_kappa;
  const size_t fixed =
      tma_fixed_smem(m, half) + (tc ? linear_tc_b_bytes(m.n_classes) : 0) + linear_epi_bytes(sched, m.n_classes);
  const int stage_bytes = linear_stage_bytes(sched);
  int stages = static_cast<int>((static_cast<size_t>(kMaxSmemBytes) - fixed) / stage_bytes);
  stages = std::min(stages, 64);
  // test hook: the shallowest legal ring (stages == scoring warps) stresses the barrier protocol
  const int warps = linear_ring_units(sched);
  if (const char* env = getenv("UML_B200_STAGES")) stages = std::max(warps, std::min(stages, atoi(env)));
  p.num_stages = stages;
  // margin > 2 err guarantees the fp32 argmax is the exact argmax; err <= (F+4) 2^-24 A (1 + F 2^-21), see DESIGN.md
  p.thr = linear_margin_thr(m.n_features);
  // UML_B200_TC_REPLAY=0 (read per call; a test hook): in the tensor-core schedules p.thr is read only by tier 2's
  // replay, which then certifies no row, so every row tier 1 leaves goes to fp64 and n_flagged counts exactly those
  // rows (DESIGN.md 3.2).  The kernels are unchanged.
  const char* replay_env = getenv("UML_B200_TC_REPLAY");
  if (tc && replay_env && replay_env[0] == '0') p.thr = INFINITY;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.x = l.x;
  p.x64 = l.x64;
  p.src = l.src;
  p.ld = l.ld;
  p.ld64 = l.ld64;
  p.w64 = m.w64;
  p.w64_stride = m.w64_stride;
  p.b64 = m.b64;
  p.n_classes = m.n_classes;
  p.n_features = m.n_features;
  p.fold_rel = m.fold_rel;
  p.binary = m.binary;
  p.counters = flags.counters;
  const size_t smem = fixed + static_cast<size_t>(stages) * stage_bytes;
  const long long slots = (p.num_tiles + warps - 1) / warps;
  const int grid = static_cast<int>(std::min<long long>(sm_count, std::max<long long>(1, slots)));
  if (x_elem_bytes) *x_elem_bytes = half ? 2 : 4;  // (kByteMma multiplies the fp16 values kHalfMma reads)
  if (x_read_bytes) *x_read_bytes = bytes ? 1 : half ? 2 : 4;
  using S = LinearSched;
  if (sched == S::kByteMma) return dispatch_classes<true, true, S::kByteMma>(m.n_classes, *byte_map, p, grid, smem, stream);
  if (sched == S::kHalfMma) return dispatch_classes<true, true, S::kHalfMma>(m.n_classes, *half_map, p, grid, smem, stream);
  if (sched == S::kHalf) {
    const CUtensorMap& hmap = *half_map;
    if (!exact) return dispatch_classes<false, false, S::kHalf>(m.n_classes, hmap, p, grid, smem, stream);
    return inline_rescore ? dispatch_classes<true, true, S::kHalf>(m.n_classes, hmap, p, grid, smem, stream)
                          : dispatch_classes<true, false, S::kHalf>(m.n_classes, hmap, p, grid, smem, stream);
  }
  if (sched == S::kWhole) {
    if (!exact) return dispatch_classes<false, false, S::kWhole>(m.n_classes, xmap, p, grid, smem, stream);
    return inline_rescore ? dispatch_classes<true, true, S::kWhole>(m.n_classes, xmap, p, grid, smem, stream)
                          : dispatch_classes<true, false, S::kWhole>(m.n_classes, xmap, p, grid, smem, stream);
  }
  if (!exact) return dispatch_classes<false, false, S::kChunked>(m.n_classes, xmap, p, grid, smem, stream);
  return inline_rescore ? dispatch_classes<true, true, S::kChunked>(m.n_classes, xmap, p, grid, smem, stream)
                        : dispatch_classes<true, false, S::kChunked>(m.n_classes, xmap, p, grid, smem, stream);
}

cudaError_t launch_rescore_f64(const LinearDeviceModel& m, const LinearLaunch& l, const FlagList& flags, bool all_rows,
                               int sm_count, cudaStream_t stream) {
  if (l.n_rows <= 0) return cudaSuccess;
  RescoreParams p{};
  p.x = l.x;
  p.x64 = l.x64;
  p.src = l.src;
  p.ld = l.ld;
  p.ld64 = l.ld64;
  p.n_rows = l.n_rows;
  p.w64 = m.w64;
  p.w64_stride = m.w64_stride;
  p.b64 = m.b64;
  p.n_classes = m.n_classes;
  p.n_features = m.n_features;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.all_rows = all_rows ? 1 : 0;
  p.targets = l.targets;
  p.counters = flags.counters;
  p.fold_rel = m.fold_rel;
  p.binary = m.binary;
  // shared-memory copy of W, b (with the bias magnitudes) when it fits next to nothing else (<= 200 KB)
  size_t smem = (static_cast<size_t>(m.n_features) * m.w64_stride + 2 * m.n_classes) * sizeof(double);
  if (smem > 200 * 1024) smem = 0;
  p.smem_weights = smem > 0 ? 1 : 0;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(rescore_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  // flagged rows are few (0.02 % on cfg 2): a grid of <= 2 blocks per SM starts and drains faster than 8; the all-rows
  // path (generic shapes) wants every resident warp
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rescore_f64_kernel, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  long long blocks = static_cast<long long>(sm_count) * (all_rows ? per_sm : std::min(per_sm, 2));
  if (all_rows) blocks = std::min<long long>(blocks, (l.n_rows + 7) / 8);
  return launch_dependent(rescore_f64_kernel, static_cast<int>(std::max<long long>(1, blocks)), 256, smem, stream, p);
}

}  // namespace uml
