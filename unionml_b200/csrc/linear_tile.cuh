// What both families of the linear tile kernel run (sm_90a): the CUDA-core schedules of linear_argmax_tma_kernel
// (linear_kernels.cu) and the tensor-core schedules of linear_argmax_tc_kernel (linear_tc_kernels.cu).  Their
// parameters, the schedules, the float64 row scorer, the queue's constants, the shared-memory carve-up and prologue,
// the claimed-tile producer, the diagnostic builds' hooks and the launch geometry.
#pragma once

#include <cuda.h>
#include <stdint.h>

#include <cmath>
#include <cstddef>

#include "uml_common.cuh"
#include "label_store.cuh"
#include "tma_ring.cuh"
#include "rescore_util.cuh"

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
// TMA tile kernels
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

constexpr int kTileSentinel = -1;        // claimed schedules: ring item that ends a scoring warp's loop
constexpr int kQueueCap = 2048;           // flagged-row queue of the QUEUE kernels (power of two)

// Diagnostic builds of the tile kernels (tools/linear_probe.cu defines these; the library defines neither):
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
// The first three are linear_argmax_tma_kernel's (CUDA cores), the last two linear_argmax_tc_kernel's (tensor cores).
// kWhole, kHalf and the tensor-core schedules claim their tiles in groups of NCU (the units that take ring items: the
// scoring warps, or the two warpgroups) from a global counter; ring item n goes to unit n % NCU.
enum class LinearSched { kChunked, kWhole, kHalf, kHalfMma, kByteMma };
__host__ __device__ constexpr bool linear_tc_sched(LinearSched s) { return s == LinearSched::kHalfMma || s == LinearSched::kByteMma; }

// scoring warps of a CUDA-core schedule; the producer is warp NCW and the QUEUE kernels' re-score warp NCW + 1
__host__ __device__ constexpr int linear_consumer_warps(LinearSched s) {
  return s == LinearSched::kHalf ? kHalfConsumerWarps : kConsumerWarps;
}
// units that take ring items (and the ring's floor): the scoring warps, or the tensor-core schedules' two warpgroups
constexpr int kTcWarpgroups = 2;
__host__ __device__ constexpr int linear_ring_units(LinearSched s) {
  return linear_tc_sched(s) ? kTcWarpgroups : linear_consumer_warps(s);
}
// bytes of one ring stage: in kHalf and kHalfMma two 16 KiB fp16 boxes
__host__ __device__ constexpr int linear_stage_bytes(LinearSched s) {
  return s == LinearSched::kHalf || s == LinearSched::kHalfMma ? 2 * kStageBytes : kStageBytes;
}

// The dynamic shared memory of a tile kernel, from the 1 KiB-aligned base (SWIZZLE_128B wants it): the ring of S
// stages of STAGE_BYTES (smem), LEAD bytes (the tensor-core schedules' B operand), W^T [f_pad][CP] (wt_s) and the bias
// [CP] (bias_s), the `full` and `empty` barriers of the stages, the queue, the tile index of each stage (64 slots the
// host reserves), then what the host adds (kByteMma's score slots).  tma_fixed_smem is the host's side of this layout.
//  q_slots, q_ctl  QUEUE kernels: rows flagged by the scoring warps travel through this shared-memory queue to the
//                  re-score warp (slot value = row + 1, 0 = empty); ctl[0] = tail (reserved), ctl[1] = head (tickets
//                  claimed), ctl[2] = publishing warps done, ctl[3] = slots consumed
//  tile_slot       claimed schedules: the tile each stage holds, written by the producer before the stage's `full`
//                  arrive (whose release makes it visible to the waiters); kTileSentinel ends a scoring warp's loop
// A macro that declares these pointers in the kernel, rather than a function that returns them: behind an inlined
// function NVVM associates kByteMma's stage addresses differently, and the kernel's SASS changes.
#define UML_LINEAR_SMEM(CP, STAGE_BYTES, LEAD, S, F_PAD)                                                              \
  extern __shared__ uint8_t smem_raw[];                                                                             \
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);                                     \
  float* wt_s = reinterpret_cast<float*>(smem + static_cast<size_t>(S) * (STAGE_BYTES) + (LEAD));                   \
  float* bias_s = wt_s + (F_PAD) * (CP);                                                                            \
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + (CP));                                                  \
  uint64_t* empty_bar = full_bar + (S);                                                                             \
  int* q_slots = reinterpret_cast<int*>(empty_bar + (S));                                                           \
  int* q_ctl = q_slots + kQueueCap;                                                                                 \
  int* tile_slot = q_ctl + 4

// stage W^T (with its wmax column) and the bias once per CTA; they stay resident for every tile this CTA scores
template <int CP>
__device__ __forceinline__ void stage_weights(const TmaKernelParams& p, float* wt_s, float* bias_s) {
  const float4* src = reinterpret_cast<const float4*>(p.wt);
  float4* dst = reinterpret_cast<float4*>(wt_s);
  const int n4 = p.f_pad * CP / 4;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = __ldg(src + i);
  if (threadIdx.x < CP) bias_s[threadIdx.x] = __ldg(p.bias + threadIdx.x);
}
__device__ __forceinline__ void zero_queue(int* q_slots) {
  for (int i = threadIdx.x; i < kQueueCap + 4; i += blockDim.x) q_slots[i] = 0;
}
// (thread 0) `full` takes the producer's arrive; `empty` the arrives of the warps that hand a stage back
__device__ __forceinline__ void init_ring_barriers(uint64_t* full_bar, uint64_t* empty_bar, int S,
                                                   uint32_t empty_arrivals) {
  for (int s = 0; s < S; ++s) {
    mbar_init(&full_bar[s], 1);
    mbar_init(&empty_bar[s], empty_arrivals);
  }
}

// The claimed schedules' producer (one elected lane of warp NCW).  Tiles are claimed, NCU at a time, from a counter
// shared by the grid: with a static split, CTAs with equal tile counts finished up to ~0.24 ms apart (SMs draw unequal
// shares of HBM bandwidth), and the launch lasted as long as the slowest one.  Ring item n is one tile with both halves
// of its rows and goes to unit n % NCU; a group claimed past the end hands every unit kTileSentinel.  The next group is
// claimed while this one is issued, so the atomic's round trip stays off the ring.  F16: two {64, 128} fp16 boxes per
// stage; TWO_BOXES (kWhole): two {32, 64} fp32 boxes side by side; otherwise one box of kStageBytes (kByteMma).
// num_tiles is p.num_tiles, which the kernel has loaded for its consumers.  Returns the clock64() cycles spent in
// `empty` waits (UML_PROBE_WAIT_CLOCKS builds; 0 otherwise).
template <int TILE, int NCU, int STAGE_BYTES, int BOX_BYTES, bool F16, bool TWO_BOXES>
__device__ __forceinline__ long long produce_claimed_tiles(const CUtensorMap* xmap, const TmaKernelParams& p,
                                                           uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar,
                                                           int* tile_slot, int S, long long num_tiles) {
  long long probe_wait = 0;
  tma_prefetch_desc(xmap);
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
          uint8_t* dst = ring + static_cast<size_t>(stage) * STAGE_BYTES;
          const int row = static_cast<int>(tile * TILE);
          const bool second = row + kTileRows < p.n_rows;
          mbar_arrive_expect_tx(&full_bar[stage], second ? STAGE_BYTES : BOX_BYTES);
          tma_load_2d(dst, xmap, &full_bar[stage], 0, row, policy);
          if (second) tma_load_2d(dst + BOX_BYTES, xmap, &full_bar[stage], 0, row + kTileRows, policy);
        } else {
          // (kByteMma: one {64, 256} box; rows past the batch are filled with zeros and never stored)
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          uint8_t* dst = ring + static_cast<size_t>(stage) * kStageBytes;
          const int row = static_cast<int>(tile * TILE);
          tma_load_2d(dst, xmap, &full_bar[stage], 0, row, policy);
          if constexpr (TWO_BOXES) tma_load_2d(dst + BOX_BYTES, xmap, &full_bar[stage], kChunkF, row, policy);
        }
#ifdef UML_PROBE_TIMELINE
        if (probe_first_issue) UML_PROBE_STAMP(1);
        probe_first_issue = false;
#endif
      } else {
        mbar_arrive(&full_bar[stage]);  // past the last tile: nothing to load, the unit skips or stops
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
  return probe_wait;
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// Launch geometry of one schedule for one batch (linear_kernels.cu): what launch_linear_tma and tools/linear_probe.cu
// launch with.  stages honours UML_B200_STAGES (read per call), in the probe as in the library.
struct LinearGeometry {
  long long num_tiles;
  int tile_rows;    // rows per tile = per ring stage
  int stage_bytes;
  int stages;
  size_t smem;      // dynamic shared memory: the ring and UML_LINEAR_SMEM's regions (tma_fixed_smem), and
                    // linear_tc_extra_smem in the tensor-core schedules
  int grid;
};
LinearGeometry linear_geometry(const LinearDeviceModel& m, LinearSched sched, long long n_rows, int sm_count);
// linear_tc_kernels.cu: the tensor-core schedules' shared memory besides UML_LINEAR_SMEM's regions (the B operand,
// kByteMma's score slots), and the launch of linear_argmax_tc_kernel<m.n_classes, sched> with p and m's tensor-core
// operands
size_t linear_tc_extra_smem(LinearSched sched, int C);
cudaError_t launch_linear_tc(LinearSched sched, const LinearDeviceModel& m, const CUtensorMap& xmap, TmaKernelParams p,
                             int grid, size_t smem, cudaStream_t stream);

}  // namespace uml
