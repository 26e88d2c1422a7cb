// Scoring kernels for the linear predictor  X . W^T + b -> argmax   (sm_90a).
//
// Replaces the numeric body of sklearn's LinearClassifierMixin.predict (sklearn/linear_model/_base.py:366-427), which
// is what the reference's canonical predictor runs (unionml:README.md:87-92).
//
//  * linear_argmax_tma_kernel<C, EXACT, QUEUE, SCHED>: the CUDA-core schedules of the tile kernel (kChunked, kWhole,
//    kHalf), persistent, warp-specialised.  One producer warp streams X
//    through a 16 KiB-per-stage shared-memory ring with TMA + mbarriers: 128-row x 32-feature boxes (128B-swizzled), or
//    at 33 <= F <= 64 (kWhole) stages of 64 complete rows, or (kHalf) 32 KiB stages of 256 complete rows from the
//    batch's compact fp16 copy; eight consumer warps (four in kHalf) each own one tile at a time (4, 2 or 8
//    rows per lane), read X with conflict-free LDS.128, W as warp-uniform broadcast
//    LDS.128 from a transposed copy in shared memory, keep C (+1) fp32 accumulators per row in registers, and fuse
//    bias, argmax (first maximum wins, like np.argmax) and the label store.  In EXACT mode one extra accumulator
//    carries A = max|b| + sum_f |x_f| * max_c |w_cf|; rows whose top-2 margin is not provably larger than the fp32
//    rounding error (2 (F+4) 2^-24 A) are appended to a list and re-scored in fp64 by rescore_f64_kernel.  The
//    tensor-core schedules are linear_argmax_tc_kernel's (linear_tc_kernels.cu); launch_linear_tma chooses among all
//    five.
//  * rescore_f64_kernel: warp per row, lanes over features, fp64 FMA + shuffle reduction; serves the flagged rows of
//    EXACT mode and is the generic (any F, any C) path when the tile kernel's shape limits do not hold.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "linear_tile.cuh"

#ifndef UML_RESCORE_QUEUE_DEFAULT
#define UML_RESCORE_QUEUE_DEFAULT 1  // one launch per step; the few flagged rows (0.02 % on digits) cost the queue little
#endif


namespace uml {

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

constexpr int kQueueHeadroom = 1024;      // a warp publishes only while this many slots are free (8 warps x 128 rows)
// the scoring warps, the producer and (QUEUE kernels) the re-score warp
__host__ __device__ constexpr int linear_threads(LinearSched s, bool queue) { return (linear_consumer_warps(s) + (queue ? 2 : 1)) * 32; }

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
  constexpr bool HALF = SCHED == LinearSched::kHalf;          // 256-row stages of the compact fp16 rows, two boxes
  constexpr bool CLAIMED = WHOLE || HALF;                     // tiles claimed from kCounterTileClaim, one tile per stage
  static_assert(!linear_tc_sched(SCHED), "the tensor-core schedules are linear_argmax_tc_kernel's");
  constexpr int NCW = linear_consumer_warps(SCHED);
  constexpr int TILE = HALF ? kHalfTileRows : WHOLE ? kWholeTileRows : kTileRows;  // rows per tile = per ring stage
  // free queue slots a scoring warp wants before it publishes (kHalf: every one may publish all its rows of a tile at
  // once)
  constexpr int HEADROOM = HALF ? NCW * TILE : kQueueHeadroom;
  static_assert(HEADROOM <= kQueueCap, "the queue holds one tile of every scoring warp");
  // rows per lane held in registers at once (kHalf: one pass, NPASS passes per tile)
  constexpr int R = HALF ? kHalfPassRows : TILE / 32;
  constexpr int NPASS = TILE / 32 / R;
  static_assert(NPASS * R * 32 == TILE && (!HALF || R % 4 == 0), "a pass is whole 128-row boxes");
  // one box: 8 KiB (two per kWhole stage) or 16 KiB (two per kHalf stage)
  constexpr int BOX_BYTES = (HALF ? kTileRows : TILE) * kChunkF * 4;
  constexpr int STAGE_BYTES = linear_stage_bytes(SCHED);
  static_assert(!HALF || (BOX_BYTES == kTileRows * kHalfBoxF * 2 && STAGE_BYTES == 2 * BOX_BYTES),
                "an fp16 stage is two boxes");
  // fp32x2 accumulator pairs (see the accumulator comment below).  Not in the fp16 schedule: fma2 is two fmaf, so the
  // scores are the same bits, and without the 64-bit register pairs ptxas schedules its 128 registers better
  // (0.534 -> 0.523 ms at cfg 2, DESIGN.md 5.1)
  constexpr bool USE_F2 = EXACT && !HALF;

  const int S = p.num_stages;
  UML_LINEAR_SMEM(CP, STAGE_BYTES, 0, S, p.f_pad);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) UML_PROBE_STAMP(0);

  stage_weights<CP>(p, wt_s, bias_s);
  if constexpr (QUEUE) zero_queue(q_slots);
  if (threadIdx.x == 0) {
    init_ring_barriers(full_bar, empty_bar, S, 1);
    fence_barrier_init();
  }
  __syncthreads();

  pdl_launch_dependents();  // the re-score kernel behind this launch may be scheduled now; it waits for this grid to finish
  const long long G = gridDim.x;
  const long long num_tiles = p.num_tiles;
  const int KC = p.kc;
  [[maybe_unused]] long long probe_wait = 0;
#ifdef UML_PROBE_WAIT_CLOCKS
  const long long probe_start = clock64();
#endif

  if (warp == NCW) {
    // ===================== TMA producer (one elected lane) =====================
    if (elect_one_sync()) {
      if constexpr (CLAIMED) {
        probe_wait = produce_claimed_tiles<TILE, NCW, STAGE_BYTES, BOX_BYTES, HALF, WHOLE>(&xmap, p, smem, full_bar,
                                                                                          empty_bar, tile_slot, S,
                                                                                          num_tiles);
      } else {
        tma_prefetch_desc(&xmap);
        const uint64_t policy = make_evict_first_policy();  // X is read exactly once
        int stage = 0;
        uint32_t phase = 0;
        auto next_stage = [&] {
          if (++stage == S) {
            stage = 0;
            phase ^= 1u;
          }
        };
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
    const bool scoring_warp = warp < NCW;
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

    if constexpr (CLAIMED) {
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
      if (warp < NCW) {
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
      long long probe_busy = 0, probe_rows = 0;
#endif
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
            if (v == 0 && atomicAdd(&q_ctl[2], 0) == NCW) {
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
#ifdef UML_PROBE_WAIT_CLOCKS
      if (warp == NCW + 1 && lane == 0) {
        atomicAdd(&p.probe_clocks[5], static_cast<unsigned long long>(probe_busy));
        atomicAdd(&p.probe_clocks[6], static_cast<unsigned long long>(clock64() - probe_start));
        atomicAdd(&p.probe_clocks[10], static_cast<unsigned long long>(probe_busy));
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

LinearGeometry linear_geometry(const LinearDeviceModel& m, LinearSched sched, long long n_rows, int sm_count) {
  const bool tc = linear_tc_sched(sched);
  LinearGeometry g{};
  // the kernels' TILE: by schedule, not by f_pad (tools/linear_probe.cu runs kChunked at f_pad 64 too)
  g.tile_rows = sched == LinearSched::kHalf || tc ? kHalfTileRows
                : sched == LinearSched::kWhole     ? kWholeTileRows
                                                   : kTileRows;
  g.num_tiles = (n_rows + g.tile_rows - 1) / g.tile_rows;
  g.stage_bytes = linear_stage_bytes(sched);
  const size_t fixed = tma_fixed_smem(m, sched != LinearSched::kChunked) + (tc ? linear_tc_extra_smem(sched, m.n_classes) : 0);
  int stages = static_cast<int>((static_cast<size_t>(kMaxSmemBytes) - fixed) / g.stage_bytes);
  stages = std::min(stages, 64);
  // test hook: the shallowest legal ring (stages == the units that take ring items) stresses the barrier protocol
  const int units = linear_ring_units(sched);
  if (const char* env = getenv("UML_B200_STAGES")) stages = std::max(units, std::min(stages, atoi(env)));
  g.stages = stages;
  g.smem = fixed + static_cast<size_t>(stages) * g.stage_bytes;
  const long long slots = (g.num_tiles + units - 1) / units;
  g.grid = static_cast<int>(std::min<long long>(sm_count, std::max<long long>(1, slots)));
  return g;
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
  const LinearGeometry g = linear_geometry(m, sched, l.n_rows, sm_count);
  p.num_tiles = g.num_tiles;
  p.f_pad = m.f_pad;
  p.kc = m.f_pad / kChunkF;
  p.num_stages = g.stages;
  // margin > 2 err guarantees the fp32 argmax is the exact argmax; err <= (F+4) 2^-24 A (1 + F 2^-21), see DESIGN.md
  p.thr = linear_margin_thr(m.n_features);
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
  const int grid = g.grid;
  const size_t smem = g.smem;
  if (x_elem_bytes) *x_elem_bytes = half ? 2 : 4;  // (kByteMma multiplies the fp16 values kHalfMma reads)
  if (x_read_bytes) *x_read_bytes = bytes ? 1 : half ? 2 : 4;
  using S = LinearSched;
  if (tc) return launch_linear_tc(sched, m, bytes ? *byte_map : *half_map, p, grid, smem, stream);
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
