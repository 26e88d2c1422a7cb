// Tensor-core schedules of the linear tile kernel  X . W^T + b -> argmax   (sm_90a, DESIGN.md 3.1, 3.2).
//
//  * linear_argmax_tc_kernel<C, SCHED>, SCHED = kHalfMma (the batch's compact fp16 rows) or kByteMma (its byte rows):
//    persistent, warp-specialised, always exact with the in-launch queue.  The producer warp streams 256-row tiles
//    through the shared-memory ring of linear_tile.cuh; two MMA warpgroups score them with wgmma (f16 x f16 -> fp32,
//    W^T as scaled hi | lo pieces, the bound column beside the classes) and tier 1 certifies a row when its margin
//    exceeds kappa A.  kByteMma hands each item's scores to four epilogue warps through score slots.  Rows tier 1 leaves
//    go through the queue to the drain, which replays the fp32 route on them 32 at a time (tier 2) and re-scores the
//    rest in fp64.
//  * build_tc_operands: the B operand image and kappa, built on the host at model load.
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "linear_tile.cuh"
#include "wgmma.cuh"

namespace uml {

// The tensor-core schedules' fp64 scores of one row, from the batch's float64 copy when it keeps one (its fp32 rows are
// not the caller's values) and from the fp32 rows otherwise; no source view reaches these schedules (launch_linear_tma's
// dispatch).  C is known, so this is one copy of score_row_f64 with its 2 C accumulators in registers, instead of the
// CUDA-core drain's three copies with sixteen of each in local memory.
template <int C>
__device__ __noinline__ int rescore_row_tc(const TmaKernelParams& p, long long row, int lane) {
  const float* xr = p.x + row * p.ld;
  const double* xr64 = p.x64 ? p.x64 + row * p.ld64 : nullptr;
  const RowScore r = score_row_f64<C, true>([&](int f) { return xr64 ? xr64[f] : static_cast<double>(xr[f]); }, p.w64,
                                            p.w64_stride, p.b64, p.n_features, C, p.fold_rel, p.binary != 0, lane);
  if (lane == 0) count_rescored_row(p, r.bad, r.ambiguous);
  return r.idx;
}

// warps: kHalfMma two MMA warpgroups (warps 0-7); kByteMma the same and a pair of epilogue warps per warpgroup (8-11).
// The producer is warp NCW and the drain's own warp NCW + 1.  kByteMma's feed takes half of kHalfMma's time, so the time
// per item outside the tensor cores is the limit: the epilogue warps take the per-row tail (top-2, tier 1, label
// stores, queue hand-off) off the warpgroups, which then keep up with the feed in two.  Two epilogue warps for three
// warpgroups (16 warps) could not: 0.349 against 0.280 ms (DESIGN.md 5.1).
constexpr int kByteWarpgroups = 2;
constexpr int kByteEpiWarps = 2 * kByteWarpgroups;
static_assert(kByteWarpgroups == kTcWarpgroups && kConsumerWarps == 4 * kTcWarpgroups, "two MMA warpgroups");
__host__ __device__ constexpr int linear_tc_warps(LinearSched s) {
  return s == LinearSched::kByteMma ? 4 * kByteWarpgroups + kByteEpiWarps : kConsumerWarps;
}
// bytes of the B operand in shared memory (rounded up to the 1 KiB that keeps what follows aligned)
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
// the CUDA-core kernel's sequential best / second loop and the same p.thr comparison.  A lane whose row that route
// certifies stores its label and returns true; the caller sends the others to fp64.  W^T rows are read as warp-uniform
// LDS.128 (broadcast; CP % 4 == 0).  Out of line, so that the MMA and epilogue loops keep their register allocation, and
// small: it runs a few times per CTA per launch, from a cold instruction cache, so the FMAs of one 32-feature half are
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

template <int C, LinearSched SCHED>
__global__ void __launch_bounds__((linear_tc_warps(SCHED) + 2) * 32, 1)
linear_argmax_tc_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ TmaKernelParams p) {
  static_assert(linear_tc_sched(SCHED), "kHalfMma or kByteMma");
  constexpr int CP = (C + 1 + 3) / 4 * 4;    // padded columns of wt in shared memory (the CUDA-core kernel's layout)
  constexpr bool BYTES = SCHED == LinearSched::kByteMma;    // 256-row stages of the byte rows, one box
  constexpr bool F16 = SCHED == LinearSched::kHalfMma;      // 256-row stages of the compact fp16 rows, two boxes
  constexpr int NCW = linear_tc_warps(SCHED);
  constexpr int NCU = kTcWarpgroups;
  constexpr int TILE = kHalfTileRows;  // rows per tile = per ring stage
  // warps that publish to the queue (kByteMma: the epilogue warps, warps NMW .. NCW - 1)
  constexpr int NMW = BYTES ? 4 * kByteWarpgroups : NCW;
  constexpr int NPUB = BYTES ? kByteEpiWarps : NCW;
  static_assert(!BYTES || NMW + NPUB == NCW, "warps NMW .. NCW - 1 are the epilogue warps");
  // free queue slots a publishing warp wants before it publishes: every one may publish all its rows of a tile at once
  // (kHalfMma: the 64 rows of the tile a warp stores; kByteMma: an epilogue warp's 128, half a tile)
  constexpr int HEADROOM = BYTES ? NPUB * TILE / 2 : NCW * 64;
  static_assert(HEADROOM <= kQueueCap, "the queue holds one tile of every scoring warp");
  // one box: 16 KiB (two per kHalfMma stage, one per kByteMma stage)
  constexpr int BOX_BYTES = BYTES ? kHalfTileRows * kByteRowBytes : kTileRows * kChunkF * 4;
  constexpr int STAGE_BYTES = linear_stage_bytes(SCHED);
  static_assert(!F16 || (BOX_BYTES == kTileRows * kHalfBoxF * 2 && STAGE_BYTES == 2 * BOX_BYTES),
                "an fp16 stage is two boxes");
  static_assert(!BYTES || STAGE_BYTES == BOX_BYTES, "a byte stage is one box");

  const int S = p.num_stages;
  // the B operand (1 KiB aligned, as SWIZZLE_128B wants) between the ring and W^T
  UML_LINEAR_SMEM(CP, STAGE_BYTES, linear_tc_b_bytes(C), S, p.f_pad);
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

  stage_weights<CP>(p, wt_s, bias_s);
  {
    const uint4* bsrc = static_cast<const uint4*>(p.tc_ops);
    uint4* bdst = reinterpret_cast<uint4*>(smem + static_cast<size_t>(S) * STAGE_BYTES);
    for (int i = threadIdx.x; i < linear_tc_cols(C) * 8; i += blockDim.x) bdst[i] = __ldg(bsrc + i);
    fence_proxy_async_smem();  // st.shared -> visible to the wgmma reads
  }
  zero_queue(q_slots);
  if (threadIdx.x == 0) {
    init_ring_barriers(full_bar, empty_bar, S, 4);  // every warp of the warpgroup hands the stage back
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
  const long long num_tiles = p.num_tiles;
#ifdef UML_PROBE_WAIT_CLOCKS
  long long probe_wait = 0;
  const long long probe_start = clock64();
#endif

  if (warp == NCW) {
    // ===================== TMA producer (one elected lane) =====================
    if (elect_one_sync()) {
      [[maybe_unused]] const long long waited =
          produce_claimed_tiles<TILE, NCU, STAGE_BYTES, BOX_BYTES, F16, false>(&xmap, p, smem, full_bar, empty_bar,
                                                                               tile_slot, S, num_tiles);
#ifdef UML_PROBE_WAIT_CLOCKS
      atomicAdd(&p.probe_clocks[0], static_cast<unsigned long long>(waited));
      atomicAdd(&p.probe_clocks[1], static_cast<unsigned long long>(clock64() - probe_start));
#endif
    }
  } else {
    // ===================== MMA warpgroups (kByteMma: and epilogue warps); warp NCW + 1 drains the queue ==========
    const bool scoring_warp = warp < NMW;  // (kByteMma: the MMA warps)
#ifdef UML_PROBE_WAIT_CLOCKS
    long long probe_hold = 0;
#endif
#ifdef UML_PROBE_TIMELINE
    unsigned long long probe_last_release = 0;
#endif
    // warpgroup wg = warp / 4 takes ring items wg, wg + NCU, ...; per item four m64 blocks of 64 rows x NT columns,
    // f_pad / 16 k16 steps each.  Fragment (WgmmaTf32's layout): thread (warp w, lane l) holds fragment rows 16 (w % 4)
    // + l / 4 and the row 8 below of each block, columns 8 i + 2 (l % 4) + {0, 1}: class c's hi piece at c, its lo
    // piece at NH + c, the bound column at C - all of a row in one quad
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
        // the (few) uncertified rows go to the drain, as in the CUDA-core kernel: the labels above are provisional.
        // When the queue is backed up (most rows near-ties) the warp waits for room instead of settling its rows itself:
        // a call from this loop made ptxas save the loop's live registers around it, spill stores and loads in the hot
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
    if (BYTES ? warp >= NMW && warp < NCW : warp < NCW) {  // the publishers: kByteMma's epilogue warps, kHalfMma's MMA warps
      __syncwarp();
      if (lane == 0) {
        __threadfence_block();
        atomicAdd(&q_ctl[2], 1);  // this warp has published everything it will ever publish
      }
    }
    // ===================== the drain: warp NCW + 1 settles the queue's rows while the others stream; every warp that
    // has finished its own work joins in.  Tier 2 in batches of 32 rows, one per lane.  While publishers are still
    // running a batch starts only when 32 tickets are reserved (at about one row every few thousand cycles, smaller
    // batches would mostly hold one row); once all have published, what is left is split evenly over the NCW + 1
    // warps that drain, so that the float64 rows of the CTA's last batch do not run one after another in one warp.
    // Labels are due at the end of the grid only, and the queue holds 2048 rows against ~100 per CTA, so the wait
    // costs nothing.  Tickets are claimed with a CAS on the head, so every claimed ticket is reserved and its row is
    // being published. =====================
    int n_done = 0;
#ifdef UML_PROBE_WAIT_CLOCKS
    long long probe_busy = 0, probe_f64 = 0, probe_rows = 0;
#endif
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
#ifdef UML_PROBE_WAIT_CLOCKS
    if (warp == NCW + 1 && lane == 0) {
      atomicAdd(&p.probe_clocks[5], static_cast<unsigned long long>(probe_busy));
      atomicAdd(&p.probe_clocks[6], static_cast<unsigned long long>(clock64() - probe_start));
      atomicAdd(&p.probe_clocks[10], static_cast<unsigned long long>(probe_f64));
    }
    if (lane == 0 && probe_rows > 0) atomicAdd(&p.probe_clocks[11], static_cast<unsigned long long>(probe_rows));
#endif
    if (lane == 0 && n_done > 0) atomicAdd(&p.counters[kCounterFlagged], static_cast<unsigned long long>(n_done));
  }
#ifdef UML_PROBE_TIMELINE
  if (lane == 0) atomicMax(&p.probe_timeline[blockIdx.x * kProbeStamps + 4], probe_globaltimer());
#endif
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// ---- tensor-core operands (DESIGN.md 3.1, 3.2) ----
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

size_t linear_tc_extra_smem(LinearSched sched, int C) {
  return static_cast<size_t>(linear_tc_b_bytes(C)) + linear_epi_bytes(sched, C);
}

template <int C, LinearSched SCHED>
static cudaError_t launch_tc(const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                             cudaStream_t stream) {
  auto kern = linear_argmax_tc_kernel<C, SCHED>;
  static size_t configured = 0;  // per instantiation (one device per process): set the attribute once, not per launch
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  kern<<<grid, (linear_tc_warps(SCHED) + 2) * 32, smem, stream>>>(xmap, p);
  return cudaGetLastError();
}

template <LinearSched SCHED>
static cudaError_t dispatch_tc_classes(int C, const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                                       cudaStream_t stream) {
  switch (C) {
#define UML_CASE(N) \
  case N:           \
    return launch_tc<N, SCHED>(xmap, p, grid, smem, stream);
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

cudaError_t launch_linear_tc(LinearSched sched, const LinearDeviceModel& m, const CUtensorMap& xmap, TmaKernelParams p,
                             int grid, size_t smem, cudaStream_t stream) {
  p.tc_ops = m.tc_ops;
  p.tc_kappa = m.tc_kappa;
  // UML_B200_TC_REPLAY=0 (read per call; a test hook): in the tensor-core schedules p.thr is read only by tier 2's
  // replay, which then certifies no row, so every row tier 1 leaves goes to fp64 and n_flagged counts exactly those
  // rows (DESIGN.md 3.2).  The kernels are unchanged.
  const char* replay_env = getenv("UML_B200_TC_REPLAY");
  if (replay_env && replay_env[0] == '0') p.thr = INFINITY;
  const int C = m.n_classes;
  if (sched == LinearSched::kByteMma) return dispatch_tc_classes<LinearSched::kByteMma>(C, xmap, p, grid, smem, stream);
  if (sched == LinearSched::kHalfMma) return dispatch_tc_classes<LinearSched::kHalfMma>(C, xmap, p, grid, smem, stream);
  return cudaErrorInvalidValue;
}

}  // namespace uml
