// Scoring kernels for the linear predictor  X . W^T + b -> argmax   (sm_90a).
//
// Replaces the numeric body of sklearn's LinearClassifierMixin.predict (sklearn/linear_model/_base.py:366-427), which
// is what the reference's canonical predictor runs (unionml:README.md:87-92).
//
//  * linear_argmax_tma_kernel<C, EXACT, QUEUE, WHOLE>: persistent, warp-specialised.  One producer warp streams X
//    through a 16 KiB-per-stage shared-memory ring with TMA + mbarriers: 128-row x 32-feature boxes (128B-swizzled), or
//    at 33 <= F <= 64 (WHOLE) stages of 64 complete rows; eight consumer warps each own one tile at a time (4 or 2
//    rows per lane), read X with conflict-free LDS.128, W as warp-uniform broadcast
//    LDS.128 from a transposed copy in shared memory, keep C (+1) fp32 accumulators per row in registers, and fuse
//    bias, argmax (first maximum wins, like np.argmax) and the label store.  In EXACT mode one extra accumulator
//    carries A = max|b| + sum_f |x_f| * max_c |w_cf|; rows whose top-2 margin is not provably larger than the fp32
//    rounding error (2 (F+4) 2^-24 A) are appended to a list and re-scored in fp64 by rescore_f64_kernel.
//  * rescore_f64_kernel: warp per row, lanes over features, fp64 FMA + shuffle reduction; serves the flagged rows of
//    EXACT mode and is the generic (any F, any C) path when the tile kernel's shape limits do not hold.
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "uml_common.cuh"
#include "tma_ring.cuh"
#include "rescore_util.cuh"

#ifndef UML_RESCORE_QUEUE_DEFAULT
#define UML_RESCORE_QUEUE_DEFAULT 1  // one launch per step; the few flagged rows (0.02 % on digits) cost the queue little
#endif


namespace uml {

// one element of the caller's raw source chunk as float64 (exact for every dtype the ABI takes)
__device__ __forceinline__ double load_src(const SrcView& v, long long row, int f) {
  const long long i = row * v.row_stride + static_cast<long long>(f) * v.col_stride;
  switch (v.dtype) {
    case UML_F64: return static_cast<const double*>(v.base)[i];
    case UML_I64: return static_cast<double>(static_cast<const long long*>(v.base)[i]);
    case UML_I32: return static_cast<double>(static_cast<const int*>(v.base)[i]);
    case UML_U8: return static_cast<double>(static_cast<const unsigned char*>(v.base)[i]);
    default: return static_cast<double>(static_cast<const float*>(v.base)[i]);
  }
}

struct RowScore {
  int idx;
  bool bad;        // NaN/Inf in the row
  bool ambiguous;  // fp64 top-2 margin inside the fp64 rounding bound: a true tie, decided by the first-index rule
};

// float64 scores of one row by one warp, first maximum wins like np.argmax.  Lanes split the features; classes are
// scored sixteen at a time (32 independent fp64 chains per lane), the sixteen sums are reduced with warp_reduce16 and
// the arg-max / runner-up found by a butterfly over the lanes.  LOAD(f) yields feature f of the row as double.
// w64 is feature-major, w64[f * S + c]: a lane fetches the classes of its feature with 16-byte loads off ONE address
// (immediate offsets) - the class-major table this replaces cost a 64-bit multiply-add per weight, half of the kernel's
// instructions at F = 784.
template <typename LOAD>
__device__ __forceinline__ RowScore score_row_f64(LOAD load, const double* __restrict__ w64, int S,
                                                  const double* __restrict__ b64, int F, int C, int lane) {
  const double u = 1.1102230246251565e-16;  // 2^-53
  bool bad = false;
  double best = 0.0, second = -INFINITY, amax = 0.0;
  int idx = 0;
  for (int c0 = 0; c0 < C; c0 += 16) {
    const int pairs = min(8, (C - c0 + 1) / 2);  // 16-byte loads per feature this round (an odd C ends in a zero pad)
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
    const double sv = warp_reduce16(s, lane), av = warp_reduce16(a, lane);
    const int cl = c0 + (lane >> 1);  // the class this lane pair now holds
    const bool valid = cl < C;
    Top2 t;
    t.best = valid ? sv + b64[cl] : -INFINITY;
    t.second = -INFINITY;
    t.idx = cl;
    top2_butterfly(t, 2);
    amax = fmax(amax, warp_max(valid ? av + fabs(b64[cl]) : 0.0, 2));
    if (c0 == 0) {
      best = t.best;
      second = t.second;
      idx = t.idx;
    } else if (t.best > best) {  // strict: a tie keeps the earlier (lower) class
      second = fmax(best, t.second);
      best = t.best;
      idx = t.idx;
    } else {
      second = fmax(second, t.best);
    }
  }
  if (idx >= C) idx = 0;  // only reachable with NaN scores, which are reported through `bad`
  RowScore r;
  r.idx = idx;
  r.bad = __any_sync(0xffffffffu, bad);
  // fp64 error of each score <= (F/32 + 7) u a  (<= 32-way split FMA chains + 5 shuffle adds + bias add)
  const double err = (static_cast<double>(F) / 32.0 + 8.0) * u * amax;
  r.ambiguous = !((best - second) > 2.0 * err);
  return r;
}

// ---------------------------------------------------------------------------------------------------------------
// TMA fp32 tile kernel
// ---------------------------------------------------------------------------------------------------------------
struct TmaKernelParams {
  const float* wt;    // [f_pad][CP]
  const float* bias;  // [CP]
  int32_t* labels;
  void* peers[8];
  int n_peers;
  int wire_u8;  // peer vectors hold one byte per label (classes <= 256) instead of int32
  long long row_offset;
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
  unsigned long long* counters;  // [0] ambiguous, [1] nonfinite, [2] re-scored rows
#ifdef UML_PROBE_WAIT_CLOCKS
  unsigned long long* probe_clocks;  // [4], see the diagnostic builds below
#endif
};

// fp64 scores of one row by the whole warp (kept out of line so the hot loop's register allocation is untouched)
__device__ __noinline__ int rescore_row_inline(const TmaKernelParams& p, long long row, int lane) {
  RowScore r;
  if (p.src.base) {
    const SrcView v = p.src;
    r = score_row_f64([&](int f) { return load_src(v, row, f); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, lane);
  } else if (p.x64) {
    const double* xr64 = p.x64 + row * p.ld64;
    r = score_row_f64([&](int f) { return xr64[f]; }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, lane);
  } else {
    const float* xr = p.x + row * p.ld;
    r = score_row_f64([&](int f) { return static_cast<double>(xr[f]); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, lane);
  }
  if (lane == 0) {
    if (r.bad) atomicAdd(&p.counters[1], 1ull);
    if (r.ambiguous) atomicAdd(&p.counters[0], 1ull);
  }
  return r.idx;
}

constexpr int kQueueCap = 2048;           // flagged-row queue of the QUEUE kernels (power of two)
constexpr int kQueueHeadroom = 1024;      // a warp publishes only while this many slots are free (8 warps x 128 rows)
constexpr int kThreadsQueue = kThreads + 32;  // + 1 fp64 re-score warp

// the final label of a re-scored row into every target the launch writes (one lane)
__device__ __forceinline__ void store_final_label(const TmaKernelParams& p, long long row, int idx) {
  if (p.labels) p.labels[row] = idx;
  for (int i = 0; i < p.n_peers; ++i) {
    if (p.wire_u8) static_cast<uint8_t*>(p.peers[i])[p.row_offset + row] = static_cast<uint8_t>(idx);
    else static_cast<int32_t*>(p.peers[i])[p.row_offset + row] = idx;
  }
}

// Diagnostic builds of this file (tools/linear_probe.cu defines these; the library defines neither):
//  UML_PROBE_FEED_ONLY    the scoring warps hand each stage back as soon as it has landed, without the math: what the
//                         ring (producer, order, barriers) delivers on its own
//  UML_PROBE_WAIT_CLOCKS  clock64() totals added into p.probe_clocks: [0] the producer's `empty` waits, [1] its whole
//                         loop, [2] the scoring warps' waits for their data, [3] their whole loops
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
#else
#define UML_PROBE_TIMED(total, ...) __VA_ARGS__
#endif

// WHOLE (f_pad == 64, linear_whole_rows): one ring stage is one 64-row tile with all its features, loaded as two
// {32 features, 64 rows} boxes onto one barrier; warp w scores the CTA's tiles w, w + 8, ... (2 rows per lane).
// Otherwise one stage is a 128-row x 32-feature box and a tile takes f_pad / 32 stages (4 rows per lane).
template <int C, bool EXACT, bool QUEUE, bool WHOLE>
__global__ void __launch_bounds__(kThreadsQueue, 1)
linear_argmax_tma_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ TmaKernelParams p) {
  constexpr int NCOL = C + (EXACT ? 1 : 0);  // accumulators per row (classes + error-bound column)
  constexpr int CP = (C + 1 + 3) / 4 * 4;    // padded columns of wt in shared memory (layout shared by both modes)
  constexpr int NW4 = (NCOL + 3) / 4;        // float4 loads of W per feature
  constexpr int TILE = WHOLE ? kWholeTileRows : kTileRows;  // rows per tile = rows per TMA box
  constexpr int R = TILE / 32;                               // rows per lane
  constexpr int BOX_BYTES = TILE * kChunkF * 4;              // one {32, TILE} box: 8 KiB (two per stage) or 16 KiB
  constexpr bool USE_F2 = EXACT;  // fp32x2 accumulator pairs (see the accumulator comment below)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // SWIZZLE_128B wants 1 KiB alignment

  const int S = p.num_stages;
  float* wt_s = reinterpret_cast<float*>(smem + static_cast<size_t>(S) * kStageBytes);
  float* bias_s = wt_s + p.f_pad * CP;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + CP);
  uint64_t* empty_bar = full_bar + S;
  // QUEUE kernels: rows flagged by the scoring warps travel through this shared-memory queue to the re-score warp
  // (slot value = row + 1, 0 = empty); ctl[0] = tail (reserved), ctl[1] = head (tickets claimed), ctl[2] = scoring
  // warps done, ctl[3] = slots consumed
  int* q_slots = reinterpret_cast<int*>(empty_bar + S);
  int* q_ctl = q_slots + kQueueCap;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // stage W^T (with its wmax column) and the bias once per CTA; they stay resident for every tile this CTA scores
  {
    const float4* src = reinterpret_cast<const float4*>(p.wt);
    float4* dst = reinterpret_cast<float4*>(wt_s);
    const int n4 = p.f_pad * CP / 4;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = __ldg(src + i);
    if (threadIdx.x < CP) bias_s[threadIdx.x] = __ldg(p.bias + threadIdx.x);
    if constexpr (QUEUE) {
      for (int i = threadIdx.x; i < kQueueCap + 4; i += blockDim.x) q_slots[i] = 0;
    }
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);
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

  if (warp == kConsumerWarps) {
    // ===================== TMA producer (one elected lane) =====================
    if (elect_one_sync()) {
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
      if constexpr (WHOLE) {
        // ring item n of this CTA = its n-th tile (tile blockIdx.x + n*G): both halves of its rows land together
        for (long long tile = blockIdx.x; tile < num_tiles; tile += G) {
          UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u));
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          uint8_t* dst = smem + static_cast<size_t>(stage) * kStageBytes;
          const int row = static_cast<int>(tile * TILE);
          tma_load_2d(dst, &xmap, &full_bar[stage], 0, row, policy);
          tma_load_2d(dst + BOX_BYTES, &xmap, &full_bar[stage], kChunkF, row, policy);
          next_stage();
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
    const bool scoring_warp = warp < kConsumerWarps;
    // lane l owns rows l, l+32, ... of the tile.  In every box row r sits at byte r*128 with its 16-byte chunks
    // XOR-swizzled by (r & 7); r & 7 == l & 7 for all of a lane's rows, so one swizzle term serves them all and the
    // eight lanes of every LDS.128 phase (lanes 8i..8i+7: l & 7 = 0..7) hit eight distinct bank groups.  The whole-row
    // stage is two such boxes (features 0-31, then 32-63 at +8 KiB), so the same holds in both halves.
    const uint32_t lanebase = static_cast<uint32_t>(lane) * 128u + static_cast<uint32_t>(lane & 7) * 16u;

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
          for (int j = 0; j < R; ++j) {
            const float x = e == 0 ? xv[j].x : e == 1 ? xv[j].y : e == 2 ? xv[j].z : xv[j].w;
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
          }
        }
      }
    };

    // ---- fused epilogue: argmax (first maximum wins), margin guard, label store (+ peer stores) ----
    auto finish_tile = [&](long long tile) {
      if constexpr (USE_F2) {
#pragma unroll
        for (int j = 0; j < R; ++j) {
#pragma unroll
          for (int i = 0; i < NPAIR; ++i) unpack2(acc2[j][i], acc[j][2 * i], acc[j][2 * i + 1]);
          if (ODD) acc[j][C - 1] = acc_last[j];
          acc[j][C] = acc_bound[j];
        }
      }
      const long long row0 = tile * TILE;
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
        if (row < p.n_rows) {
          if (p.labels) p.labels[row] = idxs[j];
          if (!p.wire_u8)
            for (int i = 0; i < p.n_peers; ++i) static_cast<int32_t*>(p.peers[i])[p.row_offset + row] = idxs[j];
        }
        if constexpr (EXACT && !QUEUE) {
          const unsigned mask = __ballot_sync(0xffffffffu, flag[j]);
          if (mask != 0u) {
            int base = 0;
            if (lane == 0) base = atomicAdd(p.flag_count, __popc(mask));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (flag[j]) {
              const int pos = base + __popc(mask & ((1u << lane) - 1u));
              if (pos < p.flag_cap) p.flag_rows[pos] = static_cast<int32_t>(row);
            }
          }
        }
      }
      if (p.wire_u8 && p.n_peers > 0) {
        // byte labels: transpose through shuffles so lane l < TILE/4 holds rows 4l..4l+3 of the tile and the whole
        // tile leaves as ONE coalesced TILE-byte store per target (instead of R int32 stores).  Row 4l+t sits in byte
        // (4l+t)/32 = l/8 of lane (4l+t) % 32's packed word.
        uint32_t packed = 0, word = 0;
#pragma unroll
        for (int j = 0; j < R; ++j) packed |= static_cast<uint32_t>(idxs[j]) << (8 * j);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const uint32_t w = __shfl_sync(0xffffffffu, packed, (4 * lane + t) & 31);
          word |= ((w >> (8 * (lane >> 3))) & 0xffu) << (8 * t);
        }
        const long long row4 = row0 + 4 * lane;
        const long long at = p.row_offset + row4;
        if (4 * lane < TILE) {
          if (row4 + 3 < p.n_rows && (at & 3) == 0) {
            for (int i = 0; i < p.n_peers; ++i)
              *reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(p.peers[i]) + at) = word;
          } else {
            for (int t = 0; t < 4; ++t)
              if (row4 + t < p.n_rows)
                for (int i = 0; i < p.n_peers; ++i)
                  static_cast<uint8_t*>(p.peers[i])[at + t] = static_cast<uint8_t>((word >> (8 * t)) & 0xffu);
          }
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
            if (tail - consumed <= kQueueCap - kQueueHeadroom) base = atomicAdd(&q_ctl[0], total);
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
                if (lane == 0) store_final_label(p, row, idx64);
              }
            }
            if (lane == 0) atomicAdd(&p.counters[2], static_cast<unsigned long long>(total));
          }
        }
      }
    };

    if constexpr (WHOLE) {
      // this warp's ring items are n = warp, warp + 8, ... (stage n % S, phase (n / S) & 1); S >= 8 lets stage and
      // phase advance without a division.  Both waits keep the invariant argued below: the next item is n + 8 <= n + S.
      uint32_t stage = static_cast<uint32_t>(warp), phase = 0;
      for (long long tile = blockIdx.x + warp * G; scoring_warp && tile < num_tiles; tile += G * kConsumerWarps) {
        init_acc();
        UML_PROBE_TIMED(probe_wait, mbar_wait(&empty_bar[stage], phase ^ 1u); mbar_wait(&full_bar[stage], phase));
        const uint8_t* xs = smem + static_cast<size_t>(stage) * kStageBytes;
        fma_box(xs, wt_s);
        fma_box(xs + BOX_BYTES, wt_s + kChunkF * CP);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);  // hand the stage back to the producer
        stage += kConsumerWarps;
        if (stage >= static_cast<uint32_t>(S)) {
          stage -= S;
          phase ^= 1u;
        }
        finish_tile(tile);
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
            fma_box(smem + static_cast<size_t>(stage) * kStageBytes, wt_s + k * kChunkF * CP);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);  // hand the stage back to the producer
          }
          finish_tile(tile);
        }
        seq_base += static_cast<uint32_t>(KC * nv);
      }
    }
#ifdef UML_PROBE_WAIT_CLOCKS
    if (scoring_warp && lane == 0) {
      atomicAdd(&p.probe_clocks[2], static_cast<unsigned long long>(probe_wait));
      atomicAdd(&p.probe_clocks[3], static_cast<unsigned long long>(clock64() - probe_start));
    }
#endif
    if constexpr (EXACT && QUEUE) {
      if (warp < kConsumerWarps) {
        __syncwarp();
        if (lane == 0) {
          __threadfence_block();
          atomicAdd(&q_ctl[2], 1);  // this scoring warp has published everything it will ever publish
        }
      }
      // ===================== fp64 re-score: warp 9 drains the queue while the scoring warps stream; a scoring warp
      // that has finished its tiles joins in, so a long tail of flagged rows (wide rows, many near-ties) is shared
      // by all ten warps instead of waiting for one =====================
      int n_done = 0;
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
            if (v == 0 && atomicAdd(&q_ctl[2], 0) == kConsumerWarps) {
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
        const int idx64 = rescore_row_inline(p, row, lane);
        if (lane == 0) store_final_label(p, row, idx64);
        ++n_done;
      }
      if (lane == 0 && n_done > 0) atomicAdd(&p.counters[2], static_cast<unsigned long long>(n_done));
    }
  }
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
  int32_t* labels;
  void* peers[8];
  int n_peers;
  int wire_u8;
  long long row_offset;
  unsigned long long* counters;  // [0] ambiguous, [1] nonfinite, [2] flagged (re-scored) rows
  int smem_weights;              // W, b staged in dynamic shared memory ((C F + C) doubles)
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
      r = score_row_f64([&](int f) { return load_src(v, row, f); }, w64, S, b64, F, C, lane);
    } else if (p.x64) {
      const double* xr64 = p.x64 + row * p.ld64;
      r = score_row_f64([&](int f) { return xr64[f]; }, w64, S, b64, F, C, lane);
    } else {
      const float* xr = p.x + row * p.ld;
      r = score_row_f64([&](int f) { return static_cast<double>(xr[f]); }, w64, S, b64, F, C, lane);
    }
    if (lane == 0) {
      if (p.labels) p.labels[row] = r.idx;
      for (int q = 0; q < p.n_peers; ++q) {
        if (p.wire_u8) static_cast<uint8_t*>(p.peers[q])[p.row_offset + row] = static_cast<uint8_t>(r.idx);
        else static_cast<int32_t*>(p.peers[q])[p.row_offset + row] = r.idx;
      }
      if (r.bad) atomicAdd(&p.counters[1], 1ull);
      if (r.ambiguous) atomicAdd(&p.counters[0], 1ull);
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
    for (int i = threadIdx.x; i < p.n_classes; i += blockDim.x) rs_w[nw + i] = p.b64[i];
    __syncthreads();
  }
  pdl_wait_for_predecessor();  // the flag list is written by the scoring kernel this launch depends on
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long n = p.all_rows ? p.n_rows : static_cast<long long>(min(*p.flag_count, p.flag_cap));
  if (!p.all_rows && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&p.counters[2], static_cast<unsigned long long>(n));
  if (p.smem_weights) {
    const double* ws = rs_w;
    rescore_rows(p, ws, ws + nw, n, lane, warp_global, warps_total);
  } else {
    rescore_rows(p, p.w64, p.b64, n, lane, warp_global, warps_total);
  }
  // hand the flag list back empty: every block has read *flag_count before it gets here, so the last one to finish may
  // reset it (and the ticket) for the next scoring launch on this stream - no memset between steps
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned long long ticket = atomicAdd(&p.counters[3], 1ull);
    if (ticket == static_cast<unsigned long long>(gridDim.x) - 1ull) {
      *const_cast<int*>(p.flag_count) = 0;
      p.counters[3] = 0ull;
      __threadfence();
    }
  }
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
  SmallResult* out;
};

__global__ void __launch_bounds__(256) linear_small_kernel(const SmallParams p) {
  const int lane = threadIdx.x & 31;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= p.n_rows) return;
  const SrcView v = p.src;
  const RowScore r = score_row_f64([&](int f) { return load_src(v, row, f); }, p.w64, p.w64_stride, p.b64, p.n_features, p.n_classes, lane);
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
static size_t tma_fixed_smem(const LinearDeviceModel& m) {
  // alignment slack + W^T + bias + barriers (64 stages max) + the flagged-row queue of the QUEUE kernels
  return 1024 + static_cast<size_t>(m.f_pad) * m.cp * 4 + static_cast<size_t>(m.cp) * 4 + 2 * 64 * 8 + (kQueueCap + 4) * 4;
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

template <int C, bool EXACT, bool QUEUE, bool WHOLE>
static cudaError_t launch_one(const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                              cudaStream_t stream) {
  auto kern = linear_argmax_tma_kernel<C, EXACT, QUEUE, WHOLE>;
  static size_t configured = 0;  // per instantiation (one device per process): set the attribute once, not per launch
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  kern<<<grid, QUEUE ? kThreadsQueue : kThreads, smem, stream>>>(xmap, p);
  return cudaGetLastError();
}

template <bool EXACT, bool QUEUE, bool WHOLE>
static cudaError_t dispatch_classes(int C, const CUtensorMap& xmap, const TmaKernelParams& p, int grid, size_t smem,
                                    cudaStream_t stream) {
  switch (C) {
#define UML_CASE(N) \
  case N:           \
    return launch_one<N, EXACT, QUEUE, WHOLE>(xmap, p, grid, smem, stream);
    UML_CASE(2) UML_CASE(3) UML_CASE(4) UML_CASE(5) UML_CASE(6) UML_CASE(7) UML_CASE(8) UML_CASE(9) UML_CASE(10)
    UML_CASE(11) UML_CASE(12) UML_CASE(13) UML_CASE(14) UML_CASE(15) UML_CASE(16)
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

cudaError_t launch_linear_tma(const CUtensorMap& xmap, const LinearDeviceModel& m, const LinearLaunch& l, bool exact,
                              const FlagList& flags, int sm_count, cudaStream_t stream, std::string* err,
                              bool* rescore_kernel_needed) {
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
  p.labels = l.labels;
  p.n_peers = l.n_peers;
  p.wire_u8 = l.wire_u8;
  for (int i = 0; i < 8; ++i) p.peers[i] = i < l.n_peers ? l.peers[i] : nullptr;
  p.row_offset = l.row_offset;
  p.n_rows = l.n_rows;
  const bool whole = linear_whole_rows(m.f_pad);
  const int tile_rows = linear_box_rows(m.f_pad);
  p.num_tiles = (l.n_rows + tile_rows - 1) / tile_rows;
  p.f_pad = m.f_pad;
  p.kc = m.f_pad / kChunkF;
  const size_t fixed = tma_fixed_smem(m);
  int stages = static_cast<int>((static_cast<size_t>(kMaxSmemBytes) - fixed) / kStageBytes);
  stages = std::min(stages, 64);
  // test hook: the shallowest legal ring (stages == consumer warps) stresses the barrier protocol
  if (const char* env = getenv("UML_B200_STAGES")) stages = std::max(kConsumerWarps, std::min(stages, atoi(env)));
  p.num_stages = stages;
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
  p.counters = flags.counters;
  const size_t smem = fixed + static_cast<size_t>(stages) * kStageBytes;
  const long long slots = (p.num_tiles + kConsumerWarps - 1) / kConsumerWarps;
  const int grid = static_cast<int>(std::min<long long>(sm_count, std::max<long long>(1, slots)));
  if (whole) {
    if (!exact) return dispatch_classes<false, false, true>(m.n_classes, xmap, p, grid, smem, stream);
    return inline_rescore ? dispatch_classes<true, true, true>(m.n_classes, xmap, p, grid, smem, stream)
                          : dispatch_classes<true, false, true>(m.n_classes, xmap, p, grid, smem, stream);
  }
  if (!exact) return dispatch_classes<false, false, false>(m.n_classes, xmap, p, grid, smem, stream);
  return inline_rescore ? dispatch_classes<true, true, false>(m.n_classes, xmap, p, grid, smem, stream)
                        : dispatch_classes<true, false, false>(m.n_classes, xmap, p, grid, smem, stream);
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
  p.labels = l.labels;
  p.n_peers = l.n_peers;
  p.wire_u8 = l.wire_u8;
  for (int i = 0; i < 8; ++i) p.peers[i] = i < l.n_peers ? l.peers[i] : nullptr;
  p.row_offset = l.row_offset;
  p.counters = flags.counters;
  // shared-memory copy of W, b when it fits next to nothing else (<= 200 KB)
  size_t smem = (static_cast<size_t>(m.n_features) * m.w64_stride + m.n_classes) * sizeof(double);
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
