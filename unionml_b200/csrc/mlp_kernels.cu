// Scoring kernels for the 2-layer MLP predictor  argmax(softmax(W2 relu(W1 x + b1) + b2)) = argmax of the logits.
//
// Replaces PytorchModel.forward + .argmax(1) of the reference's torch quickstart
// (unionml:tests/integration/pytorch_app/quickstart.py:14-24, 68-70; hyperparameters 64 -> 32 -> 10 at :80).
//
//  * mlp_argmax_tma_kernel<H, C, EXACT>: the same persistent TMA + mbarrier ring (128-row x 32-feature boxes) as the
//    linear kernel; consumer warps work in pairs on a box (64 rows each, 2 rows x H hidden accumulators per lane).  Layer 1 runs per
//    landed box (W1^T rows are warp-uniform broadcast LDS.128 from shared memory), then ReLU, layer 2 and the argmax are
//    fused in registers.  EXACT mode carries two bound accumulators (A1 over layer 1, A2 over layer 2) and re-scores
//    rows whose logit margin is inside the propagated fp32 error bound in fp64.
//    PROBA instantiations store softmax(logits) instead of the label: each warp's 32 consecutive rows per j leave as one
//    coalesced run through shared memory (mlp_proba.cuh).
//    TOPK instantiations store the k largest logits' class indices (and probabilities) the same way; EXACT ones flag
//    rows whose top k + 1 logits are not separated by the bound (mlp_topk.cuh, DESIGN.md 3.8).
//  * mlp_topk_f64_kernel: the fp64 top-k of those flagged rows, or of every row for shapes / k no tile kernel takes.
//  * mlp_rescore_f64_kernel: warp per row, lane per hidden unit, fp64; flagged rows of EXACT mode, or every row for
//    shapes the tile kernel is not instantiated for.
//  * mlp_proba_f64_kernel: class probabilities for those shapes - the same fp64 scorer, then a float64 softmax - or
//    for the rows a tensor-core PROBA launch flagged as not tf32 values.
//  * mlp_small_kernel: the online path (B <= 64 rows): the same fp64 scorer on the request block in pinned host memory,
//    writing labels, class probabilities or top-k records.
//
// This is CUDA-core fp32 (FFMA): 4 736 flop/row puts the HBM roofline (25 G rows/s) above the FFMA peak, so this kernel
// is FMA-pipe bound (~0.66 ms per 10M rows at 1.9 GHz).  It serves batches whose features are NOT tf32 values (general
// floats); tf32-representable batches (integer / pixel domains) take the tensor-core kernel in mlp_tc_kernels.cu.
#include <algorithm>
#include <cstdlib>

#include "uml_common.cuh"
#include "label_store.cuh"
#include "tma_ring.cuh"
#include "mlp_rescore.cuh"
#include "mlp_proba.cuh"
#include "mlp_topk.cuh"

#ifndef UML_MLP_UNROLL_Q
#define UML_MLP_UNROLL_Q 8  // feature-quad unroll of the layer-1 loop
#endif
#define UML_PRAGMA_(x) _Pragma(#x)
#define UML_UNROLL(n) UML_PRAGMA_(unroll n)

namespace uml {

// 8 consumer warps work as 4 PAIRS: a pair shares one 128-row x 32-feature box, warp 2p takes rows 0..63 and warp 2p+1
// rows 64..127 (2 rows per lane x 32 hidden accumulators = 64 registers, inside the 168-register cap of a 9-warp CTA)
// and two warps per SM sub-partition hide each other's LDS / barrier latency.  A stage is released by both warps.
constexpr int kMlpPairs = 4;
constexpr int kMlpConsumerWarps = 2 * kMlpPairs;
constexpr int kMlpThreads = (kMlpConsumerWarps + 1) * 32;
constexpr int kMlpTileRows = kTileRows;                      // 128 rows x 32 features, same boxes as the linear kernel
constexpr int kMlpStageBytes = kStageBytes;                  // 16 KiB
constexpr int kMlpRowsPerLane = 2;                           // rows per lane within a warp's 64-row half

struct MlpKernelParams {
  const float* w1t;  // [f_pad][H + 4]   column H = max_n |w1_nf|
  const float* b1;   // [H + 4]          entry  H = max_n |b1_n|
  const float* w2t;  // [H][CP]          column C = max_c |w2_cn|
  const float* b2;   // [CP]             entry  C = max_c |b2_c|
  int32_t* labels;
  long long n_rows;
  long long num_tiles;
  int f_pad;
  int kc;
  int num_stages;
  float e1_scale;  // (F+4) 2^-24 (1+slack) * max_c sum_n |w2_cn|   -> layer-1 error as it reaches a logit
  float e2_scale;  // (H+4) 2^-24 (1+slack)                          -> layer-2 accumulation error
  int* flag_count;
  int32_t* flag_rows;
  int flag_cap;
  float* proba;  // PROBA kernels: [n_rows][C] row-major
};

// TOPK kernels take the parameters in this longer form (a longer MlpKernelParams changes the code ptxas makes for
// every other instantiation)
struct MlpTopkKernelParams : MlpKernelParams {
  int32_t* topk_idx;  // [n_rows][topk_k] class indices
  float* topk_proba;  // [n_rows][topk_k] their probabilities, or nullptr: not written
  int topk_k;
};

template <int H, int C, bool EXACT, bool PROBA, bool TOPK = false, class Params = MlpKernelParams>
__global__ void __launch_bounds__(kMlpThreads, 1)
mlp_argmax_tma_kernel(const __grid_constant__ CUtensorMap xmap, const Params p) {
  constexpr int HP = H + 4;
  constexpr int CP = (C + 1 + 3) / 4 * 4;
  constexpr int NC2 = C + (EXACT ? 1 : 0);
  constexpr int NW2 = (NC2 + 3) / 4;
  constexpr int R = kMlpRowsPerLane;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int S = p.num_stages;
  float* w1_s = reinterpret_cast<float*>(smem + static_cast<size_t>(S) * kMlpStageBytes);
  float* b1_s = w1_s + p.f_pad * HP;
  float* w2_s = b1_s + HP;
  float* b2_s = w2_s + H * CP;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(b2_s + CP);
  uint64_t* empty_bar = full_bar + S;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  {
    const float4* src = reinterpret_cast<const float4*>(p.w1t);
    float4* dst = reinterpret_cast<float4*>(w1_s);
    for (int i = threadIdx.x; i < p.f_pad * HP / 4; i += kMlpThreads) dst[i] = __ldg(src + i);
    for (int i = threadIdx.x; i < H * CP; i += kMlpThreads) w2_s[i] = __ldg(p.w2t + i);
    if (threadIdx.x < HP) b1_s[threadIdx.x] = __ldg(p.b1 + threadIdx.x);
    if (threadIdx.x < CP) b2_s[threadIdx.x] = __ldg(p.b2 + threadIdx.x);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // both warps of the pair that read the stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  pdl_launch_dependents();  // see linear_kernels.cu: the re-score kernel may be scheduled while this grid drains
  const long long G = gridDim.x;
  const long long num_tiles = p.num_tiles;
  const int KC = p.kc;

  if (warp == kMlpConsumerWarps) {
    if (elect_one_sync()) {
      tma_prefetch_desc(&xmap);
      const uint64_t policy = make_evict_first_policy();
      int stage = 0;
      uint32_t phase = 0;
      for (long long first = blockIdx.x; first < num_tiles; first += G * kMlpPairs) {
        const int nv = static_cast<int>(min(static_cast<long long>(kMlpPairs), (num_tiles - first + G - 1) / G));
        for (int k = 0; k < KC; ++k) {
          for (int w = 0; w < nv; ++w) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            mbar_arrive_expect_tx(&full_bar[stage], kMlpStageBytes);
            tma_load_2d(smem + static_cast<size_t>(stage) * kMlpStageBytes, &xmap, &full_bar[stage], k * kChunkF,
                        static_cast<int>((first + w * G) * kMlpTileRows), policy);
            if (++stage == S) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
    }
  } else {
    const int pair = warp >> 1;
    const int half = warp & 1;
    const uint32_t lanebase = static_cast<uint32_t>(half * 64 + lane) * 128u + static_cast<uint32_t>(lane & 7) * 16u;
    uint32_t seq_base = 0;
    for (long long first = blockIdx.x; first < num_tiles; first += G * kMlpPairs) {
      const int nv = static_cast<int>(min(static_cast<long long>(kMlpPairs), (num_tiles - first + G - 1) / G));
      if (pair < nv) {
        const long long tile = first + pair * G;
        uint64_t h2[R][H / 2];  // hidden accumulators as fp32x2 pairs (units 2i, 2i+1)
        float a1[R];
#pragma unroll
        for (int j = 0; j < R; ++j) {
#pragma unroll
          for (int n = 0; n < H / 2; ++n) h2[j][n] = pack2(b1_s[2 * n], b1_s[2 * n + 1]);
          a1[j] = b1_s[H];
        }
        for (int k = 0; k < KC; ++k) {
          const uint32_t seq = seq_base + static_cast<uint32_t>(k * nv + pair);
          const uint32_t stage = seq % static_cast<uint32_t>(S);
          const uint32_t phase = (seq / static_cast<uint32_t>(S)) & 1u;
          mbar_wait(&empty_bar[stage], phase ^ 1u);  // previous occupant released (see linear_kernels.cu)
          mbar_wait(&full_bar[stage], phase);
          const uint8_t* xs = smem + static_cast<size_t>(stage) * kMlpStageBytes;
          const float* wk = w1_s + k * kChunkF * HP;
          UML_UNROLL(UML_MLP_UNROLL_Q)
          for (int q = 0; q < kChunkF / 4; ++q) {
            float4 xv[R];
            const uint32_t off = lanebase ^ static_cast<uint32_t>(q * 16);
#pragma unroll
            for (int j = 0; j < R; ++j) xv[j] = *reinterpret_cast<const float4*>(xs + off + j * 32 * 128);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float* wrow = wk + (q * 4 + e) * HP;
              float x[R];
#pragma unroll
              for (int j = 0; j < R; ++j) x[j] = e == 0 ? xv[j].x : e == 1 ? xv[j].y : e == 2 ? xv[j].z : xv[j].w;
#pragma unroll
              for (int m = 0; m < H / 4; ++m) {
                const float4 t = *reinterpret_cast<const float4*>(wrow + m * 4);
                const uint64_t w01 = pack2(t.x, t.y), w23 = pack2(t.z, t.w);
#pragma unroll
                for (int j = 0; j < R; ++j) {
                  const uint64_t xx = pack2(x[j], x[j]);
                  h2[j][m * 2 + 0] = fma2(xx, w01, h2[j][m * 2 + 0]);
                  h2[j][m * 2 + 1] = fma2(xx, w23, h2[j][m * 2 + 1]);
                }
              }
              if (EXACT) {
                const float wmax = wrow[H];
#pragma unroll
                for (int j = 0; j < R; ++j) a1[j] = fmaf(fabsf(x[j]), wmax, a1[j]);
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }

        // ---- ReLU, layer 2 (hidden unit outermost: each W2^T row is loaded once for the lane's 4 rows) ----
        constexpr int NZ2 = (NC2 + 1) / 2;  // logit accumulators as pairs (a padding lane multiplies a zero weight)
        uint64_t z2[R][NZ2];
#pragma unroll
        for (int j = 0; j < R; ++j)
#pragma unroll
          for (int c = 0; c < NZ2; ++c) z2[j][c] = pack2(b2_s[2 * c], 2 * c + 1 < CP ? b2_s[2 * c + 1] : 0.f);
#pragma unroll
        for (int n2 = 0; n2 < H / 2; ++n2) {
          float hv[R][2];
#pragma unroll
          for (int j = 0; j < R; ++j) {
            unpack2(h2[j][n2], hv[j][0], hv[j][1]);
            hv[j][0] = fmaxf(hv[j][0], 0.f);
            hv[j][1] = fmaxf(hv[j][1], 0.f);
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int n = 2 * n2 + u;
            uint64_t w2p[NW2 * 2];
#pragma unroll
            for (int m = 0; m < NW2; ++m) {
              const float4 t = *reinterpret_cast<const float4*>(w2_s + n * CP + m * 4);
              w2p[m * 2 + 0] = pack2(t.x, t.y);
              w2p[m * 2 + 1] = pack2(t.z, t.w);
            }
#pragma unroll
            for (int j = 0; j < R; ++j) {
              const uint64_t hh = pack2(hv[j][u], hv[j][u]);
#pragma unroll
              for (int c = 0; c < NZ2; ++c) z2[j][c] = fma2(hh, w2p[c], z2[j][c]);
            }
          }
        }
        float z[R][2 * NZ2];
#pragma unroll
        for (int j = 0; j < R; ++j)
#pragma unroll
          for (int c = 0; c < NZ2; ++c) unpack2(z2[j][c], z[j][2 * c], z[j][2 * c + 1]);
        // ---- argmax (first maximum wins), margin guard, label store ----
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const long long row = tile * kMlpTileRows + half * 64 + lane + 32 * j;
          if constexpr (PROBA) {
            // the warp's rows 32 j .. 32 j + 31 of its half: lane l's C probabilities at l C of the warp's strip
            float* strip = reinterpret_cast<float*>(empty_bar + S) + warp * 32 * C;
            float pr[C];
            mlp_softmax_f32<C>(z[j], pr);
#pragma unroll
            for (int c = 0; c < C; ++c) strip[lane * C + c] = pr[c];
            __syncwarp();
            mlp_proba_store_run<C, 32>(strip, p.proba, row - lane, p.n_rows, lane);
            __syncwarp();  // the strip is rewritten for the next run
            continue;
          }
          if constexpr (TOPK) {
            // lane l's k indices at l k of the warp's strip, its k probabilities at l k of the strip's second half
            constexpr int M = C < kMlpTopkMax + 1 ? C : kMlpTopkMax + 1;
            const int k = p.topk_k;
            const bool want_p = p.topk_proba != nullptr;
            float pr[C];
            if (want_p) {
              mlp_softmax_f32<C>(z[j], pr);
            } else {
#pragma unroll
              for (int c = 0; c < C; ++c) pr[c] = 0.f;
            }
            float v[M], pv[M];
            int id[M];
            mlp_topk_select<C, M>(z[j], pr, v, id, pv);
            int32_t* si = reinterpret_cast<int32_t*>(empty_bar + S) + warp * kMlpTopkStripWords;
            float* sp = reinterpret_cast<float*>(si + 32 * kMlpTopkMax);
#pragma unroll
            for (int r = 0; r < M; ++r) {
              if (r < k) {
                si[lane * k + r] = id[r];
                sp[lane * k + r] = pv[r];
              }
            }
            __syncwarp();
            mlp_topk_store_run<32>(si, p.topk_idx, row - lane, p.n_rows, k, lane);
            if (want_p) mlp_topk_store_run<32>(sp, p.topk_proba, row - lane, p.n_rows, k, lane);
            __syncwarp();  // the strip is rewritten for the next run
            if (EXACT) {
              const float err = p.e1_scale * a1[j] + p.e2_scale * z[j][C];
              const bool certain = mlp_topk_certain<M>(v, min(k, C - 1), 2.0f * err);
              mlp_topk_flag(row < p.n_rows && !certain, row, p.flag_count, p.flag_rows, p.flag_cap, lane);
            }
            continue;
          }
          float best = z[j][0];
          float second = -INFINITY;
          int idx = 0;
#pragma unroll
          for (int c = 1; c < C; ++c) {
            if (z[j][c] > best) {
              second = best;
              best = z[j][c];
              idx = c;
            } else {
              second = fmaxf(second, z[j][c]);
            }
          }
          const bool in_range = row < p.n_rows;
          if (in_range) p.labels[row] = idx;
          if (EXACT) {
            // |z_c - true| <= E1 * sum_n |w2_cn| + (H+4) u A2, E1 = (F+4) u A1 (ReLU is 1-Lipschitz)
            const float err = p.e1_scale * a1[j] + p.e2_scale * z[j][C];
            const bool certain = (best - second) > 2.0f * err;
            flag_rows_warp(in_range && !certain, row, p, lane);
          }
        }
      }
      seq_base += static_cast<uint32_t>(KC * nv);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// fp64 re-score / generic kernel: warp per row, lane per hidden unit
// ---------------------------------------------------------------------------------------------------------------
struct MlpRescoreParams {
  const float* x;
  long long ld;
  long long n_rows;
  const double* pack;  // the shared-memory image of the fp64 operands (mlp_rs_build_pack)
  int F, H, C;
  const int* flag_count;
  const int32_t* flag_rows;
  int flag_cap;
  int all_rows;
  LabelTargets targets;
  unsigned long long* counters;
};

constexpr int kMlpRsRows = 4;  // rows per warp pass (mlp_rescore.cuh: shared-memory wavefronts per row fall 3 -> 1)

// Shared-memory version (mlp_rescore.cuh): the fp64 image of the model (W1 [F][H], W2 [C][H+1], biases, bound vectors;
// built on the host at load) is copied once per block; a warp scores four rows per pass - their features and hidden
// activations interleaved in the warp's own strip, so every W element it reads from shared memory is used four times.
// Layer 1: lane per hidden unit.  Layer 2: lane per class (no warp reductions), then one butterfly per row for arg-max
// and runner-up.
__global__ void __launch_bounds__(256) mlp_rescore_f64_kernel(const MlpRescoreParams p) {
  extern __shared__ __align__(16) double rs_smem[];
  constexpr int R = kMlpRsRows;
  // (weights are staged first: they do not depend on the scoring kernel; the flag list does - see the wait below)
  MlpRsView view = mlp_rs_stage(rs_smem, p.pack, p.F, p.H, p.C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* xs = rs_smem + mlp_rs_weight_doubles(p.F, p.H, p.C) + warp * mlp_rs_strip_doubles(p.F, p.H, R);
  double* hv = xs + p.F * R;
  __syncthreads();
  mlp_rs_finish_stage(view);

  pdl_wait_for_predecessor();  // from here on: the flag list and labels of the scoring kernel this launch depends on
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long n = flag_list_rows(p);
  // warp w takes entries [w*R, w*R + R) of the list, then strides by all warps: a short list spreads over many warps
  for (long long i = warp_global * R; i < n; i += warps_total * R) {
    long long row[R];
    const float* xr[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long j = i + r < n ? i + r : i;  // unused slots repeat the first row (result ignored)
      row[r] = p.all_rows ? j : static_cast<long long>(p.flag_rows[j]);
      xr[r] = p.x + row[r] * p.ld;
    }
    MlpRowResult res[R];
    mlp_rs_rows<R>(view, xr, xs, hv, lane, res);
    if (lane < R && i + lane < n) {
      // lane r publishes row r (R <= 4 lanes, one per row)
      long long my_row = row[0];
      MlpRowResult mine = res[0];
#pragma unroll
      for (int r = 1; r < R; ++r) {
        if (lane == r) {
          my_row = row[r];
          mine = res[r];
        }
      }
      store_label(p.targets, my_row, mine.idx);
      count_rescored_row(p, mine.bad, mine.ambiguous);
    }
  }
  flag_list_hand_back(p);
}

// One row's float64 outputs from the logits a pass of the fp64 scorer left in its strip (logit c at zr[c R]): the
// softmax (max, exp(z - m), lane sum, true division), each probability rounded once to fp32, and for top-k each class's
// rank in the stable descending order (the logits above it, and equal logits of lower index) - no sort, any k <= C.
// proba: the row's C probabilities by class, or nullptr.  k > 0: idx / kproba receive slot `rank` of a class of rank < k
// (kproba may be nullptr).  Returns, in every lane, whether a consecutive gap among ranks 0 .. min(k, C - 1) is within
// twice err (the labels' top-2 margin rule).  Every float64 probability and top-k of the MLP leaves through this one
// routine (mlp_proba_f64_kernel, mlp_topk_f64_kernel, mlp_small_kernel), so their bits agree by construction.
__device__ __noinline__ bool mlp_f64_row_outputs(const double* zr, int R, int C, int lane, float* proba, int k,
                                                 int32_t* idx, float* kproba, double err) {
  double m = -INFINITY;
  for (int c = lane; c < C; c += 32) m = fmax(m, zr[c * R]);
  m = warp_max(m, 1);
  double s = 0.0;
  for (int c = lane; c < C; c += 32) s += exp(zr[c * R] - m);
  s = warp_sum(s);
  const int kk = min(k, C - 1);
  bool ambiguous = false;
  for (int c = lane; c < C; c += 32) {
    const double zc = zr[c * R];
    const float pc = proba || kproba ? static_cast<float>(exp(zc - m) / s) : 0.f;
    if (proba) proba[c] = pc;
    if (k > 0) {
      int rank = 0;
      double above = INFINITY;  // the smallest logit ranked above c: its neighbour one rank up
      for (int o = 0; o < C; ++o) {
        const double zo = zr[o * R];
        if (zo > zc || (zo == zc && o < c)) {
          ++rank;
          above = fmin(above, zo);
        }
      }
      if (rank < k) {
        idx[rank] = c;
        if (kproba) kproba[rank] = pc;
      }
      if (rank >= 1 && rank <= kk && !((above - zc) > 2.0 * err)) ambiguous = true;
    }
  }
  return __any_sync(0xffffffffu, ambiguous);
}

// class probabilities for shapes no tile kernel takes: the logits of the fp64 scorer above (mlp_rs_rows), then
// mlp_f64_row_outputs.  A warp scores kMlpRsRows rows per pass; lane per class, so each row's C floats leave as
// consecutive stores.  Every row (all_rows), or the rows on the flag list: those the tensor-core PROBA kernel in front of
// this launch scored from features that are not tf32 values, whose probabilities this overwrites.
struct MlpProbaF64Params {
  const float* x;
  long long ld;
  long long n_rows;
  const double* pack;
  int F, H, C;
  float* proba;
  const int* flag_count;
  const int32_t* flag_rows;
  int flag_cap;
  int all_rows;
  unsigned long long* counters;
};

__global__ void __launch_bounds__(256) mlp_proba_f64_kernel(const MlpProbaF64Params p) {
  extern __shared__ __align__(16) double rs_smem[];
  constexpr int R = kMlpRsRows;
  MlpRsView view = mlp_rs_stage(rs_smem, p.pack, p.F, p.H, p.C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* xs = rs_smem + mlp_rs_weight_doubles(p.F, p.H, p.C) + warp * (mlp_rs_strip_doubles(p.F, p.H, R) + p.C * R);
  double* hv = xs + p.F * R;
  double* zs = hv + p.H * R;  // the pass's logits, [c][R]
  __syncthreads();
  mlp_rs_finish_stage(view);

  pdl_wait_for_predecessor();  // flagged mode: the flag list and outputs of the tile kernel this launch depends on
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long n = flag_list_rows(p);
  for (long long i = warp_global * R; i < n; i += warps_total * R) {
    long long row[R];
    const float* xr[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long j = i + r < n ? i + r : i;  // unused slots repeat the first row (result ignored)
      row[r] = p.all_rows ? j : static_cast<long long>(p.flag_rows[j]);
      xr[r] = p.x + row[r] * p.ld;
    }
    MlpRowResult res[R];
    mlp_rs_rows<R, true>(view, xr, xs, hv, lane, res, zs);
    for (int r = 0; r < R && i + r < n; ++r) {
      mlp_f64_row_outputs(zs + r, R, p.C, lane, p.proba + row[r] * p.C, 0, nullptr, nullptr, 0.0);
      if (!p.all_rows && lane == 0) count_rescored_row(p, res[r].bad, false);
    }
    __syncwarp();  // the strip is rewritten by the next pass
  }
  if (!p.all_rows) flag_list_hand_back(p);
}

// top-k of the float64 network: the flagged rows of a TOPK tile kernel (EXACT mode, or rows that are not tf32 values),
// or every row for a shape or k no tile kernel takes.  The fp64 scorer above (logits and their bound kept), then
// mlp_f64_row_outputs: a row where a consecutive gap among ranks 0 .. min(k, C - 1) is within twice the fp64 logit
// bound counts as ambiguous, as the labels' top-2 margin does.
struct MlpTopkF64Params {
  const float* x;
  long long ld;
  long long n_rows;
  const double* pack;
  int F, H, C;
  int k;
  int32_t* idx;   // [n_rows][k]
  float* proba;   // [n_rows][k] or nullptr
  const int* flag_count;
  const int32_t* flag_rows;
  int flag_cap;
  int all_rows;
  unsigned long long* counters;
};

__global__ void __launch_bounds__(256) mlp_topk_f64_kernel(const MlpTopkF64Params p) {
  extern __shared__ __align__(16) double rs_smem[];
  constexpr int R = kMlpRsRows;
  MlpRsView view = mlp_rs_stage(rs_smem, p.pack, p.F, p.H, p.C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* xs = rs_smem + mlp_rs_weight_doubles(p.F, p.H, p.C) + warp * (mlp_rs_strip_doubles(p.F, p.H, R) + p.C * R);
  double* hv = xs + p.F * R;
  double* zs = hv + p.H * R;  // the pass's logits, [c][R]
  __syncthreads();
  mlp_rs_finish_stage(view);

  pdl_wait_for_predecessor();  // flagged mode: the flag list and outputs of the tile kernel this launch depends on
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long n = flag_list_rows(p);
  const int k = p.k;
  for (long long i = warp_global * R; i < n; i += warps_total * R) {
    long long row[R];
    const float* xr[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long j = i + r < n ? i + r : i;  // unused slots repeat the first row (result ignored)
      row[r] = p.all_rows ? j : static_cast<long long>(p.flag_rows[j]);
      xr[r] = p.x + row[r] * p.ld;
    }
    MlpRowResult res[R];
    double err[R];
    mlp_rs_rows<R, true, true>(view, xr, xs, hv, lane, res, zs, err);
    for (int r = 0; r < R && i + r < n; ++r) {
      const long long at = (p.all_rows ? i + r : static_cast<long long>(p.flag_rows[i + r])) * k;
      const bool ambiguous = mlp_f64_row_outputs(zs + r, R, p.C, lane, nullptr, k, p.idx + at,
                                                 p.proba ? p.proba + at : nullptr, err[r]);
      if (lane == 0) count_rescored_row(p, res[r].bad, ambiguous);
    }
    __syncwarp();  // the strip is rewritten by the next pass
  }
  flag_list_hand_back(p);
}

// small-batch kernel of the online path (fastapi.py /predict, B <= 64 rows): the fp64 scorer above on the request's
// raw feature block, which the kernel reads straight from pinned host memory - no staging pass, no tile kernel, no
// guard, exact by construction.  Each warp casts its four rows to fp32 as the staging kernels do (convert_one: the
// value as double, then to float), so this route scores the same fp32 features as the chunk pipeline and as the
// reference predictor (`torch.from_numpy(values).float()`), into an fp32 strip in its own shared memory.
// OUT (kSmallLabels / kSmallProba / kSmallTopk): what it writes besides each row's status - the label, or through
// mlp_f64_row_outputs the row's record in p.rec: C fp32 probabilities, or k int32 class indices then their k fp32
// probabilities.  The record forms keep the pass's logits in a further C x 4 doubles of the warp's strip.
struct MlpSmallParams {
  SrcView src;
  int n_rows;
  const double* pack;
  int F, H, C;
  SmallResult* out;
};

struct MlpSmallRecParams : MlpSmallParams {
  void* rec;  // [n_rows][C] fp32, or [n_rows][2k] words
  int k;
};

template <int OUT, class Params>
__global__ void __launch_bounds__(256) mlp_small_kernel(const Params p) {
  extern __shared__ __align__(16) double rs_smem[];
  constexpr int R = kMlpRsRows;
  constexpr bool kRec = OUT != kSmallLabels;
  MlpRsView view = mlp_rs_stage(rs_smem, p.pack, p.F, p.H, p.C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // per warp: the scorer's strip, then the four rows as fp32 (F x R doubles hold 2 F x R floats: room to spare), then
  // (records) the logits
  double* xs = rs_smem + mlp_rs_weight_doubles(p.F, p.H, p.C) +
               warp * (mlp_rs_strip_doubles(p.F, p.H, R) + 2 * p.F + (kRec ? p.C * R : 0));
  double* hv = xs + p.F * R;
  float* x32 = reinterpret_cast<float*>(hv + p.H * R);
  __syncthreads();
  mlp_rs_finish_stage(view);

  const int i = (blockIdx.x * (blockDim.x >> 5) + warp) * R;
  if (i >= p.n_rows) return;
  // x32[r F + f] = feature f of row r.  Every load is a PCIe round trip to pinned host memory, so a lane issues a
  // batch of them before it stores any (a store in between would serialise them: the source may alias shared memory)
  constexpr int kLoads = 8;
  const int total = R * p.F;
  for (int k0 = lane; k0 < total; k0 += 32 * kLoads) {
    double v[kLoads];
#pragma unroll
    for (int j = 0; j < kLoads; ++j) {
      const int k = min(k0 + 32 * j, total - 1);  // (past the end: a valid element, not stored; no branch per load)
      const int r = k / p.F;
      const int row = i + r < p.n_rows ? i + r : i;  // unused slots repeat the first row (result ignored)
      v[j] = load_src(p.src, row, k - r * p.F);
    }
#pragma unroll
    for (int j = 0; j < kLoads; ++j)
      if (k0 + 32 * j < total) x32[k0 + 32 * j] = static_cast<float>(v[j]);
  }
  const float* xr[R];
#pragma unroll
  for (int r = 0; r < R; ++r) xr[r] = x32 + r * p.F;
  __syncwarp();
  MlpRowResult res[R];
  if constexpr (!kRec) {
    mlp_rs_rows<R>(view, xr, xs, hv, lane, res);
  } else {
    double* zs = xs + mlp_rs_strip_doubles(p.F, p.H, R) + 2 * p.F;  // the pass's logits, [c][R]
    double err[R];
    mlp_rs_rows<R, true, true>(view, xr, xs, hv, lane, res, zs, err);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (i + r >= p.n_rows) continue;  // (unrolled: res[] stays in registers)
      if constexpr (OUT == kSmallProba) {
        mlp_f64_row_outputs(zs + r, R, p.C, lane, static_cast<float*>(p.rec) + static_cast<long long>(i + r) * p.C, 0,
                            nullptr, nullptr, 0.0);
      } else {
        int32_t* at = static_cast<int32_t*>(p.rec) + static_cast<long long>(i + r) * 2 * p.k;
        // top-k rows are ambiguous by the rank rule of mlp_topk_f64_kernel, not by the labels' top-2 margin
        res[r].ambiguous = mlp_f64_row_outputs(zs + r, R, p.C, lane, nullptr, p.k, at, reinterpret_cast<float*>(at + p.k),
                                               err[r]);
      }
    }
  }
  if (lane < R && i + lane < p.n_rows) {
    MlpRowResult mine = res[0];
#pragma unroll
    for (int r = 1; r < R; ++r)
      if (lane == r) mine = res[r];
    p.out[i + lane].label = mine.idx;
    // (probabilities have no ranks to be ambiguous about)
    p.out[i + lane].status = (mine.bad ? 1 : 0) | (mine.ambiguous && OUT != kSmallProba ? 2 : 0);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
size_t mlp_small_smem_bytes(int n_in, int n_hidden, int n_classes, bool records) {
  const size_t per_warp = mlp_rs_strip_doubles(n_in, n_hidden, kMlpRsRows) + 2 * static_cast<size_t>(n_in) +
                          (records ? static_cast<size_t>(n_classes) * kMlpRsRows : 0);
  const size_t smem = (mlp_rs_weight_doubles(n_in, n_hidden, n_classes) + 8 * per_warp) * sizeof(double);
  return smem > static_cast<size_t>(kMaxSmemBytes) ? 0 : smem;
}

template <int OUT, class Params>
static cudaError_t mlp_small_reserve_one(size_t smem) {
  static size_t configured = 0;
  if (smem <= configured) return cudaSuccess;
  cudaError_t err = cudaFuncSetAttribute(mlp_small_kernel<OUT, Params>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
  if (err == cudaSuccess) configured = smem;
  return err;
}

cudaError_t mlp_small_reserve(size_t smem, bool records) {
  if (!records) return mlp_small_reserve_one<kSmallLabels, MlpSmallParams>(smem);
  const cudaError_t err = mlp_small_reserve_one<kSmallProba, MlpSmallRecParams>(smem);
  return err != cudaSuccess ? err : mlp_small_reserve_one<kSmallTopk, MlpSmallRecParams>(smem);
}

cudaError_t launch_mlp_small(const MlpDeviceModel& m, const SrcView& src, int n_rows, SmallResult* out, size_t smem,
                             cudaStream_t stream, int kind, int k, void* rec) {
  if (n_rows <= 0) return cudaSuccess;
  MlpSmallRecParams p{};
  p.src = src;
  p.n_rows = n_rows;
  p.pack = m.rs_pack;
  p.F = m.n_in;
  p.H = m.n_hidden;
  p.C = m.n_classes;
  p.out = out;
  p.rec = rec;
  p.k = k;
  constexpr int rows_per_block = 8 * kMlpRsRows;
  const int grid = (n_rows + rows_per_block - 1) / rows_per_block;
  if (kind == kSmallProba) mlp_small_kernel<kSmallProba><<<grid, 256, smem, stream>>>(p);
  else if (kind == kSmallTopk) mlp_small_kernel<kSmallTopk><<<grid, 256, smem, stream>>>(p);
  else mlp_small_kernel<kSmallLabels><<<grid, 256, smem, stream>>>(static_cast<const MlpSmallParams&>(p));
  return cudaGetLastError();
}

static size_t mlp_fixed_smem(const MlpDeviceModel& m, bool proba = false, bool topk = false) {
  return 1024 + (static_cast<size_t>(m.f_pad) * (m.n_hidden + 4) + (m.n_hidden + 4) + static_cast<size_t>(m.n_hidden) * m.cp + m.cp) * 4 +
         2 * 64 * 8 + (proba ? static_cast<size_t>(kMlpConsumerWarps) * 32 * m.n_classes * 4 : 0) +  // + a staging strip per warp
         (topk ? static_cast<size_t>(kMlpConsumerWarps) * kMlpTopkStripWords * 4 : 0);
}

bool mlp_tma_supported(const MlpDeviceModel& m, std::string* why, bool proba, bool topk) {
  const bool shape_ok = (m.n_hidden == 32 || m.n_hidden == 16) && (m.n_classes == 10 || m.n_classes == 2 || m.n_classes == 3);
  if (!shape_ok) {
    if (why) *why = "tile kernel instantiated for hidden in {16, 32} and classes in {2, 3, 10}";
    return false;
  }
  if (mlp_fixed_smem(m, proba, topk) + kMlpPairs * static_cast<size_t>(kMlpStageBytes) > static_cast<size_t>(kMaxSmemBytes)) {
    if (why) *why = "W1^T does not fit in shared memory next to a 4-stage ring";
    return false;
  }
  return true;
}

template <int H, int C, bool EXACT, bool PROBA = false, bool TOPK = false, class Params = MlpKernelParams>
static cudaError_t mlp_launch_one(const CUtensorMap& xmap, const Params& p, int grid, size_t smem, cudaStream_t stream) {
  auto kern = mlp_argmax_tma_kernel<H, C, EXACT, PROBA, TOPK, Params>;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  kern<<<grid, kMlpThreads, smem, stream>>>(xmap, p);
  return cudaGetLastError();
}

template <bool EXACT, bool PROBA = false, bool TOPK = false, class Params = MlpKernelParams>
static cudaError_t mlp_dispatch(int H, int C, const CUtensorMap& xmap, const Params& p, int grid, size_t smem,
                                cudaStream_t stream) {
#define UML_MLP_CASE(HH, CC) \
  if (H == HH && C == CC) return mlp_launch_one<HH, CC, EXACT, PROBA, TOPK, Params>(xmap, p, grid, smem, stream);
  UML_MLP_CASE(32, 10) UML_MLP_CASE(32, 2) UML_MLP_CASE(32, 3) UML_MLP_CASE(16, 10) UML_MLP_CASE(16, 2) UML_MLP_CASE(16, 3)
#undef UML_MLP_CASE
  return cudaErrorInvalidValue;
}

// the parameters, grid and shared memory of one tile-kernel launch; `fixed` = mlp_fixed_smem of the kernel's form
static MlpKernelParams mlp_tma_params(const MlpDeviceModel& m, int64_t n_rows, int32_t* labels, const FlagList& flags,
                                      float* proba, size_t fixed, int sm_count, int* grid, size_t* smem) {
  MlpKernelParams p{};
  p.w1t = m.w1t;
  p.b1 = m.b1;
  p.w2t = m.w2t;
  p.b2 = m.b2;
  p.labels = labels;
  p.n_rows = n_rows;
  p.num_tiles = (n_rows + kMlpTileRows - 1) / kMlpTileRows;
  p.f_pad = m.f_pad;
  p.kc = m.f_pad / kChunkF;
  int stages = static_cast<int>((static_cast<size_t>(kMaxSmemBytes) - fixed) / kMlpStageBytes);
  stages = std::min(stages, 64);
  if (const char* env = getenv("UML_B200_STAGES")) stages = std::max(kMlpPairs, std::min(stages, atoi(env)));
  p.num_stages = stages;
  // the absolute (underflow) part of the bound is in entry C of b2 (uml_mlp_load)
  const double F = m.n_in;
  p.e1_scale = static_cast<float>((F + 4.0) * kU * (1.0 + F * 4.76837158203125e-07) * 1.0001 * m.w2_abs_row_sum_max);
  p.e2_scale = mlp_e2_scale(m.n_hidden);
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.proba = proba;
  *smem = fixed + static_cast<size_t>(stages) * kMlpStageBytes;
  const long long slots = (p.num_tiles + kMlpPairs - 1) / kMlpPairs;
  *grid = static_cast<int>(std::min<long long>(sm_count, std::max<long long>(1, slots)));
  return p;
}

cudaError_t launch_mlp_tma(const CUtensorMap& xmap, const MlpDeviceModel& m, const float* x, int64_t n_rows,
                           int32_t* labels, bool exact, const FlagList& flags, int sm_count, cudaStream_t stream,
                           float* proba) {
  (void)x;
  if (n_rows <= 0) return cudaSuccess;
  const bool want_proba = proba != nullptr;
  int grid = 0;
  size_t smem = 0;
  const MlpKernelParams p = mlp_tma_params(m, n_rows, labels, flags, proba, mlp_fixed_smem(m, want_proba), sm_count, &grid, &smem);
  if (want_proba) return mlp_dispatch<false, true>(m.n_hidden, m.n_classes, xmap, p, grid, smem, stream);
  return exact ? mlp_dispatch<true>(m.n_hidden, m.n_classes, xmap, p, grid, smem, stream)
               : mlp_dispatch<false>(m.n_hidden, m.n_classes, xmap, p, grid, smem, stream);
}

cudaError_t launch_mlp_tma_topk(const CUtensorMap& xmap, const MlpDeviceModel& m, int64_t n_rows, int k, int32_t* idx,
                                float* proba, bool exact, const FlagList& flags, int sm_count, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  if (k < 1 || k > std::min(m.n_classes, kMlpTopkMax)) return cudaErrorInvalidValue;
  int grid = 0;
  size_t smem = 0;
  MlpTopkKernelParams p{};
  static_cast<MlpKernelParams&>(p) =
      mlp_tma_params(m, n_rows, nullptr, flags, nullptr, mlp_fixed_smem(m, false, true), sm_count, &grid, &smem);
  p.topk_idx = idx;
  p.topk_proba = proba;
  p.topk_k = k;
  return exact ? mlp_dispatch<true, false, true>(m.n_hidden, m.n_classes, xmap, p, grid, smem, stream)
               : mlp_dispatch<false, false, true>(m.n_hidden, m.n_classes, xmap, p, grid, smem, stream);
}

cudaError_t launch_mlp_rescore_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows,
                                   const MlpTcLaunch& out, const FlagList& flags, bool all_rows, int sm_count,
                                   cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  MlpRescoreParams p{};
  p.x = x;
  p.ld = ld;
  p.n_rows = n_rows;
  p.pack = m.rs_pack;
  p.F = m.n_in;
  p.H = m.n_hidden;
  p.C = m.n_classes;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.all_rows = all_rows ? 1 : 0;
  p.targets = out.targets;
  p.counters = flags.counters;
  // shared memory: W1 + padded W2 + biases + the two bound vectors + one strip (x, hidden values) per warp
  const size_t smem = (mlp_rs_weight_doubles(m.n_in, m.n_hidden, m.n_classes) + 8 * mlp_rs_strip_doubles(m.n_in, m.n_hidden, kMlpRsRows)) * sizeof(double);
  if (smem > static_cast<size_t>(kMaxSmemBytes)) return cudaErrorInvalidValue;  // uml_mlp_load bounds F * H
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(mlp_rescore_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mlp_rescore_f64_kernel, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  long long blocks = static_cast<long long>(sm_count) * per_sm;  // persistent: every resident warp loops over rows
  if (all_rows) blocks = std::min<long long>(blocks, (n_rows + 8 * kMlpRsRows - 1) / (8 * kMlpRsRows));
  cudaError_t lerr = launch_dependent(mlp_rescore_f64_kernel, static_cast<int>(std::max<long long>(1, blocks)), 256, smem, stream, p);
  if (lerr != cudaSuccess) return lerr;
  return cudaGetLastError();
}

cudaError_t launch_mlp_proba_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, float* proba,
                                 const FlagList& flags, bool all_rows, int sm_count, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  MlpProbaF64Params p{};
  p.x = x;
  p.ld = ld;
  p.n_rows = n_rows;
  p.pack = m.rs_pack;
  p.F = m.n_in;
  p.H = m.n_hidden;
  p.C = m.n_classes;
  p.proba = proba;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.all_rows = all_rows ? 1 : 0;
  p.counters = flags.counters;
  // the re-score kernel's shared memory plus C x kMlpRsRows logits per warp
  const size_t strip = mlp_rs_strip_doubles(m.n_in, m.n_hidden, kMlpRsRows) + static_cast<size_t>(m.n_classes) * kMlpRsRows;
  const size_t smem = (mlp_rs_weight_doubles(m.n_in, m.n_hidden, m.n_classes) + 8 * strip) * sizeof(double);
  if (smem > static_cast<size_t>(kMaxSmemBytes)) return cudaErrorInvalidValue;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(mlp_proba_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mlp_proba_f64_kernel, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  long long blocks = static_cast<long long>(sm_count) * per_sm;  // persistent: every resident warp loops over rows
  if (all_rows) {
    blocks = std::min<long long>(blocks, (n_rows + 8 * kMlpRsRows - 1) / (8 * kMlpRsRows));
    mlp_proba_f64_kernel<<<static_cast<int>(std::max<long long>(1, blocks)), 256, smem, stream>>>(p);
    return cudaGetLastError();
  }
  cudaError_t lerr = launch_dependent(mlp_proba_f64_kernel, static_cast<int>(std::max<long long>(1, blocks)), 256, smem, stream, p);
  if (lerr != cudaSuccess) return lerr;
  return cudaGetLastError();
}

cudaError_t launch_mlp_topk_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, int k, int32_t* idx,
                                float* proba, const FlagList& flags, bool all_rows, int sm_count, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  MlpTopkF64Params p{};
  p.x = x;
  p.ld = ld;
  p.n_rows = n_rows;
  p.pack = m.rs_pack;
  p.F = m.n_in;
  p.H = m.n_hidden;
  p.C = m.n_classes;
  p.k = k;
  p.idx = idx;
  p.proba = proba;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  p.all_rows = all_rows ? 1 : 0;
  p.counters = flags.counters;
  // the shared memory of mlp_proba_f64_kernel
  const size_t strip = mlp_rs_strip_doubles(m.n_in, m.n_hidden, kMlpRsRows) + static_cast<size_t>(m.n_classes) * kMlpRsRows;
  const size_t smem = (mlp_rs_weight_doubles(m.n_in, m.n_hidden, m.n_classes) + 8 * strip) * sizeof(double);
  if (smem > static_cast<size_t>(kMaxSmemBytes)) return cudaErrorInvalidValue;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(mlp_topk_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mlp_topk_f64_kernel, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  long long blocks = static_cast<long long>(sm_count) * per_sm;  // persistent: every resident warp loops over rows
  if (all_rows) blocks = std::min<long long>(blocks, (n_rows + 8 * kMlpRsRows - 1) / (8 * kMlpRsRows));
  cudaError_t lerr = launch_dependent(mlp_topk_f64_kernel, static_cast<int>(std::max<long long>(1, blocks)), 256, smem, stream, p);
  if (lerr != cudaSuccess) return lerr;
  return cudaGetLastError();
}

}  // namespace uml
