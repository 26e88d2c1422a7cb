// Tensor-core scoring kernel for the 2-layer MLP predictor (cfg 5): layer 1 on Hopper wgmma (tf32), fp32 accumulators
// in the registers of the consuming warpgroup.
//
// Replaces PytorchModel.forward + .argmax(1) of UnionML's torch quickstart
// (tests/integration/pytorch_app/quickstart.py:14-24, 68-70; hyperparameters 64 -> 32 -> 10 at :80).
//
// Why tensor cores here and not in the linear kernel: layer 1 is a real [rows x F] . [F x H] contraction (4 096 of the
// 4 736 flop per row); on CUDA cores it is the bulk of the kernel's FMA issue.
//
// Exactness with 10-bit tf32 mantissas.  The MMA multiplies tf32 x tf32 exactly and accumulates in fp32, so the only
// approximation is what the operands lose when they become tf32:
//   * X: this kernel is dispatched for batches whose features ARE tf32 values (low 13 mantissa bits zero - integer /
//     pixel domains such as the reference's digits and MNIST frames; the staging pass records it).  Every row is
//     re-checked here (scan warps OR the low bits): a row that is not tf32-exact gets A1 = +inf and is therefore
//     flagged for the fp64 re-score, so the answer is right for any input - only slower.  The PROBA form, and the
//     TOPK form in FAST mode, flag such rows too when the launch has a flag list (the chunk pipeline, whose kernel
//     choice is a guess from the first rows), and the float64 kernels behind them overwrite those rows.
//   * W1: split on the host as w = hi + lo + r with hi, lo tf32 (round to nearest) and |r| <= 2^-22 |w|; B holds
//     [hi | lo] as 2H columns, so ONE MMA per K step yields main = x.hi and small = x.lo in separate accumulator
//     columns (the small terms never lose bits against the large accumulator), summed in fp32 in the epilogue.
// EXACT mode bounds the error per row, |h_n - h_n_true| <= E1 = (32 n_mma + 12) 2^-24 A1 with
// A1 = max|b1| + sum_f |x_f| max_n |w1_nf| (n_mma = F_pad / 8 accumulating MMA steps; the per-step term covers a
// truncating 9-addend aligner with no guard bits, DESIGN.md 3.3), propagates it through layer 2 exactly like the
// CUDA-core kernel, and re-scores rows whose logit margin is inside the bound in fp64 (mlp_rescore_f64_kernel).
//
// Roles (13 warps, one CTA per SM, persistent over 128-row tiles):
//   warp 12  : TMA producer - 128 x 32 fp32 boxes of X (16 KiB, SWIZZLE_128B) into an S-stage ring
//   warps 0-3: scan         - thread per row: A1 bound + tf32-exactness of the row from the same box (LDS.128)
//   warps 4-7, 8-11: two consumer warpgroups taking alternate tiles, so one runs its epilogue while the other's MMAs
//             are in flight.  Per box 2 x 4 wgmma m64nNk8 (N = 2H; rows 0-63 and 64-127 of the box as A, K-major SW128,
//             the resident W1 tile as B), then from the accumulator registers: + b1, ReLU, layer 2 over the lane's
//             hidden units, a quad reduce-scatter that leaves each lane one row's logits, argmax (first maximum
//             wins), margin guard, label store (+ peer stores); PROBA kernels instead take the softmax of the logits
//             and store each warp's two 16-row runs of probabilities through shared memory (mlp_proba.cuh); TOPK
//             kernels select the k largest logits and store indices / probabilities the same way (mlp_topk.cuh)
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "uml_common.cuh"
#include "label_store.cuh"
#include "wgmma.cuh"
#include "mlp_proba.cuh"
#include "mlp_topk.cuh"

namespace uml {

constexpr int kTcThreads = 416;
constexpr int kTcProducerWarp = 12;
// __launch_bounds__ thread count: the register budget of 544 threads, not the 416 the kernel launches with.  Every
// measurement of this kernel was taken with it; with a bound of 416, ptxas (CUDA 12.9) gives H=32 C=10 EXACT 128
// registers instead of 95 and H=16 C=10 EXACT 92 instead of 80, and changes their code.  Raising the budget is a
// performance change to be measured on its own.
constexpr int kTcRegBudgetThreads = 544;
constexpr int kTcEpilogueWarps = 8;
constexpr int kTcSlots = 24;       // A1 hand-off slots (scan -> epilogue); > the scan warps' maximum lead over the epilogue
constexpr int kTcMaxFpad = 128;    // features (padded to 32) the resident W1 tile is sized for

template <int H, int C>
struct MlpTcParams {
  static constexpr int CP = (C + 1 + 3) / 4 * 4;
  float w2[H][CP];          // [n][c], column C = max_c |w2_cn| (EXACT bound), rest zero
  float b1[H];
  float b2[CP];             // entry C = max_c |b2_c|
  float w1max[kTcMaxFpad];  // max_n |w1_nf| per feature (zero padded)
  float b1max;
  float e1_scale, e2_scale;
  const float* w1_tiles;    // [KC][2H rows][32 floats], rows 128-byte swizzled exactly as the wgmma descriptor reads them
  LabelTargets targets;
  long long n_rows;
  long long num_tiles;
  int kc;
  int num_stages;
  int* flag_count;
  int32_t* flag_rows;
  int flag_cap;
  float* proba;  // PROBA kernels: [n_rows][C] row-major
  // TOPK kernels: [n_rows][topk_k] class indices and (optional, nullptr: not written) their probabilities
  int32_t* topk_idx;
  float* topk_proba;
  int topk_k;
};

// consumer lane l of warp wq (in its warpgroup) ends the epilogue owning one row of the 128-row tile: the quad
// (l / 4) holds rows 16 wq + l / 4 (+ 8) of both 64-row halves, and lane l % 4 keeps the (half, +8) pair it names
__device__ __forceinline__ int tc_row_of_lane(int wq, int l) { return 64 * ((l & 3) >> 1) + 16 * wq + (l >> 2) + 8 * (l & 1); }

// FLAG_TF32 (PROBA, and TOPK in FAST mode): rows that are not tf32 values go onto the flag list (a template argument,
// not a runtime test of the list: the forms without it keep their code and their measured time)
template <int H, int C, bool EXACT, bool PROBA, bool TOPK = false, bool FLAG_TF32 = false>
__global__ void __launch_bounds__(kTcRegBudgetThreads, 1)
mlp_argmax_tc_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ MlpTcParams<H, C> p) {
  constexpr int N = 2 * H;     // accumulator columns per row: [main | small]
  constexpr int NACC = N / 2;  // fp32 accumulator registers per thread and 64-row half
  static_assert(N == 32 || N == 64, "wgmma kind tf32 is instantiated for N in {32, 64}");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int S = p.num_stages;
  const int KC = p.kc;
  uint8_t* ring = smem;                                                  // S x 16 KiB
  uint8_t* btile = ring + static_cast<size_t>(S) * kStageBytes;          // KC x (N x 128 B), 1 KiB aligned
  float* a1_s = reinterpret_cast<float*>(btile + static_cast<size_t>(KC) * N * 128);  // [kTcSlots][128]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(a1_s + kTcSlots * kTileRows);
  uint64_t* empty_bar = full_bar + S;
  uint64_t* a1_bar = empty_bar + S;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // W1 tile (already in the swizzled layout) -> shared memory, once per CTA
  {
    const float4* src = reinterpret_cast<const float4*>(p.w1_tiles);
    float4* dst = reinterpret_cast<float4*>(btile);
    const int n4 = KC * N * 32 / 4;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = __ldg(src + i);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1 + 4);  // the consuming warpgroup + the four scan warps
    }
    for (int s = 0; s < kTcSlots; ++s) mbar_init(&a1_bar[s], kTileRows);  // every scan thread arrives for its own row
    fence_barrier_init();
  }
  fence_proxy_async_smem();  // the W1 tile was written with st.shared; wgmma reads it through the async proxy
  __syncthreads();

  pdl_launch_dependents();  // the fp64 re-score behind this launch may stage its weights while this grid runs
  const long long G = gridDim.x;
  const long long num_tiles = p.num_tiles;

  if (warp == kTcProducerWarp) {
    // ===================== TMA producer =====================
    if (elect_one_sync()) {
      tma_prefetch_desc(&xmap);
      const uint64_t policy = make_evict_first_policy();
      int stage = 0;
      uint32_t phase = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += G) {
        for (int k = 0; k < KC; ++k) {
          mbar_wait_relaxed(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(ring + static_cast<size_t>(stage) * kStageBytes, &xmap, &full_bar[stage], k * kChunkF,
                      static_cast<int>(tile * kTileRows), policy);
          if (++stage == S) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else if (warp < 4) {
    // ===================== scan warps: thread per row, A1 bound + tf32 exactness =====================
    const int row = threadIdx.x;  // 0..127
    const uint32_t rowbase = static_cast<uint32_t>(row) * 128u;
    const uint32_t sw = static_cast<uint32_t>(row & 7) * 16u;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t it = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += G, ++it) {
      float a1 = 0.f;
      uint32_t lowbits = 0u;
      for (int k = 0; k < KC; ++k) {
        mbar_wait_relaxed(&full_bar[stage], phase);
        const uint8_t* xs = ring + static_cast<size_t>(stage) * kStageBytes;
#pragma unroll
        for (int q = 0; q < kChunkF / 4; ++q) {
          const float4 v = *reinterpret_cast<const float4*>(xs + rowbase + ((static_cast<uint32_t>(q) * 16u) ^ sw));
          if (EXACT) {
            const float* wm = p.w1max + k * kChunkF + q * 4;
            a1 = fmaf(fabsf(v.x), wm[0], a1);
            a1 = fmaf(fabsf(v.y), wm[1], a1);
            a1 = fmaf(fabsf(v.z), wm[2], a1);
            a1 = fmaf(fabsf(v.w), wm[3], a1);
          }
          lowbits |= __float_as_uint(v.x) | __float_as_uint(v.y) | __float_as_uint(v.z) | __float_as_uint(v.w);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == S) {
          stage = 0;
          phase ^= 1u;
        }
      }
      // a row whose features are not tf32 values was scored from truncated inputs: A1 = +inf sends it to the fp64 re-score
      const uint32_t slot = it % kTcSlots;
      a1_s[slot * kTileRows + row] = (lowbits & 0x1fffu) ? INFINITY : (a1 + p.b1max);
      mbar_arrive(&a1_bar[slot]);  // release: this thread's A1 is visible to whoever completes the wait
    }
  } else if (warp < 4 + kTcEpilogueWarps) {
    // ===================== consumer warpgroups: warps 4-7 even tiles, warps 8-11 odd tiles =====================
    // layer 1 as two m64 wgmma chains (rows 0-63, 64-127 of the tile) per K step, then the epilogue from the registers
    const int wq = warp & 3;
    const int set = (warp - 4) >> 2;
    const int q = lane & 3;
    const int row_in_tile = tc_row_of_lane(wq, lane);
    uint32_t it = static_cast<uint32_t>(set);
    for (long long tile = blockIdx.x + set * G; tile < num_tiles; tile += 2 * G, it += 2) {
      // the ring carries this CTA's tiles in order, KC chunks each: chunk k of local tile `it` is number it * KC + k
      const uint32_t first_chunk = it * static_cast<uint32_t>(KC);
      float acc[2][NACC];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < NACC; ++r) {
          acc[h][r] = 0.f;
          wgmma_fence_operand(acc[h][r]);
        }
      wgmma_fence();
      for (int k = 0; k < KC; ++k) {
        const uint32_t chunk = first_chunk + static_cast<uint32_t>(k);
        const uint32_t stage = chunk % static_cast<uint32_t>(S);
        mbar_wait_bounded(&full_bar[stage], (chunk / static_cast<uint32_t>(S)) & 1u);
        const uint32_t a_base = smem_u32(ring + static_cast<size_t>(stage) * kStageBytes);
        const uint32_t b_base = smem_u32(btile + static_cast<size_t>(k) * N * 128);
#pragma unroll
        for (int j = 0; j < kChunkF / 8; ++j) {  // K = 8 tf32 (32 bytes) per MMA
          const uint32_t scale_d = (k | j) != 0 ? 1u : 0u;
          const uint64_t b_desc = wgmma_desc_k_sw128(b_base + j * 32);
          WgmmaTf32<N>::mma(acc[0], wgmma_desc_k_sw128(a_base + j * 32), b_desc, scale_d);
          WgmmaTf32<N>::mma(acc[1], wgmma_desc_k_sw128(a_base + 64 * 128 + j * 32), b_desc, scale_d);
        }
      }
      wgmma_commit();
      const uint32_t slot = it % kTcSlots;
      mbar_wait_bounded(&a1_bar[slot], (it / kTcSlots) & 1u);
      // read before the ring stages are released: the scan warps cannot reach this slot's next tile until they are
      const float a1 = a1_s[slot * kTileRows + row_in_tile];
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < NACC; ++r) wgmma_fence_operand(acc[h][r]);
      if (wq == 0 && lane == 0)
        for (int k = 0; k < KC; ++k) mbar_arrive(&empty_bar[(first_chunk + static_cast<uint32_t>(k)) % static_cast<uint32_t>(S)]);

      // ---- + b1, ReLU, layer 2 over this lane's hidden units for the quad's four rows ----
      // row j of the quad: half j >> 1, + 8 for odd j; this lane's hidden units n = 8 i + 2 q + e (i < H / 8, e < 2):
      // main term acc[j >> 1][4 i + 2 (j & 1) + e], small term the same entry of column group i + H / 8
      constexpr int NZ = C + (EXACT ? 1 : 0);
      float part[4][NZ];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int c = 0; c < NZ; ++c) part[j][c] = 0.f;
#pragma unroll
        for (int i = 0; i < H / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 8 * i + 2 * q + e;
            const int at = 4 * i + 2 * (j & 1) + e;
            const float hv = fmaxf((acc[j >> 1][at + 4 * (H / 8)] + acc[j >> 1][at]) + p.b1[n], 0.f);
#pragma unroll
            for (int c = 0; c < NZ; ++c) part[j][c] = fmaf(hv, p.w2[n][c], part[j][c]);
          }
      }
      // quad reduce-scatter: lane q ends with the complete logits of row j = q (xor 2 splits the rows by half, xor 1
      // by the + 8 pair)
      const bool hi2 = (q & 2) != 0, hi1 = (q & 1) != 0;
      float z[NZ];
#pragma unroll
      for (int c = 0; c < NZ; ++c) {
        float s[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float keep = hi2 ? part[2 + r][c] : part[r][c];
          const float send = hi2 ? part[r][c] : part[2 + r][c];
          s[r] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        const float keep = hi1 ? s[1] : s[0];
        const float send = hi1 ? s[0] : s[1];
        z[c] = (keep + __shfl_xor_sync(0xffffffffu, send, 1)) + p.b2[c];
      }
      if constexpr (PROBA) {
        // this warp's staging strip (32 rows x C floats behind the A1 hand-off barriers): row r of run h at
        // (16 h + r) C, so each run is 64 C contiguous bytes, as it is in the output
        float* strip = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(a1_bar + kTcSlots) + 15u) & ~static_cast<uintptr_t>(15)) +
                       (warp - 4) * 32 * C;
        float pr[C];
        mlp_softmax_f32<C>(z, pr);
        float* mine = strip + (16 * ((lane & 3) >> 1) + (lane >> 2) + 8 * (lane & 1)) * C;
#pragma unroll
        for (int c = 0; c < C; ++c) mine[c] = pr[c];
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h)
          mlp_proba_store_run<C, 16>(strip + 16 * h * C, p.proba, tile * kTileRows + 64 * h + 16 * wq, p.n_rows, lane);
        __syncwarp();  // the strip is rewritten by this warp's next tile
        // given a flag list: a row that is not a tf32 value (A1 = +inf) was scored from truncated features, and the
        // float64 probabilities behind this launch replace its values
        if constexpr (FLAG_TF32) {
          const long long row = tile * kTileRows + row_in_tile;
          flag_rows_warp(row < p.n_rows && isinf(a1), row, p, lane);
        }
        continue;
      }
      if constexpr (TOPK) {
        // this warp's staging strip, laid out as the PROBA strip with k words per row: indices, then probabilities
        constexpr int M = C < kMlpTopkMax + 1 ? C : kMlpTopkMax + 1;
        const int k = p.topk_k;
        const bool want_p = p.topk_proba != nullptr;
        float pr[C];
        if (want_p) {
          mlp_softmax_f32<C>(z, pr);
        } else {
#pragma unroll
          for (int c = 0; c < C; ++c) pr[c] = 0.f;
        }
        float v[M], pv[M];
        int id[M];
        mlp_topk_select<C, M>(z, pr, v, id, pv);
        int32_t* si = reinterpret_cast<int32_t*>((reinterpret_cast<uintptr_t>(a1_bar + kTcSlots) + 15u) & ~static_cast<uintptr_t>(15)) +
                      (warp - 4) * kMlpTopkStripWords;
        float* sp = reinterpret_cast<float*>(si + 32 * kMlpTopkMax);
        const int mine = (16 * ((lane & 3) >> 1) + (lane >> 2) + 8 * (lane & 1)) * k;
#pragma unroll
        for (int r = 0; r < M; ++r) {
          if (r < k) {
            si[mine + r] = id[r];
            sp[mine + r] = pv[r];
          }
        }
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row0 = tile * kTileRows + 64 * h + 16 * wq;
          mlp_topk_store_run<16>(si + 16 * h * k, p.topk_idx, row0, p.n_rows, k, lane);
          if (want_p) mlp_topk_store_run<16>(sp + 16 * h * k, p.topk_proba, row0, p.n_rows, k, lane);
        }
        __syncwarp();  // the strip is rewritten by this warp's next tile
        if (EXACT) {
          const long long row = tile * kTileRows + row_in_tile;
          const float err = p.e1_scale * a1 + p.e2_scale * z[C];
          const bool certain = mlp_topk_certain<M>(v, min(k, C - 1), 2.0f * err);
          flag_rows_warp(row < p.n_rows && !certain, row, p, lane);
        }
        if constexpr (!EXACT && FLAG_TF32) {  // only the rows that are not tf32 values (EXACT flags them through err = inf)
          const long long row = tile * kTileRows + row_in_tile;
          flag_rows_warp(row < p.n_rows && isinf(a1), row, p, lane);
        }
        continue;
      }
      const long long row = tile * kTileRows + row_in_tile;
      float best = z[0];
      float second = -INFINITY;
      int idx = 0;
#pragma unroll
      for (int c = 1; c < C; ++c) {
        if (z[c] > best) {
          second = best;
          best = z[c];
          idx = c;
        } else {
          second = fmaxf(second, z[c]);
        }
      }
      const bool in_range = row < p.n_rows;
      if (in_range) store_label_i32(p.targets, row, idx);
      if (p.targets.wire_u8 && p.targets.n_peers > 0) {
        // byte labels: the warp's rows are two runs of 16 (rows 16 wq + 0..15 of each half); lanes 0..7 gather 4
        // consecutive rows each -> the warp's 32 labels leave as eight 4-byte words
        const int run = (lane >> 2) & 1;
        const int r0 = 4 * (lane & 3);
        uint32_t word = 0;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int r = (r0 + t) & 15;
          const int src = 4 * (r & 7) + 2 * run + (r >> 3);  // the lane that owns row r of the run
          word |= (static_cast<uint32_t>(__shfl_sync(0xffffffffu, idx, src)) & 0xffu) << (8 * t);
        }
        store_label_word_u8(p, tile * kTileRows + 64 * run + 16 * wq + r0, word, lane < 8);
      }
      if (EXACT) {
        // |z_c - true| <= E1 * max_c sum_n |w2_cn| + (H+4) u A2   (ReLU is 1-Lipschitz); NaN/Inf -> comparison false
        const float err = p.e1_scale * a1 + p.e2_scale * z[C];
        const bool certain = (best - second) > 2.0f * err;
        flag_rows_warp(in_range && !certain, row, p, lane);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static float tf32_round(float v) {  // round to nearest tf32 (10 mantissa bits), ties away from zero
  uint32_t b;
  memcpy(&b, &v, 4);
  if ((b & 0x7f800000u) == 0x7f800000u) return v;  // Inf / NaN
  b = (b + 0x1000u) & 0xffffe000u;
  float r;
  memcpy(&r, &b, 4);
  return r;
}

// B operand of layer 1: per 32-feature chunk, 2H rows ([hi rows | lo rows]) of 32 floats, each row's 16-byte chunks
// XOR-swizzled by (row & 7) - the SWIZZLE_128B K-major layout the wgmma descriptor (and TMA) use
std::vector<float> mlp_tc_build_w1_tiles(const float* w1 /*[H][F]*/, int H, int F, int f_pad) {
  const int KC = f_pad / kChunkF, N = 2 * H;
  std::vector<float> tiles(static_cast<size_t>(KC) * N * 32, 0.f);
  for (int kc = 0; kc < KC; ++kc)
    for (int n = 0; n < N; ++n)
      for (int j = 0; j < 32; ++j) {
        const int f = kc * 32 + j;
        float v = 0.f;
        if (f < F) {
          const float w = w1[static_cast<size_t>(n % H) * F + f];
          const float hi = tf32_round(w);
          v = n < H ? hi : tf32_round(w - hi);  // w - hi is exact in fp32
        }
        const size_t off = (static_cast<size_t>(kc) * N + n) * 32 + static_cast<size_t>(((j / 4) ^ (n & 7)) * 4 + (j % 4));
        tiles[off] = v;
      }
  return tiles;
}

static size_t mlp_tc_fixed_smem(const MlpDeviceModel& m, bool proba = false, bool topk = false) {
  const size_t kc = m.f_pad / kChunkF;
  size_t bytes = 1024 + kc * (2 * m.n_hidden) * 128 + static_cast<size_t>(kTcSlots) * kTileRows * 4 +
                 (2 * 64 + kTcSlots) * 8 + 16;
  if (proba) bytes += 16 + static_cast<size_t>(kTcEpilogueWarps) * 32 * m.n_classes * 4;  // one staging strip per epilogue warp
  if (topk) bytes += 16 + static_cast<size_t>(kTcEpilogueWarps) * kMlpTopkStripWords * 4;
  return bytes;
}

bool mlp_tc_supported(const MlpDeviceModel& m, std::string* why, bool topk) {
  const bool shape_ok = (m.n_hidden == 32 || m.n_hidden == 16) && (m.n_classes == 10 || m.n_classes == 2 || m.n_classes == 3);
  if (!shape_ok) {
    if (why) *why = "tensor-core kernel instantiated for hidden in {16, 32} and classes in {2, 3, 10}";
    return false;
  }
  if (m.f_pad > kTcMaxFpad || m.w1_tiles == nullptr) {
    if (why) *why = "more than 128 features: the resident W1 tile is sized for F_pad <= 128";
    return false;
  }
  return mlp_tc_fixed_smem(m, false, topk) + 6 * static_cast<size_t>(kStageBytes) <= static_cast<size_t>(kMaxSmemBytes);
}

template <int H, int C, bool EXACT, bool PROBA = false, bool TOPK = false, bool FLAG_TF32 = false>
static cudaError_t mlp_tc_launch_one(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l,
                                     const FlagList& flags, int sm_count, cudaStream_t stream) {
  using Params = MlpTcParams<H, C>;
  static_assert(sizeof(Params) < 4000, "kernel parameters must stay below the 4 KiB limit");
  Params p;
  memset(&p, 0, sizeof(p));
  const MlpHostModel& hm = *m.host;
  for (int n = 0; n < H; ++n) {
    p.b1[n] = hm.b1[n];
    for (int c = 0; c < C; ++c) p.w2[n][c] = hm.w2[static_cast<size_t>(c) * H + n];
    float wmax = 0.f;
    for (int c = 0; c < C; ++c) wmax = fmaxf(wmax, fabsf(hm.w2[static_cast<size_t>(c) * H + n]));
    p.w2[n][C] = wmax;
  }
  float b2max = 0.f, b1max = 0.f;
  for (int c = 0; c < C; ++c) {
    p.b2[c] = hm.b2[c];
    b2max = fmaxf(b2max, fabsf(hm.b2[c]));
  }
  for (int n = 0; n < H; ++n) b1max = fmaxf(b1max, fabsf(hm.b1[n]));
  p.b1max = b1max;
  // Below FLT_MIN (DESIGN.md 3.3): the hi / lo split leaves |r| <= 2^-22 |w| only while w - hi is normal; for
  // |w| < 2^-115 the remainder, or a lo / hi operand the tensor cores flush, is up to FLT_MIN = 4 u 2^-104.  Flooring
  // w1max_f at 2^-104 puts that inside the split term of e1.
  double w1max_sum = 0.0;
  for (int f = 0; f < m.n_in; ++f) {
    float wmax = 0.f;
    for (int n = 0; n < H; ++n) wmax = fmaxf(wmax, fabsf(hm.w1[static_cast<size_t>(n) * m.n_in + f]));
    p.w1max[f] = fmaxf(wmax, 0x1p-104f);
    w1max_sum += p.w1max[f];
  }
  const double F = m.n_in, n_mma = m.f_pad / 8.0;
  // layer-1 error as it reaches a logit: per accumulating MMA step <= 32 u (running |.| sum) - a truncating 9-addend
  // aligner without guard bits gives (9 * 2 + 2) u = 20 u -, + 4 u for the W1 split remainder, + 8 u for the small
  // accumulator and the two fp32 adds of the epilogue; A1 itself is an fp32 sum of F terms (factor 1 + F 2^-21)
  p.e1_scale = static_cast<float>((32.0 * n_mma + 12.0) * kU * (1.0 + F * 4.76837158203125e-07) * 1.0001 * m.w2_abs_row_sum_max);
  p.e2_scale = mlp_e2_scale(H);
  // absolute error of a hidden unit if the tensor cores flush what falls below FLT_MIN: per step and accumulator
  // (main, small) 8 products and the sum, a subnormal feature |x_f| w1max_f, and 3 for the bias and epilogue adds
  p.b2[C] = mlp_a2_bias_entry(b2max, (18.0 * n_mma + 3.0 + w1max_sum) * kFltMin, m.w2_abs_row_sum_max, H);
  p.w1_tiles = m.w1_tiles;
  p.targets = l.targets;
  p.n_rows = l.n_rows;
  p.num_tiles = (l.n_rows + kTileRows - 1) / kTileRows;
  p.kc = m.f_pad / kChunkF;
  p.proba = l.proba;
  p.topk_idx = l.topk_idx;
  p.topk_proba = l.topk_proba;
  p.topk_k = l.topk_k;
  const size_t fixed = mlp_tc_fixed_smem(m, PROBA, TOPK);
  int stages = static_cast<int>((static_cast<size_t>(kMaxSmemBytes) - fixed) / kStageBytes);
  stages = std::min(stages, 64);
  if (const char* env = getenv("UML_B200_STAGES")) stages = std::max(4, std::min(stages, atoi(env)));
  // the A1 hand-off has kTcSlots slots: a consumer reads its tile's A1 before it frees the tile's ring stages, so the
  // scan warps lead it by at most S / KC tiles
  stages = std::min(stages, (kTcSlots - 2) * p.kc);
  p.num_stages = stages;
  p.flag_count = flags.count;
  p.flag_rows = flags.rows;
  p.flag_cap = flags.capacity;
  const size_t smem = fixed + static_cast<size_t>(stages) * kStageBytes;
  auto kern = mlp_argmax_tc_kernel<H, C, EXACT, PROBA, TOPK, FLAG_TF32>;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  const int grid = static_cast<int>(std::min<long long>(sm_count, std::max<long long>(1, p.num_tiles)));
  kern<<<grid, kTcThreads, smem, stream>>>(xmap, p);
  return cudaGetLastError();
}

cudaError_t launch_mlp_tc(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l, bool exact,
                          const FlagList& flags, int sm_count, cudaStream_t stream) {
  if (l.n_rows <= 0) return cudaSuccess;
#define UML_TC_CASE(HH, CC)                                                                                  \
  if (m.n_hidden == HH && m.n_classes == CC)                                                                 \
    return exact ? mlp_tc_launch_one<HH, CC, true>(xmap, m, l, flags, sm_count, stream)                      \
                 : mlp_tc_launch_one<HH, CC, false>(xmap, m, l, flags, sm_count, stream);
  UML_TC_CASE(32, 10) UML_TC_CASE(32, 2) UML_TC_CASE(32, 3) UML_TC_CASE(16, 10) UML_TC_CASE(16, 2) UML_TC_CASE(16, 3)
#undef UML_TC_CASE
  return cudaErrorInvalidValue;
}

cudaError_t launch_mlp_tc_proba(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l,
                                const FlagList& flags, int sm_count, cudaStream_t stream) {
  if (l.n_rows <= 0) return cudaSuccess;
#define UML_TC_CASE(HH, CC)                                                                                  \
  if (m.n_hidden == HH && m.n_classes == CC)                                                                 \
    return flags.count ? mlp_tc_launch_one<HH, CC, false, true, false, true>(xmap, m, l, flags, sm_count, stream) \
                       : mlp_tc_launch_one<HH, CC, false, true>(xmap, m, l, flags, sm_count, stream);
  UML_TC_CASE(32, 10) UML_TC_CASE(32, 2) UML_TC_CASE(32, 3) UML_TC_CASE(16, 10) UML_TC_CASE(16, 2) UML_TC_CASE(16, 3)
#undef UML_TC_CASE
  return cudaErrorInvalidValue;
}

cudaError_t launch_mlp_tc_topk(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l, bool exact,
                               const FlagList& flags, int sm_count, cudaStream_t stream) {
  if (l.n_rows <= 0) return cudaSuccess;
  if (l.topk_k < 1 || l.topk_k > std::min(m.n_classes, kMlpTopkMax)) return cudaErrorInvalidValue;
#define UML_TC_CASE(HH, CC)                                                                                  \
  if (m.n_hidden == HH && m.n_classes == CC)                                                                 \
    return exact         ? mlp_tc_launch_one<HH, CC, true, false, true>(xmap, m, l, flags, sm_count, stream)        \
           : flags.count ? mlp_tc_launch_one<HH, CC, false, false, true, true>(xmap, m, l, flags, sm_count, stream) \
                         : mlp_tc_launch_one<HH, CC, false, false, true>(xmap, m, l, flags, sm_count, stream);
  UML_TC_CASE(32, 10) UML_TC_CASE(32, 2) UML_TC_CASE(32, 3) UML_TC_CASE(16, 10) UML_TC_CASE(16, 2) UML_TC_CASE(16, 3)
#undef UML_TC_CASE
  return cudaErrorInvalidValue;
}

}  // namespace uml
