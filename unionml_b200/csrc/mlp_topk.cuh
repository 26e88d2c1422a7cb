// Top-k epilogue of the MLP tile kernels (the quickdraw template's predictor: softmax(module(x)) then
// torch.topk(probabilities, 3)): the k largest logits of one row in registers, the rank guard of EXACT mode, and the
// warp's coalesced store of its rows' k indices / probabilities.  DESIGN.md 3.8.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace uml {

// largest k the tile kernels select in registers; larger k is served by the float64 kernel (mlp_topk_f64_kernel)
constexpr int kMlpTopkMax = 5;

// The M largest of the C logits z[0..C-1], in descending order with ties to the lower class index (np.argmax's rule
// for rank 1, a stable descending sort below it), each carried with its class index and pr[c].  Insertion into a
// sorted list: the classes arrive in index order and an equal logit never passes an earlier one.  Slots not filled
// yet hold index C, which any class passes.  M = min(C, kMlpTopkMax + 1): one rank beyond k for the guard.
template <int C, int M>
__device__ __forceinline__ void mlp_topk_select(const float* z, const float* pr, float (&v)[M], int (&id)[M],
                                                float (&pv)[M]) {
#pragma unroll
  for (int j = 0; j < M; ++j) {
    v[j] = -INFINITY;
    id[j] = C;
    pv[j] = 0.f;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    float x = z[c], xp = pr[c];
    int xi = c;
    bool ins = false;
#pragma unroll
    for (int j = 0; j < M; ++j) {
      ins = ins || id[j] >= C || x > v[j];  // once in, every later slot shifts down by one
      if (ins) {
        const float tv = v[j], tp = pv[j];
        const int ti = id[j];
        v[j] = x;
        pv[j] = xp;
        id[j] = xi;
        x = tv;
        xp = tp;
        xi = ti;
      }
    }
  }
}

// EXACT mode: the order of the top k and the boundary between rank k and rank k + 1 are those of the exact logits
// when every consecutive gap ẑ_(r) − ẑ_(r+1), r < kk = min(k, C − 1), exceeds err2 = 2δ.  kk = 1 is the label guard.
// NaN fails the comparison, so such a row is flagged.
template <int M>
__device__ __forceinline__ bool mlp_topk_certain(const float (&v)[M], int kk, float err2) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j + 1 < M; ++j)
    if (j < kk) ok = ok && (v[j] - v[j + 1]) > err2;
  return ok;
}

// One warp copies RUN consecutive rows of k 4-byte values, staged contiguously in shared memory at `s` (16-byte
// aligned), to out[row0 * k ...]: float4-sized stores for a whole run at a 16-byte aligned destination (RUN * k is a
// multiple of 4 for RUN in {16, 32}), consecutive scalar stores otherwise.  Nothing past row n_rows - 1 is written.
template <int RUN, class T>
__device__ __forceinline__ void mlp_topk_store_run(const T* s, T* out, long long row0, long long n_rows, int k, int lane) {
  static_assert(sizeof(T) == 4 && RUN % 4 == 0, "4-byte values, runs of whole 16-byte groups");
  T* dst = out + row0 * k;
  if (row0 + RUN <= n_rows && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
    for (int i = lane; i < RUN * k / 4; i += 32) reinterpret_cast<int4*>(dst)[i] = reinterpret_cast<const int4*>(s)[i];
  } else {
    const long long left = n_rows - row0;
    const int n = left >= RUN ? RUN * k : (left > 0 ? static_cast<int>(left) * k : 0);
    for (int i = lane; i < n; i += 32) dst[i] = s[i];
  }
}

// a warp's staging strip: 32 rows x kMlpTopkMax indices, then as many probabilities (4-byte words)
constexpr int kMlpTopkStripWords = 2 * 32 * kMlpTopkMax;

// flag_rows_warp (label_store.cuh) with the flag list's fields read before the ballot, for the top-k form of
// mlp_argmax_tma_kernel: read after it, as flag_rows_warp does, ptxas gives that form different code (H = 16, C = 10:
// 134 registers instead of 128)
__device__ __forceinline__ void mlp_topk_flag(bool flagged, long long row, int* flag_count, int32_t* flag_rows, int flag_cap,
                                              int lane) {
  const unsigned mask = __ballot_sync(0xffffffffu, flagged);
  if (mask != 0u) {
    int base = 0;
    if (lane == 0) base = atomicAdd(flag_count, __popc(mask));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (flagged) {
      const int pos = base + __popc(mask & ((1u << lane) - 1u));
      if (pos < flag_cap) flag_rows[pos] = static_cast<int32_t>(row);
    }
  }
}

}  // namespace uml
