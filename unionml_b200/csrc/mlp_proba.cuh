// Class-probability epilogue of the MLP tile kernels (PytorchModel.forward of the torch quickstart returns
// softmax(logits, dim=1)): the fp32 softmax of one row's logits and the warp's coalesced store of its rows.
// DESIGN.md 3.6 derives the error bound of mlp_softmax_f32.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace uml {

// softmax over the C logits z[0..C-1] of one row, fp32: max, expf(z - max), running sum, one reciprocal.  expf and the
// reciprocal are the accurate library forms (no fast-math), which the bound assumes.
template <int C>
__device__ __forceinline__ void mlp_softmax_f32(const float* z, float* pr) {
  float m = z[0];
#pragma unroll
  for (int c = 1; c < C; ++c) m = fmaxf(m, z[c]);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    pr[c] = expf(z[c] - m);
    s += pr[c];
  }
  const float inv = 1.0f / s;  // s >= 1: the maximum's term is expf(0) = 1
#pragma unroll
  for (int c = 0; c < C; ++c) pr[c] *= inv;
}

// One warp copies RUN consecutive rows of C probabilities, staged contiguously in shared memory at `s` (16-byte
// aligned), to out[row0 * C ...].  A whole run at a 16-byte aligned destination leaves as float4 stores; a run cut by
// the batch end, or a destination that is only 4-byte aligned, as consecutive scalar stores (still one 128-byte line
// per warp instruction).  Nothing past row n_rows - 1 is written.
template <int C, int RUN>
__device__ __forceinline__ void mlp_proba_store_run(const float* s, float* out, long long row0, long long n_rows, int lane) {
  static_assert(RUN * C % 4 == 0, "a whole run is a whole number of float4");
  float* dst = out + row0 * C;
  if (row0 + RUN <= n_rows && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
#pragma unroll
    for (int i = lane; i < RUN * C / 4; i += 32) reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(s)[i];
  } else {
    const long long left = n_rows - row0;
    const int n = left >= RUN ? RUN * C : (left > 0 ? static_cast<int>(left) * C : 0);
    for (int i = lane; i < n; i += 32) dst[i] = s[i];
  }
}

}  // namespace uml
