// Warp-level helpers of the float64 re-score kernels: they are latency-bound (a handful of rows per warp), so the
// reductions are arranged to need few dependent shuffle rounds.
#pragma once

#include <cuda_runtime.h>
#include <math.h>

namespace uml {

// c ? a : b as one selp on values already in registers (the compiler cannot turn it into a select of addresses)
__device__ __forceinline__ double select_reg(bool c, double a, double b) {
  double r;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\tselp.f64 %0, %1, %2, p;\n\t}" : "=d"(r) : "d"(a), "d"(b), "r"((unsigned)c));
  return r;
}

// one butterfly step of warp_reduce16<true>: lanes with bit 2 M set keep the upper M of their 2 M values
template <int M>
__device__ __forceinline__ void reduce16_step(double (&v)[16], int lane) {
  const bool upper = (lane & (2 * M)) != 0;
#pragma unroll
  for (int i = 0; i < M; ++i) {
    const double send = select_reg(upper, v[i], v[i + M]);
    const double keep = select_reg(upper, v[i + M], v[i]);
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2 * M);
  }
}

// Sum 16 per-lane values across the warp with 16 shuffles instead of 16 x 5: every butterfly step halves the number
// of values a lane is still responsible for (lanes with the offset bit set keep the upper half).  On return lane l
// holds the complete sum of value (l >> 1); the two lanes of a pair hold the same one.  REGS: the same additions of the
// same values, with every step's trip count a constant and the lane-dependent choice of the half made on values
// (select_reg), so that v can live in registers.  (The loop nest below leaves each step's trip count to the outer loop
// and chooses between addresses: v is kept in local memory.)
template <bool REGS = false>
__device__ __forceinline__ double warp_reduce16(double (&v)[16], int lane) {
  if constexpr (REGS) {
    reduce16_step<8>(v, lane);
    reduce16_step<4>(v, lane);
    reduce16_step<2>(v, lane);
    reduce16_step<1>(v, lane);
  } else {
#pragma unroll
    for (int m = 8; m >= 1; m >>= 1) {
      const int o = 2 * m;  // 16, 8, 4, 2
      const bool upper = (lane & o) != 0;
#pragma unroll
      for (int i = 0; i < m; ++i) {
        const double send = upper ? v[i] : v[i + m];
        const double keep = upper ? v[i + m] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
  }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

// Running (best, second, argmax) with numpy's first-maximum rule; `second` is the largest of the OTHER scores, so an
// exact tie gives second == best (margin 0 -> "ambiguous").  NaN follows np.argmax too: a NaN score is the maximum, and
// the first NaN wins among several (finite features can overflow to inf - inf in float64).  best = NaN then makes the
// margin test fail, so such a row is counted as ambiguous.
struct Top2 {
  double best, second;
  int idx;
};

// does candidate (ob, oi) beat the current best (b, bi) under np.argmax's rule?
__device__ __forceinline__ bool argmax_takes(double ob, int oi, double b, int bi) {
  if (isnan(ob)) return !isnan(b) || oi < bi;
  return !isnan(b) && (ob > b || (ob == b && oi < bi));
}

// NAN_RULE = false: the caller's scores cannot be NaN (the MLP stage's logits of finite fp32 inputs, DESIGN.md 3.3)
template <bool NAN_RULE = true>
__device__ __forceinline__ void top2_merge(Top2& t, double ob, double os, int oi) {
  const bool take = NAN_RULE ? argmax_takes(ob, oi, t.best, t.idx) : (ob > t.best || (ob == t.best && oi < t.idx));
  const double loser = take ? t.best : ob;
  t.second = fmax(fmax(t.second, os), loser);
  if (take) {
    t.best = ob;
    t.idx = oi;
  }
}

// all-lanes top-2 over per-lane candidates; first_offset = 2 when lane pairs hold the same class (after warp_reduce16)
template <bool NAN_RULE = true>
__device__ __forceinline__ void top2_butterfly(Top2& t, int first_offset) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    if (o < first_offset) break;
    const double ob = __shfl_xor_sync(0xffffffffu, t.best, o);
    const double os = __shfl_xor_sync(0xffffffffu, t.second, o);
    const int oi = __shfl_xor_sync(0xffffffffu, t.idx, o);
    top2_merge<NAN_RULE>(t, ob, os, oi);
  }
}

__device__ __forceinline__ double warp_max(double v, int first_offset) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    if (o < first_offset) break;
    v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  }
  return v;
}

}  // namespace uml
