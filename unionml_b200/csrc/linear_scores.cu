// float64 decision_function scores of the linear predictor (sm_90a):
//
//     out[r][j] = sum_f x_rf w64[f][c0 + j] + b_{c0 + j}
//
// LinearClassifierMixin.decision_function (sklearn/linear_model/_base.py:366-396), X @ coef_.T + intercept_, computed
// from the caller's own values (any dtype, either memory order: the SrcView of a raw chunk, a resident batch's float64
// copy, or fp32 rows that are the caller's values).  A binary model is stored expanded as [0, s]; only s is written
// (c0 = 1, one double per row), the (n,) shape of scikit-learn's binary decision_function.
//
// linear_scores_f64_kernel<PAIRS, WSMEM>: one thread per row, 128-row tiles on a persistent grid.  A tile's rows are
// staged through shared memory 32 features at a time with coalesced loads (consecutive threads take consecutive
// addresses in either memory order; a thread issues 16 loads before it stores the first), converted to
// float64 there, and each thread runs one sequential fp64 FMA chain per class over its row's features in order, then
// adds the bias: the summation order, and so the error bound, do not depend on the schedule (DESIGN.md 3.7).  Classes
// go in groups of 2 * PAIRS <= 16 (register accumulators); a model with more classes re-reads the tile per group.
// W sits in shared memory when it fits (WSMEM, zero padded to whole groups), else it is read from global memory.
// The scores leave through a shared-memory strip in output order, as whole runs of consecutive doubles.
//
// KIND selects what leaves: the scores (kF64Scores), or scikit-learn's predict_proba (kF64Proba) or predict_log_proba
// (kF64LogProba) of them, n_classes doubles per row ([1 - p, p] for a binary model).  proba_row turns a row's scores
// into them in float64: on the thread's strip row before the store for a model of one class group (C <= 16, binary
// included), and for a grouped model on the tile's rows in global memory, re-read by the block that wrote them after
// the tile's last group (DESIGN.md 3.9).
#include <algorithm>

#include "uml_common.cuh"

namespace uml {
namespace {

constexpr int kScoreRows = 128;        // rows per tile = threads per block (one row per thread)
constexpr int kScoreF = 32;            // features per staged chunk
constexpr int kScoreLd = kScoreF + 2;  // doubles per staged row: even, so a thread reads two features as one 16-byte
                                       // LDS.128, and 17 16-byte units, so a quarter-warp's eight rows fall into eight
                                       // different bank groups
constexpr int kScoreGroup = 16;        // classes per pass at most (2 * PAIRS)
constexpr size_t kTileBytes = static_cast<size_t>(kScoreRows) * kScoreLd * sizeof(double);

struct ScoresParams {
  SrcView src;
  long long n_rows;
  long long num_tiles;
  const double* w64;  // [F][S], feature-major, zero padded
  const double* b64;  // biases (then the bias magnitudes of the fp64 bound, unused here)
  int S, F, C;
  int c_first;  // 1 for the binary layout [0, s], else 0: the scores output starts at that class, probabilities take both
  int n_out;    // doubles per output row: C - c_first for the scores, C for the probabilities
  int sp;       // WSMEM: doubles per feature of the shared-memory copy of W (C rounded up to whole groups)
  double* out;
  unsigned long long* nonfinite;  // rows with NaN / Inf features
};

// features [f0, f0 + kScoreF) of rows [row0, row0 + kScoreRows) -> xs[r][f] as float64 (zero beyond the batch / row)
template <typename T>
__device__ __forceinline__ void load_chunk(const ScoresParams& p, long long row0, int f0, double* xs) {
  const T* base = static_cast<const T*>(p.src.base);
  const long long rs = p.src.row_stride, cs = p.src.col_stride;
  const long long rows = min(static_cast<long long>(kScoreRows), p.n_rows - row0);
  const int nf = min(kScoreF, p.F - f0);
  const int t = threadIdx.x;
  constexpr int kBatch = kScoreF / 2;  // loads in flight per thread before the first is stored (two batches)
#pragma unroll
  for (int h = 0; h < kScoreF; h += kBatch) {
    T v[kBatch];
    if (cs == 1) {
      // row-major: a warp reads 32 consecutive features of one row per load
      const int f = t % kScoreF;
#pragma unroll
      for (int k = 0; k < kBatch; ++k) {
        const int r = (h + k) * (kScoreRows / kScoreF) + t / kScoreF;
        v[k] = (r < rows && f < nf) ? __ldcs(base + (row0 + r) * rs + f0 + f) : T(0);
      }
#pragma unroll
      for (int k = 0; k < kBatch; ++k)
        xs[((h + k) * (kScoreRows / kScoreF) + t / kScoreF) * kScoreLd + f] = static_cast<double>(v[k]);
    } else {
      // feature-major: a warp reads 32 consecutive rows of one feature per load
#pragma unroll
      for (int k = 0; k < kBatch; ++k)
        v[k] = (t < rows && h + k < nf) ? __ldcs(base + (row0 + t) * rs + static_cast<long long>(f0 + h + k) * cs) : T(0);
#pragma unroll
      for (int k = 0; k < kBatch; ++k) xs[t * kScoreLd + h + k] = static_cast<double>(v[k]);
    }
  }
}

// a row's scores v[0, n) -> their probabilities or log-probabilities, in place, in float64 with scikit-learn's formula
// and order: softmax of sklearn/utils/extmath.py (m = max, e_c = exp(s_c - m), S = sum of e_c in class order,
// p_c = e_c / S), or for the binary layout v = [0, s] scipy's expit p = 1 / (1 + exp(-s)) and the columns [1 - p, p]
// (LinearClassifierMixin._predict_proba_lr); the logs are np.log of those.  NaN propagates through the max as np.max
// does, so scores that overflowed give numpy's NaN / 0 / 1 pattern.  Not inlined: both epilogues run one body (v is a
// generic pointer, to shared or global memory), and the kernel around the call keeps the scores form's registers.
template <int KIND>
__device__ __noinline__ void proba_row(double* v, int n, bool binary) {
  constexpr bool kLog = KIND == kF64LogProba;
  if (binary) {
    const double p = 1.0 / (1.0 + exp(-v[1]));
    const double q = 1.0 - p;
    v[0] = kLog ? log(q) : q;
    v[1] = kLog ? log(p) : p;
    return;
  }
  double m = v[0];
  for (int c = 1; c < n; ++c) {
    const double s = v[c];
    if (s > m || isnan(s)) m = s;
  }
  double sum = 0.0;
  for (int c = 0; c < n; ++c) {
    const double e = exp(v[c] - m);
    v[c] = e;
    sum += e;
  }
  for (int c = 0; c < n; ++c) {
    const double pc = v[c] / sum;
    v[c] = kLog ? log(pc) : pc;
  }
}

template <int PAIRS, bool WSMEM, int KIND = kF64Scores>
__global__ void __launch_bounds__(kScoreRows, 3) linear_scores_f64_kernel(const ScoresParams p) {
  extern __shared__ __align__(16) double sc_smem[];
  double* xs = sc_smem;                          // [kScoreRows][kScoreLd]: the staged chunk, then the output strip
  double* ws = sc_smem + kScoreRows * kScoreLd;  // WSMEM: W as [F][sp], zero padded
  constexpr int G = 2 * PAIRS;
  if constexpr (WSMEM) {
    for (int i = threadIdx.x; i < p.F * p.sp; i += kScoreRows) {
      const int f = i / p.sp, c = i % p.sp;
      ws[i] = c < p.C ? p.w64[static_cast<size_t>(f) * p.S + c] : 0.0;
    }
    // (the first chunk's __syncthreads below orders these stores before any read)
  }
  const int t = threadIdx.x;
  const double* xr = xs + t * kScoreLd;
  for (long long tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const long long row0 = tile * kScoreRows;
    const int rows = static_cast<int>(min(static_cast<long long>(kScoreRows), p.n_rows - row0));
    for (int c0 = 0; c0 < p.C; c0 += G) {
      double acc[G];
#pragma unroll
      for (int q = 0; q < G; ++q) acc[q] = 0.0;
      // global W: the last group of a model with more than 16 classes stops at C (uniform branch)
      const int pairs = WSMEM ? PAIRS : min(PAIRS, (p.C - c0 + 1) / 2);
      bool bad = false;
      for (int f0 = 0; f0 < p.F; f0 += kScoreF) {
        __syncthreads();  // every thread is done with the previous chunk (or output strip) in xs
        switch (p.src.dtype) {
          case UML_F64: load_chunk<double>(p, row0, f0, xs); break;
          case UML_I64: load_chunk<long long>(p, row0, f0, xs); break;
          case UML_I32: load_chunk<int>(p, row0, f0, xs); break;
          case UML_U8: load_chunk<unsigned char>(p, row0, f0, xs); break;
          default: load_chunk<float>(p, row0, f0, xs); break;
        }
        __syncthreads();
        const int nf = min(kScoreF, p.F - f0);
        for (int f = 0; f < nf; f += 2) {
          const double2 xv = *reinterpret_cast<const double2*>(xr + f);
          bad |= !isfinite(xv.x) || !isfinite(xv.y);  // (a feature past F was staged as 0)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (e == 1 && f + 1 >= nf) break;
            const double x = e == 0 ? xv.x : xv.y;
            const int fg = f0 + f + e;
            if constexpr (WSMEM) {
              const double2* wp = reinterpret_cast<const double2*>(ws + static_cast<size_t>(fg) * p.sp + c0);
#pragma unroll
              for (int q = 0; q < PAIRS; ++q) {
                const double2 w = wp[q];
                acc[2 * q] = fma(x, w.x, acc[2 * q]);
                acc[2 * q + 1] = fma(x, w.y, acc[2 * q + 1]);
              }
            } else {
              const double2* wp = reinterpret_cast<const double2*>(p.w64 + static_cast<size_t>(fg) * p.S + c0);
#pragma unroll
              for (int q = 0; q < PAIRS; ++q) {
                if (q < pairs) {
                  const double2 w = __ldg(wp + q);
                  acc[2 * q] = fma(x, w.x, acc[2 * q]);
                  acc[2 * q + 1] = fma(x, w.y, acc[2 * q + 1]);
                }
              }
            }
          }
        }
      }
      if (c0 == 0) {  // NaN / Inf rows, counted once per row
        const unsigned mask = __ballot_sync(0xffffffffu, bad && t < rows);
        if ((t & 31) == 0 && mask) atomicAdd(p.nonfinite, static_cast<unsigned long long>(__popc(mask)));
      }
      // this group's output columns [j0, j0 + gc): classes max(c0, c_first) .. min(c0 + G, C) - 1 of the scores, every
      // class of the probabilities
      const int c_first = KIND == kF64Scores ? p.c_first : 0;
      const int cb = max(c0, c_first), ce = min(c0 + G, p.C);
      const int gc = ce - cb, j0 = cb - c_first;
      __syncthreads();  // xs is free: every thread has read its last chunk
      double* strip = xs;  // [rows][gc] in output order
#pragma unroll
      for (int q = 0; q < G; ++q) {
        const int c = c0 + q;
        if (c >= cb && c < ce) strip[t * gc + (c - cb)] = acc[q] + p.b64[c];
      }
      if constexpr (KIND != kF64Scores) {
        if (p.C <= G) proba_row<KIND>(strip + t * gc, gc, p.c_first != 0);  // one group: the whole row is in the strip
      }
      __syncthreads();
      // whole runs: one run of rows * n_out doubles when the group covers every output column, else one run of gc
      // doubles per row; consecutive threads store consecutive doubles either way, and nothing past row n_rows
      double* dst = p.out + row0 * p.n_out;
      const int total = rows * gc;
      if (gc == p.n_out) {
        for (int i = t; i < total; i += kScoreRows) __stcs(dst + i, strip[i]);
      } else {
        for (int i = t; i < total; i += kScoreRows) {
          const int r = i / gc, j = i - r * gc;
          __stcs(dst + static_cast<long long>(r) * p.n_out + j0 + j, strip[i]);
        }
      }
    }
    if constexpr (KIND != kF64Scores) {
      if (p.C > G) {  // grouped: every group of the tile's rows is written; each thread normalises its own row
        __syncthreads();  // makes the block's stores of the other threads visible
        if (t < rows) proba_row<KIND>(p.out + (row0 + t) * p.n_out, p.C, false);
      }
    }
  }
}

template <int PAIRS, bool WSMEM, int KIND>
cudaError_t launch_scores(const ScoresParams& p, int sm_count, size_t smem, cudaStream_t stream) {
  auto kern = linear_scores_f64_kernel<PAIRS, WSMEM, KIND>;
  static size_t configured = 0;  // per instantiation (one device per process): set the attribute once
  if (smem > configured) {
    const cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err != cudaSuccess) return err;
    configured = smem;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kScoreRows, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const long long grid = std::min<long long>(p.num_tiles, static_cast<long long>(per_sm) * sm_count);
  kern<<<static_cast<int>(std::max<long long>(1, grid)), kScoreRows, smem, stream>>>(p);
  return cudaGetLastError();
}

template <bool WSMEM, int KIND>
cudaError_t dispatch_pairs(int pairs, const ScoresParams& p, int sm_count, size_t smem, cudaStream_t stream) {
  switch (pairs) {
    case 1: return launch_scores<1, WSMEM, KIND>(p, sm_count, smem, stream);
    case 2: return launch_scores<2, WSMEM, KIND>(p, sm_count, smem, stream);
    case 3: return launch_scores<3, WSMEM, KIND>(p, sm_count, smem, stream);
    case 4: return launch_scores<4, WSMEM, KIND>(p, sm_count, smem, stream);
    case 5: return launch_scores<5, WSMEM, KIND>(p, sm_count, smem, stream);
    case 6: return launch_scores<6, WSMEM, KIND>(p, sm_count, smem, stream);
    case 7: return launch_scores<7, WSMEM, KIND>(p, sm_count, smem, stream);
    default: return launch_scores<8, WSMEM, KIND>(p, sm_count, smem, stream);
  }
}

template <int KIND>
cudaError_t dispatch_smem(int pairs, const ScoresParams& p, int sm_count, size_t w_bytes, cudaStream_t stream) {
  if (kTileBytes + w_bytes <= static_cast<size_t>(kMaxSmemBytes))
    return dispatch_pairs<true, KIND>(pairs, p, sm_count, kTileBytes + w_bytes, stream);
  return dispatch_pairs<false, KIND>(pairs, p, sm_count, kTileBytes, stream);
}

}  // namespace

cudaError_t launch_linear_scores_f64(const LinearDeviceModel& m, const SrcView& src, int64_t n_rows, double* out,
                                     unsigned long long* nonfinite, int sm_count, cudaStream_t stream, int kind) {
  if (n_rows <= 0) return cudaSuccess;
  ScoresParams p{};
  p.src = src;
  p.n_rows = n_rows;
  p.num_tiles = (n_rows + kScoreRows - 1) / kScoreRows;
  p.w64 = m.w64;
  p.b64 = m.b64;
  p.S = m.w64_stride;
  p.F = m.n_features;
  p.C = m.n_classes;
  p.c_first = m.binary ? 1 : 0;
  p.n_out = linear_f64_width(m, kind);
  p.out = out;
  p.nonfinite = nonfinite;
  const int pairs = std::min(kScoreGroup, m.n_classes + (m.n_classes & 1)) / 2;
  p.sp = (m.n_classes + 2 * pairs - 1) / (2 * pairs) * (2 * pairs);
  const size_t w_bytes = static_cast<size_t>(m.n_features) * p.sp * sizeof(double);
  switch (kind) {
    case kF64Proba: return dispatch_smem<kF64Proba>(pairs, p, sm_count, w_bytes, stream);
    case kF64LogProba: return dispatch_smem<kF64LogProba>(pairs, p, sm_count, w_bytes, stream);
    default: return dispatch_smem<kF64Scores>(pairs, p, sm_count, w_bytes, stream);
  }
}

}  // namespace uml
