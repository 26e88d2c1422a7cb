// Staging kernels: feature rows in the caller's dtype/order (already copied to a device scratch chunk) -> the
// engine's resident layout: fp32 row-major [rows][ld] (optionally also an fp64 row-major copy for exact re-scoring).
//
// Replaces the host-side pandas/numpy copies of Dataset.get_features (unionml:unionml/dataset.py:350-359,
// 506-520: pd.DataFrame(features)[cols]) and sklearn's check_array finiteness scan
// (sklearn/utils/validation.py:107): the scan for NaN/Inf and the "is the fp32 copy lossless" test are fused into
// the conversion pass, so each element is touched once.
#include <cstring>
#include <type_traits>

#include "uml_common.cuh"

namespace uml {

template <typename T>
__device__ __forceinline__ double load_as_double(const T* p) {
  return static_cast<double>(*p);
}

// flag bits accumulated per thread: 1 = NaN/Inf, 2 = fp32 copy differs from the source value, 4 = fp32 value is not
// a tf32 value (low 13 mantissa bits set)
template <typename T>
__device__ __forceinline__ void convert_one(T v, float* out32, double* out64, unsigned& nonfinite, unsigned& lossy) {
  const double d = static_cast<double>(v);
  const float f = static_cast<float>(d);
  *out32 = f;
  if (out64) *out64 = d;
  if (!isfinite(d)) {
    nonfinite |= 1u;
  } else if (static_cast<double>(f) != d) {
    lossy |= 1u;
  }
  if (__float_as_uint(f) & 0x1fffu) lossy |= 2u;  // second bit of `lossy`: not a tf32 value
}

__device__ __forceinline__ void publish_flags(unsigned nonfinite, unsigned lossy, StageResult* result) {
  if (__any_sync(0xffffffffu, nonfinite) && (threadIdx.x & 31) == 0) atomicAdd(&result->nonfinite, 1ull);
  if (__any_sync(0xffffffffu, lossy & 1u) && (threadIdx.x & 31) == 0) atomicAdd(&result->lossy, 1ull);
  if (__any_sync(0xffffffffu, lossy & 2u) && (threadIdx.x & 31) == 0) atomicAdd(&result->not_tf32, 1ull);
}

// source is row-major: element (r, f) at src[r * pitch + f]
template <typename T>
__global__ void __launch_bounds__(256) stage_rowmajor_kernel(const T* __restrict__ src, long long pitch, long long rows,
                                                             int F, float* __restrict__ dst, long long ld,
                                                             double* __restrict__ dst64, long long ld64,
                                                             StageResult* result) {
  unsigned nonfinite = 0, lossy = 0;
  const long long total = rows * static_cast<long long>(ld);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / ld;
    const int f = static_cast<int>(i - r * ld);
    if (f < F) {
      convert_one(src[r * pitch + f], dst + i, dst64 ? dst64 + r * ld64 + f : nullptr, nonfinite, lossy);
    } else {
      dst[i] = 0.f;  // padding columns up to ld
    }
  }
  publish_flags(nonfinite, lossy, result);
}

// source is feature-major (a pandas block): element (r, f) at src[f * pitch + r].
// Tile = 128 rows x 32 features through shared memory.  Read side: a warp-level load covers 32 consecutive rows of one
// feature (256 B of float64, whole sectors), 16 independent loads per thread in flight before the first use (latency
// hiding by memory-level parallelism, not occupancy).  Write side: a warp writes one row segment of 32 features
// (128 B, one line) per store.  The row stride of the tile is 33 floats, so both phases are bank-conflict free.
// KEEP64 adds a float64 tile for the optional fp64 copy (resident batches staged with UML_STAGE_KEEP_F64).
constexpr int kStRows = 128;
constexpr int kStFeat = 32;

template <typename T, bool KEEP64>
__global__ void __launch_bounds__(256) stage_featmajor_kernel(const T* __restrict__ src, long long pitch,
                                                              long long rows, int F, float* __restrict__ dst,
                                                              long long ld, double* __restrict__ dst64, long long ld64,
                                                              StageResult* result) {
  using TileT = typename std::conditional<KEEP64, double, float>::type;  // one tile: the float64 values when both copies are wanted
  __shared__ TileT tile[kStRows][kStFeat + 1];
  unsigned nonfinite = 0, lossy = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;  // 8 warps
  const long long row_tiles = (rows + kStRows - 1) / kStRows;
  const int feat_tiles = static_cast<int>((ld + kStFeat - 1) / kStFeat);
  const long long tiles = row_tiles * feat_tiles;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long r0 = (t / feat_tiles) * kStRows;
    const int f0 = static_cast<int>(t % feat_tiles) * kStFeat;
    // ---- read: 32 features x 4 row groups = 128 (feature, group) pairs, 16 per warp; all loads issued first ----
    T v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int pair = warp * 16 + i;
      const int f = f0 + (pair >> 2);
      const long long r = r0 + (pair & 3) * 32 + lane;
      v[i] = (f < F && r < rows) ? __ldg(src + static_cast<long long>(f) * pitch + r) : T(0);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int pair = warp * 16 + i;
      const int fl = pair >> 2, rl = (pair & 3) * 32 + lane;
      float f32;
      double d;
      convert_one(v[i], &f32, &d, nonfinite, lossy);
      if constexpr (KEEP64) tile[rl][fl] = d;
      else tile[rl][fl] = f32;
    }
    __syncthreads();
    // ---- write: lanes along the 32 features of a row (128 B per store), 16 rows per warp ----
    const int f = f0 + lane;
#pragma unroll 4
    for (int i = 0; i < kStRows / 8; ++i) {
      const int rl = warp * (kStRows / 8) + i;
      const long long r = r0 + rl;
      if (r < rows && f < ld) {
        dst[r * ld + f] = f < F ? static_cast<float>(tile[rl][lane]) : 0.f;
        if constexpr (KEEP64) {
          if (dst64 && f < F) dst64[r * ld64 + f] = tile[rl][lane];
        }
      }
    }
    __syncthreads();
  }
  publish_flags(nonfinite, lossy, result);
}

// finiteness scan of rows that are already fp32 row-major on the device (no conversion needed)
__global__ void __launch_bounds__(256) finite_scan_kernel(const float* __restrict__ x, long long ld, long long rows,
                                                          int F, StageResult* result) {
  unsigned nonfinite = 0, low = 0;
  const long long total = rows * static_cast<long long>(ld);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int f = static_cast<int>(i % ld);
    if (f < F) {
      const float v = x[i];
      if (!isfinite(v)) nonfinite = 1u;
      low |= __float_as_uint(v);
    }
  }
  publish_flags(nonfinite, (low & 0x1fffu) ? 2u : 0u, result);
}

// dense variants (ld == F, source pitch == F): no per-element index arithmetic, 16-byte accesses
__global__ void __launch_bounds__(256) finite_scan_dense_kernel(const float4* __restrict__ x, long long n4,
                                                                StageResult* result) {
  unsigned nonfinite = 0, low = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(x + i);
    // x - x is 0 for finite x and NaN for NaN / Inf
    const float t = (v.x - v.x) + (v.y - v.y) + (v.z - v.z) + (v.w - v.w);
    if (!(t == 0.f)) nonfinite = 1u;
    low |= __float_as_uint(v.x) | __float_as_uint(v.y) | __float_as_uint(v.z) | __float_as_uint(v.w);
  }
  publish_flags(nonfinite, (low & 0x1fffu) ? 2u : 0u, result);
}

// four consecutive source elements with 16-byte loads where the type allows it
template <typename T>
__device__ __forceinline__ void load4(const T* __restrict__ p, T (&v)[4]) {
  if constexpr (sizeof(T) == 8) {
    const longlong2 a = __ldg(reinterpret_cast<const longlong2*>(p)), b = __ldg(reinterpret_cast<const longlong2*>(p) + 1);
    const long long raw[4] = {a.x, a.y, b.x, b.y};
#pragma unroll
    for (int k = 0; k < 4; ++k) memcpy(&v[k], &raw[k], 8);
  } else if constexpr (sizeof(T) == 4) {
    const int4 a = __ldg(reinterpret_cast<const int4*>(p));
    const int raw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) memcpy(&v[k], &raw[k], 4);
  } else {
    const uchar4 a = __ldg(reinterpret_cast<const uchar4*>(p));
    v[0] = static_cast<T>(a.x);
    v[1] = static_cast<T>(a.y);
    v[2] = static_cast<T>(a.z);
    v[3] = static_cast<T>(a.w);
  }
}

// dense row-major source (pitch == F == ld): no index arithmetic, 16-byte loads and stores, 2 x 4 elements per thread
// per iteration in flight
template <typename T>
__global__ void __launch_bounds__(256) stage_dense_kernel(const T* __restrict__ src, long long n, float* __restrict__ dst,
                                                          double* __restrict__ dst64, StageResult* result) {
  unsigned nonfinite = 0, lossy = 0;
  const long long n4 = n / 4;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += 2 * stride) {
    T v0[4], v1[4];
    const long long j = i + stride;
    load4(src + 4 * i, v0);
    if (j < n4) load4(src + 4 * j, v1);
    float4 o;
    float* op = &o.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) convert_one(v0[k], op + k, dst64 ? dst64 + 4 * i + k : nullptr, nonfinite, lossy);
    reinterpret_cast<float4*>(dst)[i] = o;
    if (j < n4) {
#pragma unroll
      for (int k = 0; k < 4; ++k) convert_one(v1[k], op + k, dst64 ? dst64 + 4 * j + k : nullptr, nonfinite, lossy);
      reinterpret_cast<float4*>(dst)[j] = o;
    }
  }
  publish_flags(nonfinite, lossy, result);
}

template <typename T>
static cudaError_t launch_typed(const void* src, bool feature_major, long long pitch, long long rows, int F, float* dst,
                                long long ld, double* dst64, long long ld64, StageResult* result, cudaStream_t stream) {
  static int sm_count = 0;  // grid caps scale with the device (one device per process)
  if (sm_count == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0) sm_count = 132;
  }
  const T* s = static_cast<const T*>(src);
  if (feature_major) {
    const long long tiles = ((rows + kStRows - 1) / kStRows) * ((ld + kStFeat - 1) / kStFeat);
    const long long cap = static_cast<long long>(sm_count) * 8;
    const int grid = static_cast<int>(tiles < cap ? (tiles < 1 ? 1 : tiles) : cap);
    if (dst64) stage_featmajor_kernel<T, true><<<grid, 256, 0, stream>>>(s, pitch, rows, F, dst, ld, dst64, ld64, result);
    else stage_featmajor_kernel<T, false><<<grid, 256, 0, stream>>>(s, pitch, rows, F, dst, ld, nullptr, 0, result);
  } else if (pitch == F && ld == F && (dst64 == nullptr || ld64 == F) && (F % 4) == 0 &&
             (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const long long want = (rows * ld / 8 + 255) / 256;
    const long long cap = static_cast<long long>(sm_count) * 16;
    const int grid = static_cast<int>(want < cap ? (want < 1 ? 1 : want) : cap);
    stage_dense_kernel<T><<<grid, 256, 0, stream>>>(s, rows * ld, dst, dst64, result);
  } else {
    const long long total = rows * ld;
    const long long want = (total + 255) / 256;
    const long long cap = static_cast<long long>(sm_count) * 16;
    const int grid = static_cast<int>(want < cap ? (want < 1 ? 1 : want) : cap);
    stage_rowmajor_kernel<T><<<grid, 256, 0, stream>>>(s, pitch, rows, F, dst, ld, dst64, ld64, result);
  }
  return cudaGetLastError();
}

cudaError_t launch_stage_convert(const void* src, int src_dtype, bool feature_major, int64_t src_pitch_elems,
                                 int64_t rows, int n_features, float* dst, int64_t ld, double* dst64, int64_t ld64,
                                 StageResult* result, bool check_finite, cudaStream_t stream) {
  (void)check_finite;  // the check is fused and free; the caller decides whether to act on the counter
  if (rows <= 0) return cudaSuccess;
  switch (src_dtype) {
    case UML_F32:
      return launch_typed<float>(src, feature_major, src_pitch_elems, rows, n_features, dst, ld, dst64, ld64, result, stream);
    case UML_F64:
      return launch_typed<double>(src, feature_major, src_pitch_elems, rows, n_features, dst, ld, dst64, ld64, result, stream);
    case UML_I64:
      return launch_typed<long long>(src, feature_major, src_pitch_elems, rows, n_features, dst, ld, dst64, ld64, result, stream);
    case UML_I32:
      return launch_typed<int>(src, feature_major, src_pitch_elems, rows, n_features, dst, ld, dst64, ld64, result, stream);
    case UML_U8:
      return launch_typed<unsigned char>(src, feature_major, src_pitch_elems, rows, n_features, dst, ld, dst64, ld64, result, stream);
    default:
      return cudaErrorInvalidValue;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// label push: copy this rank's slice of the label vector into the peers' vectors (or the NVLS multicast alias)
// ---------------------------------------------------------------------------------------------------------------
struct PushParams {
  const unsigned char* src;
  unsigned char* dst[8];
  int n_dst;
  long long bytes;
};

__global__ void __launch_bounds__(256) push_bytes_kernel(const PushParams p) {
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  bool aligned = (reinterpret_cast<uintptr_t>(p.src) & 15) == 0;
  for (int d = 0; d < p.n_dst; ++d) aligned = aligned && (reinterpret_cast<uintptr_t>(p.dst[d]) & 15) == 0;
  const long long n16 = aligned ? p.bytes / 16 : 0;
  for (long long i = tid; i < n16; i += nthreads) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(p.src) + i);
    for (int d = 0; d < p.n_dst; ++d) reinterpret_cast<uint4*>(p.dst[d])[i] = v;
  }
  for (long long i = n16 * 16 + tid; i < p.bytes; i += nthreads) {
    const unsigned char v = p.src[i];
    for (int d = 0; d < p.n_dst; ++d) p.dst[d][i] = v;
  }
}

cudaError_t launch_push_bytes(const void* src, void* const* dst, int n_dst, int64_t bytes, int sm_count,
                              cudaStream_t stream) {
  if (bytes <= 0 || n_dst <= 0) return cudaSuccess;
  PushParams p{};
  p.src = static_cast<const unsigned char*>(src);
  p.n_dst = n_dst;
  for (int d = 0; d < 8; ++d) p.dst[d] = d < n_dst ? static_cast<unsigned char*>(dst[d]) : nullptr;
  p.bytes = bytes;
  const long long want = (bytes / 16 + 255) / 256;
  const int grid = static_cast<int>(want < 1 ? 1 : (want < sm_count ? want : sm_count));  // a thin kernel: <= 1 CTA per SM
  push_bytes_kernel<<<grid, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// label post-processing (SURVEY.md 8f-4): classes_.take on the device and the evaluator's match count
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) labels_take_kernel(const void* __restrict__ labels, int label_bytes, long long n,
                                                          const double* __restrict__ classes, int n_classes,
                                                          double* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int idx = label_bytes == 1 ? static_cast<int>(static_cast<const unsigned char*>(labels)[i])
                                     : static_cast<const int*>(labels)[i];
    out[i] = idx >= 0 && idx < n_classes ? __ldg(classes + idx) : nan("");
  }
}

__global__ void __launch_bounds__(256) labels_count_equal_kernel(const void* __restrict__ labels, int label_bytes,
                                                                 long long n, const double* __restrict__ classes,
                                                                 int n_classes, const double* __restrict__ targets,
                                                                 unsigned long long* count) {
  unsigned long long local = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int idx = label_bytes == 1 ? static_cast<int>(static_cast<const unsigned char*>(labels)[i])
                                     : static_cast<const int*>(labels)[i];
    if (idx >= 0 && idx < n_classes && __ldg(classes + idx) == targets[i]) ++local;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

// int32 labels -> every target vector of a fused exchange
struct ScatterParams {
  const int32_t* labels;
  long long n;
  void* peers[8];
  int n_peers;
  int wire_u8;
  long long row_offset;
};

__global__ void __launch_bounds__(256) labels_scatter_kernel(const ScatterParams p) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < p.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int idx = p.labels[i];
    for (int q = 0; q < p.n_peers; ++q) {
      if (p.wire_u8) static_cast<unsigned char*>(p.peers[q])[p.row_offset + i] = static_cast<unsigned char>(idx);
      else static_cast<int32_t*>(p.peers[q])[p.row_offset + i] = idx;
    }
  }
}

cudaError_t launch_labels_scatter(const int32_t* labels, int64_t n, void* const* peers, int n_peers, int wire_u8,
                                  int64_t row_offset, int sm_count, cudaStream_t stream) {
  if (n <= 0 || n_peers <= 0) return cudaSuccess;
  ScatterParams p{};
  p.labels = labels;
  p.n = n;
  p.n_peers = n_peers;
  p.wire_u8 = wire_u8;
  p.row_offset = row_offset;
  for (int i = 0; i < 8; ++i) p.peers[i] = i < n_peers ? peers[i] : nullptr;
  const long long want = (n + 255) / 256;
  const int grid = static_cast<int>(want < static_cast<long long>(sm_count) * 4 ? want : static_cast<long long>(sm_count) * 4);
  labels_scatter_kernel<<<grid, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_labels_take(const void* labels, int label_bytes, int64_t n, const double* classes, int n_classes,
                               double* out, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long want = (n + 255) / 256;
  const int grid = static_cast<int>(want < 132 * 16 ? want : 132 * 16);
  labels_take_kernel<<<grid, 256, 0, stream>>>(labels, label_bytes, n, classes, n_classes, out);
  return cudaGetLastError();
}

cudaError_t launch_labels_count_equal(const void* labels, int label_bytes, int64_t n, const double* classes,
                                      int n_classes, const double* targets, unsigned long long* count,
                                      cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long want = (n + 255) / 256;
  const int grid = static_cast<int>(want < 132 * 8 ? want : 132 * 8);
  labels_count_equal_kernel<<<grid, 256, 0, stream>>>(labels, label_bytes, n, classes, n_classes, targets, count);
  return cudaGetLastError();
}

cudaError_t launch_finite_scan(const float* x, int64_t ld, int64_t rows, int n_features, StageResult* result,
                               cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  if (ld == n_features && (ld % 4) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const long long n4 = rows * ld / 4;
    const long long want4 = (n4 + 255) / 256;
    const int grid4 = static_cast<int>(want4 < 132 * 32 ? (want4 < 1 ? 1 : want4) : 132 * 32);
    finite_scan_dense_kernel<<<grid4, 256, 0, stream>>>(reinterpret_cast<const float4*>(x), n4, result);
    return cudaGetLastError();
  }
  const long long want = (rows * ld + 255) / 256;
  const int grid = static_cast<int>(want < 132 * 16 ? (want < 1 ? 1 : want) : 132 * 16);
  finite_scan_kernel<<<grid, 256, 0, stream>>>(x, ld, rows, n_features, result);
  return cudaGetLastError();
}

}  // namespace uml
