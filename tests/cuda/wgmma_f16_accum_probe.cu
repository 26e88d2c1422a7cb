// Test-only probe of the Hopper f16 wgmma accumulation that the tensor-core schedule of the linear tile kernel relies on
// (DESIGN.md 3.2).  It runs the product's own WgmmaF16<N>::mma and wgmma_desc_k_sw128 on chosen operands:
// D[64 x N] = sum over n_steps accumulating k16 steps of A[64 x 16 n_steps] . B[N x 16 n_steps]^T, as
// linear_argmax_tma_kernel<..., kHalfMma> issues them (first step scale_d = 0, one commit group, wait 0), and returns D
// row-major.  tests/test_gpu_wgmma_f16_accum.py compares D with exact sums.  Built by
// unionml_b200/_build.py:build_test_probes into build/tests/; the product never loads it.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../unionml_b200/csrc/wgmma.cuh"

namespace {

constexpr int kRows = 64;
constexpr int kMaxSteps = 4;  // K = 64: one 128-byte swizzle atom per row, the kernel's widest rows

// element (r, k) of a K-major SWIZZLE_128B f16 operand with K <= 64: row r at 64 r, its 16-byte pieces (8 halves)
// XOR-swizzled by (r & 7) - the layout of the fp16 TMA boxes and of build_tc_operands
__device__ __forceinline__ int sw128_index(int r, int k) { return r * 64 + (((k / 8) ^ (r & 7)) * 8) + (k % 8); }

template <int N>
__global__ void __launch_bounds__(128, 1) wgmma_f16_probe_kernel(const float* a, const float* b, float* d, int n_steps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (uml::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int K = 16 * n_steps;
  __half* as = reinterpret_cast<__half*>(smem);
  __half* bs = as + kRows * 64;
  for (int i = threadIdx.x; i < kRows * 64; i += blockDim.x) as[i] = __float2half_rn(0.f);
  for (int i = threadIdx.x; i < N * 64; i += blockDim.x) bs[i] = __float2half_rn(0.f);
  __syncthreads();
  for (int i = threadIdx.x; i < kRows * K; i += blockDim.x) as[sw128_index(i / K, i % K)] = __float2half_rn(a[i]);
  for (int i = threadIdx.x; i < N * K; i += blockDim.x) bs[sw128_index(i / K, i % K)] = __float2half_rn(b[i]);
  uml::fence_proxy_async_smem();
  __syncthreads();

  float acc[N / 2];
#pragma unroll
  for (int r = 0; r < N / 2; ++r) {
    acc[r] = 0.f;
    uml::wgmma_fence_operand(acc[r]);
  }
  uml::wgmma_fence();
  const uint32_t a_base = uml::smem_u32(as), b_base = uml::smem_u32(bs);
  for (int s = 0; s < n_steps; ++s)
    uml::WgmmaF16<N>::mma(acc, uml::wgmma_desc_k_sw128(a_base + s * 32), uml::wgmma_desc_k_sw128(b_base + s * 32),
                          s != 0 ? 1u : 0u);
  uml::wgmma_commit();
  uml::wgmma_wait<0>();
#pragma unroll
  for (int r = 0; r < N / 2; ++r) uml::wgmma_fence_operand(acc[r]);
  const int t = threadIdx.x;
  const int row = 16 * (t / 32) + (t % 32) / 4;
#pragma unroll
  for (int i = 0; i < N / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) d[(row + 8 * (e >> 1)) * N + 8 * i + 2 * (t % 4) + (e & 1)] = acc[4 * i + e];
}

template <int N>
cudaError_t run(const float* a, const float* b, float* d, int n_steps) {
  const size_t smem = 1024 + static_cast<size_t>(kRows + N) * 128;
  float *da = nullptr, *db = nullptr, *dd = nullptr;
  cudaError_t e = cudaMalloc(&da, sizeof(float) * kRows * 16 * n_steps);
  if (e == cudaSuccess) e = cudaMalloc(&db, sizeof(float) * N * 16 * n_steps);
  if (e == cudaSuccess) e = cudaMalloc(&dd, sizeof(float) * kRows * N);
  if (e == cudaSuccess) e = cudaMemcpy(da, a, sizeof(float) * kRows * 16 * n_steps, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(db, b, sizeof(float) * N * 16 * n_steps, cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(wgmma_f16_probe_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e == cudaSuccess) {
    wgmma_f16_probe_kernel<N><<<1, 128, smem>>>(da, db, dd, n_steps);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(d, dd, sizeof(float) * kRows * N, cudaMemcpyDeviceToHost);
  cudaFree(da);
  cudaFree(db);
  cudaFree(dd);
  return e;
}

}  // namespace

// a: [64][16 n_steps], b: [n][16 n_steps], d: [64][n], row-major fp32 holding fp16 values; n in {16, 32}.
// Returns 0 or the cudaError_t code.
extern "C" __attribute__((visibility("default"))) int uml_probe_wgmma_f16(const float* a, const float* b, float* d, int n,
                                                                           int n_steps) {
  if (n_steps < 1 || n_steps > kMaxSteps) return static_cast<int>(cudaErrorInvalidValue);
  if (n == 32) return static_cast<int>(run<32>(a, b, d, n_steps));
  if (n == 16) return static_cast<int>(run<16>(a, b, d, n_steps));
  return static_cast<int>(cudaErrorInvalidValue);
}
