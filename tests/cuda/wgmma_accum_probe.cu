// Test-only probe of the Hopper tf32 wgmma accumulation that the tensor-core MLP kernel's error bound relies on
// (DESIGN.md 3.3).  It runs the product's own WgmmaTf32<N>::mma and wgmma_desc_k_sw128 on chosen operands:
// D[64 x N] = sum over n_steps accumulating k8 steps of A[64 x 8 n_steps] . B[N x 8 n_steps]^T, exactly as
// mlp_argmax_tc_kernel issues them (first step scale_d = 0, one commit group, wait 0), and returns D row-major.
// tests/test_gpu_wgmma_accum.py compares D with exact sums.  Built by unionml_b200/_build.py:build_test_probes into
// build/tests/; the product never loads it.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../unionml_b200/csrc/wgmma.cuh"

namespace {

constexpr int kRows = 64;
constexpr int kMaxSteps = 16;  // K = 128 = four 32-wide swizzle atoms per row

// element (r, k) of a K-major SWIZZLE_128B operand: per 32-wide K chunk a block of rows x 128 B, each row's 16-byte
// pieces XOR-swizzled by (r & 7) - the layout of mlp_tc_build_w1_tiles and of the TMA boxes
__device__ __forceinline__ int sw128_index(int r, int k, int rows) {
  return (k / 32) * rows * 32 + r * 32 + (((k % 32) / 4) ^ (r & 7)) * 4 + (k % 4);
}

template <int N>
__global__ void __launch_bounds__(128, 1) wgmma_accum_probe_kernel(const float* a, const float* b, float* d, int n_steps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (uml::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int K = 8 * n_steps, kc = (K + 31) / 32;
  float* as = reinterpret_cast<float*>(smem);
  float* bs = as + kc * kRows * 32;
  for (int i = threadIdx.x; i < kc * kRows * 32; i += blockDim.x) as[i] = 0.f;
  for (int i = threadIdx.x; i < kc * N * 32; i += blockDim.x) bs[i] = 0.f;
  __syncthreads();
  for (int i = threadIdx.x; i < kRows * K; i += blockDim.x) as[sw128_index(i / K, i % K, kRows)] = a[i];
  for (int i = threadIdx.x; i < N * K; i += blockDim.x) bs[sw128_index(i / K, i % K, N)] = b[i];
  uml::fence_proxy_async_smem();  // st.shared -> visible to the async proxy that wgmma reads through
  __syncthreads();

  float acc[N / 2];
#pragma unroll
  for (int r = 0; r < N / 2; ++r) {
    acc[r] = 0.f;
    uml::wgmma_fence_operand(acc[r]);
  }
  uml::wgmma_fence();
  const uint32_t a_base = uml::smem_u32(as), b_base = uml::smem_u32(bs);
  for (int s = 0; s < n_steps; ++s) {
    const int chunk = s / 4, j = s % 4;
    uml::WgmmaTf32<N>::mma(acc, uml::wgmma_desc_k_sw128(a_base + chunk * kRows * 128 + j * 32),
                           uml::wgmma_desc_k_sw128(b_base + chunk * N * 128 + j * 32), s != 0 ? 1u : 0u);
  }
  uml::wgmma_commit();
  uml::wgmma_wait<0>();
#pragma unroll
  for (int r = 0; r < N / 2; ++r) uml::wgmma_fence_operand(acc[r]);
  // fragment layout of the WgmmaTf32 comment: d[4i + {0,1}] = row 16 (t / 32) + (t % 32) / 4, columns
  // 8 i + 2 (t % 4) + {0, 1}; d[4i + {2,3}] = the same columns of the row 8 below
  const int t = threadIdx.x;
  const int row = 16 * (t / 32) + (t % 32) / 4;
#pragma unroll
  for (int i = 0; i < N / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = 8 * i + 2 * (t % 4) + (e & 1);
      d[(row + 8 * (e >> 1)) * N + col] = acc[4 * i + e];
    }
}

template <int N>
cudaError_t run(const float* a, const float* b, float* d, int n_steps) {
  const int kc = (8 * n_steps + 31) / 32;
  const size_t smem = 1024 + static_cast<size_t>(kc) * (kRows + N) * 128;
  float *da = nullptr, *db = nullptr, *dd = nullptr;
  cudaError_t e = cudaMalloc(&da, sizeof(float) * kRows * 8 * n_steps);
  if (e == cudaSuccess) e = cudaMalloc(&db, sizeof(float) * N * 8 * n_steps);
  if (e == cudaSuccess) e = cudaMalloc(&dd, sizeof(float) * kRows * N);
  if (e == cudaSuccess) e = cudaMemcpy(da, a, sizeof(float) * kRows * 8 * n_steps, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(db, b, sizeof(float) * N * 8 * n_steps, cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(wgmma_accum_probe_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e == cudaSuccess) {
    wgmma_accum_probe_kernel<N><<<1, 128, smem>>>(da, db, dd, n_steps);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(d, dd, sizeof(float) * kRows * N, cudaMemcpyDeviceToHost);
  cudaFree(da);
  cudaFree(db);
  cudaFree(dd);
  return e;
}

}  // namespace

// a: [64][8 n_steps], b: [n][8 n_steps], d: [64][n], all row-major fp32 (tf32 values); n in {32, 64}.
// Returns 0 or the cudaError_t code.
extern "C" __attribute__((visibility("default"))) int uml_probe_wgmma_tf32(const float* a, const float* b, float* d,
                                                                            int n, int n_steps) {
  if (n_steps < 1 || n_steps > kMaxSteps) return static_cast<int>(cudaErrorInvalidValue);
  if (n == 64) return static_cast<int>(run<64>(a, b, d, n_steps));
  if (n == 32) return static_cast<int>(run<32>(a, b, d, n_steps));
  return static_cast<int>(cudaErrorInvalidValue);
}
