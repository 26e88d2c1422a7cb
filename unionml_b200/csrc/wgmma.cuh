// PTX building blocks for the Hopper warpgroup tensor-core MMA (wgmma) on sm_90a.
//
// A warpgroup (four consecutive warps, 128 threads) issues wgmma.mma_async together; both operands are shared-memory
// matrix descriptors (K-major, 128-byte swizzle - the layout TMA's SWIZZLE_128B boxes already have) and the fp32
// accumulator lives in the registers of the 128 threads.  SASS: HGMMA, WARPGROUP.ARRIVE / WARPGROUP.DEPBAR.
#pragma once

#include <stdint.h>

#include "tma_ring.cuh"

namespace uml {

// ---- shared-memory matrix descriptor (64 bit): K-major operand, SWIZZLE_128B, rows of 128 bytes ---------------------
//   bits [0,14)  start address >> 4          bits [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   bits [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B between 8-row groups)
//   bits [62,64) layout type = 1 (SWIZZLE_128B)
// The tile base must be 1024-byte aligned; stepping K by 8 tf32 (32 bytes) inside the 128-byte swizzle atom adds
// 32 >> 4 = 2 to the start-address field.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3ffffu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// keeps the compiler from moving accesses of an accumulator register across the asynchronous MMA
__device__ __forceinline__ void wgmma_fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 x tf32 -> fp32, one K = 8 step (32 bytes of tf32 per row); scale_d = 0
// overwrites D.  Thread t of the warpgroup holds, for i < N / 8: d[4i], d[4i+1] = row 16 (t / 32) + (t % 32) / 4,
// columns 8i + 2 (t % 4) + {0, 1}; d[4i+2], d[4i+3] = the same columns of the row 8 below.
template <int N>
struct WgmmaTf32;

template <>
struct WgmmaTf32<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d)
        : "memory");
  }
};

template <>
struct WgmmaTf32<32> {
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d)
        : "memory");
  }
};

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, f16 x f16 -> fp32, one K = 16 step (32 bytes of f16 per row), both operands
// K-major (transpose immediates 0, 0); scale_d = 0 overwrites D.  Same fragment layout as WgmmaTf32.  N: the widths the
// linear tile kernel's tensor-core schedules use (linear_tc_cols).
// mma_ra: the same with A from registers (f16 A fragment of the PTX ISA): thread t of the warpgroup holds row
// r = 16 (t / 32) + (t % 32) / 4 and column group q = t % 4 as a[0] = (r, 2q..2q+1), a[1] = (r + 8, 2q..2q+1),
// a[2] = (r, 2q+8..2q+9), a[3] = (r + 8, 2q+8..2q+9), each an f16x2 with the lower column in the low half.  The
// registers are read asynchronously: the caller keeps them unchanged until the wgmma_wait that covers the MMA.
template <int N>
struct WgmmaF16;

#define UML_WGMMA_F16(N, REGS, NA, NB, NS, RA, RB, RS, ...)                                                   \
  template <>                                                                                                 \
  struct WgmmaF16<N> {                                                                                        \
    static __device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc,           \
                                               uint32_t scale_d) {                                            \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" NS ", 0;\n\t"                                     \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, %" NA ", %" NB         \
                   ", p, 1, 1, 0, 0;\n\t}"                                                                    \
                   : __VA_ARGS__                                                                              \
                   : "l"(a_desc), "l"(b_desc), "r"(scale_d)                                                   \
                   : "memory");                                                                               \
    }                                                                                                         \
    static __device__ __forceinline__ void mma_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc, \
                                                  uint32_t scale_d) {                                         \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" RS ", 0;\n\t"                                     \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, {" RA "}, %" RB        \
                   ", p, 1, 1, 0;\n\t}"                                                                       \
                   : __VA_ARGS__                                                                              \
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d)                    \
                   : "memory");                                                                               \
    }                                                                                                         \
  };
#define UML_R4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
UML_WGMMA_F16(16, "%0, %1, %2, %3, %4, %5, %6, %7", "8", "9", "10", "%8, %9, %10, %11", "12", "13", UML_R4(0),
              UML_R4(4))
UML_WGMMA_F16(24, "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11", "12", "13", "14", "%12, %13, %14, %15", "16",
              "17", UML_R4(0), UML_R4(4), UML_R4(8))
UML_WGMMA_F16(32, "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15", "16", "17", "18",
              "%16, %17, %18, %19", "20", "21", UML_R4(0), UML_R4(4), UML_R4(8), UML_R4(12))
UML_WGMMA_F16(40, "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19", "20",
              "21", "22", "%20, %21, %22, %23", "24", "25", UML_R4(0), UML_R4(4), UML_R4(8), UML_R4(12), UML_R4(16))
#undef UML_R4
#undef UML_WGMMA_F16

// keeps the compiler from reusing an A register of a register-A wgmma before the wgmma_wait that covers it
__device__ __forceinline__ void wgmma_fence_operand(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }

// two bytes of w (bytes 2i, 2i + 1) -> f16x2 with the lower byte in the low half, exactly: PRMT places each byte under
// an exponent byte 0x64 (the f16 value 1024 + byte), HADD2 subtracts 1024
__device__ __forceinline__ uint32_t bytes_to_half2(uint32_t w, int i) {
  uint32_t h, r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(h) : "r"(w), "r"(0x64646464u), "r"(i == 0 ? 0x4140u : 0x4342u));
  asm("add.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(h), "r"(0xe400e400u));
  return r;
}

// generic-proxy writes to shared memory (st.shared) -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// bounded mbarrier wait: a protocol bug traps (an error the host sees) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}
// the same for roles that are ahead of the critical path (producer, scan): back off between polls so the spinning
// does not take issue slots from the MMA / epilogue warps sharing the sub-partition
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(64);
    if (++spins > (1u << 24)) __trap();
  }
}

}  // namespace uml
