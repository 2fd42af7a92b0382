// Hopper (sm_90a) tensor-core helpers shared by the 3xTF32 kernels: warpgroup MMA (wgmma, kind tf32, fp32
// accumulators in registers), shared-memory matrix descriptors, mbarrier and the async-proxy fence.
//
// Register fragments of one warpgroup (128 threads; w = warp % 4, g = lane / 4, q = lane % 4), m64nNk8:
//   accumulator d[4 * j + i]  = D[16 w + g + 8 * (i / 2)][8 j + 2 q + (i % 2)]        j < N / 8
//   A operand   a[i]          = A[16 w + g + 8 * (i % 2)][q + 4 * (i / 2)]
// An accumulator therefore feeds the next MMA's A operand without a shuffle when k-slot s of every 8-wide k-step holds
// column kperm8(s) of the accumulator: a = {d[4j], d[4j + 2], d[4j + 1], d[4j + 3]}; the B operand of that MMA stores
// its k dimension in the same permuted order (a reduction does not care about the order of its terms).
#pragma once
#include <stdint.h>

namespace co {
namespace wg {

// k-slot s (0..7) of a k-step <-> column / key kperm8(s) of the 8-wide group
__host__ __device__ constexpr int kperm8(int s) { return s < 4 ? 2 * s : 2 * (s - 4) + 1; }
// inverse: the k-slot that holds column c (0..7)
__host__ __device__ constexpr int kslot8(int c) { return (c & 1) ? 4 + (c >> 1) : (c >> 1); }

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Shared-memory matrix descriptor, K-major: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), swizzle mode [62,64)
// (0 = none, 1 = 128 B).  128-B swizzle: rows of 128 B, 8-row atoms SBO apart, LBO unused.  No swizzle: 8 x 16 B core
// matrices, LBO apart along K and SBO apart along M / N.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint64_t desc_plain(uint32_t saddr, uint32_t sbo, uint32_t lbo) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// keeps the compiler from moving uses of an accumulator across the asynchronous MMAs that write it
template <int R>
__device__ __forceinline__ void pin(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define CO_WG_ACC8(d, o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])

// D[64 x 128] (+)= A[64 x 8] B[128 x 8]^T, both operands through shared-memory descriptors
__device__ __forceinline__ void mma_ss_n128(float (&d)[64], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : CO_WG_ACC8(d, 0), CO_WG_ACC8(d, 8), CO_WG_ACC8(d, 16), CO_WG_ACC8(d, 24), CO_WG_ACC8(d, 32), CO_WG_ACC8(d, 40),
        CO_WG_ACC8(d, 48), CO_WG_ACC8(d, 56)
      : "l"(a), "l"(b), "r"(accumulate)
      : "memory");
}
// the same with the A operand from registers (tf32 bit patterns in the fragment layout above)
__device__ __forceinline__ void mma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : CO_WG_ACC8(d, 0), CO_WG_ACC8(d, 8), CO_WG_ACC8(d, 16), CO_WG_ACC8(d, 24), CO_WG_ACC8(d, 32), CO_WG_ACC8(d, 40),
        CO_WG_ACC8(d, 48), CO_WG_ACC8(d, 56)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate)
      : "memory");
}
// D[64 x 32] (+)= A[64 x 8] B[32 x 8]^T and D[64 x 16] (+)= A[64 x 8] B[16 x 8]^T, A from registers
__device__ __forceinline__ void mma_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : CO_WG_ACC8(d, 0), CO_WG_ACC8(d, 8)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void mma_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
      : CO_WG_ACC8(d, 0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ float rna_tf32(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u);
}

// ---- mbarrier
__device__ __forceinline__ void bar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void bar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

}  // namespace wg
}  // namespace co
