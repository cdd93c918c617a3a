// wgmma.cuh — Hopper warpgroup MMA wrappers (sm_90a): m64nNk8 TF32 and m64nNk16 BF16, fp32
// accumulators in registers, both operands read from shared memory through matrix descriptors
// (K-major, no swizzle).  PTX names every accumulator register, so there is one specialisation
// per N (multiples of 16 up to 128).
//
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): for every 8-column
// block j, d[4j + 0..1] = row 16w + l/4, columns 8j + 2(l%4) + 0..1; d[4j + 2..3] = row + 8.
#pragma once
#include <stdint.h>

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int K>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(K) : "memory");
}
// keeps the compiler from moving accumulator reads/writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Shared-memory matrix descriptor, no swizzle: LBO = byte stride between the two 16-byte core-matrix
// columns along K, SBO = byte stride between 8-row groups along M / N (both in 16-byte units).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

template <int N> struct Wgmma;

#define AB_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), \
                   "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// N, the accumulator operand list "%0, ..., %(N/2 - 1)", the operand numbers of the two
// descriptors and of the scale-d flag, then the accumulator constraints
#define AB_WGMMA(N, REGS, A, B, S, ...)                                                          \
  template <> struct Wgmma<N> {                                                                  \
    static __device__ __forceinline__ void tf32(float (&d)[N / 2], uint64_t a, uint64_t b,       \
                                                uint32_t acc) {                                  \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" S ", 0;\n\t"                         \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 {" REGS "}, %" A    \
                   ", %" B ", p, 1, 1;\n\t}"                                                     \
                   : __VA_ARGS__ : "l"(a), "l"(b), "r"(acc));                                    \
    }                                                                                            \
    static __device__ __forceinline__ void bf16(float (&d)[N / 2], uint64_t a, uint64_t b,       \
                                                uint32_t acc) {                                  \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" S ", 0;\n\t"                         \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" REGS "}, %" A   \
                   ", %" B ", p, 1, 1, 0, 0;\n\t}"                                               \
                   : __VA_ARGS__ : "l"(a), "l"(b), "r"(acc));                                    \
    }                                                                                            \
  };

AB_WGMMA(16, "%0,%1,%2,%3,%4,%5,%6,%7", "8", "9", "10", AB_ACC8(0))
AB_WGMMA(32, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15", "16", "17", "18", AB_ACC8(0), AB_ACC8(8))
AB_WGMMA(48, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23", "24", "25", "26", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16))
AB_WGMMA(64, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31", "32", "33", "34", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16), AB_ACC8(24))
AB_WGMMA(80, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39", "40", "41", "42", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16), AB_ACC8(24), AB_ACC8(32))
AB_WGMMA(96, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47", "48", "49", "50", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16), AB_ACC8(24), AB_ACC8(32), AB_ACC8(40))
AB_WGMMA(112, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55", "56", "57", "58", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16), AB_ACC8(24), AB_ACC8(32), AB_ACC8(40), AB_ACC8(48))
AB_WGMMA(128, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63", "64", "65", "66", AB_ACC8(0), AB_ACC8(8), AB_ACC8(16), AB_ACC8(24), AB_ACC8(32), AB_ACC8(40), AB_ACC8(48), AB_ACC8(56))
#undef AB_WGMMA
#undef AB_ACC8
