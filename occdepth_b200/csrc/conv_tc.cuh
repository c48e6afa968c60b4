// wgmma / TMA / mbarrier PTX wrappers for sm_90a (hand-written; bit layouts follow the PTX ISA "wgmma" matrix
// descriptor tables).
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------- mbarrier ----------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// count arrivals at once (count >= 1)
__device__ __forceinline__ void mbar_arrive(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// Spin on the phase parity.  A bounded spin: a protocol bug traps (context error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins > (1u << 28)) __trap();
  }
}

// named barrier over the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// named barrier shared by two warpgroups: one waits (bar.sync), the other signals without waiting (bar.arrive)
__device__ __forceinline__ void pair_wait(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void pair_signal(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

// register budget hand-off between the producer warpgroup and the MMA warpgroups
template <int N> __device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------- TMA ----------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
      "%7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---------------- wgmma ----------------
// shared-memory matrix descriptor, K-major operand, swizzled rows of `row_bytes` (32/64/128):
//   bits [0,14)  start address >> 4         bits [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   bits [32,46) stride byte offset >> 4 (distance between 8-row groups)
//   bits [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B
// The TMA-written tiles start on 1024-byte boundaries and the XOR swizzle is a function of the absolute shared
// address bits on both the TMA and the wgmma side, so a start address shifted by whole rows (the halo kernels' tap
// views) or by 32 bytes of K keeps base offset 0.
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr, uint32_t row_bytes) {
  const uint32_t layout = row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : 3u);
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8u * row_bytes) >> 4) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// wait until at most n (0 <= n <= 9, warp-uniform) wgmma groups are pending
__device__ __forceinline__ void wg_wait_le(int n) {
  switch (n) {
    case 0: wg_wait<0>(); break;
    case 1: wg_wait<1>(); break;
    case 2: wg_wait<2>(); break;
    case 3: wg_wait<3>(); break;
    case 4: wg_wait<4>(); break;
    case 5: wg_wait<5>(); break;
    case 6: wg_wait<6>(); break;
    case 7: wg_wait<7>(); break;
    case 8: wg_wait<8>(); break;
    default: wg_wait<9>(); break;
  }
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int NA> __device__ __forceinline__ void acc_fence(float (&d)[NA]) {
#pragma unroll
  for (int i = 0; i < NA; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One m64nN MMA step over a 32-byte K slice: bf16 (K = 16) or TF32 (K = 8, fp32 containers whose TF32 bits the
// tensor core reads), N a multiple of 8 up to 256.  D: this thread's N / 2 fp32 accumulators of the 64 x N tile, the
// concatenation of the m64n8 fragments (warp w: rows 16 w + lane / 4 and + 8, columns 2 (lane % 4) + {0, 1} of every
// 8-column block: d[4 j .. 4 j + 3] belong to block j); scale_d == 0 overwrites them.
// OCCD_WG_R<nb> / OCCD_WG_D<nb>: the asm operand string / list of the accumulators of nb 8-column blocks; the
// predicate and the two descriptors follow them as operands nb*4, nb*4 + 1, nb*4 + 2.
#define OCCD_WG_Q(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define OCCD_WG_R1 "%0, %1, %2, %3"
#define OCCD_WG_R2 OCCD_WG_R1 ", %4, %5, %6, %7"
#define OCCD_WG_R3 OCCD_WG_R2 ", %8, %9, %10, %11"
#define OCCD_WG_R4 OCCD_WG_R3 ", %12, %13, %14, %15"
#define OCCD_WG_R5 OCCD_WG_R4 ", %16, %17, %18, %19"
#define OCCD_WG_R6 OCCD_WG_R5 ", %20, %21, %22, %23"
#define OCCD_WG_R7 OCCD_WG_R6 ", %24, %25, %26, %27"
#define OCCD_WG_R8 OCCD_WG_R7 ", %28, %29, %30, %31"
#define OCCD_WG_R9 OCCD_WG_R8 ", %32, %33, %34, %35"
#define OCCD_WG_R10 OCCD_WG_R9 ", %36, %37, %38, %39"
#define OCCD_WG_R11 OCCD_WG_R10 ", %40, %41, %42, %43"
#define OCCD_WG_R12 OCCD_WG_R11 ", %44, %45, %46, %47"
#define OCCD_WG_R13 OCCD_WG_R12 ", %48, %49, %50, %51"
#define OCCD_WG_R14 OCCD_WG_R13 ", %52, %53, %54, %55"
#define OCCD_WG_R15 OCCD_WG_R14 ", %56, %57, %58, %59"
#define OCCD_WG_R16 OCCD_WG_R15 ", %60, %61, %62, %63"
#define OCCD_WG_R17 OCCD_WG_R16 ", %64, %65, %66, %67"
#define OCCD_WG_R18 OCCD_WG_R17 ", %68, %69, %70, %71"
#define OCCD_WG_R19 OCCD_WG_R18 ", %72, %73, %74, %75"
#define OCCD_WG_R20 OCCD_WG_R19 ", %76, %77, %78, %79"
#define OCCD_WG_R21 OCCD_WG_R20 ", %80, %81, %82, %83"
#define OCCD_WG_R22 OCCD_WG_R21 ", %84, %85, %86, %87"
#define OCCD_WG_R23 OCCD_WG_R22 ", %88, %89, %90, %91"
#define OCCD_WG_R24 OCCD_WG_R23 ", %92, %93, %94, %95"
#define OCCD_WG_R25 OCCD_WG_R24 ", %96, %97, %98, %99"
#define OCCD_WG_R26 OCCD_WG_R25 ", %100, %101, %102, %103"
#define OCCD_WG_R27 OCCD_WG_R26 ", %104, %105, %106, %107"
#define OCCD_WG_R28 OCCD_WG_R27 ", %108, %109, %110, %111"
#define OCCD_WG_R29 OCCD_WG_R28 ", %112, %113, %114, %115"
#define OCCD_WG_R30 OCCD_WG_R29 ", %116, %117, %118, %119"
#define OCCD_WG_R31 OCCD_WG_R30 ", %120, %121, %122, %123"
#define OCCD_WG_R32 OCCD_WG_R31 ", %124, %125, %126, %127"
#define OCCD_WG_D1 OCCD_WG_Q(0)
#define OCCD_WG_D2 OCCD_WG_D1, OCCD_WG_Q(4)
#define OCCD_WG_D3 OCCD_WG_D2, OCCD_WG_Q(8)
#define OCCD_WG_D4 OCCD_WG_D3, OCCD_WG_Q(12)
#define OCCD_WG_D5 OCCD_WG_D4, OCCD_WG_Q(16)
#define OCCD_WG_D6 OCCD_WG_D5, OCCD_WG_Q(20)
#define OCCD_WG_D7 OCCD_WG_D6, OCCD_WG_Q(24)
#define OCCD_WG_D8 OCCD_WG_D7, OCCD_WG_Q(28)
#define OCCD_WG_D9 OCCD_WG_D8, OCCD_WG_Q(32)
#define OCCD_WG_D10 OCCD_WG_D9, OCCD_WG_Q(36)
#define OCCD_WG_D11 OCCD_WG_D10, OCCD_WG_Q(40)
#define OCCD_WG_D12 OCCD_WG_D11, OCCD_WG_Q(44)
#define OCCD_WG_D13 OCCD_WG_D12, OCCD_WG_Q(48)
#define OCCD_WG_D14 OCCD_WG_D13, OCCD_WG_Q(52)
#define OCCD_WG_D15 OCCD_WG_D14, OCCD_WG_Q(56)
#define OCCD_WG_D16 OCCD_WG_D15, OCCD_WG_Q(60)
#define OCCD_WG_D17 OCCD_WG_D16, OCCD_WG_Q(64)
#define OCCD_WG_D18 OCCD_WG_D17, OCCD_WG_Q(68)
#define OCCD_WG_D19 OCCD_WG_D18, OCCD_WG_Q(72)
#define OCCD_WG_D20 OCCD_WG_D19, OCCD_WG_Q(76)
#define OCCD_WG_D21 OCCD_WG_D20, OCCD_WG_Q(80)
#define OCCD_WG_D22 OCCD_WG_D21, OCCD_WG_Q(84)
#define OCCD_WG_D23 OCCD_WG_D22, OCCD_WG_Q(88)
#define OCCD_WG_D24 OCCD_WG_D23, OCCD_WG_Q(92)
#define OCCD_WG_D25 OCCD_WG_D24, OCCD_WG_Q(96)
#define OCCD_WG_D26 OCCD_WG_D25, OCCD_WG_Q(100)
#define OCCD_WG_D27 OCCD_WG_D26, OCCD_WG_Q(104)
#define OCCD_WG_D28 OCCD_WG_D27, OCCD_WG_Q(108)
#define OCCD_WG_D29 OCCD_WG_D28, OCCD_WG_Q(112)
#define OCCD_WG_D30 OCCD_WG_D29, OCCD_WG_Q(116)
#define OCCD_WG_D31 OCCD_WG_D30, OCCD_WG_Q(120)
#define OCCD_WG_D32 OCCD_WG_D31, OCCD_WG_Q(124)
#define OCCD_WG_STR(x) #x
template <typename T, int N> struct Mma;
#define OCCD_WG_MMA(N, NB, IS, IA, IB)                                                                             \
  template <> struct Mma<__nv_bfloat16, N> {                                                                       \
    static __device__ __forceinline__ void issue(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {              \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" OCCD_WG_STR(IS) ", 0;\n"                                     \
                   "wgmma.mma_async.sync.aligned.m64n" OCCD_WG_STR(N) "k16.f32.bf16.bf16 {" OCCD_WG_R##NB "}, %"       \
                   OCCD_WG_STR(IA) ", %" OCCD_WG_STR(IB) ", p, 1, 1, 0, 0;\n}\n"                                     \
                   : OCCD_WG_D##NB                                                                                 \
                   : "r"(scale_d), "l"(a), "l"(b));                                                                \
    }                                                                                                              \
  };                                                                                                               \
  template <> struct Mma<float, N> {                                                                               \
    static __device__ __forceinline__ void issue(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {              \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" OCCD_WG_STR(IS) ", 0;\n"                                     \
                   "wgmma.mma_async.sync.aligned.m64n" OCCD_WG_STR(N) "k8.f32.tf32.tf32 {" OCCD_WG_R##NB "}, %"        \
                   OCCD_WG_STR(IA) ", %" OCCD_WG_STR(IB) ", p, 1, 1;\n}\n"                                           \
                   : OCCD_WG_D##NB                                                                                 \
                   : "r"(scale_d), "l"(a), "l"(b));                                                                \
    }                                                                                                              \
  };
OCCD_WG_MMA(8, 1, 4, 5, 6)
OCCD_WG_MMA(16, 2, 8, 9, 10)
OCCD_WG_MMA(24, 3, 12, 13, 14)
OCCD_WG_MMA(32, 4, 16, 17, 18)
OCCD_WG_MMA(40, 5, 20, 21, 22)
OCCD_WG_MMA(48, 6, 24, 25, 26)
OCCD_WG_MMA(56, 7, 28, 29, 30)
OCCD_WG_MMA(64, 8, 32, 33, 34)
OCCD_WG_MMA(72, 9, 36, 37, 38)
OCCD_WG_MMA(80, 10, 40, 41, 42)
OCCD_WG_MMA(88, 11, 44, 45, 46)
OCCD_WG_MMA(96, 12, 48, 49, 50)
OCCD_WG_MMA(104, 13, 52, 53, 54)
OCCD_WG_MMA(112, 14, 56, 57, 58)
OCCD_WG_MMA(120, 15, 60, 61, 62)
OCCD_WG_MMA(128, 16, 64, 65, 66)
OCCD_WG_MMA(136, 17, 68, 69, 70)
OCCD_WG_MMA(144, 18, 72, 73, 74)
OCCD_WG_MMA(152, 19, 76, 77, 78)
OCCD_WG_MMA(160, 20, 80, 81, 82)
OCCD_WG_MMA(168, 21, 84, 85, 86)
OCCD_WG_MMA(176, 22, 88, 89, 90)
OCCD_WG_MMA(184, 23, 92, 93, 94)
OCCD_WG_MMA(192, 24, 96, 97, 98)
OCCD_WG_MMA(200, 25, 100, 101, 102)
OCCD_WG_MMA(208, 26, 104, 105, 106)
OCCD_WG_MMA(216, 27, 108, 109, 110)
OCCD_WG_MMA(224, 28, 112, 113, 114)
OCCD_WG_MMA(232, 29, 116, 117, 118)
OCCD_WG_MMA(240, 30, 120, 121, 122)
OCCD_WG_MMA(248, 31, 124, 125, 126)
OCCD_WG_MMA(256, 32, 128, 129, 130)
#undef OCCD_WG_MMA
#undef OCCD_WG_STR
#undef OCCD_WG_Q

}  // namespace tc
