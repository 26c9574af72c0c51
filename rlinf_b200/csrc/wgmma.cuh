// sm_90a wgmma wrappers: D[64 x N] (+)= A[64 x 16] . B[16 x N], fp16 in, fp32 accumulators in registers.  Mma: A from
// registers (the m64k16 fragment of the PTX ISA), B from a descriptor (TB = 1: MN-major).  MmaSS: both K-major descriptors.
// Accumulator fragment: for each 8-column block j, d[4j + {0,1}] = (row g, cols 8j + 2t + {0,1}) and d[4j + {2,3}] =
// (row g + 8, same cols), rows relative to 16 * (warp % 4), g = lane / 4, t = lane % 4.
#pragma once
#include <stdint.h>

namespace rb {
namespace wg {

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout [62,64): 1 = SWIZZLE_128B,
// 2 = SWIZZLE_64B (operand tiles 1024-byte aligned, base offset 0)
__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
  return (uint64_t)((saddr & 0x3ffffu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3fffu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fffu) << 32) | ((uint64_t)layout << 62);
}

#define RB_WG_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define RB_WG_D16(i) RB_WG_D4(i), RB_WG_D4(i + 4), RB_WG_D4(i + 8), RB_WG_D4(i + 12)
#define RB_WG_D64(i) RB_WG_D16(i), RB_WG_D16(i + 16), RB_WG_D16(i + 32), RB_WG_D16(i + 48)

template <int N, int TB>
struct Mma;
template <int N>
struct MmaSS;

template <int TB>
struct Mma<128, TB> {
  __device__ __forceinline__ static void run(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
                 "}, {%64, %65, %66, %67}, %68, p, 1, 1, %70;\n}\n"
                 : RB_WG_D64(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
  }
};

template <int TB>
struct Mma<256, TB> {
  __device__ __forceinline__ static void run(float (&d)[128], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
                 "}, {%128, %129, %130, %131}, %132, p, 1, 1, %134;\n}\n"
                 : RB_WG_D64(0), RB_WG_D64(64)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
  }
};

template <>
struct MmaSS<32> {
  __device__ __forceinline__ static void run(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
                 "}, %16, %17, p, 1, 1, 0, 0;\n}\n"
                 : RB_WG_D16(0)
                 : "l"(a), "l"(b), "r"(scale_d));
  }
};

template <>
struct MmaSS<64> {
  __device__ __forceinline__ static void run(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
                 "}, %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : RB_WG_D16(0), RB_WG_D16(16)
                 : "l"(a), "l"(b), "r"(scale_d));
  }
};

#undef RB_WG_D64
#undef RB_WG_D16
#undef RB_WG_D4

}  // namespace wg
}  // namespace rb
