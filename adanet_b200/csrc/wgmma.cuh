// Hopper warpgroup MMA (wgmma) helpers shared by the split-plane GEMM (planes.cu) and the conv stem
// (conv_stem_tc.cu).  Operands come from shared memory through matrix descriptors; the accumulators live in the
// registers of the issuing warpgroup (m64 x N: warp w of the warpgroup holds rows 16w + lane/4 and 16w + lane/4 + 8,
// columns 8j + 2(lane%4) + {0, 1} in d[4j + {0, 1}] and d[4j + {2, 3}]).
#pragma once
#include <stdint.h>

namespace adn {
namespace wg {

// Shared-memory matrix descriptor (sm_90 GMMA): start address >> 4 at [0,14), leading byte offset >> 4 at [16,30),
// stride byte offset >> 4 at [32,46), layout type at [62,64) (1 = 128 B swizzle).  Every operand tile here is a
// 128 B swizzled tile on a 1024 B boundary whose 8-row core groups are 1024 B apart; each instruction spans a single
// 128 B swizzle atom in the other dimension, so both offsets are 1024 B.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(1024u >> 4) << 16) | ((uint64_t)(1024u >> 4) << 32) |
         (1ull << 62);
}
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define ADN_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                  "+f"(d[i + 6]), "+f"(d[i + 7])


// D (+)= A B, fp16 operands (TA / TB = 1: the operand is MN-major in shared memory), K = 16

template <int TA, int TB>
__device__ __forceinline__ void mma_f16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
               : ADN_D8(0), ADN_D8(8), ADN_D8(16), ADN_D8(24)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

// D (+)= A B, tf32 operands (both K-major), K = 8

__device__ __forceinline__ void mma_tf32_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
               : ADN_D8(0)
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void mma_tf32_n48(float (&d)[24], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1;\n\t}"
               : ADN_D8(0), ADN_D8(8), ADN_D8(16)
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void mma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
               : ADN_D8(0), ADN_D8(8), ADN_D8(16), ADN_D8(24)
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void mma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
               : ADN_D8(0), ADN_D8(8), ADN_D8(16), ADN_D8(24), ADN_D8(32), ADN_D8(40), ADN_D8(48), ADN_D8(56)
               : "l"(da), "l"(db), "r"(scale_d));
}

#undef ADN_D8

}  // namespace wg
}  // namespace adn
