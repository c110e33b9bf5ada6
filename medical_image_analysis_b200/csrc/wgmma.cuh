// Device-side wgmma / TMA helpers shared by the tensor-core kernels (gemm_wgmma.cu, attention.cu; sm_90a).
#pragma once

#include <cuda.h>
#include <cstdint>

#include "scan_common.cuh"

namespace mia {

__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *tm, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *tm, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }

// d[64 x 128 fragment] (+)= A[smem desc, 64 x 16] . B[smem desc, 128 x 16]^T ; accumulate == 0 overwrites.  Fragment of thread t
// of the warpgroup: d[4 j + 2 h + c] = element (16 (t / 32) + (t % 32) / 4 + 8 h, 8 j + 2 (t % 4) + c).
#define MIA_WGMMA_N128(TYPE)                                                                                                          \
    asm volatile(                                                                                                                     \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                                            \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPE "." TYPE                                                                  \
        " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"    \
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,"    \
        "%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"                                                                                 \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),     \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),        \
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),        \
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),        \
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])         \
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(kAMN ? 1 : 0), "n"(kBMN ? 1 : 0)                                             \
        : "memory")
#define MIA_WGMMA_N64(TYPE)                                                                                                           \
    asm volatile(                                                                                                                     \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                                            \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE                                                                   \
        " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"   \
        " %32, %33, p, 1, 1, %35, %36;\n\t}"                                                                                          \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),     \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])                                                                          \
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(kAMN ? 1 : 0), "n"(kBMN ? 1 : 0)                                             \
        : "memory")

template <bool kF16, bool kAMN, bool kBMN>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    if (kF16) MIA_WGMMA_N128("f16"); else MIA_WGMMA_N128("bf16");
}
template <bool kF16, bool kAMN, bool kBMN>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    if (kF16) MIA_WGMMA_N64("f16"); else MIA_WGMMA_N64("bf16");
}

// Shared-memory matrix descriptor of a K-major tile staged by TMA with the 128-byte swizzle: rows of 64 elements
// (128 bytes), 8-row groups 1024 bytes apart (SBO), leading offset unused, layout type 1 (SWIZZLE_128B) in bits 62-63.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// MN-major operand (the M / N index is the contiguous one, e.g. X^T or W^T read in place): TMA boxes of [64 k-rows x 64
// mn-elements (128 bytes)] with the 128-byte swizzle, consecutive 64-wide mn slices 8192 bytes apart.  Canonical layout
// ((8,8,m),(8,k)) : ((1,8,LBO),(64,SBO)) elements: LBO = 8192 B between mn slices, SBO = 1024 B between groups of 8 k-rows.
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// Descriptor of an unswizzled operand (layout type 0) built from 8 x 16-byte core matrices, each 128 contiguous bytes.
// K-major ((8,m),(8,2k)): LBO = bytes between core matrices along K, SBO = between 8-row groups along M / N.
// MN-major ((8,m),(8,k)): SBO = bytes between 8-element groups along M / N, LBO = between 8-row groups along K.
__device__ __forceinline__ uint64_t wgmma_desc_plain(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

}  // namespace mia
