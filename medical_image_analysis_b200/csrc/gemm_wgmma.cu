// Tensor-core GEMM for the projections around the scan and for the ViT-MAE patch encode (sm_90a: wgmma + TMA).
//
//   C[M, N] = act( A[M, K] . W[N, K]^T + bias[N] )        A, W: bf16 / fp16, K contiguous ("TN", nn.Linear's layout)
//
// Replaces the cuBLAS / cuDNN calls behind nn.Linear / einsum / kernel==stride nn.Conv2d at:
//   SS2D in_proj / out_proj / x_proj            R2GenCSR/VMamba/classification/models/vmamba.py:751, 775, 386
//   Mamba in_proj / x_proj / dt_proj / out_proj */arm/Finetuning/mamba_simple.py:408-414, 686-689, 708
//   SmallPatchEmbed conv16/16, conv4/4, conv1x1 HD_Xray_Pretrain_MAE/pretrain/patch_embed.py:25-41 (as GEMMs over patches)
//   timm Block qkv / proj / fc1 / fc2           HD_Xray_Pretrain_MAE/pretrain/models/mae.py:64-66, 82-84
//
// Structure (one persistent CTA per SM, three warpgroups of 128 threads, warp-specialised):
//   warpgroup 0   TMA producer (one elected thread, the group gives its registers away with setmaxnreg): 2-D tensor-map
//                 loads (cp.async.bulk.tensor.2d, SASS UTMALDG) of [128 x 64] A and [BN x 64] W tiles with the 128-byte
//                 swizzle into a ring of kStages shared-memory stages (full / empty mbarriers);
//   warpgroups 1-2  consumers: each owns 64 of the tile's 128 rows and keeps its [64 x BN] fp32 accumulator in registers;
//                 per 64-wide K block four wgmma.mma_async.m64nNk16 (SASS HGMMA) per 128 columns read both operands from
//                 shared memory through matrix descriptors; one K block stays in flight (wgmma.wait_group 1) and the
//                 stage before it is handed back to the producer.  Epilogue from the accumulator fragment: + bias,
//                 activation, conversion, 8-byte (fp32) / 4-byte (16-bit) stores of the two columns a thread holds per
//                 8-column group; the producer already streams the next tile's stages meanwhile.
// Out-of-range rows / columns / K tail are zero-filled by TMA and masked in the epilogue, so any M, N and any K with
// K % 8 == 0 (16-byte rows) work.  No split-K: K is at most 16384 (patch-embed conv4/4) and M is large on this path.
// The SwiGLU MLP (models_mamba.py:59-83) runs on the same CTA with a paired-B tile and its own epilogues (kEpiSwiglu*);
// the GELU MLP's fc1 and fc2-dgrad (vmamba.py:495-514, timm Mlp) run on it with the GELU and its derivative in theirs (kEpiGelu*).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstring>

#include "../../include/mia_gemm.h"
#include "abi_host.h"
#include "scan_common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kBM = 128, kBK = 64;
constexpr int kGemmThreads = 384;      // producer warpgroup + two consumer warpgroups

struct GemmArgs {
    int M, N, K;
    int act, out_f32, has_bias, in_f16;
    const float *bias;
    void *C;
    long long ldc;
    int num_m_blocks, num_n_blocks, num_k_blocks;
};

// Epilogue of a tile.  kEpiLinear: act(acc + bias) into C (mia_gemm_tn / mia_gemm).  The SwiGLU pair (mia_gemm_swiglu_*):
//   kEpiSwigluFwd  paired B tile: columns [0, BN/2) of the tile are x.W1^T, [BN/2, BN) x.W2^T at the same hidden columns;
//                  a = round(acc1 + b1), b = round(acc2 + b2) -> ab (optional), h = round(silu(a) b)
//   kEpiSwigluBwd  acc = g = dy.W3 (W3 read MN-major); a, b loaded from ab at the fragment's own (row, col) ->
//                  dab = (round(g b s (1 + a (1 - s))), round(g a s)), h = round(a s b) (optional), s = sigmoid(a)
// ab / dab are (M, 2 Hp): the a / da half in columns [0, H), the b / db half in [Hp, Hp + H), pad columns written as 0.
// The GELU pair (mia_gemm_gelu_*), Hp = H rounded up to 8:
//   kEpiGeluFwd    acc = x.W1^T: p = round(acc + b1) -> ab = pre (optional), h = round(gelu(p))
//   kEpiGeluBwd    acc = g = dy.W2 (W2 read MN-major); p loaded from ab = pre at the fragment's own (row, col) ->
//                  dab = dpre = round(g gelu'(p)), h = round(gelu(p)) (optional)
// pre / dpre / h are (M, Hp) with columns [H, Hp) written as 0.
enum { kEpiLinear = 0, kEpiSwigluFwd = 1, kEpiSwigluBwd = 2, kEpiGeluFwd = 3, kEpiGeluBwd = 4 };

// Operands of the fused epilogues (every mode but kEpiLinear).
struct EpiArgs {
    const float *b1, *b2;      // fwd biases (fp32, may be NULL; b2: SwiGLU only)
    void *h;                   // (M, H), pitch ldh (bwd: may be NULL)
    void *ab;                  // saved pre-activations (SwiGLU: packed a / b; GELU: pre).  fwd: output, may be NULL; bwd: input
    void *dab;                 // bwd output: their gradients, in ab's layout
    long long ldh, ldab, lddab;
    int H, Hp;
};

using mia::tma_load_2d;
using mia::wgmma_commit;
using mia::wgmma_desc_k_sw128;
using mia::wgmma_desc_mn_sw128;
using mia::wgmma_fence;
using mia::wgmma_n128;
using mia::wgmma_n64;
using mia::wgmma_wait;

// The operation order of ATen's CUDA GELU (x 0.5 (1 + erf(x sqrt(1/2))) in fp32), so that a GELU epilogue on a rounded
// pre-activation writes what F.gelu writes for it.
__device__ __forceinline__ float gelu(float p) { return 0.5f * p * (1.f + erff(p * 0.70710678118654752f)); }

__device__ __forceinline__ float act_apply(float v, int act) {
    switch (act) {
        case MIA_ACT_RELU: return fmaxf(v, 0.f);
        case MIA_ACT_GELU: return gelu(v);
        case MIA_ACT_SILU: return v / (1.f + __expf(-v));
        default: return v;
    }
}

// two adjacent columns of one row of C: one 8-byte / 4-byte store when both are inside N and the address allows it
template <bool kF16>
__device__ __forceinline__ void store_pair(const GemmArgs &g, int row, int col, float v0, float v1) {
    const bool both = col + 1 < g.N;
    if (g.out_f32) {
        float *dst = reinterpret_cast<float *>(g.C) + (size_t)row * g.ldc + col;
        if (both && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) { *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1); return; }
        dst[0] = v0;
        if (both) dst[1] = v1;
    } else {
        uint16_t *dst = reinterpret_cast<uint16_t *>(g.C) + (size_t)row * g.ldc + col;
        uint32_t w;
        if (kF16) { __half2 h = __floats2half2_rn(v0, v1); w = *reinterpret_cast<uint32_t *>(&h); }
        else { __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1); w = *reinterpret_cast<uint32_t *>(&h); }
        if (both && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) { *reinterpret_cast<uint32_t *>(dst) = w; return; }
        dst[0] = (uint16_t)(w & 0xffffu);
        if (both) dst[1] = (uint16_t)(w >> 16);
    }
}

template <bool kF16>
__device__ __forceinline__ float round_to(float v) {
    return kF16 ? __half2float(__float2half_rn(v)) : __bfloat162float(__float2bfloat16_rn(v));
}
template <bool kF16>
__device__ __forceinline__ float2 load2(const void *base, long long ld, int row, int col) {
    const uint32_t w = *reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint16_t *>(base) + (size_t)row * ld + col);
    if (kF16) return __half22float2(*reinterpret_cast<const __half2 *>(&w));
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&w));
}
// two adjacent 16-bit elements of a row; `both` false stores the first only
template <bool kF16>
__device__ __forceinline__ void store2(void *base, long long ld, int row, int col, float v0, float v1, bool both) {
    uint16_t *dst = reinterpret_cast<uint16_t *>(base) + (size_t)row * ld + col;
    uint32_t w;
    if (kF16) { __half2 h = __floats2half2_rn(v0, v1); w = *reinterpret_cast<uint32_t *>(&h); }
    else { __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1); w = *reinterpret_cast<uint32_t *>(&h); }
    if (both) *reinterpret_cast<uint32_t *>(dst) = w;
    else dst[0] = (uint16_t)(w & 0xffffu);
}

// SwiGLU epilogues of one thread's fragment (see kEpiSwigluFwd / kEpiSwigluBwd).  Host checks make every pitch even and
// every base 16-byte aligned, so the pair stores are aligned; Hp is a multiple of 64, so a pair never straddles it.
// Both compute h as (a s) b from the rounded a and b, so the backward's recomputed h is the forward's, bit for bit.
__device__ __forceinline__ float sigmoid(float a) { return 1.f / (1.f + __expf(-a)); }
template <bool kF16>
__device__ __forceinline__ void swiglu_fwd_pair(const EpiArgs &sw, int row, int col, float acc_a0, float acc_a1, float acc_b0,
                                                float acc_b1, float ba0, float ba1, float bb0, float bb1) {
    const bool in0 = col < sw.H, in1 = col + 1 < sw.H;
    const float a0 = in0 ? round_to<kF16>(acc_a0 + ba0) : 0.f, a1 = in1 ? round_to<kF16>(acc_a1 + ba1) : 0.f;
    const float b0 = in0 ? round_to<kF16>(acc_b0 + bb0) : 0.f, b1 = in1 ? round_to<kF16>(acc_b1 + bb1) : 0.f;
    if (sw.ab) {
        store2<kF16>(sw.ab, sw.ldab, row, col, a0, a1, true);
        store2<kF16>(sw.ab, sw.ldab, row, sw.Hp + col, b0, b1, true);
    }
    if (in0) store2<kF16>(sw.h, sw.ldh, row, col, a0 * sigmoid(a0) * b0, a1 * sigmoid(a1) * b1, in1);
}

// silu'(a) / s = 1 + a (1 - s).  It has a root at a = -1.2785: around it fp32 cancels to a relative error above half an
// fp16 ulp, so where |factor| < 2^-8 (a few representable a) it is recomputed in fp64.
__device__ __noinline__ float dsilu_factor_f64(float a) {
    const double e = exp(-(double)a);
    return (float)(1.0 + (double)a * e / (1.0 + e));
}
__device__ __forceinline__ float dsilu_factor(float a, float s) {
    const float f = 1.f + a * (1.f - s);
    return fabsf(f) < 0.00390625f ? dsilu_factor_f64(a) : f;
}

template <bool kF16>
__device__ __forceinline__ void swiglu_bwd_pair(const EpiArgs &sw, int row, int col, float g0, float g1) {
    const bool in0 = col < sw.H, in1 = col + 1 < sw.H;
    const float2 a = load2<kF16>(sw.ab, sw.ldab, row, col), b = load2<kF16>(sw.ab, sw.ldab, row, sw.Hp + col);
    const float s0 = sigmoid(a.x), s1 = sigmoid(a.y);
    const float da0 = in0 ? g0 * b.x * s0 * dsilu_factor(a.x, s0) : 0.f, da1 = in1 ? g1 * b.y * s1 * dsilu_factor(a.y, s1) : 0.f;
    const float db0 = in0 ? g0 * a.x * s0 : 0.f, db1 = in1 ? g1 * a.y * s1 : 0.f;
    store2<kF16>(sw.dab, sw.lddab, row, col, da0, da1, true);
    store2<kF16>(sw.dab, sw.lddab, row, sw.Hp + col, db0, db1, true);
    if (sw.h && in0) store2<kF16>(sw.h, sw.ldh, row, col, a.x * s0 * b.x, a.y * s1 * b.y, in1);
}

// GELU epilogues of one thread's fragment (see kEpiGeluFwd / kEpiGeluBwd).  Hp is a multiple of 8 and every pitch covers
// it, so both columns of a pair are stored; pads hold p = 0, whose gelu and dpre are 0.  h is gelu of the rounded p in both,
// so it equals F.gelu(pre) and the backward's recomputed h is the forward's, bit for bit.

// gelu'(p) = Phi(p) + p phi(p).  Phi is taken from erfc, which does not cancel in the negative tail as 1 + erf does.  The
// sum has a root at p = -0.7518: around it fp32 cancels to a relative error above half an fp16 ulp, so where
// |factor| < 2^-8 (a few representable p) it is recomputed in fp64.
__device__ __noinline__ float dgelu_f64(float p) {
    const double q = (double)p;
    return (float)(0.5 * erfc(-q * 0.70710678118654752) + q * exp(-0.5 * q * q) * 0.39894228040143268);
}
__device__ __forceinline__ float dgelu(float p) {
    const float f = 0.5f * erfcf(-p * 0.70710678118654752f) + p * expf(-0.5f * p * p) * 0.3989422804014327f;
    return fabsf(f) < 0.00390625f ? dgelu_f64(p) : f;
}

template <bool kF16>
__device__ __forceinline__ void gelu_fwd_pair(const EpiArgs &ep, int row, int col, float acc0, float acc1, float b0, float b1) {
    const bool in0 = col < ep.H, in1 = col + 1 < ep.H;
    const float p0 = in0 ? round_to<kF16>(acc0 + b0) : 0.f, p1 = in1 ? round_to<kF16>(acc1 + b1) : 0.f;
    if (ep.ab) store2<kF16>(ep.ab, ep.ldab, row, col, p0, p1, true);
    store2<kF16>(ep.h, ep.ldh, row, col, gelu(p0), gelu(p1), true);
}

template <bool kF16>
__device__ __forceinline__ void gelu_bwd_pair(const EpiArgs &ep, int row, int col, float g0, float g1) {
    const bool in0 = col < ep.H, in1 = col + 1 < ep.H;
    const float2 p = load2<kF16>(ep.ab, ep.ldab, row, col);
    store2<kF16>(ep.dab, ep.lddab, row, col, in0 ? g0 * dgelu(p.x) : 0.f, in1 ? g1 * dgelu(p.y) : 0.f, true);
    if (ep.h) store2<kF16>(ep.h, ep.ldh, row, col, in0 ? gelu(p.x) : 0.f, in1 ? gelu(p.y) : 0.f, true);
}

// The two consumer warpgroups: `cw` (0 / 1) owns rows [64 cw, 64 cw + 64) of every tile of this CTA.
template <int BN, int kStages, bool kAMN, bool kBMN, bool kF16, int kEpi = kEpiLinear>
__device__ __forceinline__ void gemm_consumer(const GemmArgs &g, char *tiles, uint64_t *full, uint64_t *empty, int cw,
                                              const EpiArgs *sw = nullptr) {
    constexpr int kABytes = kBM * kBK * 2, kStageBytes = kABytes + BN * kBK * 2;
    constexpr int kUnit = BN >= 128 ? 128 : 64;          // columns per wgmma instruction
    const int t = threadIdx.x & 127, lane = t & 31;
    const int num_tiles = g.num_m_blocks * g.num_n_blocks, KB = g.num_k_blocks;
    float d[BN / kUnit][kUnit / 2];
    int s = 0, prev = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mb = tile % g.num_m_blocks, nb = tile / g.num_m_blocks;
        for (int kb = 0; kb < KB; ++kb) {
            mia::mbar_wait(full + s, ph);
            const uint32_t a_addr = mia::smem_u32(tiles + s * kStageBytes) + cw * 8192, b_addr = mia::smem_u32(tiles + s * kStageBytes) + kABytes;
            const uint64_t da = kAMN ? wgmma_desc_mn_sw128(a_addr) : wgmma_desc_k_sw128(a_addr);
            // 16 elements along K per instruction: K-major = 32 bytes inside the swizzle atom (+2 in the address field);
            // MN-major = 16 k-rows of 128 bytes = 2048 bytes (+128).  64 columns (or rows of a K-major W tile) = 8192 bytes.
            constexpr uint64_t ka = kAMN ? 128 : 2, kbb = kBMN ? 128 : 2;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k) {
#pragma unroll
                for (int u = 0; u < BN / kUnit; ++u) {
                    const uint32_t bu = b_addr + u * (kUnit / 64) * 8192;
                    const uint64_t db = kBMN ? wgmma_desc_mn_sw128(bu) : wgmma_desc_k_sw128(bu);
                    if constexpr (kUnit == 128) wgmma_n128<kF16, kAMN, kBMN>(d[u], da + ka * k, db + kbb * k, (kb | k) != 0);
                    else wgmma_n64<kF16, kAMN, kBMN>(d[u], da + ka * k, db + kbb * k, (kb | k) != 0);
                }
            }
            wgmma_commit();
            if (kb > 0) {                                   // the K block before this one has been read: its stage is free
                wgmma_wait<1>();
                if (t == 0) mia::mbar_arrive(empty + prev);
            }
            prev = s;
            if (++s == kStages) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        if (t == 0) mia::mbar_arrive(empty + prev);

        const int row0 = mb * kBM + cw * 64 + (t >> 5) * 16 + (lane >> 2);
        if constexpr (kEpi == kEpiSwigluFwd) {
            // d[0] holds x.W1^T and d[1] x.W2^T at the same (row, hidden column): the gate needs no data exchange
            static_assert(BN == 256 && !kBMN, "the paired-B tile is 2 x 128 K-major rows");
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = nb * 128 + 8 * j + 2 * (lane & 3);
                if (col < sw->Hp) {
                    const bool in0 = col < sw->H, in1 = col + 1 < sw->H;
                    const float ba0 = sw->b1 && in0 ? __ldg(sw->b1 + col) : 0.f, ba1 = sw->b1 && in1 ? __ldg(sw->b1 + col + 1) : 0.f;
                    const float bb0 = sw->b2 && in0 ? __ldg(sw->b2 + col) : 0.f, bb1 = sw->b2 && in1 ? __ldg(sw->b2 + col + 1) : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = row0 + 8 * h;
                        if (row < g.M)
                            swiglu_fwd_pair<kF16>(*sw, row, col, d[0][4 * j + 2 * h], d[0][4 * j + 2 * h + 1], d[1][4 * j + 2 * h],
                                                  d[1][4 * j + 2 * h + 1], ba0, ba1, bb0, bb1);
                    }
                }
            }
        } else if constexpr (kEpi != kEpiLinear) {
#pragma unroll
            for (int u = 0; u < BN / kUnit; ++u) {
#pragma unroll
                for (int j = 0; j < kUnit / 8; ++j) {
                    const int col = nb * BN + u * kUnit + 8 * j + 2 * (lane & 3);
                    if (col < sw->Hp) {
                        float b0 = 0.f, b1 = 0.f;
                        if constexpr (kEpi == kEpiGeluFwd) {
                            b0 = sw->b1 && col < sw->H ? __ldg(sw->b1 + col) : 0.f;
                            b1 = sw->b1 && col + 1 < sw->H ? __ldg(sw->b1 + col + 1) : 0.f;
                        }
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int row = row0 + 8 * h;
                            if (row < g.M) {
                                const float v0 = d[u][4 * j + 2 * h], v1 = d[u][4 * j + 2 * h + 1];
                                if constexpr (kEpi == kEpiSwigluBwd) swiglu_bwd_pair<kF16>(*sw, row, col, v0, v1);
                                else if constexpr (kEpi == kEpiGeluFwd) gelu_fwd_pair<kF16>(*sw, row, col, v0, v1, b0, b1);
                                else gelu_bwd_pair<kF16>(*sw, row, col, v0, v1);
                            }
                        }
                    }
                }
            }
        } else {
#pragma unroll
            for (int u = 0; u < BN / kUnit; ++u) {
#pragma unroll
                for (int j = 0; j < kUnit / 8; ++j) {
                    const int col = nb * BN + u * kUnit + 8 * j + 2 * (lane & 3);
                    if (col < g.N) {
                        const float b0 = g.has_bias ? __ldg(g.bias + col) : 0.f;
                        const float b1 = (g.has_bias && col + 1 < g.N) ? __ldg(g.bias + col + 1) : 0.f;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int row = row0 + 8 * h;
                            if (row < g.M)
                                store_pair<kF16>(g, row, col, act_apply(d[u][4 * j + 2 * h] + b0, g.act), act_apply(d[u][4 * j + 2 * h + 1] + b1, g.act));
                        }
                    }
                }
            }
        }
    }
}

// The whole CTA: barrier setup, the producer warpgroup and the two consumers.  kEpiSwigluFwd pairs the B tile: W1 rows
// [n0, n0 + 128) from tmB into its first half and W2's from tmB2 into its second, n0 = 128 nb (tmB2 is unused otherwise).
template <int BN, int kStages, bool kAMN, bool kBMN, bool kF16, int kEpi>
__device__ __forceinline__ void gemm_cta(const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmB2, const GemmArgs &g,
                                         const EpiArgs *sw) {
    extern __shared__ char smem_raw[];
    // SWIZZLE_128B tiles must sit on 1024-byte boundaries
    char *tiles = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int kABytes = kBM * kBK * 2, kBBytes = BN * kBK * 2, kStageBytes = kABytes + kBBytes;
    uint64_t *full = reinterpret_cast<uint64_t *>(tiles + kStages * kStageBytes);
    uint64_t *empty = full + kStages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mia::mbar_init(full + s, 1); mia::mbar_init(empty + s, 2); }   // one arrival per consumer warpgroup
        mia::fence_mbar_init();
    }
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    if (wg == 0) {
        // ===== TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
            const int num_tiles = g.num_m_blocks * g.num_n_blocks, KB = g.num_k_blocks;
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int mb = tile % g.num_m_blocks, nb = tile / g.num_m_blocks;     // m fastest: a column of W stays in L2
                for (int kb = 0; kb < KB; ++kb) {
                    mia::mbar_wait(empty + s, ph ^ 1);
                    mia::mbar_arrive_expect_tx(full + s, kStageBytes);
                    char *sa = tiles + s * kStageBytes, *sb = sa + kABytes;
                    if (kAMN) {
#pragma unroll
                        for (int i = 0; i < kBM / 64; ++i) tma_load_2d(sa + i * 8192, &tmA, mb * kBM + 64 * i, kb * kBK, full + s);
                    } else {
                        tma_load_2d(sa, &tmA, kb * kBK, mb * kBM, full + s);
                    }
                    if constexpr (kEpi == kEpiSwigluFwd) {
                        tma_load_2d(sb, &tmB, kb * kBK, nb * (BN / 2), full + s);
                        tma_load_2d(sb + (BN / 2) * kBK * 2, &tmB2, kb * kBK, nb * (BN / 2), full + s);
                    } else if (kBMN) {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i) tma_load_2d(sb + i * 8192, &tmB, nb * BN + 64 * i, kb * kBK, full + s);
                    } else {
                        tma_load_2d(sb, &tmB, kb * kBK, nb * BN, full + s);
                    }
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        gemm_consumer<BN, kStages, kAMN, kBMN, kF16, kEpi>(g, tiles, full, empty, wg - 1, sw);
    }
}

template <int BN, int kStages, bool kAMN, bool kBMN, bool kF16>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                  const GemmArgs g) {
    gemm_cta<BN, kStages, kAMN, kBMN, kF16, kEpiLinear>(tmA, tmB, tmB, g, nullptr);
}

// SwiGLU forward (kEpiSwigluFwd: A = x, tmB / tmB2 = W1 / W2, K-major) and backward (kEpiSwigluBwd: A = dy, tmB = W3 read
// MN-major, tmB2 unused).
template <int kEpi, int BN, int kStages, bool kBMN, bool kF16>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_swiglu_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                      const __grid_constant__ CUtensorMap tmB2, const GemmArgs g, const EpiArgs sw) {
    gemm_cta<BN, kStages, false, kBMN, kF16, kEpi>(tmA, tmB, tmB2, g, &sw);
}

// GELU MLP's fc1 (kEpiGeluFwd: A = x, tmB = W1, K-major) and fc2 dgrad (kEpiGeluBwd: A = dy, tmB = W2 read MN-major); the
// same parameters as gemm_swiglu_kernel so that one launcher serves both (tmB2 unused).
template <int kEpi, int BN, int kStages, bool kBMN, bool kF16>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_gelu_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                    const __grid_constant__ CUtensorMap tmB2, const GemmArgs g, const EpiArgs ep) {
    gemm_cta<BN, kStages, false, kBMN, kF16, kEpi>(tmA, tmB, tmB2, g, &ep);
}

// ---- host side -------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// 2-D map of a row-major [rows][cols] matrix with row pitch ld (elements); box = [box_rows][128 bytes of columns], 128B swizzle.
// dt: MIA_GEMM_F32 / F16 / BF16
int make_map(CUtensorMap *tm, const void *ptr, long long rows, long long cols, long long ld, int box_rows, int dt) {
    // rows x cols with cols contiguous; the box is [box_rows][128 bytes of columns]
    EncodeTiledFn fn = encode_fn();
    if (!fn) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const int es = dt == MIA_GEMM_F32 ? 4 : 2;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * es};
    cuuint32_t box[2] = {(cuuint32_t)(128 / es), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType cdt = dt == MIA_GEMM_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                                        : (dt == MIA_GEMM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    const CUresult r = fn(tm, cdt, 2, const_cast<void *>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "cuTensorMapEncodeTiled failed (CUresult %d): rows %lld cols %lld ld %lld", (int)r, rows, cols, ld);
    return MIA_GEMM_OK;
}

template <int BN, int kStages, bool kAMN, bool kBMN, bool kF16>
int launch_gemm(const CUtensorMap &tmA, const CUtensorMap &tmB, GemmArgs &g, int sms, cudaStream_t stream) {
    constexpr int smem = kStages * (kBM * kBK * 2 + BN * kBK * 2) + 2 * kStages * 8 + 1024;
    auto k = &gemm_tn_kernel<BN, kStages, kAMN, kBMN, kF16>;
    if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "cudaFuncSetAttribute(gemm, %d B): %s", smem, cudaGetErrorString(cudaGetLastError()));
    g.num_m_blocks = (g.M + kBM - 1) / kBM;
    g.num_n_blocks = (g.N + BN - 1) / BN;
    g.num_k_blocks = (g.K + kBK - 1) / kBK;
    const int tiles = g.num_m_blocks * g.num_n_blocks;
    const int grid = tiles < sms ? tiles : sms;
    k<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, g);
    return mia::launched(mia::kErrGemm, "gemm launch");
}

// The kernel of a fused-epilogue mode (taking only its address instantiates only it).
template <int kEpi, int BN, int kStages, bool kBMN, bool kF16>
constexpr auto epi_kernel() {
    if constexpr (kEpi == kEpiGeluFwd || kEpi == kEpiGeluBwd) return &gemm_gelu_kernel<kEpi, BN, kStages, kBMN, kF16>;
    else return &gemm_swiglu_kernel<kEpi, BN, kStages, kBMN, kF16>;
}

// Launch of a fused-epilogue kernel.  g.N is the hidden width H; a paired-B tile (SwiGLU forward) spans BN / 2 hidden
// columns, every other tile BN.
template <int kEpi, int BN, int kStages, bool kBMN, bool kF16>
int launch_epi(const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmB2, GemmArgs &g, const EpiArgs &ep, int sms,
               cudaStream_t stream) {
    constexpr int smem = kStages * (kBM * kBK * 2 + BN * kBK * 2) + 2 * kStages * 8 + 1024;
    constexpr int span = kEpi == kEpiSwigluFwd ? BN / 2 : BN;
    constexpr bool gelu = kEpi == kEpiGeluFwd || kEpi == kEpiGeluBwd;
    auto k = epi_kernel<kEpi, BN, kStages, kBMN, kF16>();
    const char *name = gelu ? "gemm_gelu" : "gemm_swiglu";
    if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "cudaFuncSetAttribute(%s, %d B): %s", name, smem, cudaGetErrorString(cudaGetLastError()));
    g.num_m_blocks = (g.M + kBM - 1) / kBM;
    g.num_n_blocks = (g.N + span - 1) / span;
    g.num_k_blocks = (g.K + kBK - 1) / kBK;
    const int tiles = g.num_m_blocks * g.num_n_blocks;
    const int grid = tiles < sms ? tiles : sms;
    k<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, tmB2, g, ep);
    return mia::launched(mia::kErrGemm, gelu ? "gemm_gelu launch" : "gemm_swiglu launch");
}

long long swiglu_pad(int H) { return ((long long)H + 63) / 64 * 64; }
long long gelu_pad(int H) { return ((long long)H + 7) / 8 * 8; }

}  // namespace

static int gemm_impl(const void *A, const void *W, const float *bias, void *C, int M, int N, int K, long long lda, long long ldw, long long ldc,
                     int a_mn, int b_mn, int in_dtype, int out_dtype, int act, void *cuda_stream) {
    if (!A || !W || !C) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: null pointer");
    if (M <= 0 || N <= 0 || K <= 0) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: empty or negative size (M %d, N %d, K %d)", M, N, K);
    if (in_dtype != MIA_GEMM_BF16 && in_dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: inputs must be bf16 or fp16");
    if (out_dtype != in_dtype && out_dtype != MIA_GEMM_F32) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: output must be the input dtype or fp32");
    if (act < 0 || act > MIA_ACT_SILU) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: unknown activation %d", act);
    if ((lda % 8) || (ldw % 8) || lda < (a_mn ? M : K) || ldw < (b_mn ? N : K))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: row pitches must cover a row and be multiples of 8 elements (lda %lld, ldw %lld, M %d, N %d, K %d)", lda, ldw, M, N, K);
    if (((uintptr_t)A | (uintptr_t)W) & 15) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: A and W must be 16-byte aligned");
    if (ldc < N) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm: ldc < N");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "gemm: cannot query the device");
    const int sms = di.sms;
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = N; g.K = K; g.act = act; g.out_f32 = out_dtype == MIA_GEMM_F32; g.has_bias = bias != nullptr; g.bias = bias;
    g.in_f16 = in_dtype == MIA_GEMM_F16; g.C = C; g.ldc = ldc;
    const int BN = N <= 64 ? 64 : (N <= 128 || (long long)((M + 127) / 128) * ((N + 255) / 256) < sms ? 128 : 256);
    CUtensorMap tmA, tmB;
    // K-major operand: [rows = M or N][cols = K], box [tile rows][64 k];  MN-major operand: stored [rows = K][cols = M or N], box [64 k][64 mn]
    if (int rc = a_mn ? make_map(&tmA, A, K, M, lda, kBK, in_dtype) : make_map(&tmA, A, M, K, lda, kBM, in_dtype)) return rc;
    if (int rc = b_mn ? make_map(&tmB, W, K, N, ldw, kBK, in_dtype) : make_map(&tmB, W, N, K, ldw, BN, in_dtype)) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
#define MIA_GEMM_LAUNCH(AMN, BMN, F16)                                                     \
    switch (BN) {                                                                          \
        case 64: return launch_gemm<64, 8, AMN, BMN, F16>(tmA, tmB, g, sms, stream);       \
        case 128: return launch_gemm<128, 6, AMN, BMN, F16>(tmA, tmB, g, sms, stream);     \
        default: return launch_gemm<256, 4, AMN, BMN, F16>(tmA, tmB, g, sms, stream);      \
    }
#define MIA_GEMM_LAUNCH_T(AMN, BMN) \
    if (g.in_f16) { MIA_GEMM_LAUNCH(AMN, BMN, true) } else { MIA_GEMM_LAUNCH(AMN, BMN, false) }
    if (!a_mn && !b_mn) { MIA_GEMM_LAUNCH_T(false, false) }
    if (!a_mn && b_mn) { MIA_GEMM_LAUNCH_T(false, true) }
    if (a_mn && b_mn) { MIA_GEMM_LAUNCH_T(true, true) }
    MIA_GEMM_LAUNCH_T(true, false)
#undef MIA_GEMM_LAUNCH_T
#undef MIA_GEMM_LAUNCH
}

extern "C" {

int mia_gemm_tn(const void *A, const void *W, const float *bias, void *C, int M, int N, int K, long long lda, long long ldw, long long ldc,
                int in_dtype, int out_dtype, int act, void *cuda_stream) {
    return gemm_impl(A, W, bias, C, M, N, K, lda, ldw, ldc, 0, 0, in_dtype, out_dtype, act, cuda_stream);
}

int mia_gemm(const void *A, const void *B, const float *bias, void *C, int M, int N, int K, long long lda, long long ldb, long long ldc,
             int a_mn_major, int b_mn_major, int in_dtype, int out_dtype, int act, void *cuda_stream) {
    return gemm_impl(A, B, bias, C, M, N, K, lda, ldb, ldc, a_mn_major != 0, b_mn_major != 0, in_dtype, out_dtype, act, cuda_stream);
}

int mia_gemm_swiglu_fwd(const void *x, const void *w1, const void *w2, const float *b1, const float *b2, void *h, void *ab, int M, int H,
                        int K, long long ldx, long long ldw1, long long ldw2, long long ldh, long long ldab, int dtype, void *cuda_stream) {
    if (!x || !w1 || !w2 || !h) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: null pointer (x, w1, w2 and h are required)");
    if (M <= 0 || H <= 0 || K <= 0) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: empty or negative size (M %d, H %d, K %d)", M, H, K);
    if (dtype != MIA_GEMM_BF16 && dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: dtype must be bf16 or fp16");
    if ((ldx | ldw1 | ldw2 | ldh) % 8 || ldx < K || ldw1 < K || ldw2 < K || ldh < H)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: row pitches must cover a row and be multiples of 8 elements "
                         "(ldx %lld, ldw1 %lld, ldw2 %lld, ldh %lld, H %d, K %d)", ldx, ldw1, ldw2, ldh, H, K);
    const long long Hp = swiglu_pad(H);
    if (ab && (ldab % 8 || ldab < 2 * Hp))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: ldab must be a multiple of 8 and at least 2 Hp = %lld (ldab %lld)", 2 * Hp, ldab);
    if (((uintptr_t)x | (uintptr_t)w1 | (uintptr_t)w2 | (uintptr_t)h | (uintptr_t)ab) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_fwd: x, w1, w2, h and ab must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "gemm_swiglu_fwd: cannot query the device");
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = H; g.K = K; g.in_f16 = dtype == MIA_GEMM_F16;
    EpiArgs sw;
    memset(&sw, 0, sizeof(sw));
    sw.b1 = b1; sw.b2 = b2; sw.h = h; sw.ab = ab; sw.ldh = ldh; sw.ldab = ldab; sw.H = H; sw.Hp = (int)Hp;
    CUtensorMap tmA, tmB, tmB2;
    if (int rc = make_map(&tmA, x, M, K, ldx, kBM, dtype)) return rc;
    if (int rc = make_map(&tmB, w1, H, K, ldw1, 128, dtype)) return rc;
    if (int rc = make_map(&tmB2, w2, H, K, ldw2, 128, dtype)) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (g.in_f16) return launch_epi<kEpiSwigluFwd, 256, 4, false, true>(tmA, tmB, tmB2, g, sw, di.sms, stream);
    return launch_epi<kEpiSwigluFwd, 256, 4, false, false>(tmA, tmB, tmB2, g, sw, di.sms, stream);
}

int mia_gemm_swiglu_bwd(const void *dy, const void *w3, const void *ab, void *dab, void *h, int M, int H, int N_out, long long lddy,
                        long long ldw3, long long ldab, long long lddab, long long ldh, int dtype, void *cuda_stream) {
    if (!dy || !w3 || !ab || !dab) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: null pointer (dy, w3, ab and dab are required)");
    if (M <= 0 || H <= 0 || N_out <= 0)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: empty or negative size (M %d, H %d, N_out %d)", M, H, N_out);
    if (dtype != MIA_GEMM_BF16 && dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: dtype must be bf16 or fp16");
    if ((lddy | ldw3) % 8 || (h && ldh % 8) || lddy < N_out || ldw3 < H || (h && ldh < H))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: row pitches must cover a row and be multiples of 8 elements "
                         "(lddy %lld, ldw3 %lld, ldh %lld, H %d, N_out %d)", lddy, ldw3, ldh, H, N_out);
    const long long Hp = swiglu_pad(H);
    if ((ldab | lddab) % 8 || ldab < 2 * Hp || lddab < 2 * Hp)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: ldab and lddab must be multiples of 8 and at least 2 Hp = %lld "
                         "(ldab %lld, lddab %lld)", 2 * Hp, ldab, lddab);
    if (((uintptr_t)dy | (uintptr_t)w3 | (uintptr_t)ab | (uintptr_t)dab | (uintptr_t)h) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_swiglu_bwd: dy, w3, ab, dab and h must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "gemm_swiglu_bwd: cannot query the device");
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = H; g.K = N_out; g.in_f16 = dtype == MIA_GEMM_F16;
    EpiArgs sw;
    memset(&sw, 0, sizeof(sw));
    sw.h = h; sw.ab = const_cast<void *>(ab); sw.dab = dab; sw.ldh = ldh; sw.ldab = ldab; sw.lddab = lddab; sw.H = H; sw.Hp = (int)Hp;
    // g = dy . W3: dy [M][N_out] K-major; W3 [N_out][H] read MN-major (rows = k), as LinearTC's dgrad reads it
    CUtensorMap tmA, tmB;
    if (int rc = make_map(&tmA, dy, M, N_out, lddy, kBM, dtype)) return rc;
    if (int rc = make_map(&tmB, w3, N_out, H, ldw3, kBK, dtype)) return rc;
    const bool wide = H > 128 && (long long)((M + 127) / 128) * ((H + 255) / 256) >= di.sms;      // gemm_impl's choice between 128 and 256
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (g.in_f16) {
        if (wide) return launch_epi<kEpiSwigluBwd, 256, 4, true, true>(tmA, tmB, tmB, g, sw, di.sms, stream);
        return launch_epi<kEpiSwigluBwd, 128, 6, true, true>(tmA, tmB, tmB, g, sw, di.sms, stream);
    }
    if (wide) return launch_epi<kEpiSwigluBwd, 256, 4, true, false>(tmA, tmB, tmB, g, sw, di.sms, stream);
    return launch_epi<kEpiSwigluBwd, 128, 6, true, false>(tmA, tmB, tmB, g, sw, di.sms, stream);
}

int mia_gemm_gelu_fwd(const void *x, const void *w1, const float *b1, void *h, void *pre, int M, int H, int K, long long ldx, long long ldw1,
                      long long ldh, long long ldpre, int dtype, void *cuda_stream) {
    if (!x || !w1 || !h) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_fwd: null pointer (x, w1 and h are required)");
    if (M <= 0 || H <= 0 || K <= 0) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_fwd: empty or negative size (M %d, H %d, K %d)", M, H, K);
    if (dtype != MIA_GEMM_BF16 && dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_fwd: dtype must be bf16 or fp16");
    if ((ldx | ldw1 | ldh) % 8 || (pre && ldpre % 8) || ldx < K || ldw1 < K || ldh < H || (pre && ldpre < H))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_fwd: row pitches must cover a row and be multiples of 8 elements "
                         "(ldx %lld, ldw1 %lld, ldh %lld, ldpre %lld, H %d, K %d)", ldx, ldw1, ldh, ldpre, H, K);
    if (((uintptr_t)x | (uintptr_t)w1 | (uintptr_t)h | (uintptr_t)pre) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_fwd: x, w1, h and pre must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "gemm_gelu_fwd: cannot query the device");
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = H; g.K = K; g.in_f16 = dtype == MIA_GEMM_F16;
    EpiArgs ep;
    memset(&ep, 0, sizeof(ep));
    ep.b1 = b1; ep.h = h; ep.ab = pre; ep.ldh = ldh; ep.ldab = ldpre; ep.H = H; ep.Hp = (int)gelu_pad(H);
    // gemm_impl's tile width for N = H, so pre has mia_gemm_tn's k order
    const int BN = H <= 64 ? 64 : (H <= 128 || (long long)((M + 127) / 128) * ((H + 255) / 256) < di.sms ? 128 : 256);
    CUtensorMap tmA, tmB;
    if (int rc = make_map(&tmA, x, M, K, ldx, kBM, dtype)) return rc;
    if (int rc = make_map(&tmB, w1, H, K, ldw1, BN, dtype)) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
#define MIA_GELU_FWD(F16)                                                                                       \
    switch (BN) {                                                                                               \
        case 64: return launch_epi<kEpiGeluFwd, 64, 8, false, F16>(tmA, tmB, tmB, g, ep, di.sms, stream);       \
        case 128: return launch_epi<kEpiGeluFwd, 128, 6, false, F16>(tmA, tmB, tmB, g, ep, di.sms, stream);     \
        default: return launch_epi<kEpiGeluFwd, 256, 4, false, F16>(tmA, tmB, tmB, g, ep, di.sms, stream);      \
    }
    if (g.in_f16) { MIA_GELU_FWD(true) }
    MIA_GELU_FWD(false)
#undef MIA_GELU_FWD
}

int mia_gemm_gelu_bwd(const void *dy, const void *w2, const void *pre, void *dpre, void *h, int M, int H, int N_out, long long lddy,
                      long long ldw2, long long ldpre, long long lddpre, long long ldh, int dtype, void *cuda_stream) {
    if (!dy || !w2 || !pre || !dpre) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_bwd: null pointer (dy, w2, pre and dpre are required)");
    if (M <= 0 || H <= 0 || N_out <= 0)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_bwd: empty or negative size (M %d, H %d, N_out %d)", M, H, N_out);
    if (dtype != MIA_GEMM_BF16 && dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_bwd: dtype must be bf16 or fp16");
    if ((lddy | ldw2 | ldpre | lddpre) % 8 || (h && ldh % 8) || lddy < N_out || ldw2 < H || ldpre < H || lddpre < H || (h && ldh < H))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_bwd: row pitches must cover a row and be multiples of 8 elements "
                         "(lddy %lld, ldw2 %lld, ldpre %lld, lddpre %lld, ldh %lld, H %d, N_out %d)", lddy, ldw2, ldpre, lddpre, ldh, H, N_out);
    if (((uintptr_t)dy | (uintptr_t)w2 | (uintptr_t)pre | (uintptr_t)dpre | (uintptr_t)h) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "gemm_gelu_bwd: dy, w2, pre, dpre and h must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "gemm_gelu_bwd: cannot query the device");
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = H; g.K = N_out; g.in_f16 = dtype == MIA_GEMM_F16;
    EpiArgs ep;
    memset(&ep, 0, sizeof(ep));
    ep.h = h; ep.ab = const_cast<void *>(pre); ep.dab = dpre; ep.ldh = ldh; ep.ldab = ldpre; ep.lddab = lddpre; ep.H = H; ep.Hp = (int)gelu_pad(H);
    // g = dy . W2: dy [M][N_out] K-major; W2 [N_out][H] read MN-major (rows = k), as LinearTC's dgrad reads it
    CUtensorMap tmA, tmB;
    if (int rc = make_map(&tmA, dy, M, N_out, lddy, kBM, dtype)) return rc;
    if (int rc = make_map(&tmB, w2, N_out, H, ldw2, kBK, dtype)) return rc;
    const bool wide = H > 128 && (long long)((M + 127) / 128) * ((H + 255) / 256) >= di.sms;      // gemm_impl's choice between 128 and 256
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (g.in_f16) {
        if (wide) return launch_epi<kEpiGeluBwd, 256, 4, true, true>(tmA, tmB, tmB, g, ep, di.sms, stream);
        return launch_epi<kEpiGeluBwd, 128, 6, true, true>(tmA, tmB, tmB, g, ep, di.sms, stream);
    }
    if (wide) return launch_epi<kEpiGeluBwd, 256, 4, true, false>(tmA, tmB, tmB, g, ep, di.sms, stream);
    return launch_epi<kEpiGeluBwd, 128, 6, true, false>(tmA, tmB, tmB, g, ep, di.sms, stream);
}

}  // extern "C"
