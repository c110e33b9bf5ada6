// ViT-MAE attention, softmax(q k^T dh^-0.5) v per (image, head), on wgmma + TMA (sm_90a).  Mirrors the
// F.scaled_dot_product_attention of timm 0.9.2's Attention (HD_Xray_Pretrain_MAE/pretrain/models/mae.py:64-66, 82-84).
//
// Layout: q / k / v are read in place from the qkv GEMM's output, (B, N, 3, H, dh) with row pitch ld_qkv, through a 3-D
// tensor map (3C, N, B): TMA zero-fills rows past token N - 1 of each image, which in memory are the next image's tokens.
// A [64 rows x dh] tile is staged as dh / 8 boxes of [64 rows x 8 elements] without swizzle, so every head dim that is a
// multiple of 16 (32, 64, 80) uses one layout: 8 x 16-byte core matrices of 128 contiguous bytes, 8-column slices 1024
// bytes apart.  The same tile is a K-major operand (S = Q K^T) and an MN-major one (O += P V).
//
// Every CTA is one consumer warpgroup (64 rows, fp32 accumulators in registers) plus one producer warp whose lane 0
// issues the TMA loads into a ring of kStages stages (full / empty mbarriers).  Tiles of keys are 64 wide.
//   attn_fwd_kernel     CTA = (64 queries, head, image).  Per key tile: S = Q K^T, online softmax in fp32 in the log2
//                       domain (p = exp2(s dh^-0.5 log2e - m)), P rounded to the input dtype, O += P V.  O / l is rounded
//                       once and written token-major (B, N, C); lse = (m + log2 l) ln2 in fp32 (B, H, N).
//   attn_bwd_dq_kernel  CTA = (64 queries, head, image).  delta = rowsum(dO o O) in fp32 (stored for the next launch),
//                       then per key tile: S, P = exp2(s dh^-0.5 log2e - lse log2e), dP = dO V^T, dS = P (dP - delta),
//                       dQ += dS K.  dq = round(dh^-0.5 dQ) into the packed dqkv.
//   attn_bwd_dkv_kernel CTA = (64 keys, head, image).  Per query tile: S^T = K Q^T, dP^T = V dO^T, P^T and dS^T as
//                       above, dV += P^T dO, dK += dS^T Q.  dk = round(dh^-0.5 dK), dv = round(dV).
// Key columns >= N are -inf (forward) / P = 0 (backward) before anything else sees them; rows >= N are never stored.  No
// atomics: every output element is summed in a fixed order, so results are bit-reproducible.
//
// Cross-attention (kX = true; the ARM pre-training decoder's CrossAttention, CXPMRG_Bench_MambaXray_VL/pretrain/
// models_pretrain.py:55-83, 395-400): q is the q GEMM's output (B, N, C) read through its own map (C, N, B), k / v the kv
// GEMM's output (B, N, 2C) through one map (2C, N, B) at columns h dh / C + h dh.  A segment-causal mask of segment length
// seg: key j is visible to query i iff j / seg <= i / seg, i.e. j < (i / seg + 1) seg.  Masked scores become -inf before
// the row max (a select, not an add) and P = 0 in the backward.  Key 0 is visible to every row, so the running max is
// finite after the first key tile and a later tile that a row cannot see adds exact zeros.  Tiles no row of a CTA can see
// are skipped: the forward / dq loops end at the key tile holding the last key visible to the CTA's last valid query row,
// and the dkv loop starts at the query tile holding the first query that sees the CTA's first key.  dq goes to (B, N, C)
// and dk / dv to a packed (B, N, 2C): the output gradients of the q and kv GEMMs.  Head dim 64 only.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "../../include/mia_gemm.h"
#include "abi_host.h"
#include "tma_host.h"
#include "wgmma.cuh"

namespace {

constexpr int kRows = 64;                 // rows of every tile: queries of a CTA, keys (forward / dq) or queries (dkv) per step
constexpr int kThreads = 160;             // consumer warpgroup + producer warp
constexpr int kStages = 2;
constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;

struct AttnArgs {
    int N, H, C;                          // C = H dh
    float scale, scale_log2;              // dh^-0.5 and dh^-0.5 log2(e)
    void *o;                              // forward: output; backward: input
    const void *dout;
    const float *lse;                     // backward input
    float *lse_out, *delta;               // forward output (may be NULL) / backward scratch
    void *dqkv;                           // self-attention: the packed dqkv; cross-attention: dq (B, N, C)
    long long ld_o, ld_do, ld_dqkv;
    void *dkv;                            // cross-attention: the packed (B, N, 2C) dk / dv
    long long ld_dkv;
    int seg;                              // cross-attention: segment length of the mask
};

// The tensor maps of a launch: self-attention reads q / k / v from one map (3C, N, B) at columns h dh, C + h dh, 2C + h dh;
// cross-attention reads q from m[0] (C, N, B) at h dh and k / v from m[1] (2C, N, B) at h dh, C + h dh.
template <bool kX>
struct Maps {
    CUtensorMap m[kX ? 2 : 1];
};
template <bool kX>
__device__ __forceinline__ const CUtensorMap *map_kv(const Maps<kX> &tm) { return &tm.m[kX ? 1 : 0]; }
template <bool kX, int DH>
__device__ __forceinline__ int col_k(const AttnArgs &a, int head) { return (kX ? 0 : a.C) + head * DH; }
template <bool kX, int DH>
__device__ __forceinline__ int col_v(const AttnArgs &a, int head) { return (kX ? a.C : 2 * a.C) + head * DH; }

// One past the last key visible to query i under the segment-causal mask, capped at N.
__device__ __forceinline__ int seg_end(int i, int seg, int N) { return min(N, (i / seg + 1) * seg); }

// Key tiles a CTA of query tile qt visits: all of them, or (kX) up to the one holding the last key its last valid row sees.
template <bool kX>
__device__ __forceinline__ int key_steps(const AttnArgs &a, int qt) {
    if (!kX) return (a.N + kRows - 1) / kRows;
    return (seg_end(min(a.N, (qt + 1) * kRows) - 1, a.seg, a.N) + kRows - 1) / kRows;
}

// d[64 x N fragment] += A[registers, 64 x 16] . B[smem desc, 16 x N], B MN-major (its N index contiguous).  A fragment of
// thread t: a[0] = (row g, k 2q..2q+1), a[1] = (g + 8, same k), a[2] = (g, 2q + 8..), a[3] = (g + 8, 2q + 8..), with
// row g = 16 (t / 32) + (t % 32) / 4 and q = t % 4: the accumulator fragment of S, rounded pairwise.
#define MIA_WGMMA_RS_N32(TYPE) \
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32." TYPE "." TYPE " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, 1, 1, 1, 1;" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b) : "memory")
#define MIA_WGMMA_RS_N64(TYPE) \
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, 1, 1, 1, 1;" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b) : "memory")
#define MIA_WGMMA_RS_N80(TYPE) \
    asm volatile("wgmma.mma_async.sync.aligned.m64n80k16.f32." TYPE "." TYPE " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, {%40,%41,%42,%43}, %44, 1, 1, 1, 1;" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]) \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b) : "memory")

template <bool kF16, int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc_b) {
    if constexpr (N == 32) { if (kF16) MIA_WGMMA_RS_N32("f16"); else MIA_WGMMA_RS_N32("bf16"); }
    else if constexpr (N == 64) { if (kF16) MIA_WGMMA_RS_N64("f16"); else MIA_WGMMA_RS_N64("bf16"); }
    else { static_assert(N == 80, "head dims 32, 64, 80"); if (kF16) MIA_WGMMA_RS_N80("f16"); else MIA_WGMMA_RS_N80("bf16"); }
}

// Descriptors of a staged [64 x DH] tile at smem address `base`, for the 16-wide step kk of the contraction: K-major when the
// contraction runs over DH (core matrices along DH 1024 bytes apart, 8-row groups 128), MN-major when it runs over the rows
// (8-row groups 128 bytes apart, 8-column slices 1024).
__device__ __forceinline__ uint64_t desc_k(uint32_t base, int kk) { return mia::wgmma_desc_plain(base + kk * 2048, 1024, 128); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t base, int kk) { return mia::wgmma_desc_plain(base + kk * 256, 128, 1024); }

// One [64 rows x DH] tile of a 3-D map (columns, tokens, images): DH / 8 boxes of [64 x 8], each 1024 contiguous bytes.
template <int DH>
__device__ __forceinline__ void load_tile(char *dst, const CUtensorMap *tm, int col, int row, int b, uint64_t *bar) {
#pragma unroll
    for (int c = 0; c < DH / 8; ++c) mia::tma_load_3d(dst + c * 1024, tm, col + 8 * c, row, b, bar);
}

template <bool kF16>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    if (kF16) { __half2 h = __floats2half2_rn(lo, hi); return *reinterpret_cast<uint32_t *>(&h); }
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}
template <bool kF16>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
    if (kF16) return __half22float2(*reinterpret_cast<const __half2 *>(&w));
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&w));
}

// The [64 x 64] fp32 fragment v as four A fragments of a 64 x 16 x N product (k = the fragment's columns), rounded.
template <bool kF16>
__device__ __forceinline__ void to_a_frags(const float (&v)[32], uint32_t (&a)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        a[kk][0] = pack2<kF16>(v[8 * kk + 0], v[8 * kk + 1]);
        a[kk][1] = pack2<kF16>(v[8 * kk + 2], v[8 * kk + 3]);
        a[kk][2] = pack2<kF16>(v[8 * kk + 4], v[8 * kk + 5]);
        a[kk][3] = pack2<kF16>(v[8 * kk + 6], v[8 * kk + 7]);
    }
}

// acc (64 x DH fragment) scaled by `scale`, rounded and stored at rows row0 + r < N, columns col0 + [0, DH) of a token-major
// (B, N, *) tensor of pitch ld, image b.
template <int DH, bool kF16>
__device__ __forceinline__ void store_rows(void *base, long long ld, int b, int N, int row0, int col0, const float (&acc)[DH / 2], float scale) {
    const int t = threadIdx.x, r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = col0 + 2 * (t & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (r + 8 * h >= N) continue;
        uint16_t *dst = reinterpret_cast<uint16_t *>(base) + ((size_t)b * N + r + 8 * h) * ld + c;
#pragma unroll
        for (int j = 0; j < DH / 8; ++j)
            *reinterpret_cast<uint32_t *>(dst + 8 * j) = pack2<kF16>(acc[4 * j + 2 * h] * scale, acc[4 * j + 2 * h + 1] * scale);
    }
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// Shared memory: `fixed` tiles loaded once, then kStages stages of two tiles each, then the barriers (one for the fixed
// tiles, full[kStages], empty[kStages]).
template <int DH>
constexpr int smem_bytes(int fixed) { return (fixed + 2 * kStages) * kRows * DH * 2 + (1 + 2 * kStages) * 8 + 128; }

struct Ring {
    char *fixed, *stages;
    uint64_t *fbar, *full, *empty;
};

template <int DH>
__device__ __forceinline__ Ring setup_ring(int fixed) {
    extern __shared__ char smem_raw[];
    constexpr int kTile = kRows * DH * 2;
    Ring r;
    r.fixed = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    r.stages = r.fixed + fixed * kTile;
    r.fbar = reinterpret_cast<uint64_t *>(r.stages + 2 * kStages * kTile);
    r.full = r.fbar + 1;
    r.empty = r.full + kStages;
    if (threadIdx.x == 0) {
        mia::mbar_init(r.fbar, 1);
        for (int s = 0; s < kStages; ++s) { mia::mbar_init(r.full + s, 1); mia::mbar_init(r.empty + s, 1); }
        mia::fence_mbar_init();
    }
    __syncthreads();
    return r;
}

// The producer (lane 0 of warp 4): the two fixed tiles (columns fcol0 / fcol1 of maps fm0 / fm1, rows frow), then for
// each of the row tiles [first, steps) the pair (columns scol0 of sm0, scol1 of sm1).
template <int DH>
__device__ __forceinline__ void produce(const Ring &r, const CUtensorMap *fm0, int fcol0, const CUtensorMap *fm1, int fcol1, int frow, int nfixed,
                                        const CUtensorMap *sm0, int scol0, const CUtensorMap *sm1, int scol1, int first, int steps, int b) {
    constexpr int kTile = kRows * DH * 2;
    asm volatile("prefetch.tensormap [%0];" ::"l"(fm0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(sm1) : "memory");
    mia::mbar_arrive_expect_tx(r.fbar, nfixed * kTile);
    load_tile<DH>(r.fixed, fm0, fcol0, frow, b, r.fbar);
    if (nfixed == 2) load_tile<DH>(r.fixed + kTile, fm1, fcol1, frow, b, r.fbar);
    int s = 0;
    uint32_t ph = 0;
    for (int i = first; i < steps; ++i) {
        mia::mbar_wait(r.empty + s, ph ^ 1);
        mia::mbar_arrive_expect_tx(r.full + s, 2 * kTile);
        char *st = r.stages + s * 2 * kTile;
        load_tile<DH>(st, sm0, scol0, i * kRows, b, r.full + s);
        load_tile<DH>(st + kTile, sm1, scol1, i * kRows, b, r.full + s);
        if (++s == kStages) { s = 0; ph ^= 1; }
    }
}

template <int DH, bool kF16, bool kX>
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(const __grid_constant__ Maps<kX> tm, const AttnArgs a) {
    constexpr int kTile = kRows * DH * 2;
    const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z, N = a.N;
    const int steps = key_steps<kX>(a, qt);
    const Ring r = setup_ring<DH>(1);
    if (threadIdx.x >= 128) {
        if (threadIdx.x == 128)
            produce<DH>(r, &tm.m[0], head * DH, &tm.m[0], 0, qt * kRows, 1, map_kv(tm), col_k<kX, DH>(a, head), map_kv(tm), col_v<kX, DH>(a, head), 0, steps, b);
        return;
    }
    const int t = threadIdx.x, q = t & 3;
    int lim[2], lim0 = 0;                     // kX: one past the last visible key of rows rl, rl + 8, and of the CTA's first row
    if constexpr (kX) {
        const int row = qt * kRows + 16 * (t >> 5) + ((t & 31) >> 2);
        lim[0] = seg_end(row, a.seg, N);
        lim[1] = seg_end(row + 8, a.seg, N);
        lim0 = seg_end(qt * kRows, a.seg, N);
    }
    float o[DH / 2], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
    const uint32_t aq = mia::smem_u32(r.fixed);
    mia::mbar_wait(r.fbar, 0);
    int s = 0;
    uint32_t ph = 0;
    for (int kt = 0; kt < steps; ++kt) {
        mia::mbar_wait(r.full + s, ph);
        const uint32_t ak = mia::smem_u32(r.stages + s * 2 * kTile), av = ak + kTile;
        float sc[32];
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) mia::wgmma_n64<kF16, false, false>(sc, desc_k(aq, kk), desc_k(ak, kk), kk);
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
        if constexpr (kX) {
            if ((kt + 1) * kRows > lim0) {        // keys a row cannot see (including those past N)
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int c = 0; c < 2; ++c)
                            if (kt * kRows + 8 * j + 2 * q + c >= lim[h]) sc[4 * j + 2 * h + c] = -INFINITY;
            }
        } else if ((kt + 1) * kRows > N) {        // keys past N: zero-filled rows that would still score 0
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c)
                    if (kt * kRows + 8 * j + 2 * q + c >= N) sc[4 * j + c] = sc[4 * j + 2 + c] = -INFINITY;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float mn = fmaxf(m[h], mx * a.scale_log2), alpha = exp2f(m[h] - mn);
            m[h] = mn;
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float p = exp2f(fmaf(sc[4 * j + 2 * h + c], a.scale_log2, -mn));
                    sc[4 * j + 2 * h + c] = p;
                    sum += p;
                }
            l[h] = l[h] * alpha + sum;
#pragma unroll
            for (int j = 0; j < DH / 8; ++j) { o[4 * j + 2 * h] *= alpha; o[4 * j + 2 * h + 1] *= alpha; }
        }
        uint32_t pa[4][4];
        to_a_frags<kF16>(sc, pa);
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<kF16, DH>(o, pa[kk], desc_mn(av, kk));
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
        if (t == 0) mia::mbar_arrive(r.empty + s);
        if (++s == kStages) { s = 0; ph ^= 1; }
    }
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        inv[h] = 1.f / l[h];
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) { o[4 * j + 2 * h] *= inv[h]; o[4 * j + 2 * h + 1] *= inv[h]; }
    }
    store_rows<DH, kF16>(a.o, a.ld_o, b, N, qt * kRows, head * DH, o, 1.f);
    if (a.lse_out && q == 0) {
        const int row = qt * kRows + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
        for (int h = 0; h < 2; ++h)
            if (row + 8 * h < N) a.lse_out[((size_t)b * a.H + head) * N + row + 8 * h] = (m[h] + log2f(l[h])) * kLn2;
    }
}

// Per-row statistics of the rows [row0, row0 + 64) of (image b, head) into smem: lse log2(e) and delta = sum dO o O (fp32,
// the two halves of a row summed in one order); delta is also stored for the dk / dv launch.  Rows >= N get 0.
template <int DH, bool kF16>
__device__ __forceinline__ void row_stats(const AttnArgs &a, int b, int head, int row0, float *lse_s, float *delta_s) {
    const int t = threadIdx.x, rr = t >> 1, row = row0 + rr, half = t & 1;
    float part = 0.f;
    if (row < a.N) {
        const uint32_t *po = reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint16_t *>(a.o) + ((size_t)b * a.N + row) * a.ld_o + head * DH + half * (DH / 2));
        const uint32_t *pd = reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint16_t *>(a.dout) + ((size_t)b * a.N + row) * a.ld_do + head * DH + half * (DH / 2));
#pragma unroll
        for (int i = 0; i < DH / 4; ++i) {
            const float2 vo = unpack2<kF16>(__ldg(po + i)), vd = unpack2<kF16>(__ldg(pd + i));
            part = fmaf(vd.x, vo.x, part);
            part = fmaf(vd.y, vo.y, part);
        }
    }
    const float lo = __shfl_sync(0xffffffffu, part, (t & 31) & ~1), hi = __shfl_sync(0xffffffffu, part, (t & 31) | 1);
    if (half == 0) {
        const size_t i = ((size_t)b * a.H + head) * a.N + row;
        delta_s[rr] = row < a.N ? lo + hi : 0.f;
        lse_s[rr] = row < a.N ? __ldg(a.lse + i) * kLog2e : 0.f;
        if (row < a.N) a.delta[i] = lo + hi;
    }
}

template <int DH, bool kF16, bool kX>
__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(const __grid_constant__ Maps<kX> tm, const __grid_constant__ CUtensorMap tm_do,
                                                             const AttnArgs a) {
    constexpr int kTile = kRows * DH * 2;
    __shared__ float lse_s[kRows], delta_s[kRows];
    const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z, N = a.N;
    const int steps = key_steps<kX>(a, qt);
    const Ring r = setup_ring<DH>(2);
    if (threadIdx.x >= 128) {
        if (threadIdx.x == 128)
            produce<DH>(r, &tm.m[0], head * DH, &tm_do, head * DH, qt * kRows, 2, map_kv(tm), col_k<kX, DH>(a, head), map_kv(tm), col_v<kX, DH>(a, head), 0,
                        steps, b);
        return;
    }
    const int t = threadIdx.x, q = t & 3, rl = 16 * (t >> 5) + ((t & 31) >> 2);
    row_stats<DH, kF16>(a, b, head, qt * kRows, lse_s, delta_s);
    consumer_sync();
    const float lse2[2] = {lse_s[rl], lse_s[rl + 8]}, dlt[2] = {delta_s[rl], delta_s[rl + 8]};
    // one past the last visible key of rows rl, rl + 8
    const int lim[2] = {kX ? seg_end(qt * kRows + rl, a.seg, N) : N, kX ? seg_end(qt * kRows + rl + 8, a.seg, N) : N};
    float dq[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) dq[i] = 0.f;
    const uint32_t aq = mia::smem_u32(r.fixed), ado = aq + kTile;
    mia::mbar_wait(r.fbar, 0);
    int s = 0;
    uint32_t ph = 0;
    for (int kt = 0; kt < steps; ++kt) {
        mia::mbar_wait(r.full + s, ph);
        const uint32_t ak = mia::smem_u32(r.stages + s * 2 * kTile), av = ak + kTile;
        float sc[32], dp[32];
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) mia::wgmma_n64<kF16, false, false>(sc, desc_k(aq, kk), desc_k(ak, kk), kk);
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) mia::wgmma_n64<kF16, false, false>(dp, desc_k(ado, kk), desc_k(av, kk), kk);
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int i = 4 * j + 2 * h + c;
                    const float p = kt * kRows + 8 * j + 2 * q + c < lim[h] ? exp2f(fmaf(sc[i], a.scale_log2, -lse2[h])) : 0.f;
                    sc[i] = p * (dp[i] - dlt[h]);
                }
        uint32_t da[4][4];
        to_a_frags<kF16>(sc, da);
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<kF16, DH>(dq, da[kk], desc_mn(ak, kk));
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
        if (t == 0) mia::mbar_arrive(r.empty + s);
        if (++s == kStages) { s = 0; ph ^= 1; }
    }
    store_rows<DH, kF16>(a.dqkv, a.ld_dqkv, b, N, qt * kRows, head * DH, dq, a.scale);
}

template <int DH, bool kF16, bool kX>
__global__ void __launch_bounds__(kThreads) attn_bwd_dkv_kernel(const __grid_constant__ Maps<kX> tm, const __grid_constant__ CUtensorMap tm_do,
                                                              const AttnArgs a) {
    constexpr int kTile = kRows * DH * 2;
    const int kt = blockIdx.x, head = blockIdx.y, b = blockIdx.z, N = a.N;
    const int steps = (N + kRows - 1) / kRows;
    const int first = kX ? kt * kRows / a.seg * a.seg / kRows : 0;     // kX: the query tile of the first query that sees key kt 64
    const Ring r = setup_ring<DH>(2);
    if (threadIdx.x >= 128) {
        if (threadIdx.x == 128)
            produce<DH>(r, map_kv(tm), col_k<kX, DH>(a, head), map_kv(tm), col_v<kX, DH>(a, head), kt * kRows, 2, &tm.m[0], head * DH, &tm_do, head * DH,
                        first, steps, b);
        return;
    }
    const int t = threadIdx.x, q = t & 3;
    int lo[2] = {0, 0};                       // kX: the first query that sees key rows rl, rl + 8
    if constexpr (kX) {
        const int key = kt * kRows + 16 * (t >> 5) + ((t & 31) >> 2);
        lo[0] = key / a.seg * a.seg;
        lo[1] = (key + 8) / a.seg * a.seg;
    }
    const float *lse = a.lse + ((size_t)b * a.H + head) * N, *delta = a.delta + ((size_t)b * a.H + head) * N;
    float dk[DH / 2], dv[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) dk[i] = dv[i] = 0.f;
    const uint32_t ak = mia::smem_u32(r.fixed), av = ak + kTile;
    mia::mbar_wait(r.fbar, 0);
    int s = 0;
    uint32_t ph = 0;
    for (int it = first; it < steps; ++it) {
        mia::mbar_wait(r.full + s, ph);
        const uint32_t aq = mia::smem_u32(r.stages + s * 2 * kTile), ado = aq + kTile;
        float sc[32], dp[32];
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) mia::wgmma_n64<kF16, false, false>(sc, desc_k(ak, kk), desc_k(aq, kk), kk);
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) mia::wgmma_n64<kF16, false, false>(dp, desc_k(av, kk), desc_k(ado, kk), kk);
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int col = it * kRows + 8 * j + 2 * q + c;
                const bool in = col < N;
                const float lse2 = in ? __ldg(lse + col) * kLog2e : 0.f, dlt = in ? __ldg(delta + col) : 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = 4 * j + 2 * h + c;
                    const float p = in && (!kX || col >= lo[h]) ? exp2f(fmaf(sc[i], a.scale_log2, -lse2)) : 0.f;
                    sc[i] = p;
                    dp[i] = p * (dp[i] - dlt);
                }
            }
        uint32_t pa[4][4], da[4][4];
        to_a_frags<kF16>(sc, pa);
        to_a_frags<kF16>(dp, da);
        mia::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<kF16, DH>(dv, pa[kk], desc_mn(ado, kk));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<kF16, DH>(dk, da[kk], desc_mn(aq, kk));
        mia::wgmma_commit();
        mia::wgmma_wait<0>();
        if (t == 0) mia::mbar_arrive(r.empty + s);
        if (++s == kStages) { s = 0; ph ^= 1; }
    }
    if constexpr (kX) {
        store_rows<DH, kF16>(a.dkv, a.ld_dkv, b, N, kt * kRows, head * DH, dk, a.scale);
        store_rows<DH, kF16>(a.dkv, a.ld_dkv, b, N, kt * kRows, a.C + head * DH, dv, 1.f);
    } else {
        store_rows<DH, kF16>(a.dqkv, a.ld_dqkv, b, N, kt * kRows, a.C + head * DH, dk, a.scale);
        store_rows<DH, kF16>(a.dqkv, a.ld_dqkv, b, N, kt * kRows, 2 * a.C + head * DH, dv, 1.f);
    }
}

// ---- host side -------------------------------------------------------------------------------------------------
// 3-D map (cols, N, B) of a token-major (B, N, cols) tensor with row pitch ld: box [1 image][64 tokens][8 elements], no
// swizzle; tokens past N of an image are zero-filled.
int make_map3(CUtensorMap *tm, const void *ptr, long long cols, int N, int B, long long ld, int dtype, const char *what) {
    mia::EncodeTiledFn fn = mia::tma_encode_fn();
    if (!fn) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "%s: cuTensorMapEncodeTiled is not available from this driver", what);
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)N, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * N};
    cuuint32_t box[3] = {8, kRows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUresult rc = fn(tm, dtype == MIA_GEMM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(ptr), dims,
                           strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS)
        return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "%s: cuTensorMapEncodeTiled failed (CUresult %d): cols %lld N %d B %d ld %lld", what, (int)rc, cols, N, B, ld);
    return MIA_GEMM_OK;
}

// The checks every entry point shares, before any CUDA call.
int check_sizes(const char *what, int B, int N, int H, int dh, int dtype) {
    if (B < 1 || N < 1 || H < 1) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: B, N and H must be at least 1 (B %d, N %d, H %d)", what, B, N, H);
    if (B > 65535 || H > 65535) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: B and H must be at most 65535 (B %d, H %d)", what, B, H);
    if (dh != 32 && dh != 64 && dh != 80) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: head dim %d is not one of 32, 64, 80", what, dh);
    if (dtype != MIA_GEMM_BF16 && dtype != MIA_GEMM_F16) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: dtype must be bf16 or fp16", what);
    return MIA_GEMM_OK;
}

bool pitch_ok(long long ld, long long row) { return ld % 8 == 0 && ld >= row; }

template <typename K, typename... Args>
int launch(K kernel, int smem, dim3 grid, cudaStream_t stream, const char *what, const Args &...args) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "cudaFuncSetAttribute(%s, %d B): %s", what, smem, cudaGetErrorString(cudaGetLastError()));
    kernel<<<grid, kThreads, smem, stream>>>(args...);
    return mia::launched(mia::kErrGemm, what);
}

template <int DH, bool kF16, bool kX = false>
int launch_fwd(const Maps<kX> &tm, const AttnArgs &a, int B, cudaStream_t stream) {
    const dim3 grid((a.N + kRows - 1) / kRows, a.H, B);
    return launch(&attn_fwd_kernel<DH, kF16, kX>, smem_bytes<DH>(1), grid, stream, kX ? "xattn_fwd launch" : "attn_fwd launch", tm, a);
}

template <int DH, bool kF16, bool kX = false>
int launch_bwd(const Maps<kX> &tm, const CUtensorMap &tmd, const AttnArgs &a, int B, cudaStream_t stream) {
    const dim3 grid((a.N + kRows - 1) / kRows, a.H, B);
    if (int rc = launch(&attn_bwd_dq_kernel<DH, kF16, kX>, smem_bytes<DH>(2), grid, stream, kX ? "xattn_bwd_dq launch" : "attn_bwd_dq launch", tm, tmd, a))
        return rc;
    return launch(&attn_bwd_dkv_kernel<DH, kF16, kX>, smem_bytes<DH>(2), grid, stream, kX ? "xattn_bwd_dkv launch" : "attn_bwd_dkv launch", tm, tmd, a);
}

// The cross-attention entries' checks besides check_sizes: head dim 64 and 1 <= seg <= N.
int check_xsizes(const char *what, int B, int N, int H, int dh, int seg, int dtype) {
    if (int rc = check_sizes(what, B, N, H, dh, dtype)) return rc;
    if (dh != 64) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: head dim %d is not 64", what, dh);
    if (seg < 1 || seg > N) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "%s: segment length %d is not in [1, N = %d]", what, seg, N);
    return MIA_GEMM_OK;
}

AttnArgs make_args(int N, int H, int dh) {
    AttnArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.H = H; a.C = H * dh;
    a.scale = 1.f / sqrtf((float)dh);
    a.scale_log2 = a.scale * kLog2e;
    return a;
}

}  // namespace

extern "C" {

int mia_attn_fwd(const void *qkv, void *o, float *lse, int B, int N, int H, int dh, long long ld_qkv, long long ld_o, int dtype, void *cuda_stream) {
    const char *what = "attn_fwd";
    if (!qkv || !o) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_fwd: null pointer (qkv and o are required)");
    if (int rc = check_sizes(what, B, N, H, dh, dtype)) return rc;
    const long long C = (long long)H * dh;
    if (!pitch_ok(ld_qkv, 3 * C) || !pitch_ok(ld_o, C))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_fwd: row pitches must cover a row and be multiples of 8 elements (ld_qkv %lld >= 3C = %lld, ld_o %lld >= C)",
                         ld_qkv, 3 * C, ld_o);
    if (((uintptr_t)qkv | (uintptr_t)o | (uintptr_t)lse) & 15) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_fwd: qkv, o and lse must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "attn_fwd: cannot query the device");
    Maps<false> tm;
    if (int rc = make_map3(&tm.m[0], qkv, 3 * C, N, B, ld_qkv, dtype, what)) return rc;
    AttnArgs a = make_args(N, H, dh);
    a.o = o; a.ld_o = ld_o; a.lse_out = lse;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const bool f16 = dtype == MIA_GEMM_F16;
    switch (dh) {
        case 32: return f16 ? launch_fwd<32, true>(tm, a, B, stream) : launch_fwd<32, false>(tm, a, B, stream);
        case 64: return f16 ? launch_fwd<64, true>(tm, a, B, stream) : launch_fwd<64, false>(tm, a, B, stream);
        default: return f16 ? launch_fwd<80, true>(tm, a, B, stream) : launch_fwd<80, false>(tm, a, B, stream);
    }
}

int mia_attn_bwd(const void *qkv, const void *o, const void *dout, const float *lse, float *delta, void *dqkv, int B, int N, int H, int dh,
                 long long ld_qkv, long long ld_o, long long ld_do, long long ld_dqkv, int dtype, void *cuda_stream) {
    const char *what = "attn_bwd";
    if (!qkv || !o || !dout || !lse || !delta || !dqkv)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_bwd: null pointer (qkv, o, dout, lse, delta and dqkv are required)");
    if (int rc = check_sizes(what, B, N, H, dh, dtype)) return rc;
    const long long C = (long long)H * dh;
    if (!pitch_ok(ld_qkv, 3 * C) || !pitch_ok(ld_o, C) || !pitch_ok(ld_do, C) || !pitch_ok(ld_dqkv, 3 * C))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_bwd: row pitches must cover a row and be multiples of 8 elements "
                         "(ld_qkv %lld, ld_dqkv %lld >= 3C = %lld; ld_o %lld, ld_do %lld >= C)", ld_qkv, ld_dqkv, 3 * C, ld_o, ld_do);
    if (((uintptr_t)qkv | (uintptr_t)o | (uintptr_t)dout | (uintptr_t)lse | (uintptr_t)delta | (uintptr_t)dqkv) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "attn_bwd: qkv, o, dout, lse, delta and dqkv must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "attn_bwd: cannot query the device");
    Maps<false> tm;
    CUtensorMap tmd;
    if (int rc = make_map3(&tm.m[0], qkv, 3 * C, N, B, ld_qkv, dtype, what)) return rc;
    if (int rc = make_map3(&tmd, dout, C, N, B, ld_do, dtype, what)) return rc;
    AttnArgs a = make_args(N, H, dh);
    a.o = const_cast<void *>(o); a.dout = dout; a.lse = lse; a.delta = delta; a.dqkv = dqkv;
    a.ld_o = ld_o; a.ld_do = ld_do; a.ld_dqkv = ld_dqkv;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const bool f16 = dtype == MIA_GEMM_F16;
    switch (dh) {
        case 32: return f16 ? launch_bwd<32, true>(tm, tmd, a, B, stream) : launch_bwd<32, false>(tm, tmd, a, B, stream);
        case 64: return f16 ? launch_bwd<64, true>(tm, tmd, a, B, stream) : launch_bwd<64, false>(tm, tmd, a, B, stream);
        default: return f16 ? launch_bwd<80, true>(tm, tmd, a, B, stream) : launch_bwd<80, false>(tm, tmd, a, B, stream);
    }
}

int mia_xattn_fwd(const void *q, const void *kv, void *o, float *lse, int B, int N, int H, int dh, int seg, long long ld_q, long long ld_kv,
                  long long ld_o, int dtype, void *cuda_stream) {
    const char *what = "xattn_fwd";
    if (!q || !kv || !o) return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_fwd: null pointer (q, kv and o are required)");
    if (int rc = check_xsizes(what, B, N, H, dh, seg, dtype)) return rc;
    const long long C = (long long)H * dh;
    if (!pitch_ok(ld_q, C) || !pitch_ok(ld_kv, 2 * C) || !pitch_ok(ld_o, C))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_fwd: row pitches must cover a row and be multiples of 8 elements "
                         "(ld_q %lld, ld_o %lld >= C = %lld; ld_kv %lld >= 2C)", ld_q, ld_o, C, ld_kv);
    if (((uintptr_t)q | (uintptr_t)kv | (uintptr_t)o | (uintptr_t)lse) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_fwd: q, kv, o and lse must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "xattn_fwd: cannot query the device");
    Maps<true> tm;
    if (int rc = make_map3(&tm.m[0], q, C, N, B, ld_q, dtype, what)) return rc;
    if (int rc = make_map3(&tm.m[1], kv, 2 * C, N, B, ld_kv, dtype, what)) return rc;
    AttnArgs a = make_args(N, H, dh);
    a.o = o; a.ld_o = ld_o; a.lse_out = lse; a.seg = seg;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    return dtype == MIA_GEMM_F16 ? launch_fwd<64, true, true>(tm, a, B, stream) : launch_fwd<64, false, true>(tm, a, B, stream);
}

int mia_xattn_bwd(const void *q, const void *kv, const void *o, const void *dout, const float *lse, float *delta, void *dq, void *dkv, int B, int N,
                  int H, int dh, int seg, long long ld_q, long long ld_kv, long long ld_o, long long ld_do, long long ld_dq, long long ld_dkv, int dtype,
                  void *cuda_stream) {
    const char *what = "xattn_bwd";
    if (!q || !kv || !o || !dout || !lse || !delta || !dq || !dkv)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_bwd: null pointer (q, kv, o, dout, lse, delta, dq and dkv are required)");
    if (int rc = check_xsizes(what, B, N, H, dh, seg, dtype)) return rc;
    const long long C = (long long)H * dh;
    if (!pitch_ok(ld_q, C) || !pitch_ok(ld_kv, 2 * C) || !pitch_ok(ld_o, C) || !pitch_ok(ld_do, C) || !pitch_ok(ld_dq, C) || !pitch_ok(ld_dkv, 2 * C))
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_bwd: row pitches must cover a row and be multiples of 8 elements "
                         "(ld_q %lld, ld_o %lld, ld_do %lld, ld_dq %lld >= C = %lld; ld_kv %lld, ld_dkv %lld >= 2C)", ld_q, ld_o, ld_do, ld_dq, C, ld_kv, ld_dkv);
    if (((uintptr_t)q | (uintptr_t)kv | (uintptr_t)o | (uintptr_t)dout | (uintptr_t)lse | (uintptr_t)delta | (uintptr_t)dq | (uintptr_t)dkv) & 15)
        return mia::fail(mia::kErrGemm, MIA_GEMM_EINVAL, "xattn_bwd: q, kv, o, dout, lse, delta, dq and dkv must be 16-byte aligned");
    mia::DeviceInfo di;
    if (mia::device_info(mia::kErrGemm, di) != MIA_OK) return mia::fail(mia::kErrGemm, MIA_GEMM_ECUDA, "xattn_bwd: cannot query the device");
    Maps<true> tm;
    CUtensorMap tmd;
    if (int rc = make_map3(&tm.m[0], q, C, N, B, ld_q, dtype, what)) return rc;
    if (int rc = make_map3(&tm.m[1], kv, 2 * C, N, B, ld_kv, dtype, what)) return rc;
    if (int rc = make_map3(&tmd, dout, C, N, B, ld_do, dtype, what)) return rc;
    AttnArgs a = make_args(N, H, dh);
    a.o = const_cast<void *>(o); a.dout = dout; a.lse = lse; a.delta = delta; a.dqkv = dq; a.dkv = dkv; a.seg = seg;
    a.ld_o = ld_o; a.ld_do = ld_do; a.ld_dqkv = ld_dq; a.ld_dkv = ld_dkv;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    return dtype == MIA_GEMM_F16 ? launch_bwd<64, true, true>(tm, tmd, a, B, stream) : launch_bwd<64, false, true>(tm, tmd, a, B, stream);
}

}  // extern "C"
