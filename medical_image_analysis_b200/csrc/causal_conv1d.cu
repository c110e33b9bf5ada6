// Depth-wise causal conv1d (+ bias, + SiLU) of the Mamba mixers, forward and backward, as sm_90a kernels.
//
// Reference semantics: `self.act(self.conv1d(x)[..., :seqlen])` with `nn.Conv1d(d, d, k, groups=d, padding=k-1)`
// (CXPMRG_Bench_MambaXray_VL/arm/Finetuning/mamba_simple.py:112-120, 673), which is what the un-vendored
// `causal_conv1d.causal_conv1d_fn(x, weight, bias, activation)` computes (:676-681):
//     pre[b, d, t] = bias[d] + sum_{k < K} w[d, k] * x[b, d, t - (K - 1) + k]        y = pre * sigmoid(pre)  (silu)
// HBM-bound (2 accesses per element forward, 3 backward).  Every thread owns 4 consecutive tokens of one (batch,
// channel) row (8- or 16-byte accesses, 256-512 B per warp instruction); the K - 1 halo tokens come from the
// neighbouring lane by shuffle.
// Backward = one CTA per channel: dx for all the batch rows of the channel, and dweight[d, :], dbias[d] reduced in
// registers -> shared memory -> one write: deterministic, no atomics.
#include <cuda_runtime.h>

#include <initializer_list>
#include <type_traits>

#include "../../include/mia_selective_scan.h"
#include "abi_host.h"
#include "scan_common.cuh"

namespace {

constexpr int kConvThreads = 256;
constexpr int kMaxW = 4;

struct ConvArgs {
    const void *x, *dy;
    void *y, *dx;
    const float *w, *bias;      // (dim, width) / (dim) fp32, bias may be null
    float *dw, *dbias;
    int batch, dim, L, width, silu;
    long long x_bs, x_ds, y_bs, y_ds, dy_bs, dy_ds, dx_bs, dx_ds;   // element strides; the sequence stride is 1
};

template <typename T> struct Tok4;   // 4 consecutive tokens <-> float[4]
template <> struct Tok4<float> {
    static __device__ __forceinline__ void ld(const void *p, float (&f)[4]) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
        f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
    }
    static __device__ __forceinline__ void st(void *p, const float (&f)[4]) { *reinterpret_cast<float4 *>(p) = make_float4(f[0], f[1], f[2], f[3]); }
};
template <> struct Tok4<__nv_bfloat16> {
    static __device__ __forceinline__ void ld(const void *p, float (&f)[4]) {
        const uint2 v = __ldg(reinterpret_cast<const uint2 *>(p));
        f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
        f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
    }
    static __device__ __forceinline__ void st(void *p, const float (&f)[4]) {
        __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
        *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<uint32_t *>(&a), *reinterpret_cast<uint32_t *>(&b));
    }
};
template <> struct Tok4<__half> {
    static __device__ __forceinline__ void ld(const void *p, float (&f)[4]) {
        uint2 v = __ldg(reinterpret_cast<const uint2 *>(p));
        const float2 a = __half22float2(*reinterpret_cast<__half2 *>(&v.x)), b = __half22float2(*reinterpret_cast<__half2 *>(&v.y));
        f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
    }
    static __device__ __forceinline__ void st(void *p, const float (&f)[4]) {
        __half2 a = __floats2half2_rn(f[0], f[1]), b = __floats2half2_rn(f[2], f[3]);
        *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<uint32_t *>(&a), *reinterpret_cast<uint32_t *>(&b));
    }
};

__device__ __forceinline__ float sigmoid_f(float v) { return mia::rcpf(1.f + mia::ex2f(-v * mia::kLog2e)); }

constexpr int kConvUnroll = 4;   // quads in flight per thread: one 8-byte load per thread cannot cover the HBM latency

// ------------------------------------------------------------------------------------------------ forward
// Rows (channels of one batch element) are contiguous, so a block's range of `rows_per_block` channels is one flat run
// of quads: quad i lives at base + 4 i elements, and only the channel (taps, from shared memory) and the row-start test
// need i / quads_per_row (a multiply-high).  grid = (channel ranges, batch).  The three halo tokens come from the
// neighbouring lane (shuffle) except at lane 0.
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kConvThreads) causal_conv1d_fwd_kernel(const ConvArgs a, const int rows_per_block, const uint32_t qpr_magic) {
    constexpr int es = (int)sizeof(T);
    constexpr int U = kConvUnroll;
    extern __shared__ float taps[];                            // [rows_per_block][kW + 1]: w[0..kW-1], bias
    const int qpr = a.L >> 2;                                  // quads per row
    const int c0 = blockIdx.x * rows_per_block, nrows = min(rows_per_block, a.dim - c0);
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < nrows * (kW + 1); i += kConvThreads) {
        const int r = i / (kW + 1), k = i - r * (kW + 1);
        taps[i] = k < kW ? __ldg(a.w + (size_t)(c0 + r) * kW + k) : (a.bias ? __ldg(a.bias + c0 + r) : 0.f);
    }
    __syncthreads();
    const int nq = nrows * qpr;
    const char *xb = (const char *)a.x + ((size_t)b * a.x_bs + (size_t)c0 * a.L) * es;
    char *yb = (char *)a.y + ((size_t)b * a.y_bs + (size_t)c0 * a.L) * es;
    const int lane = threadIdx.x & 31;
    for (int i0 = 0; i0 < nq; i0 += U * kConvThreads) {
        float cur[U][4];
#pragma unroll
        for (int u = 0; u < U; ++u) {                          // all the loads of the pass are issued before any use
            const int i = min(i0 + u * kConvThreads + (int)threadIdx.x, nq - 1);
            Tok4<T>::ld(xb + (size_t)i * (4 * es), cur[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int iu = i0 + u * kConvThreads + (int)threadIdx.x;
            const int i = min(iu, nq - 1);
            const int r = qpr_magic ? (int)__umulhi((uint32_t)i, qpr_magic) : i;   // i / qpr (magic 0: qpr == 1)
            const bool row_start = i == r * qpr;
            const float *tp = taps + r * (kW + 1);
            float prev[4], xv[8];
#pragma unroll
            for (int j = 1; j < 4; ++j) prev[j] = __shfl_up_sync(0xffffffffu, cur[u][j], 1);   // lane - 1 holds the previous quad ...
            if (lane == 0 && !row_start) Tok4<T>::ld(xb + (size_t)i * (4 * es) - 4 * es, prev);  // ... except for lane 0
            if (row_start) prev[1] = prev[2] = prev[3] = 0.f;                                  // causal zero padding
#pragma unroll
            for (int j = 1; j < 4; ++j) xv[j] = prev[j];
#pragma unroll
            for (int j = 0; j < 4; ++j) xv[4 + j] = cur[u][j];
            float y[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float acc = tp[kW];
#pragma unroll
                for (int k = 0; k < kW; ++k) acc = fmaf(tp[k], xv[j + 1 + k + (kMaxW - kW)], acc);
                y[j] = kSilu ? acc * sigmoid_f(acc) : acc;
            }
            if (iu < nq) Tok4<T>::st(yb + (size_t)i * (4 * es), y);
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward
// One CTA per channel.  The quads (batch b, quad q) of the channel are numbered j = b * qpr + q; a warp pass covers 31
// of them plus one look-ahead lane: lane l computes d pre of quad j = 31 k + l and hands its first three values to lane
// l - 1 (dx[t] needs d pre up to t + 3), so nothing is computed twice except by lane 31.
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kConvThreads) causal_conv1d_bwd_kernel(const ConvArgs a, const uint32_t qpr_magic) {
    constexpr int es = (int)sizeof(T);
    constexpr int kWarps = kConvThreads / 32;
    constexpr int U = kConvUnroll;
    __shared__ float red[kWarps][kMaxW + 1];
    const int d = blockIdx.x;
    const int qpr = a.L >> 2;
    const int total = a.batch * qpr;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float bias = a.bias ? __ldg(a.bias + d) : 0.f;
    float w[kW], dw[kW], db = 0.f;
#pragma unroll
    for (int k = 0; k < kW; ++k) { w[k] = __ldg(a.w + (size_t)d * kW + k); dw[k] = 0.f; }
    const char *xd = (const char *)a.x + (size_t)d * a.x_ds * es;
    const char *dyd = (const char *)a.dy + (size_t)d * a.dy_ds * es;
    char *dxd = (char *)a.dx + (size_t)d * a.dx_ds * es;
    for (int j00 = warp * 31; j00 < total; j00 += U * kWarps * 31) {
        int q[U], b[U];
        float cur[U][4], dyv[U][4];
#pragma unroll
        for (int u = 0; u < U; ++u) {                          // all the loads of the pass are issued before any use
            const int j = min(j00 + u * kWarps * 31 + lane, total - 1);
            b[u] = qpr_magic ? (int)__umulhi((uint32_t)j, qpr_magic) : j;   // j / qpr (magic 0: qpr == 1)
            q[u] = j - b[u] * qpr;
            Tok4<T>::ld(xd + ((size_t)b[u] * a.x_bs + 4 * q[u]) * es, cur[u]);
            Tok4<T>::ld(dyd + ((size_t)b[u] * a.dy_bs + 4 * q[u]) * es, dyv[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (j00 + u * kWarps * 31 >= total) break;        // warp-uniform
            const bool valid = j00 + u * kWarps * 31 + lane < total;
            float prev[4], xv[8];
#pragma unroll
            for (int t = 1; t < 4; ++t) prev[t] = __shfl_up_sync(0xffffffffu, cur[u][t], 1);
            if (lane == 0 && q[u] > 0) Tok4<T>::ld(xd + ((size_t)b[u] * a.x_bs + 4 * q[u] - 4) * es, prev);
            if (q[u] == 0) prev[1] = prev[2] = prev[3] = 0.f;
#pragma unroll
            for (int t = 1; t < 4; ++t) xv[t] = prev[t];
#pragma unroll
            for (int t = 0; t < 4; ++t) xv[4 + t] = cur[u][t];
            float dp[7];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                float g = valid ? dyv[u][t] : 0.f;
                if (kSilu) {
                    float pre = bias;
#pragma unroll
                    for (int k = 0; k < kW; ++k) pre = fmaf(w[k], xv[t + 1 + k + (kMaxW - kW)], pre);
                    const float s = sigmoid_f(pre);
                    g *= s * fmaf(pre, 1.f - s, 1.f);
                }
                dp[t] = g;
            }
            // d pre of the next quad of the same row (zero past the row end)
            const bool has_next = valid && q[u] + 1 < qpr;
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                const float nx = __shfl_down_sync(0xffffffffu, dp[t], 1);
                dp[4 + t] = has_next ? nx : 0.f;
            }
            if (valid && lane < 31) {                          // lane 31 only looked ahead for lane 30
                float dxv[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    float acc = 0.f;                           // dx[t] = sum_k w[k] dpre[t + (kW - 1) - k]
#pragma unroll
                    for (int k = 0; k < kW; ++k) acc = fmaf(w[k], dp[t + (kW - 1) - k], acc);
                    dxv[t] = acc;
                    db += dp[t];
#pragma unroll
                    for (int k = 0; k < kW; ++k) dw[k] = fmaf(dp[t], xv[t + 1 + k + (kMaxW - kW)], dw[k]);
                }
                Tok4<T>::st(dxd + ((size_t)b[u] * a.dx_bs + 4 * q[u]) * es, dxv);
            }
        }
    }
    // block reduction in a fixed order: lanes (shuffle tree), then warps
    float vals[kW + 1];
#pragma unroll
    for (int k = 0; k < kW; ++k) vals[k] = dw[k];
    vals[kW] = db;
#pragma unroll
    for (int v = 0; v < kW + 1; ++v) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) vals[v] += __shfl_xor_sync(0xffffffffu, vals[v], off);
    }
    if (lane == 0) {
#pragma unroll
        for (int v = 0; v < kW + 1; ++v) red[warp][v] = vals[v];
    }
    __syncthreads();
    if (threadIdx.x < kW + 1) {
        float s = 0.f;
        for (int wv = 0; wv < kWarps; ++wv) s += red[wv][threadIdx.x];
        if (threadIdx.x == kW) {
            if (a.dbias) a.dbias[d] = s;
        } else {
            a.dw[(size_t)d * kW + threadIdx.x] = s;
        }
    }
}

int conv_check(ConvArgs &a, const void *x, int batch, int dim, int L, int width, int dtype, const long long *strides, int nstrides) {
    if (!x || batch <= 0 || dim <= 0 || L <= 0) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: empty or null input");
    if (width < 1 || width > kMaxW) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d only supports width between 1 and 4");
    if (dtype != MIA_F32 && dtype != MIA_F16 && dtype != MIA_BF16) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: bad dtype");
    if (L % 4) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: seqlen must be a multiple of 4 (got %d)", L);
    for (int i = 0; i < nstrides; ++i)
        if (strides[i] % 4) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: batch / channel strides must be multiples of 4 elements");
    (void)a;
    return MIA_OK;
}

// Calls f(std::integral_constant<int, W>{}, std::integral_constant<bool, S>{}) for the conv width W (1-4, anything else as 1:
// callers validate it first) and the SiLU flag S, so that a launcher names each kernel once.
template <typename F>
void dispatch_conv(int width, int silu, F &&f) {
    const auto with_act = [&](auto w) {
        if (silu) f(w, std::true_type{});
        else f(w, std::false_type{});
    };
    switch (width) {
        case 4: with_act(std::integral_constant<int, 4>{}); break;
        case 3: with_act(std::integral_constant<int, 3>{}); break;
        case 2: with_act(std::integral_constant<int, 2>{}); break;
        default: with_act(std::integral_constant<int, 1>{}); break;
    }
}

// ------------------------------------------------------------------------------------------------ tile kernels
// The kernels of the fused Mamba inner block (mamba_inner_fn and its two siblings): the conv forward / backward and the
// SiLU gate forward / backward.  Every operand is a (batch, dim, seqlen) view with arbitrary element strides (mia_bdl), so
// that the halves of xz / dxz (channel-major (b, 2d, L), or token-major when xz is a transposed projection output), the
// (batch * seqlen, dim) activations of the projection GEMMs and the time-reversed operands of bimamba_inner_fn's backward
// direction (sequence stride -1) are read and written in place.  A CTA works on a tile of kTC channels x kTT tokens of one
// batch element staged in shared memory: each operand is moved along its contiguous dimension -- lanes along the tokens
// when the sequence stride is +-1, along the channels when the channel stride is 1 -- and the arithmetic runs on the
// staged tile (one warp per channel row, lanes along the tokens).  Odd shared-memory pitches keep both walks free of bank
// conflicts.  fp32 arithmetic; any seqlen and dim.
constexpr int kTC = 64, kTT = 64, kTileThreads = 256, kTileWarps = kTileThreads / 32, kRowsPerWarp = kTC / kTileWarps;
constexpr int kHalo = kMaxW - 1;
constexpr int kBwdTok = kTT + kHalo;                           // d pre is needed kW - 1 tokens past the tile for dx
constexpr int kMaxOps = 3;

struct Op { const void *p; long long bs, ds, ts; };          // element (b, d, t) at p + b bs + d ds + t ts

struct TileArgs {
    Op x, z, dx, dz;
    Op in[kMaxOps], out[kMaxOps];                               // summed addends / copies of one result
    int n_in, n_out;
    const float *w, *bias;
    float *part;                                                // conv backward: [parts][dim][width + 1] partial sums
    float *dw, *dbias;
    int batch, dim, L, n_tt, parts;
};

template <typename T> __device__ __forceinline__ float ldf(const void *p, long long i) {
    return mia::Cvt<T>::to_f(reinterpret_cast<const typename mia::Cvt<T>::raw *>(p)[i]);
}
template <typename T> __device__ __forceinline__ void stf(const void *p, long long i, float v) {
    reinterpret_cast<typename mia::Cvt<T>::raw *>(const_cast<void *>(p))[i] = mia::Cvt<T>::from_f(v);
}
__device__ __forceinline__ bool token_rows(const Op &o) { return o.ds == 1 && o.ts != 1 && o.ts != -1; }

// s[r][j] (+)= o(b, c0 + r, t0 + j) for r < kTC, j < nj; zero outside the tensor.  The caller synchronises before a second
// pass over the same tile (the two walks hand the elements to different threads).
template <typename T, bool kAdd>
__device__ __forceinline__ void tile_ld(float *s, int pitch, const Op &o, int b, int c0, int t0, int nj, int dim, int L) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (token_rows(o)) {
        for (int j = warp; j < nj; j += kTileWarps) {
            const int t = t0 + j;
            const bool tv = t >= 0 && t < L;
            for (int r = lane; r < kTC; r += 32) {
                const int c = c0 + r;
                const float v = (tv && c < dim) ? ldf<T>(o.p, b * o.bs + c * o.ds + t * o.ts) : 0.f;
                s[r * pitch + j] = kAdd ? s[r * pitch + j] + v : v;
            }
        }
    } else {
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps, c = c0 + r;
            for (int j = lane; j < nj; j += 32) {
                const int t = t0 + j;
                const float v = (c < dim && t >= 0 && t < L) ? ldf<T>(o.p, b * o.bs + c * o.ds + t * o.ts) : 0.f;
                s[r * pitch + j] = kAdd ? s[r * pitch + j] + v : v;
            }
        }
    }
}

// o(b, c0 + r, t0 + j) = s[r][j] for the elements of the tile inside the tensor (j < kTT).
template <typename T>
__device__ __forceinline__ void tile_st(const float *s, int pitch, const Op &o, int b, int c0, int t0, int dim, int L) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (token_rows(o)) {
        for (int j = warp; j < kTT && t0 + j < L; j += kTileWarps)
            for (int r = lane; r < kTC && c0 + r < dim; r += 32) stf<T>(o.p, b * o.bs + (c0 + r) * o.ds + (t0 + j) * o.ts, s[r * pitch + j]);
    } else {
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps, c = c0 + r;
            if (c >= dim) continue;
            for (int j = lane; j < kTT && t0 + j < L; j += 32) stf<T>(o.p, b * o.bs + c * o.ds + (t0 + j) * o.ts, s[r * pitch + j]);
        }
    }
}

template <int kW>
__device__ __forceinline__ void load_taps(float (*taps)[kW + 1], const TileArgs &a, int c0) {
    for (int i = threadIdx.x; i < kTC * (kW + 1); i += kTileThreads) {
        const int r = i / (kW + 1), k = i - r * (kW + 1), c = c0 + r;
        taps[r][k] = c >= a.dim ? 0.f : k < kW ? __ldg(a.w + (size_t)c * kW + k) : (a.bias ? __ldg(a.bias + c) : 0.f);
    }
}

// Conv forward: every out[i] = act(bias + sum_k w[d, k] x[b, d, t - (K-1) + k]), the arithmetic of causal_conv1d_fwd_kernel.
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kTileThreads) conv_fwd_ex_kernel(const TileArgs a) {
    constexpr int PX = kTT + kHalo, PY = kTT + 1;               // 67, 65: odd pitches
    __shared__ float xs[kTC * PX];                              // tokens t0 - 3 .. t0 + 63
    __shared__ float ys[kTC * PY];
    __shared__ float taps[kTC][kW + 1];
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    load_taps<kW>(taps, a, c0);
    tile_ld<T, false>(xs, PX, a.x, b, c0, t0 - kHalo, kTT + kHalo, a.dim, a.L);
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int r = warp + rr * kTileWarps;
        for (int j = lane; j < kTT; j += 32) {
            float acc = taps[r][kW];
#pragma unroll
            for (int k = 0; k < kW; ++k) acc = fmaf(taps[r][k], xs[r * PX + j + kHalo - (kW - 1) + k], acc);
            ys[r * PY + j] = kSilu ? acc * sigmoid_f(acc) : acc;
        }
    }
    __syncthreads();
    for (int i = 0; i < a.n_out; ++i) tile_st<T>(ys, PY, a.out[i], b, c0, t0, a.dim, a.L);
}

// Conv backward: dy = in[0] + in[1] + ... summed in fp32 in that order; dx written completely.  grid = (channel tiles, parts):
// a CTA walks the (batch, token tile) items part, part + parts, ... in order, and every thread accumulates dweight / dbias of
// its own (channel row, token slot) pairs in registers; the lanes of a row are reduced by a fixed shuffle tree into
// part[part][channel], which conv_bwd_ex_finalize sums over the parts in order: deterministic, no atomics.
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kTileThreads) conv_bwd_ex_kernel(const TileArgs a) {
    constexpr int PX = kBwdTok + kHalo + 1, PG = kBwdTok;       // 71, 67: odd pitches
    __shared__ float xs[kTC * PX];                              // x at tokens t0 - 3 .. t0 + 66; then dx
    __shared__ float gs[kTC * PG];                              // dy, then d pre, at tokens t0 .. t0 + 66
    __shared__ float taps[kTC][kW + 1];
    const int c0 = blockIdx.x * kTC;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    load_taps<kW>(taps, a, c0);
    float dw[kRowsPerWarp][kW + 1];
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr)
#pragma unroll
        for (int k = 0; k <= kW; ++k) dw[rr][k] = 0.f;
    const int n_items = a.batch * a.n_tt;
    for (int item = blockIdx.y; item < n_items; item += a.parts) {
        const int b = item / a.n_tt, t0 = (item - b * a.n_tt) * kTT;
        __syncthreads();                                        // the previous item is done with xs / gs
        tile_ld<T, false>(xs, PX, a.x, b, c0, t0 - kHalo, kBwdTok + kHalo, a.dim, a.L);
        tile_ld<T, false>(gs, PG, a.in[0], b, c0, t0, kBwdTok, a.dim, a.L);
        for (int i = 1; i < a.n_in; ++i) {
            __syncthreads();
            tile_ld<T, true>(gs, PG, a.in[i], b, c0, t0, kBwdTok, a.dim, a.L);
        }
        __syncthreads();
#pragma unroll
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps;
            for (int j = lane; j < kBwdTok; j += 32) {
                float g = gs[r * PG + j];
                if (kSilu) {
                    float pre = taps[r][kW];
#pragma unroll
                    for (int k = 0; k < kW; ++k) pre = fmaf(taps[r][k], xs[r * PX + j + kHalo - (kW - 1) + k], pre);
                    const float s = sigmoid_f(pre);
                    g *= s * fmaf(pre, 1.f - s, 1.f);
                    gs[r * PG + j] = g;
                }
                if (j < kTT) {                                  // the tokens past the tile belong to the next item's sums
                    dw[rr][kW] += g;
#pragma unroll
                    for (int k = 0; k < kW; ++k) dw[rr][k] = fmaf(g, xs[r * PX + j + kHalo - (kW - 1) + k], dw[rr][k]);
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps;
            for (int j = lane; j < kTT; j += 32) {
                float acc = 0.f;                                // dx[t] = sum_k w[k] dpre[t + (kW - 1) - k]
#pragma unroll
                for (int k = 0; k < kW; ++k) acc = fmaf(taps[r][k], gs[r * PG + j + (kW - 1) - k], acc);
                xs[r * PX + j] = acc;
            }
        }
        __syncthreads();
        tile_st<T>(xs, PX, a.dx, b, c0, t0, a.dim, a.L);
    }
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int c = c0 + warp + rr * kTileWarps;
#pragma unroll
        for (int k = 0; k <= kW; ++k) {
            float v = dw[rr][k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0 && c < a.dim) a.part[((size_t)blockIdx.y * a.dim + c) * (kW + 1) + k] = v;
        }
    }
}

__global__ void conv_bwd_ex_finalize(const TileArgs a, const int kw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // (channel, tap or bias)
    if (i >= a.dim * (kw + 1)) return;
    float s = 0.f;
    for (int p = 0; p < a.parts; ++p) s += a.part[(size_t)p * a.dim * (kw + 1) + i];
    const int c = i / (kw + 1), k = i - c * (kw + 1);
    if (k < kw) a.dw[(size_t)c * kw + k] = s;
    else if (a.dbias) a.dbias[c] = s;
}

struct NoScale { __device__ __forceinline__ float operator()(float v) const { return v; } };

// The SiLU gate's arithmetic on a staged tile, written once for the inner block's gate kernels and the multi-direction ones
// (which scale by 1 / divisor): forward os = scale(os silu(zs)).
template <typename Scale>
__device__ __forceinline__ void gate_fwd_rows(float *os, const float *zs, Scale scale) {
    constexpr int P = kTT + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int r = warp + rr * kTileWarps;
        for (int j = lane; j < kTT; j += 32) {
            const float zv = zs[r * P + j];
            os[r * P + j] = scale(os[r * P + j] * (zv * sigmoid_f(zv)));
        }
    }
}

// Backward, for g = scale(gs): gs = g silu(zs) (the gradient of the gated sum os), os = g os silu'(zs) (the gradient of zs).
template <typename Scale>
__device__ __forceinline__ void gate_bwd_rows(float *gs, float *os, const float *zs, Scale scale) {
    constexpr int P = kTT + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int r = warp + rr * kTileWarps;
        for (int j = lane; j < kTT; j += 32) {
            const float g = scale(gs[r * P + j]), zv = zs[r * P + j], s = sigmoid_f(zv);
            gs[r * P + j] = g * (zv * s);
            os[r * P + j] = g * os[r * P + j] * s * fmaf(zv, 1.f - s, 1.f);
        }
    }
}

// Gate forward: v = (in[0] + in[1] + ...) silu(z) -> every out[i].
template <typename T>
__global__ void __launch_bounds__(kTileThreads) gate_fwd_ex_kernel(const TileArgs a) {
    constexpr int P = kTT + 1;
    __shared__ float os[kTC * P], zs[kTC * P];
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    tile_ld<T, false>(zs, P, a.z, b, c0, t0, kTT, a.dim, a.L);
    tile_ld<T, false>(os, P, a.in[0], b, c0, t0, kTT, a.dim, a.L);
    for (int i = 1; i < a.n_in; ++i) {
        __syncthreads();
        tile_ld<T, true>(os, P, a.in[i], b, c0, t0, kTT, a.dim, a.L);
    }
    __syncthreads();
    gate_fwd_rows(os, zs, NoScale{});
    __syncthreads();
    for (int i = 0; i < a.n_out; ++i) tile_st<T>(os, P, a.out[i], b, c0, t0, a.dim, a.L);
}

// Gate backward: g = dy (in[0]), o = in[1] + in[2] + ...;  every out[i] = g silu(z) (d of the gate's input, stored as TD), dz =
// g o silu'(z).
template <typename T, typename TD>
__global__ void __launch_bounds__(kTileThreads) gate_bwd_ex_kernel(const TileArgs a) {
    constexpr int P = kTT + 1;
    extern __shared__ float gate_smem[];                        // 3 tiles: 50 KB, above the static 48 KB
    float *gs = gate_smem, *os = gs + kTC * P, *zs = os + kTC * P;
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    tile_ld<T, false>(gs, P, a.in[0], b, c0, t0, kTT, a.dim, a.L);
    tile_ld<T, false>(zs, P, a.z, b, c0, t0, kTT, a.dim, a.L);
    tile_ld<T, false>(os, P, a.in[1], b, c0, t0, kTT, a.dim, a.L);
    for (int i = 2; i < a.n_in; ++i) {
        __syncthreads();
        tile_ld<T, true>(os, P, a.in[i], b, c0, t0, kTT, a.dim, a.L);
    }
    __syncthreads();
    gate_bwd_rows(gs, os, zs, NoScale{});
    __syncthreads();
    for (int i = 0; i < a.n_out; ++i) tile_st<TD>(gs, P, a.out[i], b, c0, t0, a.dim, a.L);
    tile_st<T>(os, P, a.dz, b, c0, t0, a.dim, a.L);
}

// Parts of the conv backward: ~8 CTAs per SM of a 132-SM H100 over all channel tiles of the n directions (n = 1 for the inner
// block's kernel).  A function of the sizes only, so the order of the dweight / dbias sums (and therefore their bits) does not
// depend on the device.
int conv_bwd_parts(int n, int batch, int dim, int L) {
    const int ctiles = (dim + kTC - 1) / kTC, items = batch * ((L + kTT - 1) / kTT);
    const int want = (8 * 132 + ctiles * n - 1) / (ctiles * n);
    return want < items ? want : items;
}

// ------------------------------------------------------------------------------------------------ scan orders
// The multi-direction kernels of ARM's four-direction (bimamba v3) mixer.  Direction k's scan position t reads image token
// order_k(t) (include/mia_selective_scan.h, MIA_ORDER_*), closed-form integer arithmetic: the scan-order operands (the
// scan's u / out / du / dout, dense (batch, n_dirs dim, seqlen), and the token-major x_proj operands) are addressed at
// scan positions, the image-order ones (the halves of xz / dxz, out_proj's operands) at tokens.  The conv and its backward
// work in scan order and gather their image-order x through order_k; the gate and the dx sum over the directions work in
// image order and gather each direction's scan-order operand through order_k's inverse.
constexpr int kMaxDirs = 4;

struct Dirs { int n, L, pos, side; int code[kMaxDirs]; };

__device__ __forceinline__ int col_map(int t, int pos, int side) {    // an involution
    if (t == pos) return pos;
    const int g = t - (t > pos);
    const int r = (g % side) * side + g / side;
    return r + (r >= pos);
}
// image token read at scan position t of an order
__device__ __forceinline__ int order_tok(const Dirs &o, int k, int t) {
    switch (o.code[k]) {
        case MIA_ORDER_SEQ_REV: return o.L - 1 - t;
        case MIA_ORDER_COL: return col_map(t, o.pos, o.side);
        case MIA_ORDER_COL_REV: return col_map(o.L - 1 - t, o.pos, o.side);
        default: return t;
    }
}
// scan position of image token i in an order (order_tok's inverse)
__device__ __forceinline__ int order_pos(const Dirs &o, int k, int i) {
    switch (o.code[k]) {
        case MIA_ORDER_SEQ_REV: return o.L - 1 - i;
        case MIA_ORDER_COL: return col_map(i, o.pos, o.side);
        case MIA_ORDER_COL_REV: return o.L - 1 - col_map(i, o.pos, o.side);
        default: return i;
    }
}

// tile_ld with the tokens renamed: s[r][j] (+)= o(b, c0 + r, map(t0 + j)) for t0 + j inside [0, L), zero outside.
template <typename T, bool kAdd, typename Map>
__device__ __forceinline__ void tile_ld_map(float *s, int pitch, const Op &o, int b, int c0, int t0, int nj, int dim, int L, Map map) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (token_rows(o)) {
        for (int j = warp; j < nj; j += kTileWarps) {
            const int t = t0 + j;
            const bool tv = t >= 0 && t < L;
            const int tok = tv ? map(t) : 0;
            for (int r = lane; r < kTC; r += 32) {
                const int c = c0 + r;
                const float v = (tv && c < dim) ? ldf<T>(o.p, b * o.bs + c * o.ds + (long long)tok * o.ts) : 0.f;
                s[r * pitch + j] = kAdd ? s[r * pitch + j] + v : v;
            }
        }
    } else {
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps, c = c0 + r;
            for (int j = lane; j < nj; j += 32) {
                const int t = t0 + j;
                const float v = (c < dim && t >= 0 && t < L) ? ldf<T>(o.p, b * o.bs + c * o.ds + (long long)map(t) * o.ts) : 0.f;
                s[r * pitch + j] = kAdd ? s[r * pitch + j] + v : v;
            }
        }
    }
}

// tile_st with the tokens renamed: o(b, c0 + r, map(t0 + j)) = s[r][j] inside the tensor.
template <typename T, typename Map>
__device__ __forceinline__ void tile_st_map(const float *s, int pitch, const Op &o, int b, int c0, int t0, int dim, int L, Map map) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (token_rows(o)) {
        for (int j = warp; j < kTT && t0 + j < L; j += kTileWarps) {
            const long long tok = map(t0 + j);
            for (int r = lane; r < kTC && c0 + r < dim; r += 32) stf<T>(o.p, b * o.bs + (c0 + r) * o.ds + tok * o.ts, s[r * pitch + j]);
        }
    } else {
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps, c = c0 + r;
            if (c >= dim) continue;
            for (int j = lane; j < kTT && t0 + j < L; j += 32) stf<T>(o.p, b * o.bs + c * o.ds + (long long)map(t0 + j) * o.ts, s[r * pitch + j]);
        }
    }
}

struct DirArgs {
    Dirs o;
    Op x, z, dx, dz, y;
    Op tm[kMaxDirs];                                            // per-direction token-major operands (u_tm / dy_tm), scan order
    int has_tm;
    const void *dense;                                          // (batch, n dim, L) scan order: u (conv fwd), du (conv bwd), outs (gate)
    void *dense_out;                                            // conv fwd: u;  gate bwd: douts (fp32)
    const float *w, *bias;                                      // (n, dim, width) / (n, dim)
    float *xpart, *part;                                        // conv bwd: dx per direction (n, batch, dim, L) fp32; dw partials
    float *dw, *dbias;
    float scale;
    int batch, dim, L, n_tt, parts;
};

// direction k's slice of a dense (batch, n dim, L) operand of element type T as a (batch, dim, L) Op
template <typename T>
__device__ __forceinline__ Op dense_op(const void *p, const DirArgs &a, int k) {
    return Op{(const char *)p + (size_t)k * a.dim * a.L * sizeof(T), (long long)a.o.n * a.dim * a.L, a.L, 1};
}

template <int kW>
__device__ __forceinline__ void load_taps_dir(float (*taps)[kW + 1], const DirArgs &a, int k, int c0) {
    const float *w = a.w + (size_t)k * a.dim * kW, *bias = a.bias ? a.bias + (size_t)k * a.dim : nullptr;
    for (int i = threadIdx.x; i < kTC * (kW + 1); i += kTileThreads) {
        const int r = i / (kW + 1), j = i - r * (kW + 1), c = c0 + r;
        taps[r][j] = c >= a.dim ? 0.f : j < kW ? __ldg(w + (size_t)c * kW + j) : (bias ? __ldg(bias + c) : 0.f);
    }
}

// Conv forward of every direction, in scan order: grid = (channel tiles, token tiles, batch * n); the arithmetic of
// conv_fwd_ex_kernel on x gathered through order_k.  Writes direction k's slice of u and / or its token-major tm[k].
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kTileThreads) conv_fwd_dirs_kernel(const DirArgs a) {
    constexpr int PX = kTT + kHalo, PY = kTT + 1;
    __shared__ float xs[kTC * PX];
    __shared__ float ys[kTC * PY];
    __shared__ float taps[kTC][kW + 1];
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, k = blockIdx.z % a.o.n, b = blockIdx.z / a.o.n;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    load_taps_dir<kW>(taps, a, k, c0);
    tile_ld_map<T, false>(xs, PX, a.x, b, c0, t0 - kHalo, kTT + kHalo, a.dim, a.L, [&](int t) { return order_tok(a.o, k, t); });
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int r = warp + rr * kTileWarps;
        for (int j = lane; j < kTT; j += 32) {
            float acc = taps[r][kW];
#pragma unroll
            for (int i = 0; i < kW; ++i) acc = fmaf(taps[r][i], xs[r * PX + j + kHalo - (kW - 1) + i], acc);
            ys[r * PY + j] = kSilu ? acc * sigmoid_f(acc) : acc;
        }
    }
    __syncthreads();
    if (a.dense_out) tile_st<T>(ys, PY, dense_op<T>(a.dense_out, a, k), b, c0, t0, a.dim, a.L);
    if (a.has_tm) tile_st<T>(ys, PY, a.tm[k], b, c0, t0, a.dim, a.L);
}

// Conv backward of every direction, in scan order: grid = (channel tiles, parts, n).  conv_bwd_ex_kernel's arithmetic with
// dy = du_k (+ tm[k]) summed in fp32 and x gathered through order_k; direction k's dx goes unrounded to xpart[k] (scan
// order, dense) and its dweight / dbias partials to part[k][part][channel] for conv_bwd_dirs_finalize.
template <typename T, int kW, bool kSilu>
__global__ void __launch_bounds__(kTileThreads) conv_bwd_dirs_kernel(const DirArgs a) {
    constexpr int PX = kBwdTok + kHalo + 1, PG = kBwdTok;
    __shared__ float xs[kTC * PX];
    __shared__ float gs[kTC * PG];
    __shared__ float taps[kTC][kW + 1];
    const int c0 = blockIdx.x * kTC, k = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const auto tok = [&](int t) { return order_tok(a.o, k, t); };
    const auto same = [](int t) { return t; };
    load_taps_dir<kW>(taps, a, k, c0);
    const Op du = dense_op<T>(a.dense, a, k);
    const Op dxk{(const char *)a.xpart + (size_t)k * a.batch * a.dim * a.L * sizeof(float), (long long)a.dim * a.L, a.L, 1};
    float dw[kRowsPerWarp][kW + 1];
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr)
#pragma unroll
        for (int i = 0; i <= kW; ++i) dw[rr][i] = 0.f;
    const int n_items = a.batch * a.n_tt;
    for (int item = blockIdx.y; item < n_items; item += a.parts) {
        const int b = item / a.n_tt, t0 = (item - b * a.n_tt) * kTT;
        __syncthreads();
        tile_ld_map<T, false>(xs, PX, a.x, b, c0, t0 - kHalo, kBwdTok + kHalo, a.dim, a.L, tok);
        tile_ld_map<T, false>(gs, PG, du, b, c0, t0, kBwdTok, a.dim, a.L, same);
        if (a.has_tm) {
            __syncthreads();
            tile_ld_map<T, true>(gs, PG, a.tm[k], b, c0, t0, kBwdTok, a.dim, a.L, same);
        }
        __syncthreads();
#pragma unroll
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps;
            for (int j = lane; j < kBwdTok; j += 32) {
                float g = gs[r * PG + j];
                if (kSilu) {
                    float pre = taps[r][kW];
#pragma unroll
                    for (int i = 0; i < kW; ++i) pre = fmaf(taps[r][i], xs[r * PX + j + kHalo - (kW - 1) + i], pre);
                    const float s = sigmoid_f(pre);
                    g *= s * fmaf(pre, 1.f - s, 1.f);
                    gs[r * PG + j] = g;
                }
                if (j < kTT) {
                    dw[rr][kW] += g;
#pragma unroll
                    for (int i = 0; i < kW; ++i) dw[rr][i] = fmaf(g, xs[r * PX + j + kHalo - (kW - 1) + i], dw[rr][i]);
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int rr = 0; rr < kRowsPerWarp; ++rr) {
            const int r = warp + rr * kTileWarps;
            for (int j = lane; j < kTT; j += 32) {
                float acc = 0.f;
#pragma unroll
                for (int i = 0; i < kW; ++i) acc = fmaf(taps[r][i], gs[r * PG + j + (kW - 1) - i], acc);
                xs[r * PX + j] = acc;
            }
        }
        __syncthreads();
        tile_st<float>(xs, PX, dxk, b, c0, t0, a.dim, a.L);
    }
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int c = c0 + warp + rr * kTileWarps;
#pragma unroll
        for (int i = 0; i <= kW; ++i) {
            float v = dw[rr][i];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0 && c < a.dim) a.part[(((size_t)k * a.parts + blockIdx.y) * a.dim + c) * (kW + 1) + i] = v;
        }
    }
}

// dx[b, c, i] = sum over k = 0 .. n-1, in that order, of xpart[k] at scan position order_pos_k(i), rounded once; grid =
// (channel tiles, token tiles, batch) over image order.  The CTAs of token tile 0 / batch 0 also sum the dweight / dbias
// partials of their channels over the parts, in order.
template <typename T>
__global__ void __launch_bounds__(kTileThreads) conv_bwd_dirs_finalize(const DirArgs a, const int kw) {
    constexpr int P = kTT + 1;
    __shared__ float acc[kTC * P];
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    for (int k = 0; k < a.o.n; ++k) {
        const Op xk{(const char *)a.xpart + (size_t)k * a.batch * a.dim * a.L * sizeof(float), (long long)a.dim * a.L, a.L, 1};
        const auto pos = [&](int i) { return order_pos(a.o, k, i); };
        if (k == 0) {
            tile_ld_map<float, false>(acc, P, xk, b, c0, t0, kTT, a.dim, a.L, pos);
        } else {
            __syncthreads();
            tile_ld_map<float, true>(acc, P, xk, b, c0, t0, kTT, a.dim, a.L, pos);
        }
    }
    __syncthreads();
    tile_st<T>(acc, P, a.dx, b, c0, t0, a.dim, a.L);
    if (blockIdx.y != 0 || blockIdx.z != 0) return;
    for (int i = threadIdx.x; i < a.o.n * kTC * (kw + 1); i += kTileThreads) {
        const int k = i / (kTC * (kw + 1)), rem = i - k * kTC * (kw + 1), r = rem / (kw + 1), j = rem - r * (kw + 1), c = c0 + r;
        if (c >= a.dim) continue;
        float s = 0.f;
        for (int p = 0; p < a.parts; ++p) s += a.part[(((size_t)k * a.parts + p) * a.dim + c) * (kw + 1) + j];
        if (j < kw) a.dw[((size_t)k * a.dim + c) * kw + j] = s;
        else if (a.dbias) a.dbias[(size_t)k * a.dim + c] = s;
    }
}

// Gate forward over image order: y = scale silu(z) sum_k outs_k[order_pos_k(i)] (summed in fp32, k = 0 .. n-1), rounded once.
template <typename T>
__global__ void __launch_bounds__(kTileThreads) gate_fwd_dirs_kernel(const DirArgs a) {
    constexpr int P = kTT + 1;
    __shared__ float os[kTC * P], zs[kTC * P];
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    tile_ld<T, false>(zs, P, a.z, b, c0, t0, kTT, a.dim, a.L);
    for (int k = 0; k < a.o.n; ++k) {
        const auto pos = [&](int i) { return order_pos(a.o, k, i); };
        if (k == 0) {
            tile_ld_map<T, false>(os, P, dense_op<T>(a.dense, a, k), b, c0, t0, kTT, a.dim, a.L, pos);
        } else {
            __syncthreads();
            tile_ld_map<T, true>(os, P, dense_op<T>(a.dense, a, k), b, c0, t0, kTT, a.dim, a.L, pos);
        }
    }
    __syncthreads();
    gate_fwd_rows(os, zs, [&](float v) { return v * a.scale; });
    __syncthreads();
    tile_st<T>(os, P, a.y, b, c0, t0, a.dim, a.L);
}

// Gate backward over image order, for y above and its gradient dy: every direction's dout_k at scan position order_pos_k(i)
// = dy scale silu(z) (fp32, unrounded), dz = dy scale (sum_k outs_k) silu'(z).
template <typename T>
__global__ void __launch_bounds__(kTileThreads) gate_bwd_dirs_kernel(const DirArgs a) {
    constexpr int P = kTT + 1;
    extern __shared__ float gate_smem[];                        // 3 tiles: 50 KB, above the static 48 KB
    float *gs = gate_smem, *os = gs + kTC * P, *zs = os + kTC * P;
    const int c0 = blockIdx.x * kTC, t0 = blockIdx.y * kTT, b = blockIdx.z;
    tile_ld<T, false>(gs, P, a.y, b, c0, t0, kTT, a.dim, a.L);
    tile_ld<T, false>(zs, P, a.z, b, c0, t0, kTT, a.dim, a.L);
    for (int k = 0; k < a.o.n; ++k) {
        const auto pos = [&](int i) { return order_pos(a.o, k, i); };
        if (k == 0) {
            tile_ld_map<T, false>(os, P, dense_op<T>(a.dense, a, k), b, c0, t0, kTT, a.dim, a.L, pos);
        } else {
            __syncthreads();
            tile_ld_map<T, true>(os, P, dense_op<T>(a.dense, a, k), b, c0, t0, kTT, a.dim, a.L, pos);
        }
    }
    __syncthreads();
    gate_bwd_rows(gs, os, zs, [&](float v) { return v * a.scale; });
    __syncthreads();
    for (int k = 0; k < a.o.n; ++k)
        tile_st_map<float>(gs, P, dense_op<float>(a.dense_out, a, k), b, c0, t0, a.dim, a.L, [&](int i) { return order_pos(a.o, k, i); });
    tile_st<T>(os, P, a.dz, b, c0, t0, a.dim, a.L);
}

bool op_ok(const mia_bdl *o) { return o && o->ptr; }
Op op_of(const mia_bdl *o) { return op_ok(o) ? Op{o->ptr, o->batch_stride, o->d_stride, o->seq_stride} : Op{nullptr, 0, 0, 0}; }

// Checks shared by the tile entry points: sizes (batch * z_per_batch CTAs fit the grid's z) and dtype.
template <typename Args>
int tile_check(const char *what, Args &a, int batch, int dim, int L, int dtype, int z_per_batch) {
    if (batch <= 0 || dim <= 0 || L <= 0 || (long long)batch * z_per_batch > 65535) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: bad sizes", what);
    if (dtype != MIA_F32 && dtype != MIA_F16 && dtype != MIA_BF16) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: bad dtype", what);
    a.batch = batch; a.dim = dim; a.L = L;
    return MIA_OK;
}

// Checks of the inner block's entry points; fills a.in / a.out from the operand arrays.
int ex_check(const char *what, TileArgs &a, int batch, int dim, int L, int dtype, const mia_bdl *in, int n_in, int min_in,
             const mia_bdl *out, int n_out, int min_out) {
    if (int rc = tile_check(what, a, batch, dim, L, dtype, 1)) return rc;
    if (n_in < min_in || n_in > kMaxOps || n_out < min_out || n_out > kMaxOps || (n_in && !in) || (n_out && !out)) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: %d inputs / %d outputs (at least %d / %d, at most %d each)", what, n_in, n_out,
                         min_in, min_out, kMaxOps);
    }
    for (int i = 0; i < n_in; ++i) {
        if (!op_ok(in + i)) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: null input operand", what);
        a.in[i] = op_of(in + i);
    }
    for (int i = 0; i < n_out; ++i) {
        if (!op_ok(out + i)) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: null output operand", what);
        a.out[i] = op_of(out + i);
    }
    a.n_in = n_in; a.n_out = n_out;
    return MIA_OK;
}

// Checks of the multi-direction entry points: tile_check and the orders (a column order needs a square grid of seqlen - 1
// tokens).
int dirs_check(const char *what, DirArgs &a, const int *orders, int n_dirs, int batch, int dim, int L, int dtype) {
    if (int rc = tile_check(what, a, batch, dim, L, dtype, kMaxDirs)) return rc;
    if (!orders || n_dirs < 1 || n_dirs > kMaxDirs) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: 1-%d orders required, got %d", what, kMaxDirs, n_dirs);
    int side = 0;
    while ((side + 1) * (side + 1) <= L - 1) ++side;
    for (int k = 0; k < n_dirs; ++k) {
        const int c = orders[k];
        if (c < MIA_ORDER_SEQ || c > MIA_ORDER_COL_REV) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: unknown order %d", what, c);
        if ((c == MIA_ORDER_COL || c == MIA_ORDER_COL_REV) && (L < 2 || side * side != L - 1)) {
            return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: a column order needs seqlen - 1 to be a square, got seqlen %d", what, L);
        }
        a.o.code[k] = c;
    }
    a.o.n = n_dirs; a.o.L = L; a.o.pos = L / 2; a.o.side = side;
    return MIA_OK;
}

}  // namespace

extern "C" {

int mia_causal_conv1d_fwd(const void *x, const float *weight, const float *bias, void *y, int batch, int dim, int seqlen, int width,
                          int silu, int dtype, long long x_batch_stride, long long x_d_stride, long long y_batch_stride,
                          long long y_d_stride, void *cuda_stream) {
    ConvArgs a{};
    const long long st[4] = {x_batch_stride, x_d_stride, y_batch_stride, y_d_stride};
    if (int rc = conv_check(a, x, batch, dim, seqlen, width, dtype, st, 4)) return rc;
    const int es = dtype == MIA_F32 ? 4 : 2;
    if (!weight || !y || (((uintptr_t)x | (uintptr_t)y) & (4 * es - 1))) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_fwd: null weight / y or x / y not aligned to 4 elements");
    }
    a.x = x; a.y = y; a.w = weight; a.bias = bias; a.batch = batch; a.dim = dim; a.L = seqlen; a.width = width; a.silu = silu;
    a.x_bs = x_batch_stride; a.x_ds = x_d_stride; a.y_bs = y_batch_stride; a.y_ds = y_d_stride;
    if (x_d_stride != seqlen || y_d_stride != seqlen) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_fwd: the channel rows of x and y must be contiguous (stride == seqlen)");
    }
    // rows per block: ~2 passes of kConvUnroll quads per thread
    const int qpr = seqlen / 4;
    int rpb = (2 * kConvUnroll * kConvThreads + qpr - 1) / qpr;
    if (rpb > dim) rpb = dim;
    if ((long long)rpb * qpr * qpr >= (1LL << 32) || batch > 65535) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: sequence or batch too large");
    }
    const dim3 grid((dim + rpb - 1) / rpb, batch);
    const size_t smem = (size_t)rpb * (width + 1) * sizeof(float);
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            causal_conv1d_fwd_kernel<T, decltype(w)::value, decltype(act)::value>
                <<<grid, kConvThreads, smem, (cudaStream_t)cuda_stream>>>(a, rpb, mia::div_magic(qpr));
        });
    });
    return mia::launched(mia::kErrConv, "causal_conv1d_fwd launch");
}

int mia_causal_conv1d_bwd(const void *x, const float *weight, const float *bias, const void *dy, void *dx, float *dweight, float *dbias,
                          int batch, int dim, int seqlen, int width, int silu, int dtype, long long x_batch_stride, long long x_d_stride,
                          long long dy_batch_stride, long long dy_d_stride, long long dx_batch_stride, long long dx_d_stride,
                          void *cuda_stream) {
    ConvArgs a{};
    const long long st[6] = {x_batch_stride, x_d_stride, dy_batch_stride, dy_d_stride, dx_batch_stride, dx_d_stride};
    if (int rc = conv_check(a, x, batch, dim, seqlen, width, dtype, st, 6)) return rc;
    const int es = dtype == MIA_F32 ? 4 : 2;
    if (!weight || !dy || !dx || !dweight || (((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dx) & (4 * es - 1))) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_bwd: null pointer or x / dy / dx not aligned to 4 elements");
    }
    a.x = x; a.dy = dy; a.dx = dx; a.w = weight; a.bias = bias; a.dw = dweight; a.dbias = dbias;
    a.batch = batch; a.dim = dim; a.L = seqlen; a.width = width; a.silu = silu;
    a.x_bs = x_batch_stride; a.x_ds = x_d_stride; a.dy_bs = dy_batch_stride; a.dy_ds = dy_d_stride; a.dx_bs = dx_batch_stride; a.dx_ds = dx_d_stride;
    const int qpr = seqlen / 4;
    if ((long long)batch * qpr * qpr >= (1LL << 32)) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d: batch * sequence too large");
    }
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            causal_conv1d_bwd_kernel<T, decltype(w)::value, decltype(act)::value><<<dim, kConvThreads, 0, (cudaStream_t)cuda_stream>>>(a, mia::div_magic(qpr));
        });
    });
    return mia::launched(mia::kErrConv, "causal_conv1d_bwd launch");
}

// ---- the fused inner block's kernels (see "tile kernels" above)
int mia_causal_conv1d_fwd_ex(const mia_bdl *x, const float *weight, const float *bias, const mia_bdl *ys, int n_ys, int batch, int dim,
                             int seqlen, int width, int silu, int dtype, void *cuda_stream) {
    const char *what = "causal_conv1d_fwd_ex";
    TileArgs a{};
    if (int rc = ex_check(what, a, batch, dim, seqlen, dtype, nullptr, 0, 0, ys, n_ys, 1)) return rc;
    if (!op_ok(x) || !weight || width < 1 || width > kMaxW) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: x and weight are required, width 1-4", what);
    }
    a.x = op_of(x); a.w = weight; a.bias = bias;
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            conv_fwd_ex_kernel<T, decltype(w)::value, decltype(act)::value><<<grid, kTileThreads, 0, st>>>(a);
        });
    });
    return mia::launched(mia::kErrConv, "causal_conv1d_fwd_ex launch");
}

size_t mia_causal_conv1d_bwd_ex_workspace(int batch, int dim, int seqlen, int width) {
    if (batch <= 0 || dim <= 0 || seqlen <= 0 || width < 1 || width > kMaxW) return 0;
    return (size_t)conv_bwd_parts(1, batch, dim, seqlen) * dim * (width + 1) * sizeof(float);
}

int mia_causal_conv1d_bwd_ex(const mia_bdl *x, const float *weight, const float *bias, const mia_bdl *dys, int n_dys, const mia_bdl *dx,
                             float *dweight, float *dbias, void *workspace, size_t workspace_bytes, int batch, int dim, int seqlen, int width,
                             int silu, int dtype, void *cuda_stream) {
    const char *what = "causal_conv1d_bwd_ex";
    TileArgs a{};
    if (int rc = ex_check(what, a, batch, dim, seqlen, dtype, dys, n_dys, 1, nullptr, 0, 0)) return rc;
    if (!op_ok(x) || !op_ok(dx) || !weight || !dweight || width < 1 || width > kMaxW) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: x, dx, weight and dweight are required, width 1-4", what);
    }
    if (!workspace || workspace_bytes < mia_causal_conv1d_bwd_ex_workspace(batch, dim, seqlen, width)) {
        return mia::fail(mia::kErrConv, MIA_EWORKSPACE, "%s: workspace missing or too small", what);
    }
    a.x = op_of(x); a.dx = op_of(dx); a.w = weight; a.bias = bias; a.dw = dweight; a.dbias = dbias; a.part = (float *)workspace;
    a.n_tt = (seqlen + kTT - 1) / kTT; a.parts = conv_bwd_parts(1, batch, dim, seqlen);
    const dim3 grid((dim + kTC - 1) / kTC, a.parts);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            conv_bwd_ex_kernel<T, decltype(w)::value, decltype(act)::value><<<grid, kTileThreads, 0, st>>>(a);
        });
    });
    if (int rc = mia::launched(mia::kErrConv, "causal_conv1d_bwd_ex launch")) return rc;
    conv_bwd_ex_finalize<<<(dim * (width + 1) + 255) / 256, 256, 0, st>>>(a, width);
    return mia::launched(mia::kErrConv, "causal_conv1d_bwd_ex finalize launch");
}

int mia_silu_gate_fwd_ex(const mia_bdl *outs, int n_outs, const mia_bdl *z, const mia_bdl *out_zs, int n_out_zs, int batch, int dim, int seqlen,
                         int dtype, void *cuda_stream) {
    const char *what = "silu_gate_fwd_ex";
    TileArgs a{};
    if (int rc = ex_check(what, a, batch, dim, seqlen, dtype, outs, n_outs, 1, out_zs, n_out_zs, 1)) return rc;
    if (!op_ok(z)) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: z is required", what);
    a.z = op_of(z);
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch);
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        gate_fwd_ex_kernel<T><<<grid, kTileThreads, 0, (cudaStream_t)cuda_stream>>>(a);
    });
    return mia::launched(mia::kErrConv, "silu_gate_fwd_ex launch");
}

int mia_silu_gate_bwd_ex(const mia_bdl *dy, const mia_bdl *outs, int n_outs, const mia_bdl *z, const mia_bdl *douts, int n_douts, const mia_bdl *dz,
                         int batch, int dim, int seqlen, int dtype, int dout_dtype, void *cuda_stream) {
    const char *what = "silu_gate_bwd_ex";
    if (dout_dtype != dtype && dout_dtype != MIA_F32) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: douts must have the call's dtype or float32", what);
    }
    TileArgs a{};
    mia_bdl in[kMaxOps];
    if (!op_ok(dy) || !op_ok(z) || !op_ok(dz) || !outs || n_outs < 1 || n_outs > kMaxOps - 1) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: dy, z, dz and 1-%d outs are required", what, kMaxOps - 1);
    }
    in[0] = *dy;
    for (int i = 0; i < n_outs; ++i) in[1 + i] = outs[i];
    if (int rc = ex_check(what, a, batch, dim, seqlen, dtype, in, 1 + n_outs, 2, douts, n_douts, 1)) return rc;
    a.z = op_of(z); a.dz = op_of(dz);
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch);
    const int smem = 3 * kTC * (kTT + 1) * (int)sizeof(float);
    const cudaError_t e = mia::dispatch_dtype<cudaError_t>(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        auto k = dout_dtype == MIA_F32 ? gate_bwd_ex_kernel<T, float> : gate_bwd_ex_kernel<T, T>;
        const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) k<<<grid, kTileThreads, smem, (cudaStream_t)cuda_stream>>>(a);
        return e;
    });
    if (int rc = mia::cuda_fail(mia::kErrConv, what, e)) return rc;
    return mia::launched(mia::kErrConv, "silu_gate_bwd_ex launch");
}

// ---- ARM's multi-direction (bimamba v3) kernels (see "scan orders" above)
int mia_causal_conv1d_fwd_dirs(const mia_bdl *x, const int *orders, int n_dirs, const float *weight, const float *bias, void *u,
                               const mia_bdl *u_tm, int batch, int dim, int seqlen, int width, int silu, int dtype, void *cuda_stream) {
    const char *what = "causal_conv1d_fwd_dirs";
    DirArgs a{};
    if (int rc = dirs_check(what, a, orders, n_dirs, batch, dim, seqlen, dtype)) return rc;
    if (!op_ok(x) || !weight || width < 1 || width > kMaxW || (!u && !u_tm)) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: x, weight and u or u_tm are required, width 1-4", what);
    }
    for (int k = 0; u_tm && k < n_dirs; ++k) {
        if (!op_ok(u_tm + k)) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: null u_tm operand", what);
        a.tm[k] = op_of(u_tm + k);
    }
    a.x = op_of(x); a.w = weight; a.bias = bias; a.dense_out = u; a.has_tm = u_tm != nullptr;
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch * n_dirs);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            conv_fwd_dirs_kernel<T, decltype(w)::value, decltype(act)::value><<<grid, kTileThreads, 0, st>>>(a);
        });
    });
    return mia::launched(mia::kErrConv, "causal_conv1d_fwd_dirs launch");
}

size_t mia_causal_conv1d_bwd_dirs_workspace(int n_dirs, int batch, int dim, int seqlen, int width) {
    if (n_dirs < 1 || n_dirs > kMaxDirs || batch <= 0 || dim <= 0 || seqlen <= 0 || width < 1 || width > kMaxW) return 0;
    return ((size_t)n_dirs * batch * dim * seqlen + (size_t)n_dirs * conv_bwd_parts(n_dirs, batch, dim, seqlen) * dim * (width + 1)) *
           sizeof(float);
}

int mia_causal_conv1d_bwd_dirs(const mia_bdl *x, const int *orders, int n_dirs, const float *weight, const float *bias, const void *du,
                               const mia_bdl *dy_tm, const mia_bdl *dx, float *dweight, float *dbias, void *workspace, size_t workspace_bytes,
                               int batch, int dim, int seqlen, int width, int silu, int dtype, void *cuda_stream) {
    const char *what = "causal_conv1d_bwd_dirs";
    DirArgs a{};
    if (int rc = dirs_check(what, a, orders, n_dirs, batch, dim, seqlen, dtype)) return rc;
    if (!op_ok(x) || !du || !op_ok(dx) || !weight || !dweight || width < 1 || width > kMaxW) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: x, du, dx, weight and dweight are required, width 1-4", what);
    }
    for (int k = 0; dy_tm && k < n_dirs; ++k) {
        if (!op_ok(dy_tm + k)) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: null dy_tm operand", what);
        a.tm[k] = op_of(dy_tm + k);
    }
    if (!workspace || workspace_bytes < mia_causal_conv1d_bwd_dirs_workspace(n_dirs, batch, dim, seqlen, width)) {
        return mia::fail(mia::kErrConv, MIA_EWORKSPACE, "%s: workspace missing or too small", what);
    }
    a.x = op_of(x); a.dx = op_of(dx); a.w = weight; a.bias = bias; a.dw = dweight; a.dbias = dbias; a.dense = du; a.has_tm = dy_tm != nullptr;
    a.xpart = (float *)workspace; a.part = a.xpart + (size_t)n_dirs * batch * dim * seqlen;
    a.n_tt = (seqlen + kTT - 1) / kTT; a.parts = conv_bwd_parts(n_dirs, batch, dim, seqlen);
    const dim3 grid((dim + kTC - 1) / kTC, a.parts, n_dirs), fgrid((dim + kTC - 1) / kTC, a.n_tt, batch);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        dispatch_conv(width, silu, [&](auto w, auto act) {
            conv_bwd_dirs_kernel<T, decltype(w)::value, decltype(act)::value><<<grid, kTileThreads, 0, st>>>(a);
        });
        if (cudaPeekAtLastError() == cudaSuccess) conv_bwd_dirs_finalize<T><<<fgrid, kTileThreads, 0, st>>>(a, width);
    });
    return mia::launched(mia::kErrConv, "causal_conv1d_bwd_dirs launch");
}

int mia_silu_gate_fwd_dirs(const void *outs, const int *orders, int n_dirs, int divisor, const mia_bdl *z, const mia_bdl *y, int batch, int dim,
                           int seqlen, int dtype, void *cuda_stream) {
    const char *what = "silu_gate_fwd_dirs";
    DirArgs a{};
    if (int rc = dirs_check(what, a, orders, n_dirs, batch, dim, seqlen, dtype)) return rc;
    if (!outs || !op_ok(z) || !op_ok(y) || divisor < 1) return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: outs, z, y and a divisor >= 1 are required", what);
    a.dense = outs; a.z = op_of(z); a.y = op_of(y); a.scale = 1.f / (float)divisor;
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch);
    mia::dispatch_dtype(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        gate_fwd_dirs_kernel<T><<<grid, kTileThreads, 0, (cudaStream_t)cuda_stream>>>(a);
    });
    return mia::launched(mia::kErrConv, "silu_gate_fwd_dirs launch");
}

int mia_silu_gate_bwd_dirs(const mia_bdl *dy, const void *outs, const int *orders, int n_dirs, int divisor, const mia_bdl *z, float *douts,
                           const mia_bdl *dz, int batch, int dim, int seqlen, int dtype, void *cuda_stream) {
    const char *what = "silu_gate_bwd_dirs";
    DirArgs a{};
    if (int rc = dirs_check(what, a, orders, n_dirs, batch, dim, seqlen, dtype)) return rc;
    if (!op_ok(dy) || !outs || !op_ok(z) || !douts || !op_ok(dz) || divisor < 1) {
        return mia::fail(mia::kErrConv, MIA_EINVAL, "%s: dy, outs, z, douts, dz and a divisor >= 1 are required", what);
    }
    a.y = op_of(dy); a.dense = outs; a.z = op_of(z); a.dense_out = douts; a.dz = op_of(dz); a.scale = 1.f / (float)divisor;
    const dim3 grid((dim + kTC - 1) / kTC, (seqlen + kTT - 1) / kTT, batch);
    const int smem = 3 * kTC * (kTT + 1) * (int)sizeof(float);
    const cudaError_t e = mia::dispatch_dtype<cudaError_t>(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        const cudaError_t e = cudaFuncSetAttribute(gate_bwd_dirs_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) gate_bwd_dirs_kernel<T><<<grid, kTileThreads, smem, (cudaStream_t)cuda_stream>>>(a);
        return e;
    });
    if (int rc = mia::cuda_fail(mia::kErrConv, what, e)) return rc;
    return mia::launched(mia::kErrConv, "silu_gate_bwd_dirs launch");
}

}  // extern "C"
