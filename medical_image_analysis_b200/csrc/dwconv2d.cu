// Depth-wise 3x3 conv2d (+ bias, + SiLU) of SS2D, forward and backward, as sm_90a kernels.
//
// Reference: `x = self.act(self.conv2d(x))` with `nn.Conv2d(d_inner, d_inner, groups=d_inner, kernel_size=3, padding=1)`
// on channel-first (B, C, H, W) activations (R2GenCSR/VMamba/classification/models/vmamba.py:574-582, 1120-1122).
//     pre[b, c, h, w] = bias[c] + sum_{i, j in 0..2} wgt[c, i, j] * x[b, c, h + i - 1, w + j - 1]     y = pre * sigmoid(pre)
// HBM-bound (2 tensor passes forward, 3 backward).  A (batch, channel) plane is contiguous: planes are staged whole in
// shared memory (as fp32 with a zero border, so the 3x3 stencil is nine unpredicated loads) with 4-element global accesses.
// Backward = one CTA per channel over all the batch planes of the channel: d pre goes through shared memory for the
// transposed stencil (dx), dweight[c, :, :] and dbias[c] are reduced in registers -> shared memory -> one write:
// deterministic, no atomics.
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/mia_selective_scan.h"
#include "abi_host.h"
#include "scan_common.cuh"

namespace {

constexpr int kDwThreads = 256;

struct DwArgs {
    const void *x, *dy;
    void *y, *dx;
    const float *w, *bias;      // (C, 9) / (C) fp32, bias may be null
    float *dw, *dbias;
    int batch, C, H, W, silu;
    int planes_per_block;       // forward: planes staged per block pass; backward: batch planes per pass
    uint32_t magic_hw, magic_w; // multiply-high reciprocals of H*W and W (0: divisor 1)
};

__device__ __forceinline__ int fast_div(int i, uint32_t magic) { return magic ? (int)__umulhi((uint32_t)i, magic) : i; }
__device__ __forceinline__ float dw_sigmoid(float v) { return mia::rcpf(1.f + mia::ex2f(-v * mia::kLog2e)); }

// kV consecutive elements <-> floats (kV = 4: one 8- / 16-byte access; kV = 1: element-wise, any H*W and alignment)
template <typename T, int kV> struct Pack {
    using raw = typename mia::Cvt<T>::raw;
    static __device__ __forceinline__ void ld(const raw *p, float (&f)[kV]) {
        if constexpr (kV == 1) {
            f[0] = mia::Cvt<T>::to_f(p[0]);
        } else if constexpr (sizeof(T) == 4) {
            const float4 v = *reinterpret_cast<const float4 *>(p);
            f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
        } else {
            const uint2 v = *reinterpret_cast<const uint2 *>(p);
            f[0] = mia::Cvt<T>::to_f((raw)(v.x & 0xffffu)); f[1] = mia::Cvt<T>::to_f((raw)(v.x >> 16));
            f[2] = mia::Cvt<T>::to_f((raw)(v.y & 0xffffu)); f[3] = mia::Cvt<T>::to_f((raw)(v.y >> 16));
        }
    }
    static __device__ __forceinline__ void st(raw *p, const float (&f)[kV]) {
        if constexpr (kV == 1) {
            p[0] = mia::Cvt<T>::from_f(f[0]);
        } else if constexpr (sizeof(T) == 4) {
            *reinterpret_cast<float4 *>(p) = make_float4(f[0], f[1], f[2], f[3]);
        } else {
            const uint32_t a = (uint32_t)mia::Cvt<T>::from_f(f[0]) | ((uint32_t)mia::Cvt<T>::from_f(f[1]) << 16);
            const uint32_t b = (uint32_t)mia::Cvt<T>::from_f(f[2]) | ((uint32_t)mia::Cvt<T>::from_f(f[3]) << 16);
            *reinterpret_cast<uint2 *>(p) = make_uint2(a, b);
        }
    }
};

// Planes live in shared memory as fp32 with a one-element zero border, (H + 2) x (W + 2): the 3x3 stencil is nine
// unpredicated loads at fixed offsets.
__device__ __forceinline__ float stencil9(const float *c, int Wp, const float (&k)[9], float acc, float (&v)[9]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            v[i * 3 + j] = c[(i - 1) * Wp + (j - 1)];
            acc = fmaf(k[i * 3 + j], v[i * 3 + j], acc);
        }
    return acc;
}

__device__ __forceinline__ void zero_planes(float *s, int n) {
    for (int i = threadIdx.x; i < n; i += kDwThreads) s[i] = 0.f;
}

// Every pass of a block: (A) 4-element global loads -> bordered fp32 planes (and the raw dy planes of the backward);
// (B) ONE ELEMENT PER THREAD stencil work -- consecutive lanes read consecutive shared-memory words, no bank conflicts
// (4 elements per thread would put lanes 4 words apart) -- results staged in shared memory in the tensor's dtype;
// (C) 4-element copies of the staged results to global memory.

// copy np * HW elements global -> bordered fp32 planes
template <typename T, int kV>
__device__ __forceinline__ void load_planes(const typename mia::Cvt<T>::raw *g, size_t plane_stride, float *sx, int np, int HW, int W, int Wp,
                                            int PS, uint32_t magic_hw, uint32_t magic_w) {
    for (int i = threadIdx.x * kV; i < np * HW; i += kDwThreads * kV) {
        const int pl = fast_div(i, magic_hw);
        int l = i - pl * HW, h = fast_div(l, magic_w), w = l - h * W;
        float f[kV];
        Pack<T, kV>::ld(g + (size_t)pl * plane_stride + l, f);
#pragma unroll
        for (int j = 0; j < kV; ++j) {
            sx[pl * PS + (h + 1) * Wp + (w + 1)] = f[j];
            if (++w == W) { w = 0; ++h; }
        }
    }
}

// copy np * HW staged elements (raw T in shared memory, [plane][HW]) -> global
template <typename T, int kV>
__device__ __forceinline__ void store_planes(typename mia::Cvt<T>::raw *g, size_t plane_stride, const typename mia::Cvt<T>::raw *so, int np,
                                             int HW, uint32_t magic_hw) {
    using raw = typename mia::Cvt<T>::raw;
    for (int i = threadIdx.x * kV; i < np * HW; i += kDwThreads * kV) {
        const int pl = fast_div(i, magic_hw), l = i - pl * HW;
        raw *dst = g + (size_t)pl * plane_stride + l;
        if constexpr (kV == 1) dst[0] = so[i];
        else if constexpr (sizeof(T) == 4) *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<const uint4 *>(so + i);
        else *reinterpret_cast<uint2 *>(dst) = *reinterpret_cast<const uint2 *>(so + i);
    }
}

// The forward's dynamic shared memory, offsets in floats from its base: sx [P][(H + 2) (W + 2)], taps [P][12] (10 used),
// so [P][HW] staged results in the tensor's dtype.  sx is rounded up to 4 floats so that taps and so start on 16-byte
// boundaries for every shape: the vector path copies so out as uint4.
struct DwFwdSmem {
    int taps, so;
    size_t bytes;
};
__host__ __device__ __forceinline__ DwFwdSmem dw_fwd_smem(int P, int H, int W, int es) {
    const int sx = (P * (H + 2) * (W + 2) + 3) & ~3;
    return {sx, sx + P * 12, (size_t)(sx + P * 12) * sizeof(float) + (size_t)P * H * W * es};
}

// ------------------------------------------------------------------------------------------------ forward
template <typename T, bool kSilu, int kV>
__global__ void __launch_bounds__(kDwThreads) dwconv2d_fwd_kernel(const DwArgs a) {
    using raw = typename mia::Cvt<T>::raw;
    extern __shared__ __align__(16) char dsm[];
    const int H = a.H, W = a.W, HW = H * W, Wp = W + 2, PS = (H + 2) * Wp, P = a.planes_per_block;
    const DwFwdSmem lay = dw_fwd_smem(P, H, W, (int)sizeof(raw));
    float *sx = reinterpret_cast<float *>(dsm);
    float *taps = sx + lay.taps;
    raw *so = reinterpret_cast<raw *>(sx + lay.so);
    const int n_planes = a.batch * a.C;
    zero_planes(sx, P * PS);                                  // the borders stay zero for the whole kernel
    __syncthreads();
    for (int p0 = blockIdx.x * P; p0 < n_planes; p0 += gridDim.x * P) {
        const int np = min(P, n_planes - p0);
        load_planes<T, kV>(reinterpret_cast<const raw *>(a.x) + (size_t)p0 * HW, HW, sx, np, HW, W, Wp, PS, a.magic_hw, a.magic_w);
        for (int i = threadIdx.x; i < np * 10; i += kDwThreads) {
            const int pl = i / 10, k = i - pl * 10, c = (p0 + pl) % a.C;
            taps[pl * 12 + k] = k < 9 ? __ldg(a.w + (size_t)c * 9 + k) : (a.bias ? __ldg(a.bias + c) : 0.f);
        }
        __syncthreads();
        // a warp takes whole planes when there are enough of them (taps stay in registers for the plane), else the block
        // walks each plane together
        const int wstep = P >= kDwThreads / 32 ? kDwThreads / 32 : 1, lstep = wstep > 1 ? 32 : kDwThreads;
        for (int pl = wstep > 1 ? (int)(threadIdx.x >> 5) : 0; pl < np; pl += wstep) {
            float k[9], v[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) k[t] = taps[pl * 12 + t];
            const float bias = taps[pl * 12 + 9];
            for (int l = wstep > 1 ? (int)(threadIdx.x & 31) : (int)threadIdx.x; l < HW; l += lstep) {
                const int h = fast_div(l, a.magic_w), w = l - h * W;
                const float pre = stencil9(sx + pl * PS + (h + 1) * Wp + (w + 1), Wp, k, bias, v);
                so[pl * HW + l] = mia::Cvt<T>::from_f(kSilu ? pre * dw_sigmoid(pre) : pre);
            }
        }
        __syncthreads();
        store_planes<T, kV>(reinterpret_cast<raw *>(a.y) + (size_t)p0 * HW, HW, so, np, HW, a.magic_hw);
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ backward
template <typename T, bool kSilu, int kV>
__global__ void __launch_bounds__(kDwThreads) dwconv2d_bwd_kernel(const DwArgs a) {
    using raw = typename mia::Cvt<T>::raw;
    extern __shared__ __align__(16) char dsm[];
    __shared__ float red[kDwThreads / 32][10];
    const int H = a.H, W = a.W, HW = H * W, Wp = W + 2, PS = (H + 2) * Wp, P = a.planes_per_block;
    float *sx = reinterpret_cast<float *>(dsm);               // [P][(H + 2) (W + 2)] x
    float *sdp = sx + (size_t)P * PS;                         // same layout: d pre
    raw *sio = reinterpret_cast<raw *>(sdp + (size_t)P * PS); // [P][HW]: dy on the way in, dx on the way out
    const int c = blockIdx.x;
    float k[9], acc[10];
#pragma unroll
    for (int t = 0; t < 9; ++t) { k[t] = __ldg(a.w + (size_t)c * 9 + t); acc[t] = 0.f; }
    acc[9] = 0.f;
    const float bias = a.bias ? __ldg(a.bias + c) : 0.f;
    zero_planes(sx, 2 * P * PS);
    __syncthreads();
    const size_t pstride = (size_t)a.C * HW;                  // from one batch plane of the channel to the next
    for (int b0 = 0; b0 < a.batch; b0 += P) {
        const int np = min(P, a.batch - b0);
        const size_t goff = ((size_t)b0 * a.C + c) * HW;
        load_planes<T, kV>(reinterpret_cast<const raw *>(a.x) + goff, pstride, sx, np, HW, W, Wp, PS, a.magic_hw, a.magic_w);
        for (int i = threadIdx.x * kV; i < np * HW; i += kDwThreads * kV) {      // dy: raw copy
            const int pl = fast_div(i, a.magic_hw), l = i - pl * HW;
            const raw *src = reinterpret_cast<const raw *>(a.dy) + goff + (size_t)pl * pstride + l;
            if constexpr (kV == 1) sio[i] = src[0];
            else if constexpr (sizeof(T) == 4) *reinterpret_cast<uint4 *>(sio + i) = *reinterpret_cast<const uint4 *>(src);
            else *reinterpret_cast<uint2 *>(sio + i) = *reinterpret_cast<const uint2 *>(src);
        }
        __syncthreads();
        // d pre = dy * silu'(pre) into its own bordered plane; dweight / dbias partial sums from the same nine x values
        for (int i = threadIdx.x; i < np * HW; i += kDwThreads) {
            const int pl = fast_div(i, a.magic_hw), l = i - pl * HW, h = fast_div(l, a.magic_w), w = l - h * W;
            const int o = pl * PS + (h + 1) * Wp + (w + 1);
            float v[9];
            const float pre = stencil9(sx + o, Wp, k, bias, v);
            float gg = mia::Cvt<T>::to_f(sio[i]);
            if (kSilu) {
                const float s = dw_sigmoid(pre);
                gg *= s * fmaf(pre, 1.f - s, 1.f);
            }
            sdp[o] = gg;
            acc[9] += gg;
#pragma unroll
            for (int t = 0; t < 9; ++t) acc[t] = fmaf(gg, v[t], acc[t]);
        }
        __syncthreads();
        // dx[h, w] = sum_{i, j} wgt[i, j] * d pre[h - i + 1, w - j + 1]   (transposed stencil = stencil with flipped taps)
        for (int i = threadIdx.x; i < np * HW; i += kDwThreads) {
            const int pl = fast_div(i, a.magic_hw), l = i - pl * HW, h = fast_div(l, a.magic_w), w = l - h * W;
            const float *cdp = sdp + pl * PS + (h + 1) * Wp + (w + 1);
            float v = 0.f;
#pragma unroll
            for (int ii = 0; ii < 3; ++ii)
#pragma unroll
                for (int jj = 0; jj < 3; ++jj) v = fmaf(k[ii * 3 + jj], cdp[(1 - ii) * Wp + (1 - jj)], v);
            sio[i] = mia::Cvt<T>::from_f(v);
        }
        __syncthreads();
        store_planes<T, kV>(reinterpret_cast<raw *>(a.dx) + goff, pstride, sio, np, HW, a.magic_hw);
        __syncthreads();
    }
    // block reduction in a fixed order: lanes (shuffle tree), then warps
#pragma unroll
    for (int v = 0; v < 10; ++v) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], off);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
#pragma unroll
        for (int v = 0; v < 10; ++v) red[warp][v] = acc[v];
    }
    __syncthreads();
    if (threadIdx.x < 10) {
        float s = 0.f;
        for (int wv = 0; wv < kDwThreads / 32; ++wv) s += red[wv][threadIdx.x];
        if (threadIdx.x == 9) {
            if (a.dbias) a.dbias[c] = s;
        } else {
            a.dw[(size_t)c * 9 + threadIdx.x] = s;
        }
    }
}

constexpr size_t kDwSmemMax = 227 * 1024;   // sm_90's opt-in limit of dynamic shared memory per block

size_t dw_bwd_smem(int P, int H, int W, int es) { return (size_t)2 * P * (H + 2) * (W + 2) * sizeof(float) + (size_t)P * H * W * es; }

// Validates the call and sizes its blocks: P planes per block (forward: staged per pass, at most 16; backward: batch planes
// per pass) and the dynamic shared memory they take.  Thin planes do not fit (a 1 x 16384 fp32 forward, a 4 x 4096 fp32
// backward): they are rejected here, before any CUDA call.
int dw_check(const void *x, int batch, int C, int H, int W, int dtype, bool bwd, int &P, size_t &smem) {
    if (!x || batch <= 0 || C <= 0 || H <= 0 || W <= 0) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d: empty or null input");
    if (dtype != MIA_F32 && dtype != MIA_F16 && dtype != MIA_BF16) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d: bad dtype");
    if ((long long)H * W > 16384) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d: planes larger than 16384 elements are not supported");
    if ((long long)batch * C >= (1LL << 31) / 2) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d: batch*channels too large");
    const int es = dtype == MIA_F32 ? 4 : 2;
    P = 2048 / (H * W);
    if (P < 1) P = 1;
    if (P > (bwd ? batch : 16)) P = bwd ? batch : 16;
    smem = bwd ? dw_bwd_smem(P, H, W, es) : dw_fwd_smem(P, H, W, es).bytes;
    if (smem > kDwSmemMax) {
        return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d_%s: a %d x %d %s plane needs %zu bytes of shared memory per block, "
                         "more than the %zu-byte (227 KB) limit", bwd ? "bwd" : "fwd", H, W, es == 4 ? "float32" : "16-bit", smem, kDwSmemMax);
    }
    return MIA_OK;
}

}  // namespace

extern "C" {

int mia_dwconv2d_fwd(const void *x, const float *weight, const float *bias, void *y, int batch, int channels, int H, int W, int silu,
                     int dtype, void *cuda_stream) {
    int P;
    size_t smem;
    if (int rc = dw_check(x, batch, channels, H, W, dtype, false, P, smem)) return rc;
    if (!weight || !y) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d_fwd: null weight or y");
    const int es = dtype == MIA_F32 ? 4 : 2, HW = H * W;
    DwArgs a{};
    a.x = x; a.y = y; a.w = weight; a.bias = bias; a.batch = batch; a.C = channels; a.H = H; a.W = W; a.silu = silu;
    a.planes_per_block = P;
    a.magic_hw = mia::div_magic(HW); a.magic_w = mia::div_magic(W);
    const bool vec = (HW % 4) == 0 && ((((uintptr_t)x | (uintptr_t)y) & (4 * es - 1)) == 0);
    const long long n_planes = (long long)batch * channels;
    long long blocks = (n_planes + P - 1) / P;
    mia::DeviceInfo di;
    if (int rc = mia::device_info(mia::kErrDw, di)) return rc;
    if (blocks > (long long)di.sms * 16) blocks = (long long)di.sms * 16;
    const cudaError_t e = mia::dispatch_dtype<cudaError_t>(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        void (*kern)(const DwArgs);
        if (vec) kern = silu ? &dwconv2d_fwd_kernel<T, true, 4> : &dwconv2d_fwd_kernel<T, false, 4>;
        else kern = silu ? &dwconv2d_fwd_kernel<T, true, 1> : &dwconv2d_fwd_kernel<T, false, 1>;
        if (smem > 48 * 1024)
            if (const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
        kern<<<(int)blocks, kDwThreads, smem, (cudaStream_t)cuda_stream>>>(a);
        return cudaGetLastError();
    });
    return mia::cuda_fail(mia::kErrDw, "dwconv2d_fwd launch", e);
}

int mia_dwconv2d_bwd(const void *x, const float *weight, const float *bias, const void *dy, void *dx, float *dweight, float *dbias,
                     int batch, int channels, int H, int W, int silu, int dtype, void *cuda_stream) {
    int P;
    size_t smem;
    if (int rc = dw_check(x, batch, channels, H, W, dtype, true, P, smem)) return rc;
    if (!weight || !dy || !dx || !dweight) return mia::fail(mia::kErrDw, MIA_EINVAL, "dwconv2d_bwd: null pointer");
    const int es = dtype == MIA_F32 ? 4 : 2, HW = H * W;
    DwArgs a{};
    a.x = x; a.dy = dy; a.dx = dx; a.w = weight; a.bias = bias; a.dw = dweight; a.dbias = dbias;
    a.batch = batch; a.C = channels; a.H = H; a.W = W; a.silu = silu;
    a.planes_per_block = P;
    a.magic_hw = mia::div_magic(HW); a.magic_w = mia::div_magic(W);
    const bool vec = (HW % 4) == 0 && ((((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dx) & (4 * es - 1)) == 0);
    const cudaError_t e = mia::dispatch_dtype<cudaError_t>(dtype, [&](auto *tag) {
        using T = typename std::remove_pointer<decltype(tag)>::type;
        void (*kern)(const DwArgs);
        if (vec) kern = silu ? &dwconv2d_bwd_kernel<T, true, 4> : &dwconv2d_bwd_kernel<T, false, 4>;
        else kern = silu ? &dwconv2d_bwd_kernel<T, true, 1> : &dwconv2d_bwd_kernel<T, false, 1>;
        if (smem > 48 * 1024)
            if (const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
        kern<<<channels, kDwThreads, smem, (cudaStream_t)cuda_stream>>>(a);
        return cudaGetLastError();
    });
    return mia::cuda_fail(mia::kErrDw, "dwconv2d_bwd launch", e);
}

}  // extern "C"
