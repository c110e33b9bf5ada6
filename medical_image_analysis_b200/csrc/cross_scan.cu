// CrossScan / CrossMerge of VMamba's SS2D as single-pass sm_90a kernels.
//
// Reference: R2GenCSR/VMamba/classification/models/vmamba.py:25-67 (torch: 3-5 full-tensor copies each way) and
// csm_triton.py:7-235 (Triton; the north star forbids Triton).  One CTA stages a handful of (batch, channel) planes in
// shared memory and emits all four scan orders (row-major, column-major and their reversals) with coalesced global
// accesses; the merge is the exact adjoint (accumulated in fp32, rounded once).  HBM-bound: 1 read + 4 writes (scan),
// 4 reads + 1 write (merge) per element.
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/mia_selective_scan.h"
#include "abi_host.h"
#include "scan_common.cuh"

namespace {

constexpr int kPlanes = 4;      // planes per CTA (fewer when a plane is large: see launch_cs)
constexpr int kCsThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_scan_kernel(const typename mia::Cvt<T>::raw *__restrict__ x,
                                                                typename mia::Cvt<T>::raw *__restrict__ xs, int n_planes, int C,
                                                                int H, int W, int planes) {
    using raw = typename mia::Cvt<T>::raw;
    extern __shared__ __align__(16) char smem_raw[];
    raw *s = reinterpret_cast<raw *>(smem_raw);
    const int L = H * W;
    const int p0 = blockIdx.x * planes, np = min(planes, n_planes - p0);
    for (int i = threadIdx.x; i < np * L; i += kCsThreads) s[i] = x[(size_t)p0 * L + i];
    __syncthreads();
    for (int i = threadIdx.x; i < np * L; i += kCsThreads) {
        const int pl = i / L, l = i - pl * L;
        const int p = p0 + pl, b = p / C, c = p - b * C;
        const raw v = s[i];
        const raw vt = s[pl * L + (l % H) * W + l / H];      // column-major order: position l' = w * H + h holds x[h][w]
        raw *o = xs + ((size_t)b * 4 * C + c) * L;
        const size_t kstep = (size_t)C * L;
        o[l] = v;
        o[kstep + l] = vt;
        o[2 * kstep + (L - 1 - l)] = v;
        o[3 * kstep + (L - 1 - l)] = vt;
    }
}

template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_merge_kernel(const typename mia::Cvt<T>::raw *__restrict__ ys,
                                                                 typename mia::Cvt<T>::raw *__restrict__ y, int n_planes, int C,
                                                                 int H, int W, int planes) {
    using raw = typename mia::Cvt<T>::raw;
    extern __shared__ __align__(16) char smem_raw[];
    float *t = reinterpret_cast<float *>(smem_raw);          // column-major partial: ys1 + flip(ys3)
    const int L = H * W;
    const int p0 = blockIdx.x * planes, np = min(planes, n_planes - p0);
    const size_t kstep = (size_t)C * L;
    for (int i = threadIdx.x; i < np * L; i += kCsThreads) {
        const int pl = i / L, l = i - pl * L;
        const int p = p0 + pl, b = p / C, c = p - b * C;
        const raw *in = ys + ((size_t)b * 4 * C + c) * L;
        t[i] = mia::Cvt<T>::to_f(in[kstep + l]) + mia::Cvt<T>::to_f(in[3 * kstep + (L - 1 - l)]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < np * L; i += kCsThreads) {
        const int pl = i / L, l = i - pl * L;
        const int p = p0 + pl, b = p / C, c = p - b * C;
        const raw *in = ys + ((size_t)b * 4 * C + c) * L;
        const int h = l / W, w = l - h * W;
        const float v = mia::Cvt<T>::to_f(in[l]) + mia::Cvt<T>::to_f(in[2 * kstep + (L - 1 - l)]) + t[pl * L + w * H + h];
        y[(size_t)p * L + l] = mia::Cvt<T>::from_f(v);
    }
}

// ---- vectorised variants (L % 4 == 0, 4-element aligned tensors): 8- / 16-byte global accesses instead of one element per
// thread; the gathers of the column-major and reversed orders stay element-wise, but in shared memory.
constexpr int kPlanesVec = 8;

template <typename T> struct Q4;                 // 4 consecutive elements as one vector
template <> struct Q4<float> { using vec = uint4; };
template <> struct Q4<__half> { using vec = uint2; };
template <> struct Q4<__nv_bfloat16> { using vec = uint2; };

template <typename T>
__device__ __forceinline__ typename Q4<T>::vec pack4(typename mia::Cvt<T>::raw a, typename mia::Cvt<T>::raw b, typename mia::Cvt<T>::raw c,
                                                     typename mia::Cvt<T>::raw d) {
    if constexpr (sizeof(T) == 4) return make_uint4(a, b, c, d);
    else return make_uint2((uint32_t)a | ((uint32_t)b << 16), (uint32_t)c | ((uint32_t)d << 16));
}

__device__ __forceinline__ int cs_div(int i, uint32_t magic) { return magic ? (int)__umulhi((uint32_t)i, magic) : i; }

template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_scan_vec_kernel(const typename mia::Cvt<T>::raw *__restrict__ x,
                                                                    typename mia::Cvt<T>::raw *__restrict__ xs, int n_planes, int C,
                                                                    int H, int W, uint32_t magic_q, uint32_t magic_h, uint32_t magic_c, int planes) {
    using raw = typename mia::Cvt<T>::raw;
    using vec = typename Q4<T>::vec;
    extern __shared__ __align__(16) char smem_raw[];
    raw *s = reinterpret_cast<raw *>(smem_raw);
    const int L = H * W, Q = L >> 2;
    const int p0 = blockIdx.x * planes, np = min(planes, n_planes - p0);
    {
        const vec *gx = reinterpret_cast<const vec *>(x + (size_t)p0 * L);
        vec *sv = reinterpret_cast<vec *>(s);
        for (int i = threadIdx.x; i < np * Q; i += kCsThreads) sv[i] = gx[i];
    }
    __syncthreads();
    const size_t kstep = (size_t)C * L;
    for (int i = threadIdx.x; i < np * Q; i += kCsThreads) {
        const int pl = cs_div(i, magic_q), q = i - pl * Q, l0 = 4 * q;
        const int p = p0 + pl, b = cs_div(p, magic_c), c = p - b * C;
        const raw *sp = s + pl * L;
        raw t[4], r[4], tr[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int l = l0 + j, w = cs_div(l, magic_h), h = l - w * H;      // column-major position l holds x[h][w]
            t[j] = sp[h * W + w];
            const int lr = L - 1 - l, wr = cs_div(lr, magic_h), hr = lr - wr * H;
            r[j] = sp[lr];
            tr[j] = sp[hr * W + wr];
        }
        raw *o = xs + ((size_t)b * 4 * C + c) * L + l0;
        *reinterpret_cast<vec *>(o) = *reinterpret_cast<const vec *>(sp + l0);
        *reinterpret_cast<vec *>(o + kstep) = pack4<T>(t[0], t[1], t[2], t[3]);
        *reinterpret_cast<vec *>(o + 2 * kstep) = pack4<T>(r[0], r[1], r[2], r[3]);
        *reinterpret_cast<vec *>(o + 3 * kstep) = pack4<T>(tr[0], tr[1], tr[2], tr[3]);
    }
}

template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_merge_vec_kernel(const typename mia::Cvt<T>::raw *__restrict__ ys,
                                                                     typename mia::Cvt<T>::raw *__restrict__ y, int n_planes, int C,
                                                                     int H, int W, uint32_t magic_q, uint32_t magic_w, uint32_t magic_c, int planes) {
    using raw = typename mia::Cvt<T>::raw;
    using vec = typename Q4<T>::vec;
    extern __shared__ __align__(16) char smem_raw[];
    raw *s = reinterpret_cast<raw *>(smem_raw);               // [plane][direction][L]
    const int L = H * W, Q = L >> 2;
    const int p0 = blockIdx.x * planes, np = min(planes, n_planes - p0);
    const size_t kstep = (size_t)C * L;
    for (int i = threadIdx.x; i < np * 4 * Q; i += kCsThreads) {
        const int pd = cs_div(i, magic_q), q = i - pd * Q;      // pd = plane * 4 + direction
        const int pl = pd >> 2, k = pd & 3;
        const int p = p0 + pl, b = cs_div(p, magic_c), c = p - b * C;
        reinterpret_cast<vec *>(s)[i] = reinterpret_cast<const vec *>(ys + ((size_t)b * 4 * C + c) * L + k * kstep)[q];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < np * Q; i += kCsThreads) {
        const int pl = cs_div(i, magic_q), q = i - pl * Q, l0 = 4 * q;
        const raw *sp = s + (size_t)pl * 4 * L;
        raw o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int l = l0 + j, h = cs_div(l, magic_w), w = l - h * W, tl = w * H + h;   // x[h][w] sits at tl in the column-major orders
            const float v = mia::Cvt<T>::to_f(sp[l]) + mia::Cvt<T>::to_f(sp[2 * L + (L - 1 - l)]) + mia::Cvt<T>::to_f(sp[L + tl]) +
                            mia::Cvt<T>::to_f(sp[3 * L + (L - 1 - tl)]);
            o[j] = mia::Cvt<T>::from_f(v);
        }
        *reinterpret_cast<vec *>(y + (size_t)(p0 + pl) * L + l0) = pack4<T>(o[0], o[1], o[2], o[3]);
    }
}

// Planes too large for shared memory (H W > ~50 K elements): straight gathers from global memory, one element per thread.
// The column-major orders are strided reads (scan) / reads of two strided tensors (merge); correct for any size.
template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_scan_direct_kernel(const typename mia::Cvt<T>::raw *__restrict__ x,
                                                                       typename mia::Cvt<T>::raw *__restrict__ xs, long long total, int C,
                                                                       int H, int W) {
    using raw = typename mia::Cvt<T>::raw;
    const int L = H * W;
    const size_t kstep = (size_t)C * L;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / L;
        const int l = (int)(i - p * L);
        const int b = (int)(p / C), c = (int)(p - (long long)b * C);
        const raw *src = x + (size_t)p * L;
        const raw v = src[l], vt = src[(l % H) * W + l / H];
        raw *o = xs + ((size_t)b * 4 * C + c) * L;
        o[l] = v;
        o[kstep + l] = vt;
        o[2 * kstep + (L - 1 - l)] = v;
        o[3 * kstep + (L - 1 - l)] = vt;
    }
}

template <typename T>
__global__ void __launch_bounds__(kCsThreads) cross_merge_direct_kernel(const typename mia::Cvt<T>::raw *__restrict__ ys,
                                                                        typename mia::Cvt<T>::raw *__restrict__ y, long long total, int C,
                                                                        int H, int W) {
    using raw = typename mia::Cvt<T>::raw;
    const int L = H * W;
    const size_t kstep = (size_t)C * L;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / L;
        const int l = (int)(i - p * L);
        const int b = (int)(p / C), c = (int)(p - (long long)b * C);
        const raw *in = ys + ((size_t)b * 4 * C + c) * L;
        const int h = l / W, w = l - h * W, tl = w * H + h;
        const float v = mia::Cvt<T>::to_f(in[l]) + mia::Cvt<T>::to_f(in[2 * kstep + (L - 1 - l)]) + mia::Cvt<T>::to_f(in[kstep + tl]) +
                        mia::Cvt<T>::to_f(in[3 * kstep + (L - 1 - tl)]);
        y[(size_t)p * L + l] = mia::Cvt<T>::from_f(v);
    }
}

// out_z = out * silu(z): the gate of the mamba_ssm signature recomputed from the saved pre-gate output
// (selective_scan_cuda.bwd(..., recompute_out_z=True), test_selective_scan.py:105-108); fp32 arithmetic, one rounding.
template <typename T, typename TO>
__global__ void __launch_bounds__(256) silu_gate_kernel(const typename mia::Cvt<TO>::raw *__restrict__ out, const typename mia::Cvt<T>::raw *__restrict__ z,
                                                        typename mia::Cvt<TO>::raw *__restrict__ out_z, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float zv = mia::Cvt<T>::to_f(z[i]);
        const float y = mia::Cvt<TO>::to_f(out[i]);
        out_z[i] = mia::Cvt<TO>::from_f(y * zv * mia::rcpf(1.f + mia::ex2f(-zv * mia::kLog2e)));
    }
}

}  // namespace

// Defined ahead of the cross scan's launchers: the gate kernels are instantiated first, which fixes where they sit among
// the functions of the cubin.
extern "C" int mia_silu_gate(const void *out, const void *z, void *out_z, long long n, int z_dtype, int out_dtype, void *cuda_stream) {
    if (!out || !z || !out_z) return mia::fail(mia::kErrCs, MIA_EINVAL, "silu_gate: null pointer");
    if (n <= 0) return mia::fail(mia::kErrCs, MIA_EINVAL, "silu_gate: empty");
    if (out_dtype != z_dtype && out_dtype != MIA_F32) return mia::fail(mia::kErrCs, MIA_EINVAL, "silu_gate: out dtype must be z's dtype or float32");
    if (z_dtype != MIA_F32 && z_dtype != MIA_F16 && z_dtype != MIA_BF16)
        return mia::fail(mia::kErrCs, MIA_EINVAL, "silu_gate: dtype must be MIA_F32, MIA_F16 or MIA_BF16");
    cudaStream_t st = (cudaStream_t)cuda_stream;
    long long blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    const int g = (int)blocks;
#define MIA_GATE(T, TO) silu_gate_kernel<T, TO><<<g, 256, 0, st>>>((const typename mia::Cvt<TO>::raw *)out, (const typename mia::Cvt<T>::raw *)z, (typename mia::Cvt<TO>::raw *)out_z, n)
    mia::dispatch_dtype(z_dtype, [&](auto *tag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        if (out_dtype == MIA_F32) MIA_GATE(T, float); else MIA_GATE(T, T);
    });
#undef MIA_GATE
    return mia::launched(mia::kErrCs, "silu_gate launch");
}

namespace {

constexpr size_t kCsSmemMax = 200 * 1024;

template <typename T>
int launch_cs(bool merge, const void *in, void *out, int B, int C, int H, int W, cudaStream_t stream) {
    using raw = typename mia::Cvt<T>::raw;
    const int n_planes = B * C, L = H * W;
    const bool aligned = ((((uintptr_t)in | (uintptr_t)out) & (4 * sizeof(raw) - 1)) == 0);
    // planes per CTA: as many as fit (8 for the 14 x 14 ... 56 x 56 maps of the models, fewer for large maps)
    const size_t vplane = (size_t)L * sizeof(raw) * (merge ? 4 : 1);
    int vplanes = (int)(kCsSmemMax / vplane);
    if (vplanes > kPlanesVec) vplanes = kPlanesVec;
    if ((L % 4) == 0 && aligned && vplanes >= 1 && (long long)vplanes * L * L < (1LL << 32) / 4 &&
        (long long)n_planes * C < (1LL << 32)) {   // ranges in which the multiply-high divisions are exact
        const size_t vsmem = vplane * vplanes;
        const int grid = (n_planes + vplanes - 1) / vplanes;
        if (merge) {
            auto k = &cross_merge_vec_kernel<T>;
            if (vsmem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vsmem) != cudaSuccess)
                return mia::launched(mia::kErrCs, "cross_merge: cudaFuncSetAttribute");
            k<<<grid, kCsThreads, vsmem, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), n_planes, C, H, W,
                                                  mia::div_magic(L / 4), mia::div_magic(W), mia::div_magic(C), vplanes);
        } else {
            auto k = &cross_scan_vec_kernel<T>;
            if (vsmem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vsmem) != cudaSuccess)
                return mia::launched(mia::kErrCs, "cross_scan: cudaFuncSetAttribute");
            k<<<grid, kCsThreads, vsmem, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), n_planes, C, H, W,
                                                  mia::div_magic(L / 4), mia::div_magic(H), mia::div_magic(C), vplanes);
        }
        return mia::launched(mia::kErrCs, merge ? "cross_merge launch" : "cross_scan launch");
    }
    const size_t plane = (size_t)L * (merge ? sizeof(float) : sizeof(raw));
    int planes = (int)(kCsSmemMax / plane);
    if (planes > kPlanes) planes = kPlanes;
    if (planes >= 1) {
        const size_t smem = plane * planes;
        const int grid = (n_planes + planes - 1) / planes;
        if (merge) {
            auto k = &cross_merge_kernel<T>;
            if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
                return mia::launched(mia::kErrCs, "cross_merge: cudaFuncSetAttribute");
            k<<<grid, kCsThreads, smem, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), n_planes, C, H, W, planes);
        } else {
            auto k = &cross_scan_kernel<T>;
            if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
                return mia::launched(mia::kErrCs, "cross_scan: cudaFuncSetAttribute");
            k<<<grid, kCsThreads, smem, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), n_planes, C, H, W, planes);
        }
        return mia::launched(mia::kErrCs, merge ? "cross_merge launch" : "cross_scan launch");
    }
    // a single plane exceeds shared memory: direct gathers
    const long long total = (long long)n_planes * L;
    long long blocks = (total + kCsThreads - 1) / kCsThreads;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (merge) cross_merge_direct_kernel<T><<<(int)blocks, kCsThreads, 0, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), total, C, H, W);
    else cross_scan_direct_kernel<T><<<(int)blocks, kCsThreads, 0, stream>>>(reinterpret_cast<const raw *>(in), reinterpret_cast<raw *>(out), total, C, H, W);
    return mia::launched(mia::kErrCs, merge ? "cross_merge (direct) launch" : "cross_scan (direct) launch");
}

int cs_dispatch(bool merge, const void *in, void *out, int B, int C, int H, int W, int dtype, void *stream) {
    if (!in || !out) return mia::fail(mia::kErrCs, MIA_EINVAL, "cross scan / merge: null pointer");
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return mia::fail(mia::kErrCs, MIA_EINVAL, "cross scan / merge: empty or negative size");
    if ((long long)H * W > (1LL << 30)) return mia::fail(mia::kErrCs, MIA_EINVAL, "cross scan / merge: H * W too large");
    if (dtype != MIA_F32 && dtype != MIA_F16 && dtype != MIA_BF16)
        return mia::fail(mia::kErrCs, MIA_EINVAL, "cross scan / merge: dtype must be MIA_F32, MIA_F16 or MIA_BF16");
    return mia::dispatch_dtype<int>(dtype, [&](auto *tag) {
        return launch_cs<std::remove_pointer_t<decltype(tag)>>(merge, in, out, B, C, H, W, (cudaStream_t)stream);
    });
}

}  // namespace

extern "C" {
int mia_cross_scan(const void *x, void *xs, int batch, int channels, int H, int W, int dtype, void *cuda_stream) {
    return cs_dispatch(false, x, xs, batch, channels, H, W, dtype, cuda_stream);
}
int mia_cross_merge(const void *ys, void *y, int batch, int channels, int H, int W, int dtype, void *cuda_stream) {
    return cs_dispatch(true, ys, y, batch, channels, H, W, dtype, cuda_stream);
}
}  // extern "C"
