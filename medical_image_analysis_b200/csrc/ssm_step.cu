// Decode-step kernels of the Mamba mixers (sm_90a): one token of the selective scan with the state updated in place
// (mamba_ssm's selective_state_update, the torch branch of Mamba.step at arm/Finetuning/mamba_simple.py:747-755) and one
// token of the depth-wise causal conv1d (causal_conv1d_update, :724-738).
//
// selective_state_update is bound by the state bytes at large batch (read + write of batch x dim x dstate) and by
// launch latency at small batch, so the layout is chosen for the former and the call is one launch for the latter.
// A CTA owns one batch entry and a run of consecutive channel rows; B[b, :] and C[b, :] are staged once per CTA in
// shared memory as fp32.  LPR lanes (a power of two, up to 32) share one state row: when a row is a whole number of
// 16-byte vectors (and the strides keep them aligned) every lane moves 16 bytes per access, so a warp covers 32 / LPR
// consecutive rows and each access is coalesced (d_state 16 f32: 4 lanes per row, 8 rows per warp); other rows (d_state
// 1, odd d_state, unaligned strides) go element by element.  sum_n state C is a shuffle reduction over the row's lanes.
// Arithmetic is the scan kernels' (scan_fwd.cuh): softplus_f, A pre-multiplied by log2 e into ex2, the silu gate of
// the z path, so a step continues a prefill's last_state with the same numerics.
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/mia_selective_scan.h"
#include "abi_host.h"
#include "scan_common.cuh"

namespace {

using mia::Cvt;
using mia::kLog2e;

constexpr int kStepThreads = 128;
constexpr int kMaxN = 256;
constexpr int kConvStepThreads = 128;
constexpr int kMaxConvW = 4;

struct SsuArgs {
    void *state;
    const void *x, *dt, *z, *B, *C, *D, *bias;
    const float *A;
    void *out;
    long long s_bs, s_ds, x_bs, dt_bs, z_bs, B_bs, C_bs, out_bs, A_ds, A_ns;
    int batch, dim, N, lpr_log2, rows_per_cta, softplus, D_type, bias_type;
};

template <typename T>
__device__ __forceinline__ float ld1(const void *p, long long i) {
    return Cvt<T>::to_f(__ldg(reinterpret_cast<const typename Cvt<T>::raw *>(p) + i));
}

// a (dim)-vector parameter in whichever dtype it arrives (D, dt_bias, conv weight / bias): a warp-uniform branch
__device__ __forceinline__ float ld_any(const void *p, long long i, int dtype) {
    if (dtype == MIA_F32) return ld1<float>(p, i);
    if (dtype == MIA_F16) return ld1<__half>(p, i);
    return ld1<__nv_bfloat16>(p, i);
}

template <typename T>
__device__ __forceinline__ float round_to(float v) { return Cvt<T>::to_f(Cvt<T>::from_f(v)); }

// E consecutive state elements <-> float[E]: one 16-byte access when E * sizeof(T) == 16, else E == 1
template <typename T, int E>
__device__ __forceinline__ void ld_state(const char *p, float (&f)[E]) {
    if constexpr (E == 1) {
        f[0] = Cvt<T>::to_f(*reinterpret_cast<const typename Cvt<T>::raw *>(p));
    } else {
        const uint4 v = *reinterpret_cast<const uint4 *>(p);
        const typename Cvt<T>::raw *r = reinterpret_cast<const typename Cvt<T>::raw *>(&v);
#pragma unroll
        for (int e = 0; e < E; ++e) f[e] = Cvt<T>::to_f(r[e]);
    }
}
template <typename T, int E>
__device__ __forceinline__ void st_state(char *p, const float (&f)[E]) {
    if constexpr (E == 1) {
        *reinterpret_cast<typename Cvt<T>::raw *>(p) = Cvt<T>::from_f(f[0]);
    } else {
        uint4 v;
        typename Cvt<T>::raw *r = reinterpret_cast<typename Cvt<T>::raw *>(&v);
#pragma unroll
        for (int e = 0; e < E; ++e) r[e] = Cvt<T>::from_f(f[e]);
        *reinterpret_cast<uint4 *>(p) = v;
    }
}

template <typename TS, typename TI, bool kVec>
__global__ void __launch_bounds__(kStepThreads) ss_step_kernel(const SsuArgs a) {
    constexpr int E = kVec ? 16 / (int)sizeof(TS) : 1;      // state elements per access
    __shared__ float sB[kMaxN], sC[kMaxN];
    const int b = blockIdx.y;
    for (int n = threadIdx.x; n < a.N; n += kStepThreads) {
        sB[n] = ld1<TI>(a.B, (long long)b * a.B_bs + n);
        sC[n] = ld1<TI>(a.C, (long long)b * a.C_bs + n);
    }
    __syncthreads();
    const int lpr = 1 << a.lpr_log2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = lane & (lpr - 1);                           // lane within the row
    const int d = blockIdx.x * a.rows_per_cta + (warp << (5 - a.lpr_log2)) + (lane >> a.lpr_log2);
    const bool valid = d < a.dim;
    const int dd = valid ? d : a.dim - 1;                     // rows past the end still take part in the shuffles
    const float xv = ld1<TI>(a.x, (long long)b * a.x_bs + dd);
    float m = ld1<TI>(a.dt, (long long)b * a.dt_bs + dd);
    if (a.bias) m += ld_any(a.bias, dd, a.bias_type);
    if (a.softplus) {
        float unused;
        m = mia::softplus_f<false>(m, unused);
    }
    const float mx = m * xv;
    char *row = (char *)a.state + ((size_t)b * a.s_bs + (size_t)dd * a.s_ds) * sizeof(TS);
    const float *Ar = a.A + (size_t)dd * a.A_ds;
    const int units = a.N / E;
    float acc = 0.f;
    for (int u = j; u < units; u += lpr) {
        float h[E];
        ld_state<TS, E>(row + (size_t)u * E * sizeof(TS), h);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int n = u * E + e;
            const float dA = mia::ex2f(m * (__ldg(Ar + (size_t)n * a.A_ns) * kLog2e));
            h[e] = round_to<TS>(fmaf(dA, h[e], mx * sB[n]));
            acc = fmaf(h[e], sC[n], acc);
        }
        if (valid) st_state<TS, E>(row + (size_t)u * E * sizeof(TS), h);
    }
    for (int off = lpr >> 1; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (valid && j == 0) {
        float y = acc;
        if (a.D) y = fmaf(ld_any(a.D, d, a.D_type), xv, y);
        if (a.z) {
            const float zv = ld1<TI>(a.z, (long long)b * a.z_bs + d);
            y = y * zv * mia::rcpf(1.f + mia::ex2f(-zv * kLog2e));
        }
        reinterpret_cast<typename Cvt<TI>::raw *>(a.out)[(size_t)b * a.out_bs + d] = Cvt<TI>::from_f(y);
    }
}

struct ConvStepArgs {
    const void *x, *w, *bias;
    void *state, *out;
    long long x_bs, s_bs, s_ds, s_ws, w_ds, w_ws, out_bs;
    int batch, dim, width, silu, w_type, bias_type;
};

// one thread per (batch, channel): shift the row left, append x, dot with the taps
template <typename TX, typename TS>
__global__ void __launch_bounds__(kConvStepThreads) causal_conv1d_update_kernel(const ConvStepArgs a) {
    const int d = blockIdx.x * kConvStepThreads + threadIdx.x, b = blockIdx.y;
    if (d >= a.dim) return;
    using RS = typename Cvt<TS>::raw;
    RS *s = reinterpret_cast<RS *>(a.state) + (size_t)b * a.s_bs + (size_t)d * a.s_ds;
    float v[kMaxConvW];
#pragma unroll
    for (int k = 0; k < kMaxConvW; ++k)
        if (k + 1 < a.width) v[k] = Cvt<TS>::to_f(s[(size_t)(k + 1) * a.s_ws]);
    const RS xs = Cvt<TS>::from_f(ld1<TX>(a.x, (long long)b * a.x_bs + d));
    float acc = a.bias ? ld_any(a.bias, d, a.bias_type) : 0.f;
#pragma unroll
    for (int k = 0; k < kMaxConvW; ++k) {
        if (k >= a.width) break;
        const float sk = k + 1 < a.width ? v[k] : Cvt<TS>::to_f(xs);
        acc = fmaf(ld_any(a.w, (long long)d * a.w_ds + (long long)k * a.w_ws, a.w_type), sk, acc);
    }
#pragma unroll
    for (int k = 0; k < kMaxConvW; ++k)
        if (k + 1 < a.width) s[(size_t)k * a.s_ws] = Cvt<TS>::from_f(v[k]);
    s[(size_t)(a.width - 1) * a.s_ws] = xs;
    if (a.silu) acc = acc * mia::rcpf(1.f + mia::ex2f(-acc * kLog2e));
    reinterpret_cast<typename Cvt<TX>::raw *>(a.out)[(size_t)b * a.out_bs + d] = Cvt<TX>::from_f(acc);
}

bool good_dtype(int t) { return t == MIA_F32 || t == MIA_F16 || t == MIA_BF16; }
int esize(int t) { return t == MIA_F32 ? 4 : 2; }

}  // namespace

extern "C" {

int mia_selective_state_update(const mia_ssu_params *pp, void *cuda_stream) {
    if (!pp) return mia::fail(mia::kErrScan, MIA_EINVAL, "selective_state_update: null params");
    const mia_ssu_params &p = *pp;
    if (p.batch <= 0 || p.dim <= 0 || p.batch > 65535)
        return mia::fail(mia::kErrScan, MIA_EINVAL, "selective_state_update: batch must be in 1..65535 and dim >= 1 (got %d, %d)", p.batch, p.dim);
    if (p.dstate < 1 || p.dstate > kMaxN)
        return mia::fail(mia::kErrScan, MIA_EINVAL, "selective_state_update only supports state dimension <= 256 (got %d)", p.dstate);
    if (!good_dtype(p.state_type) || !good_dtype(p.itype) || (p.D && !good_dtype(p.D_type)) || (p.dt_bias && !good_dtype(p.dt_bias_type)))
        return mia::fail(mia::kErrScan, MIA_EINVAL, "selective_state_update: every dtype must be float32, float16 or bfloat16");
    if (!p.state || !p.x || !p.dt || !p.A || !p.B || !p.C || !p.out)
        return mia::fail(mia::kErrScan, MIA_EINVAL, "selective_state_update: null state / x / dt / A / B / C / out");
    const int es = esize(p.state_type);
    const bool vec = (p.dstate * es) % 16 == 0 && (p.state_d_stride * es) % 16 == 0 && (p.state_batch_stride * es) % 16 == 0 &&
                     ((uintptr_t)p.state & 15) == 0;
    const int units = vec ? p.dstate * es / 16 : p.dstate;
    int lpr_log2 = 0;
    while ((1 << lpr_log2) < units && lpr_log2 < 5) ++lpr_log2;
    SsuArgs a{};
    a.state = p.state; a.x = p.x; a.dt = p.dt; a.z = p.z; a.B = p.B; a.C = p.C; a.D = p.D; a.bias = p.dt_bias; a.A = p.A; a.out = p.out;
    a.s_bs = p.state_batch_stride; a.s_ds = p.state_d_stride; a.x_bs = p.x_batch_stride; a.dt_bs = p.dt_batch_stride;
    a.z_bs = p.z_batch_stride; a.B_bs = p.B_batch_stride; a.C_bs = p.C_batch_stride; a.out_bs = p.out_batch_stride;
    a.A_ds = p.A_d_stride; a.A_ns = p.A_dstate_stride;
    a.batch = p.batch; a.dim = p.dim; a.N = p.dstate; a.lpr_log2 = lpr_log2; a.softplus = p.dt_softplus != 0;
    a.D_type = p.D_type; a.bias_type = p.dt_bias_type;
    a.rows_per_cta = (kStepThreads / 32) << (5 - lpr_log2);
    const dim3 grid((p.dim + a.rows_per_cta - 1) / a.rows_per_cta, p.batch);
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(p.state_type, [&](auto *ts) {
        mia::dispatch_dtype(p.itype, [&](auto *ti) {
            using TS = typename std::remove_pointer<decltype(ts)>::type;
            using TI = typename std::remove_pointer<decltype(ti)>::type;
            if (vec) ss_step_kernel<TS, TI, true><<<grid, kStepThreads, 0, st>>>(a);
            else ss_step_kernel<TS, TI, false><<<grid, kStepThreads, 0, st>>>(a);
        });
    });
    if (int rc = mia::launched(mia::kErrScan, "selective_state_update launch")) return rc;
    mia::count_launches(1);
    return MIA_OK;
}

int mia_causal_conv1d_update(const void *x, void *conv_state, const void *weight, const void *bias, void *out, int batch, int dim,
                             int width, int silu, int x_dtype, int state_dtype, int weight_dtype, int bias_dtype,
                             long long x_batch_stride, long long state_batch_stride, long long state_d_stride, long long state_w_stride,
                             long long weight_d_stride, long long weight_w_stride, long long out_batch_stride, void *cuda_stream) {
    if (!x || !conv_state || !weight || !out) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_update: null x / conv_state / weight / out");
    if (batch <= 0 || dim <= 0 || batch > 65535)
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_update: batch must be in 1..65535 and dim >= 1 (got %d, %d)", batch, dim);
    if (width < 1 || width > kMaxConvW) return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_update only supports width between 1 and 4 (got %d)", width);
    if (!good_dtype(x_dtype) || !good_dtype(state_dtype) || !good_dtype(weight_dtype) || (bias && !good_dtype(bias_dtype)))
        return mia::fail(mia::kErrConv, MIA_EINVAL, "causal_conv1d_update: every dtype must be float32, float16 or bfloat16");
    ConvStepArgs a{};
    a.x = x; a.w = weight; a.bias = bias; a.state = conv_state; a.out = out;
    a.x_bs = x_batch_stride; a.s_bs = state_batch_stride; a.s_ds = state_d_stride; a.s_ws = state_w_stride;
    a.w_ds = weight_d_stride; a.w_ws = weight_w_stride; a.out_bs = out_batch_stride;
    a.batch = batch; a.dim = dim; a.width = width; a.silu = silu != 0; a.w_type = weight_dtype; a.bias_type = bias_dtype;
    const dim3 grid((dim + kConvStepThreads - 1) / kConvStepThreads, batch);
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    mia::dispatch_dtype(x_dtype, [&](auto *tx) {
        mia::dispatch_dtype(state_dtype, [&](auto *ts) {
            using TX = typename std::remove_pointer<decltype(tx)>::type;
            using TS = typename std::remove_pointer<decltype(ts)>::type;
            causal_conv1d_update_kernel<TX, TS><<<grid, kConvStepThreads, 0, st>>>(a);
        });
    });
    if (int rc = mia::launched(mia::kErrConv, "causal_conv1d_update launch")) return rc;
    mia::count_launches(1);
    return MIA_OK;
}

}  // extern "C"
