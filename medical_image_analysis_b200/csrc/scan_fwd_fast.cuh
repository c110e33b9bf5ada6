// Forward selective scan, fast path: d_state == 1 (R2GenCSR's vssm_base_224.yaml, the reference's own test grid),
// rows spanning the whole warp (L > 128), delta per row, no z gate.  Same staging pipeline and results as the
// generic kernel (scan_fwd.cuh); the consumer is rewritten for instruction count:
//   * softplus stays in the log2 domain: m = log2(1 + 2^x') with x' = (delta + bias) log2e, so that
//     a = exp(dl A) = 2^(m A) needs no constant and b = dl u B = m u (B ln2) folds ln2 into the hoisted B row;
//   * elementwise work is issued as packed f32x2 instructions (FFMA2 / FMUL2 / FADD2);
//   * B', C live in registers for a whole (segment, chunk); addresses are 32-bit shared-window adds.
#pragma once
#include <type_traits>

#include "scan_fwd.cuh"

namespace mia {

template <typename T, bool kSoftplus, bool kOutF32>
__global__ void __launch_bounds__(kThreadsFwd, 1) ss_fwd_fast_kernel(const __grid_constant__ ScanArgs a) {
    extern __shared__ __align__(128) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NW = a.n_consumer_warps;
    uint64_t *rfull = reinterpret_cast<uint64_t *>(smem + a.off_bars);
    uint64_t *rempty = rfull + kMaxStages;
    uint64_t *gfull = rempty + kMaxStages;
    uint64_t *gempty = gfull + kGroupStages;
    float2 *carry = reinterpret_cast<float2 *>(smem + a.off_carry);  // [RS] running (prod a, h)
    constexpr int es = (int)sizeof(T);
    constexpr int eo = kOutF32 ? 4 : es;
    using TO = typename std::conditional<kOutF32, float, T>::type;

    zero_smem(smem, a.smem_bytes);
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int s = 0; s < a.stages; ++s) { mbar_init(rfull + s, 1); mbar_init(rempty + s, NW); }
        for (int s = 0; s < kGroupStages; ++s) { mbar_init(gfull + s, 1); mbar_init(gempty + s, NW); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == NW) {
        fwd_producer<T>(a, smem, rfull, rempty, gfull, gempty, lane);
        return;
    }
    if (warp > NW) return;

    const int L = a.L, RT = a.RT;
    const int tok0 = lane * kTok;
    const uint32_t sbase = smem_u32(smem);
    const uint32_t ustepB = (uint32_t)(a.u_ds * es), dstepB = (uint32_t)(a.delta_ds * es);
    const uint32_t upitch = a.flat_u ? (uint32_t)(L * es) : (uint32_t)a.row_pitch, ustep = a.flat_u ? 0u : ustepB;
    const uint32_t dpitch = a.flat_delta ? (uint32_t)(L * es) : (uint32_t)a.row_pitch, dstep = a.flat_delta ? 0u : dstepB;
    const size_t out_step = (size_t)a.out_ds * eo;
    const size_t xstride = (size_t)a.n_chunks;
    const float2 kL2E = splat2(kLog2e);
    int kr = 0, kg = 0;
    for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
        const SegCoord sc = decode_seg(a, seg);
        const int tiles = (sc.nrows + RT - 1) / RT;
        for (int c = 0; c < a.n_chunks; ++c, ++kg) {
            const int l0 = c * kTok * 32, len = min(kTok * 32, L - l0);
            const int nval = max(0, min(kTok, len - tok0));
            const bool partial = len < kTok * 32;
            const int jl = (len - 1) / kTok, lastidx = (len - 1) % kTok;   // lane / slot of the chunk's last token
            const bool more_chunks = c + 1 < a.n_chunks;
            const int sg = kg % kGroupStages;
            mbar_wait(gfull + sg, (kg / kGroupStages) & 1);
            const char *gs = smem + a.off_groups + (size_t)sg * a.gstage_bytes;
            const uint32_t gsb = sbase + a.off_groups + sg * a.gstage_bytes;
            const uint32_t gBlo = (uint32_t)(uintptr_t)((const char *)a.B + ((size_t)sc.b * a.B_bs + (size_t)sc.g * a.B_gs + l0) * es);
            const uint32_t gClo = (uint32_t)(uintptr_t)((const char *)a.C + ((size_t)sc.b * a.C_bs + (size_t)sc.g * a.C_gs + l0) * es);
            float2 Bp[4], C2[4];
            lds8v<T>(gsb + a.goff_B + (gBlo & 15u) + tok0 * es, Bp);
            lds8v<T>(gsb + a.goff_C + (gClo & 15u) + tok0 * es, C2);
#pragma unroll
            for (int k = 0; k < 4; ++k) Bp[k] = mul2(Bp[k], splat2(kLn2));
            const float *pA = reinterpret_cast<const float *>(gs + a.goff_A);
            const float *pD = reinterpret_cast<const float *>(gs + a.goff_D);
            const float *pbias = reinterpret_cast<const float *>(gs + a.goff_bias);
            const uint32_t gu_lo = (uint32_t)(uintptr_t)((const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)sc.row_lo * a.u_ds + l0) * es);
            const uint32_t gd_lo = (uint32_t)(uintptr_t)((const char *)a.delta + ((size_t)sc.b * a.delta_bs + (size_t)sc.row_lo * a.delta_ds + l0) * es);
            char *out_seg = (char *)a.out + ((size_t)sc.b * a.out_bs + (size_t)sc.row_lo * a.out_ds + l0 + tok0) * eo;
            float2 *x_seg = reinterpret_cast<float2 *>(a.x) + ((size_t)(sc.b * a.dim + sc.row_lo) * a.n_chunks + c);
            for (int t = 0; t < tiles; ++t, ++kr) {
                const int sr = kr % a.stages;
                mbar_wait(rfull + sr, (kr / a.stages) & 1);
                const uint32_t stb = sbase + sr * a.stage_bytes;
                const int r0 = t * RT, nr = min(RT, sc.nrows - r0);
                const uint32_t u_t = stb + a.off_u + tok0 * es, ulo_t = gu_lo + r0 * ustepB;
                const uint32_t d_t = stb + a.off_delta + tok0 * es, dlo_t = gd_lo + r0 * dstepB;
                for (int r = warp; r < nr; r += NW) {
                    const int rs = r0 + r;
                    float2 d2[4], u2[4];
                    lds8v<T>(d_t + r * dpitch + ((dlo_t + r * dstep) & 15u), d2);
                    lds8v<T>(u_t + r * upitch + ((ulo_t + r * ustep) & 15u), u2);
                    const float Araw = pA[rs] * kLn2;          // the group stage holds A * log2e
                    const float Dv = pD[rs];
                    const float2 bl = splat2(pbias[rs] * kLog2e);
                    float2 y2[4], a2[4], b2[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float2 m = fma2(d2[k], kL2E, bl);       // (delta + bias) * log2e
                        if (kSoftplus) {
                            m = softplus_l2(m);   // softplus * log2e
                        }
                        y2[k] = mul2(u2[k], splat2(Dv));
                        const float2 arg = mul2(m, splat2(Araw));
                        a2[k] = make_float2(ex2f(arg.x), ex2f(arg.y));
                        b2[k] = mul2(mul2(m, u2[k]), Bp[k]);
                    }
                    float pa = 1.f, pb = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        pb = fmaf(a2[k].x, pb, b2[k].x); pa *= a2[k].x;
                        pb = fmaf(a2[k].y, pb, b2[k].y); pa *= a2[k].y;
                    }
                    float2 cin = make_float2(1.f, 0.f);
                    if (c > 0) cin = carry[rs];
                    float ea, eb;
                    seg_scan_fwd<32>(pa, pb, ea, eb, lane, 32);
                    float h = fmaf(ea, cin.y, eb);
                    float hs[kTok];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        h = fmaf(a2[k].x, h, b2[k].x); hs[2 * k] = h;
                        h = fmaf(a2[k].y, h, b2[k].y); hs[2 * k + 1] = h;
                        y2[k] = fma2(make_float2(hs[2 * k], hs[2 * k + 1]), C2[k], y2[k]);
                    }
                    // ---- state after the chunk's last token: carry + checkpoint x[b][d][chunk] = (prod a, h)
                    if (more_chunks) __syncwarp();
                    if (!partial) {
                        if (lane == 31) {
                            const float2 cout = make_float2(pa * cin.x, fmaf(pa, cin.y, pb));
                            if (more_chunks) carry[rs] = cout;
                            x_seg[(size_t)rs * xstride] = cout;
                        }
                    } else if (lane == jl) {
                        float hend = hs[0], pp = ea * cin.x;
#pragma unroll
                        for (int i = 0; i < kTok; ++i) {
                            if (i == lastidx) hend = hs[i];
                            if (i <= lastidx) pp *= (i & 1) ? a2[i >> 1].y : a2[i >> 1].x;
                        }
                        x_seg[(size_t)rs * xstride] = make_float2(pp, hend);
                    }
                    if (nval > 0) st8v<TO>(out_seg + rs * out_step, y2, nval);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(rempty + sr);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(gempty + sg);
        }
    }
}

template <typename T>
cudaError_t launch_fwd_any(const ScanArgs &a, int grid, cudaStream_t stream) {
    const bool fast = a.N == 1 && a.LPR == 32 && !a.has_z && a.delta_ratio == 1;
    if (!fast) return launch_fwd<T>(a, grid, stream);
    void (*kernel)(const ScanArgs);
    if constexpr (sizeof(T) == 4)        // fp32 inputs store fp32 outputs: kOutF32 is always set
        kernel = a.softplus ? &ss_fwd_fast_kernel<T, true, true> : &ss_fwd_fast_kernel<T, false, true>;
    else if (a.softplus) kernel = a.out_f32 ? &ss_fwd_fast_kernel<T, true, true> : &ss_fwd_fast_kernel<T, true, false>;
    else kernel = a.out_f32 ? &ss_fwd_fast_kernel<T, false, true> : &ss_fwd_fast_kernel<T, false, false>;
    return launch_smem(kernel, grid, kThreadsFwd, a.smem_bytes, stream, a);
}

}  // namespace mia
