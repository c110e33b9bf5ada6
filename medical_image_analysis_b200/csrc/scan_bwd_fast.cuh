// Backward selective scan, fast path: d_state == 1, rows spanning the whole warp (L > 128), delta per row, no z gate.
// Same pipeline, reductions and results as the generic kernel (scan_bwd.cuh); the consumer is rewritten for
// instruction count (log2-domain softplus, packed f32x2 arithmetic, hoisted B ln2 / C rows, 32-bit addressing).
//
// Log2-domain bookkeeping (m = softplus(delta + bias) * log2e, so dl = m ln2):
//   a = 2^(m A)            b = m u B'            with B' = B ln2
//   du  = D dy + g B' m    ddm = g B' u + g a h_prev (A ln2) = ln2 * d/d(dl)     ddelta = ddm * (sigmoid * log2e)
//   dA  = ln2 * sum g a h_prev m                 dB = ln2 * sum_rows (g m) u     dC = sum_rows dy h
#pragma once
#include <type_traits>

#include "scan_bwd.cuh"
#include "scan_bwd_fastn.cuh"

namespace mia {

template <typename T, bool kSoftplus, bool kOutF32>
__global__ void __launch_bounds__(kThreads, 1) ss_bwd_fast_kernel(const __grid_constant__ ScanArgs a) {
    extern __shared__ __align__(128) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NW = a.n_consumer_warps;
    uint64_t *rfull = reinterpret_cast<uint64_t *>(smem + a.off_bars);
    uint64_t *rempty = rfull + kMaxStages;
    uint64_t *gfull = rempty + kMaxStages;
    uint64_t *gempty = gfull + kGroupStages;
    const int L = a.L, RT = a.RT, RS = a.RS;
    float *carryG = reinterpret_cast<float *>(smem + a.off_carry);  // [RS] suffix value entering from the next chunk
    float *carryA = carryG + RS;                                    // [RS] dA accumulated over chunks
    float *carryD = carryA + RS;                                    // [RS]
    float *carryBias = carryD + RS;                                 // [RS]
    float *red = reinterpret_cast<float *>(smem + a.off_red);       // [NW][256]
    constexpr int es = (int)sizeof(T);
    constexpr int eso = kOutF32 ? 4 : es;
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
        bwd_producer<T>(a, smem, rfull, rempty, gfull, gempty, lane);
        return;
    }
    if (warp > NW) return;

    const int tok0 = lane * kTok;
    const uint32_t sbase = smem_u32(smem);
    const uint32_t ustepB = (uint32_t)(a.u_ds * es), dstepB = (uint32_t)(a.delta_ds * es), ostepB = (uint32_t)(a.dout_ds * eso);
    const uint32_t upitch = a.flat_u ? (uint32_t)(L * es) : (uint32_t)a.row_pitch, ustep = a.flat_u ? 0u : ustepB;
    const uint32_t dpitch = a.flat_delta ? (uint32_t)(L * es) : (uint32_t)a.row_pitch, dstep = a.flat_delta ? 0u : dstepB;
    const uint32_t opitch = a.flat_dout ? (uint32_t)(L * eso) : (uint32_t)a.rowo_pitch, ostep = a.flat_dout ? 0u : ostepB;
    const size_t du_step = (size_t)a.du_ds * es, dd_step = (size_t)a.dd_ds * es;
    const float2 kL2E = splat2(kLog2e), kLN2 = splat2(kLn2);
    int kr = 0, kg = 0;
    for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
        const SegCoord sc = decode_seg(a, seg);
        const int tiles = (sc.nrows + RT - 1) / RT;
        for (int c = a.n_chunks - 1; c >= 0; --c, ++kg) {
            const int l0 = c * kTok * 32, len = min(kTok * 32, L - l0);
            const int nval = max(0, min(kTok, len - tok0));
            const bool last_chunk = c == a.n_chunks - 1, first_chunk = c == 0;
            const int sg = kg % kGroupStages;
            mbar_wait(gfull + sg, (kg / kGroupStages) & 1);
            const char *gs = smem + a.off_groups + (size_t)sg * a.gstage_bytes;
            const uint32_t gsb = sbase + a.off_groups + sg * a.gstage_bytes;
            const uint32_t gBlo = (uint32_t)(uintptr_t)((const char *)a.B + ((size_t)sc.b * a.B_bs + (size_t)sc.g * a.B_gs + l0) * es);
            const uint32_t gClo = (uint32_t)(uintptr_t)((const char *)a.C + ((size_t)sc.b * a.C_bs + (size_t)sc.g * a.C_gs + l0) * es);
            float2 Bp[4], C2[4], dBacc[4], dCacc[4];
            lds8v<T>(gsb + a.goff_B + (gBlo & 15u) + tok0 * es, Bp);
            lds8v<T>(gsb + a.goff_C + (gClo & 15u) + tok0 * es, C2);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                Bp[k] = mul2(Bp[k], kLN2);
                dBacc[k] = dCacc[k] = make_float2(0.f, 0.f);
            }
            const float *pA = reinterpret_cast<const float *>(gs + a.goff_A);
            const float *pD = reinterpret_cast<const float *>(gs + a.goff_D);
            const float *pbias = reinterpret_cast<const float *>(gs + a.goff_bias);
            const uint32_t gu_lo = (uint32_t)(uintptr_t)((const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)sc.row_lo * a.u_ds + l0) * es);
            const uint32_t gd_lo = (uint32_t)(uintptr_t)((const char *)a.delta + ((size_t)sc.b * a.delta_bs + (size_t)sc.row_lo * a.delta_ds + l0) * es);
            const uint32_t go_lo = (uint32_t)(uintptr_t)((const char *)a.dout + ((size_t)sc.b * a.dout_bs + (size_t)sc.row_lo * a.dout_ds + l0) * eso);
            char *du_seg = (char *)a.du + ((size_t)sc.b * a.du_bs + (size_t)sc.row_lo * a.du_ds + l0 + tok0) * es;
            char *dd_seg = (char *)a.ddelta + ((size_t)sc.b * a.dd_bs + (size_t)sc.row_lo * a.dd_ds + l0 + tok0) * es;
            for (int t = 0; t < tiles; ++t, ++kr) {
                const int sr = kr % a.stages;
                mbar_wait(rfull + sr, (kr / a.stages) & 1);
                const uint32_t stb = sbase + sr * a.stage_bytes;
                const int r0 = t * RT, nr = min(RT, sc.nrows - r0);
                const uint32_t u_t = stb + a.off_u + tok0 * es, ulo_t = gu_lo + r0 * ustepB;
                const uint32_t d_t = stb + a.off_delta + tok0 * es, dlo_t = gd_lo + r0 * dstepB;
                const uint32_t o_t = stb + a.off_dout + tok0 * eso, olo_t = go_lo + r0 * ostepB;
                const float *h0s = reinterpret_cast<const float *>(smem + (size_t)sr * a.stage_bytes + a.off_h0);
                for (int r = warp; r < nr; r += NW) {
                    const int rs = r0 + r;
                    float2 m2[4], u2[4], dy2[4], sg2[4];
                    lds8v<T>(d_t + r * dpitch + ((dlo_t + r * dstep) & 15u), m2);
                    lds8v<T>(u_t + r * upitch + ((ulo_t + r * ustep) & 15u), u2);
                    lds8v<TO>(o_t + r * opitch + ((olo_t + r * ostep) & 15u), dy2);
                    // tokens past the end of the sequence come FIRST in the suffix scan: their dy must be zero
                    if (nval < kTok) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            dy2[k].x = 2 * k < nval ? dy2[k].x : 0.f;
                            dy2[k].y = 2 * k + 1 < nval ? dy2[k].y : 0.f;
                        }
                    }
                    const float A2 = pA[rs];                    // A * log2e
                    const float Araw = A2 * kLn2, Aln2 = Araw * kLn2;
                    const float Dv = pD[rs];
                    const float2 bl = splat2(pbias[rs] * kLog2e);
                    float2 a2[4], ah2[4], du2[4], dd2[4];
                    float dDv = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float2 m = fma2(m2[k], kL2E, bl);       // (delta + bias) * log2e
                        if (kSoftplus) {
                            float2 e;
                            m = softplus_l2(m, e);                                              // softplus * log2e
                            const float2 sl = fma2(e, kLN2, kLN2);                              // (1 + e) ln2
                            sg2[k] = mul2(e, make_float2(rcpf(sl.x), rcpf(sl.y)));              // sigmoid * log2e
                        } else {
                            sg2[k] = kL2E;
                        }
                        m2[k] = m;
                        du2[k] = mul2(dy2[k], splat2(Dv));
                        dDv = fmaf(dy2[k].x, u2[k].x, dDv);
                        dDv = fmaf(dy2[k].y, u2[k].y, dDv);
                        const float2 arg = mul2(m, splat2(Araw));
                        a2[k] = make_float2(ex2f(arg.x), ex2f(arg.y));
                        ah2[k] = mul2(mul2(m, u2[k]), Bp[k]);   // b_t for now
                    }
                    // ---- forward recompute
                    float pa = 1.f, pb = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        pb = fmaf(a2[k].x, pb, ah2[k].x); pa *= a2[k].x;
                        pb = fmaf(a2[k].y, pb, ah2[k].y); pa *= a2[k].y;
                    }
                    const float h0 = first_chunk ? 0.f : h0s[r];
                    float ea, eb;
                    seg_scan_fwd<32>(pa, pb, ea, eb, lane, 32);
                    float hm = fmaf(ea, h0, eb);
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float2 hh;
                        float tt = a2[k].x * hm; hm = tt + ah2[k].x; ah2[k].x = tt; hh.x = hm;   // a_t h_{t-1}, then h_t
                        tt = a2[k].y * hm; hm = tt + ah2[k].y; ah2[k].y = tt; hh.y = hm;
                        dCacc[k] = fma2(dy2[k], hh, dCacc[k]);
                    }
                    // ---- suffix scan of G_t = a_t (dy_t C_t + G_{t+1})
                    float ra = 1.f, rb = 0.f;
                    float2 dyC[4];
#pragma unroll
                    for (int k = 3; k >= 0; --k) {
                        dyC[k] = mul2(dy2[k], C2[k]);
                        rb = a2[k].y * (dyC[k].y + rb); ra *= a2[k].y;
                        rb = a2[k].x * (dyC[k].x + rb); ra *= a2[k].x;
                    }
                    const float gin = last_chunk ? 0.f : carryG[rs];
                    seg_scan_rev<32>(ra, rb, ea, eb, lane, 32);
                    float Gn = fmaf(ea, gin, eb);               // G entering from the first token after this lane
                    float dAm = 0.f;
#pragma unroll
                    for (int k = 3; k >= 0; --k) {
                        float2 g;
                        g.y = dyC[k].y + Gn; Gn = a2[k].y * g.y;
                        g.x = dyC[k].x + Gn; Gn = a2[k].x * g.x;
                        const float2 gB = mul2(g, Bp[k]);                   // g B ln2
                        du2[k] = fma2(gB, m2[k], du2[k]);
                        const float2 gah = mul2(g, ah2[k]);
                        float2 ddm = mul2(gB, u2[k]);
                        ddm = fma2(gah, splat2(Aln2), ddm);
                        dd2[k] = mul2(ddm, sg2[k]);                          // ddelta
                        dAm = fmaf(gah.x, m2[k].x, dAm);
                        dAm = fmaf(gah.y, m2[k].y, dAm);
                        dBacc[k] = fma2(mul2(g, m2[k]), u2[k], dBacc[k]);
                    }
                    if (!first_chunk) {
                        __syncwarp();
                        if (lane == 0) carryG[rs] = Gn;         // G at this chunk's first token, for chunk c-1
                    }
                    float dbv = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) dbv += dd2[k].x + dd2[k].y;
                    if (nval > 0) {
                        st8v<T>(du_seg + rs * du_step, du2, nval);
                        st8v<T>(dd_seg + rs * dd_step, dd2, nval);
                    }
                    // one 6-shuffle reduction for (dA, dD, dbias): totals land in lanes 0 / 16 / 8
                    const float tot = warp_sum3(dAm * kLn2, dDv, dbv, lane);
                    if (lane == 0 || lane == 16 || lane == 8) {
                        float *cr = lane == 0 ? carryA : (lane == 16 ? carryD : carryBias);
                        float *gp = lane == 0 ? a.part_dA : (lane == 16 ? a.part_dD : a.part_dbias);
                        const float t2 = last_chunk ? tot : tot + cr[rs];
                        if (first_chunk) gp[(size_t)sc.b * a.dim + sc.row_lo + rs] = t2; else cr[rs] = t2;
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(rempty + sr);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(gempty + sg);

            // ---- fold this warp's dB/dC (summed over its rows of the segment) with the other warps' and emit the segment
            // partial.  Slot p = lane*8 + i = token.  Fixed order -> bit-reproducible.
            const int tid = threadIdx.x;
#pragma unroll
            for (int which = 0; which < 2; ++which) {
                float4 *mine = reinterpret_cast<float4 *>(red + warp * 256 + lane * kTok);
                const float2 *src = which == 0 ? dBacc : dCacc;
                mine[0] = make_float4(src[0].x, src[0].y, src[1].x, src[1].y);
                mine[1] = make_float4(src[2].x, src[2].y, src[3].x, src[3].y);
                asm volatile("bar.sync 1, %0;" ::"r"(NW * 32) : "memory");
                if (tid < len) {
                    float sum = 0.f;
                    for (int w = 0; w < NW; ++w) sum += red[w * 256 + tid];
                    float *dst = (which == 0 ? a.acc_dB : a.acc_dC) + (size_t)seg * L + l0 + tid;
                    *dst = which == 0 ? sum * kLn2 : sum;
                }
                asm volatile("bar.sync 1, %0;" ::"r"(NW * 32) : "memory");
            }
        }
    }
}

template <typename T>
cudaError_t launch_bwd_any(const ScanArgs &a, int grid, cudaStream_t stream) {
    const bool fast = a.LPR == 32 && a.delta_ratio == 1 && (a.N > 1 || !a.has_z);
    if (!fast) return launch_bwd<T>(a, grid, stream);
    void (*kernel)(const ScanArgs);
    if constexpr (sizeof(T) == 4) {      // fp32 inputs read fp32 douts: kOutF32 is always set
        if (a.N == 1) kernel = a.softplus ? &ss_bwd_fast_kernel<T, true, true> : &ss_bwd_fast_kernel<T, false, true>;
        else kernel = a.softplus ? &ss_bwd_fastn_kernel<T, true, true> : &ss_bwd_fastn_kernel<T, false, true>;
    } else if (a.N == 1) {
        if (a.softplus) kernel = a.out_f32 ? &ss_bwd_fast_kernel<T, true, true> : &ss_bwd_fast_kernel<T, true, false>;
        else kernel = a.out_f32 ? &ss_bwd_fast_kernel<T, false, true> : &ss_bwd_fast_kernel<T, false, false>;
    } else {
        if (a.softplus) kernel = a.out_f32 ? &ss_bwd_fastn_kernel<T, true, true> : &ss_bwd_fastn_kernel<T, true, false>;
        else kernel = a.out_f32 ? &ss_bwd_fastn_kernel<T, false, true> : &ss_bwd_fastn_kernel<T, false, false>;
    }
    return launch_smem(kernel, grid, kThreads, a.smem_bytes, stream, a);
}

// The deterministic d_state > 1 backward: the same kernel choice as launch_bwd_any, kDet instantiations
// (a.N > 1; a.off_det / a.off_det_acc / a.det_smem_acc carved by the host for them).
template <typename T>
cudaError_t launch_bwd_det(const ScanArgs &a, int grid, cudaStream_t stream) {
    if (a.N == 1) return cudaErrorInvalidValue;
    const bool fast = a.LPR == 32 && a.delta_ratio == 1;
    if (!fast) return launch_bwd<T, true>(a, grid, stream);
    void (*kernel)(const ScanArgs);
    if constexpr (sizeof(T) == 4)        // fp32 inputs read fp32 douts: kOutF32 is always set
        kernel = a.softplus ? &ss_bwd_fastn_kernel<T, true, true, true> : &ss_bwd_fastn_kernel<T, false, true, true>;
    else if (a.softplus) kernel = a.out_f32 ? &ss_bwd_fastn_kernel<T, true, true, true> : &ss_bwd_fastn_kernel<T, true, false, true>;
    else kernel = a.out_f32 ? &ss_bwd_fastn_kernel<T, false, true, true> : &ss_bwd_fastn_kernel<T, false, false, true>;
    return launch_smem(kernel, grid, kThreads, a.smem_bytes, stream, a);
}

}  // namespace mia
