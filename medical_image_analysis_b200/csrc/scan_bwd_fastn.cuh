// Backward selective scan, fast path for d_state > 1: rows spanning the whole warp (L > 128), delta per row, with or
// without the z gate of the mamba_ssm signature.
// Same pipeline (producer warp, group / row stages), reductions and results as the generic kernel (scan_bwd.cuh); the
// consumer is rewritten for instruction count -- the generic kernel executes about twice the
// instructions the arithmetic needs:
//   * everything that does not depend on the state index is hoisted out of the state loop and kept as float2 pairs:
//     m = softplus(delta + bias) log2e, m u ln2, D dy, the accumulators of du (in units of m) and of d(dl);
//   * a_n = 2^(m A_n) needs no constant; ln2 is folded into m u once per row and into du / dA once per row at the end;
//   * the sigmoid of the softplus derivative is rebuilt from m after the state loop (1 - 2^-m) instead of being held in
//     8 registers across it;
//   * (dA, dD, dbias) leave through the 6-shuffle warp_sum3 of the d_state = 1 path where possible.
// (Pre-converting the B / C chunk to aligned fp32 in shared memory was tried and removed: it cut ~45 instructions per
// (row, state) but cost a row stage and two consumer barriers per chunk, and the kernel got slower, not faster.)
// dB / dC are still vector reductions into the L2-resident accumulator (red.global.add.v4.f32): shared-memory fp32
// atomics are CAS loops (ATOMS.CAST.SPIN) and 2 x N x 256 register accumulators do not exist.
#pragma once
#include <type_traits>

#include "scan_bwd.cuh"

namespace mia {

template <typename T, bool kSoftplus, bool kOutF32>
__global__ void __launch_bounds__(kThreads, 1) ss_bwd_fastn_kernel(const __grid_constant__ ScanArgs a) {
    extern __shared__ __align__(128) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NW = a.n_consumer_warps;
    uint64_t *rfull = reinterpret_cast<uint64_t *>(smem + a.off_bars);
    uint64_t *rempty = rfull + kMaxStages;
    uint64_t *gfull = rempty + kMaxStages;
    uint64_t *gempty = gfull + kGroupStages;
    const int N = a.N, L = a.L, RT = a.RT, RS = a.RS;
    float *carryG = reinterpret_cast<float *>(smem + a.off_carry);  // [RS][N] suffix value entering from the next chunk
    float *carryA = carryG + RS * N;                                // [RS][N] dA accumulated over chunks
    float *carryD = carryA + RS * N;                                // [RS]
    float *carryBias = carryD + RS;                                 // [RS]
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
    const int Lp = (L + 3) & ~3;                      // row pitch of the atomic dB/dC accumulators
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
            const char *gB = (const char *)a.B + ((size_t)sc.b * a.B_bs + (size_t)sc.g * a.B_gs + l0) * es;
            const char *gC = (const char *)a.C + ((size_t)sc.b * a.C_bs + (size_t)sc.g * a.C_gs + l0) * es;
            const RowView vB = make_view(gs + a.goff_B, gB, a.B_ns, len, es, a.bc_pitch, a.flat_B);
            const RowView vC = make_view(gs + a.goff_C, gC, a.C_ns, len, es, a.bc_pitch, a.flat_C);
            const float *pA = reinterpret_cast<const float *>(gs + a.goff_A);
            const float *pD = reinterpret_cast<const float *>(gs + a.goff_D);
            const float *pbias = reinterpret_cast<const float *>(gs + a.goff_bias);
            const uint32_t gu_lo = (uint32_t)(uintptr_t)((const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)sc.row_lo * a.u_ds + l0) * es);
            const uint32_t gd_lo = (uint32_t)(uintptr_t)((const char *)a.delta + ((size_t)sc.b * a.delta_bs + (size_t)sc.row_lo * a.delta_ds + l0) * es);
            const uint32_t go_lo = (uint32_t)(uintptr_t)((const char *)a.dout + ((size_t)sc.b * a.dout_bs + (size_t)sc.row_lo * a.dout_ds + l0) * eso);
            char *du_seg = (char *)a.du + ((size_t)sc.b * a.du_bs + (size_t)sc.row_lo * a.du_ds + l0 + tok0) * es;
            char *dd_seg = (char *)a.ddelta + ((size_t)sc.b * a.dd_bs + (size_t)sc.row_lo * a.dd_ds + l0 + tok0) * es;
            char *dz_seg = a.has_z ? (char *)a.dz + ((size_t)sc.b * a.dz_bs + (size_t)sc.row_lo * a.dz_ds + l0 + tok0) * es : nullptr;
            const size_t dz_step = (size_t)a.dz_ds * es;
            float *accB = a.acc_dB + (size_t)(sc.b * a.G + sc.g) * N * Lp + l0 + tok0;
            float *accC = a.acc_dC + (size_t)(sc.b * a.G + sc.g) * N * Lp + l0 + tok0;
            for (int t = 0; t < tiles; ++t, ++kr) {
                const int sr = kr % a.stages;
                mbar_wait(rfull + sr, (kr / a.stages) & 1);
                const uint32_t stb = sbase + sr * a.stage_bytes;
                const int r0 = t * RT, nr = min(RT, sc.nrows - r0);
                const uint32_t u_t = stb + a.off_u + tok0 * es, ulo_t = gu_lo + r0 * ustepB;
                const uint32_t d_t = stb + a.off_delta + tok0 * es, dlo_t = gd_lo + r0 * dstepB;
                const uint32_t o_t = stb + a.off_dout + tok0 * eso, olo_t = go_lo + r0 * ostepB;
                const float *h0s = reinterpret_cast<const float *>(smem + (size_t)sr * a.stage_bytes + a.off_h0);
                RowView vz{}, vo{};
                if (a.has_z) {
                    const char *st = smem + (size_t)sr * a.stage_bytes;
                    const size_t d0 = (size_t)sc.row_lo + r0;
                    vz = make_view(st + a.off_z, (const char *)a.z + ((size_t)sc.b * a.z_bs + d0 * a.z_ds + l0) * es, a.z_ds, len, es,
                                   a.row_pitch, a.flat_z);
                    vo = make_view(st + a.off_osaved, (const char *)a.out_saved + ((size_t)sc.b * a.osaved_bs + d0 * a.osaved_ds + l0) * eso,
                                   a.osaved_ds, len, eso, a.rowo_pitch, a.flat_osaved);
                }
                for (int r = warp; r < nr; r += NW) {
                    const int rs = r0 + r;
                    float2 m2[4], u2[4], dy2[4];
                    lds8v<T>(d_t + r * dpitch + ((dlo_t + r * dstep) & 15u), m2);
                    lds8v<T>(u_t + r * upitch + ((ulo_t + r * ustep) & 15u), u2);
                    lds8v<TO>(o_t + r * opitch + ((olo_t + r * ostep) & 15u), dy2);
                    if (a.has_z) {
                        // out_z = y silu(z):  dy = dout silu(z);  dz = dout y sigmoid(z) (1 + z (1 - sigmoid(z)))   (y = saved `out`)
                        float2 z2[4], o2[4], dz2[4];
                        lds8v<T>(vz.row(r) + tok0 * es, z2);
                        lds8v<TO>(vo.row(r) + tok0 * eso, o2);
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const float2 sz = make_float2(rcpf(1.f + ex2f(-z2[k].x * kLog2e)), rcpf(1.f + ex2f(-z2[k].y * kLog2e)));
                            const float2 dsz = mul2(dy2[k], sz);
                            dz2[k] = mul2(mul2(dsz, o2[k]), make_float2(fmaf(z2[k].x, 1.f - sz.x, 1.f), fmaf(z2[k].y, 1.f - sz.y, 1.f)));
                            dy2[k] = mul2(dsz, z2[k]);
                        }
                        if (nval > 0) st8v<T>(dz_seg + (size_t)rs * dz_step, dz2, nval);
                    }
                    // tokens past the end of the sequence come FIRST in the suffix scan: their dy must be zero
                    if (nval < kTok) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            dy2[k].x = 2 * k < nval ? dy2[k].x : 0.f;
                            dy2[k].y = 2 * k + 1 < nval ? dy2[k].y : 0.f;
                        }
                    }
                    const float Dv = pD[rs];
                    const float2 bl = splat2(pbias[rs] * kLog2e);
                    float2 mul2v[4], dum2[4], ddl2[4];       // m u ln2 (= dl u); du in units of 1/ln2; d(dl)
                    float dDv = 0.f, msum = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float2 m = fma2(m2[k], kL2E, bl);       // (delta + bias) * log2e
                        if (kSoftplus) {
                            m = softplus_l2(m);      // softplus * log2e
                        }
                        m2[k] = m;
                        msum += m.x + m.y;
                        mul2v[k] = mul2(mul2(m, u2[k]), kLN2);
                        dum2[k] = make_float2(0.f, 0.f);
                        ddl2[k] = make_float2(0.f, 0.f);
                        dDv = fmaf(dy2[k].x, u2[k].x, dDv);
                        dDv = fmaf(dy2[k].y, u2[k].y, dDv);
                    }
                    const float *pAr = pA + rs * N;
                    const float *h0r = h0s + r * N;
                    float *cGr = carryG + rs * N, *cAr = carryA + rs * N;
                    float *gdA = a.part_dA + (size_t)(sc.b * a.dim + sc.row_lo + rs) * N;
                    float *pB = accB, *pC = accC;            // accumulator rows of state n (advance by Lp per state)
#pragma unroll 1
                    for (int n = 0; n < N; ++n) {
                        const float Araw = pAr[n] * kLn2;       // the group stage holds A * log2e
                        float2 B2[4], C2[4], a2[4], ah2[4];
                        lds8v<T>(vB.row(n) + tok0 * es, B2);
                        lds8v<T>(vC.row(n) + tok0 * es, C2);
                        // ---- forward recompute: lane aggregate, warp scan, per-token states
                        float pa = ex2f(msum * Araw), pb = 0.f;  // product of the lane's 8 a: one MUFU instead of 8 FMUL
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const float2 arg = mul2(m2[k], splat2(Araw));
                            a2[k] = make_float2(ex2f(arg.x), ex2f(arg.y));
                            ah2[k] = mul2(mul2v[k], B2[k]);     // b_t for now
                            pb = fmaf(a2[k].x, pb, ah2[k].x);
                            pb = fmaf(a2[k].y, pb, ah2[k].y);
                        }
                        float ra = pa, rb = 0.f;                 // the suffix scan multiplies the same 8 factors
                        const float h0 = first_chunk ? 0.f : h0r[n];
                        float ea, eb;
                        seg_scan_fwd<32>(pa, pb, ea, eb, lane, 32);
                        float hm = fmaf(ea, h0, eb);
                        float2 dCv[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float2 hh;
                            float tt = a2[k].x * hm; hm = tt + ah2[k].x; ah2[k].x = tt; hh.x = hm;   // a_t h_{t-1}, then h_t
                            tt = a2[k].y * hm; hm = tt + ah2[k].y; ah2[k].y = tt; hh.y = hm;
                            dCv[k] = mul2(dy2[k], hh);
                        }
                        if (nval > 0) {
                            red_add_v4(pC, dCv[0].x, dCv[0].y, dCv[1].x, dCv[1].y);
                            if (nval > 4) red_add_v4(pC + 4, dCv[2].x, dCv[2].y, dCv[3].x, dCv[3].y);
                        }
                        // ---- suffix scan of G_t = a_t (dy_t C_t + G_{t+1})
#pragma unroll
                        for (int k = 3; k >= 0; --k) {
                            C2[k] = mul2(dy2[k], C2[k]);        // dy C
                            rb = a2[k].y * (C2[k].y + rb);
                            rb = a2[k].x * (C2[k].x + rb);
                        }
                        const float gin = last_chunk ? 0.f : cGr[n];
                        seg_scan_rev<32>(ra, rb, ea, eb, lane, 32);
                        float Gn = fmaf(ea, gin, eb);           // G entering from the first token after this lane
                        float2 dAm2 = make_float2(0.f, 0.f);
#pragma unroll
                        for (int k = 3; k >= 0; --k) {
                            float2 g;
                            g.y = C2[k].y + Gn; Gn = a2[k].y * g.y;
                            g.x = C2[k].x + Gn; Gn = a2[k].x * g.x;
                            const float2 gB = mul2(g, B2[k]);
                            dum2[k] = fma2(gB, m2[k], dum2[k]);                 // du / ln2
                            const float2 gah = mul2(g, ah2[k]);
                            ddl2[k] = fma2(gB, u2[k], ddl2[k]);
                            ddl2[k] = fma2(gah, splat2(Araw), ddl2[k]);
                            dAm2 = fma2(gah, m2[k], dAm2);                      // dA / ln2
                            B2[k] = mul2(g, mul2v[k]);                          // dB
                        }
                        if (nval > 0) {
                            red_add_v4(pB, B2[0].x, B2[0].y, B2[1].x, B2[1].y);
                            if (nval > 4) red_add_v4(pB + 4, B2[2].x, B2[2].y, B2[3].x, B2[3].y);
                        }
                        pB += Lp; pC += Lp;
                        if (!first_chunk) {
                            __syncwarp();
                            if (lane == 0) cGr[n] = Gn;         // G at this chunk's first token, for chunk c-1
                        }
                        // ---- dA: reduce over the row's lanes, accumulate over chunks
                        const float dAv = seg_sum<32>((dAm2.x + dAm2.y) * kLn2, 32);
                        if (lane == 0) {
                            const float tot = last_chunk ? dAv : dAv + cAr[n];
                            if (first_chunk) gdA[n] = tot; else cAr[n] = tot;
                        }
                    }
                    // ---- per-row epilogue
                    float dbv = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        dum2[k] = fma2(dy2[k], splat2(Dv), mul2(dum2[k], kLN2));
                        if (kSoftplus) {
                            ddl2[k] = mul2(ddl2[k], sigmoid_of_softplus_l2(m2[k], 1.f));     // sigmoid(x) = 1 - 2^(-m)
                        }
                        dbv += ddl2[k].x + ddl2[k].y;
                    }
                    if (nval > 0) {
                        st8v<T>(du_seg + rs * du_step, dum2, nval);
                        st8v<T>(dd_seg + rs * dd_step, ddl2, nval);
                    }
                    // one 6-shuffle reduction for (-, dD, dbias): totals land in lanes 16 / 8
                    const float tot = warp_sum3(0.f, dDv, dbv, lane);
                    if (lane == 16 || lane == 8) {
                        float *cr = lane == 16 ? carryD : carryBias;
                        float *gp = lane == 16 ? a.part_dD : a.part_dbias;
                        const float t2 = last_chunk ? tot : tot + cr[rs];
                        if (first_chunk) gp[(size_t)sc.b * a.dim + sc.row_lo + rs] = t2; else cr[rs] = t2;
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(rempty + sr);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(gempty + sg);
        }
    }
}

}  // namespace mia
