// Forward selective scan for sm_90a.
//
// Replaces selective_scan_fwd_kernel of the reference
// (R2GenCSR/VMamba/kernels/selective_scan/csrc/selective_scan/cusoflex/selective_scan_fwd_kernel_oflex.cuh:68-181):
//   delta' = softplus(delta + bias);  h_n[l] = exp(delta' A_n) h_n[l-1] + delta' u B_n[l];
//   y[l]   = sum_n C_n[l] h_n[l] + D u[l];   (optional) out_z = y * silu(z)
// and writes the per-chunk (prod a, h) checkpoints x that the backward restarts from.
//
// Not a port: instead of one CTA per (batch, row) with CUB block loads/scans and 2 __syncthreads per state,
// a persistent CTA walks (batch, group, row-range) segments; a producer warp TMA-stages the B/C chunk and the
// per-row parameters once per (segment, chunk) and streams the rows through an mbarrier ring; each consumer warp
// scans its rows with register-serial 8-token pieces + one warp-shuffle scan per state.  No block-wide
// synchronisation in the steady state.
#pragma once
#include "scan_common.cuh"

namespace mia {

// ===================== producer warp: TMA-stage group + row stages =====================
template <typename T>
__device__ __forceinline__ void fwd_producer(const ScanArgs &a, char *smem, uint64_t *rfull, uint64_t *rempty, uint64_t *gfull,
                                             uint64_t *gempty, int lane) {
    constexpr int es = (int)sizeof(T);
    const int N = a.N, L = a.L, CH = a.CH, RT = a.RT;
    {
        const float *Ap = reinterpret_cast<const float *>(a.A);
        const float *Dp = reinterpret_cast<const float *>(a.D);
        const float *biasp = reinterpret_cast<const float *>(a.delta_bias);
        int kr = 0, kg = 0;
        for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
            const SegCoord sc = decode_seg(a, seg);
            const int tiles = (sc.nrows + RT - 1) / RT;
            for (int c = 0; c < a.n_chunks; ++c) {
                const int l0 = c * CH, len = min(CH, L - l0);
                {
                    const int sg = kg % kGroupStages, ug = kg / kGroupStages;
                    if (ug > 0) mbar_wait(gempty + sg, (ug - 1) & 1);
                    char *gs = smem + a.off_groups + (size_t)sg * a.gstage_bytes;
                    uint32_t tx = 0;
                    const char *gB = (const char *)a.B + ((size_t)sc.b * a.B_bs + (size_t)sc.g * a.B_gs + l0) * es;
                    tx += stage_rows(gs + a.goff_B, gB, a.B_ns, N, len, es, a.bc_pitch, a.flat_B, gfull + sg, lane);
                    const char *gC = (const char *)a.C + ((size_t)sc.b * a.C_bs + (size_t)sc.g * a.C_gs + l0) * es;
                    tx += stage_rows(gs + a.goff_C, gC, a.C_ns, N, len, es, a.bc_pitch, a.flat_C, gfull + sg, lane);
                    float *pA = reinterpret_cast<float *>(gs + a.goff_A);
                    float *pD = reinterpret_cast<float *>(gs + a.goff_D);
                    float *pb = reinterpret_cast<float *>(gs + a.goff_bias);
                    for (int rs = lane; rs < sc.nrows; rs += 32) {
                        const int d = sc.row_lo + rs;
                        for (int n = 0; n < N; ++n) pA[rs * N + n] = __ldg(Ap + (size_t)d * a.A_ds + (size_t)n * a.A_ns) * kLog2e;
                        pD[rs] = Dp ? __ldg(Dp + d) : 0.f;
                        pb[rs] = biasp ? __ldg(biasp + d / a.delta_ratio) : 0.f;
                    }
                    tx = __reduce_add_sync(0xffffffffu, tx);
                    if (lane == 0) mbar_arrive_expect_tx(gfull + sg, tx);
                    ++kg;
                }
                for (int t = 0; t < tiles; ++t, ++kr) {
                    const int sr = kr % a.stages, ur = kr / a.stages;
                    if (ur > 0) mbar_wait(rempty + sr, (ur - 1) & 1);
                    char *st = smem + (size_t)sr * a.stage_bytes;
                    const int r0 = t * RT, nr = min(RT, sc.nrows - r0), d0 = sc.row_lo + r0;
                    uint32_t tx = 0;
                    const char *gu = (const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)d0 * a.u_ds + l0) * es;
                    tx += stage_rows(st + a.off_u, gu, a.u_ds, nr, len, es, a.row_pitch, a.flat_u, rfull + sr, lane);
                    const int dg0 = d0 / a.delta_ratio, ndr = (d0 + nr - 1) / a.delta_ratio - dg0 + 1;
                    const char *gd = (const char *)a.delta + ((size_t)sc.b * a.delta_bs + (size_t)dg0 * a.delta_ds + l0) * es;
                    tx += stage_rows(st + a.off_delta, gd, a.delta_ds, ndr, len, es, a.row_pitch, a.flat_delta, rfull + sr, lane);
                    if (a.has_z) {
                        const char *gz = (const char *)a.z + ((size_t)sc.b * a.z_bs + (size_t)d0 * a.z_ds + l0) * es;
                        tx += stage_rows(st + a.off_z, gz, a.z_ds, nr, len, es, a.row_pitch, a.flat_z, rfull + sr, lane);
                    }
                    tx = __reduce_add_sync(0xffffffffu, tx);
                    if (lane == 0) mbar_arrive_expect_tx(rfull + sr, tx);
                }
            }
        }
    }
}

template <typename T, bool kSoftplus, bool kN1, int kLPR>
__global__ void __launch_bounds__(kThreadsFwd, 1) ss_fwd_kernel(const __grid_constant__ ScanArgs a) {
    extern __shared__ __align__(128) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NW = a.n_consumer_warps;
    uint64_t *rfull = reinterpret_cast<uint64_t *>(smem + a.off_bars);
    uint64_t *rempty = rfull + kMaxStages;
    uint64_t *gfull = rempty + kMaxStages;
    uint64_t *gempty = gfull + kGroupStages;
    float2 *carry = reinterpret_cast<float2 *>(smem + a.off_carry);  // [RS][N] running (prod a, h)
    constexpr int es = (int)sizeof(T);

    zero_smem(smem, a.smem_bytes);
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int s = 0; s < a.stages; ++s) { mbar_init(rfull + s, 1); mbar_init(rempty + s, NW); }
        for (int s = 0; s < kGroupStages; ++s) { mbar_init(gfull + s, 1); mbar_init(gempty + s, NW); }
        fence_mbar_init();
    }
    __syncthreads();

    const int N = kN1 ? 1 : a.N, L = a.L, CH = a.CH, RT = a.RT;

    if (warp == NW) {
        fwd_producer<T>(a, smem, rfull, rempty, gfull, gempty, lane);
    } else if (warp < NW) {
        // ===================== consumer warps: scan rows =====================
        const int LPR = kLPR == 32 ? 32 : a.LPR, RPP = kLPR == 32 ? 1 : 32 / LPR;
        const int sub = kLPR == 32 ? 0 : lane / LPR, j = kLPR == 32 ? lane : lane % LPR;
        const int tok0 = j * kTok;
        const int eo = a.out_f32 ? 4 : es;
        int kr = 0, kg = 0;
        for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
            const SegCoord sc = decode_seg(a, seg);
            const int tiles = (sc.nrows + RT - 1) / RT;
            for (int c = 0; c < a.n_chunks; ++c, ++kg) {
                const int l0 = c * CH, len = min(CH, L - l0);
                const int nval = max(0, min(kTok, len - tok0));
                // lane / slot of the chunk's last token: that lane owns the end state (carry + checkpoint); tokens behind
                // it hold arbitrary finite data and only feed later tokens, so only that lane needs masking
                const int jl = (len - 1) / kTok, lastidx = (len - 1) % kTok;
                const bool more_chunks = c + 1 < a.n_chunks;
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
                float B8[kTok], C8[kTok];
                if (kN1) {
                    lds8<T>(vB.row(0) + tok0 * es, B8);
                    lds8<T>(vC.row(0) + tok0 * es, C8);
                }
                // per-(segment, chunk) global bases; tiles and rows only add strides
                const char *gu_seg = (const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)sc.row_lo * a.u_ds + l0) * es;
                const char *gd_seg = (const char *)a.delta + ((size_t)sc.b * a.delta_bs + l0) * es;
                char *out_seg = (char *)a.out + ((size_t)sc.b * a.out_bs + (size_t)sc.row_lo * a.out_ds + l0 + tok0) * eo;
                const size_t out_step = (size_t)a.out_ds * eo;
                const size_t xstride = (size_t)a.n_chunks * N;
                float2 *x_seg = reinterpret_cast<float2 *>(a.x) + ((size_t)(sc.b * a.dim + sc.row_lo) * a.n_chunks + c) * N;
                for (int t = 0; t < tiles; ++t, ++kr) {
                    const int sr = kr % a.stages;
                    mbar_wait(rfull + sr, (kr / a.stages) & 1);
                    const char *st = smem + (size_t)sr * a.stage_bytes;
                    const int r0 = t * RT, nr = min(RT, sc.nrows - r0), d0 = sc.row_lo + r0;
                    const int dg0 = d0 / a.delta_ratio;
                    const char *gu = gu_seg + (size_t)r0 * a.u_ds * es;
                    const char *gd = gd_seg + (size_t)dg0 * a.delta_ds * es;
                    const RowView vu = make_view(st + a.off_u, gu, a.u_ds, len, es, a.row_pitch, a.flat_u);
                    const RowView vd = make_view(st + a.off_delta, gd, a.delta_ds, len, es, a.row_pitch, a.flat_delta);
                    char *out_tile = out_seg + r0 * out_step;
                    float2 *xrow = x_seg + r0 * xstride;

                    for (int rb = warp * RPP; rb < nr; rb += NW * RPP) {
                        const bool active = rb + sub < nr;
                        const int r = active ? rb + sub : nr - 1;  // idle sub-rows shadow a valid row, never store
                        const int rs = r0 + r, d = d0 + r;
                        const int rdelta = a.delta_ratio == 1 ? r : d / a.delta_ratio - dg0;
                        float u8[kTok], dl[kTok], y[kTok];
                        lds8<T>(vu.row(r) + tok0 * es, u8);
                        lds8<T>(vd.row(rdelta) + tok0 * es, dl);
                        const float bias = pbias[rs], Dv = pD[rs];
#pragma unroll
                        for (int i = 0; i < kTok; ++i) {
                            float sgm;
                            const float xv = dl[i] + bias;
                            dl[i] = kSoftplus ? softplus_f<false>(xv, sgm) : xv;
                            y[i] = Dv * u8[i];
                            u8[i] *= dl[i];  // from here on u8 holds delta' * u
                        }
                        if (j == jl && lastidx < kTok - 1) {   // make the padding tokens of the last lane identities (a = 1, b = 0)
#pragma unroll
                            for (int i = 1; i < kTok; ++i) {
                                dl[i] = i <= lastidx ? dl[i] : 0.f;
                                u8[i] = i <= lastidx ? u8[i] : 0.f;
                            }
                        }
                        for (int n = 0; n < N; ++n) {
                            const float A2 = pA[rs * N + n];
                            if (!kN1) {
                                lds8<T>(vB.row(n) + tok0 * es, B8);
                                lds8<T>(vC.row(n) + tok0 * es, C8);
                            }
                            float2 cin = make_float2(1.f, 0.f);
                            if (c > 0) cin = carry[rs * N + n];
                            float av[kTok], bv[kTok];
                            float pa = 1.f, pb = 0.f;
#pragma unroll
                            for (int i = 0; i < kTok; ++i) {
                                av[i] = ex2f(dl[i] * A2);
                                bv[i] = u8[i] * B8[i];
                                pb = fmaf(av[i], pb, bv[i]);
                                pa *= av[i];
                            }
                            float ea, eb;
                            seg_scan_fwd<kLPR>(pa, pb, ea, eb, j, LPR);
                            float h = fmaf(ea, cin.y, eb);
#pragma unroll
                            for (int i = 0; i < kTok; ++i) {
                                h = fmaf(av[i], h, bv[i]);
                                y[i] = fmaf(h, C8[i], y[i]);
                            }
                            // ---- state after the chunk's last token: carry to the next chunk + checkpoint
                            if (more_chunks) __syncwarp();
                            if (j == jl && active) {
                                const float2 cout = make_float2(pa * cin.x, fmaf(pa, cin.y, pb));
                                if (more_chunks) carry[rs * N + n] = cout;
                                // reference layout: x[b][d][chunk][2n] = prod a, [2n+1] = h  (fwd kernel :164-167)
                                xrow[(size_t)r * xstride + n] = cout;
                            }
                        }
                        if (active && nval > 0) {
                            char *go = out_tile + r * out_step;
                            if (a.out_f32) st8<float>(go, y, nval); else st8<T>(go, y, nval);
                            if (a.has_z) {
                                const char *gz = (const char *)a.z + ((size_t)sc.b * a.z_bs + (size_t)d0 * a.z_ds + l0) * es;
                                const RowView vz = make_view(st + a.off_z, gz, a.z_ds, len, es, a.row_pitch, a.flat_z);
                                float z8[kTok];
                                lds8<T>(vz.row(r) + tok0 * es, z8);
#pragma unroll
                                for (int i = 0; i < kTok; ++i) {
                                    const float sg = rcpf(1.f + ex2f(-z8[i] * kLog2e));
                                    y[i] = y[i] * z8[i] * sg;
                                }
                                char *gzo = (char *)a.out_z + ((size_t)sc.b * a.outz_bs + (size_t)d * a.outz_ds + l0 + tok0) * eo;
                                if (a.out_f32) st8<float>(gzo, y, nval); else st8<T>(gzo, y, nval);
                            }
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
}

template <typename T>
cudaError_t launch_fwd(const ScanArgs &a, int grid, cudaStream_t stream) {
    void (*kernel)(const ScanArgs);
    const bool n1 = a.N == 1, w32 = a.LPR == 32;
#define MIA_PICK(SP, N1) (w32 ? &ss_fwd_kernel<T, SP, N1, 32> : &ss_fwd_kernel<T, SP, N1, 0>)
    if (a.softplus) kernel = n1 ? MIA_PICK(true, true) : MIA_PICK(true, false);
    else kernel = n1 ? MIA_PICK(false, true) : MIA_PICK(false, false);
#undef MIA_PICK
    return launch_smem(kernel, grid, kThreadsFwd, a.smem_bytes, stream, a);
}

}  // namespace mia
