// Backward selective scan for sm_90a.
//
// Replaces selective_scan_bwd_kernel of the reference
// (R2GenCSR/VMamba/kernels/selective_scan/csrc/selective_scan/cusoflex/selective_scan_bwd_kernel_oflex.cuh:74-291).
// Gradient algebra (same quantities as lines 216-224 / 245-259 there, re-derived):
//   h_t  = a_t h_{t-1} + b_t,  a_t = exp(dl_t A),  b_t = dl_t u_t B_t,  y_t = sum_n C_t h_t + D u_t
//   G_t  = a_t (dy_t C_t + G_{t+1})              (suffix scan; G_{L} = 0)
//   g_t  = dy_t C_t + G_{t+1}                     (= dL/dh_t)
//   du_t = D dy_t + sum_n g_t B_t dl_t            ddl_t = sum_n g_t (B_t u_t + A a_t h_{t-1})
//   dA   = sum_t g_t dl_t a_t h_{t-1}             dB_t = sum_rows g_t dl_t u_t      dC_t = sum_rows dy_t h_t
//   ddelta_t = ddl_t * sigmoid(delta_t + bias) when softplus;  dD = sum dy u;  dbias = sum ddelta
// Chunks are walked last-to-first; the forward state at a chunk start comes from the checkpoints x written by
// the forward kernel (gathered into the row stage by the producer), the suffix value G crosses chunks through
// a shared-memory carry.
//
// Reductions are deterministic for d_state == 1 (the reference's shipped configuration and its own test grid):
// dB/dC are summed in registers over all the rows a warp owns inside a (segment, chunk), then across warps through
// shared memory, and leave the CTA as one partial per segment; dA/dD/dbias leave as per-(batch,row) partials.
// A finalize kernel (scan_api.cu) folds the partials in a fixed order.  For d_state > 1 dB/dC use fp32 vector
// reductions into an L2-resident accumulator (red.global.add.v4.f32), like the reference's atomics, unless the kernel is
// instantiated with kDet (mia_selective_scan_bwd_deterministic; DESIGN.md 3.3):
//
// Deterministic d_state > 1 (kDet).  dB / dC leave as one partial per segment, [seg][N][L] in acc_dB / acc_dC, which the
// non-atomic branch of the finalize folds in segment order - the layout of the d_state 1 kernels.  Inside a
// (segment, chunk) the rows are added in ascending order:
//   * a ROW GROUP is what one warp handles at once - one row (LPR = 32) or the RPP = 32 / LPR rows rb .. rb + RPP - 1
//     (L <= 128), which are first summed by a butterfly over the sub-rows (shfl_xor at LPR, 2 LPR, .., 16: every lane ends
//     with the same bits).  Group q = t ceil(RT / RPP) + rb / RPP, numbered consecutively 0 .. nq - 1 over the tiles.
//   * group 0 writes its values, groups 1 .. nq - 1 read the running sum, add theirs (sum + own) and write it back, so
//     every element is ((g_0 + g_1) + g_2) + .. in group order; the last group writes the sum into the segment's partial.
//     The running sum lives in shared memory, [2][N][CH] at off_det_acc, when 2 N CH floats fit in 32 KB (det_smem_acc),
//     otherwise in the partial itself.
//   * the order is enforced per (state, dB or dC) by a ticket in shared memory (off_det, [2][N] ints, counting groups
//     over the CTA's whole life): group q of the k-th (segment, chunk) waits until ticket == base_k + q (acquire, CTA
//     scope), adds, then sets base_k + q + 1 (release); base_{k+1} = base_k + nq_k.
// The order depends on the sizes and the plan only, never on timing.
// Progress: order the work items (k, q) lexicographically.  Every wait of item (k, q) is on an item strictly before it:
// the ticket on (k, q - 1), or (k - 1, last) when q = 0; a row stage on every warp having released tile T - stages, i.e.
// on items of earlier tiles; a group stage on chunk k - 2.  A warp meets its items in increasing order, so the least
// unfinished item never waits on anything unfinished and the chain cannot close into a cycle.  In -DMIA_DEBUG builds a wait
// gives up after about 2^26 polls and raises *det_status, which the host reports as an error.
#pragma once
#include "scan_common.cuh"

namespace mia {

__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- ordered accumulation of the deterministic backward (see the header comment)
__device__ __forceinline__ int ld_acquire_cta(const int *p) {
    int v;
    asm volatile("ld.acquire.cta.shared::cta.b32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_cta(int *p, int v) {
    asm volatile("st.release.cta.shared::cta.b32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void det_wait(const int *ticket, int want, int *status) {
#ifdef MIA_DEBUG
    for (long long it = 0; ld_acquire_cta(ticket) != want; ++it) {
        if (it > (1LL << 26)) { if (status) atomicExch(status, 1); break; }
        __nanosleep(32);
    }
#else
    (void)status;
    while (ld_acquire_cta(ticket) != want) __nanosleep(32);
#endif
}
// One row group's 8 tokens (nval of them valid) of one (state, dB or dC): wait for the group before it, add, publish.
// acc: running sum (shared or global), part: the segment's partial; both already offset to this lane's first token.
__device__ __forceinline__ void det_ordered_add(float *acc, float *part, int *ticket, int want, bool first, bool last, bool writer,
                                                const float (&v)[kTok], int nval, int lane, int *status) {
    det_wait(ticket, want, status);
    if (writer) {
        float *dst = last ? part : acc;
#pragma unroll
        for (int i = 0; i < kTok; ++i)
            if (i < nval) dst[i] = first ? v[i] : acc[i] + v[i];
    }
    __syncwarp();
    if (lane == 0) st_release_cta(ticket, want + 1);
}

__device__ __forceinline__ void consumer_bar(int nthreads) { asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory"); }

// ===================== producer warp: TMA-stage group + row stages (chunks last-to-first) =====================
template <typename T>
__device__ __forceinline__ void bwd_producer(const ScanArgs &a, char *smem, uint64_t *rfull, uint64_t *rempty, uint64_t *gfull,
                                             uint64_t *gempty, int lane) {
    constexpr int es = (int)sizeof(T);
    const int eso = a.out_f32 ? 4 : es;
    const int N = a.N, L = a.L, CH = a.CH, RT = a.RT;
    {
        const float *Ap = reinterpret_cast<const float *>(a.A);
        const float *Dp = reinterpret_cast<const float *>(a.D);
        const float *biasp = reinterpret_cast<const float *>(a.delta_bias);
        int kr = 0, kg = 0;
        for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
            const SegCoord sc = decode_seg(a, seg);
            const int tiles = (sc.nrows + RT - 1) / RT;
            for (int c = a.n_chunks - 1; c >= 0; --c) {
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
                    const char *gdo = (const char *)a.dout + ((size_t)sc.b * a.dout_bs + (size_t)d0 * a.dout_ds + l0) * eso;
                    tx += stage_rows(st + a.off_dout, gdo, a.dout_ds, nr, len, eso, a.rowo_pitch, a.flat_dout, rfull + sr, lane);
                    if (a.has_z) {
                        const char *gz = (const char *)a.z + ((size_t)sc.b * a.z_bs + (size_t)d0 * a.z_ds + l0) * es;
                        tx += stage_rows(st + a.off_z, gz, a.z_ds, nr, len, es, a.row_pitch, a.flat_z, rfull + sr, lane);
                        const char *gos = (const char *)a.out_saved + ((size_t)sc.b * a.osaved_bs + (size_t)d0 * a.osaved_ds + l0) * eso;
                        tx += stage_rows(st + a.off_osaved, gos, a.osaved_ds, nr, len, eso, a.rowo_pitch, a.flat_osaved, rfull + sr, lane);
                    }
                    if (c > 0) {  // forward state at the start of this chunk = checkpoint of chunk c-1
                        float *h0 = reinterpret_cast<float *>(st + a.off_h0);
                        for (int idx = lane; idx < nr * N; idx += 32) {
                            const int r = idx / N, n = idx - r * N;
                            h0[idx] = __ldg(a.x + (((size_t)(sc.b * a.dim + d0 + r) * a.n_chunks + (c - 1)) * N + n) * 2 + 1);
                        }
                    }
                    tx = __reduce_add_sync(0xffffffffu, tx);
                    if (lane == 0) mbar_arrive_expect_tx(rfull + sr, tx);
                }
            }
        }
    }
}

template <typename T, bool kSoftplus, bool kN1, int kLPR, bool kDet = false>
__global__ void __launch_bounds__(kThreads, 1) ss_bwd_kernel(const __grid_constant__ ScanArgs a) {
    extern __shared__ __align__(128) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NW = a.n_consumer_warps;
    uint64_t *rfull = reinterpret_cast<uint64_t *>(smem + a.off_bars);
    uint64_t *rempty = rfull + kMaxStages;
    uint64_t *gfull = rempty + kMaxStages;
    uint64_t *gempty = gfull + kGroupStages;
    const int N = kN1 ? 1 : a.N, L = a.L, CH = a.CH, RT = a.RT, RS = a.RS;
    float *carryG = reinterpret_cast<float *>(smem + a.off_carry);  // [RS][N] suffix value entering from the next chunk
    float *carryA = carryG + RS * N;                                // [RS][N] dA accumulated over chunks
    float *carryD = carryA + RS * N;                                // [RS]
    float *carryBias = carryD + RS;                                 // [RS]
    float *red = reinterpret_cast<float *>(smem + a.off_red);       // [NW][256]
    constexpr int es = (int)sizeof(T);
    const int eso = a.out_f32 ? 4 : es;

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
    } else if (warp < NW) {
        // ===================== consumer warps =====================
        const int LPR = kLPR == 32 ? 32 : a.LPR, RPP = kLPR == 32 ? 1 : 32 / LPR;
        const int sub = kLPR == 32 ? 0 : lane / LPR, j = kLPR == 32 ? lane : lane % LPR;
        const int tok0 = j * kTok;
        const int Lp = (L + 3) & ~3;  // row pitch of the atomic dB/dC accumulators
        int kr = 0, kg = 0;
        int *det_tick = reinterpret_cast<int *>(smem + a.off_det);            // kDet: [2][N] (dC, dB)
        float *det_sacc = reinterpret_cast<float *>(smem + a.off_det_acc);    // kDet, det_smem_acc: [2][N][CH] (dB, dC)
        const int det_gpt = (RT + RPP - 1) / RPP;                              // row groups per full tile
        int det_base = 0;
        for (int seg = blockIdx.x; seg < a.n_seg; seg += gridDim.x) {
            const SegCoord sc = decode_seg(a, seg);
            const int tiles = (sc.nrows + RT - 1) / RT;
            const int det_nq = (tiles - 1) * det_gpt + (sc.nrows - (tiles - 1) * RT + RPP - 1) / RPP;
            for (int c = a.n_chunks - 1; c >= 0; --c, ++kg) {
                const int l0 = c * CH, len = min(CH, L - l0);
                const int nval = max(0, min(kTok, len - tok0));
                const bool last_chunk = c == a.n_chunks - 1, first_chunk = c == 0;
                float *det_partB = a.acc_dB + (size_t)seg * N * L + l0 + tok0, *det_partC = a.acc_dC + (size_t)seg * N * L + l0 + tok0;
                float *det_runB = a.det_smem_acc ? det_sacc + tok0 : det_partB;
                float *det_runC = a.det_smem_acc ? det_sacc + (size_t)N * CH + tok0 : det_partC;
                const size_t det_rstep = a.det_smem_acc ? (size_t)CH : (size_t)L;
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
                float dBacc[kTok], dCacc[kTok];
                if (kN1) {
                    lds8<T>(vB.row(0) + tok0 * es, B8);
                    lds8<T>(vC.row(0) + tok0 * es, C8);
#pragma unroll
                    for (int i = 0; i < kTok; ++i) dBacc[i] = dCacc[i] = 0.f;
                }
                const char *gu_seg = (const char *)a.u + ((size_t)sc.b * a.u_bs + (size_t)sc.row_lo * a.u_ds + l0) * es;
                const char *gd_seg = (const char *)a.delta + ((size_t)sc.b * a.delta_bs + l0) * es;
                const char *gdo_seg = (const char *)a.dout + ((size_t)sc.b * a.dout_bs + (size_t)sc.row_lo * a.dout_ds + l0) * eso;
                char *du_seg = (char *)a.du + ((size_t)sc.b * a.du_bs + (size_t)sc.row_lo * a.du_ds + l0 + tok0) * es;
                char *dd_seg = (char *)a.ddelta + ((size_t)sc.b * a.dd_bs + (size_t)sc.row_lo * a.dd_ds + l0 + tok0) * es;
                const size_t du_step = (size_t)a.du_ds * es, dd_step = (size_t)a.dd_ds * es;
                for (int t = 0; t < tiles; ++t, ++kr) {
                    const int sr = kr % a.stages;
                    mbar_wait(rfull + sr, (kr / a.stages) & 1);
                    const char *st = smem + (size_t)sr * a.stage_bytes;
                    const int r0 = t * RT, nr = min(RT, sc.nrows - r0), d0 = sc.row_lo + r0;
                    const int dg0 = d0 / a.delta_ratio;
                    const char *gu = gu_seg + (size_t)r0 * a.u_ds * es;
                    const char *gd = gd_seg + (size_t)dg0 * a.delta_ds * es;
                    const char *gdo = gdo_seg + (size_t)r0 * a.dout_ds * eso;
                    const RowView vu = make_view(st + a.off_u, gu, a.u_ds, len, es, a.row_pitch, a.flat_u);
                    const RowView vd = make_view(st + a.off_delta, gd, a.delta_ds, len, es, a.row_pitch, a.flat_delta);
                    const RowView vdo = make_view(st + a.off_dout, gdo, a.dout_ds, len, eso, a.rowo_pitch, a.flat_dout);
                    const float *h0s = reinterpret_cast<const float *>(st + a.off_h0);
                    char *du_tile = du_seg + r0 * du_step;
                    char *dd_tile = dd_seg + r0 * dd_step;

                    for (int rb = warp * RPP; rb < nr; rb += NW * RPP) {
                        const bool active = rb + sub < nr;
                        const int r = active ? rb + sub : nr - 1;
                        const int rs = r0 + r, d = d0 + r;
                        const int rdelta = a.delta_ratio == 1 ? r : d / a.delta_ratio - dg0;
                        float u8[kTok], dl[kTok], dy[kTok], du[kTok], ddl[kTok], sg[kTok];
                        lds8<T>(vu.row(r) + tok0 * es, u8);
                        lds8<T>(vd.row(rdelta) + tok0 * es, dl);
                        if (a.out_f32) lds8<float>(vdo.row(r) + tok0 * 4, dy); else lds8<T>(vdo.row(r) + tok0 * es, dy);
                        if (a.has_z) {
                            // out_z = y * silu(z):  dy = dout * silu(z);  dz = dout * y * sigmoid(z) * (1 + z (1 - sigmoid(z)))
                            const char *gz = (const char *)a.z + ((size_t)sc.b * a.z_bs + (size_t)d0 * a.z_ds + l0) * es;
                            const char *gos = (const char *)a.out_saved + ((size_t)sc.b * a.osaved_bs + (size_t)d0 * a.osaved_ds + l0) * eso;
                            const RowView vz = make_view(st + a.off_z, gz, a.z_ds, len, es, a.row_pitch, a.flat_z);
                            const RowView vo = make_view(st + a.off_osaved, gos, a.osaved_ds, len, eso, a.rowo_pitch, a.flat_osaved);
                            float z8[kTok], o8[kTok], dz[kTok];
                            lds8<T>(vz.row(r) + tok0 * es, z8);
                            if (a.out_f32) lds8<float>(vo.row(r) + tok0 * 4, o8); else lds8<T>(vo.row(r) + tok0 * es, o8);
#pragma unroll
                            for (int i = 0; i < kTok; ++i) {
                                const float sz = rcpf(1.f + ex2f(-z8[i] * kLog2e));
                                dz[i] = dy[i] * o8[i] * sz * (1.f + z8[i] * (1.f - sz));
                                dy[i] = dy[i] * z8[i] * sz;
                            }
                            if (active && nval > 0) {
                                char *gdz = (char *)a.dz + ((size_t)sc.b * a.dz_bs + (size_t)d * a.dz_ds + l0 + tok0) * es;
                                st8<T>(gdz, dz, nval);
                            }
                        }
                        // tokens past the end of the sequence come FIRST in the suffix scan: their dy must be zero
                        // (everything they could contribute is proportional to dy or to the G chain it starts)
                        // -- and idle sub-rows (shadowing a valid row) must not reach the register accumulators.
                        if (nval < kTok || !active) {
                            const int nv = active ? nval : 0;
#pragma unroll
                            for (int i = 0; i < kTok; ++i) dy[i] = i < nv ? dy[i] : 0.f;
                        }
                        const float bias = pbias[rs], Dv = pD[rs];
                        float dDv = 0.f, dA1 = 0.f;
#pragma unroll
                        for (int i = 0; i < kTok; ++i) {
                            const float xv = dl[i] + bias;
                            sg[i] = 1.f;
                            dl[i] = kSoftplus ? softplus_f<true>(xv, sg[i]) : xv;
                            du[i] = Dv * dy[i];
                            dDv = fmaf(dy[i], u8[i], dDv);
                            ddl[i] = 0.f;
                        }
                        for (int n = 0; n < N; ++n) {
                            const float A2 = pA[rs * N + n];
                            const float Araw = A2 * kLn2;
                            if (!kN1) {
                                lds8<T>(vB.row(n) + tok0 * es, B8);
                                lds8<T>(vC.row(n) + tok0 * es, C8);
                            }
                            // ---- forward recompute: lane aggregate, warp scan, per-token states
                            float av[kTok], ah[kTok];
                            float pa = 1.f, pb = 0.f;
#pragma unroll
                            for (int i = 0; i < kTok; ++i) {
                                av[i] = ex2f(dl[i] * A2);
                                ah[i] = dl[i] * u8[i] * B8[i];      // b_t for now
                                pb = fmaf(av[i], pb, ah[i]);
                                pa *= av[i];
                            }
                            const float h0 = first_chunk ? 0.f : h0s[r * N + n];
                            float ea, eb;
                            seg_scan_fwd<kLPR>(pa, pb, ea, eb, j, LPR);
                            float hm = fmaf(ea, h0, eb);
                            float dCv[kTok];
#pragma unroll
                            for (int i = 0; i < kTok; ++i) {
                                const float tt = av[i] * hm;         // a_t h_{t-1}
                                hm = tt + ah[i];                     // h_t
                                ah[i] = tt;
                                if (kN1) dCacc[i] = fmaf(dy[i], hm, dCacc[i]); else dCv[i] = dy[i] * hm;
                            }
                            // ---- suffix scan of G
                            float ra = 1.f, rb2 = 0.f;
#pragma unroll
                            for (int i = kTok - 1; i >= 0; --i) {
                                rb2 = av[i] * fmaf(dy[i], C8[i], rb2);
                                ra *= av[i];
                            }
                            const float gin = last_chunk ? 0.f : carryG[rs * N + n];
                            seg_scan_rev<kLPR>(ra, rb2, ea, eb, j, LPR);
                            float Gn = fmaf(ea, gin, eb);            // G entering from the first token after this lane
                            float dAv = 0.f;
                            float dBv[kTok];
#pragma unroll
                            for (int i = kTok - 1; i >= 0; --i) {
                                const float g = fmaf(dy[i], C8[i], Gn);
                                const float gB2 = g * B8[i];
                                du[i] = fmaf(gB2, dl[i], du[i]);
                                const float gah = g * ah[i];
                                ddl[i] = fmaf(gB2, u8[i], ddl[i]);
                                ddl[i] = fmaf(gah, Araw, ddl[i]);
                                dAv = fmaf(gah, dl[i], dAv);
                                const float gdl = g * dl[i];
                                if (kN1) dBacc[i] = fmaf(gdl, u8[i], dBacc[i]); else dBv[i] = gdl * u8[i];
                                Gn = av[i] * g;
                            }
                            if (!first_chunk) {
                                __syncwarp();
                                if (j == 0 && active) carryG[rs * N + n] = Gn;   // G at this chunk's first token, for chunk c-1
                            }
                            // ---- dA: reduce over the row's lanes, accumulate over chunks (d_state == 1 on full warps: fused with
                            //      dD / dbias below)
                            if (!(kN1 && kLPR == 32)) {
                                dAv = seg_sum<kLPR>(dAv, LPR);
                                if (j == 0 && active) {
                                    const float tot = last_chunk ? dAv : dAv + carryA[rs * N + n];
                                    if (first_chunk) a.part_dA[(size_t)(sc.b * a.dim + d) * N + n] = tot;
                                    else carryA[rs * N + n] = tot;
                                }
                            } else {
                                dA1 = dAv;
                            }
                            // ---- dB / dC over rows (d_state > 1): vector reductions into the L2-resident accumulator, or
                            //      (kDet) sub-rows folded by a butterfly, then the ordered add of the row group
                            if (kDet && !kN1) {
#pragma unroll
                                for (int i = 0; i < kTok; ++i) {
                                    dBv[i] = active ? dBv[i] : 0.f;
                                    dCv[i] = active ? dCv[i] : 0.f;
                                }
                                if (kLPR != 32) {
                                    for (int off = LPR; off < 32; off <<= 1) {
#pragma unroll
                                        for (int i = 0; i < kTok; ++i) {
                                            dBv[i] += __shfl_xor_sync(0xffffffffu, dBv[i], off);
                                            dCv[i] += __shfl_xor_sync(0xffffffffu, dCv[i], off);
                                        }
                                    }
                                }
                                const int q = t * det_gpt + rb / RPP;
                                det_ordered_add(det_runC + n * det_rstep, det_partC + (size_t)n * L, det_tick + n, det_base + q, q == 0,
                                                q == det_nq - 1, sub == 0, dCv, nval, lane, a.det_status);
                                det_ordered_add(det_runB + n * det_rstep, det_partB + (size_t)n * L, det_tick + N + n, det_base + q,
                                                q == 0, q == det_nq - 1, sub == 0, dBv, nval, lane, a.det_status);
                            }
                            if (!kDet && !kN1 && active && nval > 0) {
                                float *pB = a.acc_dB + ((size_t)(sc.b * a.G + sc.g) * N + n) * Lp + l0 + tok0;
                                float *pC = a.acc_dC + ((size_t)(sc.b * a.G + sc.g) * N + n) * Lp + l0 + tok0;
                                red_add_v4(pB, dBv[0], dBv[1], dBv[2], dBv[3]);
                                red_add_v4(pC, dCv[0], dCv[1], dCv[2], dCv[3]);
                                if (nval > 4) {
                                    red_add_v4(pB + 4, dBv[4], dBv[5], dBv[6], dBv[7]);
                                    red_add_v4(pC + 4, dCv[4], dCv[5], dCv[6], dCv[7]);
                                }
                            }
                        }
                        // ---- per-row epilogue
                        float dbv = 0.f;
#pragma unroll
                        for (int i = 0; i < kTok; ++i) {
                            if (kSoftplus) ddl[i] *= sg[i];
                            dbv += ddl[i];
                        }
                        if (active && nval > 0) {
                            st8<T>(du_tile + r * du_step, du, nval);
                            if (a.delta_ratio == 1) {
                                st8<T>(dd_tile + r * dd_step, ddl, nval);
                            } else {
                                float *gdd = a.ddelta_full + ((size_t)(sc.b * a.dim + d)) * L + l0 + tok0;
                                st8<float>(gdd, ddl, nval);
                            }
                        }
                        if (kN1 && kLPR == 32) {
                            // one 6-shuffle reduction for (dA, dD, dbias): totals land in lanes 0 / 16 / 8
                            const float tot = warp_sum3(dA1, dDv, dbv, lane);
                            if (active && (lane == 0 || lane == 16 || lane == 8)) {
                                float *cr = lane == 0 ? carryA : (lane == 16 ? carryD : carryBias);
                                float *gp = lane == 0 ? a.part_dA : (lane == 16 ? a.part_dD : a.part_dbias);
                                const float t2 = last_chunk ? tot : tot + cr[rs];
                                if (first_chunk) gp[(size_t)sc.b * a.dim + d] = t2; else cr[rs] = t2;
                            }
                        } else {
                            dDv = seg_sum<kLPR>(dDv, LPR);
                            dbv = seg_sum<kLPR>(dbv, LPR);
                            if (j == 0 && active) {
                                const float tD = last_chunk ? dDv : dDv + carryD[rs];
                                const float tb = last_chunk ? dbv : dbv + carryBias[rs];
                                if (first_chunk) {
                                    a.part_dD[(size_t)sc.b * a.dim + d] = tD;
                                    a.part_dbias[(size_t)sc.b * a.dim + d] = tb;
                                } else {
                                    carryD[rs] = tD;
                                    carryBias[rs] = tb;
                                }
                            }
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(rempty + sr);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(gempty + sg);
                det_base += det_nq;

                if (kN1) {
                    // ---- fold this warp's dB/dC (summed over its rows of the segment) with the other warps' and emit the
                    // segment partial.  Slot p = lane*8 + i = sub*CH + token.  Fixed order -> bit-reproducible.
                    const int tid = threadIdx.x;  // consumer threads are 0 .. NW*32-1
#pragma unroll
                    for (int which = 0; which < 2; ++which) {
                        float4 *mine = reinterpret_cast<float4 *>(red + warp * 256 + lane * kTok);
                        if (which == 0) { mine[0] = make_float4(dBacc[0], dBacc[1], dBacc[2], dBacc[3]); mine[1] = make_float4(dBacc[4], dBacc[5], dBacc[6], dBacc[7]); }
                        else { mine[0] = make_float4(dCacc[0], dCacc[1], dCacc[2], dCacc[3]); mine[1] = make_float4(dCacc[4], dCacc[5], dCacc[6], dCacc[7]); }
                        consumer_bar(NW * 32);
                        if (tid < len) {
                            float sum = 0.f;
                            for (int w = 0; w < NW; ++w)
                                for (int sb = 0; sb < RPP; ++sb) sum += red[w * 256 + sb * CH + tid];
                            float *dst = (which == 0 ? a.acc_dB : a.acc_dC) + (size_t)seg * L + l0 + tid;
                            *dst = sum;
                        }
                        consumer_bar(NW * 32);
                    }
                }
            }
        }
    }
}

// kDet: the deterministic d_state > 1 instantiations (d_state 1 is deterministic without them)
template <typename T, bool kDet = false>
cudaError_t launch_bwd(const ScanArgs &a, int grid, cudaStream_t stream) {
    void (*kernel)(const ScanArgs);
    const bool n1 = a.N == 1, w32 = a.LPR == 32;
#define MIA_PICK(SP, N1) (w32 ? &ss_bwd_kernel<T, SP, N1, 32, kDet> : &ss_bwd_kernel<T, SP, N1, 0, kDet>)
    if constexpr (kDet) {
        kernel = a.softplus ? MIA_PICK(true, false) : MIA_PICK(false, false);
    } else {
        if (a.softplus) kernel = n1 ? MIA_PICK(true, true) : MIA_PICK(true, false);
        else kernel = n1 ? MIA_PICK(false, true) : MIA_PICK(false, false);
    }
#undef MIA_PICK
    return launch_smem(kernel, grid, kThreads, a.smem_bytes, stream, a);
}

}  // namespace mia
