// Host side of libmia_scan.so: argument validation (the reference's TORCH_CHECKs,
// selective_scan_oflex.cpp:152-204 / 245-312), tile planning, launches, the finalize kernel that folds the
// backward's deterministic partials, and the extern "C" surface declared in include/mia_selective_scan.h.
#include <algorithm>
#include <initializer_list>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "../../include/mia_selective_scan.h"
#include "abi_host.h"
#include "scan_common.cuh"
#include "scan_bwd_rows.cuh"
#include "scan_bwd_rowsn.cuh"
#include "scan_bwd_cw.cuh"
#include "tma_host.h"
#include "scan_fwd_rowsn.cuh"
#include "scan_fwd_stream.cuh"
#include "scan_fwd_chunks.cuh"
#include "scan_fwd_cw.cuh"

namespace mia {
template <typename T> cudaError_t launch_fwd_rows(const RowsArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_fwd_rowsn(const RowsNArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_fwd_stream(const StreamArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_fwd_chunks(const ChunkArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_fwd_cw(const CUtensorMap *, const CwFwdArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_bwd_rows(const RowsBwdArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_bwd_rowsn(const RowsNBwdArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_bwd_cw(const CUtensorMap *, const CwBwdArgs &, int, bool, cudaStream_t);
template <typename T> cudaError_t launch_fwd_any(const ScanArgs &, int, cudaStream_t);
template <typename T> cudaError_t launch_bwd_any(const ScanArgs &, int, cudaStream_t);
template <typename T> cudaError_t launch_bwd_det(const ScanArgs &, int, cudaStream_t);
}  // namespace mia

namespace {

#define MIA_CHECK(cond, ...) \
    do { if (!(cond)) return mia::fail(mia::kErrScan, MIA_EINVAL, __VA_ARGS__); } while (0)
#define MIA_CUDA(expr) \
    do { if (int rc__ = mia::cuda_fail(mia::kErrScan, #expr, (expr))) return rc__; } while (0)

using mia::DeviceInfo;

// Debugging knobs (force a kernel family, move the half split) exist only in -DMIA_DEBUG builds; the release library
// reads no environment variable and has no mode that alters results.
#ifdef MIA_DEBUG
bool dbg_knob(const char *name) { return getenv(name) != nullptr; }
int dbg_int(const char *name, int dflt) { const char *v = getenv(name); return v ? atoi(v) : dflt; }
#define MIA_TRACE(...) do { if (getenv("MIA_TRACE")) { fprintf(stderr, "[mia] " __VA_ARGS__); fputc('\n', stderr); } } while (0)
#else
#define MIA_TRACE(...) do { } while (0)
constexpr bool dbg_knob(const char *) { return false; }
constexpr int dbg_int(const char *, int dflt) { return dflt; }
#endif

int esize(int dt) { return dt == MIA_F32 ? 4 : 2; }
int round_up(int x, int m) { return (x + m - 1) / m * m; }

int lanes_per_row(int L) {
    if (L > 128) return 32;
    int need = (L + mia::kTok - 1) / mia::kTok, lpr = 4;
    while (lpr < need) lpr <<= 1;
    return lpr;
}

struct WorkspaceLayout {
    size_t part_dA = 0, part_dD = 0, part_dbias = 0, acc_dB = 0, acc_dC = 0, ddelta_full = 0, total = 0;
    size_t acc_bytes = 0;
    bool bc_atomic = false;
};

// Work plan shared by fwd and bwd (the checkpoint geometry must match between them).
struct Plan {
    int LPR, CH, n_chunks, RPP, NW, RT, RS, split, tiles_per_seg, n_seg;
};

void set_split(Plan &pl, const mia_ss_params &p, int split) {
    const int rpg = p.dim / p.n_groups;
    pl.RS = (rpg + split - 1) / split;
    pl.split = (rpg + pl.RS - 1) / pl.RS;
    pl.tiles_per_seg = (pl.RS + pl.RT - 1) / pl.RT;
    pl.n_seg = p.batch * p.n_groups * pl.split;
}

// det: the deterministic d_state > 1 backward, whose dB / dC leave as one partial per segment (N L floats each): it aims at
// ~1 segment per SM instead of ~6, which bounds those partials at about (SMs + 3 B G) 8 N L bytes.
Plan make_plan(const mia_ss_params &p, int sms, bool bwd, bool det = false) {
    Plan pl;
    pl.LPR = lanes_per_row(p.seqlen);
    pl.CH = pl.LPR * mia::kTok;
    pl.n_chunks = (p.seqlen + pl.CH - 1) / pl.CH;
    pl.RPP = 32 / pl.LPR;
    pl.NW = (bwd ? mia::kThreads : mia::kThreadsFwd) / 32 - 1;
    pl.RT = pl.NW * pl.RPP * (bwd ? 4 : 3);   // row passes per warp and row stage (amortises the per-stage bookkeeping)
    const int rpg = p.dim / p.n_groups;
    // Segments: (batch, group, row range).  Aim at >= ~6 segments per SM with the best last-wave balance; a segment
    // keeps its carries in shared memory, so bound rows * d_state.
    const long long bg = (long long)p.batch * p.n_groups;
    int max_split = (rpg + pl.RPP - 1) / pl.RPP;
    int min_split = 1;
    while ((long long)((rpg + min_split - 1) / min_split) * p.dstate > 4096 && min_split < max_split) ++min_split;
    int want = (int)(((det ? 1LL : 6LL) * sms + bg - 1) / bg);
    if (want < min_split) want = min_split;
    if (want > max_split) want = max_split;
    int best = want;
    double best_eff = -1.0;
    for (int sp = want; sp <= want + 3 && sp <= max_split; ++sp) {
        Plan t = pl;
        set_split(t, p, sp);
        const double waves = (double)t.n_seg / sms;
        const double eff = waves / (double)((t.n_seg + sms - 1) / sms);
        if (eff > best_eff + 1e-9) { best_eff = eff; best = sp; }
    }
    set_split(pl, p, best);
    return pl;
}

// Work split of the deterministic d_state 16 backward (scan_bwd_rowsn.cuh): sizes only, shared by the workspace query and
// the launch.  Returns false when the shape is not one it takes.
struct RowsNSplit { int n_oct, oct_per_cta, oct_per_group, grid, max_parts; };
bool rowsn_bwd_split(const mia_ss_params &p, int sms, int ctas_per_sm, RowsNSplit &sp) {
    const int rpg = p.dim / p.n_groups;
    if (p.dstate != 16 || p.delta_dim != p.dim || p.seqlen > 256 || (rpg % mia::kRnOct)) return false;
    sp.n_oct = (int)((long long)p.batch * p.dim / mia::kRnOct);
    sp.oct_per_group = rpg / mia::kRnOct;
    const int slots = sms * ctas_per_sm;
    sp.oct_per_cta = (sp.n_oct + slots - 1) / slots;
    sp.grid = (sp.n_oct + sp.oct_per_cta - 1) / sp.oct_per_cta;
    sp.max_parts = (sp.oct_per_group + sp.oct_per_cta - 2) / sp.oct_per_cta + 1;   // CTAs a group's octets can straddle
    return true;
}
constexpr int kRowsNCtasPerSm = 3;   // the split (hence the partial layout) is fixed at 3 CTAs per SM: launching fewer
                                     // resident CTAs (z gate, fp32) only queues them

WorkspaceLayout workspace_layout(const mia_ss_params &p, const Plan &pl, int sms, bool det = false) {
    WorkspaceLayout w;
    auto take = [&](size_t nfloat) { size_t off = w.total; w.total += (nfloat * 4 + 255) / 256 * 256; return off; };
    w.bc_atomic = p.dstate > 1 && !det;     // det: per-segment partials at every d_state
    w.part_dA = take((size_t)p.batch * p.dim * p.dstate);
    w.part_dD = take((size_t)p.batch * p.dim);
    w.part_dbias = take((size_t)p.batch * p.dim);
    // d_state == 1: one partial row per segment (warp-scan kernels) or per 32-row batch (row-serial kernel); the query
    // cannot know which of the two will run (it depends on strides and alignment), so size for the larger.
    const int rpg = p.dim / p.n_groups;
    const size_t row_items = (p.dstate == 1 && rpg % 32 == 0) ? (size_t)p.batch * p.n_groups * (rpg / 32) : 0;
    const size_t parts = row_items > (size_t)pl.n_seg ? row_items : (size_t)pl.n_seg;
    size_t nacc = w.bc_atomic ? (size_t)p.batch * p.n_groups * p.dstate * ((p.seqlen + 3) & ~3) : parts * p.dstate * p.seqlen;
    RowsNSplit rs;
    if (rowsn_bwd_split(p, sms, kRowsNCtasPerSm, rs)) {   // whichever d_state 16 kernel runs (it depends on strides), its buffer fits
        const size_t need = (size_t)p.batch * p.n_groups * rs.max_parts * p.dstate * p.seqlen;
        if (need > nacc) nacc = need;
    }
    w.acc_dB = take(nacc);
    w.acc_dC = take(nacc);
    w.acc_bytes = nacc * 4;
    if (p.dim != p.delta_dim) w.ddelta_full = take((size_t)p.batch * p.dim * p.seqlen);
    return w;
}

int validate_sizes(const mia_ss_params &p) {
    MIA_CHECK(p.itype == MIA_F32 || p.itype == MIA_F16 || p.itype == MIA_BF16, "u must be float32, float16 or bfloat16");
    MIA_CHECK(p.otype == p.itype || p.otype == MIA_F32, "out/dout dtype must be the input dtype or float32");
    MIA_CHECK(p.batch > 0 && p.dim > 0 && p.seqlen > 0 && p.dstate > 0 && p.n_groups > 0 && p.delta_dim > 0, "empty or negative size");
    MIA_CHECK(p.dim % p.n_groups == 0, "dims should be dividable by n_groups");
    MIA_CHECK(p.dim % p.delta_dim == 0, "dims should be dividable by delta_dim");
    MIA_CHECK(p.dstate <= 256, "selective_scan only supports state dimension <= 256");
    MIA_CHECK((long long)p.batch * p.dim < (1LL << 31) / 2, "batch*dim too large");
    return MIA_OK;
}

int validate_common(const mia_ss_params &p) {
    if (int rc = validate_sizes(p)) return rc;
    MIA_CHECK(p.u && p.delta && p.A && p.B && p.C, "u, delta, A, B, C must not be null");
    MIA_CHECK(p.n_chunks == mia_ss_num_chunks(p.seqlen), "x must have %d chunks for seqlen %d (got %d)", mia_ss_num_chunks(p.seqlen),
              p.seqlen, p.n_chunks);
    return MIA_OK;
}

void fill_common(mia::ScanArgs &a, const mia_ss_params &p, const Plan &pl) {
    memset(&a, 0, sizeof(a));
    a.batch = p.batch; a.dim = p.dim; a.L = p.seqlen; a.N = p.dstate; a.G = p.n_groups; a.delta_dim = p.delta_dim;
    a.rows_per_group = p.dim / p.n_groups;
    a.delta_ratio = p.dim / p.delta_dim;
    a.softplus = p.delta_softplus; a.has_z = p.z != nullptr; a.out_f32 = (p.otype == MIA_F32) && (p.itype != MIA_F32);
    a.RT = pl.RT; a.RS = pl.RS; a.split = pl.split; a.tiles_per_seg = pl.tiles_per_seg; a.LPR = pl.LPR; a.CH = pl.CH;
    a.n_chunks = pl.n_chunks; a.n_seg = pl.n_seg; a.n_consumer_warps = pl.NW;
    a.u = p.u; a.delta = p.delta; a.A = p.A; a.B = p.B; a.C = p.C; a.D = p.D; a.delta_bias = p.delta_bias; a.z = p.z;
    a.x = p.x;
    a.u_bs = p.u_batch_stride; a.u_ds = p.u_d_stride; a.delta_bs = p.delta_batch_stride; a.delta_ds = p.delta_d_stride;
    a.z_bs = p.z_batch_stride; a.z_ds = p.z_d_stride; a.A_ds = p.A_d_stride; a.A_ns = p.A_dstate_stride;
    a.B_bs = p.B_batch_stride; a.B_gs = p.B_group_stride; a.B_ns = p.B_dstate_stride;
    a.C_bs = p.C_batch_stride; a.C_gs = p.C_group_stride; a.C_ns = p.C_dstate_stride;
    const bool whole = pl.n_chunks == 1;
    a.flat_u = whole && p.u_d_stride == p.seqlen;
    a.flat_delta = whole && p.delta_d_stride == p.seqlen;
    a.flat_z = a.has_z && whole && p.z_d_stride == p.seqlen;
    a.flat_B = whole && p.B_dstate_stride == p.seqlen;
    a.flat_C = whole && p.C_dstate_stride == p.seqlen;
}

// Shared-memory carve-up.  Returns false if not even two row stages fit.  det: also the tickets and (det_acc, and 2 N CH
// floats fit in 32 KB) the running sums of the deterministic d_state > 1 backward (scan_bwd.cuh).
bool layout_smem(mia::ScanArgs &a, int es, int eso, bool bwd, int smem_max, bool det = false, bool det_acc = false) {
    const int span = a.CH < a.L ? a.CH : a.L;
    a.row_pitch = round_up(span * es, 16) + 16;
    a.rowo_pitch = round_up(span * eso, 16) + 16;
    a.bc_pitch = a.row_pitch;
    const int slack = a.CH * 4 + 16;   // an 8-token vector read may run past the last row of a region
    int off = 0;
    auto region = [&](int rows, int pitch) { int o = off; off += round_up(rows * pitch + slack, 128); return o; };
    a.off_u = region(a.RT, a.row_pitch);
    a.off_delta = region(a.RT, a.row_pitch);
    if (a.has_z) a.off_z = region(a.RT, a.row_pitch);
    if (bwd) {
        a.off_dout = region(a.RT, a.rowo_pitch);
        if (a.has_z) a.off_osaved = region(a.RT, a.rowo_pitch);
        a.off_h0 = off; off += round_up(a.RT * a.N * 4, 128);
    }
    a.stage_bytes = off;
    off = 0;
    a.goff_B = region(a.N, a.bc_pitch);
    a.goff_C = region(a.N, a.bc_pitch);
    a.goff_A = off; off += round_up(a.RS * a.N * 4, 128);
    a.goff_D = off; off += round_up(a.RS * 4, 128);
    a.goff_bias = off; off += round_up(a.RS * 4, 128);
    a.gstage_bytes = off;
    const int bars = round_up((2 * mia::kMaxStages + 2 * mia::kGroupStages) * 8, 128);
    const int carry = round_up(bwd ? (2 * a.RS * a.N + 2 * a.RS) * 4 : a.RS * a.N * 8, 128);
    const int red = bwd ? a.n_consumer_warps * 256 * 4 : 0;
    const int tickets = round_up(2 * a.N * 4, 128);
    a.det_smem_acc = det && det_acc && 2 * a.N * a.CH * 4 <= 32768;
    const int det_bytes = det ? tickets + (a.det_smem_acc ? 2 * a.N * a.CH * 4 : 0) : 0;
    const int fixed = mia::kGroupStages * a.gstage_bytes + bars + carry + red + det_bytes;
    int stages = (smem_max - fixed) / a.stage_bytes;
    if (stages > mia::kMaxStages) stages = mia::kMaxStages;
    if (stages < 2) return false;
    a.stages = stages;
    a.off_groups = stages * a.stage_bytes;
    a.off_bars = a.off_groups + mia::kGroupStages * a.gstage_bytes;
    a.off_carry = a.off_bars + bars;
    a.off_red = a.off_carry + carry;
    a.smem_bytes = a.off_red + red;
    if (det) {
        a.off_det = a.smem_bytes;
        a.off_det_acc = a.off_det + tickets;
        a.smem_bytes += det_bytes;
    }
    return true;
}

// Pick the work plan and carve shared memory; if it does not fit, first cut segments finer (smaller carries and
// parameter blocks), then halve the row tile; det: as a last resort keep the running sums in the partials, not in shared memory.
int plan_and_layout(const mia_ss_params &p, const DeviceInfo &di, bool bwd, Plan &pl, mia::ScanArgs &a, bool det = false) {
    pl = make_plan(p, di.sms, bwd, det);
    bool det_acc = det;
    const int es = esize(p.itype), eso = esize(p.otype);
    const int rpg = p.dim / p.n_groups;
    for (;;) {
        fill_common(a, p, pl);
        if (bwd) {
            const bool whole = pl.n_chunks == 1;
            a.flat_dout = whole && p.dout_d_stride == p.seqlen;
            a.flat_osaved = a.has_z && whole && p.out_saved_d_stride == p.seqlen;
        }
        if (layout_smem(a, es, eso, bwd, di.smem_optin, det, det_acc)) return MIA_OK;
        if (pl.RS > pl.RT) {
            set_split(pl, p, pl.split * 2 < rpg ? pl.split * 2 : rpg);
        } else if (det_acc && pl.RT <= pl.RPP) {
            det_acc = false;
            pl = make_plan(p, di.sms, bwd, det);
        } else {
            MIA_CHECK(pl.RT > pl.RPP, "tile does not fit in shared memory (dstate %d, seqlen %d)", p.dstate, p.seqlen);
            pl.RT = pl.RT / 2 < pl.RPP ? pl.RPP : pl.RT / 2;
            set_split(pl, p, pl.split);
        }
    }
}

// Eligibility checks shared by the planners below.  Each plan_* states only what is particular to its family.
struct RowStrides { long long bs, ds; };   // one (batch, dim, L) operand: batch and row strides in elements
#define MIA_ROWS(t) RowStrides{p.t##_batch_stride, p.t##_d_stride}

// The operands are dense (batch, dim, L) rows: rows L elements apart, batches dim L apart.
bool dense_rows(const mia_ss_params &p, std::initializer_list<RowStrides> ops) {
    for (const RowStrides &o : ops)
        if (o.ds != p.seqlen || o.bs != (long long)p.dim * p.seqlen) return false;
    return true;
}

// Every pointer is a multiple of `bytes` (a power of two).
bool aligned(uintptr_t bytes, std::initializer_list<const void *> ptrs) {
    uintptr_t bits = 0;
    for (const void *q : ptrs) bits |= (uintptr_t)q;
    return (bits & (bytes - 1)) == 0;
}

// What every d_state 1 row-serial kernel needs: one delta row per row, no gate, whole 32-row batches in a group, rows of
// whole 4-token pieces.
bool rowwise_n1(const mia_ss_params &p) {
    return p.dstate == 1 && !p.z && p.delta_dim == p.dim && (p.dim / p.n_groups) % 32 == 0 && p.seqlen % 4 == 0;
}

// The d_state 1 row-serial kernels read A as one float per row.
bool a_per_row(const mia_ss_params &p) { return p.A_d_stride == 1 || p.dim == 1; }

// Shared memory per SM as the planners count it: the 227 KB one CTA may opt in to.
constexpr int kSmemPerSm = 227 * 1024;

// Grid of a persistent kernel: as many CTAs per SM as `capacity` bytes of shared memory hold at `smem` bytes each (plus the
// 1 KB the SM reserves per CTA), at most hi, on every SM, at most one per item; 0 when fewer than lo fit (the family declines).
int resident_grid(const DeviceInfo &di, int smem, int capacity, int lo, int hi, int n_items) {
    const int per_sm = std::min(capacity / (smem + 1024), hi);
    return per_sm < lo ? 0 : std::min(di.sms * per_sm, n_items);
}

template <typename R, typename = void> struct HasRows : std::false_type {};
template <typename R> struct HasRows<R, std::void_t<decltype(R::u)>> : std::true_type {};
template <typename R, typename = void> struct HasOut : std::false_type {};
template <typename R> struct HasOut<R, std::void_t<decltype(R::out)>> : std::true_type {};

// Zero a row-serial or column-walk argument block and fill the fields they all share.
template <typename R>
void fill_rows_common(R &r, const mia_ss_params &p) {
    memset(&r, 0, sizeof(r));
    r.batch = p.batch; r.dim = p.dim; r.L = p.seqlen; r.G = p.n_groups; r.rows_per_group = p.dim / p.n_groups;
    r.softplus = p.delta_softplus;
    r.A = p.A; r.B = p.B; r.C = p.C; r.D = p.D; r.delta_bias = p.delta_bias;
    r.B_bs = p.B_batch_stride; r.B_gs = p.B_group_stride; r.C_bs = p.C_batch_stride; r.C_gs = p.C_group_stride;
    if constexpr (HasRows<R>::value) { r.u = p.u; r.delta = p.delta; }
    if constexpr (HasOut<R>::value) r.out = p.out;
}

// Geometry of the column-walk kernels (scan_fwd_cw.cuh / scan_bwd_cw.cuh): g rows per tensor-map row.  A pure function of the
// problem's sizes and dtypes (and the SM count) -- it also fixes the LAYOUT of the block states (hblk), which forward and backward must agree on.
// A tensor-map row must be a multiple of 16 bytes (else the map cannot be encoded); it SHOULD be a multiple of 32 (else every
// other row starts mid-sector and every 64-byte box row touches three sectors instead of two, e.g.
// L = 196 bf16 with g = 2).  2-byte types: the smallest g in {1, 2, 4} with g L a multiple of 16 elements, falling back to a
// smaller legal g when rows_per_group is not a multiple of 32 g or when the item count falls between one and two rounds; g > 1
// only for rows of one checkpoint chunk (L <= 256: the kernels write x at row ends only when they walk several rows per
// lane).  fp32 rows (L % 4 == 0) are always legal: g = 1.
bool cw_geometry(const mia_ss_params &p, int sms, int &g) {
    const int es = esize(p.itype), L = p.seqlen;
    if (!rowwise_n1(p)) return false;
    const int rpg = p.dim / p.n_groups;
    if (es == 4) { g = 1; return true; }
    const int want = (L % 16 == 0) ? 1 : (L % 8 == 0) ? 2 : 4;
    // Items are 32 g rows: a larger g halves their number, and a problem that fills the resident slots a little more than once
    // pays a whole second round -> take the preferred g when its items fit one round or make at least two, else the next smaller
    // legal one.  (~9 resident warps per SM with fp32 outputs / gradients, 12 otherwise; the same estimate for both directions,
    // since forward and backward must pick the same g.)
    const long long slots = (long long)sms * ((esize(p.otype) == 4) ? 9 : 12);
    int fallback = 0;
    for (int c = want; c >= 1; c >>= 1) {
        if (((long long)c * L * es) % 16) break;                 // not a legal tensor-map row any more
        if (c > 1 && L > 256) continue;
        if (rpg % (32 * c)) continue;
        const long long n_items = (long long)p.batch * p.n_groups * (rpg / (32 * c));
        if (n_items <= slots || n_items >= 2 * slots) { g = c; return true; }
        if (!fallback) fallback = c;
    }
    if (fallback) { g = fallback; return true; }
    return false;
}

// Row-serial forward (scan_fwd_rows.cuh): eligibility + argument block.  Returns false when the warp-scan kernels must run.
bool plan_rows_fwd(const mia_ss_params &p, const DeviceInfo &di, mia::RowsArgs &r, int &grid) {
    const int es = esize(p.itype), L = p.seqlen;
    if (!rowwise_n1(p)) return false;
    if (dbg_knob("MIA_NO_ROWS_FWD")) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(out)}) || !a_per_row(p) || !aligned(16, {p.u, p.delta, p.out})) return false;
    const int budget = 13 * 1024;                               // bytes of one [32 x chunk] tile (8 warps per SM at 2-byte dtypes)
    int Lc = L;
    if (32 * L * es > budget) {
        if ((L * es) % 16) return false;                        // per-row pieces must start 16-byte aligned
        Lc = budget / (32 * es) / 8 * 8;
    }
    fill_rows_common(r, p);
    r.Lc = Lc; r.n_lchunks = (L + Lc - 1) / Lc;
    r.n_items = p.batch * p.n_groups * (r.rows_per_group / 32);
    r.tile_bytes = round_up(32 * Lc * es, 128);
    r.off_bc32 = 2 * r.tile_bytes;
    r.stage_bytes = r.off_bc32 + round_up(2 * Lc * 4, 128);
    r.smem_bytes = r.stage_bytes + 128;
    if (r.smem_bytes > di.smem_optin) return false;
    r.xchunks = mia_ss_num_chunks(L); r.xchunk_tokens = mia_ss_chunk_len(L);
    r.x = p.x;
    grid = di.smem_optin / (r.smem_bytes + 1024) > 0 ? resident_grid(di, r.smem_bytes, kSmemPerSm, 1, 8, r.n_items) : 0;
    if (!grid) grid = std::min(di.sms, r.n_items);              // a tile that leaves no room for the 1 KB reserve: one per SM
    return true;
}

// Column-walk forward (scan_fwd_cw.cuh): eligibility, argument block, tensor maps (u, delta, out).
bool plan_cw_fwd(const mia_ss_params &p, const DeviceInfo &di, mia::CwFwdArgs &r, CUtensorMap *tm, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    int g = 0;
    if (!cw_geometry(p, di.sms, g)) return false;
    if (dbg_knob("MIA_NO_CW_FWD")) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(out)}) || !a_per_row(p) || !aligned(16, {p.u, p.delta, p.out})) return false;
    const unsigned long long trows = (unsigned long long)p.batch * p.dim / g, tcols = (unsigned long long)g * L;
    if (tcols >= (1ull << 31) || trows >= (1ull << 31)) return false;
    const int n_items = p.batch * p.n_groups * (p.dim / p.n_groups / (32 * g));
    // few long rows: the chunk-parallel kernel (scan_fwd_chunks.cuh) has more warps to offer than one per 32 rows
    if (n_items < 4 * di.sms && (L + mia::kChunkTok - 1) / mia::kChunkTok >= 2 && !dbg_knob("MIA_FORCE_CW_FWD")) return false;
    fill_rows_common(r, p);
    r.zero = 0;                                                  // (the kernel XORs parameter loads with it: scan_fwd_cw.cuh, settle)
    r.g = g; r.n_items = n_items;
    r.nwin = (g * L + mia::kCwTok - 1) / mia::kCwTok;
    r.ngrp = (g * L + 15) / 16;
    const bool of32 = eo == 4 && es != 4;
    const int tile_i = 32 * mia::kCwTok * es, tile_o = 32 * mia::kCwTok * eo;
    r.stage_bytes = 2 * tile_i;
    r.ns = dbg_int("MIA_CW_STAGES", 3);                          // 3 stages, at most 6 resident warps per SM: see below
    r.off_out = r.ns * r.stage_bytes;
    r.off_bc32 = r.off_out + (of32 ? 2 * tile_o : 0);
    r.off_bar = r.off_bc32 + 2 * mia::kCwTok * 4;
    r.smem_bytes = r.off_bar + 8 * r.ns + 16;
    r.xchunks = mia_ss_num_chunks(L); r.xchunk_tokens = mia_ss_chunk_len(L);
    r.x = p.x; r.hblk = p.hblk;
    const void *ptrs[3] = {p.u, p.delta, p.out};
    for (int i = 0; i < 3; ++i) {
        const int e = i == 2 ? eo : es;
        const int trc = mia::tma_make_2d(&tm[i], ptrs[i], trows, tcols, tcols * e, 32, mia::kCwTok, e, mia::kCwTok * e);
        if (trc != 0) { MIA_TRACE("cw fwd: tensor map %d rejected (CUresult %d)", i, trc); return false; }
    }
    // At most 6 resident warps per SM.  The kernel is bound by DRAM, not by issue, and fewer concurrent row streams per SM move
    // its bytes faster: on an H100 (80GB HBM3, 700 W; bf16, R = 3072; debug-build knobs MIA_CW_STAGES / MIA_CW_MAXPERSM) 3 stages at 6 warps take 0.214 ms at B = 132, L = 196 and
    // 0.831 ms at B = 16, L = 6400, against 0.241 / 0.866 ms for 4 stages at 13 warps; 8 warps: 0.223 / 0.830 ms, 4 warps:
    // 0.225 / 0.876 ms, 2 stages: >= 0.232 / 0.926 ms, 4-10 stages at 6 warps: 0.225-0.235 / 0.856-0.885 ms.
    const int fill = resident_grid(di, r.smem_bytes, kSmemPerSm, 1, dbg_int("MIA_CW_MAXPERSM", 6), n_items);
    if (!fill) return false;
    const int rounds = (n_items + fill - 1) / fill;
    grid = (n_items + rounds - 1) / rounds;                      // equal rounds per CTA
    return true;
}

// Chunk-parallel forward for long rows and few 32-row batches (scan_fwd_chunks.cuh): eligibility + argument block.
bool plan_chunks_fwd(const mia_ss_params &p, const DeviceInfo &di, mia::ChunkArgs &r, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    if (!rowwise_n1(p)) return false;
    if (dbg_knob("MIA_NO_ROWS_FWD") || dbg_knob("MIA_NO_CHUNKS_FWD")) return false;
    const int nch = (L + mia::kChunkTok - 1) / mia::kChunkTok;
    if (nch < 2 || mia_ss_chunk_len(L) != mia::kChunkTok || ((L * es) % 16) || ((L * eo) % 16)) return false;
    const int n_batches = p.batch * p.n_groups * (p.dim / p.n_groups / 32);
    if (n_batches >= 4 * di.sms) return false;                 // enough rows: the serial row walk fills the machine
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(out)}) || !a_per_row(p) || !aligned(16, {p.u, p.delta, p.out})) return false;
    fill_rows_common(r, p);
    r.n_chunks = nch;
    r.n_items = n_batches * nch;
    r.tile_bytes = round_up(32 * (mia::kChunkTok * es + 16), 128);
    r.off_bc32 = 2 * r.tile_bytes;
    r.off_bar = r.off_bc32 + 2 * mia::kChunkTok * 4;
    r.smem_bytes = r.off_bar + 128;
    r.x = p.x;
    grid = resident_grid(di, r.smem_bytes, kSmemPerSm, 3, 8, r.n_items);
    return grid > 0;
}

// Streaming row-serial forward (scan_fwd_stream.cuh): eligibility + argument block.
bool plan_stream_fwd(const mia_ss_params &p, const DeviceInfo &di, mia::StreamArgs &r, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    if (!rowwise_n1(p)) return false;
    if (dbg_knob("MIA_NO_ROWS_FWD") || dbg_knob("MIA_NO_STREAM_FWD")) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(out)}) || !a_per_row(p)) return false;
    if (!aligned(4 * es, {p.u, p.delta}) || !aligned(4 * eo, {p.out})) return false;   // every row start is a multiple of one 4-token piece
    if (L > 256 && mia_ss_chunk_len(L) != 256) return false;
    fill_rows_common(r, p);
    r.n_items = p.batch * p.n_groups * (r.rows_per_group / 32);
    r.Lp = (L + 3) & ~3;
    const int pitch = mia::kStreamTok * es + 4 * es;
    r.off_bc32 = round_up(2 * 2 * 32 * pitch, 128);             // 2 stages x (u, delta)
    r.smem_bytes = r.off_bc32 + round_up(2 * r.Lp * 4, 128);
    if (r.smem_bytes > di.smem_optin) return false;
    r.xchunks = mia_ss_num_chunks(L);
    r.x = p.x;
    grid = resident_grid(di, r.smem_bytes, kSmemPerSm, 4, 16, r.n_items);   // at most 16: 128 registers per thread
    return grid > 0;
}

// Row-serial forward for d_state > 1 (scan_fwd_rowsn.cuh): eligibility + argument block.
bool plan_rowsn_fwd(const mia_ss_params &p, const DeviceInfo &di, mia::RowsNArgs &r, int &grid) {
    const int es = esize(p.itype), L = p.seqlen, N = p.dstate;
    const int rpg = p.dim / p.n_groups;
    if ((N != 16 && N != 8) || p.delta_dim != p.dim || (rpg % 32)) return false;
    if (dbg_knob("MIA_NO_ROWS_FWD")) return false;
    if (mia_ss_num_chunks(L) != 1) return false;                // whole rows, one checkpoint
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(out)}) || !aligned(16, {p.u, p.delta, p.out})) return false;
    if (p.z && (!dense_rows(p, {MIA_ROWS(z), MIA_ROWS(out_z)}) || !aligned(16, {p.z, p.out_z}))) return false;
    if ((32 * L * es) % 16) return false;
    fill_rows_common(r, p);
    r.N = N;
    r.warps = p.z ? 2 : mia::kRowsNWarps;
    r.tiles_per_warp = p.z ? 3 : 2;
    const int W = r.warps;
    r.units_per_group = (rpg / 32 + W - 1) / W;
    r.n_units = p.batch * p.n_groups * r.units_per_group;
    r.tile_bytes = round_up(32 * L * es, 128);
    r.off_bc = W * r.tiles_per_warp * r.tile_bytes;
    r.off_bar = r.off_bc + round_up(2 * L * N * es, 128);
    r.smem_bytes = r.off_bar + 128;
    if (r.smem_bytes > di.smem_optin) return false;
    r.x = p.x; r.z = p.z; r.out_z = p.out_z;
    r.A_ds = p.A_d_stride; r.A_ns = p.A_dstate_stride; r.B_ns = p.B_dstate_stride; r.C_ns = p.C_dstate_stride;
    // This family counts the SM's whole 228 KB, not kSmemPerSm: counting 227 KB would change its grid at some sizes.
    grid = resident_grid(di, r.smem_bytes, 228 * 1024, 1, 4, r.n_units);
    return grid > 0;
}

// Row-serial backward (scan_bwd_rows.cuh): eligibility + argument block.  Returns false when the warp-scan kernels must run.
bool plan_rows_bwd(const mia_ss_params &p, const DeviceInfo &di, mia::RowsBwdArgs &r, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    if (!rowwise_n1(p)) return false;
    if (dbg_knob("MIA_NO_ROWS_BWD")) return false;
    const int CH = mia::kRowsChunk;
    const int nch = (L + CH - 1) / CH;
    // long rows: x must hold a checkpoint every 256 tokens, and the per-row pieces of a tile must be 16-byte aligned
    if (nch > 1 && (mia_ss_chunk_len(L) != CH || !p.x || ((L * es) % 16) || ((L * eo) % 16))) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(dout), MIA_ROWS(du), MIA_ROWS(ddelta)}) || !a_per_row(p) ||
        !aligned(16, {p.u, p.delta, p.dout, p.du, p.ddelta})) return false;
    fill_rows_common(r, p);
    r.n_chunks = nch;
    const int span = nch == 1 ? L : CH;                         // tokens of a row resident at a time
    r.t0_pct = dbg_int("MIA_T0_PCT", 52);   // share of a chunk for the half that has no Gs to accumulate
    const int T0 = (span * r.t0_pct / 100) / 4 * 4;
    const int longer = T0 > span - T0 ? T0 : span - T0;
    r.nblk = (longer + mia::kBlk - 1) / mia::kBlk;
    r.Lp = (span + mia::kBlk - 1) / mia::kBlk * mia::kBlk + mia::kBlk;
    r.n_items = p.batch * p.n_groups * (r.rows_per_group / 32);
    r.tile_bytes = round_up(32 * (span * es + (nch > 1 ? 16 : 0)), 128);
    r.tileo_bytes = round_up(32 * (span * eo + (nch > 1 ? 16 : 0)), 128);
    r.off_delta = r.tile_bytes;
    r.off_dout = 2 * r.tile_bytes;
    r.off_bc32 = r.off_dout + r.tileo_bytes;
    r.off_ck = r.off_bc32 + round_up(2 * r.Lp * 4, 128);
    r.off_xch = r.off_ck + 3 * r.nblk * 128;                    // ck of both halves + ckm
    r.off_bar = r.off_xch + 7 * 128;
    r.smem_bytes = r.off_bar + 128;
    r.dout = p.dout; r.du = p.du; r.ddelta = p.ddelta; r.x = p.x;
    // at least 3 resident CTAs to hide the dependent chains; at most 5: 64 threads x 168 registers, 3 warps per scheduler
    grid = resident_grid(di, r.smem_bytes, kSmemPerSm, 3, 5, r.n_items);
    // Long rows: a CTA walks its 32 rows chunk by chunk and each chunk is latency-bound (load -> phase 1 -> exchange ->
    // phase 2 -> store), so this path only wins while every item gets its own resident CTA.
    return grid > 0 && !(nch > 1 && r.n_items > grid);
}

// Column-walk backward (scan_bwd_cw.cuh): eligibility, argument block, tensor maps (u, delta, dout, du, ddelta).
bool plan_cw_bwd(const mia_ss_params &p, const DeviceInfo &di, mia::CwBwdArgs &r, CUtensorMap *tm, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    // Only on the forward's block states (one warp per 32 g rows, phase 2 only).  Short rows always; rows of more than one
    // 256-token chunk only with enough 32-row items to fill the SMs (four per SM): below that a one-warp-per-item walk leaves
    // the SMs short of warps and the warp-scan kernel is used.
    const long long items32 = (long long)p.batch * (p.dim / 32);
    if (!p.hblk || !(L <= mia::kRowsChunk || items32 >= 4LL * di.sms || dbg_knob("MIA_FORCE_CW_BWD"))) return false;
    int g = 0;
    if (!cw_geometry(p, di.sms, g)) return false;
    if (dbg_knob("MIA_NO_CW_BWD")) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(dout), MIA_ROWS(du), MIA_ROWS(ddelta)}) || !a_per_row(p) ||
        !aligned(16, {p.u, p.delta, p.dout, p.du, p.ddelta})) return false;
    const unsigned long long trows = (unsigned long long)p.batch * p.dim / g, tcols = (unsigned long long)g * L;
    if (tcols >= (1ull << 31) || trows >= (1ull << 31)) return false;
    fill_rows_common(r, p);
    r.g = g;
    r.n_items = p.batch * p.n_groups * (r.rows_per_group / (32 * g));
    r.ngrp = (g * L + mia::kCwGrp - 1) / mia::kCwGrp;
    r.nwin = (g * L + mia::kCwWin - 1) / mia::kCwWin;
    const int tile_i = 32 * mia::kCwWin * es, tile_o = 32 * mia::kCwWin * eo;
    r.stage_bytes = 2 * tile_i + tile_o;
    r.ns = dbg_int("MIA_CW_STAGES", 4);                          // 4 stages, at most 4 resident warps per SM: see below
    r.off_bc32 = r.ns * r.stage_bytes;
    r.off_pf = r.off_bc32 + 2 * mia::kCwWin * 4;                // two 512-byte prefetch slots (raw B, raw C, block states of 2 groups)
    r.off_red = r.off_pf + 1024;                                // [32][20] fp32 scratch of the row reductions
    r.off_bar = r.off_red + 32 * 20 * 4;
    r.smem_bytes = r.off_bar + 8 * r.ns + 16;
    if (!aligned(4, {p.B, p.C}) || ((p.B_batch_stride | p.B_group_stride | p.C_batch_stride | p.C_group_stride) * es) % 4) return false;
    r.hblk = p.hblk;
    const void *ptrs[5] = {p.u, p.delta, p.dout, p.du, p.ddelta};
    for (int i = 0; i < 5; ++i) {
        const int e = i == 2 ? eo : es;
        const int trc = mia::tma_make_2d(&tm[i], ptrs[i], trows, tcols, tcols * e, 32, mia::kCwWin, e, mia::kCwWin * e);
        if (trc != 0) { MIA_TRACE("cw bwd: tensor map %d rejected (CUresult %d)", i, trc); return false; }
    }
    // At most 4 resident warps per SM.  The kernel is bound by DRAM, not by issue, and fewer concurrent row streams per SM with
    // a deeper ring move its bytes faster: on an H100 (80GB HBM3, 700 W; tools/bwd_variants.py, bf16, R = 3072, debug-build knobs
    // MIA_CW_STAGES / MIA_CW_MAXPERSM) 4 stages at 4 warps take 0.418 ms at B = 132, L = 196 and 1.340 ms at B = 16, L = 6400,
    // against 0.448 / 1.405 ms for 3 / 2 stages at 8 warps; 3 stages at 4 warps: 0.413 / 1.388 ms; 2 stages: 0.445 / 1.542 ms;
    // 5-8 stages at 4 warps: 0.417 / 1.341 ms; 3 warps: >= 0.496 / 1.729 ms; 4 stages at 5-8 warps (smem allows 7):
    // 0.429-0.461 / 1.346-1.458 ms.  Never more than 8: the kernel's register budget (scan_bwd_cw.cuh).
    const int fill = resident_grid(di, r.smem_bytes, kSmemPerSm, 1, std::min(dbg_int("MIA_CW_MAXPERSM", 4), 8), r.n_items);
    if (!fill) return false;
    const int rounds = (r.n_items + fill - 1) / fill;
    grid = (r.n_items + rounds - 1) / rounds;                    // equal rounds per CTA
    return true;
}

// Deterministic d_state 16 backward (scan_bwd_rowsn.cuh): eligibility + argument block.
bool plan_rowsn_bwd(const mia_ss_params &p, const DeviceInfo &di, mia::RowsNBwdArgs &r, int &grid) {
    const int es = esize(p.itype), eo = esize(p.otype), L = p.seqlen;
    RowsNSplit sp;
    if (!rowsn_bwd_split(p, di.sms, kRowsNCtasPerSm, sp)) return false;
    if (dbg_knob("MIA_NO_ROWS_BWD")) return false;
    if (!dense_rows(p, {MIA_ROWS(u), MIA_ROWS(delta), MIA_ROWS(dout), MIA_ROWS(du), MIA_ROWS(ddelta)}) ||
        !aligned(16, {p.u, p.delta, p.dout})) return false;
    if (p.z && (!dense_rows(p, {MIA_ROWS(z), MIA_ROWS(out_saved), MIA_ROWS(dz)}) || !aligned(16, {p.z, p.out_saved}))) return false;
    fill_rows_common(r, p);
    r.has_z = p.z != nullptr;
    r.n_oct = sp.n_oct; r.oct_per_cta = sp.oct_per_cta; r.oct_per_group = sp.oct_per_group; r.max_parts = sp.max_parts;
    r.nblk = (L + mia::kRnBlk - 1) / mia::kRnBlk;
    r.Lp = r.nblk * mia::kRnBlk;
    r.pitch_s = r.Lp + 4;
    r.pitch_acc = r.Lp + 4;
    // B / C rows [16 states][pitch]: consecutive state rows 16 bytes apart modulo 128, so that the 8 state pairs of a
    // quarter warp read 8 different 16-byte bank windows
    r.pitch_bc = r.Lp;
    while ((r.pitch_bc * es) % 128 != 16) r.pitch_bc += 16 / es;
    int off = 0;
    auto take = [&](int bytes) { int o = off; off += round_up(bytes, 128); return o; };
    r.off_raw_u = take(mia::kRnOct * L * es);
    r.off_raw_d = take(mia::kRnOct * L * es);
    r.off_raw_o = take(mia::kRnOct * L * eo);
    if (p.z) { r.off_raw_z = take(mia::kRnOct * L * es); r.off_raw_os = take(mia::kRnOct * L * eo); }
    r.off_sm = take(4 * r.pitch_s * 4);
    r.off_su = take(4 * r.pitch_s * 4);
    r.off_sy = take(4 * r.pitch_s * 4);
    r.off_b = take(16 * r.pitch_bc * es);
    r.off_c = take(16 * r.pitch_bc * es);
    r.off_acc = take(2 * 16 * r.pitch_acc * 4);
    r.off_ck = take(r.nblk * 32 * 8);
    r.off_ckm = take(r.nblk * 4 * 4);
    r.off_x = take((4 * mia::kRnWarps * 32 + mia::kRnWarps * 4) * 8);
    r.off_bar = take(8);
    r.smem_bytes = off;
    if (r.smem_bytes > di.smem_optin) return false;
    r.dout = p.dout; r.z = p.z; r.out_saved = p.out_saved; r.du = p.du; r.ddelta = p.ddelta; r.dz = p.dz;
    r.A_ds = p.A_d_stride; r.A_ns = p.A_dstate_stride; r.B_ns = p.B_dstate_stride; r.C_ns = p.C_dstate_stride;
    grid = sp.grid;
    return true;
}

template <typename P> using elem_t = std::remove_pointer_t<P>;

// One launch for the input dtype: `f` receives a null pointer of the element type and returns the launch's error.  On success
// counts `n_launches` kernel launches; on failure reports "<what> launch: <error>".
template <typename F>
int launch(int itype, const char *what, int n_launches, F &&f) {
    const cudaError_t e = mia::dispatch_dtype<cudaError_t>(itype, f);
    if (e != cudaSuccess) return mia::fail(mia::kErrScan, MIA_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
    mia::count_launches(n_launches);
    return MIA_OK;
}

// ---------------------------------------------------------------------------------------------
// Finalize: fold the backward's partials in a fixed order (deterministic) and cast to the output dtypes.
struct FinArgs {
    int batch, dim, L, N, G, delta_dim, ratio, tiles, bc_atomic, Lp, has_D, has_bias;
    int oct_per_cta, oct_per_group;          // > 0: partials of scan_bwd_rowsn.cuh, group bg has (c_hi - c_lo + 1) <= tiles of them
    const float *part_dA, *part_dD, *part_dbias, *acc_dB, *acc_dC, *ddelta_full;
    float *dA, *dD, *dbias;
    void *dB, *dC, *ddelta;
    long long dA_ds, dA_ns, dB_bs, dB_gs, dB_ns, dC_bs, dC_gs, dC_ns, dd_bs, dd_ds;
    long long n_bc, n_dA, n_dD, n_db, n_dd;
};

// thread items: dB, dC (sum of the per-segment partials / cast of the atomic accumulator) and the ddelta group fold;
// warp items: dA, dD, dbias (sum over the batch, lanes stride over b, shuffle-reduced in a fixed order).
template <typename T>
__global__ void ss_finalize_kernel(const __grid_constant__ FinArgs f) {
    using raw = typename mia::Cvt<T>::raw;
    const long long n_thread_items = 2 * f.n_bc + f.n_dd;
    const long long t1 = (n_thread_items + 31) / 32 * 32;
    const long long n_warp_items = f.n_dA + f.n_dD + f.n_db;
    const long long total = t1 + 32 * n_warp_items;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        if (idx < t1) {
            long long i = idx;
            if (i >= n_thread_items) continue;
            if (i < 2 * f.n_bc) {
                const bool isC = i >= f.n_bc;
                if (isC) i -= f.n_bc;
                const int l = (int)(i % f.L);
                long long t = i / f.L;
                const int n = (int)(t % f.N); t /= f.N;
                const int g = (int)(t % f.G);
                const int b = (int)(t / f.G);
                const float *acc = isC ? f.acc_dC : f.acc_dB;
                float sum = 0.f;
                if (f.bc_atomic) {
                    sum = acc[((size_t)(b * f.G + g) * f.N + n) * f.Lp + l];
                } else {
                    const float *p0 = acc + (((size_t)(b * f.G + g) * f.tiles) * f.N + n) * f.L + l;
                    const size_t step = (size_t)f.N * f.L;
                    int nt = f.tiles;
                    if (f.oct_per_cta > 0) {             // partial slots actually written for this group (CTAs it straddles)
                        const long long o0 = (long long)(b * f.G + g) * f.oct_per_group;
                        nt = (int)((o0 + f.oct_per_group - 1) / f.oct_per_cta - o0 / f.oct_per_cta) + 1;
                    }
#pragma unroll 4
                    for (int tl = 0; tl < nt; ++tl) sum += p0[tl * step];
                }
                raw *dst = reinterpret_cast<raw *>(isC ? f.dC : f.dB);
                const long long o = isC ? (b * f.dC_bs + g * f.dC_gs + n * f.dC_ns + l) : (b * f.dB_bs + g * f.dB_gs + n * f.dB_ns + l);
                dst[o] = mia::Cvt<T>::from_f(sum);
            } else {   // ddelta fold over the delta group (selective_scan_oflex.cpp:348-350)
                i -= 2 * f.n_bc;
                const int l = (int)(i % f.L);
                long long t = i / f.L;
                const int dg = (int)(t % f.delta_dim);
                const int b = (int)(t / f.delta_dim);
                float sum = 0.f;
                for (int r = 0; r < f.ratio; ++r) sum += f.ddelta_full[((size_t)b * f.dim + dg * f.ratio + r) * f.L + l];
                reinterpret_cast<raw *>(f.ddelta)[b * f.dd_bs + dg * f.dd_ds + l] = mia::Cvt<T>::from_f(sum);
            }
            continue;
        }
        // ---- warp items (idx - t1 is warp aligned, so the whole warp takes this path together)
        long long w = (idx - t1) >> 5;
        const int lane = (int)(idx & 31);
        float sum = 0.f;
        float *dst;
        if (w < f.n_dA) {
            const int n = (int)(w % f.N), d = (int)(w / f.N);
            for (int b = lane; b < f.batch; b += 32) sum += f.part_dA[((size_t)b * f.dim + d) * f.N + n];
            dst = f.dA + d * f.dA_ds + n * f.dA_ns;
        } else if (w < f.n_dA + f.n_dD) {
            w -= f.n_dA;
            for (int b = lane; b < f.batch; b += 32) sum += f.part_dD[(size_t)b * f.dim + w];
            dst = f.dD + w;
        } else {
            w -= f.n_dA + f.n_dD;
            for (int k = lane; k < f.batch * f.ratio; k += 32) {
                const int b = k / f.ratio, r = k - b * f.ratio;
                sum += f.part_dbias[(size_t)b * f.dim + w * f.ratio + r];
            }
            dst = f.dbias + w;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
        if (lane == 0) *dst = sum;
    }
}

}  // namespace

// =================================================================================================
extern "C" {

int mia_abi_version(void) { return MIA_ABI_VERSION; }

int mia_ss_chunk_len(int seqlen) { return lanes_per_row(seqlen) * mia::kTok; }
int mia_ss_num_chunks(int seqlen) {
    const int ch = mia_ss_chunk_len(seqlen);
    return (seqlen + ch - 1) / ch;
}

size_t mia_ss_block_state_floats(const mia_ss_params *pp) {
    if (!pp || validate_sizes(*pp) != MIA_OK) return 0;
    const mia_ss_params &p = *pp;
    if (p.dstate != 1 || ((p.dim / p.n_groups) % 32)) return 0;
    return (size_t)p.batch * p.dim * ((p.seqlen + 15) / 16);
}

int mia_ss_fwd_writes_block_states(const mia_ss_params *pp) {
    if (!pp || !pp->hblk || validate_sizes(*pp) != MIA_OK || !pp->u || !pp->delta || !pp->out) return 0;
    DeviceInfo di;
    if (mia::device_info(mia::kErrScan, di) != MIA_OK) return 0;
    mia::CwFwdArgs rw;
    CUtensorMap tm[3];
    int grid = 0;
    return plan_cw_fwd(*pp, di, rw, tm, grid) ? 1 : 0;          // the column-walk forward is the kernel that fills hblk
}

int mia_selective_scan_fwd(const mia_ss_params *pp, void *cuda_stream) {
    if (!pp) return mia::fail(mia::kErrScan, MIA_EINVAL, "null params");
    const mia_ss_params &p = *pp;
    if (int rc = validate_common(p)) return rc;
    MIA_CHECK(p.out && p.x, "out and x must not be null");
    MIA_CHECK(!p.z || p.out_z, "out_z is required when z is given");
    DeviceInfo di;
    if (int rc = mia::device_info(mia::kErrScan, di)) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const bool of32 = p.otype == MIA_F32 && p.itype != MIA_F32;
    int grid = 0;
    // The first family that takes the problem runs: column-walk, chunk-parallel, resident-row, streaming, d_state 8 / 16
    // row-serial, warp-scan.
    {
        mia::CwFwdArgs r;
        CUtensorMap tm[3];
        if (plan_cw_fwd(p, di, r, tm, grid)) {
            MIA_TRACE("fwd: cw g=%d ns=%d nwin=%d grid=%d smem=%d", r.g, r.ns, r.nwin, grid, r.smem_bytes);
            return launch(p.itype, "selective_scan_fwd (column-walk)", 1,
                          [&](auto *t) { return mia::launch_fwd_cw<elem_t<decltype(t)>>(tm, r, grid, of32, stream); });
        }
    }
    {
        mia::ChunkArgs r;
        if (plan_chunks_fwd(p, di, r, grid))
            return launch(p.itype, "selective_scan_fwd (chunk-parallel)", 3,
                          [&](auto *t) { return mia::launch_fwd_chunks<elem_t<decltype(t)>>(r, grid, of32, stream); });
    }
    {
        mia::RowsArgs r;
        if (plan_rows_fwd(p, di, r, grid))
            return launch(p.itype, "selective_scan_fwd (row-serial)", 1,
                          [&](auto *t) { return mia::launch_fwd_rows<elem_t<decltype(t)>>(r, grid, of32, stream); });
    }
    {
        mia::StreamArgs r;
        if (plan_stream_fwd(p, di, r, grid))
            return launch(p.itype, "selective_scan_fwd (streaming)", 1,
                          [&](auto *t) { return mia::launch_fwd_stream<elem_t<decltype(t)>>(r, grid, of32, stream); });
    }
    {
        mia::RowsNArgs r;
        if (plan_rowsn_fwd(p, di, r, grid))
            return launch(p.itype, "selective_scan_fwd (row-serial, d_state 8 / 16)", 1,
                          [&](auto *t) { return mia::launch_fwd_rowsn<elem_t<decltype(t)>>(r, grid, of32, stream); });
    }
    Plan pl;
    mia::ScanArgs a;
    if (int rc = plan_and_layout(p, di, false, pl, a)) return rc;
    a.out = p.out; a.out_z = p.out_z;
    a.out_bs = p.out_batch_stride; a.out_ds = p.out_d_stride; a.outz_bs = p.out_z_batch_stride; a.outz_ds = p.out_z_d_stride;
    grid = a.n_seg < di.sms ? a.n_seg : di.sms;
    return launch(p.itype, "selective_scan_fwd", 1, [&](auto *t) { return mia::launch_fwd_any<elem_t<decltype(t)>>(a, grid, stream); });
}

}  // extern "C"

namespace {

// det: mia_selective_scan_bwd_deterministic.  It changes the plan and the workspace only for d_state > 1 (d_state 1 is
// deterministic on every path), and there only the warp-scan kernels' dB / dC reduction.
size_t bwd_workspace(const mia_ss_params *pp, bool det) {
    if (!pp) return 0;
    if (validate_sizes(*pp) != MIA_OK) return 0;     // sizes that the backward itself would reject
    det = det && pp->dstate > 1;
    DeviceInfo di;
    if (mia::device_info(mia::kErrScan, di) != MIA_OK) { di.sms = 132; di.smem_optin = 232448; }
    Plan pl;
    mia::ScanArgs a;
    if (plan_and_layout(*pp, di, true, pl, a, det) != MIA_OK) return 0;
    return workspace_layout(*pp, pl, di.sms, det).total;
}

#ifdef MIA_DEBUG
int *det_status_word() {          // raised by a deterministic-backward wait that gave up (scan_bwd.cuh, det_wait)
    static int *w = nullptr;
    if (!w && cudaMalloc(&w, sizeof(int)) != cudaSuccess) w = nullptr;
    return w;
}
#endif

int bwd_impl(const mia_ss_params *pp, void *cuda_stream, bool det) {
    if (!pp) return mia::fail(mia::kErrScan, MIA_EINVAL, "null params");
    const mia_ss_params &p = *pp;
    if (int rc = validate_common(p)) return rc;
    MIA_CHECK(p.dout && p.du && p.ddelta && p.dA && p.dB && p.dC, "dout, du, ddelta, dA, dB, dC must not be null");
    MIA_CHECK(!p.D || p.dD, "dD is required when D is given");
    MIA_CHECK(!p.delta_bias || p.ddelta_bias, "ddelta_bias is required when delta_bias is given");
    MIA_CHECK(!p.z || (p.dz && p.out_saved), "dz and out_saved are required when z is given");
    MIA_CHECK(p.n_chunks == 1 || p.x, "x is required when the sequence spans more than one chunk");
    det = det && p.dstate > 1;
    DeviceInfo di;
    if (int rc = mia::device_info(mia::kErrScan, di)) return rc;
    Plan pl;
    mia::ScanArgs a;
    if (int rc = plan_and_layout(p, di, true, pl, a, det)) return rc;
    a.dout = p.dout; a.out_saved = p.out_saved; a.du = p.du; a.ddelta = p.ddelta; a.dz = p.dz;
    a.dout_bs = p.dout_batch_stride; a.dout_ds = p.dout_d_stride;
    a.osaved_bs = p.out_saved_batch_stride; a.osaved_ds = p.out_saved_d_stride;
    a.du_bs = p.du_batch_stride; a.du_ds = p.du_d_stride; a.dd_bs = p.ddelta_batch_stride; a.dd_ds = p.ddelta_d_stride;
    a.dz_bs = p.dz_batch_stride; a.dz_ds = p.dz_d_stride;
    const WorkspaceLayout w = workspace_layout(p, pl, di.sms, det);
    if (!p.workspace || p.workspace_bytes < w.total)
        return mia::fail(mia::kErrScan, MIA_EWORKSPACE, "workspace too small: need %zu bytes, got %zu", w.total, p.workspace ? p.workspace_bytes : (size_t)0);
    MIA_CHECK(((uintptr_t)p.workspace & 255) == 0, "workspace must be 256-byte aligned");
    char *ws = (char *)p.workspace;
    a.part_dA = (float *)(ws + w.part_dA); a.part_dD = (float *)(ws + w.part_dD); a.part_dbias = (float *)(ws + w.part_dbias);
    a.acc_dB = (float *)(ws + w.acc_dB); a.acc_dC = (float *)(ws + w.acc_dC);
    a.ddelta_full = (float *)(ws + w.ddelta_full);
    a.bc_atomic = w.bc_atomic;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const bool of32 = p.otype == MIA_F32 && p.itype != MIA_F32;
    auto give_partials = [&](auto &r) {
        r.part_dA = a.part_dA; r.part_dD = a.part_dD; r.part_dbias = a.part_dbias; r.acc_dB = a.acc_dB; r.acc_dC = a.acc_dC;
    };
    // The first family that takes the problem runs: d_state 16 row-serial, column-walk, resident-row, (deterministic)
    // warp-scan.  Then the finalize kernel folds the partials.
    mia::RowsNBwdArgs rn;
    mia::CwBwdArgs cwb;
    mia::RowsBwdArgs rb;
    CUtensorMap tmaps[5];
    int rc, grid = 0, bc_parts = pl.split;
    const bool use_rowsn = plan_rowsn_bwd(p, di, rn, grid);
    if (use_rowsn) {
        a.bc_atomic = 0;
        give_partials(rn);
        bc_parts = rn.max_parts;
        rc = launch(p.itype, "selective_scan_bwd", 1, [&](auto *t) { return mia::launch_bwd_rowsn<elem_t<decltype(t)>>(rn, grid, of32, stream); });
    } else if (plan_cw_bwd(p, di, cwb, tmaps, grid)) {
        MIA_TRACE("bwd: cw g=%d ns=%d ngrp=%d grid=%d smem=%d", cwb.g, cwb.ns, cwb.ngrp, grid, cwb.smem_bytes);
        give_partials(cwb);
        bc_parts = cwb.rows_per_group / 32;
        rc = launch(p.itype, "selective_scan_bwd", 1, [&](auto *t) { return mia::launch_bwd_cw<elem_t<decltype(t)>>(tmaps, cwb, grid, of32, stream); });
    } else if (plan_rows_bwd(p, di, rb, grid)) {
        give_partials(rb);
        bc_parts = rb.rows_per_group / 32;
        rc = launch(p.itype, "selective_scan_bwd", 1, [&](auto *t) { return mia::launch_bwd_rows<elem_t<decltype(t)>>(rb, grid, of32, stream); });
    } else {
        if (a.bc_atomic) {
            MIA_CUDA(cudaMemsetAsync(a.acc_dB, 0, w.acc_bytes, stream));
            MIA_CUDA(cudaMemsetAsync(a.acc_dC, 0, w.acc_bytes, stream));
            mia::count_launches(2);
        }
        grid = a.n_seg < di.sms ? a.n_seg : di.sms;
        if (det) {
#ifdef MIA_DEBUG
            a.det_status = det_status_word();
            if (a.det_status) MIA_CUDA(cudaMemsetAsync(a.det_status, 0, sizeof(int), stream));
#endif
            MIA_TRACE("bwd: deterministic warp-scan N=%d LPR=%d split=%d n_seg=%d RT=%d stages=%d smem=%d smem_acc=%d grid=%d", p.dstate,
                      a.LPR, a.split, a.n_seg, a.RT, a.stages, a.smem_bytes, a.det_smem_acc, grid);
            rc = launch(p.itype, "selective_scan_bwd", 1, [&](auto *t) { return mia::launch_bwd_det<elem_t<decltype(t)>>(a, grid, stream); });
        } else {
            rc = launch(p.itype, "selective_scan_bwd", 1, [&](auto *t) { return mia::launch_bwd_any<elem_t<decltype(t)>>(a, grid, stream); });
        }
    }
    if (rc) return rc;

    FinArgs f;
    memset(&f, 0, sizeof(f));
    f.batch = p.batch; f.dim = p.dim; f.L = p.seqlen; f.N = p.dstate; f.G = p.n_groups; f.delta_dim = p.delta_dim;
    f.ratio = p.dim / p.delta_dim; f.tiles = bc_parts; f.bc_atomic = a.bc_atomic; f.Lp = (p.seqlen + 3) & ~3;
    if (use_rowsn) { f.oct_per_cta = rn.oct_per_cta; f.oct_per_group = rn.oct_per_group; }
    f.part_dA = a.part_dA; f.part_dD = a.part_dD; f.part_dbias = a.part_dbias; f.acc_dB = a.acc_dB; f.acc_dC = a.acc_dC;
    f.ddelta_full = a.ddelta_full;
    f.dA = p.dA; f.dD = p.dD; f.dbias = p.ddelta_bias; f.dB = p.dB; f.dC = p.dC; f.ddelta = p.ddelta;
    f.dA_ds = p.dA_d_stride; f.dA_ns = p.dA_dstate_stride;
    f.dB_bs = p.dB_batch_stride; f.dB_gs = p.dB_group_stride; f.dB_ns = p.dB_dstate_stride;
    f.dC_bs = p.dC_batch_stride; f.dC_gs = p.dC_group_stride; f.dC_ns = p.dC_dstate_stride;
    f.dd_bs = p.ddelta_batch_stride; f.dd_ds = p.ddelta_d_stride;
    f.n_bc = (long long)p.batch * p.n_groups * p.dstate * p.seqlen;
    f.n_dA = (long long)p.dim * p.dstate;
    f.n_dD = p.D ? p.dim : 0;
    f.n_db = p.delta_bias ? p.delta_dim : 0;
    f.n_dd = f.ratio > 1 ? (long long)p.batch * p.delta_dim * p.seqlen : 0;
    const long long total = (2 * f.n_bc + f.n_dd + 31) / 32 * 32 + 32 * (f.n_dA + f.n_dD + f.n_db);
    long long blocks = (total + 255) / 256;
    if (blocks > di.sms * 8) blocks = di.sms * 8;
    rc = launch(p.itype, "selective_scan_bwd finalize", 1, [&](auto *t) {
        ss_finalize_kernel<elem_t<decltype(t)>><<<(int)blocks, 256, 0, stream>>>(f);
        return cudaGetLastError();
    });
    if (rc) return rc;
#ifdef MIA_DEBUG
    if (a.det_status) {
        int st = 0;
        MIA_CUDA(cudaMemcpyAsync(&st, a.det_status, sizeof(int), cudaMemcpyDeviceToHost, stream));
        MIA_CUDA(cudaStreamSynchronize(stream));
        if (st) return mia::fail(mia::kErrScan, MIA_ECUDA, "selective_scan_bwd_deterministic: an ordering wait timed out (results are wrong)");
    }
#endif
    return MIA_OK;
}

}  // namespace

extern "C" {

size_t mia_selective_scan_bwd_workspace(const mia_ss_params *pp) { return bwd_workspace(pp, false); }
int mia_selective_scan_bwd(const mia_ss_params *pp, void *cuda_stream) { return bwd_impl(pp, cuda_stream, false); }
size_t mia_selective_scan_bwd_deterministic_workspace(const mia_ss_params *pp) { return bwd_workspace(pp, true); }
int mia_selective_scan_bwd_deterministic(const mia_ss_params *pp, void *cuda_stream) { return bwd_impl(pp, cuda_stream, true); }

}  // extern "C"
