// Developer probe (GPU): where the column-walk scan kernels' bandwidth goes.  One JSON line per case.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o build/cw_probe tools/cw_probe.cu    (no -lcuda: the tensor
//   maps are encoded through the runtime's driver entry point, as in the library)
//   ./build/cw_probe [--iters N]
//
// 1. Ceilings: plain coalesced 16-byte-per-thread streaming kernels over the headline sizes -- read-only, 2 reads : 1 write (the
//    forward's mix), 3 reads : 2 writes (the backward's mix).
// 2. The column-walk data movement with the arithmetic removed: one-warp CTAs, [32 rows x W columns] 2-D TMA boxes through a ring
//    of `ns` stages, refilled behind cp.async.bulk.wait_group.read exactly as scan_fwd_cw.cuh / scan_bwd_cw.cuh do (two stages:
//    the refill is issued before the step's stores, as the kernels' half-step-early refill), grid sized by the planner's
//    equal-rounds rule.  The forward skeleton moves 2 box loads and 1 box store per window, the backward 3 loads and 2 stores.
//    Geometries: L = 6400, g = 1 (49 152 rows of 12 800 B) and L = 196, g = 4 (405 504 rows walked as 101 376 tensor-map rows
//    of 1568 B), bf16.  Variants: box rows of 64 / 128 / 256 bytes, stage counts, and L2 promotion 128 / 256 B / none.
// The first line names the card and its power limit (nvidia-smi --query-gpu, read-only).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../medical_image_analysis_b200/csrc/scan_bwd_cw.cuh"
#include "../medical_image_analysis_b200/csrc/tma_host.h"

#define CK(x)                                                                                     \
    do {                                                                                          \
        cudaError_t e_ = (x);                                                                     \
        if (e_ != cudaSuccess) {                                                                  \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));    \
            exit(1);                                                                              \
        }                                                                                         \
    } while (0)

// ---------------------------------------------------------------------------------------------------------------- ceilings
template <int kR, int kW>
__global__ void __launch_bounds__(512) stream_kernel(const int4 *__restrict__ in, int4 *__restrict__ out, size_t n16, size_t plane) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
        int4 v[kR];
#pragma unroll
        for (int r = 0; r < kR; ++r) v[r] = __ldcs(in + r * plane + i);
        int x = 0, y = 0, z = 0, w = 0;
#pragma unroll
        for (int r = 0; r < kR; ++r) { x ^= v[r].x; y ^= v[r].y; z ^= v[r].z; w ^= v[r].w; }
        if constexpr (kW == 0) {
            if ((x & y & z & w) == 0x7f3a9c1d) out[0] = make_int4(x, y, z, w);   // never true for the zero-filled input
        } else {
#pragma unroll
            for (int o = 0; o < kW; ++o) __stcs(out + o * plane + i, make_int4(x + o, y, z, w));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- skeleton
struct SkelArgs {
    int n_items, nwin, ns, stage_bytes, box_bytes, box_cols;
};

// kLoads boxes in (u, delta[, dout]), kStores boxes out (y / du[, ddelta]) per window; the window order is the forward's
// (ascending) -- the backward's descending walk touches the same lines in the same rounds.
template <int kLoads, int kStores>
__global__ void __launch_bounds__(32, 16) skel_kernel(const __grid_constant__ CUtensorMap tm_in0, const __grid_constant__ CUtensorMap tm_in1,
                                                       const __grid_constant__ CUtensorMap tm_in2, const __grid_constant__ CUtensorMap tm_out0,
                                                       const __grid_constant__ CUtensorMap tm_out1, const SkelArgs a) {
    extern __shared__ __align__(1024) char smem[];
    const int lane = threadIdx.x, ns = a.ns, nwin = a.nwin, W = a.box_cols;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + ns * a.stage_bytes);
    if (lane == 0) {
        for (int s = 0; s < ns; ++s) mia::mbar_init(full + s, 1);
        mia::fence_mbar_init();
    }
    __syncwarp();
    int ld_item = blockIdx.x, ld_w = 0, ld_stage = 0;
    auto issue_load = [&]() {
        if (ld_item < a.n_items) {
            char *st = smem + ld_stage * a.stage_bytes;
            mia::mbar_arrive_expect_tx(full + ld_stage, (uint32_t)(kLoads * a.box_bytes));
            mia::tma_box_g2s(st, &tm_in0, ld_w * W, ld_item * 32, full + ld_stage);
            mia::tma_box_g2s(st + a.box_bytes, &tm_in1, ld_w * W, ld_item * 32, full + ld_stage);
            if (kLoads > 2) mia::tma_box_g2s(st + 2 * a.box_bytes, &tm_in2, ld_w * W, ld_item * 32, full + ld_stage);
            if (++ld_w == nwin) { ld_w = 0; ld_item += gridDim.x; }
        }
        ld_stage = ld_stage + 1 == ns ? 0 : ld_stage + 1;
    };
    if (lane == 0)
        for (int s = 0; s < ns - 1; ++s) issue_load();
    uint32_t phbits = 0;
    int stage = 0;
    for (int item = blockIdx.x; item < a.n_items; item += gridDim.x) {
        for (int w = 0; w < nwin; ++w) {
            mia::mbar_wait(full + stage, (phbits >> stage) & 1u);
            phbits ^= 1u << stage;
            char *st = smem + stage * a.stage_bytes;
            mia::fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                if (ns == 2) {                    // the stage the next window needs: refill before this window's stores
                    mia::bulk_wait_read<0>();
                    issue_load();
                }
                mia::tma_box_s2g(&tm_out0, st, w * W, item * 32);
                if (kStores > 1) mia::tma_box_s2g(&tm_out1, st + a.box_bytes, w * W, item * 32);
                mia::bulk_commit();
                if (ns > 2) {
                    mia::bulk_wait_read<1>();
                    issue_load();
                }
            }
            stage = stage + 1 == ns ? 0 : stage + 1;
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

static int encode(CUtensorMap *tm, void *ptr, unsigned long long rows, unsigned long long cols, unsigned box_cols, int l2) {
    mia::EncodeTiledFn fn = mia::tma_encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 2};
    cuuint32_t box[2] = {box_cols, 32};
    cuuint32_t estr[2] = {1, 1};
    const unsigned rb = box_cols * 2;
    const CUtensorMapSwizzle sw = rb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : rb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE;
    return (int)fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   l2 == 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : l2 == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

template <typename F>
static float time_ms(F &&launch, int iters) {
    for (int i = 0; i < 3; ++i) launch();
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    std::vector<float> t(iters);
    for (int i = 0; i < iters; ++i) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&t[i], e0, e1));
    }
    CK(cudaGetLastError());
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    std::sort(t.begin(), t.end());
    return t[iters / 2];
}

int main(int argc, char **argv) {
    int iters = 20;
    for (int i = 1; i < argc; ++i)
        if (!strcmp(argv[i], "--iters") && i + 1 < argc) iters = atoi(argv[++i]);
    {
        std::string info;
        if (FILE *f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem --format=csv,noheader -i 0", "r")) {
            char buf[256];
            while (fgets(buf, sizeof buf, f)) info += buf;
            pclose(f);
        }
        while (!info.empty() && (info.back() == '\n' || info.back() == '\r')) info.pop_back();
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, 0));
        printf("{\"card\": \"%s\", \"nvidia_smi\": \"%s\", \"sms\": %d}\n", prop.name, info.c_str(), prop.multiProcessorCount);
    }
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));

    struct Geo { const char *name; unsigned long long rows, cols; };
    const Geo geos[2] = {{"L6400_g1", 49152, 6400}, {"L196_g4", 101376, 784}};
    const size_t max_plane = 49152ull * 6400 * 2;               // bytes of one bf16 tensor at either geometry (L = 6400 is larger)
    char *buf = nullptr;
    CK(cudaMalloc(&buf, 5 * max_plane));
    CK(cudaMemset(buf, 0, 5 * max_plane));

    // ---- ceilings
    for (const Geo &g : geos) {
        const size_t plane = g.rows * g.cols * 2, n16 = plane / 16;
        const int4 *in = reinterpret_cast<const int4 *>(buf);
        int4 *out = reinterpret_cast<int4 *>(buf + 3 * max_plane);
        const size_t pl16 = max_plane / 16;
        const int grid = sms * 4;
        struct { const char *mix; int r, w; } mixes[3] = {{"read_only_3r", 3, 0}, {"fwd_2r1w", 2, 1}, {"bwd_3r2w", 3, 2}};
        for (auto &m : mixes) {
            float ms;
            if (m.w == 0) ms = time_ms([&] { stream_kernel<3, 0><<<grid, 512>>>(in, out, n16, pl16); }, iters);
            else if (m.r == 2) ms = time_ms([&] { stream_kernel<2, 1><<<grid, 512>>>(in, out, n16, pl16); }, iters);
            else ms = time_ms([&] { stream_kernel<3, 2><<<grid, 512>>>(in, out, n16, pl16); }, iters);
            const double bytes = (double)plane * (m.r + m.w);
            printf("{\"probe\": \"ceiling\", \"geometry\": \"%s\", \"mix\": \"%s\", \"bytes\": %.0f, \"ms\": %.4f, \"TBps\": %.3f}\n", g.name, m.mix,
                   bytes, ms, bytes / ms * 1e-9);
        }
    }

    // ---- skeletons
    struct Var { int dir; int box_bytes; int l2; int ns; int cap; };   // dir 0: forward, 1: backward
    const std::vector<Var> vars = {
        // forward: 64-byte boxes as today (4 stages; 3 and 5 stages), promotion 128 / 256 / none; 128-byte boxes with 2 / 3
        // stages; 256-byte boxes
        {0, 64, 128, 4, 16}, {0, 64, 128, 3, 16}, {0, 64, 128, 5, 16}, {0, 64, 256, 4, 16}, {0, 64, 0, 4, 16}, {0, 128, 128, 2, 16}, {0, 128, 128, 3, 16}, {0, 128, 256, 2, 16}, {0, 256, 128, 2, 16},
        // backward: 64-byte boxes as today (2 and 3 stages; 4 stages), promotion 256 / none; 128-byte boxes with 2 / 3 stages;
        // 256-byte boxes
        {1, 64, 128, 2, 8}, {1, 64, 128, 3, 8}, {1, 64, 128, 4, 8}, {1, 64, 256, 2, 8}, {1, 64, 256, 3, 8}, {1, 64, 0, 3, 8}, {1, 128, 128, 2, 8}, {1, 128, 128, 3, 8},
        {1, 128, 256, 2, 8}, {1, 256, 128, 2, 8}};
    for (const Geo &g : geos) {
        for (const Var &v : vars) {
            const int nload = v.dir ? 3 : 2, nstore = v.dir ? 2 : 1;
            const int box_cols = v.box_bytes / 2;
            CUtensorMap tm[5];
            bool ok = true;
            for (int i = 0; i < 5; ++i) ok = ok && encode(&tm[i], buf + (size_t)i * max_plane, g.rows, g.cols, box_cols, v.l2) == 0;
            if (!ok) { printf("{\"probe\": \"skeleton\", \"error\": \"tensor map rejected\"}\n"); continue; }
            SkelArgs a;
            a.n_items = (int)(g.rows / 32);
            a.box_cols = box_cols;
            a.box_bytes = 32 * v.box_bytes;
            a.nwin = (int)((g.cols + box_cols - 1) / box_cols);
            a.ns = v.ns;
            a.stage_bytes = nload * a.box_bytes;
            // the real kernels' scratch next to the ring: B / C as fp32, prefetch slots and the reduction scratch (backward)
            const int scratch = v.dir ? 2 * box_cols * 4 + 2 * (2 * box_cols * 2 + (box_cols / 16) * 128) + 32 * 20 * 4 : 2 * box_cols * 4;
            const int smem = v.ns * a.stage_bytes + scratch + 8 * v.ns + 16;
            int per_sm = (227 * 1024) / (smem + 1024);
            per_sm = std::min(per_sm, v.cap);
            const long long slots = (long long)sms * per_sm, rounds = (a.n_items + slots - 1) / slots;
            const int grid = (int)((a.n_items + rounds - 1) / rounds);
            void (*k)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const SkelArgs) =
                v.dir ? &skel_kernel<3, 2> : &skel_kernel<2, 1>;
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            const float ms = time_ms([&] { k<<<grid, 32, smem>>>(tm[0], tm[1], tm[2], tm[3], tm[4], a); }, iters);
            const double bytes = (double)g.rows * g.cols * 2 * (nload + nstore);
            printf("{\"probe\": \"skeleton\", \"geometry\": \"%s\", \"dir\": \"%s\", \"box_row_bytes\": %d, \"l2_promotion\": %d, \"stages\": %d, "
                   "\"smem\": %d, \"warps_per_sm\": %d, \"grid\": %d, \"rounds\": %lld, \"bytes\": %.0f, \"ms\": %.4f, \"TBps\": %.3f}\n",
                   g.name, v.dir ? "bwd" : "fwd", v.box_bytes, v.l2, v.ns, smem, per_sm, grid, rounds, bytes, ms, bytes / ms * 1e-9);
            fflush(stdout);
        }
    }
    CK(cudaFree(buf));
    return 0;
}
