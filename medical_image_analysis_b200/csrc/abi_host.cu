// The error channels, launch counter and device attributes declared in abi_host.h, and the C ABI's getters for them.
#include "abi_host.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/mia_gemm.h"

namespace {

thread_local char g_err[mia::kErrChannels][512];
std::atomic<uint64_t> g_launches{0};

}  // namespace

namespace mia {

int fail(ErrChannel ch, int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    char *msg = g_err[ch];
    vsnprintf(msg, sizeof(g_err[ch]), fmt, ap);
    va_end(ap);
    return code;
}

int cuda_fail(ErrChannel ch, const char *what, cudaError_t e) {
    if (e == cudaSuccess) return MIA_OK;
    return fail(ch, MIA_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

void count_launches(int n) { g_launches.fetch_add(n); }

#define MIA_QUERY(expr) \
    do { if (int rc__ = cuda_fail(ch, #expr, (expr))) return rc__; } while (0)

int device_info(ErrChannel ch, DeviceInfo &di) {
    static thread_local int cached_dev = -1;
    static thread_local DeviceInfo cached;
    int dev = 0;
    MIA_QUERY(cudaGetDevice(&dev));
    if (dev != cached_dev) {
        // Binds the device's primary context to this thread.  cudaGetDevice alone does not, and the driver calls that follow
        // (cuTensorMapEncodeTiled) fail with CUDA_ERROR_INVALID_CONTEXT on a thread whose first CUDA work is one of ours,
        // e.g. autograd's device thread when a backward starts with one of our ops.
        MIA_QUERY(cudaSetDevice(dev));
        MIA_QUERY(cudaDeviceGetAttribute(&cached.sms, cudaDevAttrMultiProcessorCount, dev));
        MIA_QUERY(cudaDeviceGetAttribute(&cached.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        cached_dev = dev;
    }
    di = cached;
    return MIA_OK;
}

#undef MIA_QUERY

}  // namespace mia

extern "C" {

const char *mia_last_error(void) { return g_err[mia::kErrScan]; }
const char *mia_conv_last_error(void) { return g_err[mia::kErrConv]; }
const char *mia_cs_last_error(void) { return g_err[mia::kErrCs]; }
const char *mia_dwconv2d_last_error(void) { return g_err[mia::kErrDw]; }
const char *mia_gemm_last_error(void) { return g_err[mia::kErrGemm]; }
uint64_t mia_launch_count(void) { return g_launches.load(); }

}  // extern "C"
