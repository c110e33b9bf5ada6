// Host side of the C ABI, shared by every unit that exports entry points: the thread-local error channels behind the
// five documented *_last_error getters, the dtype dispatch, the launch counter and the cached device attributes.
// Host code only: no kernel header includes it.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/mia_selective_scan.h"

namespace mia {

// One thread-local message per channel (abi_host.cu):
//   kErrScan  mia_last_error            scan, selective_state_update
//   kErrConv  mia_conv_last_error       causal conv1d, the *_ex entry points, causal_conv1d_update
//   kErrCs    mia_cs_last_error         cross scan / merge, silu_gate
//   kErrDw    mia_dwconv2d_last_error   depth-wise conv2d
//   kErrGemm  mia_gemm_last_error       GEMM
enum ErrChannel { kErrScan, kErrConv, kErrCs, kErrDw, kErrGemm, kErrChannels };

// Writes the formatted message into the channel and returns `code`.
int fail(ErrChannel ch, int code, const char *fmt, ...) __attribute__((format(printf, 3, 4)));

// MIA_OK for cudaSuccess; otherwise writes "<what>: <cudaGetErrorString(e)>" into the channel and returns MIA_ECUDA.
int cuda_fail(ErrChannel ch, const char *what, cudaError_t e);

// The check after a launch: cuda_fail of cudaGetLastError().
inline int launched(ErrChannel ch, const char *what) { return cuda_fail(ch, what, cudaGetLastError()); }

// Adds to the count mia_launch_count() reports.
void count_launches(int n);

struct DeviceInfo { int sms = 0; int smem_optin = 0; };
// SM count and opt-in shared memory per block of the current device, cached per thread for the last device queried.
// A failed query is reported through the channel as MIA_ECUDA.
int device_info(ErrChannel ch, DeviceInfo &di);

// Multiply-high reciprocal of d: floor(i / d) == __umulhi(i, div_magic(d)) for 0 <= i with i * d < 2^32 (0: divisor 1).
inline uint32_t div_magic(int d) { return d == 1 ? 0u : (uint32_t)((0x100000000ULL + (uint64_t)d - 1) / (uint64_t)d); }

// Calls f with a null pointer of the element type of a MIA_F32 / MIA_F16 / MIA_BF16 code and returns its R; any other
// code is taken as bf16, so callers validate the code first.  R is stated, not deduced: deducing it would instantiate
// f's kernels at the call instead of at the end of the unit, which reorders the functions in the cubin.
template <typename R = void, typename F>
R dispatch_dtype(int code, F &&f) {
    switch (code) {
        case MIA_F32: return f((float *)nullptr);
        case MIA_F16: return f((__half *)nullptr);
        default: return f((__nv_bfloat16 *)nullptr);
    }
}

}  // namespace mia
