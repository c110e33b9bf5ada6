"""``mia_silu_gate`` (csrc/cross_scan.cu), called through the C ABI: out_z = out * silu(z), the gate that
selective_scan_cuda.bwd(..., recompute_out_z=True) recomputes from the saved pre-gate output.  Against out * silu(z) in
float64 on the same rounded inputs, for every (z, out) dtype pair the launcher accepts (out in z's dtype, or float32 for
16-bit z), at 1 element, a partial block and more elements than one sweep of its grid (capped at 132 x 16 blocks of 256
threads) covers.  A 16-bit out_z by ``cmp_stored``, a float32 one by ``cmp_f32`` (tests/parity.py).  The kernel instance
of each dtype pair is recorded by torch.profiler in a child process (tests/kernel_trace.py)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests.kernel_trace import in_child, names_of, targs
from tests.parity import cmp_f32, cmp_stored

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
T_NAME = {F32: "float", F16: "__half", BF16: "__nv_bfloat16"}
GRID_THREADS = 132 * 16 * 256
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]


def _gate(out, z, out_z):
    from medical_image_analysis_b200 import _lib
    dt = {F32: _lib.MIA_F32, F16: _lib.MIA_F16, BF16: _lib.MIA_BF16}
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream) if out.is_cuda else None
    return _lib.lib().mia_silu_gate(out.data_ptr(), z.data_ptr(), out_z.data_ptr(), out.numel(), dt[z.dtype], dt[out.dtype], stream)


def kernel_paths():
    """{(z dtype, out dtype): kernels one call launches} under the profiler."""
    out = {}
    for z_dtype, out_dtype in PAIRS:
        o, z = torch.randn(4096, device="cuda").to(out_dtype), torch.randn(4096, device="cuda").to(z_dtype)
        out[f"{z_dtype}|{out_dtype}"] = names_of(lambda: _gate(o, z, torch.empty_like(o)), r"\bsilu_gate_kernel<")
    return out


@pytest.fixture(scope="module")
def paths():
    return in_child("tests.test_silu_gate_gpu:kernel_paths")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 1023, 700_000])
@pytest.mark.parametrize("z_dtype,out_dtype", PAIRS, ids=["f32-f32", "bf16-bf16", "f16-f16", "bf16-f32", "f16-f32"])
def test_silu_gate_parity(paths, z_dtype, out_dtype, n):
    assert n < 1024 or n > GRID_THREADS
    g = torch.Generator().manual_seed(n)
    z = (torch.randn(n, generator=g) * 4).to(z_dtype)          # SiLU from saturated to linear
    z[:: 97] = 0
    out = torch.randn(n, generator=g).to(out_dtype)
    zg, og = z.cuda(), out.cuda()
    out_z = torch.full_like(og, float("nan"))
    assert _gate(og, zg, out_z) == 0
    k = paths[f"{z_dtype}|{out_dtype}"]
    assert len(k) == 1 and targs(k[0], "silu_gate_kernel<") == [T_NAME[z_dtype], T_NAME[out_dtype]], k
    ref = out.double() * F.silu(z.double())
    if out_dtype == F32:
        cmp_f32(out_z, ref, f"silu_gate {z_dtype}->{out_dtype} n={n}")
    else:
        cmp_stored(out_z, ref, out_dtype, f"silu_gate {z_dtype}->{out_dtype} n={n}")


@pytest.mark.parametrize("z_dtype,out_dtype", [(F32, BF16), (F32, F16), (F16, BF16), (BF16, F16)])
def test_silu_gate_rejects_a_mismatched_out_dtype(z_dtype, out_dtype):
    """out must be in z's dtype or float32; anything else is refused before any CUDA call (so this needs no GPU)."""
    from medical_image_analysis_b200 import _lib
    out, z = torch.zeros(8, dtype=out_dtype), torch.zeros(8, dtype=z_dtype)
    assert _gate(out, z, torch.empty_like(out)) == -1
    assert b"out dtype must be z's dtype or float32" in _lib.lib().mia_cs_last_error()
