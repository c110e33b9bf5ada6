"""CPU-only checks of the SwiGLU GEMM entry points' C ABI (mia_gemm_swiglu_fwd / _bwd): every bad argument is refused before
any CUDA call, on the GEMM channel, so no device is needed to see it."""
import ctypes

import pytest

from medical_image_analysis_b200 import _lib

M, H, K, N = 394, 176, 64, 64
HP = 192                                                             # H rounded up to 64


@pytest.fixture(scope="module")
def p():
    _lib.lib()
    buf = ctypes.create_string_buffer(256)
    addr = ctypes.cast(buf, ctypes.c_void_p).value
    return buf, (addr + 15) // 16 * 16                              # a 16-byte aligned host address: never dereferenced


def _fwd(ptr, null=None, **kw):
    a = dict(x=ptr, w1=ptr, w2=ptr, b1=None, b2=None, h=ptr, ab=ptr, M=M, H=H, K=K, ldx=K, ldw1=K, ldw2=K, ldh=HP, ldab=2 * HP, dtype=_lib.MIA_BF16)
    a.update(kw)
    if null:
        a[null] = None
    return tuple(a.values())


def _bwd(ptr, null=None, **kw):
    a = dict(dy=ptr, w3=ptr, ab=ptr, dab=ptr, h=ptr, M=M, H=H, N_out=N, lddy=N, ldw3=HP, ldab=2 * HP, lddab=2 * HP, ldh=HP, dtype=_lib.MIA_BF16)
    a.update(kw)
    if null:
        a[null] = None
    return tuple(a.values())


def _refused(name, args, match):
    with pytest.raises(RuntimeError, match=match) as e:
        _lib.call(name, name, None, *args)
    assert "(code -1)" in str(e.value)
    assert _lib.lib().mia_gemm_last_error().decode() in str(e.value)


def test_symbols_exported():
    L = _lib.lib()
    for name in ("mia_gemm_swiglu_fwd", "mia_gemm_swiglu_bwd"):
        assert hasattr(L, name)
        assert _lib.ABI[name][2] == "mia_gemm_last_error"


@pytest.mark.parametrize("null", ["x", "w1", "w2", "h"])
def test_fwd_null_pointers(p, null):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], null), "null pointer")


@pytest.mark.parametrize("null", ["dy", "w3", "ab", "dab"])
def test_bwd_null_pointers(p, null):
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], null), "null pointer")


@pytest.mark.parametrize("dtype", [_lib.MIA_F32, 7, -1])
def test_bad_dtype(p, dtype):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")


@pytest.mark.parametrize("size", [dict(M=0), dict(H=0), dict(K=-8)])
def test_fwd_empty_sizes(p, size):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], **size), "empty or negative size")


@pytest.mark.parametrize("size", [dict(M=0), dict(H=-1), dict(N_out=0)])
def test_bwd_empty_sizes(p, size):
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], **size), "empty or negative size")


@pytest.mark.parametrize("pitch", [dict(ldx=K + 4), dict(ldw1=K + 2), dict(ldw2=K + 1), dict(ldh=HP + 4), dict(ldh=H - 8), dict(ldx=K - 8)])
def test_fwd_pitches(p, pitch):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("pitch", [dict(lddy=N + 4), dict(ldw3=HP + 2), dict(ldh=HP + 1), dict(ldw3=H - 8)])
def test_bwd_pitches(p, pitch):
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("ldab", [2 * HP - 8, 2 * H, 2 * HP + 4])
def test_ab_pitch(p, ldab):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], ldab=ldab), f"at least 2 Hp = {2 * HP}")
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], ldab=ldab), f"at least 2 Hp = {2 * HP}")
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], lddab=ldab), f"at least 2 Hp = {2 * HP}")


def test_fwd_without_ab_skips_its_pitch_and_bwd_without_h_skips_its_pitch(p):
    """ab (forward) and h (backward) are optional: NULL lifts their pitch rules, so the call gets past them to the
    alignment rule."""
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1] + 2, null="ab", ldab=0), "16-byte aligned")
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1] + 2, null="h", ldh=3), "16-byte aligned")


def test_alignment(p):
    _refused("mia_gemm_swiglu_fwd", _fwd(p[1], ab=p[1] + 8), "16-byte aligned")
    _refused("mia_gemm_swiglu_bwd", _bwd(p[1], dab=p[1] + 2), "16-byte aligned")


def test_op_refuses_cpu_and_fp32():
    import torch
    from medical_image_analysis_b200.arm import swiglu_fn
    w1, w3 = torch.zeros(16, 8), torch.zeros(8, 16)
    with pytest.raises(RuntimeError, match="no CPU path"):
        swiglu_fn(torch.zeros(3, 8), w1, None, w1, None, w3, None)
    with pytest.raises(ValueError, match="checkpoint_lvl"):
        swiglu_fn(torch.zeros(3, 8), w1, None, w1, None, w3, None, checkpoint_lvl=2)


def test_cpu_module_takes_the_composition():
    import torch
    from medical_image_analysis_b200.arm import SwiGLU
    torch.manual_seed(0)
    m = SwiGLU(8, 16)
    x = torch.randn(2, 5, 8)
    assert not m._fused_ok(x)
    assert torch.equal(m(x), m._forward_composed(x))
