"""CPU-only checks of the GELU MLP GEMM entry points' C ABI (mia_gemm_gelu_fwd / _bwd): every bad argument is refused before
any CUDA call, on the GEMM channel, so no device is needed to see it."""
import ctypes

import pytest

from medical_image_analysis_b200 import _lib

M, H, K, N = 591, 202, 64, 64
HP = 208                                                             # H rounded up to 8


@pytest.fixture(scope="module")
def p():
    _lib.lib()
    buf = ctypes.create_string_buffer(256)
    addr = ctypes.cast(buf, ctypes.c_void_p).value
    return buf, (addr + 15) // 16 * 16                              # a 16-byte aligned host address: never dereferenced


def _fwd(ptr, null=None, **kw):
    a = dict(x=ptr, w1=ptr, b1=None, h=ptr, pre=ptr, M=M, H=H, K=K, ldx=K, ldw1=K, ldh=HP, ldpre=HP, dtype=_lib.MIA_BF16)
    a.update(kw)
    if null:
        a[null] = None
    return tuple(a.values())


def _bwd(ptr, null=None, **kw):
    a = dict(dy=ptr, w2=ptr, pre=ptr, dpre=ptr, h=ptr, M=M, H=H, N_out=N, lddy=N, ldw2=HP, ldpre=HP, lddpre=HP, ldh=HP, dtype=_lib.MIA_BF16)
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
    for name in ("mia_gemm_gelu_fwd", "mia_gemm_gelu_bwd"):
        assert hasattr(L, name)
        assert _lib.ABI[name][2] == "mia_gemm_last_error"


@pytest.mark.parametrize("null", ["x", "w1", "h"])
def test_fwd_null_pointers(p, null):
    _refused("mia_gemm_gelu_fwd", _fwd(p[1], null), "null pointer")


@pytest.mark.parametrize("null", ["dy", "w2", "pre", "dpre"])
def test_bwd_null_pointers(p, null):
    _refused("mia_gemm_gelu_bwd", _bwd(p[1], null), "null pointer")


@pytest.mark.parametrize("dtype", [_lib.MIA_F32, 7, -1])
def test_bad_dtype(p, dtype):
    _refused("mia_gemm_gelu_fwd", _fwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")
    _refused("mia_gemm_gelu_bwd", _bwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")


@pytest.mark.parametrize("size", [dict(M=0), dict(H=0), dict(K=-8)])
def test_fwd_empty_sizes(p, size):
    _refused("mia_gemm_gelu_fwd", _fwd(p[1], **size), "empty or negative size")


@pytest.mark.parametrize("size", [dict(M=-1), dict(H=0), dict(N_out=0)])
def test_bwd_empty_sizes(p, size):
    _refused("mia_gemm_gelu_bwd", _bwd(p[1], **size), "empty or negative size")


@pytest.mark.parametrize("pitch", [dict(ldx=K + 4), dict(ldw1=K + 2), dict(ldh=HP + 4), dict(ldh=H - 2), dict(ldpre=HP - 8),
                                   dict(ldpre=HP + 1), dict(ldx=K - 8)])
def test_fwd_pitches(p, pitch):
    _refused("mia_gemm_gelu_fwd", _fwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("pitch", [dict(lddy=N + 4), dict(ldw2=HP + 2), dict(ldw2=H - 2), dict(ldpre=HP - 8), dict(lddpre=H),
                                   dict(lddpre=HP + 4), dict(ldh=HP + 1), dict(lddy=N - 8)])
def test_bwd_pitches(p, pitch):
    _refused("mia_gemm_gelu_bwd", _bwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


def test_fwd_without_pre_skips_its_pitch_and_bwd_without_h_skips_its_pitch(p):
    """pre (forward) and h (backward) are optional: NULL lifts their pitch rules, so the call gets past them to the
    alignment rule."""
    _refused("mia_gemm_gelu_fwd", _fwd(p[1] + 2, null="pre", ldpre=3), "16-byte aligned")
    _refused("mia_gemm_gelu_bwd", _bwd(p[1] + 2, null="h", ldh=3), "16-byte aligned")


@pytest.mark.parametrize("which", ["x", "w1", "h", "pre"])
def test_fwd_alignment(p, which):
    _refused("mia_gemm_gelu_fwd", _fwd(p[1], **{which: p[1] + 8}), "16-byte aligned")


@pytest.mark.parametrize("which", ["dy", "w2", "pre", "dpre", "h"])
def test_bwd_alignment(p, which):
    _refused("mia_gemm_gelu_bwd", _bwd(p[1], **{which: p[1] + 2}), "16-byte aligned")


def test_op_refuses_cpu_bad_shapes_and_levels():
    import torch
    from medical_image_analysis_b200.gemm import gelu_mlp_fn
    w1, w2 = torch.zeros(32, 8), torch.zeros(8, 32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        gelu_mlp_fn(torch.zeros(3, 8), w1, None, w2, None)
    with pytest.raises(ValueError, match="checkpoint_lvl"):
        gelu_mlp_fn(torch.zeros(3, 8), w1, None, w2, None, checkpoint_lvl=2)


def test_cpu_modules_take_the_composition():
    import torch
    from medical_image_analysis_b200 import gemm, mae, vmamba
    torch.manual_seed(0)
    x = torch.randn(2, 5, 16, requires_grad=True)
    for m in (vmamba.Mlp(16, 64), mae.Mlp(16, 64)):
        assert not gemm.gelu_mlp_eligible(m, x, True)
        assert torch.equal(m(x), m._forward_composed(x))
