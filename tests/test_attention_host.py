"""CPU-only checks of the attention entry points' C ABI (mia_attn_fwd / _bwd): every bad argument is refused before any CUDA
call, on the GEMM channel, so no device is needed to see it; and the in-tree object runs on wgmma and TMA."""
import ctypes
import os
import shutil
import subprocess

import pytest

from medical_image_analysis_b200 import _lib

B, N, H, DH = 2, 61, 4, 32
C = H * DH


@pytest.fixture(scope="module")
def p():
    _lib.lib()
    buf = ctypes.create_string_buffer(256)
    addr = ctypes.cast(buf, ctypes.c_void_p).value
    return buf, (addr + 15) // 16 * 16                              # a 16-byte aligned host address: never dereferenced


def _fwd(ptr, null=None, **kw):
    a = dict(qkv=ptr, o=ptr, lse=ptr, B=B, N=N, H=H, dh=DH, ld_qkv=3 * C, ld_o=C, dtype=_lib.MIA_BF16)
    a.update(kw)
    if null:
        a[null] = None
    return tuple(a.values())


def _bwd(ptr, null=None, **kw):
    a = dict(qkv=ptr, o=ptr, dout=ptr, lse=ptr, delta=ptr, dqkv=ptr, B=B, N=N, H=H, dh=DH, ld_qkv=3 * C, ld_o=C, ld_do=C, ld_dqkv=3 * C,
             dtype=_lib.MIA_BF16)
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
    for name in ("mia_attn_fwd", "mia_attn_bwd"):
        assert hasattr(L, name)
        assert _lib.ABI[name][2] == "mia_gemm_last_error"


@pytest.mark.parametrize("null", ["qkv", "o"])
def test_fwd_null_pointers(p, null):
    _refused("mia_attn_fwd", _fwd(p[1], null), "null pointer")


@pytest.mark.parametrize("null", ["qkv", "o", "dout", "lse", "delta", "dqkv"])
def test_bwd_null_pointers(p, null):
    _refused("mia_attn_bwd", _bwd(p[1], null), "null pointer")


@pytest.mark.parametrize("dh", [16, 48, 96, 128, 0, -32])
def test_head_dims_outside_the_set(p, dh):
    _refused("mia_attn_fwd", _fwd(p[1], dh=dh, ld_qkv=max(3 * H * dh, 8), ld_o=max(H * dh, 8)), "head dim")
    _refused("mia_attn_bwd", _bwd(p[1], dh=dh, ld_qkv=max(3 * H * dh, 8), ld_o=max(H * dh, 8), ld_do=max(H * dh, 8),
                                  ld_dqkv=max(3 * H * dh, 8)), "head dim")


@pytest.mark.parametrize("size", [dict(B=0), dict(N=0), dict(H=0), dict(N=-1), dict(B=65536)])
def test_sizes(p, size):
    _refused("mia_attn_fwd", _fwd(p[1], **size), "must be at (least|most)")
    _refused("mia_attn_bwd", _bwd(p[1], **size), "must be at (least|most)")


@pytest.mark.parametrize("dtype", [_lib.MIA_F32, 7, -1])
def test_bad_dtype(p, dtype):
    _refused("mia_attn_fwd", _fwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")
    _refused("mia_attn_bwd", _bwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")


@pytest.mark.parametrize("pitch", [dict(ld_qkv=3 * C - 8), dict(ld_qkv=3 * C + 4), dict(ld_o=C - 8), dict(ld_o=C + 2)])
def test_fwd_pitches(p, pitch):
    _refused("mia_attn_fwd", _fwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("pitch", [dict(ld_qkv=3 * C - 8), dict(ld_o=C + 4), dict(ld_do=C - 8), dict(ld_do=C + 1),
                                   dict(ld_dqkv=C), dict(ld_dqkv=3 * C + 2)])
def test_bwd_pitches(p, pitch):
    _refused("mia_attn_bwd", _bwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("which", ["qkv", "o", "lse"])
def test_fwd_alignment(p, which):
    _refused("mia_attn_fwd", _fwd(p[1], **{which: p[1] + 8}), "16-byte aligned")


def test_fwd_without_lse_gets_past_its_alignment(p):
    """lse is optional (inference): NULL is accepted, so a misaligned o is what the call then refuses."""
    _refused("mia_attn_fwd", _fwd(p[1] + 2, null="lse", qkv=p[1]), "16-byte aligned")


@pytest.mark.parametrize("which", ["qkv", "o", "dout", "lse", "delta", "dqkv"])
def test_bwd_alignment(p, which):
    _refused("mia_attn_bwd", _bwd(p[1], **{which: p[1] + 4}), "16-byte aligned")


def test_op_refuses_cpu_bad_head_dims_and_levels():
    import torch
    from medical_image_analysis_b200.mae import attention_fn
    wq, wp = torch.zeros(3 * 64, 64), torch.zeros(64, 64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        attention_fn(torch.zeros(1, 3, 64), wq, None, wp, None, 2)
    with pytest.raises(ValueError, match="checkpoint_lvl"):
        attention_fn(torch.zeros(1, 3, 64), wq, None, wp, None, 2, checkpoint_lvl=2)


def test_cpu_and_fp32_attention_takes_the_composition():
    import torch
    from medical_image_analysis_b200 import mae
    torch.manual_seed(0)
    m = mae.Attention(64, num_heads=2, qkv_bias=True)
    x = torch.randn(2, 5, 64, requires_grad=True)
    assert not mae.attention_eligible(m, x)
    assert torch.equal(m(x), m._forward_composed(x))


def test_sass_runs_on_wgmma_and_tma():
    obj = os.path.join(os.path.dirname(_lib.LIB_PATH), "build", "attention.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("no in-tree attention.o or no cuobjdump")
    sass = subprocess.run([tool, "-sass", obj], stdout=subprocess.PIPE, text=True, check=True).stdout
    for kernel in ("attn_fwd_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel"):
        assert kernel in sass, kernel
    assert "HGMMA" in sass and "UTMALDG" in sass
