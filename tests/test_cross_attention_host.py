"""CPU-only checks of the cross-attention entry points' C ABI (mia_xattn_fwd / _bwd): every bad argument is refused before
any CUDA call, on the GEMM channel; the op's own refusals; the CPU / fp32 module is the composition; and the in-tree object
holds the cross-attention instantiations on wgmma and TMA."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from medical_image_analysis_b200 import _lib, arm_pretrain

B, N, H, DH, SEG = 2, 48, 2, 64, 16
C = H * DH


@pytest.fixture(scope="module")
def p():
    _lib.lib()
    buf = ctypes.create_string_buffer(256)
    addr = ctypes.cast(buf, ctypes.c_void_p).value
    return buf, (addr + 15) // 16 * 16                              # a 16-byte aligned host address: never dereferenced


def _fwd(ptr, null=None, **kw):
    a = dict(q=ptr, kv=ptr, o=ptr, lse=ptr, B=B, N=N, H=H, dh=DH, seg=SEG, ld_q=C, ld_kv=2 * C, ld_o=C, dtype=_lib.MIA_BF16)
    a.update(kw)
    if null:
        a[null] = None
    return tuple(a.values())


def _bwd(ptr, null=None, **kw):
    a = dict(q=ptr, kv=ptr, o=ptr, dout=ptr, lse=ptr, delta=ptr, dq=ptr, dkv=ptr, B=B, N=N, H=H, dh=DH, seg=SEG, ld_q=C, ld_kv=2 * C, ld_o=C,
             ld_do=C, ld_dq=C, ld_dkv=2 * C, dtype=_lib.MIA_BF16)
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
    for name in ("mia_xattn_fwd", "mia_xattn_bwd"):
        assert hasattr(L, name)
        assert _lib.ABI[name][2] == "mia_gemm_last_error"


@pytest.mark.parametrize("null", ["q", "kv", "o"])
def test_fwd_null_pointers(p, null):
    _refused("mia_xattn_fwd", _fwd(p[1], null), "null pointer")


@pytest.mark.parametrize("null", ["q", "kv", "o", "dout", "lse", "delta", "dq", "dkv"])
def test_bwd_null_pointers(p, null):
    _refused("mia_xattn_bwd", _bwd(p[1], null), "null pointer")


@pytest.mark.parametrize("dh", [32, 80, 16, 128, 0])
def test_head_dim_must_be_64(p, dh):
    ld = dict(ld_q=max(H * dh, 8), ld_kv=max(2 * H * dh, 8), ld_o=max(H * dh, 8))
    _refused("mia_xattn_fwd", _fwd(p[1], dh=dh, **ld), "head dim")
    _refused("mia_xattn_bwd", _bwd(p[1], dh=dh, ld_do=ld["ld_o"], ld_dq=ld["ld_q"], ld_dkv=ld["ld_kv"], **ld), "head dim")


@pytest.mark.parametrize("size", [dict(B=0), dict(N=0), dict(H=0), dict(N=-1), dict(B=65536), dict(H=65536)])
def test_sizes(p, size):
    _refused("mia_xattn_fwd", _fwd(p[1], **size), "must be at (least|most)")
    _refused("mia_xattn_bwd", _bwd(p[1], **size), "must be at (least|most)")


@pytest.mark.parametrize("seg", [0, -16, N + 1])
def test_segment_length(p, seg):
    _refused("mia_xattn_fwd", _fwd(p[1], seg=seg), "segment length")
    _refused("mia_xattn_bwd", _bwd(p[1], seg=seg), "segment length")


@pytest.mark.parametrize("dtype", [_lib.MIA_F32, 7, -1])
def test_bad_dtype(p, dtype):
    _refused("mia_xattn_fwd", _fwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")
    _refused("mia_xattn_bwd", _bwd(p[1], dtype=dtype), "dtype must be bf16 or fp16")


@pytest.mark.parametrize("pitch", [dict(ld_q=C - 8), dict(ld_q=C + 4), dict(ld_kv=C), dict(ld_kv=2 * C + 2), dict(ld_o=C - 8), dict(ld_o=C + 1)])
def test_fwd_pitches(p, pitch):
    _refused("mia_xattn_fwd", _fwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("pitch", [dict(ld_q=C - 8), dict(ld_kv=2 * C - 8), dict(ld_o=C + 4), dict(ld_do=C - 8), dict(ld_do=C + 1),
                                   dict(ld_dq=C - 8), dict(ld_dq=C + 2), dict(ld_dkv=C), dict(ld_dkv=2 * C + 4)])
def test_bwd_pitches(p, pitch):
    _refused("mia_xattn_bwd", _bwd(p[1], **pitch), "row pitches must cover a row and be multiples of 8")


@pytest.mark.parametrize("which", ["q", "kv", "o", "lse"])
def test_fwd_alignment(p, which):
    _refused("mia_xattn_fwd", _fwd(p[1], **{which: p[1] + 8}), "16-byte aligned")


def test_fwd_without_lse_gets_past_its_alignment(p):
    """lse is optional (inference): NULL is accepted, so a misaligned o is what the call then refuses."""
    _refused("mia_xattn_fwd", _fwd(p[1], null="lse", o=p[1] + 2), "16-byte aligned")


@pytest.mark.parametrize("which", ["q", "kv", "o", "dout", "lse", "delta", "dq", "dkv"])
def test_bwd_alignment(p, which):
    _refused("mia_xattn_bwd", _bwd(p[1], **{which: p[1] + 4}), "16-byte aligned")


def test_op_refuses_cpu_and_bad_levels():
    wq, wkv, wp = torch.zeros(C, C), torch.zeros(2 * C, C), torch.zeros(C, C)
    x = torch.zeros(1, 32, C)
    with pytest.raises(RuntimeError, match="no CPU path"):
        arm_pretrain.cross_attention_fn(x, x, wq, None, wkv, None, wp, None, H, 16)
    with pytest.raises(ValueError, match="checkpoint_lvl"):
        arm_pretrain.cross_attention_fn(x, x, wq, None, wkv, None, wp, None, H, 16, checkpoint_lvl=2)


def test_cpu_and_fp32_cross_attention_takes_the_composition():
    torch.manual_seed(0)
    m = arm_pretrain.CrossAttention(C, num_heads=H, qkv_bias=True)
    mask = arm_pretrain.VisionMamba.mask_generate(3, 16)
    q, kv = torch.randn(2, 48, C, requires_grad=True), torch.randn(2, 48, C, requires_grad=True)
    assert arm_pretrain.mask_segment(mask, 48) == 16
    assert not arm_pretrain.cross_attention_eligible(m, q, kv, mask)
    assert torch.equal(m(q, kv, mask), m._forward_composed(q, kv, mask))


def test_mask_segment_reads_the_pattern():
    mask = arm_pretrain.VisionMamba.mask_generate(8, 16)
    assert arm_pretrain.mask_segment(mask, 128) == 16
    assert arm_pretrain.mask_segment(mask, 64) is None                       # wrong size
    assert arm_pretrain.mask_segment(torch.zeros(128, 128), 128) == 128      # all visible: one segment of N
    assert arm_pretrain.mask_segment(torch.randn(128, 128), 128) is None
    causal = torch.zeros(128, 128).masked_fill(torch.ones(128, 128, dtype=torch.bool).triu(1), float("-inf"))
    assert arm_pretrain.mask_segment(causal, 128) == 1                        # token-causal is seg 1
    mask[5, 100] = 0.0                                                       # a mutated buffer is read again
    assert arm_pretrain.mask_segment(mask, 128) is None
    mask[5, 100] = float("-inf")
    assert arm_pretrain.mask_segment(mask, 128) == 16


def test_sass_runs_on_wgmma_and_tma():
    obj = os.path.join(os.path.dirname(_lib.LIB_PATH), "build", "attention.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("no in-tree attention.o or no cuobjdump")
    sass = subprocess.run([tool, "-sass", obj], stdout=subprocess.PIPE, text=True, check=True).stdout
    bodies = re.split(r"\n\s+Function : ", sass)
    for kernel in ("attn_fwd_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel"):
        for f16 in (0, 1):                                                   # <64, f16, cross = true>
            body = [b for b in bodies if re.match(rf"\S*{kernel}ILi64ELb{f16}ELb1E", b)]
            assert len(body) == 1, (kernel, f16)
            assert "HGMMA" in body[0] and "UTMALDG" in body[0], (kernel, f16)
