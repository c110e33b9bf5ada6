"""GPU parity of the depth-wise 3x3 conv2d (+ bias, + SiLU) kernels (csrc/dwconv2d.cu, through the C ABI) against the
reference's own definition, `self.act(self.conv2d(x))` with nn.Conv2d(C, C, 3, padding=1, groups=C)
(R2GenCSR/VMamba/classification/models/vmamba.py:574-582, 1120-1122), evaluated by torch on the CPU in float64 on the
same rounded inputs.

Criteria (tests/parity.py): y and dx of bf16 / fp16 by ``cmp_stored`` (1 ulp of the rounded oracle + 1e-3 RMS), of fp32
by ``cmp_f32``; dweight / dbias are fp32 sums over B x H x W products, also by ``cmp_f32``.  Worst err / tol measured on
an H100 80GB HBM3 at 700 W (MIA_PARITY_LOG, every case of this file): y 0.94 (bf16 / fp16), 0.028 (fp32); dx 0.96
(bf16 / fp16), 0.075 (fp32); dweight 0.049; dbias 0.036.  The 16-bit values near 1 are elements whose fp32 value lies
across a rounding boundary from the oracle's: one ulp, which the criterion allows.  No criterion was widened.

Every case asserts the kernel instances its configuration launches (recorded by torch.profiler in a child process,
tests/kernel_trace.py): the vector (4-element) or element-wise instance; and, restated from the launchers, how many
planes a block stages, how many times the forward's grid (capped at 16 blocks per SM) sweeps the planes and how many
batch passes the backward takes.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.kernel_trace import in_child, names_of, targs
from tests.parity import cmp_f32, cmp_stored

pytestmark = pytest.mark.gpu

DW_KERNEL = r"\bdwconv2d_(fwd|bwd)_kernel<"
T_NAME = {torch.float32: "float", torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}


def geometry(B, C, H, W, sms):
    """The launchers' choices: planes per forward block, forward grid sweeps, backward batch passes."""
    P = max(1, 2048 // (H * W))
    pf, pb = min(P, 16), min(P, B)
    blocks = min(math.ceil(B * C / pf), 16 * sms)
    return dict(planes=pf, sweeps=math.ceil(B * C / (pf * blocks)), bwd_passes=math.ceil(B / pb),
                # fp32 staged results would start 8 bytes off a 16-byte boundary without the padding of the planes region
                odd_pad=(H * W) % 4 == 0 and pf * ((H + 2) * (W + 2) + 12) % 4 != 0)


# (B, C, H, W) -> what the shape reaches (entries of `geometry`; sweeps = 2 means "at least 2" on any H100)
SHAPES = {
    (2, 8, 14, 14): {}, (3, 96, 7, 7): {}, (1, 5, 1, 1): {}, (2, 16, 28, 28): {}, (1, 4, 80, 80): {}, (2, 768, 14, 14): {},
    (2, 6, 3, 17): {},
    (32, 768, 14, 14): dict(planes=10, sweeps=2, bwd_passes=4),     # forward grid-stride loop, 4 backward passes
    (3, 4, 80, 80): dict(planes=1, bwd_passes=3),
    (45, 8, 7, 7): dict(planes=16, bwd_passes=2),                   # element-wise (H W % 4 != 0)
    (2, 16, 16, 16): dict(planes=8),                                # a warp per plane
    (2, 16, 20, 20): dict(planes=5),                                # the block walks each plane
    (2, 8, 11, 12): dict(planes=15, odd_pad=True), (2, 8, 12, 11): dict(planes=15, odd_pad=True),
    (2, 8, 7, 32): dict(planes=9, odd_pad=True), (2, 8, 8, 17): dict(planes=15, odd_pad=True),
    (1, 4, 33, 32): dict(planes=1, odd_pad=True),
    (1, 2, 128, 128): dict(planes=1),                               # the largest plane
}


def _on_gpu(t, offset=0):
    """``t`` on the GPU, contiguous, its storage starting ``offset`` elements into a buffer."""
    buf = torch.empty(offset + t.numel(), dtype=t.dtype, device="cuda")
    buf[offset:].copy_(t.reshape(-1))
    return buf[offset:].view(t.shape)


def _reference(x, w, b, dy, silu):
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    br = None if b is None else b.double().requires_grad_(True)
    pre = F.conv2d(xr, wr, br, padding=1, groups=x.shape[1])
    yr = F.silu(pre) if silu else pre
    yr.backward(dy.double())
    return pre.detach(), (yr.detach(), xr.grad, wr.grad, None if b is None else br.grad)


DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
UNALIGNED = (2, 8, 16, 16)           # the shape of the unaligned-input and edge-value cases


def _key(shape, dtype, silu, has_bias, offset=0):
    return f"{tuple(shape)}|{dtype}|{silu}|{has_bias}|{offset}"


def _configs():
    for shape in SHAPES:
        for dtype in DTYPES.values():
            for silu, has_bias in ((True, True), (False, False), (True, False)):
                yield shape, dtype, silu, has_bias, 0
    for dtype in DTYPES.values():
        for offset in (1, 3):
            yield UNALIGNED, dtype, True, True, offset
        for silu in (True, False):
            yield UNALIGNED, dtype, silu, True, 0


def kernel_paths():
    """{configuration: [forward kernels, backward kernels]} under the profiler, for every configuration the tests run."""
    from medical_image_analysis_b200.vmamba import DWConv2dFn
    out = {}
    for shape, dtype, silu, has_bias, offset in _configs():
        x = _on_gpu(torch.randn(*shape, device="cuda").to(dtype), offset).requires_grad_(True)
        w = torch.randn(shape[1], 1, 3, 3, device="cuda", requires_grad=True)
        b = torch.randn(shape[1], device="cuda", requires_grad=True) if has_bias else None
        leaves = [t for t in (x, w, b) if t is not None]
        kf = names_of(lambda: DWConv2dFn.apply(x, w, b, silu), DW_KERNEL)
        y = DWConv2dFn.apply(x, w, b, silu)
        kb = names_of(lambda: torch.autograd.grad(y, leaves, torch.ones_like(y), retain_graph=True), DW_KERNEL)
        out[_key(shape, dtype, silu, has_bias, offset)] = [kf, kb]
    return out


@pytest.fixture(scope="module")
def paths():
    return in_child("tests.test_dwconv2d_gpu:kernel_paths")


def _check(tag, paths, x, w, b, dy, silu, x_offset=0, vec=None):
    """Forward and backward on the GPU against the float64 oracle, and the kernel instances of the configuration."""
    from medical_image_analysis_b200.vmamba import DWConv2dFn
    dtype = x.dtype
    _, ref = _reference(x, w, b, dy, silu)
    xg = _on_gpu(x, x_offset).requires_grad_(True)
    wg = w.cuda().requires_grad_(True)
    bg = None if b is None else b.cuda().requires_grad_(True)
    y = DWConv2dFn.apply(xg, wg, bg, silu)
    assert y.dtype == dtype and y.shape == x.shape
    leaves = [t for t in (xg, wg, bg) if t is not None]
    grads = torch.autograd.grad(y, leaves, dy.cuda())
    if vec is None:
        vec = (x.shape[2] * x.shape[3]) % 4 == 0
    kf, kb = paths[_key(x.shape, dtype, silu, b is not None, x_offset)]
    for names, kind in ((kf, "fwd"), (kb, "bwd")):
        assert len(names) == 1 and f"dwconv2d_{kind}_kernel<" in names[0], names
        assert targs(names[0], f"dwconv2d_{kind}_kernel<") == [T_NAME[dtype], str(silu).lower(), "4" if vec else "1"], names
    got = [y] + list(grads) + ([None] if b is None else [])
    for what, g, r in zip(("y", "dx", "dweight", "dbias"), got, ref):
        if r is None:
            continue
        if what in ("y", "dx") and dtype != torch.float32:
            cmp_stored(g, r, dtype, f"dwconv2d {tag} {what}")
        else:
            assert g.dtype == torch.float32
            cmp_f32(g, r, f"dwconv2d {tag} {what}")


def _inputs(B, C, H, W, dtype, has_bias, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, C, H, W, generator=g) * scale).to(dtype)
    w = torch.randn(C, 1, 3, 3, generator=g) * 0.4
    b = torch.randn(C, generator=g) if has_bias else None
    dy = torch.randn(B, C, H, W, generator=g).to(dtype)
    return x, w, b, dy


@pytest.mark.parametrize("shape", list(SHAPES), ids=str)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("silu,has_bias", [(True, True), (False, False), (True, False)])
def test_dwconv2d_parity(paths, shape, dtype, silu, has_bias):
    B, C, H, W = shape
    geo = geometry(B, C, H, W, torch.cuda.get_device_properties(0).multi_processor_count)
    for k, v in SHAPES[shape].items():
        assert (geo[k] >= v) if k == "sweeps" else geo[k] == v, (k, geo)
    x, w, b, dy = _inputs(B, C, H, W, dtype, has_bias, B * 1000 + C + H * W)
    _check(f"{shape} {dtype} silu={silu} bias={has_bias}", paths, x, w, b, dy, silu)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("offset", [1, 3])
def test_dwconv2d_unaligned_input(paths, dtype, offset):
    """A contiguous input at an odd element offset: the element-wise instances run although H W % 4 == 0."""
    x, w, b, dy = _inputs(*UNALIGNED, dtype, True, 7 + offset)
    _check(f"off{offset} {dtype}", paths, x, w, b, dy, True, x_offset=offset, vec=False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("silu", [True, False])
def test_dwconv2d_edge_values(paths, dtype, silu):
    """Pre-activations spanning about +-100 (SiLU saturates both ways), exact zeros, and a channel with all-zero taps."""
    x, w, b, dy = _inputs(*UNALIGNED, dtype, True, 11, scale=25.0)
    x[:, :, ::3] = 0                     # zero rows
    x[1, 5] = 0                          # a zero plane
    w[2] = 0                             # a channel whose output is its bias
    pre, _ = _reference(x, w, b, dy, silu)
    assert pre.max() > 80 and pre.min() < -80 and (pre[:, 2] == b[2].double()).all()
    _check(f"edge {dtype} silu={silu}", paths, x, w, b, dy, silu)


def test_dwconv2d_backward_is_deterministic():
    """Two backward runs at a multi-pass shape (4 batch passes) give bit-identical dx, dweight and dbias."""
    from medical_image_analysis_b200.vmamba import DWConv2dFn
    x, w, b, dy = _inputs(32, 64, 14, 14, torch.bfloat16, True, 5)
    assert geometry(32, 64, 14, 14, 132)["bwd_passes"] == 4
    xg, wg, bg = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = DWConv2dFn.apply(xg, wg, bg, True)
    g1 = torch.autograd.grad(y, (xg, wg, bg), dy.cuda(), retain_graph=True)
    g2 = torch.autograd.grad(y, (xg, wg, bg), dy.cuda())
    for what, a, c in zip(("dx", "dweight", "dbias"), g1, g2):
        assert torch.equal(a, c), what


def test_ss2d_uses_the_fused_conv_and_matches_torch():
    """SS2D.forward with the fused conv + SiLU equals the same module evaluated with nn.Conv2d + nn.SiLU (fwd + grads)."""
    from medical_image_analysis_b200 import vmamba
    torch.manual_seed(0)
    m = vmamba.SS2D(d_model=32, d_state=1, ssm_ratio=2.0, dt_rank="auto", d_conv=3, forward_type="v2").cuda()
    x = torch.randn(2, 14, 14, 32, device="cuda", requires_grad=True)
    y = m(x)
    y.square().mean().backward()
    g1 = [p.grad.clone() for p in m.parameters()]
    gx1 = x.grad.clone()
    m.zero_grad(); x.grad = None
    orig = vmamba.dwconv2d_silu
    vmamba.dwconv2d_silu = lambda t, conv, silu=True: F.silu(conv(t))
    try:
        y2 = m(x)
        y2.square().mean().backward()
    finally:
        vmamba.dwconv2d_silu = orig
    assert torch.allclose(y, y2, rtol=1e-4, atol=1e-5)
    assert torch.allclose(gx1, x.grad, rtol=1e-3, atol=1e-5)
    for a, p in zip(g1, m.parameters()):
        assert torch.allclose(a, p.grad, rtol=2e-3, atol=1e-5), (a - p.grad).abs().max()
