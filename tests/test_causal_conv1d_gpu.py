"""GPU parity of the depth-wise causal conv1d kernels (csrc/causal_conv1d.cu, through the C ABI) against the reference's
own definition of the op, `self.act(self.conv1d(x)[..., :seqlen])` with a depth-wise nn.Conv1d(padding = k - 1)
(arm/Finetuning/mamba_simple.py:112-120, 673), evaluated by torch on the CPU in float64 on the same rounded inputs.

Criteria (tests/parity.py): y and dx of bf16 / fp16 by ``cmp_stored`` (1 ulp of the rounded oracle + 1e-3 RMS), of fp32
by ``cmp_f32``; dweight / dbias are fp32 sums over B x L products, also by ``cmp_f32``.  Worst err / tol measured on an
H100 80GB HBM3 at 700 W (MIA_PARITY_LOG, every case of this file): y 0.96 (bf16 / fp16), 0.019 (fp32); dx 0.97
(bf16 / fp16), 0.073 (fp32); dweight 0.040; dbias 0.030.  The 16-bit values near 1 are elements whose fp32 value lies
across a rounding boundary from the oracle's: one ulp, which the criterion allows.  No criterion was widened.

Every case asserts the kernel instances its configuration launches (recorded by torch.profiler in a child process,
tests/kernel_trace.py): their dtype, width and activation; and, restated from the launchers, how many channel rows a
forward block takes and how many passes the backward's 8 warps x 4 x 31 quads take over the channel's batch x L / 4 quads.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.kernel_trace import in_child, names_of, targs
from tests.parity import cmp_f32, cmp_stored

pytestmark = pytest.mark.gpu

CONV_KERNEL = r"\bcausal_conv1d_(fwd|bwd)_kernel<"
T_NAME = {torch.float32: "float", torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}


def geometry(B, D, L):
    """The launchers' choices at seqlen L (padded to a multiple of 4): rows per forward block, backward passes."""
    qpr = -(-L // 4)
    return dict(rows_per_block=min(math.ceil(2 * 4 * 256 / qpr), D), bwd_passes=math.ceil(B * qpr / (4 * 8 * 31)))


# (batch, dim, seqlen) -> what the shape reaches (entries of `geometry`)
SHAPES = {
    (2, 8, 16): {}, (3, 96, 196): {}, (1, 5, 4): {}, (2, 64, 1024): {}, (2, 1536, 196): {}, (2, 24, 197): {}, (3, 7, 50): {},
    (4, 64, 1024): dict(bwd_passes=2),                       # 1024 quads: a partial second backward pass
    (24, 1536, 197): dict(bwd_passes=2),                     # the ARM mixer's width, padded to 200: 1200 quads
    (2, 16, 6400): dict(rows_per_block=2, bwd_passes=4),     # long rows: 3200 quads
    (1, 8, 8200): dict(rows_per_block=1, bwd_passes=3),
}


def _ref(x, w, b, silu):
    x64, w64 = x.double(), w.double()
    y = F.conv1d(x64, w64.unsqueeze(1), None if b is None else b.double(), padding=w.shape[1] - 1, groups=w.shape[0])[..., : x.shape[-1]]
    return F.silu(y) if silu else y


def _compare(tag, dtype, got, ref):
    for what, g, r in zip(("y", "dx", "dweight", "dbias"), got, ref):
        if r is None:
            continue
        if what in ("y", "dx") and dtype != torch.float32:
            cmp_stored(g, r, dtype, f"causal_conv1d {tag} {what}")
        else:
            assert g.dtype == torch.float32
            cmp_f32(g, r, f"causal_conv1d {tag} {what}")


def _assert_instances(kf, kb, dtype, width, silu):
    for names, kind in ((kf, "fwd"), (kb, "bwd")):
        assert len(names) == 1 and f"causal_conv1d_{kind}_kernel<" in names[0], names
        assert targs(names[0], f"causal_conv1d_{kind}_kernel<") == [T_NAME[dtype], str(width), str(silu).lower()], names


EDGE = (3, 16, 256)                  # the shape of the edge-value cases
XZ = (4, 32, 300)                    # (batch, d, seqlen) of the xz[:, :d] case


def _key(shape, dtype, width, silu, has_bias):
    return f"{tuple(shape)}|{dtype}|{width}|{silu}|{has_bias}"


def kernel_paths():
    """{configuration: [forward kernels, backward kernels]} under the profiler, for every configuration the tests run; for
    the xz[:, :d] view, every kernel and copy its forward launches."""
    from medical_image_analysis_b200.selective_scan_interface import causal_conv1d_fn
    configs = [(shape, dtype, width, silu, has_bias) for shape in SHAPES for dtype in (torch.float32, torch.bfloat16, torch.float16)
               for width in (4, 3, 2, 1) for silu, has_bias in ((True, True), (False, False))]
    configs += [(EDGE, dtype, 4, silu, True) for dtype in (torch.float32, torch.bfloat16, torch.float16) for silu in (True, False)]
    out = {}
    for shape, dtype, width, silu, has_bias in configs + [("xz", torch.bfloat16, 4, True, True)]:
        if shape == "xz":
            B, D, L = XZ
            x = torch.randn(B, 2 * D, L, device="cuda").to(dtype).requires_grad_(True)[:, :D]
            fwd_pattern = r"kernel|Memcpy"
        else:
            B, D, L = shape
            x = torch.randn(B, D, L, device="cuda").to(dtype).requires_grad_(True)
            fwd_pattern = CONV_KERNEL
        w = torch.randn(D, width, device="cuda", requires_grad=True)
        b = torch.randn(D, device="cuda", requires_grad=True) if has_bias else None
        act = "silu" if silu else None
        kf = names_of(lambda: causal_conv1d_fn(x, w, b, act), fwd_pattern)
        y = causal_conv1d_fn(x, w, b, act)
        leaves = [t for t in (x, w, b) if t is not None]
        kb = names_of(lambda: torch.autograd.grad(y, leaves, torch.ones_like(y), retain_graph=True), CONV_KERNEL)
        out[_key(shape, dtype, width, silu, has_bias)] = [kf, kb]
    return out


@pytest.fixture(scope="module")
def paths():
    return in_child("tests.test_causal_conv1d_gpu:kernel_paths")


def _check(tag, paths, x, w, b, dy, silu):
    """Forward and backward through causal_conv1d_fn against the float64 oracle, and the kernel instances of the
    configuration."""
    from medical_image_analysis_b200.selective_scan_interface import causal_conv1d_fn
    xr = x.double().requires_grad_(True)
    wr = w.double().requires_grad_(True)
    br = None if b is None else b.double().requires_grad_(True)
    yr = _ref(xr, wr, br, silu)
    yr.backward(dy.double())
    xg, wg = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    bg = None if b is None else b.cuda().requires_grad_(True)
    y = causal_conv1d_fn(xg, wg, bg, "silu" if silu else None)
    assert y.dtype == x.dtype and y.shape == x.shape
    grads = torch.autograd.grad(y, [t for t in (xg, wg, bg) if t is not None], dy.cuda())
    _assert_instances(*paths[_key(x.shape, x.dtype, w.shape[1], silu, b is not None)], x.dtype, w.shape[1], silu)
    _compare(tag, x.dtype, [y] + list(grads), [yr.detach(), xr.grad, wr.grad, None if b is None else br.grad])


def _inputs(B, D, L, width, dtype, has_bias, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, D, L, generator=g) * scale).to(dtype)
    w = torch.randn(D, width, generator=g) * 0.5
    b = torch.randn(D, generator=g) if has_bias else None
    dy = torch.randn(B, D, L, generator=g).to(dtype)
    return x, w, b, dy


@pytest.mark.parametrize("shape", list(SHAPES), ids=str)
@pytest.mark.parametrize("width", [4, 3, 2, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("silu,has_bias", [(True, True), (False, False)])
def test_causal_conv1d_parity(paths, shape, width, dtype, silu, has_bias):
    B, D, L = shape
    geo = geometry(B, D, L)
    for k, v in SHAPES[shape].items():
        assert geo[k] == v, (k, geo)
    x, w, b, dy = _inputs(B, D, L, width, dtype, has_bias, B * 1000 + D + L + width)
    _check(f"{shape} w{width} {dtype} silu={silu}", paths, x, w, b, dy, silu)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("silu", [True, False])
def test_causal_conv1d_edge_values(paths, dtype, silu):
    """Pre-activations spanning about +-100 (SiLU saturates both ways), exact zeros, and a channel with all-zero taps."""
    x, w, b, dy = _inputs(*EDGE, 4, dtype, True, 13, scale=20.0)
    x[:, :, 100:140] = 0                 # a run of zeros in every row
    x[1, 5] = 0                          # a zero row
    w[2] = 0                             # a channel whose output is its bias
    pre = _ref(x, w, b, False)
    assert pre.max() > 80 and pre.min() < -80 and (pre[:, 2] == b[2].double()).all()
    _check(f"edge {dtype} silu={silu}", paths, x, w, b, dy, silu)


def test_causal_conv1d_on_xz_view_and_errors(paths):
    """x is the first half of xz (mamba_simple.py:666): batch stride 2 d L, read in place by the forward and the backward
    (the forward launches the conv kernel and nothing else: no copy); gradients reach xz's first half only; bad shapes
    raise."""
    from medical_image_analysis_b200.selective_scan_interface import causal_conv1d_fn
    g = torch.Generator().manual_seed(0)
    B, d, L = XZ
    xz0 = torch.randn(B, 2 * d, L, generator=g).bfloat16()
    w = torch.randn(d, 4, generator=g) * 0.5
    b = torch.randn(d, generator=g)
    dy = torch.randn(B, d, L, generator=g).bfloat16()
    xzr = xz0.double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = _ref(xzr[:, :d], wr, br, True)
    yr.backward(dy.double())
    xz = xz0.cuda().requires_grad_(True)
    wg, bg = w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    x = xz[:, :d]
    assert x.stride(0) == 2 * d * L
    y = causal_conv1d_fn(x, wg, bg, "silu")
    grads = torch.autograd.grad(y, (xz, wg, bg), dy.cuda())
    _assert_instances(*paths[_key("xz", torch.bfloat16, 4, True, True)], torch.bfloat16, 4, True)
    _compare("xz view", torch.bfloat16, [y, grads[0][:, :d], grads[1], grads[2]], [yr.detach(), xzr.grad[:, :d], wr.grad, br.grad])
    assert not grads[0][:, d:].any()
    with pytest.raises(RuntimeError):
        causal_conv1d_fn(torch.randn(2, 16, 12, device="cuda"), wg, None, "silu")        # channel mismatch
    with pytest.raises(NotImplementedError):
        causal_conv1d_fn(x, wg, None, "gelu")


def test_causal_conv1d_backward_is_deterministic():
    """Two backward runs at a multi-pass shape (2 passes) give bit-identical dx, dweight and dbias."""
    from medical_image_analysis_b200.selective_scan_interface import causal_conv1d_fn
    x, w, b, dy = _inputs(4, 64, 1024, 4, torch.bfloat16, True, 3)
    assert geometry(4, 64, 1024)["bwd_passes"] == 2
    xg, wg, bg = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = causal_conv1d_fn(xg, wg, bg, "silu")
    g1 = torch.autograd.grad(y, (xg, wg, bg), dy.cuda(), retain_graph=True)
    g2 = torch.autograd.grad(y, (xg, wg, bg), dy.cuda())
    for what, a, c in zip(("dx", "dweight", "dbias"), g1, g2):
        assert torch.equal(a, c), what
