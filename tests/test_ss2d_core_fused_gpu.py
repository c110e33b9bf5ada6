"""The fused SS2D core (vmamba.SS2DCoreFn): the epilogue kernel pair against the torch statement of its tail on the same scan
output, the whole op against the composition it replaces, CrossScan1b1 / its adjoint against the torch statement, checkpoint
levels, the saved-tensor bound, the kernel path, determinism, routing and the error paths."""
import ctypes
import math
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import kernel_trace
from tests.parity import cmp_f32

gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------- fixtures
def _module(ft, d_inner, N, seed=0):
    from medical_image_analysis_b200.vmamba import SS2D
    torch.manual_seed(seed)
    m = SS2D(d_model=d_inner // 2, d_state=N, ssm_ratio=2.0, forward_type=ft)
    with torch.no_grad():                       # a LayerNorm that is not the identity, so its gradients are exercised
        m.out_norm.weight.uniform_(0.5, 1.5)
        m.out_norm.bias.uniform_(-0.2, 0.2)
    return m.cuda()


def _run(m, x, mode, composed, seed=9, **kw):
    """-> (output, {name: grad}) of one forward + backward; mode fp32 / bf16 (module and input in bf16) / autocast (bf16) /
    autocast_fp16."""
    x = x.detach().clone().requires_grad_()
    for p in m.parameters():
        p.grad = None
    fwd = m._forward_composed if composed else m.forward
    if mode.startswith("autocast"):
        with torch.autocast("cuda", dtype=torch.float16 if mode == "autocast_fp16" else torch.bfloat16):
            out = fwd(x)
    else:
        out = fwd(x)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).to(out.device)
    (out.float() * w).sum().backward()
    return out, {"x": x.grad, **{n: p.grad for n, p in m.named_parameters()}}


def _close(got, ref, what, rel_rms, worst_rms):
    """Relative RMS error and worst element error in units of RMS(ref).  The two paths differ in the summation order of the
    projections, so a value next to a bf16 rounding boundary (the reference's cast of the merged scan output, and every
    bf16 operand) can land one bf16 ulp apart: sparse 0.4-0.8 % steps that the LayerNorm and the gradients carry on."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape and torch.isfinite(got).all(), what
    rms = ref.pow(2).mean().sqrt().item() + 1e-30
    err = (got - ref).abs()
    rel, worst = err.pow(2).mean().sqrt().item() / rms, err.max().item() / rms
    assert rel <= rel_rms and worst <= worst_rms, f"{what}: rel RMS err {rel:.3e}, worst err / RMS(ref) {worst:.3e}"


# ---------------------------------------------------------------------------------------------------------- the epilogue
def _tail_ref(ys, H, W, weight, bias, eps, z, gate, out_dtype):
    """The composition's tail in torch on the same scan output: CrossMerge, the bf16 cast, LayerNorm in fp32, the gate."""
    from medical_image_analysis_b200.vmamba import cross_merge_fwd
    B, K, D, L = ys.shape
    y = cross_merge_fwd(ys, H, W) if not ys.requires_grad else _merge(ys, H, W)
    yb = y.to(torch.bfloat16)
    o = F.layer_norm(yb.float().transpose(1, 2), (D,), weight, bias, eps).to(out_dtype).view(B, H, W, D)
    if gate == 1:
        o = o * z
    elif gate == 2:
        o = o * F.silu(z)
    return yb.transpose(1, 2), o


def _merge(ys, H, W):
    from medical_image_analysis_b200.vmamba import CrossMerge
    B, K, D, L = ys.shape
    return CrossMerge.apply(ys.view(B, K, D, H, W))


def _epilogue(ys, H, W, weight, bias, eps, z, gate, out_dtype, dy=None):
    """mia_ss2d_merge_norm_fwd (and _bwd when dy is given) called directly."""
    from medical_image_analysis_b200 import _lib
    from medical_image_analysis_b200.vmamba import _tok_view
    B, K, D, L = ys.shape
    dev = ys.device
    out = torch.empty((B, H, W, D), dtype=out_dtype, device=dev)
    yb = torch.empty((B, L, D), dtype=torch.bfloat16, device=dev)
    mean, rstd = torch.empty((B, L), device=dev), torch.empty((B, L), device=dev)
    ln = _lib.MiaLn(weight.data_ptr(), bias.data_ptr(), eps)
    none = _lib.MiaBdl(None, 0, 0, 0)
    zb = _tok_view(z, H, W) if gate else none
    _lib.call("mia_ss2d_merge_norm_fwd", "fwd", dev, ys.data_ptr(), ctypes.byref(ln), ctypes.byref(zb), gate, out.data_ptr(), yb.data_ptr(),
              mean.data_ptr(), rstd.data_ptr(), B, D, H, W, _lib.dtype_code(ys.dtype), _lib.dtype_code(out_dtype))
    if dy is None:
        return out, yb
    dout = torch.empty((B, 4, D, L), device=dev)
    dz = torch.empty_like(out) if gate else None
    dw, db = torch.empty(D, device=dev), torch.empty(D, device=dev)
    ws = torch.empty(int(_lib.lib().mia_ss2d_merge_norm_bwd_workspace(B, D, H, W)), dtype=torch.uint8, device=dev)
    _lib.call("mia_ss2d_merge_norm_bwd", "bwd", dev, dy.data_ptr(), yb.data_ptr(), mean.data_ptr(), rstd.data_ptr(), ctypes.byref(ln),
              ctypes.byref(zb), gate, ctypes.byref(_tok_view(dz, H, W) if gate else none), dout.data_ptr(), dw.data_ptr(), db.data_ptr(),
              ws.data_ptr(), ws.numel(), B, D, H, W, _lib.dtype_code(out_dtype))
    return out, yb, dout, dz, dw, db


# (B, D, H, W): the merge's staged order (H W % 4 != 0) and its vectorised order, partial tiles, D up to 2048 and the largest
# D the shared memory holds (3626)
EPI_SHAPES = [(3, 16, 6, 5), (1, 96, 7, 9), (2, 192, 14, 14), (1, 768, 14, 14), (1, 64, 80, 80), (1, 2048, 7, 7), (1, 3626, 3, 2)]


class _RoundGrad(torch.autograd.Function):
    """Identity whose backward rounds the gradient to `dtype`: where the module's backward computes a product in that dtype."""

    @staticmethod
    def forward(ctx, x, dtype):
        ctx.dtype = dtype
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dtype).double(), None


def _stored(t, dtype):
    """t rounded to dtype in the forward, identity in the backward, and the gradient reaching it rounded to dtype."""
    return _RoundGrad.apply(t + (t.to(dtype).double() - t).detach(), dtype)


def _tail64(yb, weight, bias, eps, z, gate, dy, out_dtype):
    """float64 statement of the tail after the cast, on the kernel's bf16 pre-norm plane, with the module's roundings: the
    LayerNorm output and silu(z) stored in out_dtype, the gate's product and its gradients computed in out_dtype
    -> (out, d yb, dz, dweight, dbias)."""
    B, L, D = yb.shape
    x = yb.double().cpu().requires_grad_()
    w, b = weight.double().cpu().requires_grad_(), bias.double().cpu().requires_grad_()
    zz = z.double().cpu().reshape(B, L, D).requires_grad_()
    o = F.layer_norm(x, (D,), w, b, eps)
    if gate:
        o = _stored(o, out_dtype) * _stored(F.silu(zz) if gate == 2 else zz, out_dtype)
    o.backward(dy.double().cpu().reshape(B, L, D))
    return o.detach(), x.grad, zz.grad, w.grad, b.grad


@gpu
@pytest.mark.parametrize("gate", [0, 1, 2])
@pytest.mark.parametrize("dt", ["f32", "bf16", "bf16_ys_f32"])
@pytest.mark.parametrize("shape", EPI_SHAPES, ids=[f"B{s[0]}_D{s[1]}_{s[2]}x{s[3]}" for s in EPI_SHAPES])
def test_epilogue_matches_statement(shape, dt, gate):
    """yb is bit-identical to CrossMerge(ys).to(bfloat16); the output, dz and the scan's dout (bf16-valued) against a float64
    statement of the rest by the tests/parity.py criteria (two ulp where the kernel rounds twice: the gated output, dz);
    dout holds the same value at the token's position in all four orders."""
    from medical_image_analysis_b200.vmamba import cross_scan_fwd
    from tests.parity import cmp_stored
    B, D, H, W = shape
    L = H * W
    g = torch.Generator().manual_seed(B * D * L + gate)
    ys_dtype = torch.float32 if dt != "bf16" else torch.bfloat16
    out_dtype = torch.float32 if dt == "f32" else torch.bfloat16
    ys = (torch.randn(B, 4, D, L, generator=g) + 0.3).to(ys_dtype).cuda()
    weight = (torch.rand(D, generator=g) + 0.5).cuda()
    bias = (torch.rand(D, generator=g) - 0.5).cuda()
    buf = torch.randn(B, H, W, 2 * D, generator=g).to(out_dtype).cuda()
    z = buf[..., D:]                                                      # read in place, token stride 2 D
    dy = torch.randn(B, H, W, D, generator=g).to(out_dtype).cuda()
    out, yb, dout, dz, dw, db = _epilogue(ys, H, W, weight, bias, 1e-5, z, gate, out_dtype, dy)
    yb_ref, _ = _tail_ref(ys, H, W, weight, bias, 1e-5, z, gate, out_dtype)
    assert torch.equal(yb.view(B, L, D), yb_ref.contiguous()), "yb differs from CrossMerge(ys).to(bfloat16)"
    o64, dyb64, dz64, dw64, db64 = _tail64(yb, weight, bias, 1e-5, z, gate, dy, out_dtype)
    n = 2.0 if gate else 1.0
    if out_dtype == torch.float32:
        cmp_f32(out.view(B, L, D), o64, "out")
    else:
        cmp_stored(out.view(B, L, D), o64, out_dtype, "out", n_ulp=n)
    assert torch.equal(dout, cross_scan_fwd(dout[:, 0].reshape(B, D, H, W).contiguous())), "dout differs between the four orders"
    cmp_stored(dout[:, 0].transpose(1, 2).to(torch.bfloat16), dyb64, torch.bfloat16, "dout")
    if gate:
        if out_dtype == torch.float32:
            cmp_f32(dz.view(B, L, D), dz64, "dz", rtol=1e-4, atol_rms=1e-4)
        else:
            cmp_stored(dz.view(B, L, D), dz64, out_dtype, "dz", n_ulp=2.0)
    for got, ref, what in ((dw, dw64, "dweight"), (db, db64, "dbias")):
        _close(got, ref, what, 1e-4, 1e-3)


# ---------------------------------------------------------------------------------------------------------- the whole op
FT_CASES = [("v3noz", 1, 16, 6, 5), ("v3", 16, 32, 7, 9), ("v2", 4, 32, 14, 14), ("v4", 1, 64, 14, 14), ("v4noz", 4, 32, 7, 9),
            ("v3nozact", 1, 32, 6, 5), ("v2no32", 16, 32, 14, 14), ("v3noz", 1, 768, 14, 14), ("v3", 1, 192, 80, 80),
            ("v3noz", 1, 2048, 6, 5)]
TOL = {"fp32": (2e-3, 6e-2), "bf16": (2e-2, 0.5), "autocast": (2e-2, 0.5), "autocast_fp16": (2e-2, 0.5)}


@gpu
@pytest.mark.parametrize("mode", ["fp32", "bf16", "autocast", "autocast_fp16"])
@pytest.mark.parametrize("case", FT_CASES, ids=[f"{c[0]}_N{c[1]}_D{c[2]}_{c[3]}x{c[4]}" for c in FT_CASES])
def test_fused_matches_composition(case, mode):
    ft, N, D, H, W = case
    if ft == "v2no32" and mode == "fp32":
        pytest.skip("no32 only differs from v2 for low-precision activations")
    m = _module(ft, D, N)
    B = 3 if D * H * W <= 4096 else 1
    x = torch.randn(B, H, W, D // 2, generator=torch.Generator().manual_seed(1)).cuda()
    if mode == "bf16":
        m, x = m.bfloat16(), x.bfloat16()
    assert m._fused_core_args(x) is not None
    out, grads = _run(m, x, mode, composed=False)
    ref, rgrads = _run(m, x, mode, composed=True)
    assert out.dtype == ref.dtype
    rel, worst = TOL[mode]
    _close(out, ref, f"{case} {mode} out", rel, worst)
    for k in rgrads:
        _close(grads[k], rgrads[k], f"{case} {mode} d{k}", rel * 2, worst * 2)


@gpu
@pytest.mark.parametrize("no_einsum", [False, True])
def test_free_function_routes_and_matches(no_einsum):
    from medical_image_analysis_b200 import vmamba
    from medical_image_analysis_b200.selective_scan_interface import SelectiveScanOflex
    m = _module("v3noz", 64, 1)
    x = torch.randn(2, 64, 14, 14, device="cuda", requires_grad=True)
    args = (m.x_proj_weight, None, m.dt_projs_weight, m.dt_projs_bias, m.A_logs, m.Ds)
    kw = dict(out_norm=m.out_norm, SelectiveScan=SelectiveScanOflex, no_einsum=no_einsum)
    out = vmamba.cross_selective_scan(x, *args, **kw)
    assert out.grad_fn is not None and "SS2DCoreFn" in type(out.grad_fn).__name__
    ref = vmamba._cross_selective_scan_composed(x, *args, **kw)
    _close(out, ref, "out", 2e-3, 6e-2)
    w = torch.randn_like(out)
    g = torch.autograd.grad((out * w).sum(), [x, *args[:1], *args[2:]])
    rg = torch.autograd.grad((ref * w).sum(), [x, *args[:1], *args[2:]])
    for a, b, n in zip(g, rg, ("x", "xw", "dtw", "dtb", "A_logs", "Ds")):
        _close(a, b, n, 4e-3, 0.12)


# ---------------------------------------------------------------------------------------------------------- CrossScan1b1
def _torch_1b1(x):
    return torch.stack([x[:, 0].flatten(2), x[:, 1].transpose(2, 3).flatten(2), x[:, 2].flatten(2).flip(-1),
                        x[:, 3].transpose(2, 3).flatten(2).flip(-1)], dim=1)


# (B, C, H, W) -> expected launch path for (fp32, bf16)
P1B1 = {(2, 5, 14, 14): ("vec", "vec"), (1, 3, 7, 9): ("staged", "staged"), (2, 3, 6, 5): ("staged", "staged"),
        (1, 2, 256, 256): ("direct", "vec"), (1, 1, 227, 227): ("direct", "staged")}
K1B1 = r"\bcross_1b1_(direct_)?kernel<"


def _path_1b1(names):
    assert len(names) == 1, names
    if "direct" in names[0]:
        return "direct"
    return "vec" if kernel_trace.targs(names[0], "cross_1b1_kernel<")[1] == "true" else "staged"


def paths_1b1():
    from medical_image_analysis_b200.vmamba import cross_merge_1b1_fwd, cross_scan_1b1_fwd
    res = {}
    for (B, C, H, W) in P1B1:
        for dt in (torch.float32, torch.bfloat16):
            x = torch.randn(B, 4, C, H, W, device="cuda").to(dt)
            ys = torch.randn(B, 4, C, H * W, device="cuda").to(dt)
            res[f"{(B, C, H, W)}|{dt}"] = [_path_1b1(kernel_trace.names_of(lambda: cross_scan_1b1_fwd(x), K1B1)),
                                           _path_1b1(kernel_trace.names_of(lambda: cross_merge_1b1_fwd(ys, H, W), K1B1))]
    return res


@pytest.fixture(scope="module")
def p1b1():
    return kernel_trace.in_child("tests.test_ss2d_core_fused_gpu:paths_1b1")


@gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("shape", list(P1B1))
def test_cross_scan_1b1_bit_identical(p1b1, shape, dt):
    from medical_image_analysis_b200.vmamba import CrossScan1b1
    B, C, H, W = shape
    x = torch.randn(B, 4, C, H, W, device="cuda").to(dt).requires_grad_()
    xr = x.detach().clone().requires_grad_()
    y, yr = CrossScan1b1.apply(x), _torch_1b1(xr)
    assert torch.equal(y, yr)
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g)
    assert torch.equal(x.grad, xr.grad)
    want = P1B1[shape][0 if dt == torch.float32 else 1]
    assert p1b1[f"{shape}|{dt}"] == [want, want]


# ---------------------------------------------------------------------------------------------------------- levels / saved
def _core_inputs(m, B, H, W, dtype, seed=3):
    """Leaf inputs of SS2DCoreFn at SS2D's shapes: x (B, D, H, W), and z as the second half of an in_proj-shaped buffer."""
    D = m.d_inner
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, H, W, generator=g).to(dtype).cuda().requires_grad_()
    buf = torch.randn(B, H, W, 2 * D, generator=g).to(dtype).cuda()
    z = buf[..., D:].detach().requires_grad_()
    return x, z


def _core(m, x, z, gate, lvl=1, out_float=True):
    from medical_image_analysis_b200.vmamba import ss2d_core
    return ss2d_core(x, z, m.x_proj_weight, m.dt_projs_weight, m.dt_projs_bias, m.A_logs, m.Ds, m.out_norm, gate, False, out_float,
                     checkpoint_lvl=lvl)


def _core_grads(m, x, z, gate, lvl):
    named = dict(x=x, z=z, **dict(m.named_parameters()))
    for t in named.values():
        t.grad = None
    out = _core(m, x, z, gate, lvl)
    out.float().pow(2).sum().backward()
    return out, {k: t.grad.clone() for k, t in named.items() if t.grad is not None}


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("N", [1, 16])
def test_checkpoint_levels_are_bit_identical(dtype, N):
    m = _module("v3", 128, N).to(dtype)
    x, z = _core_inputs(m, 2, 14, 14, dtype)
    o1, g1 = _core_grads(m, x, z, 2, 1)
    o0, g0 = _core_grads(m, x, z, 2, 0)
    assert torch.equal(o0, o1) and g0.keys() == g1.keys() and len(g1) == 9
    for k in g1:
        assert torch.equal(g0[k], g1[k]), k


@gpu
@pytest.mark.parametrize("lvl", [0, 1])
def test_level0_keeps_and_level1_recomputes(lvl, monkeypatch):
    """Level 0 takes xs and delta from what the forward kept: its backward runs no CrossScan of x; level 1 runs one."""
    from medical_image_analysis_b200 import vmamba
    m = _module("v3", 64, 1)
    x, z = _core_inputs(m, 2, 7, 9, torch.float32)
    calls = []
    real = vmamba.cross_scan_fwd
    monkeypatch.setattr(vmamba, "cross_scan_fwd", lambda t: calls.append(1) or real(t))
    out = _core(m, x, z, 2, lvl)
    assert len(calls) == 1
    out.float().sum().backward()
    assert len(calls) == 1 + lvl


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_inference_writes_only_the_output(dtype, monkeypatch):
    """Without grad mode the epilogue is given no pre-norm plane / statistics to write (nor the scan block states); the
    output is the same bits as with grad mode."""
    from medical_image_analysis_b200 import _lib
    m = _module("v3", 128, 1).to(dtype)
    x, z = _core_inputs(m, 2, 14, 14, dtype)
    seen = []
    real = _lib.call
    monkeypatch.setattr(_lib, "call", lambda name, *a: (seen.append((name, a)), real(name, *a))[1])
    ref = _core(m, x, z, 2)
    with torch.no_grad():
        out = _core(m, x, z, 2)
    epi = [a for name, a in seen if name == "mia_ss2d_merge_norm_fwd"]
    assert len(epi) == 2
    assert all(v is not None for v in epi[0][7:10]) and all(v is None for v in epi[1][7:10])   # yb, mean, rstd
    assert out.grad_fn is None and torch.equal(out, ref)


def _saved_bytes(fn, params):
    ptrs = {p.untyped_storage().data_ptr() for p in params}
    saved = {}

    def pack(t):
        st = t.untyped_storage()
        if st.data_ptr() not in ptrs:
            saved[st.data_ptr()] = st.nbytes()
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = fn()
    return sum(saved.values()), out


@gpu
@pytest.mark.parametrize("lvl", [0, 1])
def test_saved_tensor_bound(lvl):
    """Unique storages the op saves, parameters aside (module_timings shape, bf16): level 1 = x + Z + yb + mean / rstd + the
    scan checkpoints (+ block states) + z's storage; level 0 adds xs and delta (4 planes each).  Also below what the
    composition saves for the same layer."""
    from medical_image_analysis_b200 import scan_op
    B, H, W, N = 64, 14, 14, 1
    m = _module("v3noz", 768, N).bfloat16()
    D, L, K = m.d_inner, H * W, 4
    C = m.x_proj_weight.shape[1]
    x, _ = _core_inputs(m, B, H, W, torch.bfloat16)
    params = list(m.parameters())
    total, out = _saved_bytes(lambda: _core(m, x, None, 0, lvl), params)
    plane = B * D * L * 2
    ck = B * K * D * scan_op.num_chunks(L) * 2 * N * 4
    hblk = B * K * D * ((L + 15) // 16) * 4 * 2                         # block states: generous (<= 8 bytes per 16 tokens per row)
    small = 4 * (K * D * (2 * N + 2) + 2 * D)                            # fp32 A (and exp's result), D, delta_bias, LayerNorm w / b
    bound = plane + B * K * C * L * 2 + plane + 2 * B * L * 4 + ck + hblk + small
    if lvl == 0:
        bound += 2 * K * plane
    assert total <= bound, f"saved {total} bytes > bound {bound} (level {lvl})"
    out.float().sum().backward()
    # the composition at the same shape (SS2D v3noz without z: x is the conv output, as here)
    xc = x.detach().requires_grad_()
    from medical_image_analysis_b200.vmamba import _cross_selective_scan_composed
    comp, _ = _saved_bytes(lambda: _cross_selective_scan_composed(xc, m.x_proj_weight, None, m.dt_projs_weight, m.dt_projs_bias, m.A_logs,
                                                                  m.Ds, out_norm=m.out_norm), params)
    assert total < comp, (total, comp)


# ---------------------------------------------------------------------------------------------------------- kernel path
FULL_OPS = ("aten::copy_", "aten::cat", "aten::add", "aten::add_", "aten::mul", "aten::native_layer_norm", "aten::clone",
            "aten::contiguous", "aten::flip", "aten::stack")


def kernel_path():
    """Run in a child interpreter: kernels of the epilogue and aten ops on (B, D, L)-sized tensors, fwd and bwd."""
    res = {}
    m = _module("v3", 256, 1).bfloat16()
    B, H, W = 4, 14, 14
    x, z = _core_inputs(m, B, H, W, torch.bfloat16)
    torch.cuda.synchronize()
    out = None
    for phase in ("fwd", "bwd"):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                    record_shapes=True) as prof:
            if phase == "fwd":
                out = _core(m, x, z, 2)
            else:
                out.backward(torch.randn_like(out))
            torch.cuda.synchronize()
        big = []
        for e in prof.events():
            if e.name in FULL_OPS and any(shp and math.prod(shp) >= B * m.d_inner * H * W for shp in e.input_shapes):
                outer, p = [], e.cpu_parent
                while p is not None:
                    outer.append(p.name)
                    p = p.cpu_parent
                big.append(f"{e.name}{e.input_shapes[0]} in {outer}")
        kern = sorted({mm.group(1) for e in prof.events() for mm in [re.search(r"(merge_norm_\w+|cross_1b1_\w+)", e.name)] if mm})
        res[phase] = {"kernels": kern, "full_size_ops": big}
    return res


@gpu
def test_kernel_path():
    path = kernel_trace.in_child("tests.test_ss2d_core_fused_gpu:kernel_path")
    fwd, bwd = path["fwd"], path["bwd"]
    assert "merge_norm_fwd_kernel" in fwd["kernels"] and "cross_1b1_kernel" in fwd["kernels"], fwd
    assert {"merge_norm_bwd_kernel", "merge_norm_bwd_finalize", "cross_1b1_kernel"} <= set(bwd["kernels"]), bwd
    assert not fwd["full_size_ops"], fwd["full_size_ops"]
    # the one full-size copy left: torch's in-place baddbmm_ (dx += W_x^T dZ on the merge output) stages its result once
    assert len(bwd["full_size_ops"]) <= 1 and all("aten::baddbmm_" in op for op in bwd["full_size_ops"]), bwd["full_size_ops"]


def kernel_path_fp16():
    """Run in a child interpreter: the epilogue and CrossScan1b1 kernels of one VSSM forward + backward under fp16 autocast."""
    from medical_image_analysis_b200.vmamba import VSSM
    torch.manual_seed(0)
    model = VSSM(depths=[1], dims=[32], num_classes=10, drop_path_rate=0.0, forward_type="v3").cuda()
    x = torch.randn(2, 3, 32, 32, device="cuda")
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        with torch.autocast("cuda", dtype=torch.float16):
            out = model(x)
        out.float().sum().backward()
        torch.cuda.synchronize()
    rx = re.compile(r"\b(merge_norm_\w+?|cross_1b1_(?:direct_)?kernel)(?=[<(])")
    names = set()
    for e in prof.events():
        m = rx.search(e.name)
        if m:
            rest = e.name[m.end():]
            names.add(m.group(1) + (f"<{', '.join(kernel_trace.targs(e.name, m.group(1) + '<'))}>" if rest.startswith("<") else ""))
    return sorted(names)


@gpu
def test_kernel_path_fp16_autocast():
    """Under fp16 autocast the activations reach the op as fp16: the v3 core's fp32 scan output is merged into an fp16 output
    (merge_norm_fwd_kernel<float, __half>), the backward runs in fp16, and CrossScan1b1 moves fp16 planes."""
    names = kernel_trace.in_child("tests.test_ss2d_core_fused_gpu:kernel_path_fp16")
    assert "merge_norm_fwd_kernel<float, __half>" in names, names
    assert {"merge_norm_bwd_kernel<__half>", "merge_norm_bwd_finalize"} <= set(names), names
    assert any(n.startswith("cross_1b1_kernel<__half, ") for n in names), names


# ---------------------------------------------------------------------------------------------------------- determinism
@gpu
def test_deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    m = _module("v3", 256, 16).bfloat16()
    x, z = _core_inputs(m, 3, 14, 14, torch.bfloat16)
    o1, g1 = _core_grads(m, x, z, 2, 1)
    o2, g2 = _core_grads(m, x, z, 2, 1)
    for k in ("out_norm.weight", "out_norm.bias"):                             # always
        assert torch.equal(g1[k], g2[k]), k
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        o1, g1 = _core_grads(m, x, z, 2, 1)
        o2, g2 = _core_grads(m, x, z, 2, 1)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(o1, o2) and len(g1) == 9
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


# ---------------------------------------------------------------------------------------------------------- routing
ELIGIBLE = ["v2", "v3", "v4", "v3noz", "v4noz", "v3nozact", "v2no32"]
INELIGIBLE = [dict(forward_type=t) for t in ("v01", "v1", "v31d", "v32d", "v3none", "v3dwconv3", "v3softmax", "v3sigmoid", "v0",
                                             "xv1a")] + \
             [dict(forward_type="v3", channel_first=True), dict(forward_type="v3", act_layer=nn.GELU)]


@gpu
@pytest.mark.parametrize("kw", [dict(forward_type=t) for t in ELIGIBLE] + INELIGIBLE, ids=lambda kw: "-".join(map(str, kw.values())))
def test_routing(kw, monkeypatch):
    from medical_image_analysis_b200 import vmamba
    calls = []
    real = vmamba.SS2DCoreFn.apply
    monkeypatch.setattr(vmamba.SS2DCoreFn, "apply", lambda *a: calls.append(1) or real(*a))
    torch.manual_seed(0)
    m = vmamba.SS2D(d_model=16, d_state=2, **kw).cuda()
    x = torch.randn(2, 6, 5, 16, device="cuda")
    if kw.get("channel_first"):
        x = x.permute(0, 3, 1, 2).contiguous()
    # the dwconv3 out_norm is an fp32 Conv2d on the reference's bf16 cast of the merged output: it runs under autocast only
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=kw["forward_type"] == "v3dwconv3"):
        out = m(x)
    out.float().sum().backward()
    assert bool(calls) == (kw in [dict(forward_type=t) for t in ELIGIBLE]), (kw, calls)


# ---------------------------------------------------------------------------------------------------------- error paths
def _ptr():
    buf = ctypes.create_string_buffer(64)
    return buf, ctypes.cast(buf, ctypes.c_void_p).value


def test_epilogue_rejects_unsupported_sizes_before_any_launch():
    """Refused in the host checks (no device, null stream), through _lib.call."""
    from medical_image_analysis_b200 import _lib
    keep, p = _ptr()
    ln = _lib.MiaLn(p, p, 1e-5)
    none = _lib.MiaBdl(None, 0, 0, 0)
    args = lambda D, gate=0, B=1: (p, ctypes.byref(ln), ctypes.byref(none), gate, p, p, p, p, B, D, 14, 14, _lib.MIA_F32, _lib.MIA_BF16)
    with pytest.raises(RuntimeError, match=r"D = 4096 needs \d+ bytes of shared memory per block, more than the 232448-byte"):
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", None, *args(4096))
    with pytest.raises(RuntimeError, match="the gate needs z"):
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", None, *args(64, gate=2))
    with pytest.raises(RuntimeError, match="bad sizes"):
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", None, *args(64, B=0))
    with pytest.raises(RuntimeError, match="workspace missing or too small"):
        _lib.call("mia_ss2d_merge_norm_bwd", "ss2d_merge_norm_bwd", None, p, p, p, p, ctypes.byref(ln), ctypes.byref(none), 0,
                  ctypes.byref(none), p, p, p, p, 16, 2, 64, 14, 14, _lib.MIA_BF16)
    with pytest.raises(RuntimeError, match=r"D = 3627 needs 232576 bytes of shared memory per block, more than the 232448-byte"):
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", None, *args(3627))
    with pytest.raises(RuntimeError, match="yb, mean and rstd are all given or all NULL"):
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", None, p, ctypes.byref(ln), ctypes.byref(none), 0, p, None, p, p, 1, 64,
                  14, 14, _lib.MIA_F32, _lib.MIA_BF16)
    with pytest.raises(RuntimeError, match="1b1: tensor too large"):
        _lib.call("mia_cross_scan_1b1", "cross_scan_1b1", None, p, p, 65536, 65536, 32, 32, _lib.MIA_F32)
    with pytest.raises(RuntimeError, match="1b1: tensor too large"):          # B * 4 * C planes beyond int range at a tiny map
        _lib.call("mia_cross_merge_1b1", "cross_merge_1b1", None, p, p, 1 << 29, 1, 1, 1, _lib.MIA_F32)


@gpu
def test_fused_op_rejects_wrong_shapes():
    m = _module("v3", 64, 1)
    x, z = _core_inputs(m, 2, 6, 5, torch.float32)
    with pytest.raises(RuntimeError, match="z must be"):
        _core(m, x, z[:, :, :4], 2)
    with pytest.raises(RuntimeError, match="do not fit"):
        _core(m, x[:, :32], None, 0)
    with pytest.raises(ValueError, match="checkpoint_lvl"):
        _core(m, x, None, 0, lvl=2)
