"""The GELU MLP as one op (gemm.GeluMlpFn / gelu_mlp_fn): fc1's pre-activation and GELU against gemm.linear and F.gelu, the
backward epilogue against a float64 statement over every representable pre-activation in [-8, 8], the routed vmamba / mae
Mlp against the composition it replaces (Mlp._forward_composed), the whole op against float64, checkpoint levels, the
saved-tensor bound, the kernel path, routing and determinism."""
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import kernel_trace

pytestmark = pytest.mark.gpu

SHAPES = [(64, 202), (128, 512), (512, 2048), (1024, 4096)]       # (in, H): H = 202 is not a multiple of 8 (padded pitches)
DTYPES = [torch.bfloat16, torch.float16]
MS = [197 * 3, 61 * 5, 1]


def _lib():
    from medical_image_analysis_b200 import _lib
    return _lib


def _pad8(n):
    return (n + 7) // 8 * 8


def _fwd_kernel(x, w1, b1, with_pre=True):
    """mia_gemm_gelu_fwd on NaN-filled outputs -> (h (M, Hp), pre (M, Hp) or None), pad columns included."""
    lib = _lib()
    M, K = x.shape
    H, Hp = w1.shape[0], _pad8(w1.shape[0])
    h = torch.full((M, Hp), float("nan"), dtype=x.dtype, device="cuda")
    pre = torch.full((M, Hp), float("nan"), dtype=x.dtype, device="cuda") if with_pre else None
    b1f = None if b1 is None else b1.float().contiguous()
    lib.call("mia_gemm_gelu_fwd", "gelu_fwd", x.device, x.data_ptr(), w1.data_ptr(), None if b1f is None else b1f.data_ptr(), h.data_ptr(),
             None if pre is None else pre.data_ptr(), M, H, K, x.stride(0), w1.stride(0), h.stride(0), 0 if pre is None else pre.stride(0),
             lib.dtype_code(x.dtype))
    return h, pre


def _bwd_kernel(dy, w2, pre, H):
    """mia_gemm_gelu_bwd -> (dpre (M, Hp), h (M, Hp)); w2 (N, ldw2 >= H) with a pitch that is a multiple of 8."""
    lib = _lib()
    M, N = dy.shape
    Hp = _pad8(H)
    dpre = torch.full((M, Hp), float("nan"), dtype=dy.dtype, device="cuda")
    h = torch.full((M, Hp), float("nan"), dtype=dy.dtype, device="cuda")
    lib.call("mia_gemm_gelu_bwd", "gelu_bwd", dy.device, dy.data_ptr(), w2.data_ptr(), pre.data_ptr(), dpre.data_ptr(), h.data_ptr(), M, H, N,
             dy.stride(0), w2.stride(0), pre.stride(0), dpre.stride(0), h.stride(0), lib.dtype_code(dy.dtype))
    return dpre, h


def _ulp(v, dtype):
    """One unit in the last place of dtype at |v| (float64)."""
    mant, tiny = (7, 2.0 ** -133) if dtype == torch.bfloat16 else (10, 2.0 ** -24)
    e = torch.floor(torch.log2(v.abs().clamp_min(tiny)))
    return (2.0 ** (e - mant)).clamp_min(tiny)


def _within_ulp(got, ref, what):
    got64 = got.double()
    tol = torch.maximum(_ulp(ref, got.dtype), _ulp(got64, got.dtype))
    bad = (got64 - ref).abs() > tol
    assert torch.isfinite(got64).all(), what
    assert not bad.any(), f"{what}: {int(bad.sum())} elements more than 1 ulp off, e.g. got {got64[bad][:4].tolist()} want {ref[bad][:4].tolist()}"


def _dgelu64(p):
    """gelu'(p) = Phi(p) + p phi(p) in float64."""
    return 0.5 * torch.erfc(-p * 0.5 ** 0.5) + p * torch.exp(-0.5 * p * p) * (2 * torch.pi) ** -0.5


# ---------------------------------------------------------------------------------------------------------- fc1 epilogue
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_pre_and_h_are_gemm_linear_and_f_gelu_bit_for_bit(shape, dtype, M, bias):
    """pre is what gemm.linear writes for fc1(x) (the same k order and fp32 bias add, rounded once) and h is F.gelu(pre);
    pad columns of both are exactly zero; without pre (inference) h has the same bits."""
    from medical_image_analysis_b200 import gemm
    K, H = shape
    g = torch.Generator().manual_seed(K + M)
    w1 = (torch.randn(H, K, generator=g) * K ** -0.5).cuda().to(dtype)
    b1 = (torch.randn(H, generator=g) * 0.5).cuda().to(dtype) if bias else None
    x = torch.randn(M, K, generator=g).cuda().to(dtype)
    h, pre = _fwd_kernel(x, w1, b1)
    assert torch.equal(pre[:, :H], gemm.linear(x, w1, b1))
    assert torch.equal(h[:, :H], F.gelu(pre[:, :H]))
    assert (pre[:, H:] == 0).all() and (h[:, H:] == 0).all()
    h_inf, none = _fwd_kernel(x, w1, b1, with_pre=False)
    assert none is None and torch.equal(h_inf, h)


# ---------------------------------------------------------------------------------------------------------- fc2-dgrad epilogue
def _rank1(M, N, H, dtype, g):
    """dy (M, N) and W2 (N, Hp) with one non-zero k: g = dy[:, 0] W2[0, :] is exact in fp32, a given fp64 g."""
    u = torch.zeros(M, N, dtype=dtype)
    u[:, 0] = torch.randn(M, generator=g)
    w2 = torch.zeros(N, _pad8(H), dtype=dtype)
    w2[0, :H] = torch.randn(H, generator=g)
    return u.cuda(), w2.cuda()


def _check_bwd(dy, w2, pre, H, what):
    dpre, h = _bwd_kernel(dy, w2, pre, H)
    gg = dy[:, :1].double() * w2[:1, :H].double()
    p = pre[:, :H].double()
    _within_ulp(dpre[:, :H], gg * _dgelu64(p), f"{what} dpre")
    assert (dpre[:, H:] == 0).all(), what
    assert (h[:, H:] == 0).all(), what
    return h


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_bwd_epilogue_against_float64(shape, M, dtype):
    """dpre from the backward epilogue is within 1 ulp of float64 for a given g and pre (here pre over a wide range, 3 N(0, 1));
    its pad columns are zero; the recomputed h is the forward's, bit for bit."""
    K, H = shape
    N = K
    g = torch.Generator().manual_seed(H + M)
    w1 = (torch.randn(H, K, generator=g) * K ** -0.5).cuda().to(dtype)
    b1 = (torch.randn(H, generator=g) * 0.5).cuda().to(dtype)
    x = torch.randn(M, K, generator=g).cuda().to(dtype)
    h_fwd, pre = _fwd_kernel(x, w1, b1)
    dy, w2 = _rank1(M, N, H, dtype, g)
    assert torch.equal(_check_bwd(dy, w2, pre, H, "fc1 pre"), h_fwd)
    wide = pre.clone()
    wide[:, :H] = (torch.randn(M, H, generator=g) * 3).cuda().to(dtype)
    _check_bwd(dy, w2, wide, H, "wide pre")


def _all_values(dtype, lo=-8.0, hi=8.0):
    """Every finite value of dtype in [lo, hi] (one zero)."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype).float()
    return torch.unique(v[torch.isfinite(v) & (v >= lo) & (v <= hi)]).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_bwd_epilogue_sweep_of_every_pre_in_range(dtype):
    """Every representable pre in [-8, 8], which covers gelu''s root at -0.7518 (fp64 repair) and the negative tail (Phi from
    erfc): dpre within 1 ulp of float64, and the epilogue's h equals F.gelu(pre) bit for bit at every one of them."""
    H = 202
    vals = _all_values(dtype)
    M = -(-vals.numel() // H)
    g = torch.Generator().manual_seed(7)
    flat = torch.zeros(M * H, dtype=dtype)
    flat[:vals.numel()] = vals
    pre = torch.zeros(M, _pad8(H), dtype=dtype)
    pre[:, :H] = flat.view(M, H)
    pre = pre.cuda()
    dy, w2 = _rank1(M, 64, H, dtype, g)
    h = _check_bwd(dy, w2, pre, H, f"sweep of {vals.numel()} values")
    assert torch.equal(h[:, :H], F.gelu(pre[:, :H]))


# ---------------------------------------------------------------------------------------------------------- routed modules
def _vmamba_mlp(K, H, seed, dtype=torch.float32):
    from medical_image_analysis_b200.vmamba import Mlp
    torch.manual_seed(seed)
    m = Mlp(K, H).cuda()
    with torch.no_grad():                                              # non-zero biases of a realistic scale
        for lin in (m.fc1, m.fc2):
            lin.bias.normal_(0, 0.2)
    return m.to(dtype)


def _mae_mlp(K, H, seed, dtype=torch.float32):
    from medical_image_analysis_b200.mae import Mlp
    torch.manual_seed(seed)
    m = Mlp(K, H).cuda()
    with torch.no_grad():
        for lin in (m.fc1, m.fc2):
            lin.bias.normal_(0, 0.2)
    return m.to(dtype)


@pytest.mark.parametrize("mode", ["bf16", "f16", "autocast"])
@pytest.mark.parametrize("family", ["vmamba", "mae"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_routed_forward_is_the_composition_bit_for_bit(shape, family, mode):
    """In training mode (a backward follows) the routed Mlp writes what _forward_composed writes, bit for bit."""
    from medical_image_analysis_b200 import gemm
    K, H = shape
    dtype = {"bf16": torch.bfloat16, "f16": torch.float16, "autocast": torch.float32}[mode]
    m = (_vmamba_mlp if family == "vmamba" else _mae_mlp)(K, H, 4, dtype)
    m.train()
    x = torch.randn(3, 197, K, device="cuda", dtype=dtype, requires_grad=True)
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "autocast" else torch.autocast("cuda", enabled=False)
    with ctx:
        assert gemm.gelu_mlp_eligible(m, x, True)
        out, comp = m(x), m._forward_composed(x)
    assert out.dtype == comp.dtype and torch.equal(out, comp)


def _grads(m, x, fn, w):
    m.zero_grad()
    x = x.detach().clone().requires_grad_()
    out = fn(m, x)
    (out.float() * w).sum().backward()
    return out.detach(), {"x": x.grad, **{n: p.grad.clone() for n, p in m.named_parameters()}}


def _ref64(m, x, w):
    """float64 statement of fc2(gelu(fc1(x))) on CPU."""
    P = {n: p.detach().double().cpu().requires_grad_() for n, p in m.named_parameters()}
    x64 = x.detach().double().cpu().requires_grad_()
    out = F.linear(F.gelu(F.linear(x64, P["fc1.weight"], P["fc1.bias"])), P["fc2.weight"], P["fc2.bias"])
    (out * w.double().cpu()).sum().backward()
    return out, {"x": x64.grad, **{n: p.grad for n, p in P.items()}}


def _rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    rms = ref.pow(2).mean().sqrt().item() + 1e-30
    err = (got - ref).abs()
    return err.pow(2).mean().sqrt().item() / rms, err.max().item() / rms


@pytest.mark.parametrize("mode", ["bf16", "f16", "autocast"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_whole_op_no_further_than_the_composition(shape, mode):
    """bf16 / fp16 parameters, or bf16 autocast over fp32 ones: output, dx and the four weight / bias gradients against a
    float64 evaluation on the same inputs, within the fused ops' bf16 criterion, and no further from it than the
    composition (which rounds the hidden gradient and then dpre), up to 25 % of its error."""
    K, H = shape
    dtype = {"bf16": torch.bfloat16, "f16": torch.float16, "autocast": torch.float32}[mode]
    m = _vmamba_mlp(K, H, 12, dtype)
    T = torch.float16 if mode == "f16" else torch.bfloat16
    x = torch.randn(2, 197, K, device="cuda").to(T)
    w = torch.randn(2, 197, K, device="cuda")
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "autocast" else torch.autocast("cuda", enabled=False)
    with ctx:
        out, grads = _grads(m, x, lambda m, x: m(x), w)
        cout, cgrads = _grads(m, x, lambda m, x: m._forward_composed(x), w)
    assert out.dtype == T
    ref, rgrads = _ref64(m, x, w)
    assert set(grads) == set(rgrads) == {"x", "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias"}
    for k, (got, comp, r) in {"out": (out, cout, ref), **{k: (grads[k], cgrads[k], rgrads[k]) for k in grads}}.items():
        assert got.dtype == comp.dtype, k
        rel, worst = _rel(got, r)
        crel, cworst = _rel(comp, r)
        assert rel <= 0.02 and worst <= 0.5, f"{k}: rel RMS err {rel:.3e}, worst err / RMS(ref) {worst:.3e}"
        assert rel <= 1.25 * crel + 1e-4, f"{k}: rel RMS err {rel:.3e}, the composition's {crel:.3e}"


# ---------------------------------------------------------------------------------------------------------- levels and memory
def _op_inputs(K, H, dtype, bias=True, seed=5, b=3, L=197):
    g = torch.Generator().manual_seed(seed)
    P = dict(x=torch.randn(b, L, K, generator=g), w1=torch.randn(H, K, generator=g) * K ** -0.5, b1=torch.randn(H, generator=g) * 0.2,
             w2=torch.randn(K, H, generator=g) * H ** -0.5, b2=torch.randn(K, generator=g) * 0.2)
    if not bias:
        P = {k: v for k, v in P.items() if not k.startswith("b")}
    return {k: v.cuda().to(dtype).requires_grad_() for k, v in P.items()}


def _op(P, **kw):
    from medical_image_analysis_b200.gemm import gelu_mlp_fn
    return gelu_mlp_fn(P["x"], P["w1"], P.get("b1"), P["w2"], P.get("b2"), **kw)


def _op_run(P, seed=9, **kw):
    for v in P.values():
        v.grad = None
    out = _op(P, **kw)
    out.backward(torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).to(out.device, out.dtype))
    return out.detach(), {k: v.grad.clone() for k, v in P.items()}


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_checkpoint_levels_are_bit_identical(shape, dtype, bias):
    P = _op_inputs(*shape, dtype, bias)
    o0, g0 = _op_run(P, checkpoint_lvl=0)
    o1, g1 = _op_run(P, checkpoint_lvl=1)
    o2, g2 = _op_run(P, checkpoint_lvl=0)
    assert torch.equal(o0, o1) and torch.equal(o0, o2)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
        assert torch.equal(g0[k], g2[k]), k
    with pytest.raises(ValueError):
        _op(P, checkpoint_lvl=2)


def test_autocast_over_fp32_parameters_levels():
    P = _op_inputs(512, 2048, torch.float32)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        o0, g0 = _op_run(P, checkpoint_lvl=0)
        o1, g1 = _op_run(P, checkpoint_lvl=1)
    assert o0.dtype == torch.bfloat16 and torch.equal(o0, o1)
    for k in g0:
        assert g0[k].dtype == torch.float32 and torch.equal(g0[k], g1[k]), k


def _saved_bytes(fn, exclude):
    ptrs = {t.untyped_storage().data_ptr() for t in exclude}
    saved = {}

    def pack(t):
        st = t.untyped_storage()
        if st.data_ptr() not in ptrs:
            saved[st.data_ptr()] = st.nbytes()
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = fn()
    return sum(saved.values()), out


@pytest.mark.parametrize("shape", [(512, 2048), (64, 202)], ids=["in512_H2048", "in64_H202"])
def test_saved_tensor_bound(shape):
    """Parameters aside, level 0 keeps x and pre (M Hp elements), level 1 x only; both less than the composition.  Under
    no_grad, or with nothing requiring a gradient, no pre buffer is allocated."""
    from medical_image_analysis_b200.gemm import gelu_mlp_fn
    K, H = shape
    Hp = _pad8(H)
    m = _vmamba_mlp(K, H, 3, torch.bfloat16)
    x = torch.randn(8, 197, K, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    M = x.shape[0] * x.shape[1]
    params = list(m.parameters())
    args = lambda: (x, m.fc1.weight, m.fc1.bias, m.fc2.weight, m.fc2.bias)
    s0, out = _saved_bytes(lambda: gelu_mlp_fn(*args(), checkpoint_lvl=0), params)
    out.float().sum().backward()
    s1, out = _saved_bytes(lambda: gelu_mlp_fn(*args(), checkpoint_lvl=1), params)
    out.float().sum().backward()
    comp, out = _saved_bytes(lambda: m._forward_composed(x), params)
    print(f"saved bytes: level 0 {s0}, level 1 {s1}, composition {comp}")
    assert s0 <= x.nbytes + M * Hp * 2, s0
    assert s1 <= x.nbytes, s1
    assert s0 < comp and s1 < comp

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        y = fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, y

    h_bytes, y_bytes = M * Hp * 2, M * K * 2
    with torch.no_grad():
        p_ng, y = peak(lambda: gelu_mlp_fn(*args()))
    xd = x.detach()
    with torch.no_grad():
        for p in params:
            p.requires_grad_(False)
    try:
        p_nr, y2 = peak(lambda: gelu_mlp_fn(xd, *args()[1:]))
    finally:
        for p in params:
            p.requires_grad_(True)
    assert torch.equal(y, y2)
    w2_pad = K * Hp * 2 if H % 8 else 0                                # W2 zero-padded to an aligned pitch
    for p_ in (p_ng, p_nr):                                            # h, the output and W2's pad copy; no pre buffer
        assert p_ <= h_bytes + y_bytes + w2_pad + (1 << 20), (p_, h_bytes, y_bytes, w2_pad)


# ---------------------------------------------------------------------------------------------------------- kernel path
BIG_OPS = ("aten::gelu", "aten::gelu_backward", "aten::erf", "aten::exp", "aten::mul", "aten::add", "aten::add_", "aten::copy_")
GELU = re.compile(r"\bgemm_gelu_kernel<(\d)")
GEMM = re.compile(r"\bgemm_tn_kernel<")
REDUCE = re.compile(r"reduce_kernel")


def _want(lvl, phase):
    if phase == "fwd":
        return {"gelu_fwd": 1, "gemm": 1}
    want = {"gelu_bwd": 1, "gemm": 3, "reduce": 2}
    if lvl == 1:
        want["gelu_fwd"] = 1                                           # pre (and h) recomputed by the forward kernel
    return want


def _capture(lvl, phase, K, H, b):
    """One profiled fwd or bwd of a fresh op -> kernel launch counts and (M, H)-sized aten ops."""
    M = b * 197
    P = _op_inputs(K, H, torch.bfloat16, b=b)
    out = dout = None
    if phase == "bwd":
        out = _op(P, checkpoint_lvl=lvl)
        dout = torch.randn_like(out)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                record_shapes=True) as prof:
        if phase == "fwd":
            _op(P, checkpoint_lvl=lvl)
        else:
            out.backward(dout)
        torch.cuda.synchronize()
    big, counts = [], {}
    for e in prof.events():
        if e.name in BIG_OPS:
            for shp in e.input_shapes:
                n = 1
                for s in shp:
                    n *= s
                if shp and n >= M * H:
                    big.append(f"{e.name}{shp}")
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = GELU.search(e.name)
            key = ("gelu_fwd" if m.group(1) == "3" else "gelu_bwd") if m else ("gemm" if GEMM.search(e.name) else
                                                                             ("reduce" if REDUCE.search(e.name) else None))
            if key:
                counts[key] = counts.get(key, 0) + 1
    return {"counts": counts, "big_ops": big}


def kernel_path():
    """Run in a child interpreter: kernel launch counts and (M, H)-sized aten ops, fwd and bwd separately, per level.  A
    capture missing expected launches is taken again (kernel_trace.retry); the last capture is returned either way."""
    res = {}
    for lvl in (0, 1):
        for phase in ("fwd", "bwd"):
            want = _want(lvl, phase)
            res[f"{lvl}/{phase}"] = kernel_trace.retry(lambda: _capture(lvl, phase, 512, 2048, 16),
                                                       lambda r: all(r["counts"].get(k, 0) >= n for k, n in want.items()))
    return res


@pytest.fixture(scope="module")
def path():
    return kernel_trace.in_child("tests.test_gelu_mlp_fused_gpu:kernel_path")


@pytest.mark.parametrize("lvl", [0, 1])
def test_kernel_path(path, lvl):
    fwd, bwd = path[f"{lvl}/fwd"], path[f"{lvl}/bwd"]
    assert fwd["counts"] == _want(lvl, "fwd"), fwd
    assert bwd["counts"] == _want(lvl, "bwd"), bwd
    assert not fwd["big_ops"], fwd["big_ops"]
    assert not bwd["big_ops"], bwd["big_ops"]


# ---------------------------------------------------------------------------------------------------------- routing
@pytest.fixture
def op_calls(monkeypatch):
    from medical_image_analysis_b200 import gemm
    calls = []
    real = gemm.gelu_mlp_fn

    def spy(*a, **k):
        calls.append(a[0].shape)
        return real(*a, **k)

    monkeypatch.setattr(gemm, "gelu_mlp_fn", spy)
    return calls


def test_blocks_take_the_op(op_calls):
    from medical_image_analysis_b200.mae import Block
    from medical_image_analysis_b200.vmamba import VSSBlock
    torch.manual_seed(0)
    blk = VSSBlock(hidden_dim=64, ssm_d_state=16, ssm_ratio=1.0, forward_type="v2", mlp_ratio=4.0).cuda()
    x = torch.randn(2, 14, 14, 64, device="cuda", requires_grad=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        blk(x).float().sum().backward()
    assert len(op_calls) == 1
    vit = Block(64, 4, 4.0, qkv_bias=True).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        vit(torch.randn(2, 61, 64, device="cuda", requires_grad=True)).float().sum().backward()
    assert len(op_calls) == 2


def test_other_cases_take_the_composition(op_calls):
    from medical_image_analysis_b200 import mae, vmamba
    torch.manual_seed(0)
    x = torch.randn(2, 17, 64, device="cuda", requires_grad=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        vmamba.Mlp(64, 256).cuda()(x)
        assert len(op_calls) == 1
        vmamba.Mlp(64, 256, drop=0.1).cuda().eval()(x)                   # inactive dropout: the op
        assert len(op_calls) == 2
        vmamba.Mlp(64, 256, channels_first=True).cuda()(x.permute(0, 2, 1)[..., None].contiguous())   # Linear2d
        vmamba.Mlp(64, 256, act_layer=lambda: nn.GELU(approximate="tanh")).cuda()(x)
        vmamba.Mlp(64, 256, act_layer=nn.ReLU).cuda()(x)
        vmamba.Mlp(64, 256, drop=0.1).cuda().train()(x)
        with torch.no_grad():
            vmamba.Mlp(64, 256).cuda()(x)
            mae.Mlp(64, 256).cuda()(x)
        vmamba.Mlp(64, 256).cuda().requires_grad_(False)(x.detach())   # nothing to differentiate
    vmamba.Mlp(64, 256).cuda()(x)                                      # fp32 activations: the library path, as gemm.linear
    mae.Mlp(64, 256).cuda()(x)
    assert len(op_calls) == 2


def _two_runs(model, run):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        runs = []
        for _ in range(2):
            model.zero_grad()
            y = run()
            runs.append((y.detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(runs[0][0], runs[1][0])
    assert runs[0][1].keys() == runs[1][1].keys()
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k
    return runs[0][1]


def test_vssm_routing_and_determinism(op_calls, monkeypatch):
    """A small VSSM under bf16 autocast runs the op in every block; its fwd + bwd is bit-reproducible."""
    from medical_image_analysis_b200.vmamba import VSSM
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.manual_seed(0)
    model = VSSM(depths=[1, 2], dims=[32, 64], num_classes=10, drop_path_rate=0.0).cuda()
    img = torch.randn(2, 3, 64, 64, device="cuda")

    def run():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = model(img)
        y.float().square().mean().backward()
        return y

    grads = _two_runs(model, run)
    assert len(op_calls) == 2 * 3
    assert any(k.endswith("mlp.fc1.weight") for k in grads)


def test_mae_routing_and_determinism(op_calls, monkeypatch):
    """A small MaskedAutoencoderViT under bf16 autocast runs the op in every encoder and decoder block; its fwd + bwd is
    bit-reproducible (attention on SDPA's math backend: the cuDNN one has no deterministic backward)."""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from medical_image_analysis_b200.mae import MaskedAutoencoderViT
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.manual_seed(0)
    net = MaskedAutoencoderViT(embed_dim=64, depth=2, num_heads=2, decoder_embed_dim=32, decoder_depth=1, decoder_num_heads=2,
                               patch_embed_dims=(1, 64, 32)).cuda()
    img = torch.randn(1, 1, 1280, 1280, device="cuda")
    noise = torch.rand(1, 400, device="cuda")

    def run():
        with torch.autocast("cuda", dtype=torch.bfloat16), sdpa_kernel(SDPBackend.MATH):
            loss, _ = net(img, 0, 0.85, 0.95, noise=noise)
        loss.mean().backward()
        return loss

    grads = _two_runs(net, run)
    assert len(op_calls) == 2 * 3
    assert any(k.endswith("mlp.fc1.weight") for k in grads)
