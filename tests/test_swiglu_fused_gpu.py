"""ARM's SwiGLU MLP as one op (arm.SwiGLUFn / swiglu_fn): the dual GEMM's a / b against gemm.linear, both epilogues against
float64 statements, the whole op against a float64 statement of the module and against the composition it replaces
(SwiGLU._forward_composed), checkpoint levels, the saved-tensor bound, the kernel path, determinism and routing."""
import re

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_trace

pytestmark = pytest.mark.gpu

SHAPES = [(64, 176), (768, 2048), (1024, 2730)]                      # (in, H): a small H, arm_base, arm_large (H % 8 != 0)
DTYPES = [torch.bfloat16, torch.float16]
MS = [2 * 197, 3 * 197, 1]


def _lib():
    from medical_image_analysis_b200 import _lib
    return _lib


def _pad64(n):
    return (n + 63) // 64 * 64


def _weights(K, H, dtype, bias, seed):
    g = torch.Generator().manual_seed(seed)
    w1, w2 = (torch.randn(H, K, generator=g) * K ** -0.5 for _ in range(2))
    b1, b2 = (torch.randn(H, generator=g) * 0.5 if bias else None for _ in range(2))
    cast = lambda t: None if t is None else t.cuda().to(dtype)
    return cast(w1), cast(b1), cast(w2), cast(b2)


def _fwd_kernel(x, w1, b1, w2, b2, with_ab=True):
    """mia_gemm_swiglu_fwd on NaN-filled outputs -> (h (M, H), ab (M, 2 Hp) or None)."""
    lib = _lib()
    M, K = x.shape
    H, Hp = w1.shape[0], _pad64(w1.shape[0])
    h = torch.full((M, Hp), float("nan"), dtype=x.dtype, device="cuda")
    ab = torch.full((M, 2 * Hp), float("nan"), dtype=x.dtype, device="cuda") if with_ab else None
    f32 = lambda t: None if t is None else t.float().contiguous()
    b1f, b2f = f32(b1), f32(b2)
    lib.call("mia_gemm_swiglu_fwd", "swiglu_fwd", x.device, x.data_ptr(), w1.data_ptr(), w2.data_ptr(), None if b1f is None else b1f.data_ptr(),
             None if b2f is None else b2f.data_ptr(), h.data_ptr(), None if ab is None else ab.data_ptr(), M, H, K, x.stride(0), w1.stride(0),
             w2.stride(0), h.stride(0), 0 if ab is None else ab.stride(0), lib.dtype_code(x.dtype))
    return h[:, :H], ab


def _bwd_kernel(dy, w3, ab, H):
    """mia_gemm_swiglu_bwd -> (dab (M, 2 Hp), h (M, H)); w3 (N, ldw3 >= H) with a pitch that is a multiple of 8."""
    lib = _lib()
    M, N = dy.shape
    Hp = _pad64(H)
    dab = torch.full((M, 2 * Hp), float("nan"), dtype=dy.dtype, device="cuda")
    h = torch.full((M, Hp), float("nan"), dtype=dy.dtype, device="cuda")
    lib.call("mia_gemm_swiglu_bwd", "swiglu_bwd", dy.device, dy.data_ptr(), w3.data_ptr(), ab.data_ptr(), dab.data_ptr(), h.data_ptr(), M, H, N,
             dy.stride(0), w3.stride(0), ab.stride(0), dab.stride(0), h.stride(0), lib.dtype_code(dy.dtype))
    return dab, h[:, :H]


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


# ---------------------------------------------------------------------------------------------------------- dual GEMM
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_ab_is_gemm_linear_bit_for_bit(shape, dtype, M, bias):
    """a / b are what gemm.linear writes for w1(x) / w2(x): the same k order and the same fp32 bias add, rounded once.
    h is silu(a) b from those rounded values, within 1 ulp of float64; pad columns are exactly zero."""
    from medical_image_analysis_b200 import gemm
    K, H = shape
    Hp = _pad64(H)
    w1, b1, w2, b2 = _weights(K, H, dtype, bias, seed=K + M)
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).cuda().to(dtype)
    h, ab = _fwd_kernel(x, w1, b1, w2, b2)
    assert torch.equal(ab[:, :H], gemm.linear(x, w1, b1))
    assert torch.equal(ab[:, Hp:Hp + H], gemm.linear(x, w2, b2))
    assert (ab[:, H:Hp] == 0).all() and (ab[:, Hp + H:] == 0).all()
    a, b = ab[:, :H].double(), ab[:, Hp:Hp + H].double()
    _within_ulp(h, a * torch.sigmoid(a) * b, "h")
    h_inf, none = _fwd_kernel(x, w1, b1, w2, b2, with_ab=False)          # inference: h only, the same bits
    assert none is None and torch.equal(h_inf, h)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"in{s[0]}_H{s[1]}" for s in SHAPES])
def test_bwd_epilogue_against_float64(shape, M, dtype):
    """g = dy . W3 with one non-zero k, so g = dy[:, 0] W3[0, :] is exact in fp32: a given g.  da, db and h from the
    backward epilogue are within 1 ulp of float64; dab's pad columns are exactly zero; the recomputed h is the forward's."""
    K, H = shape
    Hp = _pad64(H)
    N = K
    g = torch.Generator().manual_seed(H + M)
    w1, b1, w2, b2 = _weights(K, H, dtype, True, seed=H)
    x = torch.randn(M, K, generator=g).cuda().to(dtype)
    h_fwd, ab = _fwd_kernel(x, w1, b1, w2, b2)
    ab[:, :H] = (torch.randn(M, H, generator=g) * 3).cuda().to(dtype)     # also a wide range of a: sigmoid saturates
    ab[:, Hp:Hp + H] = torch.randn(M, H, generator=g).cuda().to(dtype)
    u = torch.zeros(M, N, dtype=dtype)
    u[:, 0] = torch.randn(M, generator=g)
    w3 = torch.zeros(N, _pad64(H), dtype=dtype)
    w3[0, :H] = torch.randn(H, generator=g)
    dy, w3 = u.cuda(), w3.cuda()
    dab, h = _bwd_kernel(dy, w3, ab, H)
    gg = dy[:, :1].double() * w3[:1, :H].double()
    a, b = ab[:, :H].double(), ab[:, Hp:Hp + H].double()
    s = torch.sigmoid(a)
    _within_ulp(dab[:, :H], gg * b * s * (1 + a * (1 - s)), "da")
    _within_ulp(dab[:, Hp:Hp + H], gg * a * s, "db")
    _within_ulp(h, a * s * b, "h")
    assert (dab[:, H:Hp] == 0).all() and (dab[:, Hp + H:] == 0).all()
    _, ab = _fwd_kernel(x, w1, b1, w2, b2)                                # untouched a / b: the bwd h is the fwd h, bit for bit
    assert torch.equal(_bwd_kernel(dy, w3, ab, H)[1], h_fwd)


# ---------------------------------------------------------------------------------------------------------- whole op
def _mlp(K, H, seed, dtype=torch.float32):
    from medical_image_analysis_b200.arm import SwiGLU
    torch.manual_seed(seed)
    m = SwiGLU(K, H).cuda()
    with torch.no_grad():                                              # non-zero biases (nn.Linear's init) and a third scale
        for lin in (m.w1, m.w2, m.w3):
            lin.bias.normal_(0, 0.2)
    return m.to(dtype)


def _grads(m, x, fn, w):
    m.zero_grad()
    x = x.detach().clone().requires_grad_()
    out = fn(m, x)
    (out.float() * w).sum().backward()
    return out.detach(), {"x": x.grad, **{n: p.grad.clone() for n, p in m.named_parameters()}}


def _ref64(m, x, w):
    """float64 statement of the module (models_mamba.py:59-83, subln False) on CPU."""
    P = {n: p.detach().double().cpu().requires_grad_() for n, p in m.named_parameters()}
    x64 = x.detach().double().cpu().requires_grad_()
    hidden = F.silu(F.linear(x64, P["w1.weight"], P["w1.bias"])) * F.linear(x64, P["w2.weight"], P["w2.bias"])
    out = F.linear(hidden, P["w3.weight"], P["w3.bias"])
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
    """bf16 / fp16 parameters, or bf16 autocast over fp32 ones: output, dx and the six weight / bias gradients against a
    float64 evaluation on the same inputs, within the fused mixers' bf16 criterion, and no further from it than the
    composition (which rounds w1(x), silu(w1(x)), the product and the hidden gradient separately), up to 25 % of its error."""
    K, H = shape
    dtype = {"bf16": torch.bfloat16, "f16": torch.float16, "autocast": torch.float32}[mode]
    m = _mlp(K, H, 12, dtype)
    T = torch.float16 if mode == "f16" else torch.bfloat16
    x = torch.randn(2, 197, K, device="cuda").to(T)
    w = torch.randn(2, 197, K, device="cuda")
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "autocast" else torch.autocast("cuda", enabled=False)
    with ctx:
        assert m._fused_ok(x)
        out, grads = _grads(m, x, lambda m, x: m(x), w)
        cout, cgrads = _grads(m, x, lambda m, x: m._forward_composed(x), w)
    assert out.dtype == T
    ref, rgrads = _ref64(m, x, w)
    assert set(grads) == set(rgrads) == {"x", "w1.weight", "w1.bias", "w2.weight", "w2.bias", "w3.weight", "w3.bias"}
    for k, (got, comp, r) in {"out": (out, cout, ref), **{k: (grads[k], cgrads[k], rgrads[k]) for k in grads}}.items():
        assert got.dtype == comp.dtype, k
        rel, worst = _rel(got, r)
        crel, cworst = _rel(comp, r)
        assert rel <= 0.02 and worst <= 0.5, f"{k}: rel RMS err {rel:.3e}, worst err / RMS(ref) {worst:.3e}"
        assert rel <= 1.25 * crel + 1e-4, f"{k}: rel RMS err {rel:.3e}, the composition's {crel:.3e}"


def _op_inputs(K, H, dtype, bias=True, seed=5):
    g = torch.Generator().manual_seed(seed)
    P = dict(x=torch.randn(3, 197, K, generator=g), w1=torch.randn(H, K, generator=g) * K ** -0.5, b1=torch.randn(H, generator=g) * 0.2,
             w2=torch.randn(H, K, generator=g) * K ** -0.5, b2=torch.randn(H, generator=g) * 0.2, w3=torch.randn(K, H, generator=g) * H ** -0.5,
             b3=torch.randn(K, generator=g) * 0.2)
    if not bias:
        P = {k: v for k, v in P.items() if not k.startswith("b")}
    return {k: v.cuda().to(dtype).requires_grad_() for k, v in P.items()}


def _op(P, **kw):
    from medical_image_analysis_b200.arm import swiglu_fn
    return swiglu_fn(P["x"], P["w1"], P.get("b1"), P["w2"], P.get("b2"), P["w3"], P.get("b3"), **kw)


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
    P = _op_inputs(768, 2048, torch.float32)
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


@pytest.mark.parametrize("shape", [(768, 2048), (1024, 2730)], ids=["in768_H2048", "in1024_H2730"])
def test_saved_tensor_bound(shape):
    """Parameters aside, level 0 keeps x and the packed a / b (2 M Hp elements), level 1 x only; both less than the
    composition.  Under no_grad, or with nothing requiring a gradient, no a / b buffer is allocated."""
    K, H = shape
    Hp = _pad64(H)
    m = _mlp(K, H, 3, torch.bfloat16)
    x = torch.randn(8, 197, K, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    M = x.shape[0] * x.shape[1]
    params = list(m.parameters())
    args = lambda: (x, m.w1.weight, m.w1.bias, m.w2.weight, m.w2.bias, m.w3.weight, m.w3.bias)
    from medical_image_analysis_b200.arm import swiglu_fn
    s0, out = _saved_bytes(lambda: swiglu_fn(*args(), checkpoint_lvl=0), params)
    out.float().sum().backward()
    s1, out = _saved_bytes(lambda: swiglu_fn(*args(), checkpoint_lvl=1), params)
    out.float().sum().backward()
    comp, out = _saved_bytes(lambda: m._forward_composed(x), params)
    print(f"saved bytes: level 0 {s0}, level 1 {s1}, composition {comp}")
    assert s0 <= x.nbytes + 2 * M * Hp * 2, s0
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
        p_ng, y = peak(lambda: swiglu_fn(*args()))
    xd = x.detach()
    with torch.no_grad():
        for p in params:
            p.requires_grad_(False)
    try:
        p_nr, y2 = peak(lambda: swiglu_fn(xd, *args()[1:]))
    finally:
        for p in params:
            p.requires_grad_(True)
    assert torch.equal(y, y2)
    w3_pad = K * Hp * 2 if H % 8 else 0                                # W3 zero-padded to an aligned pitch (arm_large)
    for p_ in (p_ng, p_nr):                                            # h, the output and W3's pad copy; no (M, 2 Hp) buffer
        assert p_ <= h_bytes + y_bytes + w3_pad + (1 << 20), (p_, h_bytes, y_bytes, w3_pad)


# ---------------------------------------------------------------------------------------------------------- kernel path
BIG_OPS = ("aten::silu", "aten::silu_backward", "aten::mul", "aten::add", "aten::add_", "aten::cat", "aten::copy_")
SWIGLU = re.compile(r"\bgemm_swiglu_kernel<(\d)")
GEMM = re.compile(r"\bgemm_tn_kernel<")
REDUCE = re.compile(r"reduce_kernel")


def _want(lvl, phase):
    if phase == "fwd":
        return {"swiglu_fwd": 1, "gemm": 1}
    want = {"swiglu_bwd": 1, "gemm": 3, "reduce": 2}
    if lvl == 1:
        want["swiglu_fwd"] = 1                                         # a / b (and h) recomputed by the forward kernel
    return want


def _capture(lvl, phase, K, H, b):
    """One profiled fwd or bwd of a fresh op -> kernel launch counts and (M, H)-sized aten ops."""
    M = b * 197
    P = _op_inputs(K, H, torch.bfloat16)
    P["x"] = torch.randn(b, 197, K, device="cuda", dtype=torch.bfloat16, requires_grad=True)
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
            m = SWIGLU.search(e.name)
            key = ("swiglu_fwd" if m.group(1) == "1" else "swiglu_bwd") if m else ("gemm" if GEMM.search(e.name) else
                                                                                  ("reduce" if REDUCE.search(e.name) else None))
            if key:
                counts[key] = counts.get(key, 0) + 1
    return {"counts": counts, "big_ops": big}


def kernel_path():
    """Run in a child interpreter: kernel launch counts and (M, H)-sized aten ops, fwd and bwd separately, per level.  A
    capture missing expected launches is taken again (kernel_trace.retry: a profiler session now and then loses kernel
    records); the last capture is returned either way, so a wrong launch path still fails the test."""
    res = {}
    for lvl in (0, 1):
        for phase in ("fwd", "bwd"):
            want = _want(lvl, phase)
            res[f"{lvl}/{phase}"] = kernel_trace.retry(lambda: _capture(lvl, phase, 768, 2048, 16),
                                                       lambda r: all(r["counts"].get(k, 0) >= n for k, n in want.items()))
    return res


@pytest.fixture(scope="module")
def path():
    return kernel_trace.in_child("tests.test_swiglu_fused_gpu:kernel_path")


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
    from medical_image_analysis_b200 import arm
    calls = []
    real = arm.swiglu_fn

    def spy(*a, **k):
        calls.append(a[0].shape)
        return real(*a, **k)

    monkeypatch.setattr(arm, "swiglu_fn", spy)
    return calls


def test_routing(op_calls):
    from medical_image_analysis_b200.arm import SwiGLU
    torch.manual_seed(0)
    x = torch.randn(2, 17, 64, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        SwiGLU(64, 176).cuda()(x)
    assert len(op_calls) == 1
    SwiGLU(64, 176).cuda().bfloat16()(x.bfloat16())
    assert len(op_calls) == 2
    with torch.autocast("cuda", dtype=torch.bfloat16):
        SwiGLU(64, 176, subln=True).cuda()(x)
        SwiGLU(64, 176, act_layer=torch.nn.GELU).cuda()(x)
    SwiGLU(64, 176).cuda()(x)                                          # fp32: the library path, as gemm.linear
    SwiGLU(64, 176)(x.cpu())
    assert len(op_calls) == 2


def test_encoder_routing_and_determinism(op_calls, monkeypatch):
    """arm_base_pz16 under bf16 autocast runs the op in every block; with deterministic algorithms its fwd + bwd is
    bit-reproducible."""
    from medical_image_analysis_b200.arm import arm_base_pz16
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")            # the mixers' dt_proj GEMMs are cuBLAS calls
    torch.manual_seed(0)
    model = arm_base_pz16(drop_path_rate=0.0).cuda()
    img = torch.randn(2, 3, 224, 224, device="cuda")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            model.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = model(img)
            y.float().square().mean().backward()
            runs.append((y.detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert len(op_calls) == 2 * len(model.layers)
    assert torch.equal(runs[0][0], runs[1][0])
    assert runs[0][1].keys() == runs[1][1].keys() and any(k.endswith("mlp.w1.weight") for k in runs[0][1])
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k
