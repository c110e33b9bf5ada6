"""The ARM pre-training decoder's segment-causal cross-attention as one op (arm_pretrain.CrossAttentionFn, the cross-attention
instantiations of csrc/attention.cu) on the H100.

Kernel parity: o, lse, dq and dk / dv of mia_xattn_fwd / _bwd against a float64 statement of softmax(q k^T dh^-0.5 + mask) v
on the same rounded inputs, with the tolerances of test_attention_fused_gpu.py and an RMS error no more than 1.25x that of
SDPA's default backend given the same additive mask.  Then causality, image isolation, edge logits, the whole op against a
float64 statement of the composition, determinism, checkpoint levels, the saved set, routing, the kernel path and the toy
pre-training model."""
import pytest
import torch
import torch.nn.functional as F

from medical_image_analysis_b200 import _lib, arm_pretrain
from tests import kernel_trace
from tests.parity import cmp_f32, cmp_stored
from tests.test_attention_fused_gpu import EDGE, G_RMS, G_ULP, O_RMS, O_ULP, SDPA_FACTOR, _rms_err

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DH = 64


def _mask(N, seg, device="cuda"):
    i = torch.arange(N, device=device)
    return torch.zeros(N, N, device=device).masked_fill(i[None, :] // seg > i[:, None] // seg, float("-inf"))


def _inputs(B, N, H, dtype, kind="random", seed=0):
    """q (B N, C), kv (B N, 2C) in the packed (B, N, 2, H, dh) layout and dO (B N, C)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = (torch.randn(B, N, H, DH, device="cuda", generator=g) for _ in range(3))
    if kind == "large":
        q, k = q * 15 ** 0.5, k * 15 ** 0.5
    elif kind == "dominant":
        k = 4 * q
    elif kind == "equal":
        k = k[:, :1].expand_as(k).contiguous()
    do = torch.randn(B * N, H * DH, device="cuda", generator=g).to(dtype)
    return q.reshape(B * N, H * DH).to(dtype), torch.stack((k, v), 2).reshape(B * N, 2 * H * DH).to(dtype), do


def _kernels(q, kv, do, B, N, H, seg):
    C, dtype = H * DH, q.dtype
    o = torch.empty(B * N, C, dtype=dtype, device="cuda")
    lse = torch.empty(B, H, N, dtype=torch.float32, device="cuda")
    _lib.call("mia_xattn_fwd", "xattn fwd", q.device, q.data_ptr(), kv.data_ptr(), o.data_ptr(), lse.data_ptr(), B, N, H, DH, seg, q.stride(0),
              kv.stride(0), o.stride(0), _lib.dtype_code(dtype))
    delta = torch.empty(B, H, N, dtype=torch.float32, device="cuda")
    dq = torch.full((B * N, C), float("nan"), dtype=dtype, device="cuda")
    dkv = torch.full((B * N, 2 * C), float("nan"), dtype=dtype, device="cuda")
    _lib.call("mia_xattn_bwd", "xattn bwd", q.device, q.data_ptr(), kv.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(), delta.data_ptr(),
              dq.data_ptr(), dkv.data_ptr(), B, N, H, DH, seg, q.stride(0), kv.stride(0), o.stride(0), do.stride(0), dq.stride(0), dkv.stride(0),
              _lib.dtype_code(dtype))
    return o, lse, dq, dkv


def _heads(t, B, N, H):
    return t.view(B, N, H, DH).transpose(1, 2)


def _split(q, kv, B, N, H):
    k, v = kv.view(B, N, 2, H, DH).permute(2, 0, 3, 1, 4).unbind(0)
    return _heads(q, B, N, H), k, v


def _pack(dq, dk, dv, B, N, H):
    return dq.transpose(1, 2).reshape(B * N, H * DH), torch.stack((dk, dv), 0).permute(1, 3, 0, 2, 4).reshape(B * N, 2 * H * DH)


def _reference(q, kv, do, B, N, H, seg):
    qh, k, v = (t.double() for t in _split(q, kv, B, N, H))
    dO = _heads(do, B, N, H).double()
    s = qh @ k.transpose(-1, -2) * DH ** -0.5 + _mask(N, seg).double()
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    dv = p.transpose(-1, -2) @ dO
    dp = dO @ v.transpose(-1, -2)
    ds = p * (dp - (dp * p).sum(-1, keepdim=True))
    dq, dk = ds @ k * DH ** -0.5, ds.transpose(-1, -2) @ qh * DH ** -0.5
    return (o.transpose(1, 2).reshape(B * N, H * DH), lse) + _pack(dq, dk, dv, B, N, H)


def _sdpa(q, kv, do, B, N, H, seg):
    qh, k, v = (t.detach().clone().requires_grad_() for t in _split(q, kv, B, N, H))
    o = F.scaled_dot_product_attention(qh, k, v, attn_mask=_mask(N, seg).to(q.dtype))
    o.backward(_heads(do, B, N, H))
    return (o.detach().transpose(1, 2).reshape(B * N, H * DH),) + _pack(qh.grad, k.grad, v.grad, B, N, H)


def _check(B, N, H, seg, dtype, kind="random"):
    q, kv, do = _inputs(B, N, H, dtype, kind)
    o, lse, dq, dkv = _kernels(q, kv, do, B, N, H, seg)
    r_o, r_lse, r_dq, r_dkv = _reference(q, kv, do, B, N, H, seg)
    tag = f"B{B} N{N} H{H} seg{seg} {dtype} {kind}"
    f = 1.0 if kind == "random" else EDGE
    cmp_stored(o, r_o, dtype, f"{tag} o", O_ULP * f, O_RMS * f)
    cmp_f32(lse, r_lse, f"{tag} lse", 1e-5, 1e-5)
    pack = torch.cat((dq, dkv), 1)                    # one yardstick: dq of a query that sees only its own segment can be ~0
    r_pack = torch.cat((r_dq, r_dkv), 1)
    cmp_stored(pack, r_pack, dtype, f"{tag} dq|dkv", G_ULP * f, G_RMS * f)
    s_o, s_dq, s_dkv = _sdpa(q, kv, do, B, N, H, seg)
    assert _rms_err(o, r_o) <= SDPA_FACTOR * _rms_err(s_o, r_o) + 1e-7, (tag, "o", _rms_err(o, r_o), _rms_err(s_o, r_o))
    floor = 2.0 ** -14 * float(r_pack.pow(2).mean().sqrt())
    C = H * DH
    for name, ours, ref, theirs in (("dq", dq, r_dq, s_dq), ("dk", dkv[:, :C], r_dkv[:, :C], s_dkv[:, :C]), ("dv", dkv[:, C:], r_dkv[:, C:], s_dkv[:, C:])):
        a, b = _rms_err(ours, ref), _rms_err(theirs, ref)
        assert a <= SDPA_FACTOR * b + floor, (tag, name, a, b)


# ------------------------------------------------------------------------------------------------------ kernel parity
CASES = [(N, seg) for N in (16, 48, 128, 129, 384) for seg in sorted({1, 16, 24, N}) if seg <= N]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H", [(1, 1), (3, 8)])
@pytest.mark.parametrize("N,seg", CASES)
def test_kernels_against_float64(N, seg, B, H, dtype):
    _check(B, N, H, seg, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["large", "dominant", "equal"])
def test_kernels_edge_inputs(kind, dtype):
    _check(2, 129, 4, 16, dtype, kind)


@pytest.mark.parametrize("N,seg", [(128, 16), (129, 16), (384, 16), (384, 24)])
def test_later_segments_do_not_reach_earlier_queries(N, seg):
    """Perturbing k / v of the keys in segments after s leaves o, lse and dq of the queries in segments <= s bit-identical."""
    B, H = 2, 4
    q, kv, do = _inputs(B, N, H, torch.bfloat16)
    o, lse, dq, _ = _kernels(q, kv, do, B, N, H, seg)
    for s in (0, (N - 1) // seg // 2):
        cut = (s + 1) * seg
        kv2 = kv.view(B, N, -1).clone()
        kv2[:, cut:] = kv2[:, cut:] * -2 + 1
        o2, lse2, dq2, _ = _kernels(q, kv2.view(B * N, -1), do, B, N, H, seg)
        for b in range(B):
            rows = slice(b * N, b * N + cut)
            assert torch.equal(o[rows], o2[rows]) and torch.equal(dq[rows], dq2[rows]), (s, b)
            assert torch.equal(lse[b, :, :cut], lse2[b, :, :cut]), (s, b)


@pytest.mark.parametrize("N", [48, 129])
def test_images_are_isolated(N):
    B, H = 3, 4
    q, kv, do = _inputs(B, N, H, torch.bfloat16)
    outs = _kernels(q, kv, do, B, N, H, 16)
    q2, kv2, do2 = q.clone(), kv.clone(), do.clone()
    q2[N:2 * N], kv2[N:2 * N], do2[N:2 * N] = q2[N:2 * N] * 3 + 1, kv2[N:2 * N] * 3 - 1, -do2[N:2 * N]
    outs2 = _kernels(q2, kv2, do2, B, N, H, 16)
    for b in (0, 2):
        rows = slice(b * N, (b + 1) * N)
        for i in (0, 2, 3):
            assert torch.equal(outs[i][rows], outs2[i][rows]), (b, i)
        assert torch.equal(outs[1][b], outs2[1][b]), b


# ------------------------------------------------------------------------------------------------------ the op
def _weights(C, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: (torch.randn(*s, device="cuda", generator=g) / s[-1] ** 0.5).requires_grad_()
    return [mk(C, C), (0.1 * torch.randn(C, device="cuda", generator=g)).requires_grad_(), mk(2 * C, C),
            (0.1 * torch.randn(2 * C, device="cuda", generator=g)).requires_grad_(), mk(C, C), (0.1 * torch.randn(C, device="cuda", generator=g)).requires_grad_()]


def _composition64(q_in, kv_in, w, H, mask):
    """float64 statement of the reference's CrossAttention.forward."""
    B, N, C = q_in.shape
    q = F.linear(q_in, w[0], w[1]).view(B, N, H, DH).transpose(1, 2)
    k, v = F.linear(kv_in, w[2], w[3]).view(B, N, 2, H, DH).permute(2, 0, 3, 1, 4).unbind(0)
    a = (q @ k.transpose(-1, -2) * DH ** -0.5 + mask).softmax(-1)
    return F.linear((a @ v).transpose(1, 2).reshape(B, N, C), w[4], w[5])


def _grads(fn, q_in, kv_in, w, g):
    leaves = [q_in.detach().clone().requires_grad_(), kv_in.detach().clone().requires_grad_()] + [t.detach().clone().requires_grad_() for t in w]
    y = fn(leaves[0], leaves[1], leaves[2:])
    y.backward(g.to(y.dtype))
    return [y.detach()] + [t.grad for t in leaves]


def _module_run(m, routed, mask, mode, H):
    """CrossAttention m through its forward with the given parameter leaves, routed to the op or to the composition."""
    def fn(qi, ki, ws):
        params = dict(zip(("q.weight", "q.bias", "kv.weight", "kv.bias", "proj.weight", "proj.bias"), ws))
        real = arm_pretrain.cross_attention_eligible
        if not routed:
            arm_pretrain.cross_attention_eligible = lambda *a: False
        try:
            if mode == "autocast":
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    return torch.func.functional_call(m, params, (qi, ki, mask))
            return torch.func.functional_call(m, params, (qi, ki, mask))
        finally:
            arm_pretrain.cross_attention_eligible = real
    return fn


@pytest.mark.parametrize("mode", ["bf16", "fp16", "autocast"])
@pytest.mark.parametrize("N", [128, 384])
def test_op_against_float64_composition(N, mode):
    """The op is no further from float64 than the composition, on the output and every gradient."""
    B, C, H, seg = 4, 512, 8, 16
    mask = _mask(N, seg)
    gen = torch.Generator(device="cuda").manual_seed(2)
    q_in, kv_in = torch.randn(B, N, C, device="cuda", generator=gen), torch.randn(B, N, C, device="cuda", generator=gen)
    g = torch.randn(B, N, C, device="cuda", generator=gen)
    w = _weights(C)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16, "autocast": None}[mode]
    if dt is not None:                                   # the float64 statement starts from the same rounded values
        q_in, kv_in, w = q_in.to(dt), kv_in.to(dt), [t.detach().to(dt) for t in w]
    m = arm_pretrain.CrossAttention(C, H, qkv_bias=True).cuda()
    calls = []
    real = arm_pretrain.cross_attention_fn
    arm_pretrain.cross_attention_fn = lambda *a, **k: calls.append(1) or real(*a, **k)
    try:
        ours = _grads(_module_run(m, True, mask, mode, H), q_in, kv_in, w, g)
        comp = _grads(_module_run(m, False, mask, mode, H), q_in, kv_in, w, g)
    finally:
        arm_pretrain.cross_attention_fn = real
    assert len(calls) == 1
    ref = _grads(lambda a, b, ws: _composition64(a, b, ws, H, mask.double()), q_in.double(), kv_in.double(), [t.double() for t in w], g.double())
    names = ["y", "dq_in", "dkv_in", "dWq", "dbq", "dWkv", "dbkv", "dWp", "dbp"]
    for name, a, c, r in zip(names, ours, comp, ref):
        ea, ec = _rms_err(a, r), _rms_err(c, r)
        assert ea <= SDPA_FACTOR * ec + 1e-6 * float(r.pow(2).mean().sqrt()), (mode, N, name, ea, ec)


def _op_run(lvl, B=3, N=128, C=512, H=8, dtype=torch.bfloat16):
    gen = torch.Generator(device="cuda").manual_seed(5)
    q_in = torch.randn(B, N, C, device="cuda", generator=gen).to(dtype).requires_grad_()
    kv_in = torch.randn(B, N, C, device="cuda", generator=gen).to(dtype).requires_grad_()
    w = _weights(C)
    y = arm_pretrain.cross_attention_fn(q_in, kv_in, *w, H, 16, checkpoint_lvl=lvl)
    y.backward(torch.randn(y.shape, device="cuda", generator=gen).to(dtype))
    return [y.detach(), q_in.grad, kv_in.grad] + [t.grad for t in w]


def test_reproducible_and_levels_identical():
    a, b, c = _op_run(0), _op_run(0), _op_run(1)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


@pytest.mark.parametrize("lvl", [0, 1])
def test_saved_tensor_bound(lvl):
    B, N, C, H = 3, 128, 512, 8
    saved = []

    def pack(t):
        saved.append(t)
        return t
    q_in = torch.randn(B, N, C, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    kv_in = torch.randn(B, N, C, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    w = _weights(C)
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        arm_pretrain.cross_attention_fn(q_in, kv_in, *w, H, 16, checkpoint_lvl=lvl)
    act = sum(t.numel() * t.element_size() for t in saved if t.dim() != 1 and tuple(t.shape[-2:]) != (C, C) and tuple(t.shape) != (2 * C, C))
    bound = 2 * B * N * C * 2 + (4 * B * N * C * 2 + B * H * N * 4 if lvl == 0 else 0)
    assert act <= bound, (act, bound)
    with torch.no_grad():
        saved.clear()
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            arm_pretrain.cross_attention_fn(q_in, kv_in, *w, H, 16)
        assert not saved


def test_routing():
    C, H, N = 128, 2, 48
    m = arm_pretrain.CrossAttention(C, H, qkv_bias=True).cuda()
    mask = _mask(N, 16)
    x = torch.randn(2, N, C, device="cuda")
    el = arm_pretrain.cross_attention_eligible
    assert not el(m, x, x, mask)                                              # fp32
    assert el(m, x.bfloat16(), x.bfloat16(), mask) and el(m, x.half(), x.half(), mask)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert el(m, x, x, mask)
    assert not el(m.cpu(), x.cpu().bfloat16(), x.cpu().bfloat16(), mask.cpu())
    m.cuda()
    assert not el(arm_pretrain.CrossAttention(96, 2).cuda(), torch.randn(2, N, 96, device="cuda").bfloat16(), torch.randn(2, N, 96, device="cuda").bfloat16(), mask)
    d = arm_pretrain.CrossAttention(C, H, attn_drop=0.1).cuda()
    assert not el(d.train(), x.bfloat16(), x.bfloat16(), mask) and el(d.eval(), x.bfloat16(), x.bfloat16(), mask)
    assert not el(m, x.bfloat16(), x.bfloat16(), torch.randn(N, N, device="cuda"))     # not a segment mask
    buf = mask.clone()
    assert el(m, x.bfloat16(), x.bfloat16(), buf)
    buf[3, 40] = 0.0                                                          # mutated: composition
    assert not el(m, x.bfloat16(), x.bfloat16(), buf)
    buf[3, 40] = float("-inf")                                                # restored: the op again
    assert el(m, x.bfloat16(), x.bfloat16(), buf)


BIG_OPS = {"aten::bmm", "aten::matmul", "aten::softmax", "aten::_softmax", "aten::_softmax_backward_data", "aten::add", "aten::add_"}
COPY_OPS = {"aten::copy_", "aten::cat", "aten::contiguous", "aten::clone"}


def kernel_path():
    """One training step of a bf16 CrossAttention on bf16 activations, profiled: attention kernel counts and the aten ops
    that touch a (B, H, N, N) tensor or copy a (B, N, C) one (under autocast, fp32 activations are cast to bf16 once, as
    for any autocast op)."""
    B, N, C, H = 2, 128, 512, 8
    torch.manual_seed(0)
    m = arm_pretrain.CrossAttention(C, H, qkv_bias=True).cuda().bfloat16()
    mask = _mask(N, 16)
    q_in = torch.randn(B, N, C, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    kv_in = torch.randn(B, N, C, device="cuda", dtype=torch.bfloat16, requires_grad=True)

    def capture():
        m(q_in, kv_in, mask)                              # the mask check runs once, before the trace
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                    record_shapes=True) as prof:
            y = m(q_in, kv_in, mask)
            y.backward(torch.ones_like(y))
            torch.cuda.synchronize()
        counts, bad = {}, []
        for e in prof.events():
            shapes = [tuple(x) for x in (e.input_shapes or []) if x]
            if e.name in BIG_OPS and ((B, H, N, N) in shapes or (B * H, N, N) in shapes):
                bad.append(f"{e.name}{shapes}")
            if e.name in COPY_OPS and (B, N, C) in shapes:
                bad.append(f"{e.name}{shapes}")
            if e.device_type == torch.autograd.DeviceType.CUDA:
                for k in ("attn_fwd_kernel<", "attn_bwd_dq_kernel<", "attn_bwd_dkv_kernel<"):
                    if k in e.name:
                        key = k + ",".join(kernel_trace.targs(e.name, k))
                        counts[key] = counts.get(key, 0) + 1
        return {"counts": counts, "bad": bad}
    return kernel_trace.retry(capture, lambda r: sum(r["counts"].values()) >= 3)


def test_kernel_path():
    r = kernel_trace.in_child("tests.test_cross_attention_fused_gpu:kernel_path")
    assert r["counts"] == {"attn_fwd_kernel<64,false,true": 1, "attn_bwd_dq_kernel<64,false,true": 1, "attn_bwd_dkv_kernel<64,false,true": 1}, r
    assert not r["bad"], r["bad"]


# ------------------------------------------------------------------------------------------------------ the toy model
TOY = dict(img_size=128, patch_size=16, stride=16, embed_dim=32, depth=12, dec_embed_dim=128, rms_norm=True, residual_in_fp32=True,
           fused_add_norm=True, if_abs_pos_embed=True, bimamba_type="None", drop_path_rate=0.0, ssm_cfg=dict(d_state=4))


def _toy_step(m, img, routed=True):
    m.zero_grad(set_to_none=True)
    calls = []
    real = arm_pretrain.cross_attention_fn

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    arm_pretrain.cross_attention_fn = spy
    real_el = arm_pretrain.cross_attention_eligible
    if not routed:
        arm_pretrain.cross_attention_eligible = lambda *a: False
    try:
        x = img.clone().requires_grad_()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = m(x)
        w = torch.linspace(-1, 1, loss.numel(), device="cuda")
        (loss * w).sum().backward()
    finally:
        arm_pretrain.cross_attention_fn, arm_pretrain.cross_attention_eligible = real, real_el
    return [loss.detach(), x.grad] + [p.grad for p in m.parameters() if p.requires_grad], len(calls)


def test_toy_model_bit_reproducible_and_no_further_from_fp32_golden():
    from tests.test_arm_pretrain_golden import _image, _model
    torch.use_deterministic_algorithms(True)
    try:
        m, c = _model(128)
        m = m.cuda()
        img = _image(128).cuda()
        a, na = _toy_step(m, img)
        b, _ = _toy_step(m, img)
        assert na == len(m.dec_block) == 4
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        comp, nc = _toy_step(m, img, routed=False)
        assert nc == 0
    finally:
        torch.use_deterministic_algorithms(False)
    # the yardstick: the fp32 model, whose loss is the golden's, on the same image and weights w
    w = torch.linspace(-1, 1, a[0].numel())
    names = ["loss"] + [n for n, p in m.named_parameters() if p.requires_grad]
    m32, _ = _model(128)
    m32 = m32.cuda()
    x32 = img.clone().requires_grad_()
    loss32 = m32(x32)
    (loss32 * w.cuda()).sum().backward()
    ref = [loss32.detach()] + [p.grad for p in m32.parameters() if p.requires_grad]
    assert torch.allclose(ref[0].cpu(), torch.from_numpy(c["loss"]), rtol=5e-4, atol=5e-4)
    for name, o, k, r in zip(names, [a[0]] + a[2:], [comp[0]] + comp[2:], ref):
        eo, ek = _rms_err(o, r), _rms_err(k, r)
        assert eo <= SDPA_FACTOR * ek + 1e-3 * float(r.double().pow(2).mean().sqrt()), (name, eo, ek)
