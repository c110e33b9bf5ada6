"""Every instantiation of the wgmma GEMM (csrc/gemm_wgmma.cu) against float64, at the shapes where a tiled kernel goes wrong.

The host picks the kernel from M, N and the device's SM count.  A Python replica of each rule (``gemm_bn``) builds, for each
of the 40 instantiations, cases that land on it with more tiles than SMs (the persistent loop carries the mbarrier ring
phase from tile to tile), a partial last M tile, a ragged last N tile, a K tail whose block count is not a multiple of the
stage count and a single K block.  Outputs go into NaN-filled buffers with a row pitch wider than N (an odd one for the
plain GEMM): everything outside the written region must still be that NaN, bit for bit.  A child interpreter records
the kernel each case launched (kernel_trace), so a rule change that moves a case off its target fails; a CPU test checks
the list of 40 against the built library, and another shows that the criteria reject subtly wrong results."""
import os
import re
import shutil
import subprocess
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_trace
from tests.parity import cmp_f32, cmp_stored
from tests.test_attention_fused_gpu import SDPA_FACTOR, _float64_block, _rms_err
from tests.test_attention_fused_gpu import _grads as _attn_grads
from tests.test_attention_fused_gpu import _params as _attn_params
from tests.test_gelu_mlp_fused_gpu import _dgelu64, _rel, _vmamba_mlp
from tests.test_gelu_mlp_fused_gpu import _grads as _gelu_grads
from tests.test_gelu_mlp_fused_gpu import _ref64 as _gelu_ref64
from tests.test_swiglu_fused_gpu import _grads as _swiglu_grads
from tests.test_swiglu_fused_gpu import _mlp as _swiglu_mlp
from tests.test_swiglu_fused_gpu import _within_ulp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "medical_image_analysis_b200", "libmia_scan.so")
gpu = pytest.mark.gpu

# Every kernel the library holds: gemm_tn_kernel<BN, kStages, kAMN, kBMN, kF16> and the fused-epilogue
# gemm_{gelu,swiglu}_kernel<kEpi, BN, kStages, kBMN, kF16> (kEpi 1 / 2 SwiGLU fwd / bwd, 3 / 4 GELU fwd / bwd).
INSTANTIATIONS = [
    "gemm_tn_kernel<64, 8, false, false, false>", "gemm_tn_kernel<64, 8, false, false, true>",
    "gemm_tn_kernel<64, 8, false, true, false>", "gemm_tn_kernel<64, 8, false, true, true>",
    "gemm_tn_kernel<64, 8, true, true, false>", "gemm_tn_kernel<64, 8, true, true, true>",
    "gemm_tn_kernel<64, 8, true, false, false>", "gemm_tn_kernel<64, 8, true, false, true>",
    "gemm_tn_kernel<128, 6, false, false, false>", "gemm_tn_kernel<128, 6, false, false, true>",
    "gemm_tn_kernel<128, 6, false, true, false>", "gemm_tn_kernel<128, 6, false, true, true>",
    "gemm_tn_kernel<128, 6, true, true, false>", "gemm_tn_kernel<128, 6, true, true, true>",
    "gemm_tn_kernel<128, 6, true, false, false>", "gemm_tn_kernel<128, 6, true, false, true>",
    "gemm_tn_kernel<256, 4, false, false, false>", "gemm_tn_kernel<256, 4, false, false, true>",
    "gemm_tn_kernel<256, 4, false, true, false>", "gemm_tn_kernel<256, 4, false, true, true>",
    "gemm_tn_kernel<256, 4, true, true, false>", "gemm_tn_kernel<256, 4, true, true, true>",
    "gemm_tn_kernel<256, 4, true, false, false>", "gemm_tn_kernel<256, 4, true, false, true>",
    "gemm_gelu_kernel<3, 64, 8, false, false>", "gemm_gelu_kernel<3, 64, 8, false, true>",
    "gemm_gelu_kernel<3, 128, 6, false, false>", "gemm_gelu_kernel<3, 128, 6, false, true>",
    "gemm_gelu_kernel<3, 256, 4, false, false>", "gemm_gelu_kernel<3, 256, 4, false, true>",
    "gemm_gelu_kernel<4, 128, 6, true, false>", "gemm_gelu_kernel<4, 128, 6, true, true>",
    "gemm_gelu_kernel<4, 256, 4, true, false>", "gemm_gelu_kernel<4, 256, 4, true, true>",
    "gemm_swiglu_kernel<1, 256, 4, false, false>", "gemm_swiglu_kernel<1, 256, 4, false, true>",
    "gemm_swiglu_kernel<2, 128, 6, true, false>", "gemm_swiglu_kernel<2, 128, 6, true, true>",
    "gemm_swiglu_kernel<2, 256, 4, true, false>", "gemm_swiglu_kernel<2, 256, 4, true, true>",
]
STAGES = {64: 8, 128: 6, 256: 4}
KERNEL = re.compile(r"\b(gemm_(?:tn|gelu|swiglu)_kernel)<")


def _cdiv(a, b):
    return -(-a // b)


def gemm_bn(M, N, sms):
    """The tile width gemm_impl picks (and mia_gemm_gelu_fwd for N = H).  The backward epilogues take the 256 tile exactly
    when this is 256 for N = H, and the 128 tile otherwise."""
    return 64 if N <= 64 else (128 if N <= 128 or _cdiv(M, 128) * _cdiv(N, 256) < sms else 256)


def _tf(v):
    return "true" if v else "false"


def short_name(name):
    """'void (anonymous namespace)::gemm_tn_kernel<64, 8, ...>(CUtensorMap_st, ...)' -> 'gemm_tn_kernel<64, 8, ...>'."""
    kern = KERNEL.search(name).group(1)
    return f"{kern}<{', '.join(kernel_trace.targs(name, kern + '<'))}>"


# ---------------------------------------------------------------------------------------------------------- the case table
@dataclass
class Case:
    """One launch.  kind: gemm (mia_gemm), gelu_fwd / gelu_bwd / swiglu_fwd / swiglu_bwd (the fused entries); N is the hidden
    width H for the fused kinds; K the contraction (N_out for the backward kinds).  M = 128 (m_blocks(sms) - 1) + tail."""
    id: str
    kind: str
    f16: bool
    N: int
    K: int
    tail: int
    wide_m: bool = False      # m_blocks = 3 sms / 2 (one N tile per row block) instead of 3 sms / 4
    amn: bool = False
    bmn: bool = False
    out_f32: bool = False
    ldc_extra: int = 0
    bias: bool = False
    act: int = 0
    swiglu_rows: str = ""     # SwiGLU row-block rules: "narrow" (5 sms / 12) or "quarter" (sms / 4)

    @property
    def dtype(self):
        return torch.float16 if self.f16 else torch.bfloat16

    def m_blocks(self, sms):
        if self.swiglu_rows == "narrow":
            return 5 * sms // 12
        if self.swiglu_rows == "quarter":
            return sms // 4
        return 3 * sms // 2 if self.wide_m else 3 * sms // 4

    def M(self, sms):
        return 128 * (self.m_blocks(sms) - 1) + self.tail

    def target(self, sms):
        """The instantiation the host rules select for this case."""
        M, f = self.M(sms), _tf(self.f16)
        if self.kind == "gemm":
            bn = gemm_bn(M, self.N, sms)
            return f"gemm_tn_kernel<{bn}, {STAGES[bn]}, {_tf(self.amn)}, {_tf(self.bmn)}, {f}>"
        if self.kind == "swiglu_fwd":
            return f"gemm_swiglu_kernel<1, 256, 4, false, {f}>"
        bn = gemm_bn(M, self.N, sms)
        if self.kind == "gelu_fwd":
            return f"gemm_gelu_kernel<3, {bn}, {STAGES[bn]}, false, {f}>"
        bn = 256 if bn == 256 else 128
        epi, kern = (4, "gelu") if self.kind == "gelu_bwd" else (2, "swiglu")
        return f"gemm_{kern}_kernel<{epi}, {bn}, {STAGES[bn]}, true, {f}>"

    def tiles(self, sms):
        M = self.M(sms)
        span = 128 if self.kind == "swiglu_fwd" else gemm_bn(M, self.N, sms) if self.kind in ("gemm", "gelu_fwd") else \
            int(self.target(sms).split("<")[1].split(",")[1])
        return _cdiv(M, 128) * _cdiv(self.N, span)


# K = 600: ten K blocks, a 24-wide tail, 10 not a multiple of 8, 6 or 4 stages.  K = 8: one K block, fewer than the stages.
# N per tile width: (40, 56) for BN 64; (200, 120) for BN 128 (two N tiles at 3 sms / 4 row blocks, one at 3 sms / 2);
# (296, 424) for BN 256: the last tile's upper 128 columns wholly (296 = 40 mod 256) / partly (424 = 168 mod 256) beyond
# N.  A K-major B takes N + 1 for the second N (a one-column ragged edge); MN-major operands need multiples of 8.
_N = {64: (40, 56), 128: (200, 120), 256: (296, 424)}


def _gemm_cases():
    out = []
    for bn, (na, nb) in _N.items():
        for amn, bmn in ((False, False), (False, True), (True, True), (True, False)):
            for f16 in (False, True):
                mode = f"a{'mn' if amn else 'k'}_b{'mn' if bmn else 'k'}"
                for i, (N, K, out_f32, extra, tail) in enumerate(((na, 600, True, 1, 40), (nb + (not bmn), 600, False, 8, 104),
                                                                  (na, 8, False, 1, 104), (nb + (not bmn), 8, True, 0, 40))):
                    bias = not (amn or bmn) or i % 2 == 0        # K-major x K-major: bias with every activation
                    out.append(Case(f"gemm-BN{bn}-{mode}-{'f16' if f16 else 'bf16'}-N{N}-K{K}-{'f32' if out_f32 else '16b'}"
                                    f"-ldc+{extra}-act{i}{'-bias' if bias else ''}", "gemm", f16, N, K, tail, wide_m=N <= 128,
                                    amn=amn, bmn=bmn, out_f32=out_f32, ldc_extra=extra, bias=bias, act=i))
    return out


def _fused_cases():
    out = []
    for f16 in (False, True):
        d = "f16" if f16 else "bf16"
        for H in (44, 196, 300):                                         # BN 64, 128, 256
            out.append(Case(f"gelu_fwd-{d}-H{H}-K600-bias", "gelu_fwd", f16, H, 600, 40, wide_m=H <= 128, bias=True))
            out.append(Case(f"gelu_fwd-{d}-H{H}-K8", "gelu_fwd", f16, H, 8, 104, wide_m=H <= 128))
        # 128 tile (H = 120 with more row blocks than SMs: the 256 tile's upper half would be all padding); 256 tile with
        # the last tile's upper half wholly (H = 300) / partly (H = 420) beyond Hp
        for H, K, tail in ((196, 600, 40), (120, 600, 104), (300, 600, 104), (420, 136, 40)):
            out.append(Case(f"gelu_bwd-{d}-H{H}-N{K}", "gelu_bwd", f16, H, K, tail, wide_m=H <= 128))
        for H, K, tail, rows in ((300, 600, 40, "narrow"), (120, 600, 104, ""), (300, 600, 104, ""), (424, 136, 40, "")):
            out.append(Case(f"swiglu_bwd-{d}-H{H}-N{K}{'-narrow' if rows else ''}", "swiglu_bwd", f16, H, K, tail,
                            wide_m=H <= 128, swiglu_rows=rows))
        out.append(Case(f"swiglu_fwd-{d}-H2730-K1064-bias", "swiglu_fwd", f16, 2730, 1064, 40, bias=True, swiglu_rows="quarter"))
        out.append(Case(f"swiglu_fwd-{d}-H2730-K8", "swiglu_fwd", f16, 2730, 8, 104, swiglu_rows="quarter"))
    return out


GEMM_CASES = _gemm_cases()
FUSED_CASES = _fused_cases()
CASES = {c.id: c for c in GEMM_CASES + FUSED_CASES}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lib():
    from medical_image_analysis_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _nan(rows, cols, dtype):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device="cuda")


def _untouched(buf, rows, cols, what):
    """Every element of ``buf`` outside [0, rows) x [0, cols) is still the NaN the buffer was filled with, bit for bit."""
    bits = {2: torch.int16, 4: torch.int32}[buf.element_size()]
    nan = torch.full((1,), float("nan"), dtype=buf.dtype, device=buf.device).view(bits)
    b = buf.view(bits)
    outside = torch.cat([b[rows:].reshape(-1), b[:rows, cols:].reshape(-1)])
    bad = int((outside != nan).sum())
    assert bad == 0, f"{what}: {bad} elements written outside [0, {rows}) x [0, {cols})"


def _same_bits(a, b):
    """Bit-for-bit equality that also holds over the NaN sentinel (torch.equal sees NaN != NaN)."""
    bits = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(bits), b.view(bits))


def check_c(c, ref, M, N, what):
    """C[:M, :N] against the float64 ``ref`` with test_gemm_gpu.py's criteria; nothing written outside it."""
    if c.dtype == torch.float32:
        cmp_f32(c[:M, :N], ref, what, rtol=1e-4, atol_rms=1e-4)
    else:
        cmp_stored(c[:M, :N], ref, c.dtype, what)
    _untouched(c, M, N, what)


def _ref_gemm(a, w, bias, act):
    y = a.double() @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    return {0: lambda t: t, 1: torch.relu, 2: F.gelu, 3: F.silu}[act](y)


# ---------------------------------------------------------------------------------------------------------- launches
def _inputs(case, sms):
    """Seeded operands of a case (as test_gemm_gpu.py scales them).  The backward kinds also run the forward kernel here,
    for the saved pre-activations and the forward's h."""
    M, N, K, dt = case.M(sms), case.N, case.K, case.dtype
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if case.kind == "gemm":
        return dict(a=(rn(M, K) / K ** 0.5).to(dt), w=rn(N, K).to(dt), bias=rn(N) if case.bias else None)
    if case.kind in ("gelu_fwd", "gelu_bwd"):
        Kf = K if case.kind == "gelu_fwd" else 96
        inp = dict(x=rn(M, Kf).to(dt), w1=(rn(N, Kf) * Kf ** -0.5).to(dt),
                   b1=(rn(N) * 0.5).to(dt) if case.bias or case.kind == "gelu_bwd" else None)
        if case.kind == "gelu_bwd":
            inp["h_fwd"], inp["pre"] = _gelu_fwd(inp["x"], inp["w1"], inp["b1"], True)
            inp["dy"], inp["w2"] = rn(M, K).to(dt), (rn(K, _pad8(N)) * K ** -0.5).to(dt)
        return inp
    Kf = K if case.kind == "swiglu_fwd" else 96
    inp = dict(x=rn(M, Kf).to(dt), w1=(rn(N, Kf) * Kf ** -0.5).to(dt), w2=(rn(N, Kf) * Kf ** -0.5).to(dt))
    inp["b1"], inp["b2"] = ((rn(N) * 0.5).to(dt), (rn(N) * 0.5).to(dt)) if case.bias or case.kind == "swiglu_bwd" else (None, None)
    if case.kind == "swiglu_bwd":
        inp["h_fwd"], inp["ab"] = _swiglu_fwd(inp["x"], inp["w1"], inp["b1"], inp["w2"], inp["b2"], True)
        inp["dy"], inp["w3"] = rn(M, K).to(dt), (rn(K, _pad64(N)) * K ** -0.5).to(dt)
    return inp


def _pad8(n):
    return (n + 7) // 8 * 8


def _pad64(n):
    return (n + 63) // 64 * 64


def _gemm(case, inp):
    """mia_gemm on a NaN-filled (M + 3, N + ldc_extra) C, bias and activation passed through the C ABI in every mode."""
    lib = _lib()
    a, w, bias = inp["a"], inp["w"], inp["bias"]
    M, K = a.shape
    N = w.shape[0]
    a_dev = a.t().contiguous() if case.amn else a                      # stored [K][M] when MN-major
    w_dev = w.t().contiguous() if case.bmn else w
    c = _nan(M + 3, N + case.ldc_extra, torch.float32 if case.out_f32 else a.dtype)
    lib.call("mia_gemm", "mia_gemm", a.device, a_dev.data_ptr(), w_dev.data_ptr(), _ptr(bias), c.data_ptr(), M, N, K, a_dev.stride(0),
             w_dev.stride(0), c.stride(0), int(case.amn), int(case.bmn), lib.dtype_code(a.dtype), lib.dtype_code(c.dtype), case.act)
    return c


def _gelu_fwd(x, w1, b1, with_pre):
    """mia_gemm_gelu_fwd into NaN-filled (M + 3, Hp + 8) buffers -> (h, pre or None)."""
    lib = _lib()
    M, K = x.shape
    H = w1.shape[0]
    h = _nan(M + 3, _pad8(H) + 8, x.dtype)
    pre = _nan(M + 3, _pad8(H) + 8, x.dtype) if with_pre else None
    b1f = None if b1 is None else b1.float().contiguous()
    lib.call("mia_gemm_gelu_fwd", "gelu_fwd", x.device, x.data_ptr(), w1.data_ptr(), _ptr(b1f), h.data_ptr(), _ptr(pre), M, H, K,
             x.stride(0), w1.stride(0), h.stride(0), 0 if pre is None else pre.stride(0), lib.dtype_code(x.dtype))
    return h, pre


def _gelu_bwd(dy, w2, pre, H):
    """mia_gemm_gelu_bwd into NaN-filled (M + 3, Hp + 8) buffers -> (dpre, h)."""
    lib = _lib()
    M, N = dy.shape
    dpre, h = _nan(M + 3, _pad8(H) + 8, dy.dtype), _nan(M + 3, _pad8(H) + 8, dy.dtype)
    lib.call("mia_gemm_gelu_bwd", "gelu_bwd", dy.device, dy.data_ptr(), w2.data_ptr(), pre.data_ptr(), dpre.data_ptr(), h.data_ptr(), M, H, N,
             dy.stride(0), w2.stride(0), pre.stride(0), dpre.stride(0), h.stride(0), lib.dtype_code(dy.dtype))
    return dpre, h


def _swiglu_fwd(x, w1, b1, w2, b2, with_ab):
    """mia_gemm_swiglu_fwd into NaN-filled h (M + 3, Hp + 8) and ab (M + 3, 2 Hp + 8) -> (h, ab or None)."""
    lib = _lib()
    M, K = x.shape
    H, Hp = w1.shape[0], _pad64(w1.shape[0])
    h = _nan(M + 3, Hp + 8, x.dtype)
    ab = _nan(M + 3, 2 * Hp + 8, x.dtype) if with_ab else None
    b1f, b2f = (None if b is None else b.float().contiguous() for b in (b1, b2))
    lib.call("mia_gemm_swiglu_fwd", "swiglu_fwd", x.device, x.data_ptr(), w1.data_ptr(), w2.data_ptr(), _ptr(b1f), _ptr(b2f), h.data_ptr(),
             _ptr(ab), M, H, K, x.stride(0), w1.stride(0), w2.stride(0), h.stride(0), 0 if ab is None else ab.stride(0),
             lib.dtype_code(x.dtype))
    return h, ab


def _swiglu_bwd(dy, w3, ab, H):
    """mia_gemm_swiglu_bwd into NaN-filled dab (M + 3, 2 Hp + 8) and h (M + 3, Hp + 8) -> (dab, h)."""
    lib = _lib()
    M, N = dy.shape
    Hp = _pad64(H)
    dab, h = _nan(M + 3, 2 * Hp + 8, dy.dtype), _nan(M + 3, Hp + 8, dy.dtype)
    lib.call("mia_gemm_swiglu_bwd", "swiglu_bwd", dy.device, dy.data_ptr(), w3.data_ptr(), ab.data_ptr(), dab.data_ptr(), h.data_ptr(), M, H, N,
             dy.stride(0), w3.stride(0), ab.stride(0), dab.stride(0), h.stride(0), lib.dtype_code(dy.dtype))
    return dab, h


def _launch(case, inp):
    """The launch of the case's target kernel (the forward kinds: with and without the saved pre-activations)."""
    if case.kind == "gemm":
        return _gemm(case, inp)
    if case.kind == "gelu_fwd":
        return _gelu_fwd(inp["x"], inp["w1"], inp["b1"], True), _gelu_fwd(inp["x"], inp["w1"], inp["b1"], False)[0]
    if case.kind == "gelu_bwd":
        return _gelu_bwd(inp["dy"], inp["w2"], inp["pre"], case.N)
    if case.kind == "swiglu_fwd":
        args = (inp["x"], inp["w1"], inp["b1"], inp["w2"], inp["b2"])
        return _swiglu_fwd(*args, True), _swiglu_fwd(*args, False)[0]
    return _swiglu_bwd(inp["dy"], inp["w3"], inp["ab"], case.N)


# ---------------------------------------------------------------------------------------------------------- 2. plain GEMM
@gpu
@pytest.mark.parametrize("cid", [c.id for c in GEMM_CASES])
def test_gemm_parity(cid):
    """C[:M, :N] of every gemm_tn_kernel instantiation against float64 on the same rounded operands; the NaN sentinel
    around it (pitch ldc > N, three extra rows) untouched."""
    case, sms = CASES[cid], _sms()
    assert case.tiles(sms) > sms, (cid, case.tiles(sms), sms)
    inp = _inputs(case, sms)
    c = _launch(case, inp)
    ref = _ref_gemm(inp["a"], inp["w"], inp["bias"], case.act)
    check_c(c, ref, case.M(sms), case.N, f"{cid} M{case.M(sms)}")


# ---------------------------------------------------------------------------------------------------------- 3. fused epilogues
@gpu
@pytest.mark.parametrize("cid", [c.id for c in FUSED_CASES if c.kind == "gelu_fwd"])
def test_gelu_fwd_parity(cid):
    """pre is gemm.linear's fc1 bit for bit (both on the same tile width), h is F.gelu(pre), pads [H, Hp) are 0, nothing is
    written beyond Hp or M, and without pre h has the same bits."""
    from medical_image_analysis_b200 import gemm
    case, sms = CASES[cid], _sms()
    M, H, Hp = case.M(sms), case.N, _pad8(case.N)
    assert case.tiles(sms) > sms
    inp = _inputs(case, sms)
    (h, pre), h_inf = _launch(case, inp)
    assert torch.equal(pre[:M, :H], gemm.linear(inp["x"], inp["w1"], inp["b1"])), cid
    assert torch.equal(h[:M, :H], F.gelu(pre[:M, :H])), cid
    assert (pre[:M, H:Hp] == 0).all() and (h[:M, H:Hp] == 0).all(), cid
    cmp_stored(pre[:M, :H], _ref_gemm(inp["x"], inp["w1"], inp["b1"], 0), case.dtype, f"{cid} pre")
    for buf, nm in ((h, "h"), (pre, "pre"), (h_inf, "h (no pre)")):
        _untouched(buf, M, Hp, f"{cid} {nm}")
    assert _same_bits(h_inf, h), cid


@gpu
@pytest.mark.parametrize("cid", [c.id for c in FUSED_CASES if c.kind == "gelu_bwd"])
def test_gelu_bwd_parity(cid):
    """Full-rank dy and W2: dpre against float64 g gelu'(pre) with g the float64 contraction (an RMS-tied atol, g is an fp32
    accumulation); the recomputed h is the forward's bit for bit; pads are 0; nothing is written beyond Hp or M."""
    case, sms = CASES[cid], _sms()
    M, H, Hp = case.M(sms), case.N, _pad8(case.N)
    assert case.tiles(sms) > sms
    inp = _inputs(case, sms)
    dpre, h = _launch(case, inp)
    g = inp["dy"].double() @ inp["w2"][:, :H].double()
    cmp_stored(dpre[:M, :H], g * _dgelu64(inp["pre"][:M, :H].double()), case.dtype, f"{cid} dpre")
    assert torch.equal(h[:M, :Hp], inp["h_fwd"][:M, :Hp]), cid
    assert (dpre[:M, H:Hp] == 0).all() and (h[:M, H:Hp] == 0).all(), cid
    _untouched(dpre, M, Hp, f"{cid} dpre")
    _untouched(h, M, Hp, f"{cid} h")


@gpu
@pytest.mark.parametrize("cid", [c.id for c in FUSED_CASES if c.kind == "swiglu_bwd"])
def test_swiglu_bwd_parity(cid):
    """Full-rank dy and W3: da / db against float64 (g b s (1 + a (1 - s)), g a s) with g the float64 contraction; the
    recomputed h is the forward's bit for bit; dab's pads are 0; nothing is written beyond 2 Hp, H (h) or M."""
    case, sms = CASES[cid], _sms()
    M, H, Hp = case.M(sms), case.N, _pad64(case.N)
    assert case.tiles(sms) > sms
    inp = _inputs(case, sms)
    dab, h = _launch(case, inp)
    ab = inp["ab"]
    g = inp["dy"].double() @ inp["w3"][:, :H].double()
    a, b = ab[:M, :H].double(), ab[:M, Hp:Hp + H].double()
    s = torch.sigmoid(a)
    cmp_stored(dab[:M, :H], g * b * s * (1 + a * (1 - s)), case.dtype, f"{cid} da")
    cmp_stored(dab[:M, Hp:Hp + H], g * a * s, case.dtype, f"{cid} db")
    assert torch.equal(h[:M, :H], inp["h_fwd"][:M, :H]), cid
    assert (dab[:M, H:Hp] == 0).all() and (dab[:M, Hp + H:2 * Hp] == 0).all(), cid
    _untouched(dab, M, 2 * Hp, f"{cid} dab")
    _untouched(h, M, H, f"{cid} h")


@gpu
@pytest.mark.parametrize("cid", [c.id for c in FUSED_CASES if c.kind == "swiglu_fwd"])
def test_swiglu_fwd_parity(cid):
    """The paired tile at a wide M: a / b are gemm.linear's bit for bit and within one rounding of float64, h within 1 ulp
    of float64 silu(a) b, pads 0, nothing written beyond 2 Hp, H (h) or M, and without ab h has the same bits."""
    from medical_image_analysis_b200 import gemm
    case, sms = CASES[cid], _sms()
    M, H, Hp = case.M(sms), case.N, _pad64(case.N)
    assert case.tiles(sms) > sms and gemm_bn(M, H, sms) == 256
    inp = _inputs(case, sms)
    (h, ab), h_inf = _launch(case, inp)
    x = inp["x"]
    assert torch.equal(ab[:M, :H], gemm.linear(x, inp["w1"], inp["b1"])), cid
    assert torch.equal(ab[:M, Hp:Hp + H], gemm.linear(x, inp["w2"], inp["b2"])), cid
    cmp_stored(ab[:M, :H], _ref_gemm(x, inp["w1"], inp["b1"], 0), case.dtype, f"{cid} a")
    cmp_stored(ab[:M, Hp:Hp + H], _ref_gemm(x, inp["w2"], inp["b2"], 0), case.dtype, f"{cid} b")
    assert (ab[:M, H:Hp] == 0).all() and (ab[:M, Hp + H:2 * Hp] == 0).all(), cid
    a, b = ab[:M, :H].double(), ab[:M, Hp:Hp + H].double()
    _within_ulp(h[:M, :H], a * torch.sigmoid(a) * b, f"{cid} h")
    _untouched(ab, M, 2 * Hp, f"{cid} ab")
    for buf, nm in ((h, "h"), (h_inf, "h (no ab)")):
        _untouched(buf, M, H, f"{cid} {nm}")
    assert _same_bits(h_inf, h), cid


# ---------------------------------------------------------------------------------------------------------- 5. production paths
LINEAR_M = 17000                     # tokens: 133 row blocks, ragged (17000 = 104 mod 128)
VMAMBA_MLP = (96, 384, (8, 56 * 56))     # stage-1 MLP of VMamba at batch 8: in, H, (batch, tokens)
ARM_MLP = (768, 2048, (64, 197))         # ARM-base SwiGLU at batch 64
MAE_ATTN = (1024, 16, 101, 64)           # C, heads, N, B


def _linear_inputs():
    g = torch.Generator(device="cuda").manual_seed(17)
    x = (torch.randn(LINEAR_M, 768, device="cuda", generator=g) / 8).bfloat16()
    w = (torch.randn(768, 768, device="cuda", generator=g) / 8).bfloat16()
    b = torch.randn(768, device="cuda", generator=g)
    dy = torch.randn(LINEAR_M, 768, device="cuda", generator=g).bfloat16()
    return x, w, b, dy


def _linear_run(x, w, b, dy):
    from medical_image_analysis_b200.gemm import linear
    xg, wg = x.clone().requires_grad_(), w.clone().requires_grad_()
    y = linear(xg, wg, b)
    y.backward(dy)
    return y, xg.grad, wg.grad


def _gelu_op_inputs():
    K, H, lead = VMAMBA_MLP
    m = _vmamba_mlp(K, H, 12, torch.bfloat16)
    g = torch.Generator(device="cuda").manual_seed(3)
    return m, torch.randn(*lead, K, device="cuda", generator=g).bfloat16(), torch.randn(*lead, K, device="cuda", generator=g)


def _gelu_op(m, x):
    from medical_image_analysis_b200.gemm import gelu_mlp_fn
    return gelu_mlp_fn(x, m.fc1.weight, m.fc1.bias, m.fc2.weight, m.fc2.bias)


def _swiglu_op_inputs():
    K, H, lead = ARM_MLP
    m = _swiglu_mlp(K, H, 12, torch.bfloat16)
    g = torch.Generator(device="cuda").manual_seed(4)
    return m, torch.randn(*lead, K, device="cuda", generator=g).bfloat16(), torch.randn(*lead, K, device="cuda", generator=g)


def _swiglu_op(m, x):
    from medical_image_analysis_b200.arm import swiglu_fn
    return swiglu_fn(x, m.w1.weight, m.w1.bias, m.w2.weight, m.w2.bias, m.w3.weight, m.w3.bias)


def _attn_inputs():
    C, H, N, B = MAE_ATTN
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, N, C, device="cuda", generator=g).bfloat16().requires_grad_()
    dy = torch.randn(B, N, C, device="cuda", generator=g).bfloat16()
    return x, _attn_params(C, H, torch.bfloat16), dy


def _attn_op(x, params):
    from medical_image_analysis_b200 import mae
    return mae.attention_fn(x, *params, MAE_ATTN[1])


def _production_runs():
    """Name -> a callable running that op's forward and backward once."""
    def gelu():
        m, x, w = _gelu_op_inputs()
        return _gelu_grads(m, x, _gelu_op, w)

    def swiglu():
        m, x, w = _swiglu_op_inputs()
        return _swiglu_grads(m, x, _swiglu_op, w)

    def attn():
        x, params, dy = _attn_inputs()
        return _attn_grads(lambda: _attn_op(x, params), x, params, dy)

    return {"linear": lambda: _linear_run(*_linear_inputs()), "gelu_mlp_fn": gelu, "swiglu_fn": swiglu, "attention_fn": attn}


@gpu
def test_linear_at_training_size():
    """gemm.linear 768 -> 768 over 17 000 tokens: y, dx and dW (K = the token count) with test_gemm_gpu.py's criteria."""
    x, w, b, dy = _linear_inputs()
    y, dx, dw = _linear_run(x, w, b, dy)
    xr, wr = x.double().requires_grad_(), w.double().requires_grad_()
    yr = F.linear(xr, wr, b.double())
    yr.backward(dy.double())
    cmp_stored(y, yr, torch.bfloat16, "linear y")
    cmp_stored(dx, xr.grad, torch.bfloat16, "linear dx", n_ulp=2.0)
    cmp_stored(dw, wr.grad, torch.bfloat16, "linear dw", n_ulp=2.0)


def _no_further(got, comp, ref, rel_fn):
    for k, (a, c, r) in {"out": (got[0], comp[0], ref[0]), **{k: (got[1][k], comp[1][k], ref[1][k]) for k in got[1]}}.items():
        rel, worst = rel_fn(a, r)
        crel, _ = rel_fn(c, r)
        assert rel <= 0.02 and worst <= 0.5, f"{k}: rel RMS err {rel:.3e}, worst err / RMS(ref) {worst:.3e}"
        assert rel <= 1.25 * crel + 1e-4, f"{k}: rel RMS err {rel:.3e}, the composition's {crel:.3e}"


@gpu
def test_gelu_mlp_fn_at_vmamba_stage1():
    """VMamba stage-1 MLP (96 -> 384 -> 96) over 8 x 56 x 56 tokens against float64, no further from it than the composition."""
    m, x, w = _gelu_op_inputs()
    got = _gelu_grads(m, x, _gelu_op, w)
    comp = _gelu_grads(m, x, lambda m, x: m._forward_composed(x), w)
    _no_further(got, comp, _gelu_ref64(m, x, w), _rel)


def _swiglu_ref64(m, x, w):
    """test_swiglu_fused_gpu._ref64 on the device: at M = 12 608 its CPU float64 backward is ~0.4 TFLOP."""
    P = {n: p.detach().double().requires_grad_() for n, p in m.named_parameters()}
    x64 = x.detach().double().requires_grad_()
    hidden = F.silu(F.linear(x64, P["w1.weight"], P["w1.bias"])) * F.linear(x64, P["w2.weight"], P["w2.bias"])
    out = F.linear(hidden, P["w3.weight"], P["w3.bias"])
    (out * w.double()).sum().backward()
    return out, {"x": x64.grad, **{n: p.grad for n, p in P.items()}}


@gpu
def test_swiglu_fn_at_arm_base():
    """ARM-base SwiGLU (768 -> 2048 -> 768) over 64 x 197 tokens against float64, no further from it than the composition."""
    m, x, w = _swiglu_op_inputs()
    got = _swiglu_grads(m, x, _swiglu_op, w)
    comp = _swiglu_grads(m, x, lambda m, x: m._forward_composed(x), w)
    _no_further(got, comp, _swiglu_ref64(m, x, w), _rel)


@gpu
def test_attention_fn_at_mae_size():
    """ViT-MAE attention (C 1024, 16 heads, 101 tokens, batch 64) against float64, no further from it than the composition
    (test_attention_fused_gpu.py's criterion)."""
    from medical_image_analysis_b200 import mae
    C, H, N, B = MAE_ATTN
    x, params, dy = _attn_inputs()
    got = _attn_grads(lambda: _attn_op(x, params), x, params, dy)
    m = mae.Attention(C, num_heads=H, qkv_bias=True).cuda().to(torch.bfloat16)
    with torch.no_grad():
        for dst, src in zip((m.qkv.weight, m.qkv.bias, m.proj.weight, m.proj.bias), params):
            dst.copy_(src)
    comp = _attn_grads(lambda: m._forward_composed(x), x, [m.qkv.weight, m.qkv.bias, m.proj.weight, m.proj.bias], dy)
    x64 = x.detach().double().requires_grad_()
    p64 = [t.detach().double().requires_grad_() for t in params]
    y64 = _float64_block(x64, *p64, H)
    y64.backward(dy.double())
    ref = [y64.detach(), x64.grad] + [t.grad for t in p64]
    for name, a, c, r in zip(["y", "dx", "dWqkv", "dbqkv", "dWproj", "dbproj"], got, comp, ref):
        ours, theirs = _rms_err(a, r), _rms_err(c, r)
        assert ours <= SDPA_FACTOR * theirs + 1e-6 * float(r.abs().max()), (name, ours, theirs)


# ---------------------------------------------------------------------------------------------------------- 4. launched kernels
def launches():
    """Run in a child interpreter: the GEMM-family kernels each case launches (its target call only), the tile width
    gemm.linear takes for each GELU forward case's fc1, and the kernels of each production op's forward and backward."""
    sms = _sms()
    out = {"cases": {}, "linear_of_gelu_fwd": {}, "ops": {}}
    for cid, case in CASES.items():
        inp = _inputs(case, sms)
        n = 2 if case.kind in ("gelu_fwd", "swiglu_fwd") else 1
        out["cases"][cid] = [short_name(s) for s in kernel_trace.names_of(lambda: _launch(case, inp), KERNEL, n)]
        if case.kind == "gelu_fwd":
            from medical_image_analysis_b200 import gemm
            out["linear_of_gelu_fwd"][cid] = [short_name(s) for s in kernel_trace.names_of(
                lambda: gemm.linear(inp["x"], inp["w1"], inp["b1"]), KERNEL)]
        del inp
    for name, run in _production_runs().items():
        out["ops"][name] = sorted({short_name(s) for s in kernel_trace.names_of(run, KERNEL, 3)})
    return out


@pytest.fixture(scope="module")
def traced():
    return kernel_trace.in_child("tests.test_gemm_tiles_gpu:launches")


@gpu
def test_every_case_launches_its_target(traced):
    """Each case ran exactly the instantiation the Python replica of the host rules assigns it, and nothing else; each
    GELU forward case's fc1 and gemm.linear's ran on the same tile width (so pre has gemm.linear's k order)."""
    sms = _sms()
    wrong = {cid: (sorted(set(traced["cases"].get(cid, []))), c.target(sms)) for cid, c in CASES.items()
             if set(traced["cases"].get(cid, [])) != {c.target(sms)}}
    assert not wrong, wrong
    for cid, names in traced["linear_of_gelu_fwd"].items():
        bn = CASES[cid].target(sms).split(", ")[1]
        assert names and all(n.startswith(f"gemm_tn_kernel<{bn}, ") for n in names), (cid, names)


@gpu
def test_all_instantiations_launched_and_compared(traced):
    """The cases' targets are the full list of 40: every instantiation runs in at least one parity case above."""
    sms = _sms()
    targets = {c.target(sms) for c in CASES.values()}
    launched = {n for names in traced["cases"].values() for n in names}
    assert targets == set(INSTANTIATIONS) == launched, (sorted(set(INSTANTIATIONS) - targets), sorted(targets - set(INSTANTIATIONS)))
    print(f"{len(targets)}/{len(INSTANTIATIONS)} instantiations launched and compared ({len(CASES)} cases, {sms} SMs)")


@gpu
def test_production_ops_run_wide_tiles(traced):
    """At these training sizes each op runs a 256-wide tile somewhere; attention's qkv dgrad is the 256-wide MN-major-B GEMM."""
    for name, names in traced["ops"].items():
        assert any(re.search(r"kernel<(\d, )?256, ", n) for n in names), (name, names)
    assert "gemm_tn_kernel<256, 4, false, true, false>" in traced["ops"]["attention_fn"], traced["ops"]["attention_fn"]


# ---------------------------------------------------------------------------------------------------------- CPU checks
@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump and the built library (python -c 'import __graft_entry__ as g; g.build()')")
def test_instantiation_list_is_the_built_one():
    """INSTANTIATIONS is exactly the set of gemm_*_kernel functions with SASS in libmia_scan.so (cuobjdump -res-usage lists
    the functions cuobjdump -sass would disassemble, without disassembling them), so a new instantiation needs a case."""
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    built = set()
    for kern, args in re.findall(r"Function \S*?\d(gemm_(?:tn|gelu|swiglu)_kernel)I((?:L[ib]\d+E)+)E", out):
        vals = [v if t == "i" else _tf(v == "1") for t, v in re.findall(r"L([ib])(\d+)E", args)]
        built.add(f"{kern}<{', '.join(vals)}>")
    assert built == set(INSTANTIATIONS), (sorted(built - set(INSTANTIATIONS)), sorted(set(INSTANTIATIONS) - built))
    assert len(INSTANTIATIONS) == len(set(INSTANTIATIONS)) == 40


WIDE_CASES = [c for c in GEMM_CASES if c.id.startswith("gemm-BN256-ak_bk-bf16") and c.K == 600]


@pytest.mark.parametrize("out", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("cid", [c.id for c in WIDE_CASES])
def test_criteria_reject_subtly_wrong_results(cid, out):
    """The section-2 comparison (check_c) on float64 "mutants" of a correct result at the 256-wide shapes (M as on a 132-SM
    H100 SXM, K = 600): a dropped last K block, the two 64-column chunks of a 256 tile's upper half swapped, the in-range
    rows of the last partial M tile zeroed, the bias read one column off, and an fp16 output rounded as bf16 must all fail;
    the correct result, rounded to the output type, passes."""
    case = CASES[cid]
    M, N, K = case.M(132), case.N, case.K
    in_dt = torch.float16 if out == "f16" else torch.bfloat16
    out_dt = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}[out]
    g = torch.Generator().manual_seed(M + N)
    a = (torch.randn(M, K, generator=g) / K ** 0.5).to(in_dt).double()
    w = torch.randn(N, K, generator=g).to(in_dt).double()
    bias = torch.randn(N + 1, generator=g).double()
    ref = a @ w.t() + bias[:N]

    def buf(vals):
        c = torch.full((M + 3, N + 1), float("nan"), dtype=out_dt)
        c[:M, :N] = vals.to(out_dt)
        return c

    check_c(buf(ref), ref, M, N, "correct")
    kt = (K - 1) // 64 * 64
    swapped = ref.clone()
    swapped[:, 128:192], swapped[:, 192:256] = ref[:, 192:256], ref[:, 128:192]
    zeroed = ref.clone()
    zeroed[(M - 1) // 128 * 128:] = 0
    mutants = {"last K block dropped": a[:, :kt] @ w[:, :kt].t() + bias[:N], "upper-half chunks swapped": swapped,
               "last M tile zeroed": zeroed, "bias one column off": a @ w.t() + bias[1:]}
    if out == "f16":
        mutants["rounded as bf16"] = ref.to(torch.bfloat16).double()
    for what, vals in mutants.items():
        with pytest.raises(AssertionError):
            check_c(buf(vals), ref, M, N, what)
    stray = buf(ref)
    stray[M, 0] = 0                                                    # one store past the last row
    with pytest.raises(AssertionError):
        check_c(stray, ref, M, N, "stray store")
