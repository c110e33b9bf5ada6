"""Every instantiation of the SS2D core's kernels against float64: the epilogue pair of csrc/ss2d_core.cu (CrossMerge + bf16
cast + LayerNorm + z gate, and its backward with the CrossScan adjoint) and the CrossScan1b1 permutations of
csrc/cross_scan.cu, at the dtypes, shapes, layouts and values where they go wrong.

The epilogue cases call mia_ss2d_merge_norm_fwd / _bwd directly.  They cover the five (ys, out) dtype pairs and the three
backward dtypes with each gate (none, y z, y silu(z)), the inference forward without yb / mean / rstd, D from 1 to 3626 (the
largest the shared memory holds), partial 4 x 8 tiles, z read as the second half of an in_proj-shaped buffer, token-major,
channel-major or through a negative token stride, constant rows, a large common offset, fp16 gates near the top of the fp16
range, the largest batch the entry points accept and backward grids of hundreds of partial sums.  The forward copies
mia_cross_merge's summation order, which depends on the path the merge takes for these sizes (cross_merge_path): the cases
reach the vectorised path, the staged path (L % 4 != 0, ys one element off 16-byte alignment, fp32 planes too large for the
vectorised kernel, B D^2 >= 2^32), and the direct path (L > 51200).  On planted tokens the paired and unpaired orders give
different bf16 values, so yb shows which order ran.

Every operand and output sits in a NaN-filled buffer with guard bands: an input read out of bounds turns a result NaN, an
output written out of bounds shows bit for bit.  Each case runs twice with bit-identical results.  A child interpreter
records the kernels each case launched (kernel_trace).  CPU tests check the list against the built library, the Python
replicas of the launch rules against the library's workspace query, and that the criteria reject float64 mutants."""
import ctypes
import math
import os
import re
import shutil
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from oracle.ss2d_ref import cross_scan_ref
from tests import kernel_trace
from tests.parity import cmp_f32, cmp_stored
from tests.test_conv_tiles_gpu import LIB, _bits, _demangled_kernels, _same_bits
from tests.test_ss2d_core_fused_gpu import _stored, _torch_1b1

gpu = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
TNAME = {F32: "float", F16: "__half", BF16: "__nv_bfloat16"}
DT_ID = {F32: "f32", BF16: "bf16", F16: "f16"}
KTH, KTW = 4, 8                          # the epilogue's image tile: 4 rows x 8 columns = 32 tokens
CS_SMEM = 200 * 1024                     # kCsSmemMax of cross_scan.cu
EPS = 1e-5
GUARD = 64                               # NaN elements in front of and behind every operand

FWD_PAIRS = [(F32, F32), (F32, BF16), (BF16, BF16), (F32, F16), (F16, F16)]
EPI_KERNELS = ([f"merge_norm_fwd_kernel<{TNAME[y]}, {TNAME[o]}>" for y, o in FWD_PAIRS]
               + [f"merge_norm_bwd_kernel<{TNAME[t]}>" for t in (F32, BF16, F16)] + ["merge_norm_bwd_finalize"])
K1B1_KERNELS = [f"cross_1b1_kernel<{TNAME[t]}, {v}>" for t in (F32, BF16, F16) for v in ("false", "true")] + \
               [f"cross_1b1_direct_kernel<{TNAME[t]}>" for t in (F32, BF16, F16)]
INSTANTIATIONS = EPI_KERNELS + K1B1_KERNELS
CS_BASES = ("cross_scan_kernel", "cross_merge_kernel", "cross_scan_vec_kernel", "cross_merge_vec_kernel", "cross_scan_direct_kernel",
            "cross_merge_direct_kernel", "cross_1b1_kernel", "cross_1b1_direct_kernel", "silu_gate_kernel")
KERNEL = re.compile(r"\b(merge_norm_(?:fwd|bwd)_(?:kernel|finalize)|cross_1b1_(?:direct_)?kernel)\b")
MERGE = re.compile(r"\bcross_merge_(?:vec_|direct_)?kernel\b")


def _cdiv(a, b):
    return -(-a // b)


def _es(dtype):
    return torch.empty((), dtype=dtype).element_size()


# ---------------------------------------------------------------------------------------------------------- replicas
def grid_tiles(H, W):
    """CTAs per image of the epilogue pair (grid_tiles in ss2d_core.cu): one per 4 x 8 tile, the last row / column partial."""
    return _cdiv(H, KTH) * _cdiv(W, KTW)


def cross_merge_path(merge, aligned, B, C, H, W, es):
    """The kernel mia_cross_scan / mia_cross_merge launch (cross_merge_path in cross_scan.cu): vectorised when L % 4 == 0, the
    tensor is aligned, a plane's four orders fit shared memory and the multiply-high divisions are exact; else staged while
    one plane fits shared memory (as fp32 in the merge), else direct gathers."""
    L, n_planes = H * W, B * C
    vplanes = min(CS_SMEM // (L * es * (4 if merge else 1)), 8)
    if L % 4 == 0 and aligned and vplanes >= 1 and vplanes * L * L < (1 << 32) // 4 and n_planes * C < (1 << 32):
        return "vec"
    return "staged" if L * (4 if merge else es) <= CS_SMEM else "direct"


def launch_1b1(B, C, H, W, es, aligned):
    """(path, planes per CTA, CTAs) of mia_cross_scan_1b1 / mia_cross_merge_1b1 (launch_1b1 in cross_scan.cu): up to 8 planes
    per CTA in shared memory, 4-element accesses when L % 4 == 0 and both tensors are aligned; element-wise gathers over a
    grid capped at 16 CTAs per SM of a 132-SM H100 when one plane exceeds shared memory."""
    L, n_planes = H * W, B * 4 * C
    planes = min(CS_SMEM // (L * es), 8)
    if planes >= 1:
        return ("vec" if L % 4 == 0 and aligned else "staged"), planes, _cdiv(n_planes, planes)
    return "direct", 1, min(_cdiv(n_planes * L, 256), 132 * 16)


def _col(t, H, W):
    """(..., L) in column-major scan order (position w H + h holds token h W + w) -> image order."""
    return t.unflatten(-1, (W, H)).transpose(-1, -2).flatten(-2)


def merge_replica(ys, H, W, pairs, col=True):
    """mia_cross_merge in float32 on the host: (B, 4, D, L) -> (B, D, L) in ys's dtype.  The four orders at a token are
    summed as (r0 + r2) + (c1 + c3) on the staged path (pairs) and as ((r0 + r2) + c1) + c3 on the others.  col=False reads
    the column-major orders at the row-major position l instead of w H + h (a mutant)."""
    f = ys.float()
    r0, r2 = f[:, 0], f[:, 2].flip(-1)
    c1, c3 = f[:, 1], f[:, 3].flip(-1)
    if col:
        c1, c3 = _col(c1, H, W), _col(c3, H, W)
    v = (r0 + r2) + (c1 + c3) if pairs else ((r0 + r2) + c1) + c3
    return v.to(ys.dtype)


# Planted tokens: r0 = 1, r2 = R2[ys dtype], c1 = c3 = 2^-24.  Summed in pairs, c1 + c3 = 2^-23 lifts r0 + r2 (a bf16 rounding
# tie, and for fp16 ys also an fp16 one) just above the tie, so the value rounds up to 1 + 2^-7; summed one by one each
# 2^-24 is a tie lost to round-to-even, and the value rounds down to 1.
R2 = {F32: 2.0 ** -8, BF16: 2.0 ** -8, F16: 2.0 ** -8 + 2.0 ** -11}
TINY = 2.0 ** -24
PLANTED_YB = {True: 1.0 + 2.0 ** -7, False: 1.0}          # pairs -> the bf16 value of the planted token


def plant_orders(TY):
    """The bf16 values of a planted token in the paired and the unpaired order, through merge_replica."""
    ys = torch.tensor([1.0, TINY, R2[TY], TINY]).to(TY).view(1, 4, 1, 1)
    return {p: float(merge_replica(ys, 1, 1, p).to(BF16)) for p in (True, False)}


# ---------------------------------------------------------------------------------------------------------- operands
class Frame:
    """One operand in a NaN-filled flat buffer: GUARD elements in front (plus ``off`` more, to misalign it) and behind.
    ``strides`` are element strides of the operand's index order, ``start`` the offset of its element 0 in the buffer's body;
    ``rev`` names a dimension the kernel walks backwards (a negative stride: element i sits at memory index n - 1 - i)."""

    def __init__(self, shape, dtype, strides=None, numel=None, start=0, off=0, rev=None, dev="cuda"):
        self.shape, self.dtype, self.rev = tuple(shape), dtype, rev
        self.strides = tuple(strides) if strides is not None else tuple(torch.empty(shape, device="meta").stride())
        numel = math.prod(shape) if numel is None else numel
        self.base = GUARD + off + start
        self.buf = torch.full((numel + 2 * GUARD + off,), float("nan"), dtype=dtype, device=dev)

    def region(self, buf=None):
        """The operand's elements as a view of ``buf`` (default: its own), in memory order."""
        return (self.buf if buf is None else buf).as_strided(self.shape, self.strides, self.base)

    def value(self):
        r = self.region()
        return r.flip(self.rev) if self.rev is not None else r

    def set(self, v):
        self.region().copy_(v.flip(self.rev) if self.rev is not None else v)
        return self

    def ptr(self):
        return self.buf.data_ptr() + self.base * self.buf.element_size()

    def bdl(self):
        """struct mia_bdl of a (B, D, L) operand."""
        from medical_image_analysis_b200 import _lib
        s = list(self.strides)
        p = self.ptr()
        if self.rev is not None:
            p += (self.shape[self.rev] - 1) * s[self.rev] * self.buf.element_size()
            s[self.rev] = -s[self.rev]
        return _lib.MiaBdl(p, *s)

    def untouched(self, what):
        rest = self.buf.clone()
        self.region(rest).fill_(float("nan"))
        bad = int((_bits(rest) != _bits(torch.full_like(rest, float("nan")))).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the operand"


def bdl_frame(layout, B, D, L, dtype, dev="cuda"):
    """A (B, D, L) z / dz operand in one of the layouts the epilogue reads and writes in place:

    xz   the second half of an in_proj-shaped (B, H, W, 2 D) buffer (how SS2DCoreFn passes z): token stride 2 D;
    tm   a contiguous token-major (B, H, W, D) tensor;
    cm   channel-major (B, D, L);
    neg  token-major, walked from the last token: token stride -D."""
    if layout == "xz":
        return Frame((B, D, L), dtype, (2 * L * D, 1, 2 * D), B * L * 2 * D, start=D, dev=dev)
    if layout == "cm":
        return Frame((B, D, L), dtype, (D * L, L, 1), dev=dev)
    assert layout in ("tm", "neg"), layout
    return Frame((B, D, L), dtype, (L * D, 1, D), rev=2 if layout == "neg" else None, dev=dev)


# ---------------------------------------------------------------------------------------------------------- case tables
@dataclass
class Case:
    """One forward (and backward) call of the epilogue pair on (B, D, H, W).  ``off``: ys one element past 16-byte alignment;
    ``stats``: yb / mean / rstd written (False: the inference forward); ``values``: randn, const (every even token constant
    over the channels), offset (mean >> std) or huge (fp16 gates near the top of the fp16 range)."""
    ys: torch.dtype
    out: torch.dtype
    gate: int
    shape: tuple
    z: str = "xz"
    dz: str = "xz"
    off: int = 0
    stats: bool = True
    bwd: bool = True
    values: str = "randn"
    note: str = ""

    @property
    def id(self):
        B, D, H, W = self.shape
        s = f"{DT_ID[self.ys]}-{DT_ID[self.out]}-g{self.gate}-B{B}_D{D}_{H}x{W}"
        if self.gate:
            s += f"-z_{self.z}" + (f"-dz_{self.dz}" if self.bwd else "")
        s += "-off1" * (self.off == 1) + ("" if self.stats else "-infer") + ("" if self.bwd or not self.stats else "-fwd")
        return s + ("" if self.values == "randn" else f"-{self.values}") + (f"-{self.note}" if self.note else "")

    @property
    def path(self):
        B, D, H, W = self.shape
        return cross_merge_path(True, self.off % 4 == 0, B, D, H, W, _es(self.ys))

    @property
    def pairs(self):
        return self.path == "staged"

    def target(self):
        t = {f"merge_norm_fwd_kernel<{TNAME[self.ys]}, {TNAME[self.out]}>"}
        if self.bwd:
            t |= {f"merge_norm_bwd_kernel<{TNAME[self.out]}>", "merge_norm_bwd_finalize"}
        return t


SHAPES = [(3, 33, 6, 5), (2, 96, 7, 9), (1, 768, 14, 14), (2, 7, 1, 13), (1, 2048, 11, 1), (1, 3626, 3, 2), (2, 1, 14, 14),
          (1, 96, 80, 80)]
Z_LAYOUTS = ("xz", "tm", "cm", "neg")
MAX_BATCH = 65535


def _cases():
    out = []
    for i, (ys, o) in enumerate(FWD_PAIRS):
        for gate in (0, 1, 2):
            j = 3 * i + gate
            out.append(Case(ys, o, gate, SHAPES[j % 8], z=Z_LAYOUTS[j % 4], dz=Z_LAYOUTS[(j + 1) % 4]))
        # the inference forward: no yb / mean / rstd
        out.append(Case(ys, o, (i + 1) % 3, SHAPES[(i * 3 + 1) % 8], z=Z_LAYOUTS[(i + 2) % 4], stats=False, bwd=False))
    # the merge's order: staged by misalignment, fp32 planes too large for the vectorised kernel (and a 2-byte plane of the
    # same size that stays vectorised), direct gathers, and B D^2 >= 2^32 at a 2 x 2 map
    out += [Case(F32, BF16, 2, (2, 96, 14, 14), off=1), Case(BF16, BF16, 1, (1, 33, 14, 14), z="neg", off=1),
            Case(F16, F16, 2, (2, 7, 8, 8), z="cm", dz="neg", off=1),
            Case(F32, F16, 2, (1, 7, 120, 120), z="tm", dz="cm"), Case(F32, F32, 0, (1, 33, 120, 120)),
            Case(BF16, BF16, 1, (1, 7, 120, 120), z="cm", dz="tm"),
            Case(F32, BF16, 2, (1, 7, 227, 227), z="neg", dz="xz"), Case(F16, F16, 1, (1, 3, 227, 227), z="xz", dz="neg"),
            Case(BF16, BF16, 0, (1024, 2048, 2, 2), bwd=False, note="bdd")]
    # value edges
    out += [Case(F32, F32, 2, (2, 96, 7, 9), z="cm", dz="tm", values="const"), Case(BF16, BF16, 1, (1, 768, 14, 14), values="const"),
            Case(F16, F16, 2, (3, 33, 6, 5), z="tm", dz="xz", values="const"),
            Case(F32, BF16, 2, (2, 96, 14, 14), values="offset"), Case(F16, F16, 0, (3, 33, 6, 5), values="offset"),
            Case(F32, F16, 2, (2, 96, 14, 14), z="neg", dz="cm", values="huge"), Case(F16, F16, 2, (2, 33, 7, 9), values="huge"),
            Case(F16, F16, 1, (1, 768, 14, 14), z="cm", dz="xz", values="huge")]
    # the largest batch, and backward grids of 512 partial sums for the finalize
    out += [Case(BF16, BF16, 2, (MAX_BATCH, 7, 2, 3), note="maxbatch"), Case(F16, F16, 1, (MAX_BATCH, 1, 1, 1), z="tm", dz="cm", note="maxbatch"),
            Case(F32, F32, 2, (64, 96, 14, 14), note="parts"), Case(BF16, BF16, 1, (64, 96, 14, 14), z="tm", dz="neg", note="parts"),
            Case(F16, F16, 2, (64, 96, 14, 14), z="neg", dz="tm", note="parts")]
    return out


@dataclass
class Case1b1:
    """One mia_cross_scan_1b1 (merge False) or mia_cross_merge_1b1 call; ``off``: both tensors one element off alignment."""
    dtype: torch.dtype
    shape: tuple
    merge: bool
    off: int = 0

    @property
    def id(self):
        B, C, H, W = self.shape
        return f"{'merge' if self.merge else 'scan'}_1b1-{DT_ID[self.dtype]}-B{B}_C{C}_{H}x{W}" + "-off1" * (self.off == 1)

    @property
    def launch(self):
        B, C, H, W = self.shape
        return launch_1b1(B, C, H, W, _es(self.dtype), self.off % 4 == 0)

    def target(self):
        path = self.launch[0]
        if path == "direct":
            return {f"cross_1b1_direct_kernel<{TNAME[self.dtype]}>"}
        return {f"cross_1b1_kernel<{TNAME[self.dtype]}, {'true' if path == 'vec' else 'false'}>"}


def _cases_1b1():
    out = []
    for dt in (F32, BF16, F16):
        big = (1, 6, 227, 227) if dt == F32 else (1, 3, 321, 321)      # one plane over 200 KB
        for merge in (False, True):
            out += [Case1b1(dt, (1, 5, 14, 14), merge), Case1b1(dt, (1, 3, 7, 9), merge), Case1b1(dt, (1, 5, 14, 14), merge, off=1),
                    Case1b1(dt, (1, 5, 120, 120), merge), Case1b1(dt, big, merge)]
    return out


CASES = {c.id: c for c in _cases()}
CASES_1B1 = {c.id: c for c in _cases_1b1()}
assert len(CASES) == len(_cases()) and len(CASES_1B1) == len(_cases_1b1()), "case ids must be unique"


# ---------------------------------------------------------------------------------------------------------- inputs
def _planted(case):
    """(b, c, l) of the planted tokens: the last token of the last image, a middle and a second token (odd tokens only when
    the even ones have constant rows)."""
    B, D, H, W = case.shape
    L = H * W
    toks = {(B - 1, L - 1), (0, L // 2), (B // 2, 1 % L)}
    if case.values == "const":
        toks = {(b, l) for b, l in toks if l % 2 == 1}
    return sorted((b, (7 * l + b) % D, l) for b, l in toks)


def _inputs(case):
    """Seeded host operands: ys (B, 4, D, L), LayerNorm weight / bias, z (B, D, L), dy (B, L, D), and the planted tokens."""
    B, D, H, W = case.shape
    L = H * W
    TY, TO = case.ys, case.out
    g = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    if case.values == "offset":
        img = torch.randn(B, 4, D, H, W, generator=g) * 0.25 + 8.0        # the merged value: 32 +- 0.5
    else:
        img = torch.randn(B, 4, D, H, W, generator=g) * 0.5 + 0.1
    if case.values == "const":                                         # the even tokens: order 0 constant over D, others 0
        row = torch.randn(B, 1, 1, H, W, generator=g).expand(B, 1, D, H, W)
        even = (torch.arange(L) % 2 == 0).view(1, 1, 1, H, W)
        img = torch.where(even, torch.cat([row, torch.zeros(B, 3, D, H, W)], 1), img)
    planted = _planted(case)
    for b, c, l in planted:
        h, w = divmod(l, W)
        img[b, :, c, h, w] = torch.tensor([1.0, TINY, R2[TY], TINY])
    ys = _torch_1b1(img).to(TY)                                        # order k holds token (h, w) at its scan position
    del img
    if case.values == "huge":                                          # small LayerNorm output, |z| up to 65504
        weight, bias = torch.rand(D, generator=g) * 0.01 + 0.005, (torch.rand(D, generator=g) - 0.5) * 0.02
        mag = torch.rand(B, D, L, generator=g) * (65504 - 8192) + 8192
        sign = torch.where(torch.rand(B, D, L, generator=g) < 0.5, -1.0, 1.0)
        z = torch.where(torch.rand(B, D, L, generator=g) < 0.5, sign * mag, torch.randn(B, D, L, generator=g) * 4)
        dy = torch.randn(B, L, D, generator=g) * 0.01
    else:
        weight, bias = torch.rand(D, generator=g) + 0.5, torch.rand(D, generator=g) - 0.5
        z = torch.randn(B, D, L, generator=g) * 2
        dy = torch.randn(B, L, D, generator=g)
    return dict(ys=ys, w=weight, b=bias, z=z.to(TO), dy=dy.to(TO), planted=planted)


def _device(case, P):
    B, D, H, W = case.shape
    L = H * W
    return dict(ys=Frame((B, 4, D, L), case.ys, off=case.off).set(P["ys"].cuda()), w=Frame((D,), F32).set(P["w"].cuda()),
                b=Frame((D,), F32).set(P["b"].cuda()), z=bdl_frame(case.z, B, D, L, case.out).set(P["z"].cuda()) if case.gate else None,
                dy=Frame((B, L, D), case.out).set(P["dy"].cuda()) if case.bwd else None)


def _lib():
    from medical_image_analysis_b200 import _lib
    return _lib


def _launch(case, Q):
    """One forward (and backward) on NaN-framed outputs -> {name: Frame}."""
    lib = _lib()
    B, D, H, W = case.shape
    L = H * W
    dev, by, TO = torch.device("cuda"), ctypes.byref, case.out
    none = lib.MiaBdl(None, 0, 0, 0)
    ln = lib.MiaLn(Q["w"].ptr(), Q["b"].ptr(), EPS)
    zb = Q["z"].bdl() if case.gate else none
    R = {"out": Frame((B, L, D), TO)}
    if case.stats:
        R.update(yb=Frame((B, L, D), BF16), mean=Frame((B, L), F32), rstd=Frame((B, L), F32))
    p = lambda k: R[k].ptr() if k in R else None
    lib.call("mia_ss2d_merge_norm_fwd", "fwd", dev, Q["ys"].ptr(), by(ln), by(zb), case.gate, R["out"].ptr(), p("yb"), p("mean"),
             p("rstd"), B, D, H, W, lib.dtype_code(case.ys), lib.dtype_code(TO))
    if case.bwd:
        R.update(dout=Frame((B, 4, D, L), F32), dw=Frame((D,), F32), db=Frame((D,), F32))
        if case.gate:
            R["dz"] = bdl_frame(case.dz, B, D, L, TO)
        ws = torch.full((int(lib.lib().mia_ss2d_merge_norm_bwd_workspace(B, D, H, W)),), 255, dtype=torch.uint8, device=dev)   # NaN
        lib.call("mia_ss2d_merge_norm_bwd", "bwd", dev, Q["dy"].ptr(), R["yb"].ptr(), R["mean"].ptr(), R["rstd"].ptr(), by(ln), by(zb),
                 case.gate, by(R["dz"].bdl() if case.gate else none), R["dout"].ptr(), R["dw"].ptr(), R["db"].ptr(), ws.data_ptr(),
                 ws.numel(), B, D, H, W, lib.dtype_code(TO))
    return R


def _cross_merge(case, Q):
    """mia_cross_merge on the same ys view (its output aligned) -> (B, D, L) in ys's dtype."""
    B, D, H, W = case.shape
    y = torch.empty((B, D, H * W), dtype=case.ys, device="cuda")
    _lib().call("mia_cross_merge", "cross_merge", y.device, Q["ys"].ptr(), y.data_ptr(), B, D, H, W, _lib().dtype_code(case.ys))
    return y


# ---------------------------------------------------------------------------------------------------------- float64 checks
def _reference(case, P, yb):
    """float64 statement of the epilogue after the cast, on the bf16 pre-norm plane yb (B, L, D), with the module's
    roundings: the LayerNorm output and silu(z) stored in the output dtype, the gate's product and its gradients computed in
    it -> mean, rstd, out and, for the backward, d yb, dz (B, L, D), dweight, dbias."""
    B, D, H, W = case.shape
    x = yb.double().requires_grad_()
    mean = x.detach().mean(-1)
    var = (x.detach() - mean[..., None]).pow(2).mean(-1)
    w, b = P["w"].double().requires_grad_(), P["b"].double().requires_grad_()
    o = ln = F.layer_norm(x, (D,), w, b, EPS)
    ln.retain_grad()
    zz = None
    if case.gate:
        zz = P["z"].double().transpose(1, 2).contiguous().requires_grad_()
        o = _stored(o, case.out) * _stored(F.silu(zz) if case.gate == 2 else zz, case.out)
    ref = dict(mean=mean, rstd=(var + EPS).rsqrt(), out=o.detach())
    if case.bwd:
        o.backward(P["dy"].double())
        ref.update(dyb=x.grad, dw=w.grad, db=b.grad, dz=zz.grad if case.gate else None,
                   terms=ref["rstd"][..., None] * (ln.grad * w.detach()).abs())
    return ref


def _to_image(dout, H, W):
    """The four orders of a (B, 4, D, L) scan-order tensor, each brought back to image order: (B, 4, D, L)."""
    return torch.stack([dout[:, 0], _col(dout[:, 1], H, W), dout[:, 2].flip(-1), _col(dout[:, 3].flip(-1), H, W)], 1)


def _check(case, P, got, yb_ref):
    """got: the results on the host (yb / out / dout / dz token-major (B, L, D), dout (B, 4, D, L)); yb_ref: mia_cross_merge's
    value rounded to bf16, (B, L, D)."""
    B, D, H, W = case.shape
    TO = case.out
    yb = got.get("yb", yb_ref)
    if "yb" in got:
        assert _same_bits(yb, yb_ref), "yb differs from mia_cross_merge(ys) rounded to bf16"
    want, other = PLANTED_YB[case.pairs], PLANTED_YB[not case.pairs]
    for b, c, l in P["planted"]:
        v = float(yb[b, l, c])
        assert v == want != other, f"planted token (b {b}, c {c}, l {l}): yb {v}, the {case.path} path's order gives {want}"
    ref = _reference(case, P, yb_ref)
    if "mean" in got:
        cmp_f32(got["mean"], ref["mean"], "mean")
        cmp_f32(got["rstd"], ref["rstd"], "rstd")
    if TO == F32:
        cmp_f32(got["out"], ref["out"], "out")
    else:
        cmp_stored(got["out"], ref["out"], TO, "out", n_ulp=2.0 if case.gate else 1.0)
    if not case.bwd:
        return
    img = _to_image(got["dout"], H, W)
    for k in (1, 2, 3):
        assert _same_bits(img[:, k], img[:, 0]), f"dout order {k} differs from order 0"
    if D == 1:
        # the LayerNorm's input gradient is 0 at D = 1 (xhat = 0, g w - mean(g w) = 0): the kernel's value is the fp32 rounding
        # of g w amplified by rstd, bounded by 2 fp32 ulps of the terms rstd |g w|
        dx = img[:, 0].transpose(1, 2).double()
        assert bool((dx.abs() <= 2.0 ** -22 * ref["terms"]).all()), f"dout at D = 1: {float(dx.abs().max()):.3e} off 0"
    else:
        cmp_stored(img[:, 0].transpose(1, 2).to(BF16), ref["dyb"], BF16, "dout")
    if case.gate:
        if TO == F32:
            cmp_f32(got["dz"], ref["dz"], "dz", rtol=1e-4, atol_rms=1e-4)
        else:
            cmp_stored(got["dz"], ref["dz"], TO, "dz", n_ulp=2.0)
    if D == 1:                                                         # xhat = 0 exactly: so is dweight
        assert bool((got["dw"] == 0).all()), f"dweight at D = 1: {got['dw']}"
    else:
        cmp_f32(got["dw"], ref["dw"], "dweight", rtol=1e-4, atol_rms=1e-4)
    cmp_f32(got["db"], ref["db"], "dbias", rtol=1e-4, atol_rms=1e-4)


def _host(R):
    got = {k: f.value().cpu() for k, f in R.items()}
    if "dz" in got:
        got["dz"] = got["dz"].transpose(1, 2)
    return got


@gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_epilogue_parity(cid):
    """yb bit-identical to mia_cross_merge on the same ys view (and to merge_replica with the path's order), the planted tokens
    in that order; mean / rstd / out / dout / dz / dweight / dbias against float64; nothing written outside an output; the
    four orders of dout equal; a second call bit-identical to the first."""
    case = CASES[cid]
    B, D, H, W = case.shape
    P = _inputs(case)
    Q = _device(case, P)
    R = _launch(case, Q)
    again = _launch(case, Q)
    for k in R:
        assert _same_bits(R[k].buf, again[k].buf), f"{k}: two calls differ"
        R[k].untouched(k)
    for k, f in Q.items():
        if f is not None:
            f.untouched(f"input {k}")
    del again
    yb_ref = _cross_merge(case, Q).cpu()
    assert _same_bits(yb_ref, merge_replica(P["ys"], H, W, case.pairs)), "mia_cross_merge differs from the replica of its path's order"
    _check(case, P, _host(R), yb_ref.to(BF16).transpose(1, 2).contiguous())


# ---------------------------------------------------------------------------------------------------------- CrossScan1b1
def _from_1b1(ys, H, W):
    """Adjoint of _torch_1b1: (B, 4, C, L) in scan order k -> (B, 4, C, H, W) in image order."""
    B, K, C, L = ys.shape
    return _to_image(ys, H, W).view(B, K, C, H, W)


def _inputs_1b1(case):
    B, C, H, W = case.shape
    g = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    return torch.randn(B, 4, C, H * W, generator=g).to(case.dtype)


def _launch_1b1(case, X):
    B, C, H, W = case.shape
    out = Frame((B, 4, C, H * W), case.dtype, off=case.off)
    name = "mia_cross_merge_1b1" if case.merge else "mia_cross_scan_1b1"
    _lib().call(name, name, torch.device("cuda"), X.ptr(), out.ptr(), B, C, H, W, _lib().dtype_code(case.dtype))
    return out


@gpu
@pytest.mark.parametrize("cid", list(CASES_1B1))
def test_cross_1b1_parity(cid):
    """The permutation bit for bit against the torch index statement, nothing written outside the output, a second call
    bit-identical."""
    case = CASES_1B1[cid]
    B, C, H, W = case.shape
    x = _inputs_1b1(case)
    X = Frame(x.shape, case.dtype, off=case.off).set(x.cuda())
    out, again = _launch_1b1(case, X), _launch_1b1(case, X)
    assert _same_bits(out.buf, again.buf), "two calls differ"
    out.untouched("out")
    X.untouched("input")
    want = _from_1b1(x, H, W) if case.merge else _torch_1b1(x.view(B, 4, C, H, W))
    assert _same_bits(out.value().cpu().view(want.shape), want.contiguous())


# ---------------------------------------------------------------------------------------------------------- launched kernels
def _short(name, rx=KERNEL):
    m = rx.search(name)
    kern = m.group(1) if m.groups() else m.group(0)
    if name[m.end():m.end() + 1] != "<":
        return kern
    return f"{kern}<{', '.join(kernel_trace.targs(name, kern + '<'))}>"


def _merge_path(names):
    assert len(names) == 1, names
    return "vec" if "vec" in names[0] else "direct" if "direct" in names[0] else "staged"


def launches():
    """Run in a child interpreter: the kernels each case launched, and the kernel mia_cross_merge launches on its ys."""
    out = {}
    for cid, case in CASES.items():
        Q = _device(case, _inputs(case))
        out[cid] = sorted({_short(n) for n in kernel_trace.names_of(lambda: _launch(case, Q), KERNEL, len(case.target()))})
        out[cid + "|merge"] = _merge_path(kernel_trace.names_of(lambda: _cross_merge(case, Q), MERGE))
        del Q
    for cid, case in CASES_1B1.items():
        X = Frame((case.shape[0], 4, case.shape[1], case.shape[2] * case.shape[3]), case.dtype, off=case.off)
        X.set(_inputs_1b1(case).cuda())
        out[cid] = sorted({_short(n) for n in kernel_trace.names_of(lambda: _launch_1b1(case, X), KERNEL)})
    return out


@pytest.fixture(scope="module")
def traced():
    return kernel_trace.in_child("tests.test_ss2d_core_kernels_gpu:launches")


@gpu
def test_every_case_launches_its_target(traced):
    """Each case ran exactly the instantiations the replicas assign it, and mia_cross_merge on the case's ys took the path
    cross_merge_path names (the path whose order the epilogue copies)."""
    wrong = {cid: (traced.get(cid), sorted(c.target())) for cid, c in {**CASES, **CASES_1B1}.items() if set(traced.get(cid, [])) != c.target()}
    assert not wrong, wrong
    paths = {cid: (traced[cid + "|merge"], c.path) for cid, c in CASES.items() if traced[cid + "|merge"] != c.path}
    assert not paths, paths


@gpu
def test_all_instantiations_launched_and_compared(traced):
    targets = set().union(*(c.target() for c in {**CASES, **CASES_1B1}.values()))
    launched = {n for cid, names in traced.items() if not cid.endswith("|merge") for n in names}
    assert targets == set(INSTANTIATIONS) == launched, (sorted(set(INSTANTIATIONS) - launched), sorted(launched - set(INSTANTIATIONS)))
    print(f"{len(launched)}/{len(INSTANTIATIONS)} SS2D core instantiations launched and compared ({len(CASES) + len(CASES_1B1)} cases)")


# ---------------------------------------------------------------------------------------------------------- CPU checks
def test_case_table_covers_every_instantiation_and_edge():
    cases, c1 = list(CASES.values()), list(CASES_1B1.values())
    assert len(set(INSTANTIATIONS)) == 18
    assert set().union(*(c.target() for c in cases + c1)) == set(INSTANTIATIONS)
    for ys, o in FWD_PAIRS:                                            # each dtype pair with every gate; the backward too
        for gate in (0, 1, 2):
            assert any((c.ys, c.out, c.gate, c.bwd) == (ys, o, gate, True) for c in cases), (ys, o, gate)
        assert any((c.ys, c.out, c.stats) == (ys, o, False) for c in cases), (ys, o)
    assert {1, 7, 33, 96, 768, 2048, 3626} <= {c.shape[1] for c in cases}
    maps = {c.shape[2:] for c in cases}
    assert {(6, 5), (7, 9), (14, 14), (80, 80), (1, 13), (11, 1)} <= maps
    assert any(H % KTH and W % KTW for H, W in maps)
    routes = {c.path: set() for c in cases}
    for c in cases:
        B, D, H, W = c.shape
        route = ("direct" if c.path == "direct" else "L%4" if H * W % 4 else "misaligned" if c.off else "fp32 plane" if c.ys == F32 and H * W > CS_SMEM // 16
                 else "B D^2" if B * D * D >= 1 << 32 else c.path)
        routes[c.path].add(route)
    assert routes == {"vec": {"vec"}, "staged": {"L%4", "misaligned", "fp32 plane", "B D^2"}, "direct": {"direct"}}, routes
    # the B D^2 bound alone moves the merge: one batch fewer is vectorised
    assert cross_merge_path(True, True, 1024, 2048, 2, 2, 2) == "staged" and cross_merge_path(True, True, 1023, 2048, 2, 2, 2) == "vec"
    assert cross_merge_path(True, True, 1, 7, 120, 120, 2) == "vec" != cross_merge_path(True, True, 1, 7, 120, 120, 4)
    gated = [c for c in cases if c.gate]
    assert set(Z_LAYOUTS) == {c.z for c in gated} == {c.dz for c in gated if c.bwd}
    for v in ("const", "offset"):
        assert any(c.values == v for c in cases), v
    assert any(c.values == "huge" and c.out == F16 and c.gate == g for c in cases for g in (1, 2))
    assert any(c.shape[0] == MAX_BATCH and c.bwd for c in cases)
    assert max(c.shape[0] * grid_tiles(*c.shape[2:]) for c in cases if c.bwd) >= 512
    # the planted tokens tell the orders apart in every ys dtype
    for TY in (F32, BF16, F16):
        assert plant_orders(TY) == PLANTED_YB, TY
    assert all(_planted(c) for c in cases if c.shape[2] * c.shape[3] > 1)
    # 1b1: every path per dtype; a CTA straddling two orders (C not a multiple of the planes per CTA) and a partial last CTA;
    # the direct grid sweeping at least twice
    for dt in (F32, BF16, F16):
        mine = [c for c in c1 if c.dtype == dt]
        for merge in (False, True):
            assert {c.launch[0] for c in mine if c.merge == merge} == {"vec", "staged", "direct"}
        for c in mine:
            B, C, H, W = c.shape
            path, planes, ctas = c.launch
            if path == "direct":
                assert B * 4 * C * H * W > 2 * ctas * 256, c.id
            else:
                assert C % planes and (B * 4 * C) % planes, c.id
        assert any(c.off and c.launch[0] == "staged" for c in mine) and any(c.shape[2] * c.shape[3] % 4 for c in mine)


def _lib_or_skip():
    if not os.path.exists(LIB):
        pytest.skip("needs the built library (python -c 'import __graft_entry__ as g; g.build()')")
    return _lib().lib()


def test_grid_tiles_replica_is_the_library():
    """grid_tiles above gives the CTAs the library's backward launches: the workspace holds one (dweight, dbias) partial of D
    floats each per CTA.  The training-size cases sum 512 partials."""
    L_ = _lib_or_skip()
    for c in CASES.values():
        B, D, H, W = c.shape
        assert int(L_.mia_ss2d_merge_norm_bwd_workspace(B, D, H, W)) == B * grid_tiles(H, W) * 2 * D * 4, c.id
    assert grid_tiles(14, 14) * 64 == 512 and grid_tiles(6, 5) == 2 and grid_tiles(11, 1) == 3 and grid_tiles(1, 13) == 2


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump, cu++filt and the built library (python -c 'import __graft_entry__ as g; g.build()')")
def test_instantiation_list_is_the_built_one():
    """The epilogue kernels in libmia_scan.so are exactly the 9 of EPI_KERNELS, and the CrossScan1b1 kernels exactly 9 of
    cross_scan.cu's 32."""
    found = _demangled_kernels()
    epi = [full for base, full in found if base.startswith("merge_norm_")]
    cs = [full for base, full in found if base in CS_BASES]
    k1b1 = [full for base, full in found if base.startswith("cross_1b1_")]
    assert sorted(epi) == sorted(EPI_KERNELS), (sorted(epi), sorted(EPI_KERNELS))
    assert sorted(k1b1) == sorted(K1B1_KERNELS), (sorted(k1b1), sorted(K1B1_KERNELS))
    assert len(cs) == len(set(cs)) == 32


# ---------------------------------------------------------------------------------------------------------- mutants
def _correct(case, P):
    """The results a correct kernel stores, from the float64 statement and the merge replica: the same keys as _host."""
    B, D, H, W = case.shape
    yb = merge_replica(P["ys"], H, W, case.pairs).to(BF16).transpose(1, 2).contiguous()
    ref = _reference(case, P, yb)
    got = dict(yb=yb, mean=ref["mean"].float(), rstd=ref["rstd"].float(), out=ref["out"].to(case.out))
    if case.bwd:
        dx = ref["dyb"].to(BF16).float().transpose(1, 2).reshape(B, D, H, W)
        got.update(dout=cross_scan_ref(dx), dw=ref["dw"].float(), db=ref["db"].float())
        if case.gate:
            got["dz"] = ref["dz"].to(case.out)
    return got, yb


def _stats(yb, unbiased=False, eps=EPS):
    x = yb.double()
    return x.mean(-1).float(), (x.var(-1, unbiased=unbiased) + eps).rsqrt().float()


def _dx_without_term(case, P, yb):
    """d yb of the LayerNorm with rstd (g w - mean(g w)) only (gate 0: g = dy)."""
    x, w, g = yb.double(), P["w"].double(), P["dy"].double()
    mean, var = x.mean(-1, keepdim=True), x.var(-1, unbiased=False, keepdim=True)
    rstd = (var + EPS).rsqrt()
    gw = g * w
    return rstd * (gw - gw.mean(-1, keepdim=True))


def _mutate(name, case, P, got, yb):
    B, D, H, W = case.shape
    L = H * W
    if name == "merge in the other order":
        got["yb"] = merge_replica(P["ys"], H, W, not case.pairs).to(BF16).transpose(1, 2).contiguous()
    elif name == "column-major position l for w H + h":
        got["yb"] = merge_replica(P["ys"], H, W, case.pairs, col=False).to(BF16).transpose(1, 2).contiguous()
    elif name == "variance over D - 1":
        got["mean"], got["rstd"] = _stats(yb, unbiased=True)
    elif name == "eps dropped":
        got["mean"], got["rstd"] = _stats(yb, eps=0.0)
    elif name == "xhat mean(g w xhat) term of dx dropped":
        got["dout"] = cross_scan_ref(_dx_without_term(case, P, yb).to(BF16).float().transpose(1, 2).reshape(B, D, H, W))
    elif name == "dz without the SiLU backward factor":
        o = F.layer_norm(yb.double(), (D,), P["w"].double(), P["b"].double(), EPS).to(case.out).double()
        got["dz"] = (P["dy"].double() * o).to(case.out)
    elif name == "one dout order written unreversed":
        got["dout"][:, 2] = got["dout"][:, 2].flip(-1)
    elif name == "one CTA's partial missing from dweight":
        x, w = yb.double(), P["w"].double()
        xhat = (x - x.mean(-1, keepdim=True)) * (x.var(-1, unbiased=False, keepdim=True) + EPS).rsqrt()
        g = (P["dy"].double().to(case.out).double() * P["z"].double().transpose(1, 2)).to(case.out).double() if case.gate == 1 else None
        assert g is not None, "this mutant is stated for the y z gate"
        keep = torch.ones(B, H, W, dtype=torch.bool)
        keep[5, 4:8, 8:14] = False                                     # CTA (b 5, tile row 1, tile column 1)
        keep = keep.view(B, L, 1)
        assert torch.allclose((g * xhat).sum((0, 1)).float(), got["dw"], rtol=1e-4, atol=1e-3)     # the full sums are dweight
        got["dw"] = (g * xhat * keep).sum((0, 1)).float()
        got["db"] = (g * keep).sum((0, 1)).float()
    elif name == "padding tokens' statistics used":
        # a padding slot (w >= W) of a tile at the right edge sits at l = h W + w, a real token of the next row: its stats
        # (a row of zeros: mean 0, rstd eps^-1/2) land there
        mean, rstd = got["mean"].clone(), got["rstd"].clone()
        for th0 in range(0, H, KTH):
            for tw0 in range(0, W, KTW):
                for h in range(th0, min(th0 + KTH, H)):
                    for w in range(max(tw0, W), tw0 + KTW):
                        if h * W + w < L:
                            mean[:, h * W + w], rstd[:, h * W + w] = 0.0, EPS ** -0.5
        got["mean"], got["rstd"] = mean, rstd
    else:
        raise AssertionError(name)
    return got


# mutant -> the case whose shapes, dtypes and values it is stated on (and whose GPU comparison would reject it)
MUTANTS = {
    "merge in the other order": "bf16-bf16-g1-B1_D33_14x14-z_neg-dz_xz-off1",
    "column-major position l for w H + h": "f32-f32-g0-B3_D33_6x5",
    "variance over D - 1": "f32-f16-g0-B2_D96_7x9",
    "eps dropped": "f32-f32-g2-B2_D96_7x9-z_cm-dz_tm-const",
    "xhat mean(g w xhat) term of dx dropped": "f32-f16-g0-B2_D96_7x9",
    "dz without the SiLU backward factor": "f16-f16-g2-B2_D33_7x9-z_xz-dz_xz-huge",
    "one dout order written unreversed": "f32-f32-g0-B3_D33_6x5",
    "one CTA's partial missing from dweight": "bf16-bf16-g1-B64_D96_14x14-z_tm-dz_neg-parts",
    "padding tokens' statistics used": "f32-f32-g0-B3_D33_6x5",
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_criteria_reject_mutants(mutant):
    """The comparisons of test_epilogue_parity accept the correct float64 results of the named case (rounded as the kernel
    stores them) and reject the mutant: the merge summed in the other order (the planted tokens), the column-major orders
    read at the row-major position, the variance over D - 1, eps dropped on the constant rows, the xhat mean(g w xhat) term
    of dx dropped, dz without the SiLU backward factor, one dout order written unreversed, one CTA's partial missing from
    dweight / dbias out of 512, and the statistics of a partial tile's padding slots written over real tokens."""
    case = CASES[MUTANTS[mutant]]
    P = _inputs(case)
    got, yb = _correct(case, P)
    _check(case, P, got, yb)
    bad = _mutate(mutant, case, P, {k: v.clone() for k, v in got.items()}, yb)
    with pytest.raises(AssertionError):
        _check(case, P, bad, yb)
