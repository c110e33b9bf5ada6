"""Every instantiation of the conv / gate tile kernels (csrc/causal_conv1d.cu: the fused inner block's *_ex kernels and the
four-direction mixer's *_dirs kernels) against float64, at the shapes, layouts and operand counts where a 64-channel x
64-token tile goes wrong.

A case table gives each of the 114 instantiations at least one launch on a ragged shape: dims 1 to 768 around the 64-channel
tile, seqlens shorter than the conv width, around the 64-token tile and the 3 tokens the backward stages past it, and the
column-order lengths, odd grid sides included.  Operands are the halves of a channel-major or token-major xz, time-reversed
views and token-major GEMM operands with a padded row pitch, every element of their buffers outside the operand NaN: inputs
read there turn the result NaN, outputs written there are caught bit for bit.  Backward cases at training sizes have more (batch, token tile) items than CTAs per channel tile, so each CTA walks
several items; a Python replica of conv_bwd_parts, checked against the workspace queries, states it.  Every case runs twice
with bit-identical results.  A child interpreter records the kernels each case launched (kernel_trace); a CPU test checks
the list of 114 against the built library, and another shows that the criteria reject subtly wrong results."""
import ctypes
import os
import re
import shutil
import subprocess
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_trace
from tests.parity import cmp_f32, cmp_stored
from tests.test_arm_mixer_fused_gpu import TO_IMAGE, TO_SCAN, _conv_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "medical_image_analysis_b200", "libmia_scan.so")
gpu = pytest.mark.gpu

TNAME = {torch.float32: "float", torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}
DT_ID = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}
DTYPES = (torch.float32, torch.bfloat16, torch.float16)
CONV_KERNELS = ("conv_fwd_ex_kernel", "conv_bwd_ex_kernel", "conv_fwd_dirs_kernel", "conv_bwd_dirs_kernel")


def _tf(v):
    return "true" if v else "false"


# Every tile kernel the unit holds: the conv kernels <T, width, silu>, the gate kernels <T> (gate_bwd_ex_kernel<T, TD>: douts
# stored as fp32 or as T), and the finalize kernels of the conv backwards.
INSTANTIATIONS = ([f"{k}<{t}, {w}, {_tf(s)}>" for k in CONV_KERNELS for t in TNAME.values() for w in (1, 2, 3, 4) for s in (True, False)]
                  + ["conv_bwd_ex_finalize"]
                  + [f"{k}<{t}>" for k in ("gate_fwd_ex_kernel", "conv_bwd_dirs_finalize", "gate_fwd_dirs_kernel", "gate_bwd_dirs_kernel")
                     for t in TNAME.values()]
                  + [f"gate_bwd_ex_kernel<{t}, float>" for t in TNAME.values()]
                  + [f"gate_bwd_ex_kernel<{t}, {t}>" for t in ("__half", "__nv_bfloat16")])
LEGACY = ("causal_conv1d_fwd_kernel", "causal_conv1d_bwd_kernel")     # 2 x 24, covered by test_causal_conv1d_gpu.py
KERNEL = re.compile(r"\b((?:conv|gate)_(?:fwd|bwd)_(?:ex|dirs)_(?:kernel|finalize))\b")
TILE = 64                                                             # kTC = kTT


def _cdiv(a, b):
    return -(-a // b)


def conv_bwd_parts(n, b, d, L):
    """CTAs per channel tile of the conv backward (conv_bwd_parts in causal_conv1d.cu): about 8 per SM of a 132-SM H100 over
    the channel tiles of the n directions, and no more than the (batch, 64-token tile) items."""
    return min(_cdiv(8 * 132, _cdiv(d, TILE) * n), n_items(b, L))


def n_items(b, L):
    return b * _cdiv(L, TILE)


def short_name(name):
    """'void (anonymous namespace)::conv_fwd_ex_kernel<float, 4, true>((anonymous namespace)::TileArgs)' ->
    'conv_fwd_ex_kernel<float, 4, true>'."""
    m = KERNEL.search(name)
    kern = m.group(1)
    if name[m.end():m.end() + 1] != "<":
        return kern
    return f"{kern}<{', '.join(kernel_trace.targs(name, kern + '<'))}>"


# ---------------------------------------------------------------------------------------------------------- operands
class Opd:
    """A (batch, dim, seqlen) operand in one of the layouts the tile kernels read and write in place:

    cm    half ``half`` of a channel-major xz (b, 2d, L): batch stride 2 d L, the other half a gap;
    tmxz  the same half of a token-major xz (xz.transpose(1, 2).contiguous().transpose(1, 2)): channel stride 1;
    rev   cm seen time-reversed (_bdl(rev=True)): sequence stride -1;
    tm    a (b L, d) token-major GEMM operand from _tm_buffer: row pitch d rounded up to 8, pad columns when d % 8 != 0.

    The whole buffer starts NaN; ``set`` writes the operand's elements only."""

    def __init__(self, layout, b, d, L, dtype, half=0, dev="cuda"):
        from medical_image_analysis_b200.selective_scan_interface import _tm_buffer
        self.layout, self.d, self.L = layout, d, L
        if layout == "tm":
            t = _tm_buffer(b * L, d, dtype, dev)
            self.buf = t.as_strided((b * L, t.stride(0)), (t.stride(0), 1))
            self._region = lambda buf: buf[:, :d].unflatten(0, (b, L)).transpose(1, 2)
        elif layout == "tmxz":
            self.buf = torch.empty((b, L, 2 * d), dtype=dtype, device=dev)
            self._region = lambda buf: buf[:, :, half * d:(half + 1) * d].transpose(1, 2)
        else:
            assert layout in ("cm", "rev"), layout
            self.buf = torch.empty((b, 2 * d, L), dtype=dtype, device=dev)
            self._region = lambda buf: buf[:, half * d:(half + 1) * d]
        self.buf.fill_(float("nan"))

    def region(self, buf=None):
        """The operand's elements as a (b, d, L) view of ``buf`` (default: its own), in memory order."""
        return self._region(self.buf if buf is None else buf)

    def value(self):
        """The operand as the kernel addresses it: element (b, c, t)."""
        r = self.region()
        return r.flip(-1) if self.layout == "rev" else r

    def set(self, v):
        self.region().copy_(v.flip(-1) if self.layout == "rev" else v)
        return self

    def bdl(self):
        from medical_image_analysis_b200.selective_scan_interface import _bdl, _tm
        if self.layout == "tm":
            return _tm(self.buf[:, :self.d], self.L)
        return _bdl(self.region(), rev=self.layout == "rev")

    def untouched(self, what):
        """Every element of the buffer outside the operand is still the NaN it was filled with, bit for bit."""
        rest = self.buf.clone()
        self.region(rest).fill_(float("nan"))
        bad = int((_bits(rest) != _bits(torch.full_like(rest, float("nan")))).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the {self.layout} operand"


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------------------- the case table
@dataclass
class Case:
    """One call of one entry point.  ``x`` is the layout of x (conv kinds) or z (gate kinds); ``ins`` the layouts of the summed
    inputs (conv_bwd_ex: dys; gate_fwd_ex: outs; gate_bwd_ex: dy, then outs; gate_bwd_dirs: dy); ``outs`` the layouts of the
    outputs (conv_fwd_ex: ys; gate_fwd_ex: out_zs; gate_bwd_ex: douts, then dz; conv_bwd_*: dx; gate_fwd_dirs: y;
    gate_bwd_dirs: dz)."""
    kind: str
    dtype: torch.dtype
    shape: tuple
    W: int = 4
    silu: bool = True
    bias: bool = True
    x: str = "cm"
    ins: tuple = ()
    outs: tuple = ("cm",)
    dout_f32: bool = True       # gate_bwd_ex: douts in fp32 (the call Python makes) or in the call's dtype
    orders: tuple = ()
    divisor: int = 1
    dense: bool = True          # conv_fwd_dirs: u written
    tm: bool = False            # conv_fwd_dirs: u_tm written;  conv_bwd_dirs: dy_tm given
    note: str = ""

    @property
    def dirs(self):
        return self.kind.endswith("_dirs")

    @property
    def n(self):
        return len(self.orders) if self.dirs else 1

    @property
    def id(self):
        b, d, L = self.shape
        s = f"{self.kind}-{DT_ID[self.dtype]}-{b}x{d}x{L}"
        if self.kind.startswith("conv"):
            s += f"-W{self.W}{'-silu' if self.silu else ''}{'' if self.bias else '-nobias'}"
        s += f"-x_{self.x}"
        if self.ins:
            s += "-in_" + "+".join(self.ins)
        if self.kind != "conv_fwd_dirs":
            s += "-out_" + "+".join(self.outs)
        if self.kind == "gate_bwd_ex":
            s += "-dout_" + ("f32" if self.dout_f32 else DT_ID[self.dtype])
        if self.dirs:
            s += "-ord" + "".join(map(str, self.orders))
        if self.kind.startswith("gate") and self.dirs:
            s += f"-div{self.divisor}"
        if self.kind == "conv_fwd_dirs":
            s += "-u" * self.dense + "-utm" * self.tm
        if self.kind == "conv_bwd_dirs":
            s += "-dytm" * self.tm
        return s + (f"-{self.note}" if self.note else "")

    @property
    def ragged(self):
        _, d, L = self.shape
        return d % TILE != 0 or L % TILE != 0

    def target(self):
        """The instantiations the call launches."""
        t = TNAME[self.dtype]
        if self.kind.startswith("conv"):
            main = f"{self.kind}_kernel<{t}, {self.W}, {_tf(self.silu)}>"
            if self.kind == "conv_bwd_ex":
                return {main, "conv_bwd_ex_finalize"}
            if self.kind == "conv_bwd_dirs":
                return {main, f"conv_bwd_dirs_finalize<{t}>"}
            return {main}
        if self.kind == "gate_bwd_ex":
            return {f"gate_bwd_ex_kernel<{t}, {'float' if self.dout_f32 else t}>"}
        return {f"{self.kind}_kernel<{t}>"}

    def parts(self):
        b, d, L = self.shape
        return conv_bwd_parts(self.n, b, d, L)


# Every shape is ragged (d or L not a multiple of 64); together they hold dims 1, 3, 63, 64, 65, 100, 768 and seqlens 1-3
# (shorter than the width: all history is padding), 64, 65, 67 (the 3 staged tokens past a tile), 129 and 197.
EX_SHAPES = [(2, 65, 1), (3, 3, 2), (2, 63, 3), (2, 100, 64), (2, 65, 65), (1, 768, 67), (2, 64, 129), (2, 1, 197),
             (3, 100, 129), (2, 63, 67), (1, 768, 197), (2, 3, 65)]
# Column orders need seqlen - 1 = side^2: 2, 5, 65 (one tile and one token), 197, 257 (sides 1, 2, 8, 14, 16) and the odd
# sides 50, 82 (7, 9).
DIRS_SHAPES = [(2, 1, 2), (2, 3, 5), (2, 63, 65), (1, 65, 197), (1, 100, 257), (2, 64, 50), (1, 768, 197), (3, 100, 82),
               (2, 65, 2), (1, 3, 257), (2, 63, 50), (1, 768, 82)]
# n_dirs 1-4; the four n = 4 rows put every order code in every slot; repeated codes
ORDER_SETS = [(0, 1, 2, 3), (1, 2, 3, 0), (2, 3, 0, 1), (3, 0, 1, 2), (3, 3), (2,), (1, 0, 3), (0,), (2, 2, 1, 1), (3,), (1,), (0, 3, 2)]
X_LAYOUTS = ("cm", "tmxz", "rev", "tm")
COMBOS = [(dt, W, s) for dt in DTYPES for W in (1, 2, 3, 4) for s in (True, False)]
BENCH = (32, 768, 197)               # ARM-base in bench.py's module timings
RAGGED_WALK = (40, 64, 1700)         # 1080 items over 1056 parts (*_ex), 1080 over 528 (two directions)
MAX_BATCH = {"ex": 65535, "dirs": 65535 // 4}    # grid z = batch (*_ex), batch x n_dirs with n_dirs <= 4 (*_dirs)


def _cycle(seq, start, n):
    return tuple(seq[(start + j) % len(seq)] for j in range(n))


def _cases():
    out = []
    for i, (dt, W, s) in enumerate(COMBOS):
        out.append(Case("conv_fwd_ex", dt, EX_SHAPES[i * 7 % 12], W, s, bias=i % 5 != 4, x=X_LAYOUTS[i % 4],
                        outs=_cycle(("cm", "tm", "rev", "tmxz"), i, 1 + i % 3)))
        out.append(Case("conv_bwd_ex", dt, EX_SHAPES[(i * 5 + 3) % 12], W, s, bias=i % 4 != 3, x=X_LAYOUTS[(i + 1) % 4],
                        ins=_cycle(("cm", "rev", "tm", "tmxz"), i, 1 + (i + 1) % 3), outs=(X_LAYOUTS[(i + 2) % 4],)))
        dense, tm = ((True, False), (False, True), (True, True))[i % 3]
        out.append(Case("conv_fwd_dirs", dt, DIRS_SHAPES[i * 7 % 12], W, s, bias=i % 5 != 4, x=("tmxz", "cm", "rev", "tm")[i % 4],
                        orders=ORDER_SETS[i % 12], dense=dense, tm=tm))
        out.append(Case("conv_bwd_dirs", dt, DIRS_SHAPES[(i * 5 + 1) % 12], W, s, bias=i % 4 != 1, x=("tmxz", "cm", "tm", "rev")[i % 4],
                        orders=ORDER_SETS[(i + 5) % 12], tm=i % 2 == 0, outs=(("cm", "tmxz", "rev", "tm")[(i + 3) % 4],)))
    for k, dt in enumerate(DTYPES):
        for j in range(4):
            out.append(Case("gate_fwd_ex", dt, EX_SHAPES[(j * 5 + k * 3) % 12], x=("tmxz", "cm")[j % 2],
                            ins=_cycle(("cm", "rev", "tm"), j, 1 + j % 3), outs=_cycle(("tm", "cm", "tmxz", "rev"), j + k, 1 + (j + 1) % 3)))
            orders = ORDER_SETS[(j * 3 + k) % 12]
            out.append(Case("gate_fwd_dirs", dt, DIRS_SHAPES[(j * 5 + k * 3) % 12], x=("tmxz", "cm")[j % 2], orders=orders,
                            divisor=(1, 3, len(orders))[(j + k) % 3], outs=(("tm", "cm", "tmxz", "rev")[(j + k) % 4],)))
            orders = ORDER_SETS[(j * 3 + k + 1) % 12]
            out.append(Case("gate_bwd_dirs", dt, DIRS_SHAPES[(j * 7 + k * 5 + 2) % 12], x=("cm", "tmxz")[j % 2], orders=orders,
                            divisor=(3, len(orders), 1)[(j + k) % 3], ins=(("tm", "cm", "rev")[(j + k) % 3],),
                            outs=(("cm", "tmxz")[(j + k) % 2],)))
        for f32 in (True, False) if dt != torch.float32 else (True,):
            for j in range(3):
                n_outs, n_douts = 1 + (j + k) % 2, 1 + j
                out.append(Case("gate_bwd_ex", dt, EX_SHAPES[(j * 7 + k * 2 + 5 * f32) % 12], x=("cm", "tmxz")[(j + f32) % 2],
                                ins=(("tm", "cm", "rev")[j],) + _cycle(("cm", "rev"), j + k, n_outs),
                                outs=_cycle(("cm", "rev", "tm", "tmxz"), j + 2 * k, n_douts) + (("cm", "tmxz")[j % 2],), dout_f32=f32))
        # seqlen shorter than the width, and one aligned (64 x 64) shape
        for L in (1, 2, 3):
            out.append(Case("conv_fwd_ex", dt, (2, 65, L), x="tmxz", outs=("cm", "tm"), note="short"))
            out.append(Case("conv_bwd_ex", dt, (2, 65, L), x="cm", ins=("tm", "rev"), outs=("tmxz",), note="short"))
            o = (3, 2) if L == 2 else (1, 0)
            out.append(Case("conv_fwd_dirs", dt, (2, 63, L), x="tmxz", orders=o, tm=True, note="short"))
            out.append(Case("conv_bwd_dirs", dt, (2, 63, L), x="cm", orders=o, tm=True, outs=("tmxz",), note="short"))
        out.append(Case("conv_bwd_ex", dt, (2, 64, 64), W=3, silu=False, x="tmxz", ins=("cm", "tm"), outs=("tmxz",), note="aligned"))
        # multi-item backward walks: items > parts
        for W, s in ((4, True), (1, False)):
            out.append(Case("conv_bwd_ex", dt, BENCH, W, s, x="tmxz", ins=("cm", "rev", "tm"), outs=("tmxz",), note="walk"))
            out.append(Case("conv_bwd_ex", dt, RAGGED_WALK, W, s, x="cm", ins=("cm", "tm"), outs=("cm",), note="walk"))
            out.append(Case("conv_bwd_dirs", dt, BENCH, W, s, x="tmxz", orders=(0, 1, 2, 3), tm=True, outs=("tmxz",), note="walk"))
            out.append(Case("conv_bwd_dirs", dt, RAGGED_WALK, W, s, x="cm", orders=(1, 0), outs=("cm",), note="walk"))
    # the largest batch each entry point accepts (the edge of grid z)
    b, bd = MAX_BATCH["ex"], MAX_BATCH["dirs"]
    bf = torch.bfloat16
    out += [Case("conv_fwd_ex", bf, (b, 1, 3), x="tmxz", outs=("cm", "tm"), note="maxbatch"),
            Case("conv_bwd_ex", bf, (b, 1, 3), x="cm", ins=("tm",), outs=("cm",), note="maxbatch"),
            Case("gate_fwd_ex", bf, (b, 3, 1), x="tmxz", ins=("cm",), outs=("tm",), note="maxbatch"),
            Case("gate_bwd_ex", bf, (b, 3, 1), x="cm", ins=("tm", "cm"), outs=("cm", "cm"), note="maxbatch"),
            Case("conv_fwd_dirs", bf, (bd, 3, 2), x="tmxz", orders=(0, 1, 2, 3), tm=True, note="maxbatch"),
            Case("conv_bwd_dirs", bf, (bd, 3, 2), x="tmxz", orders=(0, 1, 2, 3), tm=True, outs=("tmxz",), note="maxbatch"),
            Case("gate_fwd_dirs", bf, (bd, 3, 2), x="tmxz", orders=(0, 1, 2, 3), divisor=4, outs=("tm",), note="maxbatch"),
            Case("gate_bwd_dirs", bf, (bd, 3, 2), x="tmxz", orders=(3, 2, 1, 0), divisor=4, ins=("tm",), outs=("tmxz",), note="maxbatch")]
    return out


CASES = {c.id: c for c in _cases()}
assert len(CASES) == len(_cases()), "case ids must be unique"


def _lib():
    from medical_image_analysis_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------------- launches
def _inputs(case):
    """Seeded operands of a case on the device: x / z, the taps and bias, and the summed inputs of the kind."""
    b, d, L = case.shape
    T, n = case.dtype, case.n
    g = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    rnd = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    opd = lambda layout, half=0, scale=1.0: Opd(layout, b, d, L, T, half).set(rnd(b, d, L, scale=scale).to(T))
    lead = (n,) if case.dirs else ()
    P = {}
    if case.kind.startswith("conv"):
        P["x"] = opd(case.x)
        P["w"] = rnd(*lead, d, case.W, scale=0.4).cuda()
        P["bias"] = rnd(*lead, d, scale=0.1).cuda() if case.bias else None
    else:
        P["z"] = opd(case.x, 1, 2.0)
    if case.kind in ("conv_bwd_ex", "gate_fwd_ex"):
        P["ins"] = [opd(lo) for lo in case.ins]
    elif case.kind in ("gate_bwd_ex", "gate_bwd_dirs"):
        P["dy"] = opd(case.ins[0])
        P["outs"] = [opd(lo) for lo in case.ins[1:]]
    if case.kind == "conv_bwd_dirs":
        P["du"] = rnd(b, n * d, L).to(T).cuda()
        P["dy_tm"] = [opd("tm") for _ in range(n)] if case.tm else None
    if case.kind in ("gate_fwd_dirs", "gate_bwd_dirs"):
        P["outs"] = rnd(b, n * d, L).to(T).cuda()
    return P


def _launch(case, P):
    """One call of the case's entry point on NaN-filled outputs -> the outputs."""
    from medical_image_analysis_b200.selective_scan_interface import _ops
    lib = _lib()
    b, d, L = case.shape
    T, n, W, kind = case.dtype, case.n, case.W, case.kind
    dt, dev, by = lib.dtype_code(T), torch.device("cuda"), ctypes.byref
    new = lambda layout, half=0, dtype=T: Opd(layout, b, d, L, dtype, half)
    nan = lambda *s, dtype=torch.float32: torch.full(s, float("nan"), dtype=dtype, device=dev)
    orders = (ctypes.c_int * max(1, n))(*case.orders)
    R = {}
    if kind == "conv_fwd_ex":
        R["ys"] = [new(lo) for lo in case.outs]
        arr, k = _ops(*[o.bdl() for o in R["ys"]])
        lib.call("mia_causal_conv1d_fwd_ex", kind, dev, by(P["x"].bdl()), P["w"].data_ptr(), _ptr(P["bias"]), arr, k, b, d, L, W,
                 int(case.silu), dt)
    elif kind == "conv_bwd_ex":
        R["dx"], R["dw"], R["db"] = new(case.outs[0]), nan(d, W), nan(d) if case.bias else None
        ws = torch.empty(max(1, int(lib.lib().mia_causal_conv1d_bwd_ex_workspace(b, d, L, W))), dtype=torch.uint8, device=dev)
        arr, k = _ops(*[o.bdl() for o in P["ins"]])
        lib.call("mia_causal_conv1d_bwd_ex", kind, dev, by(P["x"].bdl()), P["w"].data_ptr(), _ptr(P["bias"]), arr, k, by(R["dx"].bdl()),
                 R["dw"].data_ptr(), _ptr(R["db"]), ws.data_ptr(), ws.numel(), b, d, L, W, int(case.silu), dt)
    elif kind == "gate_fwd_ex":
        R["ys"] = [new(lo) for lo in case.outs]
        arr, k = _ops(*[o.bdl() for o in P["ins"]])
        oarr, no = _ops(*[o.bdl() for o in R["ys"]])
        lib.call("mia_silu_gate_fwd_ex", kind, dev, arr, k, by(P["z"].bdl()), oarr, no, b, d, L, dt)
    elif kind == "gate_bwd_ex":
        TD = torch.float32 if case.dout_f32 else T
        R["douts"], R["dz"] = [new(lo, 0, TD) for lo in case.outs[:-1]], new(case.outs[-1], 1)
        arr, k = _ops(*[o.bdl() for o in P["outs"]])
        darr, nd = _ops(*[o.bdl() for o in R["douts"]])
        lib.call("mia_silu_gate_bwd_ex", kind, dev, by(P["dy"].bdl()), arr, k, by(P["z"].bdl()), darr, nd, by(R["dz"].bdl()), b, d, L, dt,
                 lib.dtype_code(TD))
    elif kind == "conv_fwd_dirs":
        R["u"] = nan(b, n * d, L, dtype=T) if case.dense else None
        R["u_tm"] = [new("tm") for _ in range(n)] if case.tm else None
        tms = _ops(*[o.bdl() for o in R["u_tm"]])[0] if case.tm else None
        lib.call("mia_causal_conv1d_fwd_dirs", kind, dev, by(P["x"].bdl()), orders, n, P["w"].data_ptr(), _ptr(P["bias"]), _ptr(R["u"]),
                 tms, b, d, L, W, int(case.silu), dt)
    elif kind == "conv_bwd_dirs":
        R["dx"], R["dw"], R["db"] = new(case.outs[0]), nan(n, d, W), nan(n, d) if case.bias else None
        ws = torch.empty(max(1, int(lib.lib().mia_causal_conv1d_bwd_dirs_workspace(n, b, d, L, W))), dtype=torch.uint8, device=dev)
        tms = _ops(*[o.bdl() for o in P["dy_tm"]])[0] if case.tm else None
        lib.call("mia_causal_conv1d_bwd_dirs", kind, dev, by(P["x"].bdl()), orders, n, P["w"].data_ptr(), _ptr(P["bias"]),
                 P["du"].data_ptr(), tms, by(R["dx"].bdl()), R["dw"].data_ptr(), _ptr(R["db"]), ws.data_ptr(), ws.numel(), b, d, L, W,
                 int(case.silu), dt)
    elif kind == "gate_fwd_dirs":
        R["y"] = new(case.outs[0])
        lib.call("mia_silu_gate_fwd_dirs", kind, dev, P["outs"].data_ptr(), orders, n, case.divisor, by(P["z"].bdl()), by(R["y"].bdl()),
                 b, d, L, dt)
    else:
        R["douts"], R["dz"] = nan(b, n * d, L), new(case.outs[0], 1)
        lib.call("mia_silu_gate_bwd_dirs", kind, dev, by(P["dy"].bdl()), P["outs"].data_ptr(), orders, n, case.divisor, by(P["z"].bdl()),
                 R["douts"].data_ptr(), by(R["dz"].bdl()), b, d, L, dt)
    return R


def _flat(R):
    """name -> raw buffer of every output (operands as their whole NaN-framed buffer)."""
    out = {}
    for k, v in R.items():
        for i, t in enumerate(v if isinstance(v, list) else [v]):
            if t is not None:
                out[f"{k}[{i}]"] = t.buf if isinstance(t, Opd) else t
    return out


# ---------------------------------------------------------------------------------------------------------- float64 checks
def _cmp(got, ref, what):
    """An output the kernel stores: fp32 by cmp_f32, bf16 / fp16 within 1 ulp of the rounded float64 value (cmp_stored)."""
    if got.dtype == torch.float32:
        cmp_f32(got, ref, what)
    else:
        cmp_stored(got, ref, got.dtype, what)


def _cmp_w(got, ref, what):
    """dweight / dbias: fp32 sums over every (batch, token) of a channel, the mixer test's criterion."""
    cmp_f32(got, ref, what, rtol=1e-4, atol_rms=1e-4)


def _h(t):
    return t.detach().double().cpu()


def _leaf(t):
    return None if t is None else _h(t).requires_grad_()


def _copies(opds, ref, what):
    """Each copy of one result against ``ref``, nothing written around it, and all copies bit-identical."""
    for i, o in enumerate(opds):
        _cmp(o.value(), ref, f"{what}[{i}] ({o.layout})")
        o.untouched(f"{what}[{i}] ({o.layout})")
    for i, o in enumerate(opds[1:], 1):
        assert _same_bits(o.value(), opds[0].value()), f"{what}[{i}] differs from {what}[0]"


def _slot(t, k, d):
    return t[:, k * d:(k + 1) * d]


def _check(case, P, R):
    b, d, L = case.shape
    kind, silu = case.kind, case.silu
    if kind == "conv_fwd_ex":
        _copies(R["ys"], _conv_ref(_h(P["x"].value()), _h(P["w"]), _leaf(P["bias"]), silu), "y")
    elif kind == "conv_bwd_ex":
        x, w, bias = _leaf(P["x"].value()), _leaf(P["w"]), _leaf(P["bias"])
        dy = sum(_h(o.value()) for o in P["ins"])
        (_conv_ref(x, w, bias, silu) * dy).sum().backward()
        _copies([R["dx"]], x.grad, "dx")
        _cmp_w(R["dw"], w.grad, "dweight")
        if bias is not None:
            _cmp_w(R["db"], bias.grad, "dbias")
    elif kind == "gate_fwd_ex":
        _copies(R["ys"], sum(_h(o.value()) for o in P["ins"]) * F.silu(_h(P["z"].value())), "y")
    elif kind == "gate_bwd_ex":
        o, z = sum(_h(t.value()) for t in P["outs"]).requires_grad_(), _leaf(P["z"].value())
        (o * F.silu(z)).backward(_h(P["dy"].value()))
        _copies(R["douts"], o.grad, "dout")
        _copies([R["dz"]], z.grad, "dz")
    elif kind == "conv_fwd_dirs":
        x, w, bias = _h(P["x"].value()), _h(P["w"]), _h(P["bias"]) if case.bias else None
        for k, c in enumerate(case.orders):
            y = _conv_ref(TO_SCAN[c](x), w[k], None if bias is None else bias[k], silu)
            if case.dense:
                _cmp(_slot(R["u"], k, d), y, f"u[{k}] (order {c})")
            if case.tm:
                _copies([R["u_tm"][k]], y, f"u_tm[{k}] (order {c})")
            if case.dense and case.tm:
                assert _same_bits(_slot(R["u"], k, d), R["u_tm"][k].value()), f"u[{k}] and u_tm[{k}] differ"
    elif kind == "conv_bwd_dirs":
        x, w, bias = _leaf(P["x"].value()), _leaf(P["w"]), _leaf(P["bias"])
        loss = 0
        for k, c in enumerate(case.orders):
            dy = _h(_slot(P["du"], k, d)) + (_h(P["dy_tm"][k].value()) if case.tm else 0)
            loss = loss + (_conv_ref(TO_SCAN[c](x), w[k], None if bias is None else bias[k], silu) * dy).sum()
        loss.backward()
        _copies([R["dx"]], x.grad, "dx")
        _cmp_w(R["dw"], w.grad, "dweight")
        if bias is not None:
            _cmp_w(R["db"], bias.grad, "dbias")
    else:
        outs, z = _leaf(P["outs"]), _leaf(P["z"].value())
        y = F.silu(z) * sum(TO_IMAGE[c](_slot(outs, k, d)) for k, c in enumerate(case.orders)) / case.divisor
        if kind == "gate_fwd_dirs":
            _copies([R["y"]], y, "y")
            return
        y.backward(_h(P["dy"].value()))
        cmp_f32(R["douts"], outs.grad, "douts")
        _copies([R["dz"]], z.grad, "dz")


@gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_tile_parity(cid):
    """The case's outputs against float64 statements of the same operation on the same rounded operands, nothing written
    outside them, repeated outputs bit-identical, and a second call bit-identical to the first (dweight / dbias included)."""
    case = CASES[cid]
    P = _inputs(case)
    R = _launch(case, P)
    first, again = _flat(R), _flat(_launch(case, P))
    for k in first:
        assert _same_bits(first[k], again[k]), f"{k}: two calls differ"
    _check(case, P, R)


# ---------------------------------------------------------------------------------------------------------- launched kernels
def launches():
    """Run in a child interpreter: the tile kernels each case's call launches."""
    out = {}
    for cid, case in CASES.items():
        P = _inputs(case)
        out[cid] = sorted({short_name(s) for s in kernel_trace.names_of(lambda: _launch(case, P), KERNEL, len(case.target()))})
        del P
    return out


@pytest.fixture(scope="module")
def traced():
    return kernel_trace.in_child("tests.test_conv_tiles_gpu:launches")


@gpu
def test_every_case_launches_its_target(traced):
    """Each case ran exactly the instantiations the replica of the host dispatch assigns it, and nothing else."""
    wrong = {cid: (traced.get(cid), sorted(c.target())) for cid, c in CASES.items() if set(traced.get(cid, [])) != c.target()}
    assert not wrong, wrong


@gpu
def test_all_instantiations_launched_and_compared(traced):
    """The cases' targets are the full list of 114, and every one of them was seen running."""
    targets = set().union(*(c.target() for c in CASES.values()))
    launched = {n for names in traced.values() for n in names}
    assert targets == set(INSTANTIATIONS) == launched, (sorted(set(INSTANTIATIONS) - launched), sorted(launched - set(INSTANTIATIONS)))
    print(f"{len(launched)}/{len(INSTANTIATIONS)} tile instantiations launched and compared ({len(CASES)} cases)")


# ---------------------------------------------------------------------------------------------------------- CPU checks
def test_case_table_covers_every_instantiation_and_edge():
    """Every instantiation has a case on a ragged shape; the table holds the dims, seqlens, layouts, operand counts, orders,
    divisors and multi-item walks it is meant to."""
    cases = list(CASES.values())
    assert len(INSTANTIATIONS) == len(set(INSTANTIATIONS)) == 114
    assert set().union(*(c.target() for c in cases)) == set(INSTANTIATIONS)
    assert set().union(*(c.target() for c in cases if c.ragged)) == set(INSTANTIATIONS)
    ex, dirs = [c for c in cases if not c.dirs], [c for c in cases if c.dirs]
    assert {1, 3, 63, 64, 65, 100, 768} <= {c.shape[1] for c in ex} & {c.shape[1] for c in dirs}
    assert {1, 2, 3, 64, 65, 67, 129, 197} <= {c.shape[2] for c in ex}
    assert {2, 5, 50, 65, 82, 197, 257} <= {c.shape[2] for c in dirs if max(c.orders) >= 2}
    for kind in ("conv_fwd_ex", "conv_bwd_ex", "gate_fwd_ex", "gate_bwd_ex"):
        mine = [c for c in cases if c.kind == kind]
        assert set(X_LAYOUTS) <= {lo for c in mine for lo in c.ins + c.outs + (c.x,)}, kind
    count = lambda kind, f: {f(c) for c in cases if c.kind == kind}
    assert count("conv_fwd_ex", lambda c: len(c.outs)) == {1, 2, 3}
    assert count("conv_bwd_ex", lambda c: len(c.ins)) == {1, 2, 3}
    assert count("gate_fwd_ex", lambda c: len(c.ins)) == {1, 2, 3} == count("gate_fwd_ex", lambda c: len(c.outs))
    assert count("gate_bwd_ex", lambda c: len(c.ins) - 1) == {1, 2}
    assert count("gate_bwd_ex", lambda c: len(c.outs) - 1) == {1, 2, 3}
    assert count("gate_bwd_ex", lambda c: c.dout_f32) == {True, False}
    for kind in ("conv_fwd_dirs", "conv_bwd_dirs", "gate_fwd_dirs", "gate_bwd_dirs"):
        mine = [c for c in cases if c.kind == kind]
        assert {len(c.orders) for c in mine} == {1, 2, 3, 4}, kind
        assert {(k, o) for c in mine for k, o in enumerate(c.orders)} == {(k, o) for k in range(4) for o in range(4)}, kind
        assert any(len(set(c.orders)) < len(c.orders) for c in mine), kind
        if kind.startswith("gate"):                                     # divisors 1, 3 and n_dirs, each apart from the others
            assert any(c.divisor == 1 < c.n for c in mine), kind
            assert any(c.divisor == 3 != c.n for c in mine), kind
            assert any(c.divisor == c.n not in (1, 3) for c in mine), kind
    assert count("conv_fwd_dirs", lambda c: (c.dense, c.tm)) == {(True, False), (False, True), (True, True)}
    assert count("conv_bwd_dirs", lambda c: c.tm) == {True, False}
    walks = [c for c in cases if c.note == "walk"]
    for kind in ("conv_bwd_ex", "conv_bwd_dirs"):
        for dt in DTYPES:
            for W, s in ((4, True), (1, False)):
                assert [c for c in walks if (c.kind, c.dtype, c.W, c.silu) == (kind, dt, W, s)], (kind, dt, W, s)


def _lib_or_skip():
    if not os.path.exists(LIB):
        pytest.skip("needs the built library (python -c 'import __graft_entry__ as g; g.build()')")
    return _lib().lib()


def test_parts_replica_is_the_library():
    """conv_bwd_parts above gives the CTAs per channel tile the library launches: read back from the workspace queries
    (parts d (W + 1) floats for *_ex; dense dx plus n parts d (W + 1) floats for *_dirs) for every backward case.  The
    training-size cases walk more items than parts: 128 items over 88 (inner block) and over 22 parts (four directions) at
    ARM-base's batch 32 x 768 x 197, 1080 over 1056 at 40 x 64 x 1700."""
    L_ = _lib_or_skip()
    for c in CASES.values():
        if c.kind not in ("conv_bwd_ex", "conv_bwd_dirs"):
            continue
        b, d, L = c.shape
        per = d * (c.W + 1) * 4
        if c.kind == "conv_bwd_ex":
            ws = int(L_.mia_causal_conv1d_bwd_ex_workspace(b, d, L, c.W))
            assert ws % per == 0 and ws // per == c.parts(), (c.id, ws, c.parts())
        else:
            ws = int(L_.mia_causal_conv1d_bwd_dirs_workspace(c.n, b, d, L, c.W)) - c.n * b * d * L * 4
            assert ws % (c.n * per) == 0 and ws // (c.n * per) == c.parts(), (c.id, ws, c.parts())
        if c.note == "walk":
            assert n_items(b, L) > c.parts(), (c.id, n_items(b, L), c.parts())
    assert (n_items(32, 197), conv_bwd_parts(1, *BENCH), conv_bwd_parts(4, *BENCH)) == (128, 88, 22)
    assert (n_items(40, 1700), conv_bwd_parts(1, *RAGGED_WALK)) == (1080, 1056)


def _demangled_kernels():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"Function (\S+?):", out)
    names = subprocess.run(["cu++filt"], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout.split("\n")
    res = []
    for s in names:
        s = re.sub(r"\(int\)(-?\d+)", r"\1", s)
        s = re.sub(r"\(bool\)([01])", lambda m: _tf(m.group(1) == "1"), s)
        m = re.search(r"::(\w+)(<[^()]*>)?\(", s)
        if m:
            res.append((m.group(1), m.group(1) + (m.group(2) or "")))
    return res


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump, cu++filt and the built library (python -c 'import __graft_entry__ as g; g.build()')")
def test_instantiation_list_is_the_built_one():
    """INSTANTIATIONS is exactly the set of tile kernels with SASS in libmia_scan.so (cuobjdump -res-usage, demangled by
    cu++filt: gate_bwd_ex_kernel<T, T> mangles with a substitution), and the unit holds 162 kernels: the 114 and the 48
    legacy causal_conv1d_fwd / bwd_kernel ones."""
    bases = {n.split("<")[0] for n in INSTANTIATIONS}
    found = _demangled_kernels()
    tile = [full for base, full in found if base in bases]
    legacy = [full for base, full in found if base in LEGACY]
    assert set(tile) == set(INSTANTIATIONS), (sorted(set(tile) - set(INSTANTIATIONS)), sorted(set(INSTANTIATIONS) - set(tile)))
    assert len(tile) == len(set(tile)) == 114
    assert len(legacy) == len(set(legacy)) == 48
    assert len(tile) + len(legacy) == 162


# ---------------------------------------------------------------------------------------------------------- mutants
def _dpre(x, w, bias, dy):
    """d pre of the conv + SiLU for the output gradient dy, float64."""
    pre = _conv_ref(x, w, bias, silu=False)
    s = torch.sigmoid(pre)
    return dy * s * (1 + pre * (1 - s))


def _dx_of(dpre, w, cut_at_tile):
    """dx[t] = sum_k w[k] dpre[t + W - 1 - k]; cut_at_tile drops the terms whose dpre lies in the next 64-token tile (the
    3-token tail a tile stages past its end)."""
    W, L = w.shape[1], dpre.shape[-1]
    dx = torch.zeros_like(dpre)
    t = torch.arange(L)
    for k in range(W):
        src = t + W - 1 - k
        ok = src < L
        if cut_at_tile:
            ok &= src // TILE == t // TILE
        dx[..., t[ok]] += w[:, k:k + 1] * dpre[..., src[ok]]
    return dx


@pytest.mark.parametrize("out", ["f32", "bf16", "f16"])
def test_criteria_reject_subtly_wrong_results(out):
    """The comparisons of test_tile_parity on float64 "mutants" of a correct result (2 x 100 x 82, width 4, SiLU, four column-
    walk directions, divisor 3): taps reversed, the 3-token halo from the previous tile dropped, the 3-token dy tail from the
    next tile dropped (dx wrong only at tokens 61-63 of a tile), MIA_ORDER_COL_REV gathered as COL or as SEQ_REV, the gate
    scaled by 1 / n_dirs instead of 1 / divisor, fp32 douts rounded to bf16, and one store past the last channel of a
    ragged tile, in a channel-major half and in a token-major pad column, must all fail; the correct results pass."""
    T = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}[out]
    b, d, L, W = 2, 100, 82, 4
    g = torch.Generator().manual_seed(7)
    x = torch.randn(b, d, L, generator=g).to(T).double()
    w, bias = torch.randn(d, W, generator=g) * 0.4, torch.randn(d, generator=g) * 0.1
    w, bias = w.double(), bias.double()
    dy = torch.randn(b, d, L, generator=g).to(T).double()
    q = lambda v: v.to(T)                                              # the result as the kernel stores it

    y = _conv_ref(x, w, bias)
    halo_dropped = torch.cat([_conv_ref(x[..., t0:t0 + TILE], w, bias) for t0 in range(0, L, TILE)], -1)
    xg = x.clone().requires_grad_()
    (_conv_ref(xg, w, bias) * dy).sum().backward()
    dp = _dpre(x, w, bias, dy)
    assert torch.allclose(_dx_of(dp, w, False), xg.grad)
    u3 = _conv_ref(TO_SCAN[3](x), w, bias)
    z = torch.randn(b, d, L, generator=g).to(T).double() * 2
    outs = [torch.randn(b, d, L, generator=g).to(T).double() for _ in range(4)]
    s = sum(TO_IMAGE[c](o) for c, o in zip((0, 1, 2, 3), outs))
    gate = F.silu(z) * s / 3
    douts = dy * F.silu(z) / 3

    _cmp(q(y), y, "correct y")
    _cmp(q(xg.grad), xg.grad, "correct dx")
    _cmp(q(u3), u3, "correct u (col_rev)")
    _cmp(q(gate), gate, "correct gate")
    cmp_f32(douts.float(), douts, "correct douts")
    # MIA_ORDER_COL_REV is an involution (the column walk commutes with the reversal), so a gather through its inverse is
    # the correct gather and no comparison can tell them apart; the gathers that lose the reversal or the walk must fail.
    assert torch.equal(TO_SCAN[3](x), TO_IMAGE[3](x))
    mutants = {"taps reversed": (_conv_ref(x, w.flip(-1), bias), y),
               "halo dropped": (halo_dropped, y),
               "dy tail dropped": (_dx_of(dp, w, True), xg.grad),
               "COL_REV gathered as COL": (_conv_ref(TO_SCAN[2](x), w, bias), u3),
               "COL_REV gathered as SEQ_REV": (_conv_ref(TO_SCAN[1](x), w, bias), u3),
               "gate / n_dirs": (F.silu(z) * s / 4, gate)}
    for what, (bad, ref) in mutants.items():
        with pytest.raises(AssertionError):
            _cmp(q(bad), ref, what)
    with pytest.raises(AssertionError):
        cmp_f32(douts.to(torch.bfloat16).float(), douts, "douts rounded to bf16")

    for layout in ("cm", "tm"):                                        # one store past the last channel
        o = Opd(layout, b, d, L, T, dev="cpu")
        o.set(q(y))
        o.untouched(f"correct {layout}")
        if layout == "cm":
            o.buf[1, d, 5] = 0                                          # channel d: the other half
        else:
            o.buf[3, d] = 0                                             # pad column of a token-major row (d % 8 = 4)
        with pytest.raises(AssertionError):
            o.untouched(f"stray store ({layout})")


def test_criteria_reject_one_item_missing_from_dweight():
    """At ARM-base's size (32 x 768 x 197: 128 items per channel tile over 88 parts) dweight / dbias without one (batch,
    token tile) item's contribution fail the dweight criterion; the full sums pass."""
    b, d, L = BENCH
    W = 4
    g = torch.Generator().manual_seed(3)
    x = torch.randn(b, d, L, generator=g).bfloat16().double()
    w, bias = (torch.randn(d, W, generator=g) * 0.4).double(), (torch.randn(d, generator=g) * 0.1).double()
    dp = _dpre(x, w, bias, torch.randn(b, d, L, generator=g).bfloat16().double())
    xp = F.pad(x, (W - 1, 0))

    def sums(dpre):
        dw = torch.stack([(dpre * xp[..., k:k + L]).sum((0, 2)) for k in range(W)], -1)
        return dw, dpre.sum((0, 2))

    dw, db = sums(dp)
    _cmp_w(dw.float(), dw, "correct dweight")
    _cmp_w(db.float(), db, "correct dbias")
    missing = dp.clone()
    missing[5, :, TILE:2 * TILE] = 0                                    # item (batch 5, token tile 1)
    mdw, mdb = sums(missing)
    with pytest.raises(AssertionError):
        _cmp_w(mdw.float(), dw, "dweight without one item")
    with pytest.raises(AssertionError):
        _cmp_w(mdb.float(), db, "dbias without one item")
