"""Every selective-scan kernel instantiation (csrc/scan_*.cuh, launched from scan_api.cu) against float64, at the shapes,
dtypes and layouts where a scan kernel goes wrong.

A case table gives each of the 264 instantiations at least one launch but UNREACHED's 4, which no problem reaches on an
H100: the column-walk, chunk-parallel, resident-row, streaming and d_state 8 / 16 row-serial forwards, the warp-scan
forwards and backwards (deterministic ones included), the d_state 16 row-serial, column-walk and resident-row backwards, and the finalize kernel, in fp32, bf16 and fp16 with outputs
in the input dtype or (2-byte inputs) in fp32.  A Python replica of the planner's eligibility rules (scan_api.cu) names the
instantiations each case must launch; a child interpreter records what ran (kernel_trace) and one test holds every case to
its targets, another the targets to the full list.  Seqlens sit around the 8-token lane vector, the lanes_per_row switch,
the 16-token column groups and the 256-token checkpoint chunk; dims around the 32-row item, with ragged last rows, rows per
group that make g fall back, delta groups, 1 to 4 B / C groups and d_state 1 to 16.

Operands live in NaN-filled buffers: dense ones at a 16-byte-aligned offset between NaN guard bands, the warp-scan
families' operands also with a padded row pitch (every stride the ABI takes: u, delta, z, dout, out_saved, out, out_z, du,
ddelta, dz, and dB / dC across groups and states).  A stray read turns a result NaN; a stray write shows bit for bit.
Results are compared with the fp64 C oracle (oracle/ss_ref_c) under tests/parity.py's criteria, and the per-chunk
(prod a, h) checkpoints in x with a float64 statement of them.  Every call runs twice with bit-identical results (the
warp-scan d_state > 1 backward's dB / dC, reduced with red.global.add, only in deterministic mode).  Cases at training sizes
make the persistent kernels' CTAs walk several items, with a partial last round; the launch grids in the profiler trace
show it.  CPU tests check the list against the built library and show the criteria reject subtly wrong results."""
import ctypes
import json
import os
import re
import shutil
import tempfile
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_trace
from tests.parity import cmp_auto, cmp_f32, long_row_scale
from tests.test_conv_tiles_gpu import LIB, _bits, _demangled_kernels, _same_bits

gpu = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
TNAME = {F32: "float", F16: "__half", BF16: "__nv_bfloat16"}
# dtype id -> (input dtype, outputs / douts in fp32 while the inputs are 2-byte)
COMBOS = {"f32": (F32, False), "bf16": (BF16, False), "bf16o32": (BF16, True), "f16": (F16, False), "f16o32": (F16, True)}
KERNEL = re.compile(r"\b(ss_\w*kernel)<")
OPTIN = 227 * 1024                   # shared memory one CTA may opt in to on an H100 (the planners' kSmemPerSm)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


SMS = _sms()


def _tf(v):
    return "true" if v else "false"


def _cdiv(a, b):
    return -(-a // b)


def _round_up(x, m):
    return _cdiv(x, m) * m


# ---------------------------------------------------------------------------------------------------------- instantiations
def _instantiations():
    """The scan kernels a release build holds, as CUPTI names them (template arguments only).  fp32 inputs store and read
    fp32 directly: kOutF32 is false for the row-serial / column-walk / chunk-parallel families and true for the fast
    warp-scan kernels, the only values the host selects."""
    out = []
    for t in TNAME.values():
        two = t != "float"
        ofs = (False, True) if two else (False,)
        for sp in map(_tf, (True, False)):
            for of in map(_tf, ofs):
                for g in (1, 2, 4) if two else (1,):
                    out += [f"ss_fwd_cw_kernel<{t}, {sp}, {of}, {g}>", f"ss_bwd_cw_kernel<{t}, {sp}, {of}, {g}>"]
                out += [f"ss_fwd_rows_kernel<{t}, {sp}, {of}>", f"ss_bwd_rows_kernel<{t}, {sp}, {of}>",
                        f"ss_fwd_stream_kernel<{t}, {sp}, {of}>", f"ss_fwd_chunk_kernel<{t}, {sp}, {of}, false>"]
                out += [f"ss_fwd_rowsn_kernel<{t}, {sp}, {of}, {n}, {_tf(z)}>" for n in (8, 16) for z in (True, False)]
            out.append(f"ss_fwd_chunk_kernel<{t}, {sp}, false, true>")
            for of in map(_tf, ofs if two else (True,)):
                out += [f"ss_fwd_fast_kernel<{t}, {sp}, {of}>", f"ss_bwd_fast_kernel<{t}, {sp}, {of}>"]
                out += [f"ss_bwd_fastn_kernel<{t}, {sp}, {of}, {_tf(det)}>" for det in (False, True)]
            for to in (t, "float") if two else (t,):
                out += [f"ss_bwd_rowsn_kernel<{t}, {to}, {sp}, {_tf(z)}>" for z in (True, False)]
            for n1 in (True, False):
                for lpr in (0, 32):
                    out += [f"ss_fwd_kernel<{t}, {sp}, {_tf(n1)}, {lpr}>", f"ss_bwd_kernel<{t}, {sp}, {_tf(n1)}, {lpr}, false>"]
                    if not n1:
                        out.append(f"ss_bwd_kernel<{t}, {sp}, false, {lpr}, true>")
        out += [f"ss_fwd_chunk_combine_kernel<{t}>", f"ss_finalize_kernel<{t}>"]
    return out


INSTANTIATIONS = _instantiations()
# The fp32 resident-row and streaming forwards are built but no fp32 problem reaches them on an H100: every shape their
# planners accept (dense rows, 16-byte aligned, A per row) is taken first by the column-walk forward (rows of one
# checkpoint chunk, or at least 4 items of 32 rows per SM) or by the chunk-parallel forward (3 of its 68.7 KB fp32 CTAs fit
# an SM's 227 KB).  A 2-byte problem reaches both.
UNREACHED = {f"ss_fwd_{k}_kernel<float, {sp}, false>" for k in ("rows", "stream") for sp in ("true", "false")}


def short_name(name):
    """'void mia::ss_fwd_cw_kernel<__half, true, true, 2>(CUtensorMap_st, ...)' -> 'ss_fwd_cw_kernel<__half, true, true, 2>'."""
    m = KERNEL.search(name)
    return f"{m.group(1)}<{', '.join(kernel_trace.targs(name, m.group(1) + '<'))}>"


# ---------------------------------------------------------------------------------------------------------- planner replica
def lanes_per_row(L):
    if L > 128:
        return 32
    lpr = 4
    while lpr < _cdiv(L, 8):
        lpr <<= 1
    return lpr


def chunk_len(L):
    return lanes_per_row(L) * 8


def n_chunks(L):
    return _cdiv(L, chunk_len(L))


def warp_segments(B, dim, L, N, G, det=False):
    """Segments of the warp-scan kernels (make_plan in scan_api.cu): ~6 per SM (1 for the deterministic d_state > 1
    backward), at most one per RPP rows, with the best last-wave balance."""
    rpg, bg, rpp = dim // G, B * G, 32 // lanes_per_row(L)
    hi, lo = _cdiv(rpg, rpp), 1
    while _cdiv(rpg, lo) * N > 4096 and lo < hi:
        lo += 1
    want = min(max(_cdiv((1 if det else 6) * SMS, bg), lo), hi)
    split = lambda sp: _cdiv(rpg, _cdiv(rpg, sp))
    best, best_eff = want, -1.0
    for sp in range(want, min(want + 3, hi) + 1):
        ns = bg * split(sp)
        eff = ns / SMS / _cdiv(ns, SMS)
        if eff > best_eff + 1e-9:
            best, best_eff = sp, eff
    return bg * split(best)


# ---------------------------------------------------------------------------------------------------------- the case table
@dataclass
class Case:
    """One forward, then the backward without the forward's block states and, where the forward wrote them, on them.
    ``pitch``: every strided operand with a padded row pitch (only the warp-scan kernels take such operands);
    ``regime``: "ref" = the reference's generators (test_scan_gpu._inputs), "model" = test_scan_ranges_gpu.range_inputs;
    ``spot``: images compared against the oracle (all when empty); ``walk``: phases whose persistent kernel must give
    some CTAs a second item and leave the last round partial."""
    combo: str
    shape: tuple                 # (batch, dim, seqlen, d_state, n_groups, delta_dim)
    sp: bool = True
    D: bool = True
    bias: bool = True
    z: bool = False
    det: bool = False
    pitch: bool = False
    regime: str = "ref"
    spot: tuple = ()
    walk: tuple = ()
    fs_mult: float = 1.0
    note: str = ""

    @property
    def dtype(self):
        return COMBOS[self.combo][0]

    @property
    def o32(self):
        return COMBOS[self.combo][1]

    @property
    def otype(self):
        return F32 if self.o32 else self.dtype

    @property
    def es(self):
        return self.dtype.itemsize

    @property
    def eo(self):
        return self.otype.itemsize

    @property
    def rpg(self):
        return self.shape[1] // self.shape[4]

    @property
    def id(self):
        B, dim, L, N, G, dd = self.shape
        s = f"{self.combo}-b{B}d{dim}L{L}N{N}G{G}" + (f"dd{dd}" if dd != dim else "")
        s += "-sp" if self.sp else "-nosp"
        s += "".join(f"-{k}" for k, on in (("D", self.D), ("bias", self.bias), ("z", self.z), ("det", self.det),
                                            ("pitch", self.pitch)) if on)
        s += "-model" if self.regime == "model" else ""
        return s + (f"-{self.note}" if self.note else "")

    # ---- the planner's eligibility rules (scan_api.cu), for the operands this file builds (A contiguous, 16-byte aligned)
    def rowwise(self):
        B, dim, L, N, G, dd = self.shape
        return N == 1 and not self.z and dd == dim and self.rpg % 32 == 0 and L % 4 == 0

    def cw_g(self):
        """cw_geometry: rows per tensor-map row, 0 when the column-walk kernels decline."""
        B, dim, L, N, G, dd = self.shape
        if not self.rowwise() or self.pitch:
            return 0
        if self.es == 4:
            return 1
        slots = SMS * (9 if self.eo == 4 else 12)
        c, fallback = (1 if L % 16 == 0 else 2 if L % 8 == 0 else 4), 0
        while c >= 1:
            if (c * L * self.es) % 16:
                break
            if not (c > 1 and L > 256) and self.rpg % (32 * c) == 0:
                items = B * G * (self.rpg // (32 * c))
                if items <= slots or items >= 2 * slots:
                    return c
                fallback = fallback or c
            c >>= 1
        return fallback

    def rowsn_fwd_smem(self):
        B, dim, L, N, G, dd = self.shape
        tile = _round_up(32 * L * self.es, 128)
        return (6 if self.z else 8) * tile + _round_up(2 * L * N * self.es, 128) + 128

    def rows_bwd_ok(self):
        """plan_rows_bwd: at least 3 resident CTAs per SM, and rows of several chunks only while every item has its CTA."""
        B, dim, L, N, G, dd = self.shape
        nch = _cdiv(L, 256)
        if nch > 1 and (chunk_len(L) != 256 or (L * self.es) % 16 or (L * self.eo) % 16):
            return False
        span = L if nch == 1 else 256
        t0 = (span * 52 // 100) // 4 * 4
        nblk = _cdiv(max(t0, span - t0), 16)
        extra = 16 if nch > 1 else 0
        smem = (2 * _round_up(32 * (span * self.es + extra), 128) + _round_up(32 * (span * self.eo + extra), 128)
                + _round_up(2 * (_round_up(span, 16) + 16) * 4, 128) + 3 * nblk * 128 + 7 * 128 + 128)
        per_sm = min(OPTIN // (smem + 1024), 5)
        return per_sm >= 3 and not (nch > 1 and self.items32() > SMS * per_sm)

    def items32(self):
        B, dim, L, N, G, dd = self.shape
        return B * G * (self.rpg // 32)

    def fwd_family(self):
        B, dim, L, N, G, dd = self.shape
        if self.rowwise() and not self.pitch:
            g, nch = self.cw_g(), _cdiv(L, 256)
            if g and not (B * G * (self.rpg // (32 * g)) < 4 * SMS and nch >= 2):
                return "cw"
            if nch >= 2 and (L * self.es) % 16 == 0 and (L * self.eo) % 16 == 0 and self.items32() < 4 * SMS:
                return "chunks"
            if 32 * L * self.es <= 13 * 1024 or (L * self.es) % 16 == 0:
                return "rows"
            return "stream"
        if (N in (8, 16) and dd == dim and self.rpg % 32 == 0 and n_chunks(L) == 1 and not self.pitch
                and self.rowsn_fwd_smem() <= OPTIN):
            return "rowsn"
        return "fast" if N == 1 and lanes_per_row(L) == 32 and not self.z and dd == dim else "warp"

    def writes_hblk(self):
        return self.fwd_family() == "cw"

    def bwd_family(self, hblk):
        B, dim, L, N, G, dd = self.shape
        if N == 16 and dd == dim and L <= 256 and self.rpg % 8 == 0 and not self.pitch:
            return "rowsn"
        if hblk and (L <= 256 or B * (dim // 32) >= 4 * SMS) and self.cw_g():
            return "cw"
        if self.rowwise() and not self.pitch and self.rows_bwd_ok():
            return "rows"
        fast = lanes_per_row(L) == 32 and dd == dim
        if self.det and N > 1:
            return "fastn" if fast else "warp"
        return ("fast" if N == 1 else "fastn") if fast and (N > 1 or not self.z) else "warp"

    def nondet_bc(self):
        """The backward reduces dB / dC with red.global.add (warp-scan d_state > 1, not deterministic)."""
        return self.shape[3] > 1 and not self.det and self.bwd_family(False) in ("fastn", "warp")

    def target(self, phase):
        """The instantiations the phase ("fwd", "bwd", "bwdh") launches."""
        B, dim, L, N, G, dd = self.shape
        t, sp = TNAME[self.dtype], _tf(self.sp)
        of = _tf(self.o32)
        lpr = 32 if lanes_per_row(L) == 32 else 0
        if phase == "fwd":
            fam = self.fwd_family()
            return {"cw": {f"ss_fwd_cw_kernel<{t}, {sp}, {of}, {self.cw_g()}>"},
                    "chunks": {f"ss_fwd_chunk_kernel<{t}, {sp}, false, true>", f"ss_fwd_chunk_kernel<{t}, {sp}, {of}, false>",
                               f"ss_fwd_chunk_combine_kernel<{t}>"},
                    "rows": {f"ss_fwd_rows_kernel<{t}, {sp}, {of}>"},
                    "stream": {f"ss_fwd_stream_kernel<{t}, {sp}, {of}>"},
                    "rowsn": {f"ss_fwd_rowsn_kernel<{t}, {sp}, {of}, {N}, {_tf(self.z)}>"},
                    "fast": {f"ss_fwd_fast_kernel<{t}, {sp}, {_tf(self.o32 or t == 'float')}>"},
                    "warp": {f"ss_fwd_kernel<{t}, {sp}, {_tf(N == 1)}, {lpr}>"}}[fam]
        fam = self.bwd_family(phase == "bwdh")
        det = _tf(self.det and N > 1)
        main = {"rowsn": f"ss_bwd_rowsn_kernel<{t}, {'float' if self.o32 else t}, {sp}, {_tf(self.z)}>",
                "cw": f"ss_bwd_cw_kernel<{t}, {sp}, {of}, {self.cw_g()}>",
                "rows": f"ss_bwd_rows_kernel<{t}, {sp}, {of}>",
                "fast": f"ss_bwd_fast_kernel<{t}, {sp}, {_tf(self.o32 or t == 'float')}>",
                "fastn": f"ss_bwd_fastn_kernel<{t}, {sp}, {_tf(self.o32 or t == 'float')}, {det}>",
                "warp": f"ss_bwd_kernel<{t}, {sp}, {_tf(N == 1)}, {lpr}, {det}>"}[fam]
        return {main, f"ss_finalize_kernel<{t}>"}

    def phases(self):
        return ("fwd", "bwd", "bwdh") if self.writes_hblk() else ("fwd", "bwd")

    def items(self, phase):
        """Work items of the phase's persistent kernel (what one CTA takes per round)."""
        B, dim, L, N, G, dd = self.shape
        fam = self.fwd_family() if phase == "fwd" else self.bwd_family(phase == "bwdh")
        if fam == "cw":
            return B * G * (self.rpg // (32 * self.cw_g()))
        if fam == "chunks":
            return self.items32() * _cdiv(L, 256)
        if fam in ("rows", "stream"):
            return self.items32()
        if fam == "rowsn" and phase == "fwd":
            return B * G * _cdiv(self.rpg // 32, 2 if self.z else 4)
        if fam == "rowsn":
            return B * dim // 8                                        # octets of rows
        return warp_segments(B, dim, L, N, G, det=phase != "fwd" and self.det and N > 1)


def _mk(combo, shape, sp, k, **kw):
    """A case with D / bias rotating through their four settings, and the models' value regime every third softplus case."""
    kw.setdefault("D", k % 4 in (0, 2))
    kw.setdefault("bias", k % 4 in (0, 1))
    if sp and k % 3 == 0 and kw.get("regime", "ref") == "ref":
        kw["regime"] = "model"
    return Case(combo, shape, sp, **kw)


TWO = ("bf16", "bf16o32", "f16", "f16o32")
SPS = (True, False)

# column-walk pair; g rows per tensor-map row: L % 16 == 0 -> 1; L % 16 == 8 -> 2; L % 8 == 4 -> 4 (rows_per_group % 128 == 0)
# or 2 (rows_per_group % 64 == 0 only: g falls back)
CW = {1: [(2, 64, 256, 1, 2, 64), (3, 32, 64, 1, 1, 32), (1, 96, 16, 1, 3, 96), (2, 64, 240, 1, 1, 64), (1, 128, 128, 1, 4, 128),
          (2, 32, 32, 1, 1, 32), (2, 64, 48, 1, 2, 64), (1, 96, 144, 1, 1, 96)],
      2: [(2, 64, 200, 1, 1, 64), (1, 128, 8, 1, 2, 128), (2, 64, 24, 1, 1, 64), (1, 192, 136, 1, 3, 192), (2, 64, 196, 1, 1, 64),
          (1, 128, 36, 1, 2, 128), (2, 128, 120, 1, 2, 128), (1, 64, 4, 1, 1, 64)],
      4: [(2, 128, 196, 1, 1, 128), (1, 128, 4, 1, 1, 128), (2, 256, 12, 1, 2, 256), (1, 128, 36, 1, 1, 128), (2, 128, 204, 1, 1, 128),
          (1, 512, 252, 1, 4, 512), (2, 128, 100, 1, 1, 128), (1, 256, 132, 1, 2, 256)]}
# chunk-parallel: rows of several 256-token chunks (L % 8 == 0), few 32-row items; the last chunk of 1 to 256 tokens
CHUNKS = [(1, 64, 512, 1, 2, 64), (1, 32, 264, 1, 1, 32), (2, 32, 1000, 1, 1, 32), (1, 64, 2048, 1, 1, 64), (1, 32, 6400, 1, 1, 32),
          (1, 96, 288, 1, 3, 96), (1, 32, 776, 1, 1, 32), (2, 32, 520, 1, 1, 32), (1, 128, 264, 1, 4, 128), (1, 32, 2056, 1, 1, 32)]
# resident-row forward (2-byte): L % 8 == 4 with rows_per_group an odd multiple of 32 (no legal g), L <= 208
ROWS = [(2, 96, 196, 1, 1, 96), (3, 32, 36, 1, 1, 32), (1, 32, 4, 1, 1, 32), (2, 96, 12, 1, 3, 96), (2, 160, 204, 1, 1, 160),
        (1, 64, 100, 1, 2, 64), (2, 32, 132, 1, 1, 32), (1, 128, 20, 1, 4, 128)]
# streaming forward (2-byte): like ROWS but 208 < L <= 256, or L > 256 with L % 8 == 4 (any rows per group)
STREAM = [(2, 32, 212, 1, 1, 32), (1, 64, 260, 1, 1, 64), (2, 96, 252, 1, 3, 96), (1, 32, 300, 1, 1, 32), (1, 128, 516, 1, 2, 128),
          (1, 32, 2052, 1, 1, 32), (2, 160, 228, 1, 1, 160), (1, 64, 260, 1, 2, 64)]
# d_state 8 / 16 row-serial forward: whole rows of one checkpoint chunk, rows per group % 32 == 0
ROWSN = [(2, 64, 196, 16, 2, 64), (1, 32, 4, 16, 1, 32), (2, 96, 100, 8, 3, 96), (1, 64, 208, 16, 1, 64), (3, 32, 52, 8, 1, 32),
         (2, 64, 197, 16, 2, 64), (1, 32, 129, 8, 1, 32), (2, 32, 1, 16, 1, 32), (1, 128, 200, 8, 4, 128), (2, 32, 255, 16, 1, 32),
         (1, 64, 7, 8, 2, 64), (2, 32, 128, 16, 1, 32)]
# warp-scan families (padded pitches, or a z gate / delta groups / ragged dims that the row-serial kernels decline)
W_N1_SHORT = [(2, 33, 1, 1, 1, 33), (1, 64, 3, 1, 2, 32), (2, 8, 7, 1, 1, 8), (1, 100, 8, 1, 4, 25), (2, 64, 12, 1, 2, 64),
              (1, 40, 127, 1, 2, 20), (2, 16, 128, 1, 1, 16), (1, 96, 36, 1, 3, 48)]
W_N1_LONG = [(2, 16, 129, 1, 1, 16), (1, 64, 196, 1, 2, 32), (1, 33, 257, 1, 1, 33), (1, 12, 2049, 1, 3, 12), (2, 40, 255, 1, 2, 20),
             (1, 64, 260, 1, 4, 16), (2, 8, 200, 1, 1, 8), (1, 16, 288, 1, 2, 16)]
W_FAST = [(2, 16, 129, 1, 1, 16), (1, 64, 195, 1, 2, 64), (1, 33, 257, 1, 1, 33), (1, 8, 2049, 1, 2, 8), (2, 64, 204, 1, 4, 64),
          (1, 12, 6400, 1, 1, 12), (2, 100, 200, 1, 2, 100), (1, 64, 256, 1, 1, 64), (2, 32, 196, 1, 1, 32), (1, 48, 288, 1, 3, 48)]
W_N_SHORT = [(2, 8, 37, 4, 2, 8), (2, 6, 1, 2, 1, 6), (1, 4, 7, 2, 1, 4), (2, 16, 100, 16, 4, 16), (1, 33, 128, 8, 1, 33),
             (2, 64, 12, 16, 2, 64), (1, 96, 127, 4, 3, 96), (2, 16, 4, 8, 1, 8), (1, 64, 3, 16, 1, 32), (2, 32, 36, 2, 2, 32)]
W_N_GROUPS = [(2, 8, 256, 2, 2, 4), (1, 64, 196, 16, 2, 32), (1, 8, 257, 4, 1, 2), (2, 32, 200, 8, 4, 16), (1, 16, 129, 16, 1, 8),
              (1, 12, 600, 4, 1, 6), (2, 64, 204, 2, 2, 16), (1, 32, 288, 16, 1, 16)]
W_N_FAST = [(2, 8, 256, 2, 2, 8), (1, 64, 196, 16, 2, 64), (1, 8, 257, 4, 1, 8), (2, 32, 200, 8, 4, 32), (1, 16, 129, 16, 1, 16),
            (1, 12, 600, 4, 1, 12), (2, 64, 204, 2, 2, 64), (1, 32, 288, 16, 1, 32), (2, 100, 255, 8, 2, 100), (1, 5, 2049, 2, 1, 5)]


def _walk_cases():
    """Training-size launches: for every persistent family and dtype / output type, more items than the grid holds and an
    item count the grid does not divide (primes), so CTAs take a second item and the last round is partial.  Three images
    are compared against the oracle."""
    out = []
    spot = lambda B: (0, B // 2, B - 1)
    for i, combo in enumerate(COMBOS):
        sp = i % 2 == 0
        # column-walk pair (797 items of 32 g rows: 2 rounds), and without block states the resident-row backward (2-byte)
        shape = (797, 32, 196, 1, 1, 32) if combo == "f32" else (797, 128, 196, 1, 1, 128)
        out.append(Case(combo, shape, sp, spot=spot(797), walk=("fwd", "bwd", "bwdh") if combo != "f32" else ("fwd", "bwdh"), note="walk"))
        # chunk-parallel forward: 101 items of 32 rows x 8 chunks.  6.6 M elements per tensor: as for the 5.6 M of
        # test_scan_parity_column_walk_two_chunks, the extreme tail of the fp32 error distribution passes the criterion
        # calibrated on small cases (H100, MIA_PARITY_LOG: 1 fp32 ddelta element at 1.32) -> that criterion x 2 here
        out.append(Case(combo, (1, 3232, 2048, 1, 1, 3232), not sp, walk=("fwd",), fs_mult=2.0, note="walk"))
        # d_state 16 row-serial pair: 797 units of one 32-row batch (fwd), 3188 octets (bwd)
        out.append(Case(combo, (797, 32, 196, 16, 1, 32), sp, z=i % 2 == 1, det=i % 2 == 0, spot=spot(797), walk=("fwd", "bwd"),
                        note="walk"))
        # warp-scan pair: 139 segments of one row over the SMs
        out.append(Case(combo, (1, 139, 200, 1 if i % 2 else 4, 1, 139), not sp, pitch=True, walk=("fwd", "bwd"), note="walk"))
        if combo == "f32":
            # resident-row backward in fp32: 797 items over at most 5 per SM (short rows: 3 fp32 CTAs fit)
            out.append(Case(combo, (797, 32, 36, 1, 1, 32), sp, spot=spot(797), walk=("fwd", "bwd", "bwdh"), note="walk"))
        else:
            # resident-row pair: 1409 items over at most 8 (fwd) / 5 (bwd) per SM
            out.append(Case(combo, (1409, 32, 196, 1, 1, 32), sp, spot=spot(1409), walk=("fwd", "bwd"), note="walk"))
            # streaming forward: 2131 items over at most 16 per SM; the warp-scan fast backward
            out.append(Case(combo, (2131, 32, 260, 1, 1, 32), not sp, spot=spot(2131), walk=("fwd", "bwd"), note="walk"))
    return out


def _cases():
    out = []
    for combo in COMBOS:
        two = combo != "f32"
        for j, sp in enumerate(SPS):
            for g in (1, 2, 4) if two else (1,):
                k = len(out)
                out.append(_mk(combo, CW[g][(k * 3 + j) % len(CW[g])], sp, k))
            k = len(out)
            out.append(_mk(combo, CHUNKS[(k + j) % len(CHUNKS)], sp, k))
            if two:
                out.append(_mk(combo, ROWS[(k + 3 * j) % len(ROWS)], sp, k + 1))
                out.append(_mk(combo, STREAM[(k + 5 * j) % len(STREAM)], sp, k + 2))
            for n in (8, 16):
                for z in (True, False):
                    k = len(out)
                    pool = [s for s in ROWSN if s[3] == n]
                    shape = pool[(k + j) % len(pool)]
                    out.append(_mk(combo, shape, sp, k, z=z, det=k % 2 == 0))
            # warp-scan: d_state 1 (short rows; long rows with z or delta groups; the fast pair), d_state > 1 (short rows,
            # long rows with delta groups, the fast pair), each backward also in deterministic mode where it has a kDet form
            k = len(out)
            out.append(_mk(combo, W_N1_SHORT[(k + j) % 8], sp, k, z=k % 3 == 0, pitch=True))
            out.append(_mk(combo, W_N1_LONG[(k + j) % 8], sp, k + 1, z=W_N1_LONG[(k + j) % 8][5] == W_N1_LONG[(k + j) % 8][1], pitch=k % 2 == 0))
            out.append(_mk(combo, W_FAST[(k + j) % 10], sp, k + 2, pitch=True))
            for det in (False, True):
                k = len(out)
                out.append(_mk(combo, W_N_SHORT[(k + j) % 10], sp, k, z=k % 4 == 0, det=det, pitch=k % 3 != 2))
                out.append(_mk(combo, W_N_GROUPS[(k + j) % 8], sp, k + 1, z=k % 5 == 0, det=det, pitch=k % 2 == 1))
                out.append(_mk(combo, W_N_FAST[(k + j) % 10], sp, k + 2, z=k % 3 == 1, det=det, pitch=True))
    # 25-chunk rows: the chunk-parallel forward with its resident-row backward, and the fast warp-scan pair
    out += [Case("bf16", (1, 32, 6400, 1, 1, 32), True, note="long"), Case("f16o32", (1, 12, 6400, 1, 1, 12), False, pitch=True, note="long")]
    # more than 32 images with delta groups: the finalize's lanes take a second batch in dA / dD and a second
    # (batch, row of the group) in ddelta_bias
    out += [Case("bf16", (40, 16, 100, 4, 2, 8), True, pitch=True, note="batch40"),
            # fp32 criterion x 2: one row has A = -0.011, so its state remembers the whole row, and one out element of it sits at
            # 1.10 of the criterion (H100, MIA_PARITY_LOG).  The ss_fwd_kernel instances with and without z and delta groups and
            # the fast kernel all give that element the same error, so it comes from the fp32 arithmetic they share, whose error
            # grows with the tokens a row remembers (parity.long_row_scale), not from one instantiation
            Case("f32", (37, 64, 196, 1, 2, 32), False, z=True, fs_mult=2.0, note="batch37")]
    return out + _walk_cases()


CASES = {c.id: c for c in _cases()}
assert len(CASES) == len(_cases()), "case ids must be unique"


# ---------------------------------------------------------------------------------------------------------- operands
class Buf:
    """A tensor of ``shape`` (innermost dim contiguous) inside a NaN-filled buffer: NaN guard bands of 64 elements before
    and after it (a 16-byte-aligned offset), and with ``pad`` > 0 a row pitch of shape[-1] + pad with NaN pad elements."""
    GUARD = 64

    def __init__(self, shape, dtype, pad=0, dev="cuda"):
        self.shape, self.pitch = tuple(shape), shape[-1] + pad
        self.rows = 1
        for s in shape[:-1]:
            self.rows *= s
        self.buf = torch.full((2 * self.GUARD + self.rows * self.pitch,), float("nan"), dtype=dtype, device=dev)

    def region(self, buf=None):
        b = self.buf if buf is None else buf
        return b[self.GUARD:self.GUARD + self.rows * self.pitch].view(*self.shape[:-1], self.pitch)[..., :self.shape[-1]]

    def set(self, v):
        self.region().copy_(v)
        return self

    def untouched(self, what):
        """Every element of the buffer outside the tensor is still the NaN it was filled with, bit for bit."""
        rest = self.buf.clone()
        self.region(rest).fill_(float("nan"))
        bad = int((_bits(rest) != _bits(torch.full_like(rest, float("nan")))).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the tensor"


def _host_inputs(c):
    """Seeded float inputs of a case, rounded to their storage dtypes (CPU)."""
    from tests.test_scan_gpu import _inputs
    from tests.test_scan_ranges_gpu import range_inputs
    B, dim, L, N, G, dd = c.shape
    seed = zlib.crc32(c.id.encode())
    if c.regime == "model":
        cpu = range_inputs("model", seed, B, dim, L, N, G, dd, has_D=c.D, has_z=c.z, has_bias=c.bias, softplus=True, dtype=c.dtype)
    else:
        cpu, _ = _inputs(seed, B, dim, L, N, G, dd, c.D, c.z, c.bias, c.dtype, dev="cpu")
    if c.o32:
        cpu["dout"] = cpu["dout"].float()
    return cpu


def _device_inputs(c, cpu):
    pad = 3 if c.pitch else 0
    dev = {}
    for k, v in cpu.items():
        if v is not None:
            dev[k] = Buf(v.shape, v.dtype, pad if v.dim() >= 3 else 0).set(v.to("cuda"))
    return dev


def _params(c, I, otype):
    from medical_image_analysis_b200 import _lib
    from medical_image_analysis_b200.scan_op import _fill_inputs
    r = lambda k: I[k].region() if k in I else None
    p = _lib.MiaSSParams()
    _fill_inputs(p, r("u"), r("delta"), r("A"), r("B"), r("C"), r("D"), r("delta_bias"), r("z"), c.sp, otype)
    return p


def _fwd(c, I):
    """The forward on NaN-filled outputs -> (outputs: name -> Buf, x, hblk or None)."""
    from medical_image_analysis_b200 import _lib
    B, dim, L, N, G, dd = c.shape
    pad = 3 if c.pitch else 0
    R = {"out": Buf((B, dim, L), c.otype, pad)}
    if c.z:
        R["out_z"] = Buf((B, dim, L), c.otype, pad)
    x = torch.full((B, dim, n_chunks(L), 2 * N), float("nan"), device="cuda")
    p = _params(c, I, c.otype)
    o = R["out"].region()
    p.out, p.x, p.out_batch_stride, p.out_d_stride = o.data_ptr(), x.data_ptr(), o.stride(0), o.stride(1)
    if c.z:
        oz = R["out_z"].region()
        p.out_z, p.out_z_batch_stride, p.out_z_d_stride = oz.data_ptr(), oz.stride(0), oz.stride(1)
    hblk = None
    nfl = int(_lib.lib().mia_ss_block_state_floats(ctypes.byref(p)))
    if nfl:
        hblk = torch.full((nfl,), float("nan"), device="cuda")
        p.hblk = hblk.data_ptr()
        if not _lib.lib().mia_ss_fwd_writes_block_states(ctypes.byref(p)):
            hblk, p.hblk = None, None
    _lib.call("mia_selective_scan_fwd", c.id, torch.device("cuda"), ctypes.byref(p))
    return R, x, hblk


GRADS = ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz")


def _bwd(c, I, R, x, hblk):
    """The backward (deterministic entry point for ``det`` cases) on NaN-filled outputs -> name -> Buf."""
    from medical_image_analysis_b200 import _lib
    B, dim, L, N, G, dd = c.shape
    pad = 3 if c.pitch else 0
    T = c.dtype
    Gr = {"du": Buf((B, dim, L), T, pad), "ddelta": Buf((B, dd, L), T, pad), "dA": Buf((dim, N), F32),
          "dB": Buf((B, G, N, L), T, pad), "dC": Buf((B, G, N, L), T, pad)}
    if c.D:
        Gr["dD"] = Buf((dim,), F32)
    if c.bias:
        Gr["ddelta_bias"] = Buf((dd,), F32)
    if c.z:
        Gr["dz"] = Buf((B, dim, L), T, pad)
    p = _params(c, I, c.otype)
    p.x = x.data_ptr()
    p.hblk = None if hblk is None else hblk.data_ptr()
    g = {k: v.region() for k, v in Gr.items()}
    d = I["dout"].region()
    p.dout, p.dout_batch_stride, p.dout_d_stride = d.data_ptr(), d.stride(0), d.stride(1)
    if c.z:
        o = R["out"].region()
        p.out_saved, p.out_saved_batch_stride, p.out_saved_d_stride = o.data_ptr(), o.stride(0), o.stride(1)
        p.dz, p.dz_batch_stride, p.dz_d_stride = g["dz"].data_ptr(), g["dz"].stride(0), g["dz"].stride(1)
    p.du, p.du_batch_stride, p.du_d_stride = g["du"].data_ptr(), g["du"].stride(0), g["du"].stride(1)
    p.ddelta, p.ddelta_batch_stride, p.ddelta_d_stride = g["ddelta"].data_ptr(), g["ddelta"].stride(0), g["ddelta"].stride(1)
    p.dA, p.dA_d_stride, p.dA_dstate_stride = g["dA"].data_ptr(), g["dA"].stride(0), g["dA"].stride(1)
    p.dB, p.dB_batch_stride, p.dB_group_stride, p.dB_dstate_stride = g["dB"].data_ptr(), *g["dB"].stride()[:3]
    p.dC, p.dC_batch_stride, p.dC_group_stride, p.dC_dstate_stride = g["dC"].data_ptr(), *g["dC"].stride()[:3]
    p.dD = g["dD"].data_ptr() if c.D else None
    p.ddelta_bias = g["ddelta_bias"].data_ptr() if c.bias else None
    lib = _lib.lib()
    name = "mia_selective_scan_bwd_deterministic" if c.det else "mia_selective_scan_bwd"
    ws_bytes = int(getattr(lib, name + "_workspace")(ctypes.byref(p)))
    ws = torch.empty((max(ws_bytes, 256),), dtype=torch.uint8, device="cuda")
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws_bytes
    _lib.call(name, c.id, torch.device("cuda"), ctypes.byref(p))
    torch.cuda.synchronize()
    return Gr


# ---------------------------------------------------------------------------------------------------------- float64 checks
def x_ref(u, delta, A, B, bias, softplus):
    """float64 per-chunk checkpoints of the forward: x[b, d, c, 2n] = prod a over tokens 0 .. end of chunk c
    (= exp(A[d, n] sum delta')), x[b, d, c, 2n + 1] = h after that token; chunks of mia_ss_chunk_len(L) tokens."""
    b, dim, L = u.shape
    N, G, ratio = A.shape[1], B.shape[1], dim // delta.shape[1]
    dl = delta.double() + (bias.double()[:, None] if bias is not None else 0.0)
    dl = (F.softplus(dl) if softplus else dl).repeat_interleave(ratio, 1)
    Bx = B.double().repeat_interleave(dim // G, 1)
    A64, u64 = A.double(), u.double()
    du = dl * u64
    h = torch.zeros(b, dim, N, dtype=torch.float64)
    S = torch.zeros(b, dim, 1, dtype=torch.float64)
    CH = chunk_len(L)
    x = torch.empty(b, dim, n_chunks(L), 2 * N, dtype=torch.float64)
    for t in range(L):
        h = torch.exp(dl[:, :, t, None] * A64) * h + du[:, :, t, None] * Bx[..., t]
        S += dl[:, :, t, None]
        if (t + 1) % CH == 0 or t == L - 1:
            x[:, :, t // CH, 0::2] = torch.exp(S * A64)
            x[:, :, t // CH, 1::2] = h
    return x


def _cmp_x(got, ref, what, fs):
    """prod a and h of every checkpoint, each by cmp_f32 (scaled like every fp32 tensor of long rows)."""
    cmp_auto(got[..., 0::2], ref[..., 0::2], what + " x prod a", f32_scale=fs)
    cmp_auto(got[..., 1::2], ref[..., 1::2], what + " x h", f32_scale=fs)


def _check(c, cpu, R, x, grads):
    """Forward outputs, checkpoints and per-image gradients against float64 on images ``c.spot`` (all when empty); dA, dD and
    ddelta_bias, sums over every image, always over the whole batch: the finalize's loops over the batch and the partials
    that a CTA's later items write are checked at every batch size."""
    from oracle import ss_ref_c
    B, dim, L, N, G, dd = c.shape
    fs = long_row_scale(L) * c.fs_mult
    lowp = c.dtype != F32
    dz_ulp = 2.0 if (c.z and lowp and not c.o32) else 1.0
    # stored 2-byte gradients of multi-chunk rows at training batches: 2 ulp (test_scan_headline_batches_spot_images)
    n_ulp = 2.0 if (c.spot and L > 256) else 1.0
    ref = ss_ref_c.bwd(cpu["u"], cpu["delta"], cpu["A"], cpu["B"], cpu["C"], cpu["D"], cpu["z"], cpu["delta_bias"], cpu["dout"], c.sp)
    for path, Gr in grads.items():
        for name in ("dA", "dD", "ddelta_bias"):
            if name in Gr:
                cmp_auto(Gr[name].region(), ref[name], f"[{c.id}]{path} {name}", f32_scale=fs)
    for imgs in ([slice(b, b + 1) for b in c.spot] if c.spot else [slice(0, B)]):
        tag = f"[{c.id} img {imgs.start}]"
        s = {k: (v[imgs] if (v is not None and v.dim() >= 3) else v) for k, v in cpu.items()}
        r_out, r_out_z, _ = ss_ref_c.fwd(s["u"], s["delta"], s["A"], s["B"], s["C"], s["D"], s["z"], s["delta_bias"], c.sp)
        cmp_auto(R["out"].region()[imgs], r_out, tag + " out", f32_scale=fs)
        if c.z:
            cmp_auto(R["out_z"].region()[imgs], r_out_z, tag + " out_z", f32_scale=fs)
        _cmp_x(x[imgs], x_ref(s["u"], s["delta"], s["A"], s["B"], s["delta_bias"], c.sp), tag, fs)
        for path, Gr in grads.items():
            for name in ("du", "ddelta", "dB", "dC", "dz"):
                if name in Gr:
                    cmp_auto(Gr[name].region()[imgs], ref[name][imgs], f"{tag}{path} {name}", n_ulp=dz_ulp if name == "dz" else n_ulp,
                             f32_scale=fs)


def _same(a, b, what):
    assert _same_bits(a, b), f"{what}: two calls differ"


def run_case(c):
    cpu = _host_inputs(c)
    I = _device_inputs(c, cpu)
    R, x, hblk = _fwd(c, I)
    R2, x2, hblk2 = _fwd(c, I)
    for k in R:
        _same(R[k].buf, R2[k].buf, f"{c.id} {k}")
        R[k].untouched(f"{c.id} {k}")
    _same(x, x2, f"{c.id} x")
    assert (hblk is None) == (not c.writes_hblk()), f"{c.id}: block states {hblk is not None}"
    if hblk is not None:
        _same(hblk, hblk2, f"{c.id} hblk")
    del R2, x2, hblk2
    grads = {}
    for path, hb in (("", None),) + ((("[hblk]", hblk),) if hblk is not None else ()):
        Gr, Gr2 = _bwd(c, I, R, x, hb), _bwd(c, I, R, x, hb)
        for k in Gr:
            if not (c.nondet_bc() and k in ("dB", "dC")):
                _same(Gr[k].buf, Gr2[k].buf, f"{c.id}{path} {k}")
            Gr[k].untouched(f"{c.id}{path} {k}")
        grads[path] = Gr
    torch.cuda.synchronize()
    _check(c, cpu, R, x, grads)


@gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_scan_kernel_parity(cid):
    """The case's forward and backwards against float64 on the same rounded inputs, nothing written outside any output, and
    a second call bit-identical to the first."""
    run_case(CASES[cid])


# ---------------------------------------------------------------------------------------------------------- launched kernels
def _capture(fn):
    """[(instantiation, grid x)] of the scan kernels fn() launches, from the exported Kineto trace."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return res, [(short_name(e["name"]), e["args"]["grid"][0]) for e in events
                 if e.get("cat") == "kernel" and KERNEL.search(e.get("name", ""))]


def launches():
    """Run in a child interpreter: the scan kernels (and their grids) of each case's forward and backwards."""
    out = {}
    for cid, c in CASES.items():
        I = _device_inputs(c, _host_inputs(c))
        got = {}
        n_fwd = 3 if c.fwd_family() == "chunks" else 1
        (R, x, hblk), got["fwd"] = kernel_trace.retry(lambda: _capture(lambda: _fwd(c, I)), lambda r: len(r[1]) >= n_fwd, tries=6)
        got["bwd"] = kernel_trace.retry(lambda: _capture(lambda: _bwd(c, I, R, x, None)), lambda r: len(r[1]) >= 2, tries=6)[1]
        if hblk is not None:
            got["bwdh"] = kernel_trace.retry(lambda: _capture(lambda: _bwd(c, I, R, x, hblk)), lambda r: len(r[1]) >= 2, tries=6)[1]
        out[cid] = got
        del I, R, x, hblk
    return out


@pytest.fixture(scope="module")
def traced():
    return kernel_trace.in_child("tests.test_scan_kernels_gpu:launches")


@gpu
def test_every_case_launches_its_target(traced):
    """Each phase of each case ran exactly the instantiations the planner replica assigns it (the backward: its kernel and
    the finalize), and nothing else; the forward wrote block states exactly when it is the column-walk kernel."""
    wrong = {}
    for cid, c in CASES.items():
        for ph in ("fwd", "bwd", "bwdh"):
            want = c.target(ph) if ph in c.phases() else None
            got = traced[cid].get(ph)
            if (got is None) != (want is None) or (want is not None and {n for n, _ in got} != want):
                wrong[f"{cid} {ph}"] = (None if got is None else sorted({n for n, _ in got}), None if want is None else sorted(want))
    assert not wrong, wrong


@gpu
def test_all_instantiations_launched_and_compared(traced):
    """The cases' targets are the 264 instantiations but the 4 UNREACHED ones, and every one of them was seen running."""
    targets = set().union(*(c.target(ph) for c in CASES.values() for ph in c.phases()))
    launched = {n for phases in traced.values() for names in phases.values() for n, _ in names}
    want = set(INSTANTIATIONS) - UNREACHED
    assert targets == want == launched, (sorted(want - launched), sorted(launched - want))
    print(f"{len(launched)}/{len(INSTANTIATIONS)} scan instantiations launched and compared ({len(CASES)} cases)")


@gpu
def test_persistent_walks_take_several_items(traced):
    """In the training-size cases every persistent kernel of the walking phases had more items than CTAs, and a count its
    grid does not divide: some CTAs took a second item and the last round was partial.  Items are counted by the planner
    replica, the grid read from the trace; for the rowsn backward, whose CTAs take contiguous runs of octets, the grid must
    be the replica's run count, and the last run short."""
    seen = set()
    for cid, c in CASES.items():
        for ph in c.walk:
            items = c.items(ph)
            fam = c.fwd_family() if ph == "fwd" else c.bwd_family(ph == "bwdh")
            for name, grid in traced[cid][ph]:
                if name.startswith(("ss_finalize", "ss_fwd_chunk_combine")):
                    continue
                if fam == "rowsn" and ph != "fwd":
                    # contiguous runs of oct_per_cta octets per CTA (rowsn_bwd_split): the last CTA's run is short
                    per = _cdiv(items, SMS * 3)
                    assert grid == _cdiv(items, per) and per >= 2 and items % per != 0, (cid, ph, name, items, per, grid)
                else:                                   # items strided over the grid
                    assert items > grid and items % grid != 0, (cid, ph, name, items, grid)
                print(f"{cid} {ph} {name}: {items} items over {grid} CTAs")
                seen.add((fam, ph == "fwd", c.combo))
    fams = {(f, fwd) for f, fwd, _ in seen}
    assert {("cw", True), ("cw", False), ("rows", True), ("rows", False), ("stream", True), ("chunks", True), ("rowsn", True),
            ("rowsn", False), ("fast", True), ("fast", False), ("warp", True), ("fastn", False)} <= fams, sorted(fams)
    for f, fwd in (("cw", True), ("cw", False), ("chunks", True), ("rowsn", True), ("rowsn", False), ("rows", False)):
        assert {combo for g, w, combo in seen if (g, w) == (f, fwd)} == set(COMBOS), (f, fwd)
    for f, fwd in (("rows", True), ("stream", True)):
        assert {combo for g, w, combo in seen if (g, w) == (f, fwd)} == set(TWO), (f, fwd)


# ---------------------------------------------------------------------------------------------------------- CPU checks
def test_case_table_covers_every_instantiation_and_edge():
    """The replica assigns every instantiation to a case, and the table holds the seqlens, dims, groups, d_states, flags and
    walks it is meant to."""
    cases = list(CASES.values())
    assert len(INSTANTIATIONS) == len(set(INSTANTIATIONS)) == 264 and UNREACHED < set(INSTANTIATIONS)
    targets = set().union(*(c.target(ph) for c in cases for ph in c.phases()))
    want = set(INSTANTIATIONS) - UNREACHED
    assert targets == want, (sorted(want - targets), sorted(targets - want))
    Ls = {c.shape[2] for c in cases}
    assert {1, 3, 4, 7, 8, 12, 127, 128, 129, 36, 196, 200, 204, 255, 256, 257, 260, 288, 2049, 6400} <= Ls
    assert {c.shape[2] % 16 for c in cases if c.fwd_family() == "cw"} == {0, 4, 8, 12}
    assert {c.shape[3] for c in cases} >= {1, 2, 4, 8, 16}
    assert {c.shape[4] for c in cases} >= {1, 2, 3, 4}
    assert any(c.shape[5] < c.shape[1] for c in cases)                                     # delta groups
    assert any(c.shape[1] % 32 for c in cases)                                             # a ragged last 32-row item
    assert any(c.cw_g() == 2 and c.rpg % 128 and c.shape[2] % 8 == 4 for c in cases)       # g falls back from 4 to 2
    for fam in ("cw", "chunks", "rows", "stream", "rowsn", "fast", "warp"):
        mine = [c for c in cases if c.fwd_family() == fam]
        assert any(c.regime == "model" for c in mine), fam
        assert {(c.D, c.bias) for c in mine} == {(a, b) for a in (True, False) for b in (True, False)}, fam
    assert {c.z for c in cases if c.fwd_family() in ("rowsn", "warp")} == {True, False}
    assert any(c.pitch for c in cases if c.bwd_family(False) in ("fast", "fastn", "warp"))
    # weight gradients over more than 32 images: with delta groups, and after multi-round walks of every backward family
    assert any(c.shape[0] > 32 and c.shape[5] < c.shape[1] and c.bias for c in cases)
    walked = {c.bwd_family(ph == "bwdh") for c in cases for ph in c.walk if ph != "fwd" and c.D and c.bias}
    assert {"cw", "rows", "rowsn", "fast", "fastn"} <= walked, walked


def test_checkpoint_geometry_matches_the_library():
    """The replica's x geometry is the library's: mia_ss_chunk_len / mia_ss_num_chunks for every seqlen in the table.  (The
    replica's family and g choices are checked on the GPU, by test_every_case_launches_its_target.)"""
    if not os.path.exists(LIB):
        pytest.skip("needs the built library (python -c 'import __graft_entry__ as g; g.build()')")
    from medical_image_analysis_b200 import _lib
    for L in sorted({c.shape[2] for c in CASES.values()} | set(range(1, 300))):
        assert (_lib.lib().mia_ss_chunk_len(L), _lib.lib().mia_ss_num_chunks(L)) == (chunk_len(L), n_chunks(L)), L


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(LIB),
                    reason="needs cuobjdump, cu++filt and the built library (python -c 'import __graft_entry__ as g; g.build()')")
def test_instantiation_list_is_the_built_one():
    """INSTANTIATIONS is exactly the set of selective-scan kernels with SASS in libmia_scan.so: 264, the 3 finalize kernels
    and the 3 chunk combines among them."""
    found = {full for base, full in _demangled_kernels() if re.fullmatch(r"ss_(fwd|bwd|finalize)\w*kernel", base)}
    assert found == set(INSTANTIATIONS), (sorted(found - set(INSTANTIATIONS)), sorted(set(INSTANTIATIONS) - found))
    assert len(found) == 264
    assert sum(n.startswith("ss_finalize_kernel<") for n in found) == 3


# ---------------------------------------------------------------------------------------------------------- mutants
def _scan64(u, dl, A, Bx, Cx, D, z=None, drop_last=False, carry_lost_at=None, gate_z=False):
    """float64 scan with per-row B / C (b, dim, N, L) and delta' given: -> (out, out_z, [h after every token])."""
    b, dim, L = u.shape
    h = torch.zeros(b, dim, A.shape[1], dtype=torch.float64)
    ys, hs = [], []
    for t in range(L):
        if carry_lost_at is not None and t == carry_lost_at:
            h = torch.zeros_like(h)
        if not (drop_last and t == L - 1):
            h = torch.exp(dl[:, :, t, None] * A) * h + (dl[:, :, t] * u[:, :, t])[..., None] * Bx[..., t]
        ys.append((h * Cx[..., t]).sum(-1) + D * u[:, :, t])
        hs.append(h)
    y = torch.stack(ys, -1)
    out_z = None if z is None else y * (z if gate_z else F.silu(z))
    return y, out_z, hs


def _mutant_inputs(b, dim, L, N, T, seed):
    g = torch.Generator().manual_seed(seed)
    q = lambda t: t.to(T).double()
    u, delta, z = q(torch.randn(b, dim, L, generator=g)), q(0.5 * torch.rand(b, dim, L, generator=g)), q(torch.randn(b, dim, L, generator=g))
    A = (-0.5 * torch.rand(dim, N, generator=g)).double()
    Bx = q(torch.randn(b, 1, N, L, generator=g)).expand(b, dim, N, L).clone()
    Cx = q(torch.randn(b, 1, N, L, generator=g)).expand(b, dim, N, L).clone()
    D, bias = torch.randn(dim, generator=g).double(), (0.5 * torch.rand(dim, generator=g)).double()
    return u, delta, z, A, Bx, Cx, D, bias


@pytest.mark.parametrize("out", ["f32", "bf16", "f16"])
def test_criteria_reject_subtly_wrong_results(out):
    """test_scan_kernel_parity's comparisons on float64 "mutants" of a correct result, rounded as the kernel stores it
    (2 x 64 rows x 300 tokens, d_state 2: two 32-row items, two checkpoint chunks): the last token of a row not scanned,
    the carry lost at the 256-token chunk boundary, D u missing on one row of a 32-row item, delta_bias added twice, the
    gate applied as z instead of silu(z), one segment's dB partial missing, the ddelta group fold without its last row,
    fp32 results rounded to bf16 / fp16, the x checkpoints one chunk late (three chunks), and one store one element past a
    row end; the correct results pass."""
    T = {"f32": F32, "bf16": BF16, "f16": F16}[out]
    b, dim, L, N = 2, 64, 300, 2
    u, delta, z, A, Bx, Cx, D, bias = _mutant_inputs(b, dim, L, N, T, 11)
    dl = F.softplus(delta + bias[:, None])
    q = lambda v: v.to(T)
    cmp = lambda got, ref, what: cmp_auto(got, ref, what, f32_scale=long_row_scale(L))
    y, out_z, hs = _scan64(u, dl, A, Bx, Cx, D, z)
    cmp(q(y), y, "correct out")
    cmp(q(out_z), out_z, "correct out_z")
    D1 = D.clone()
    D1[37] = 0
    mutants = {"last token not scanned": _scan64(u, dl, A, Bx, Cx, D, drop_last=True)[0],
               "carry lost at 256": _scan64(u, dl, A, Bx, Cx, D, carry_lost_at=256)[0],
               "D u missing on row 37": _scan64(u, dl, A, Bx, Cx, D1)[0],
               "delta_bias twice": _scan64(u, F.softplus(delta + 2 * bias[:, None]), A, Bx, Cx, D)[0]}
    for what, bad in mutants.items():
        with pytest.raises(AssertionError):
            cmp(q(bad), y, what)
    with pytest.raises(AssertionError):
        cmp(q(_scan64(u, dl, A, Bx, Cx, D, z, gate_z=True)[1]), out_z, "gate z")

    # backward: dB of a group is the sum over its rows (per-segment partials), ddelta of a delta group the sum over its rows
    Bl, dll = Bx.clone().requires_grad_(), dl.clone().requires_grad_()
    dout = q(torch.randn(b, dim, L, generator=torch.Generator().manual_seed(12))).double()
    (_scan64(u, dll, A, Bl, Cx, D)[0] * dout).sum().backward()
    dB_rows, dd_rows = Bl.grad, dll.grad
    dB = dB_rows.sum(1)
    cmp(q(dB), dB, "correct dB")
    with pytest.raises(AssertionError):
        cmp(q(dB - dB_rows[:, 32:48].sum(1)), dB, "one segment's dB partial missing")
    dd = dd_rows.view(b, dim // 4, 4, L).sum(2)
    cmp(q(dd), dd, "correct ddelta (groups of 4 rows)")
    with pytest.raises(AssertionError):
        cmp(q(dd_rows.view(b, dim // 4, 4, L)[:, :, :3].sum(2)), dd, "ddelta fold without its last row")
    if T == F32:
        for lowp in (BF16, F16):
            with pytest.raises(AssertionError):
                cmp_f32(y.to(lowp).float(), y, f"fp32 out rounded to {lowp}")
            with pytest.raises(AssertionError):
                cmp_f32(dB.to(lowp).float(), dB, f"fp32 dB rounded to {lowp}")

    # x checkpoints of three chunks (L = 600), one chunk late
    u3, delta3, _, A3, Bx3, _, _, bias3 = _mutant_inputs(1, 32, 600, N, T, 13)
    Bg = Bx3[:, :1]
    xr = x_ref(u3, delta3, A3, Bg, bias3, True)
    _cmp_x(xr.float(), xr, "correct", long_row_scale(600))
    late = torch.cat([xr[:, :, 1:], xr[:, :, -1:]], 2)
    with pytest.raises(AssertionError):
        _cmp_x(late.float(), xr, "x one chunk late", long_row_scale(600))
    # and the checkpoints agree with an independent recurrence (the h of _scan64 at the chunk ends)
    hs3 = _scan64(u3, F.softplus(delta3 + bias3[:, None]), A3, Bx3, Bx3, torch.zeros(32, dtype=torch.float64))[2]
    assert torch.allclose(xr[:, :, 1, 1::2], hs3[511], rtol=1e-12, atol=1e-12)
    assert torch.allclose(xr[:, :, 2, 1::2], hs3[599], rtol=1e-12, atol=1e-12)

    # one store one element past a row end: into the guard band (dense) and into the pad of a padded pitch
    for pad in (0, 3):
        o = Buf((b, dim, L), T, pad, dev="cpu").set(q(y))
        o.untouched(f"correct (pad {pad})")
        if pad:
            o.buf[Buf.GUARD + 5 * o.pitch + L] = 0                       # row 5, first pad element
        else:
            o.buf[Buf.GUARD + b * dim * L] = 0                           # the element after the last row
        with pytest.raises(AssertionError):
            o.untouched(f"stray store (pad {pad})")


def test_criteria_reject_dA_missing_one_batch():
    """dA summed over a batch of 40 (the finalize's lanes stride over batches 0-31 and 32-39) without batch 33 fails the
    fp32 criterion; the full sum passes."""
    b, dim, L, N = 40, 4, 24, 2
    u, delta, _, A, Bx, Cx, D, bias = _mutant_inputs(b, dim, L, N, BF16, 5)
    Al = A.clone().requires_grad_()
    dout = torch.randn(b, dim, L, generator=torch.Generator().manual_seed(6)).bfloat16().double()
    y = _scan64(u, F.softplus(delta + bias[:, None]), Al, Bx, Cx, D)[0]
    parts = [torch.autograd.grad((y[i] * dout[i]).sum(), Al, retain_graph=True)[0] for i in range(b)]
    dA = sum(parts)
    cmp_f32(dA.float(), dA, "correct dA")
    with pytest.raises(AssertionError):
        cmp_f32((dA - parts[33]).float(), dA, "dA without batch 33")
