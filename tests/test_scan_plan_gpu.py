"""Which kernel family the selective-scan planner (csrc/scan_api.cu) picks, seen through the kernels a call launches.

The other scan tests see the family only through launch counts and block states, which cannot tell the resident-row,
streaming and warp-scan forwards apart, nor the resident-row and column-walk backwards when no block states are passed.
Here torch.profiler (CUPTI) lists the kernels libmia_scan.so launches for a forward, a backward without block states and,
when the forward wrote them, a backward on them.  The table has a row for every rung of both ladders
(forward: column-walk, chunk-parallel, resident-row, streaming, d_state 8 / 16 row-serial, warp-scan; backward: d_state 16
row-serial, column-walk, resident-row, warp-scan, deterministic warp-scan) and for the usual reasons a rung declines.
Item counts stay far from the gates that compare them with the SM count (4 items per SM, 12 resident warps per SM), so
the expectations hold on any H100.  Values are not checked here; the parity tests do that.
"""
import re

import pytest
import torch

from tests.kernel_trace import launched, retry, targs

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32

# (kernel-name prefix, family); the column-walk kernels' 4th template argument is g (rows per tensor-map row)
FWD_KERNELS = [("ss_fwd_cw_kernel<", "cw"), ("ss_fwd_chunk_kernel<", "chunks"), ("ss_fwd_chunk_combine_kernel<", "chunks"),
               ("ss_fwd_rows_kernel<", "rows"), ("ss_fwd_stream_kernel<", "stream"), ("ss_fwd_rowsn_kernel<", "rowsn"),
               ("ss_fwd_fast_kernel<", "fast"), ("ss_fwd_kernel<", "warp")]
BWD_KERNELS = [("ss_bwd_cw_kernel<", "cw"), ("ss_bwd_rowsn_kernel<", "rowsn"), ("ss_bwd_rows_kernel<", "rows"),
               ("ss_bwd_fast_kernel<", "fast"), ("ss_bwd_fastn_kernel<", "fastn"), ("ss_bwd_kernel<", "warp")]
SCAN_KERNEL = re.compile(r"\bss_(fwd|bwd|finalize)_\w*kernel<")


def _family(names, table):
    """The one family all scan kernels in ``names`` belong to: 'cw<g>', '<family>' or '<family>-det' (kDet instances)."""
    fams = set()
    for n in names:
        prefix, fam = next(((p, f) for p, f in table if p in n), (None, None))
        assert prefix is not None, f"unexpected scan kernel {n!r}"
        args = targs(n, prefix)
        if fam == "cw":
            fam += args[3]
        elif fam in ("fastn", "warp") and prefix.startswith("ss_bwd") and args[-1] == "true":
            fam += "-det"
        fams.add(fam)
    assert len(fams) == 1, f"kernels of several families: {names}"
    return fams.pop()


def _scan_kernels(fn):
    return launched(fn, SCAN_KERNEL)


def _inputs(batch, dim, L, N=1, G=1, ddim=None, dtype=BF16, z=False, layout=None, seed=0):
    ddim = ddim or dim
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    if layout == "u_off8":          # dense rows whose storage starts 8 bytes past a 16-byte boundary
        off = 8 // torch.empty((), dtype=dtype).element_size()
        u = rn(off + batch * dim * L).to(dtype)[off:].view(batch, dim, L)
    elif layout == "u_bstride":     # every other (dim, L) slab of a (batch, 2 dim, L) tensor
        u = rn(batch, 2 * dim, L).to(dtype)[:, :dim]
    else:
        u = rn(batch, dim, L).to(dtype)
    if layout == "bc_odd":          # B and C one element past a 4-byte boundary
        B = rn(1 + batch * G * N * L).to(dtype)[1:].view(batch, G, N, L)
        C = rn(1 + batch * G * N * L).to(dtype)[1:].view(batch, G, N, L)
    else:
        B, C = rn(batch, G, N, L).to(dtype), rn(batch, G, N, L).to(dtype)
    return dict(u=u, delta=(0.5 * torch.rand(batch, ddim, L, generator=g, device="cuda")).to(dtype),
                A=-0.5 * torch.rand(dim, N, generator=g, device="cuda"), B=B, C=C, D=rn(dim),
                z=rn(batch, dim, L).to(dtype) if z else None, delta_bias=0.5 * torch.rand(ddim, generator=g, device="cuda"),
                dout=rn(batch, dim, L).to(dtype))


# id: (shape and layout, out_float, deterministic, forward family, backward without block states, backward on them or None
# when the forward writes none)
PLANS = {
    # short rows, column-walk: L = 196 bf16 rows are 392 bytes, so 4 (rows_per_group % 128 == 0) or 2 rows per tensor-map row
    "cw_g4": (dict(batch=2, dim=256, L=196), False, False, "cw4", "rows", "cw4"),
    "cw_g4_o32": (dict(batch=2, dim=256, L=196), True, False, "cw4", "rows", "cw4"),
    "cw_g4_f16": (dict(batch=2, dim=256, L=196, dtype=F16), False, False, "cw4", "rows", "cw4"),
    "cw_g2": (dict(batch=2, dim=192, L=196), False, False, "cw2", "rows", "cw2"),
    # fp32 rows of 196 tokens: fewer than 3 resident-row backward CTAs fit an SM
    "cw_f32": (dict(batch=2, dim=64, L=196, dtype=F32), False, False, "cw1", "fast", "cw1"),
    # 96 rows per group at L = 196: no g makes a legal tensor-map row of whole 32-row items
    "rpg96": (dict(batch=2, dim=96, L=196), False, False, "rows", "rows", None),
    # B / C at an odd element: the column-walk backward's 4-byte B / C copies decline, the forward does not
    "cw_bc_odd": (dict(batch=2, dim=256, L=196, layout="bc_odd"), False, False, "cw4", "rows", "rows"),
    "u_off8": (dict(batch=2, dim=64, L=196, layout="u_off8"), False, False, "stream", "fast", None),
    "u_bstride": (dict(batch=2, dim=64, L=196, layout="u_bstride"), False, False, "fast", "fast", None),
    # long rows: few 32-row items -> chunk-parallel forward, resident-row backward; many -> column-walk both ways
    "few_long": (dict(batch=1, dim=64, L=1024), False, False, "chunks", "rows", None),
    "many_long": (dict(batch=8, dim=4096, L=1024), False, False, "cw1", "fast", "cw1"),
    "odd_L": (dict(batch=2, dim=64, L=195), False, False, "fast", "fast", None),
    "odd_L_short": (dict(batch=2, dim=64, L=101), False, False, "warp", "warp", None),
    "z_n1": (dict(batch=2, dim=64, L=196, z=True), False, False, "warp", "warp", None),
    "delta_groups": (dict(batch=2, dim=64, L=196, ddim=16), False, False, "warp", "warp", None),
    "n4_short": (dict(batch=2, dim=64, L=100, N=4), False, False, "warp", "warp", None),
    "n8": (dict(batch=2, dim=64, L=196, N=8), False, False, "rowsn", "fastn", None),
    "n8_z": (dict(batch=2, dim=64, L=196, N=8, z=True), False, False, "rowsn", "fastn", None),
    "n16": (dict(batch=2, dim=64, L=196, N=16), False, False, "rowsn", "rowsn", None),
    "n16_z": (dict(batch=2, dim=64, L=196, N=16, z=True), False, False, "rowsn", "rowsn", None),
    "n16_long": (dict(batch=2, dim=64, L=400, N=16), False, False, "warp", "fastn", None),
    "det_n4": (dict(batch=2, dim=64, L=196, N=4), False, True, "warp", "fastn-det", None),
    "det_n4_short": (dict(batch=2, dim=64, L=100, N=4), False, True, "warp", "warp-det", None),
    "det_n16": (dict(batch=2, dim=64, L=196, N=16), False, True, "rowsn", "rowsn", None),
}


def run_plan(shape, out_float, det):
    """Forward, backward and (when the forward wrote block states) backward on them under the profiler.
    -> (forward kernels, backward kernels, backward-on-block-states kernels or None)."""
    from medical_image_analysis_b200 import scan_bwd, scan_fwd
    t = _inputs(**shape)
    (out, x, _, hblk), kf = _scan_kernels(lambda: scan_fwd(t["u"], t["delta"], t["A"], t["B"], t["C"], t["D"], t["z"],
                                                            t["delta_bias"], True, out_float, want_block_states=True))
    dout = t["dout"].float() if out_float else t["dout"]
    saved = out if t["z"] is not None else None
    bwd = lambda hb: scan_bwd(t["u"], t["delta"], t["A"], t["B"], t["C"], t["D"], t["z"], t["delta_bias"], dout, x, saved, True,
                              hblk=hb)
    was_det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        _, kb = _scan_kernels(lambda: bwd(None))
        kh = _scan_kernels(lambda: bwd(hblk))[1] if hblk is not None else None
    finally:
        torch.use_deterministic_algorithms(was_det)
    return kf, kb, kh


@pytest.mark.parametrize("case", list(PLANS))
def test_scan_plan(case):
    shape, out_float, det, want_fwd, want_bwd, want_hblk = PLANS[case]
    kf, kb, kh = retry(lambda: run_plan(shape, out_float, det),
                       lambda r: len(r[0]) == (3 if "ss_fwd_chunk_kernel<" in " ".join(r[0]) else 1)
                       and all(k is None or len(k) == 2 for k in r[1:]))
    assert _family(kf, FWD_KERNELS) == want_fwd, kf
    assert len(kf) == (3 if want_fwd == "chunks" else 1), kf
    for names, want in ((kb, want_bwd), (kh, want_hblk)):
        if want is None:
            assert names is None, f"the forward wrote block states: {kf}"
            continue
        assert names is not None, f"the forward wrote no block states: {kf}"
        scan = [n for n in names if "ss_finalize_kernel<" not in n]
        assert len(scan) == 1 and len(names) == 2, names
        assert _family(scan, BWD_KERNELS) == want, names
