"""GPU parity of the selective scan at the value ranges trained models use, and with the operand layouts the models
hand it.  Same comparison as tests/test_scan_gpu.py (CUDA path through the C ABI against the fp64 C oracle, criteria of
tests/parity.py unchanged); what is new is the input generator.

Every other scan test draws from the reference's generators (A in (-0.5, 0], softplus argument in [0, 1)).  SS2D and the
ARM Mamba mixers initialise A = -(1 .. d_state) and dt_proj.bias = softplus^-1(dt), dt in [1e-3, 1e-1]: the softplus
argument sits in about [-8, -1], delta' = softplus(.) in [3e-4, 0.3], and exp(delta' A) spans 0.999 .. 0.008 per token.
There softplus(x) ~ e^x and its derivative ~ e^x are SMALL numbers whose RELATIVE error enters du, ddelta and y token by
token; an evaluation that is accurate to an ulp of 1.0 (lg2(1 + e), 1 - 2^-m) is not accurate enough.

Calibration (NVIDIA H100 80GB HBM3, 700 W; MIA_PARITY_LOG), worst err / tol per tensor class over this file, unwidened
criteria.  With softplus as lg2(1 + e) and the sigmoid as 1 - 2^-m everywhere (lower bounds: a test stops at its first
failure): model regime fp32 ddelta 5.06, last_state 1.24; 2-byte inputs last_state 1.40, dA 1.36; edges regime fp32 ddelta
22.8, ddelta_bias 2.21; the two backward families against each other, ddelta 4.13 - 30 of the 152 tests fail.  With
softplus_l2 / sigmoid_of_softplus_l2 (scan_common.cuh):
  model, fp32 tensors of fp32 runs:  out 0.10  last_state 0.14  du 0.12  ddelta 0.90 (the 5.6 M-element two-chunk shape)
                                     dB/dC 0.15  dz 0.09  dA/dD/ddelta_bias 0.22
  model, 2-byte inputs:              stored tensors 0.83 - 0.97 of an ulp; fp32 tensors last_state 0.20  dA/dD/ddelta_bias 0.29
  edges, fp32 runs:                  out 0.40  last_state 0.22  du 0.46  ddelta 0.43  dB/dC 0.35  dz 0.33  dA/dD/ddelta_bias 0.14
  edges, 2-byte inputs:              stored tensors 0.88 - 0.96 of an ulp; fp32 tensors last_state 0.26  dA/dD/ddelta_bias 0.22
  backward families against each other (fp32): du 0.04  ddelta 0.17  dB/dC 0.04  dA/dD/ddelta_bias 0.09
  ARM mixer views: fp32 all <= 0.26; bf16 stored tensors <= 0.97 of an ulp.  Unaligned operands / B, C at odd offsets: <= 0.97.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
DTYPES = [(F32, False), (BF16, False), (BF16, True), (F16, False)]
DTYPE_IDS = {(F32, False): "f32", (BF16, False): "bf16", (BF16, True): "bf16o32", (F16, False): "f16"}

# softplus arguments of the `edges` regime: deep in the e^x tail, around 0, on both sides of the x > 20 branch (20 is
# exactly representable in bf16 / fp16, so `x <= 20` itself is exercised), beyond the 2^120 clamp of the kernels
EDGE_ARGS = (-30.0, -15.0, -8.0, -1.0, 0.0, 5.0, 19.5, 20.0, 20.5, 40.0, 88.0)


def range_inputs(regime, seed, batch, dim, L, N, G, ddim, has_D=True, has_z=False, has_bias=True, softplus=True, dtype=F32):
    """CPU inputs (the dict of tests/test_scan_gpu.py::_inputs) in one of two regimes.

    ``model``: what SS2D / the ARM mixers run.  A = -(1 .. N) times a per-row factor in [0.5, 2]; with a bias,
    bias = dt + log(-expm1(-dt)), dt = exp(U(log 1e-3, log 1e-1)) and delta = 0.5 randn; without one, delta itself is
    uniform in [-8, -1].  softplus is always on.
    ``edges``: one launch covers rows with A = 0 (no decay), rows with A = -16 (the chunk product underflows) and the
    ordinary rows; with softplus the arguments are drawn from EDGE_ARGS (plus the bias, if any, in [0, 0.5)) and u, dout
    are randn / 16; without it
    delta has both signs (a > 1 on some tokens) at a magnitude that keeps |delta A| L below 60."""
    g = torch.Generator().manual_seed(seed)
    B = torch.randn(batch, G, N, L, generator=g).to(dtype)
    C = torch.randn(batch, G, N, L, generator=g).to(dtype)
    D = torch.randn(dim, generator=g) if has_D else None
    z = torch.randn(batch, dim, L, generator=g).to(dtype) if has_z else None
    u = torch.randn(batch, dim, L, generator=g).to(dtype)
    dout = torch.randn(batch, dim, L, generator=g).to(dtype)
    if regime == "model":
        assert softplus
        A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(dim, 1) * (0.5 + 1.5 * torch.rand(dim, 1, generator=g))
        if has_bias:
            dt = torch.exp(torch.rand(ddim, generator=g) * (math.log(1e-1) - math.log(1e-3)) + math.log(1e-3))
            bias = dt + torch.log(-torch.expm1(-dt))
            delta = 0.5 * torch.randn(batch, ddim, L, generator=g)
        else:
            bias = None
            delta = -8.0 + 7.0 * torch.rand(batch, ddim, L, generator=g)
    elif regime == "edges":
        bias = 0.5 * torch.rand(ddim, generator=g) if has_bias else None
        if softplus:
            A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(dim, 1) * (0.5 + 1.5 * torch.rand(dim, 1, generator=g))
            pick = torch.randint(0, len(EDGE_ARGS), (batch, ddim, L), generator=g)
            delta = torch.tensor(EDGE_ARGS)[pick]
            u, dout = u / 16, dout / 16          # delta' reaches 88 and A = 0 rows never forget: keeps fp16 results in range
        else:
            A = -0.5 * torch.rand(dim, N, generator=g)
            delta = (torch.rand(batch, ddim, L, generator=g) - 0.5) * min(1.0, 200.0 / L)
        A[0::4] = 0.0
        A[1::4] = -16.0 if softplus else -0.5
    else:
        raise ValueError(regime)
    return dict(u=u, delta=delta.to(dtype), A=A, B=B, C=C, D=D, z=z, delta_bias=bias, dout=dout)


def to_gpu(cpu):
    return {k: (None if v is None else v.cuda()) for k, v in cpu.items()}


def _check(cpu, gpu, softplus, out_float, tag, fs=1.0, fwd=None, bwd_launches=None):
    """scan_fwd / scan_bwd on ``gpu`` (same values as ``cpu``, any layout) against the fp64 C oracle on ``cpu``, criteria of
    tests/test_scan_gpu.py::_run_case.  ``fwd``: the forward family the shape was put in the table for, asserted where the
    release library shows it: "cw" = the column-walk kernel (it alone fills the block states), "chunks" = the three
    launches of the chunk-parallel forward, "one" = one launch and no block states (resident-row, streaming, d_state 8 / 16
    row-serial or warp-scan), "not-cw" = only that the planner declined the TMA path.  ``bwd_launches``: 2 = kernel +
    finalize, 4 = the warp-scan d_state > 1 backward (two memsets of its red.add accumulators in front).
    Returns (hblk, gradients without block states, gradients with them or None)."""
    from medical_image_analysis_b200 import _lib, scan_bwd, scan_fwd
    from oracle import ss_ref_c
    from tests.parity import cmp_auto
    has_z = cpu["z"] is not None
    n0 = _lib.launch_count()
    out, x, out_z, hblk = scan_fwd(gpu["u"], gpu["delta"], gpu["A"], gpu["B"], gpu["C"], gpu["D"], gpu["z"], gpu["delta_bias"],
                                   softplus, out_float, want_block_states=True)
    n_fwd = _lib.launch_count() - n0
    if fwd == "cw":
        assert hblk is not None and n_fwd == 1, f"{tag}: expected the column-walk forward (hblk {hblk is not None}, {n_fwd} launches)"
    elif fwd == "chunks":
        assert hblk is None and n_fwd == 3, f"{tag}: expected the chunk-parallel forward (hblk {hblk is not None}, {n_fwd} launches)"
    elif fwd == "one":
        assert hblk is None and n_fwd == 1, f"{tag}: expected a one-launch forward without block states (hblk {hblk is not None}, {n_fwd} launches)"
    elif fwd == "not-cw":
        assert hblk is None, f"{tag}: the column-walk forward took an operand it cannot address"
    r_out, r_out_z, r_last = ss_ref_c.fwd(cpu["u"], cpu["delta"], cpu["A"], cpu["B"], cpu["C"], cpu["D"], cpu["z"],
                                          cpu["delta_bias"], softplus)
    lowp = cpu["u"].dtype != F32
    assert out.dtype == (F32 if out_float else cpu["u"].dtype)
    cmp_auto(out, r_out, tag + " out", f32_scale=fs)
    if has_z:
        cmp_auto(out_z, r_out_z, tag + " out_z", f32_scale=fs)
    cmp_auto(x[:, :, -1, 1::2], r_last, tag + " last_state", f32_scale=fs)

    dout = gpu["dout"].float() if out_float else gpu["dout"]
    ref = ss_ref_c.bwd(cpu["u"], cpu["delta"], cpu["A"], cpu["B"], cpu["C"], cpu["D"], cpu["z"], cpu["delta_bias"],
                       cpu["dout"], softplus)
    dz_ulp = 2.0 if (has_z and lowp and not out_float) else 1.0          # see _run_case
    names = ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz")
    results = []
    for path, hb in (("", None),) + ((("[hblk]", hblk),) if hblk is not None else ()):
        n0 = _lib.launch_count()
        grads = scan_bwd(gpu["u"], gpu["delta"], gpu["A"], gpu["B"], gpu["C"], gpu["D"], gpu["z"], gpu["delta_bias"], dout, x,
                         out if has_z else None, softplus, hblk=hb)
        if bwd_launches is not None:
            assert _lib.launch_count() - n0 == bwd_launches, f"{tag}{path}: {_lib.launch_count() - n0} backward launches, expected {bwd_launches}"
        for name, got in zip(names, grads):
            if got is not None:
                cmp_auto(got, ref[name], f"{tag}{path} {name}", n_ulp=dz_ulp if name == "dz" else 1.0, f32_scale=fs)
        results.append(grads)
    return hblk, results[0], (results[1] if len(results) > 1 else None)


def _run(regime, shape, has_z, has_bias, softplus, dtype, out_float, seed, fwd=None, bwd_launches=None):
    from tests.parity import long_row_scale
    batch, dim, L, N, G, ddim = shape
    tag = (f"[{regime} b{batch} d{dim} L{L} N{N} G{G} dd{ddim} z{int(has_z)} bias{int(has_bias)} sp{int(softplus)} "
           f"{DTYPE_IDS[(dtype, out_float)]}]")
    cpu = range_inputs(regime, seed, batch, dim, L, N, G, ddim, True, has_z, has_bias, softplus, dtype)
    return _check(cpu, to_gpu(cpu), softplus, out_float, tag, long_row_scale(L), fwd, bwd_launches)


# One or two shapes per kernel family and direction (DESIGN.md section 3; planner conditions in scan_api.cu), with the family
# the shape is here for.  (batch, dim, L, N, G, ddim), z gate, (dtype, out_float) list, forward family, backward launches.
LOWP = [d for d in DTYPES if d[0] != F32]
FAMILIES = {
    # d_state 1.  32 rows per group and L = 196: 2-byte rows are not tensor-map rows (392 B) and 32 is not a multiple of
    # 64 -> resident-row forward and backward; the same shape in fp32 is a column-walk shape (g = 1)
    "rows": ((2, 64, 196, 1, 2, 64), False, LOWP, "one", 2),
    "rows_f32_cw_g1": ((2, 64, 196, 1, 2, 64), False, [(F32, False)], "cw", 2),
    "cw_g2": ((2, 128, 196, 1, 2, 128), False, DTYPES, "cw", 2),             # 64 rows per group: two rows per tensor-map row
    "cw_g4": ((2, 256, 196, 1, 2, 256), False, LOWP, "cw", 2),               # 128 rows per group: four
    "cw_short": ((3, 64, 12, 1, 1, 64), False, DTYPES, "cw", 2),             # rows shorter than one 16-column group
    # rows of two checkpoint chunks, enough 32-row items (608 >= 4 x 132) for the column-walk pair
    "cw_two_chunks": ((19, 1024, 288, 1, 1, 1024), False, [(F32, False), (BF16, False)], "cw", 2),
    # long rows, few of them: chunk-parallel forward (A / B / C passes), resident-row backward over chunks
    "chunks_b1": ((1, 256, 6400, 1, 2, 256), False, [(F32, False), (BF16, False)], "chunks", 2),
    "chunks_b2": ((2, 256, 6400, 1, 2, 256), False, [(BF16, True), (F16, False)], "chunks", 2),
    "chunks_short": ((1, 64, 512, 1, 2, 64), False, DTYPES, "chunks", 2),
    # 520-byte rows: neither tensor-map rows nor 16-byte row pieces -> streaming forward, warp-scan backward
    "stream": ((2, 32, 260, 1, 1, 32), False, LOWP, "one", 2),
    # warp-scan kernels: odd L and 11 rows per group; delta groups at d_state 4; z gate at d_state 1; d_state 4 long rows
    "ws_odd": ((2, 33, 197, 1, 3, 33), False, DTYPES, "one", 2),
    "ws_dgroups": ((2, 8, 37, 4, 2, 2), False, DTYPES, "one", 4),
    "ws_z_n1": ((2, 64, 196, 1, 2, 64), True, DTYPES, "one", 2),
    "ws_n4_long": ((1, 5, 600, 4, 1, 5), False, DTYPES, "one", 4),
    # d_state 16 / 8 row-serial forward; deterministic d_state 16 backward (2 launches), warp-scan backward at d_state 8 and
    # for L > 256 (4 launches)
    "rowsn16": ((2, 64, 196, 16, 2, 64), False, DTYPES, "one", 2),
    "rowsn16_z_odd": ((2, 64, 197, 16, 1, 64), True, DTYPES, "one", 2),
    "rowsn8": ((2, 96, 100, 8, 3, 96), False, DTYPES, "one", 4),
    "n16_long": ((1, 32, 300, 16, 1, 32), False, DTYPES, "one", 4),
    "n16_z_long": ((1, 32, 300, 16, 1, 32), True, [(F32, False), (BF16, False)], "one", 4),
}
CASES = [pytest.param(name, dt, of, id=f"{name}-{DTYPE_IDS[(dt, of)]}") for name, row in FAMILIES.items() for dt, of in row[2]]


@pytest.mark.parametrize("name,dtype,out_float", CASES)
def test_scan_parity_model_regime(name, dtype, out_float):
    """Every kernel family at the models' initialisation (softplus argument in [-8, -1], A = -(1 .. d_state)), with the bias
    and without (delta itself in [-8, -1]; not for the 5.6 M-element two-chunk column-walk shape, whose oracle run dominates)."""
    shape, has_z, _, fwd, nb = FAMILIES[name]
    _run("model", shape, has_z, True, True, dtype, out_float, 41, fwd, nb)
    if name != "cw_two_chunks":
        _run("model", shape, has_z, False, True, dtype, out_float, 42, fwd, nb)


@pytest.mark.parametrize("name,dtype,out_float", [c for c in CASES if c.values[0] != "cw_two_chunks"])
def test_scan_parity_edges_regime(name, dtype, out_float):
    """A = 0 and A = -16 rows in one launch; softplus arguments from EDGE_ARGS (with a bias: jittered by [0, 0.5); without:
    exactly those values, so x == 20 takes the log1p side of the branch and 20.5 / 40 / 88 the identity side, the last
    two past the kernels' 2^120 clamp); and without softplus a delta of both signs (growth on some tokens)."""
    shape, has_z, _, fwd, nb = FAMILIES[name]
    _run("edges", shape, has_z, True, True, dtype, out_float, 43, fwd, nb)
    _run("edges", shape, has_z, False, True, dtype, out_float, 44, fwd, nb)
    _run("edges", shape, has_z, False, False, dtype, out_float, 45, fwd, nb)


AGREE = [(2, 64, 196, 1, 2, 64), (2, 128, 196, 1, 2, 128), (3, 64, 12, 1, 1, 64),
         (9, 2048, 512, 1, 1, 2048)]      # 576 items of 32 rows: enough for the column-walk pair on two-chunk rows


@pytest.mark.parametrize("shape", AGREE, ids=lambda s: f"b{s[0]}d{s[1]}L{s[2]}G{s[4]}")
@pytest.mark.parametrize("has_bias", [True, False], ids=["bias", "nobias"])
def test_backward_families_agree_model_regime(shape, has_bias):
    """fp32, d_state 1: the backward on the forward's block states (column-walk kernel: sigmoid rebuilt from the softplus
    value) against the backward without them (resident-row / warp-scan kernels: sigmoid from e / (1 + e)), compared WITH
    EACH OTHER at the fp32 criterion - independent of the oracle."""
    from medical_image_analysis_b200 import scan_bwd, scan_fwd
    from tests.parity import cmp_f32, long_row_scale
    batch, dim, L, N, G, ddim = shape
    g = to_gpu(range_inputs("model", 46, batch, dim, L, N, G, ddim, True, False, has_bias, True, F32))
    out, x, _, hblk = scan_fwd(g["u"], g["delta"], g["A"], g["B"], g["C"], g["D"], None, g["delta_bias"], True, False, want_block_states=True)
    assert hblk is not None
    a = scan_bwd(g["u"], g["delta"], g["A"], g["B"], g["C"], g["D"], None, g["delta_bias"], g["dout"], x, None, True, hblk=hblk)
    b = scan_bwd(g["u"], g["delta"], g["A"], g["B"], g["C"], g["D"], None, g["delta_bias"], g["dout"], x, None, True, hblk=None)
    fs = long_row_scale(L)
    for nm, ta, tb in zip(("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias"), a, b):
        if ta is not None:
            cmp_f32(ta, tb, f"[agree b{batch} d{dim} L{L} bias{int(has_bias)}] {nm}", rtol=1e-5 * fs, atol_rms=2e-5 * fs)


# ------------------------------------------------------------------------------------------------------------------------
# Layouts.  Only the last dimension must be contiguous; the models hand the scan views.  (Gradients are always written to
# tensors scan_bwd allocates itself, so strided OUTPUTS are not reachable and not covered here.)

def _in_flat(t, off_elems):
    """The values of ``t`` in a view that starts ``off_elems`` elements into a fresh (512-byte aligned) flat buffer."""
    flat = torch.zeros(t.numel() + off_elems + 8, dtype=t.dtype, device=t.device)
    v = flat[off_elems:off_elems + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _batch_strided(t):
    """The values of ``t`` (batch, rows, L) as rows [0, rows) of a buffer with twice the rows: batch stride 2 rows L."""
    big = torch.zeros(t.shape[0], 2 * t.shape[1], t.shape[2], dtype=t.dtype, device=t.device)
    big[:, :t.shape[1]] = t
    return big[:, :t.shape[1]]


@pytest.mark.parametrize("L", [197, 196])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
def test_scan_arm_mixer_views(L, dtype):
    """The ARM mixer's call: u, z = xz.chunk(2, dim=1) (batch stride 2 d L), B / C = torch.split views of an x_dbl buffer
    (batch, K, R + 2 N, L), delta with padded rows, dout a row slice of a wider buffer, A transposed-contiguous; d = 768,
    d_state 16, z gate, model regime.  Forward and backward (all gradients) against the oracle on the contiguous values."""
    batch, dim, N, R = 2, 768, 16, 48
    cpu = range_inputs("model", 47, batch, dim, L, N, 1, dim, True, True, True, True, dtype)
    g = to_gpu(cpu)
    xz = torch.cat([g["u"], g["z"]], dim=1)
    u, z = xz.chunk(2, dim=1)
    x_dbl = torch.zeros(batch, 1, R + 2 * N, L, dtype=dtype, device="cuda")
    x_dbl[:, :, R:R + N] = g["B"]
    x_dbl[:, :, R + N:] = g["C"]
    _, Bv, Cv = torch.split(x_dbl, [R, N, N], dim=2)
    dpad = torch.zeros(batch, dim, L + 11, dtype=dtype, device="cuda")
    dpad[:, :, 3:3 + L] = g["delta"]
    dwide = torch.zeros(batch, dim + 4, L, dtype=dtype, device="cuda")
    dwide[:, 2:2 + dim] = g["dout"]
    views = dict(g, u=u, z=z, B=Bv, C=Cv, delta=dpad[:, :, 3:3 + L], dout=dwide[:, 2:2 + dim], A=g["A"].t().contiguous().t())
    for k in ("u", "z", "B", "C", "delta", "dout", "A"):
        assert not views[k].is_contiguous() and torch.equal(views[k], g[k]), k
    _check(cpu, views, True, False, f"[arm views L{L} {str(dtype)[6:]}]", fwd="one")


@pytest.mark.parametrize("kind", ["batch_strided", "off2", "off4", "off8"])
@pytest.mark.parametrize("which", ["u", "delta", "dout"])
def test_scan_column_walk_shape_with_unaligned_operand(which, kind):
    """A column-walk shape (2 x 128 rows of 196 bf16 tokens, d_state 1) with one of u / delta / dout batch-strided or starting
    2 / 4 / 8 bytes off a 16-byte boundary.  The TMA kernels cannot address that: u or delta -> the forward planner must
    decline (no block states) and the result must still be right; dout -> the forward is the column-walk one and the
    backward handed its block states must fall back to a kernel that can read the view."""
    cpu = range_inputs("model", 48, 2, 128, 196, 1, 2, 128, True, False, True, True, BF16)
    g = to_gpu(cpu)
    views = dict(g)
    views[which] = _batch_strided(g[which]) if kind == "batch_strided" else _in_flat(g[which], int(kind[3:]) // 2)
    assert torch.equal(views[which], g[which])
    if kind == "batch_strided":
        assert views[which].stride(0) == 2 * 128 * 196
    else:
        assert views[which].data_ptr() % 16 == int(kind[3:])
    _check(cpu, views, True, False, f"[cw shape, {which} {kind}]", fwd="cw" if which == "dout" else "not-cw", bwd_launches=2)


BC_ODD = {  # family: shape, forward family.  All bf16; B and C start one element (2 bytes) into their buffers.
    "cw": ((2, 128, 196, 1, 2, 128), "cw"),          # forward reads B / C element-wise; the backward on block states declines
    "rows": ((2, 64, 196, 1, 2, 64), "one"),
    "chunks": ((1, 64, 512, 1, 2, 64), "chunks"),
    "stream": ((2, 32, 260, 1, 1, 32), "one"),
    "rowsn16": ((2, 64, 196, 16, 2, 64), "one"),
    "ws_odd": ((2, 33, 197, 1, 3, 33), "one"),
}


@pytest.mark.parametrize("name", list(BC_ODD))
def test_scan_bc_two_bytes_off_a_word(name):
    """B / C views at an odd element offset of a bf16 buffer while u / delta / out stay dense and aligned.  Every
    forward and the resident-row, d_state 16 and warp-scan backwards load B / C one element at a time (or through
    stage_span, which copies a misaligned head / tail element-wise), so they may take such views; the column-walk backward
    moves them as 4-byte cp.async pieces and its planner declines (plan_cw_bwd)."""
    shape, fwd = BC_ODD[name]
    batch, dim, L, N, G, ddim = shape
    cpu = range_inputs("model", 49, batch, dim, L, N, G, ddim, True, False, True, True, BF16)
    g = to_gpu(cpu)
    views = dict(g, B=_in_flat(g["B"], 1), C=_in_flat(g["C"], 3))
    assert views["B"].data_ptr() % 4 == 2 and views["C"].data_ptr() % 4 == 2
    from tests.parity import long_row_scale
    _check(cpu, views, True, False, f"[B/C odd offset {name}]", long_row_scale(L), fwd, 2)
