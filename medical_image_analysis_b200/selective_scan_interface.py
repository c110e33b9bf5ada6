"""Autograd surface of the selective scan, mirroring the reference's.

* ``SelectiveScanOflex`` / ``SelectiveScanCore`` / ``SelectiveScanMamba``: the production autograd Functions of
  R2GenCSR/VMamba/classification/models/vmamba.py:294-312 / 273-291 / 250-270 (same argument lists; backward
  returns the same 11-tuple).
* ``selective_scan_fn`` / ``SelectiveScanFn``: mamba_ssm's public op as the ARM mixers call it
  (CXPMRG_Bench_MambaXray_VL/arm/Finetuning/mamba_simple.py:693-704; wrapper semantics of
  R2GenCSR/VMamba/kernels/selective_scan/test_selective_scan.py:18-165).
* ``causal_conv1d_fn``: the depth-wise causal conv (csrc/causal_conv1d.cu).
* ``mamba_inner_fn``, ``mamba_inner_fn_no_out_proj``, ``bimamba_inner_fn``: the fused inner blocks of the (un-vendored)
  Vim/ARM fork of mamba_ssm, computing what the reference's own slow path states (mamba_simple.py:665-709) as ONE
  autograd op, ``MambaInnerFn``, with mamba_ssm's saved-tensor contract and ``checkpoint_lvl`` (DESIGN.md 3.11).
* ``causal_conv1d_update`` / ``selective_state_update``: the recurrent decode step (``Mamba.step``,
  mamba_simple.py:717-762; Hugging Face ``MambaMixer``), one CUDA kernel each (csrc/ssm_step.cu), updating the conv and
  SSM states in place.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn.functional as F

from . import _lib, selective_scan_cuda, selective_scan_cuda_core, selective_scan_cuda_oflex

_fwd = torch.amp.custom_fwd(device_type="cuda")
_bwd = torch.amp.custom_bwd(device_type="cuda")


class SelectiveScanOflex(torch.autograd.Function):
    """vmamba.py:294-312."""

    @staticmethod
    @_fwd
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1, backnrows=1, oflex=True):
        ctx.delta_softplus = delta_softplus
        out, x, *rest = selective_scan_cuda_oflex.fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, 1, oflex)
        ctx.has_hblk = len(rest) > 0                       # block states for the column-walk backward (scan_bwd_cw.cuh)
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x, *rest[:1])
        return out

    @staticmethod
    @_bwd
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, x, *hb = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda_oflex.bwd(
            u, delta, A, B, C, D, delta_bias, dout, x, ctx.delta_softplus, 1, hblk=(hb[0] if hb else None))
        return (du, ddelta, dA, dB, dC, dD, ddelta_bias, None, None, None, None)


class SelectiveScanCore(torch.autograd.Function):
    """vmamba.py:273-291."""

    @staticmethod
    @_fwd
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1, backnrows=1, oflex=True):
        ctx.delta_softplus = delta_softplus
        out, x, *rest = selective_scan_cuda_core.fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, 1)
        ctx.has_hblk = len(rest) > 0                       # block states for the column-walk backward (scan_bwd_cw.cuh)
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x, *rest[:1])
        return out

    @staticmethod
    @_bwd
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, x, *hb = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda_core.bwd(
            u, delta, A, B, C, D, delta_bias, dout, x, ctx.delta_softplus, 1, hblk=(hb[0] if hb else None))
        return (du, ddelta, dA, dB, dC, dD, ddelta_bias, None, None, None, None)


class SelectiveScanMamba(torch.autograd.Function):
    """vmamba.py:250-270 (mamba_ssm's module without the z gate)."""

    @staticmethod
    @_fwd
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1, backnrows=1, oflex=True):
        ctx.delta_softplus = delta_softplus
        out, x, *rest = selective_scan_cuda.fwd(u, delta, A, B, C, D, None, delta_bias, delta_softplus)
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x)
        return out

    @staticmethod
    @_bwd
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, x = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda.bwd(
            u, delta, A, B, C, D, None, delta_bias, dout, x, None, None, ctx.delta_softplus, False)
        return (du, ddelta, dA, dB, dC, dD, ddelta_bias, None, None, None, None)


class SelectiveScanFn(torch.autograd.Function):
    """mamba_ssm.ops.selective_scan_interface.SelectiveScanFn (semantics: test_selective_scan.py:20-147)."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
        if u.stride(-1) != 1:
            u = u.contiguous()
        if delta.stride(-1) != 1:
            delta = delta.contiguous()
        if D is not None:
            D = D.contiguous()
        if B.stride(-1) != 1:
            B = B.contiguous()
        if C.stride(-1) != 1:
            C = C.contiguous()
        if z is not None and z.stride(-1) != 1:
            z = z.contiguous()
        ctx.squeeze_B = ctx.squeeze_C = False
        if B.dim() == 3:
            B = B.unsqueeze(1)
            ctx.squeeze_B = True
        if C.dim() == 3:
            C = C.unsqueeze(1)
            ctx.squeeze_C = True
        ctx.d_dtype = ctx.bias_dtype = None
        if D is not None and D.dtype != torch.float32:
            ctx.d_dtype = D.dtype
            D = D.float()
        if delta_bias is not None and delta_bias.dtype != torch.float32:
            ctx.bias_dtype = delta_bias.dtype
            delta_bias = delta_bias.float()
        out, x, *rest = selective_scan_cuda.fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus)
        ctx.delta_softplus = delta_softplus
        ctx.has_z = z is not None
        last_state = x[:, :, -1, 1::2]  # (batch, dim, dstate)
        if not ctx.has_z:
            ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x)
            return out if not return_last_state else (out, last_state)
        ctx.save_for_backward(u, delta, A, B, C, D, z, delta_bias, x, out)
        out_z = rest[0]
        return out_z if not return_last_state else (out_z, last_state)

    @staticmethod
    def backward(ctx, dout, *args):
        if not ctx.has_z:
            u, delta, A, B, C, D, delta_bias, x = ctx.saved_tensors
            z = out = None
        else:
            u, delta, A, B, C, D, z, delta_bias, x, out = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda.bwd(
            u, delta, A, B, C, D, z, delta_bias, dout, x, out, None, ctx.delta_softplus, False)
        dz = rest[0] if ctx.has_z else None
        if ctx.squeeze_B:
            dB = dB.squeeze(1)
        if ctx.squeeze_C:
            dC = dC.squeeze(1)
        if dD is not None and ctx.d_dtype is not None:
            dD = dD.to(ctx.d_dtype)
        if ddelta_bias is not None and ctx.bias_dtype is not None:
            ddelta_bias = ddelta_bias.to(ctx.bias_dtype)
        return (du, ddelta, dA, dB, dC, dD, dz, ddelta_bias, None, None)


def selective_scan_fn(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
    """mamba_ssm's op.  If return_last_state, returns (out, last_state (batch, dim, dstate)); the gradient of the
    last state is not propagated (as upstream)."""
    return SelectiveScanFn.apply(u, delta, A, B, C, D, z, delta_bias, delta_softplus, return_last_state)


# ---------------------------------------------------------------------------------------------------------
# Fused inner blocks of the Vim / ARM fork of mamba_ssm, composed (mamba_simple.py:665-709 is their definition).
def _conv_rows(t):
    """(batch, dim, L) view with contiguous channel rows and a batch stride that is a multiple of 4 elements (the first
    half of `xz` qualifies as it is); anything else is made contiguous."""
    if t.stride(2) != 1 or t.stride(1) != t.shape[2] or t.stride(0) % 4 or t.data_ptr() % (4 * t.element_size()):
        t = t.contiguous()
    return t


class CausalConv1dFn(torch.autograd.Function):
    """Depth-wise causal conv1d (+ bias, + SiLU) through the C ABI (csrc/causal_conv1d.cu)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, weight, bias, silu):
        if x.dim() != 3 or weight.dim() != 2 or weight.shape[0] != x.shape[1]:
            raise RuntimeError("causal_conv1d_fn: x must be (batch, dim, seqlen) and weight (dim, width)")
        if not x.is_cuda:
            raise RuntimeError("causal_conv1d_fn: this build has no CPU path (x must be a CUDA tensor)")
        x = _conv_rows(x)
        w32 = weight.detach().float().contiguous()
        b32 = None if bias is None else bias.detach().float().contiguous()
        y = torch.empty(x.shape, device=x.device, dtype=x.dtype)
        B, D, L = x.shape
        _lib.call("mia_causal_conv1d_fwd", "causal_conv1d_fwd", x.device, x.data_ptr(), w32.data_ptr(), 0 if b32 is None else b32.data_ptr(),
                  y.data_ptr(), B, D, L, weight.shape[1], int(silu), _lib.dtype_code(x.dtype), x.stride(0), x.stride(1), y.stride(0),
                  y.stride(1))
        ctx.save_for_backward(x, w32, b32 if b32 is not None else w32.new_empty(0))
        ctx.silu, ctx.has_bias, ctx.wdtype, ctx.bdtype = bool(silu), bias is not None, weight.dtype, None if bias is None else bias.dtype
        return y

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, w32, b32 = ctx.saved_tensors
        dy = _conv_rows(dy.to(x.dtype))
        B, D, L = x.shape
        dx = torch.empty(x.shape, device=x.device, dtype=x.dtype)
        dw = torch.empty_like(w32)
        db = torch.empty(D, device=x.device, dtype=torch.float32) if ctx.has_bias else None
        _lib.call("mia_causal_conv1d_bwd", "causal_conv1d_bwd", x.device, x.data_ptr(), w32.data_ptr(), b32.data_ptr() if ctx.has_bias else 0,
                  dy.data_ptr(), dx.data_ptr(), dw.data_ptr(), 0 if db is None else db.data_ptr(), B, D, L, w32.shape[1], int(ctx.silu),
                  _lib.dtype_code(x.dtype), x.stride(0), x.stride(1), dy.stride(0), dy.stride(1), dx.stride(0), dx.stride(1))
        return dx, dw.to(ctx.wdtype), (db.to(ctx.bdtype) if db is not None else None), None


def causal_conv1d_fn(x, weight, bias=None, activation=None):
    """causal_conv1d.causal_conv1d_fn: depthwise causal conv, x (b, d, l), weight (d, w); mamba_simple.py:673-681."""
    if activation not in (None, "silu", "swish"):
        raise NotImplementedError("activation must be None, silu or swish")
    L = x.shape[-1]
    if L % 4:   # the kernels move 4-token pieces: pad on the right (a causal filter never looks there) and cut again
        return CausalConv1dFn.apply(F.pad(x, (0, 4 - L % 4)), weight, bias, activation is not None)[..., :L]
    return CausalConv1dFn.apply(x, weight, bias, activation is not None)


def _no_cpu(op, *ts):
    ts = [t for t in ts if t is not None]
    if not all(t.is_cuda for t in ts):
        raise RuntimeError(f"{op}: this build has no CPU path (the tensors must be CUDA tensors)")
    if any(t.device != ts[0].device for t in ts):
        raise RuntimeError(f"{op}: all tensors must be on the same device")


def _rows(t):
    """a (batch, n) operand of the decode step: any batch stride, unit last stride (a copy only when it is not)."""
    return t if t.stride(-1) == 1 or t.shape[-1] == 1 else t.contiguous()


def _vec(t, n, what):
    """a (n) parameter read as stored (its own dtype) by the decode-step kernels."""
    if t.shape != (n,):
        raise RuntimeError(f"{what} must have shape ({n},), got {tuple(t.shape)}")
    if t.dtype not in _lib.DTYPE_CODES:
        raise RuntimeError(f"{what} must be float32, float16 or bfloat16")
    return t if t.stride(0) == 1 else t.contiguous()


def causal_conv1d_update(x, conv_state, weight, bias=None, activation=None):
    """causal_conv1d.causal_conv1d_update, one decode step (Mamba.step, mamba_simple.py:732-738; Hugging Face
    MambaMixer.cuda_kernels_forward): x (batch, dim), conv_state (batch, dim, width <= 4) shifted left in place with x
    written into its last column, weight (dim, width); returns act(bias + sum_k weight[:, k] conv_state[..., k]) in x's
    dtype, computed in fp32 by csrc/ssm_step.cu.  weight / bias / conv_state are read in their own dtypes."""
    if activation not in (None, "silu", "swish"):
        raise NotImplementedError("activation must be None, silu or swish")
    _no_cpu("causal_conv1d_update", x, conv_state, weight, bias)
    if x.dim() != 2 or conv_state.dim() != 3 or weight.dim() != 2:
        raise RuntimeError("causal_conv1d_update: x must be (batch, dim), conv_state (batch, dim, width) and weight (dim, width)")
    batch, dim = x.shape
    width = weight.shape[1]
    if conv_state.shape != (batch, dim, width) or weight.shape[0] != dim:
        raise RuntimeError(f"causal_conv1d_update: conv_state {tuple(conv_state.shape)} / weight {tuple(weight.shape)} do not match "
                           f"x {tuple(x.shape)}")
    for t, what in ((x, "x"), (conv_state, "conv_state"), (weight, "weight")):
        if t.dtype not in _lib.DTYPE_CODES:
            raise RuntimeError(f"causal_conv1d_update: {what} must be float32, float16 or bfloat16")
    x = _rows(x)
    bias = None if bias is None else _vec(bias, dim, "causal_conv1d_update: bias")
    out = torch.empty((batch, dim), device=x.device, dtype=x.dtype)
    code = _lib.dtype_code
    _lib.call("mia_causal_conv1d_update", "causal_conv1d_update", x.device, x.data_ptr(), conv_state.data_ptr(), weight.data_ptr(),
              0 if bias is None else bias.data_ptr(), out.data_ptr(), batch, dim, width, int(activation is not None), code(x.dtype),
              code(conv_state.dtype), code(weight.dtype), code(bias.dtype) if bias is not None else 0, x.stride(0), conv_state.stride(0),
              conv_state.stride(1), conv_state.stride(2), weight.stride(0), weight.stride(1), out.stride(0))
    return out


def selective_state_update(state, x, dt, A, B, C, D=None, z=None, dt_bias=None, dt_softplus=False):
    """mamba_ssm.ops.triton.selective_state_update.selective_state_update: one token of the selective scan, with the
    state updated in place (csrc/ssm_step.cu).

        state (batch, dim, dstate) f32 / bf16 / f16, dstate contiguous;  x, dt, z (batch, dim);  B, C (batch, dstate)
        A (dim, dstate) f32;  D, dt_bias (dim) in any of the three dtypes

    Returns out (batch, dim) in x's dtype.  No autograd (as upstream).  Grouped B / C and the Mamba-2 head layout are not
    supported."""
    _no_cpu("selective_state_update", state, x, dt, A, B, C, D, z, dt_bias)
    if state.dim() != 3:
        raise NotImplementedError("selective_state_update: only the (batch, dim, dstate) state layout (no Mamba-2 heads)")
    batch, dim, dstate = state.shape
    if state.stride(2) != 1 and dstate > 1:
        raise RuntimeError("selective_state_update: the state's dstate dimension must be contiguous (it is updated in place)")
    if x.shape != (batch, dim) or dt.shape != (batch, dim) or (z is not None and z.shape != (batch, dim)):
        raise RuntimeError(f"selective_state_update: x / dt / z must be (batch, dim) = {(batch, dim)}")
    if B.shape != (batch, dstate) or C.shape != (batch, dstate):
        raise NotImplementedError(f"selective_state_update: B and C must be (batch, dstate) = {(batch, dstate)} (no grouped B / C)")
    if A.shape != (dim, dstate):
        raise RuntimeError(f"selective_state_update: A must be (dim, dstate) = {(dim, dstate)}")
    if state.dtype not in _lib.DTYPE_CODES or x.dtype not in _lib.DTYPE_CODES:
        raise RuntimeError("selective_state_update: state and x must be float32, float16 or bfloat16")
    for t, what in ((dt, "dt"), (B, "B"), (C, "C"), (z, "z")):
        if t is not None and t.dtype != x.dtype:
            raise RuntimeError(f"selective_state_update: {what} must have x's dtype {x.dtype}, got {t.dtype}")
    x, dt, B, C = _rows(x), _rows(dt), _rows(B), _rows(C)
    z = None if z is None else _rows(z)
    A = A if A.dtype == torch.float32 else A.float()
    D = None if D is None else _vec(D, dim, "selective_state_update: D")
    dt_bias = None if dt_bias is None else _vec(dt_bias, dim, "selective_state_update: dt_bias")
    out = torch.empty((batch, dim), device=x.device, dtype=x.dtype)
    p = _lib.MiaSSUParams()
    p.batch, p.dim, p.dstate = batch, dim, dstate
    p.state_type, p.itype = _lib.dtype_code(state.dtype), _lib.dtype_code(x.dtype)
    p.D_type = _lib.dtype_code(D.dtype) if D is not None else 0
    p.dt_bias_type = _lib.dtype_code(dt_bias.dtype) if dt_bias is not None else 0
    p.dt_softplus = int(bool(dt_softplus))
    p.state, p.x, p.dt, p.B, p.C, p.A, p.out = (t.data_ptr() for t in (state, x, dt, B, C, A, out))
    p.z = z.data_ptr() if z is not None else None
    p.D = D.data_ptr() if D is not None else None
    p.dt_bias = dt_bias.data_ptr() if dt_bias is not None else None
    p.state_batch_stride, p.state_d_stride = state.stride(0), state.stride(1)
    p.x_batch_stride, p.dt_batch_stride, p.B_batch_stride, p.C_batch_stride = x.stride(0), dt.stride(0), B.stride(0), C.stride(0)
    p.z_batch_stride = z.stride(0) if z is not None else 0
    p.out_batch_stride = out.stride(0)
    p.A_d_stride, p.A_dstate_stride = A.stride(0), A.stride(1)
    _lib.call("mia_selective_state_update", "selective_state_update", x.device, ctypes.byref(p))
    return out


# ---------------------------------------------------------------------------------------------------------
# The fused inner block: one autograd Function (mamba_ssm's MambaInnerFn contract) on the conv / gate kernels of
# csrc/causal_conv1d.cu (mia_*_ex), the projection GEMMs and the CUDA scan.  See DESIGN.md section 3.11.
def _bdl(t, rev=False):
    """struct mia_bdl of a (batch, dim, seqlen) view (any strides); rev: its time-reversed view."""
    if rev:
        return _lib.MiaBdl(t.data_ptr() + (t.shape[2] - 1) * t.stride(2) * t.element_size(), t.stride(0), t.stride(1), -t.stride(2))
    return _lib.MiaBdl(t.data_ptr(), t.stride(0), t.stride(1), t.stride(2))


def _tm(t, L):
    """struct mia_bdl of a token-major (batch * L, dim) matrix seen as (batch, dim, L)."""
    return _lib.MiaBdl(t.data_ptr(), L * t.stride(0), t.stride(1), t.stride(0))


def _ops(*ops):
    return (_lib.MiaBdl * len(ops))(*ops), len(ops)


def _tm_buffer(n, d, dtype, dev):
    """(n, d) token-major activation whose row pitch is a multiple of 8 elements (the wgmma GEMM's operand rule)."""
    p = (d + 7) // 8 * 8
    return torch.empty((n, p), dtype=dtype, device=dev)[:, :d]


def _gemm_ok(*ts):
    from . import gemm as _gemm
    return all(_gemm._mn_ok(t) for t in ts)


def _mm_tn(a, w, bias=None):
    """a (M, K) @ w (N, K)^T (+ bias): the wgmma kernel (bias in its epilogue) for bf16 / fp16, the library GEMM for fp32
    (as gemm.linear)."""
    from . import gemm as _gemm
    if a.dtype != torch.float32:
        return _gemm.gemm_tn(a, w, bias)
    return a @ w.t() if bias is None else torch.addmm(bias.to(a.dtype), a, w.t())


def _mm_nn(a, w):
    """a (M, K) @ w (K, N), w read in place."""
    from . import gemm as _gemm
    if a.dtype != torch.float32 and _gemm_ok(a, w) and a.shape[1] % 8 == 0:
        return _gemm.gemm(a, w, False, True)
    return _gemm.gemm_tn(a, _gemm.transpose2d(w)) if a.dtype != torch.float32 else a @ w


def _mm_wgrad(dy, x):
    """dy (M, N)^T @ x (M, K) -> (N, K) fp32: weight gradients."""
    from . import gemm as _gemm
    if dy.dtype == torch.float32:
        return dy.t() @ x
    if _gemm_ok(dy, x):
        return _gemm.gemm(dy, x, True, True, torch.float32)
    return _gemm.gemm_tn(_gemm.transpose2d(dy), _gemm.transpose2d(x), out_dtype=torch.float32)


class MambaInnerFn(torch.autograd.Function):
    """conv1d + SiLU -> x_proj -> dt_proj -> selective scan -> SiLU(z) gate [-> out_proj] as ONE autograd op, with the
    saved-tensor contract of mamba_ssm's MambaInnerFn (checkpoint_lvl 1: xz, x_dbl, the scan's out, B, C, its
    checkpoints and the parameters; level 0 also keeps the conv output and delta; the rest is recomputed by the same
    kernels, so both levels give the same bits).  A_b given: Vim's bidirectional block, the second scan running over
    the reversed sequence with A_b (bimamba_inner_fn).  The scan runs without z on dense operands; the gate is
    mia_silu_gate_fwd_ex / _bwd_ex, which read z in place in xz and write dz in place into dxz."""

    @staticmethod
    @_fwd
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight, out_proj_bias, A, A_b, D,
                delta_bias, B_proj_bias, C_proj_bias, delta_softplus, checkpoint_lvl):
        from .scan_op import scan_fwd
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not xz.is_cuda:
            raise RuntimeError("mamba_inner_fn: this build has no CPU path (xz must be a CUDA tensor)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else xz.dtype
        if T not in _lib.DTYPE_CODES:
            raise RuntimeError("mamba_inner_fn: xz must be float32, float16 or bfloat16")
        xz = xz.to(T)
        b, d2, L = xz.shape
        d = d2 // 2
        W = conv1d_weight.shape[-1]
        R, N = delta_proj_weight.shape[1], A.shape[1]
        K = x_proj_weight.shape[0]
        if K != R + 2 * N or x_proj_weight.shape[1] != d:
            raise RuntimeError(f"mamba_inner_fn: x_proj_weight {tuple(x_proj_weight.shape)} is not (dt_rank + 2 d_state, d_inner) = "
                               f"({R + 2 * N}, {d})")
        dev = xz.device
        w32 = conv1d_weight.detach().reshape(d, W).float().contiguous()
        cb32 = None if conv1d_bias is None else conv1d_bias.detach().float().contiguous()
        wx, wdt = x_proj_weight.to(T), delta_proj_weight.to(T)
        wout = None if out_proj_weight is None else out_proj_weight.to(T)
        D32 = None if D is None else D.float().contiguous()
        db32 = None if delta_bias is None else delta_bias.float().contiguous()
        bi = A_b is not None
        ctx.sizes = (b, d, L, W, R, N, K, T, bi, checkpoint_lvl, delta_softplus)
        ctx.has = (conv1d_bias is not None, out_proj_weight is not None, out_proj_bias is not None, D is not None,
                   delta_bias is not None, B_proj_bias is not None, C_proj_bias is not None)

        u, u_rev, u_tm = MambaInnerFn._conv(xz, w32, cb32, ctx, True, True)
        x_dbl = _mm_tn(u_tm, wx)                                                     # (b l, R + 2N)
        delta, Bm, Cm = MambaInnerFn._proj(x_dbl, wdt, B_proj_bias, C_proj_bias, b, L, R, N, False)
        out_f, x_f, _ = scan_fwd(u, delta, A, Bm, Cm, D32, None, db32, delta_softplus)
        outs, saved_bi = [out_f], []
        if bi:
            delta_r, Br, Cr = MambaInnerFn._proj(x_dbl, wdt, B_proj_bias, C_proj_bias, b, L, R, N, True)
            out_b, x_b, _ = scan_fwd(u_rev, delta_r, A_b, Br, Cr, D32, None, db32, delta_softplus)
            outs.append(out_b)
            saved_bi = [out_b, x_b, A_b]
        z = xz[:, d:]
        if wout is not None:
            y_tm = MambaInnerFn._gate(outs, z, b, d, L, T, dev)
            y = _mm_tn(y_tm, wout, out_proj_bias).view(b, L, -1)
        else:
            y = torch.empty((b, d, L), dtype=T, device=dev)
            ins, n_in = _ops(_bdl(outs[0]), *([_bdl(outs[1], rev=True)] if bi else []))
            oz, n_oz = _ops(_bdl(y))
            _lib.call("mia_silu_gate_fwd_ex", "silu_gate_fwd", dev, ins, n_in, ctypes.byref(_bdl(z)), oz, n_oz, b, d, L, _lib.dtype_code(T))
        keep = [u, delta] + ([u_rev, delta_r] if bi else []) if checkpoint_lvl == 0 else []
        ctx.n_keep = len(keep)
        ctx.save_for_backward(xz, x_dbl, out_f, Bm, Cm, x_f, w32, cb32, x_proj_weight, delta_proj_weight, out_proj_weight, A, D32, db32,
                              B_proj_bias, C_proj_bias, *saved_bi, *keep)
        ctx.dtypes = (conv1d_weight.dtype, None if conv1d_bias is None else conv1d_bias.dtype, None if D is None else D.dtype,
                      None if delta_bias is None else delta_bias.dtype, None if out_proj_bias is None else out_proj_bias.dtype)
        ctx.conv_shape = conv1d_weight.shape
        return y

    @staticmethod
    def _conv(xz, w32, cb32, ctx, want_cm, want_tm):
        """conv + SiLU of xz's x half in one launch -> (u (b, d, l), its reversed copy (bimamba) | None, u token-major | None)."""
        b, d, L, W, R, N, K, T, bi, _, _ = ctx.sizes
        dev = xz.device
        u = torch.empty((b, d, L), dtype=T, device=dev) if want_cm else None
        u_rev = torch.empty((b, d, L), dtype=T, device=dev) if want_cm and bi else None
        u_tm = _tm_buffer(b * L, d, T, dev) if want_tm else None
        outs = ([_bdl(u)] if u is not None else []) + ([_bdl(u_rev, rev=True)] if u_rev is not None else []) + \
               ([_tm(u_tm, L)] if u_tm is not None else [])
        arr, n = _ops(*outs)
        _lib.call("mia_causal_conv1d_fwd_ex", "causal_conv1d_fwd_ex", dev, ctypes.byref(_bdl(xz[:, :d])), w32.data_ptr(),
                  None if cb32 is None else cb32.data_ptr(), arr, n, b, d, L, W, 1, _lib.dtype_code(T))
        return u, u_rev, u_tm

    @staticmethod
    def _proj(x_dbl, wdt, B_proj_bias, C_proj_bias, b, L, R, N, rev):
        """delta (b, d, l) = dt_proj(x_dbl[:, :R]) and B, C (b, 1, N, l) from x_dbl, over the reversed sequence when rev."""
        xd = x_dbl.view(b, L, -1)
        if rev:
            xd = xd.flip(1)                                                       # (b l, R + 2N): small
        delta = torch.bmm(wdt.expand(b, *wdt.shape), xd[:, :, :R].transpose(1, 2))   # (b, d, l), dense rows for the scan
        Bm, Cm = xd[:, :, R:R + N], xd[:, :, R + N:R + 2 * N]
        if B_proj_bias is not None:
            Bm = Bm + B_proj_bias.to(Bm.dtype)
        if C_proj_bias is not None:
            Cm = Cm + C_proj_bias.to(Cm.dtype)
        return delta, Bm.transpose(1, 2).unsqueeze(1).contiguous(), Cm.transpose(1, 2).unsqueeze(1).contiguous()

    @staticmethod
    def _gate(outs, z, b, d, L, T, dev):
        """(out_f [+ reversed out_b]) * silu(z) written token-major for out_proj."""
        y_tm = _tm_buffer(b * L, d, T, dev)
        ins, n_in = _ops(_bdl(outs[0]), *([_bdl(outs[1], rev=True)] if len(outs) > 1 else []))
        oz, n_oz = _ops(_tm(y_tm, L))
        _lib.call("mia_silu_gate_fwd_ex", "silu_gate_fwd_ex", dev, ins, n_in, ctypes.byref(_bdl(z)), oz, n_oz, b, d, L, _lib.dtype_code(T))
        return y_tm

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        from .scan_op import scan_bwd
        b, d, L, W, R, N, K, T, bi, lvl, softplus = ctx.sizes
        has_cb, has_out, has_ob, has_D, has_db, has_Bb, has_Cb = ctx.has
        sv = ctx.saved_tensors
        (xz, x_dbl, out_f, Bm, Cm, x_f, w32, cb32, x_proj_weight, delta_proj_weight, out_proj_weight, A, D32, db32,
         B_proj_bias, C_proj_bias) = sv[:16]
        rest = list(sv[16:])
        out_b, x_b, A_b = rest[:3] if bi else (None, None, None)
        keep = rest[3:] if bi else rest
        dev = xz.device
        wx, wdt = x_proj_weight.to(T), delta_proj_weight.to(T)
        # recompute what the level did not keep, with the forward's kernels (same bits)
        if lvl == 0:
            u, delta = keep[0], keep[1]
            u_rev, delta_r = (keep[2], keep[3]) if bi else (None, None)
        else:
            u, u_rev, _ = MambaInnerFn._conv(xz, w32, cb32, ctx, True, False)
            delta = MambaInnerFn._proj(x_dbl, wdt, None, None, b, L, R, N, False)[0]
            delta_r = MambaInnerFn._proj(x_dbl, wdt, None, None, b, L, R, N, True)[0] if bi else None
        z = xz[:, d:]
        outs = [out_f] + ([out_b] if bi else [])
        dxz = torch.empty_like(xz)
        d_out_w = d_out_b = None
        if has_out:
            wout = out_proj_weight.to(T)
            dy2 = dy.to(T).reshape(b * L, -1).contiguous()                         # (b l, d_model)
            y_tm = MambaInnerFn._gate(outs, z, b, d, L, T, dev)
            d_out_w = _mm_wgrad(dy2, y_tm).to(out_proj_weight.dtype)
            if has_ob:
                d_out_b = dy2.float().sum(0).to(ctx.dtypes[4])
            del y_tm
            g_tm = _mm_nn(dy2, wout)                                                 # (b l, d): d of the gate's output
            g = _tm(g_tm, L)
        else:
            g_cm = dy.to(T)
            g = _bdl(g_cm)
        # the gated gradient goes to the scan in fp32 ("oflex" dout), unrounded as when the scan applies the gate itself
        dout_f = torch.empty((b, d, L), dtype=torch.float32, device=dev)
        dout_b = torch.empty((b, d, L), dtype=torch.float32, device=dev) if bi else None
        ins, n_in = _ops(_bdl(out_f), *([_bdl(out_b, rev=True)] if bi else []))
        douts, n_do = _ops(_bdl(dout_f), *([_bdl(dout_b, rev=True)] if bi else []))
        _lib.call("mia_silu_gate_bwd_ex", "silu_gate_bwd_ex", dev, ctypes.byref(g), ins, n_in, ctypes.byref(_bdl(z)), douts, n_do,
                  ctypes.byref(_bdl(dxz[:, d:])), b, d, L, _lib.dtype_code(T), _lib.MIA_F32)
        g = g_tm = g_cm = None                                                       # transients go as soon as they are used
        du_f, dd_f, dA, dB_f, dC_f, dD, ddb, _ = scan_bwd(u, delta, A, Bm, Cm, D32, None, db32, dout_f, x_f, None, softplus)
        del dout_f, u, delta
        xd = x_dbl.view(b, L, K)
        Kp = (K + 7) // 8 * 8
        dx_dbl = torch.zeros((b * L, Kp), dtype=T, device=dev)
        dxd = dx_dbl.view(b, L, Kp)
        wdt_b = wdt.expand(b, *wdt.shape)
        dxd[:, :, :R] = torch.bmm(dd_f.transpose(1, 2), wdt_b)                       # (b, l, R), ddelta read in place
        dxd[:, :, R:R + N] = dB_f.squeeze(1).transpose(1, 2)
        dxd[:, :, R + N:K] = dC_f.squeeze(1).transpose(1, 2)
        f32 = {} if T == torch.float32 else {"out_dtype": torch.float32}             # fp32 partials per batch element
        d_wdt = torch.bmm(dd_f, xd[:, :, :R], **f32).sum(0)                           # (d, R)
        dA_b = du_b = None
        if bi:
            Br, Cr = Bm.flip(-1), Cm.flip(-1)                                       # the forward's reversed B / C, bit for bit
            du_b, dd_b, dA_b, dB_b, dC_b, dD_b, ddb_b, _ = scan_bwd(u_rev, delta_r, A_b, Br, Cr, D32, None, db32, dout_b, x_b, None, softplus)
            del dout_b, u_rev, delta_r
            dxd[:, :, :R] += torch.bmm(dd_b.transpose(1, 2), wdt_b).flip(1)
            dxd[:, :, R:R + N] += dB_b.squeeze(1).transpose(1, 2).flip(1)
            dxd[:, :, R + N:K] += dC_b.squeeze(1).transpose(1, 2).flip(1)
            d_wdt += torch.bmm(dd_b, xd.flip(1)[:, :, :R], **f32).sum(0)
            dD = None if dD is None else dD + dD_b
            ddb = None if ddb is None else ddb + ddb_b
        dxp = dx_dbl[:, :K]
        d_Bb = dxd[:, :, R:R + N].float().sum((0, 1)).to(B_proj_bias.dtype) if has_Bb else None
        d_Cb = dxd[:, :, R + N:K].float().sum((0, 1)).to(C_proj_bias.dtype) if has_Cb else None
        _, _, u_tm = MambaInnerFn._conv(xz, w32, cb32, ctx, False, True)            # x_proj's input, recomputed at both levels
        d_wx = _mm_wgrad(dxp, u_tm).to(x_proj_weight.dtype)                          # (R + 2N, d)
        del u_tm
        wx_p = wx if Kp == K else torch.cat([wx, wx.new_zeros(Kp - K, d)])
        dy_tm = _mm_nn(dx_dbl, wx_p) if T != torch.float32 else dxp @ wx               # (b l, d): x_proj's input gradient
        dys = [_bdl(du_f)] + ([_bdl(du_b, rev=True)] if bi else []) + [_tm(dy_tm, L)]
        arr, n = _ops(*dys)
        dw32 = torch.empty_like(w32)
        dcb32 = torch.empty(d, dtype=torch.float32, device=dev) if has_cb else None
        ws = torch.empty((max(1, int(_lib.lib().mia_causal_conv1d_bwd_ex_workspace(b, d, L, W))),), dtype=torch.uint8, device=dev)
        _lib.call("mia_causal_conv1d_bwd_ex", "causal_conv1d_bwd_ex", dev, ctypes.byref(_bdl(xz[:, :d])), w32.data_ptr(),
                  None if cb32 is None else cb32.data_ptr(), arr, n, ctypes.byref(_bdl(dxz[:, :d])), dw32.data_ptr(),
                  None if dcb32 is None else dcb32.data_ptr(), ws.data_ptr(), ws.numel(), b, d, L, W, 1, _lib.dtype_code(T))
        cw_dtype, cb_dtype, D_dtype, db_dtype, _ = ctx.dtypes
        return (dxz, dw32.view(ctx.conv_shape).to(cw_dtype), None if dcb32 is None else dcb32.to(cb_dtype), d_wx,
                d_wdt.to(delta_proj_weight.dtype), d_out_w, d_out_b, dA, dA_b, None if dD is None else dD.to(D_dtype),
                None if ddb is None else ddb.to(db_dtype), d_Bb, d_Cb, None, None)


def _no_given_BC(B, C):
    if B is not None or C is not None:
        raise NotImplementedError("only input-dependent B / C (B=None, C=None), as at every call site of the reference")


def mamba_inner_fn_no_out_proj(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B=None, C=None, D=None,
                               delta_bias=None, B_proj_bias=None, C_proj_bias=None, delta_softplus=True, checkpoint_lvl=1):
    """(b, 2 d_inner, l) -> gated scan output (b, d_inner, l); call sites mamba_simple.py:450-511."""
    _no_given_BC(B, C)
    return MambaInnerFn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, None, None, A, None, D, delta_bias,
                              B_proj_bias, C_proj_bias, delta_softplus, checkpoint_lvl)


def mamba_inner_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight, out_proj_bias, A,
                   B=None, C=None, D=None, delta_bias=None, B_proj_bias=None, C_proj_bias=None, delta_softplus=True, checkpoint_lvl=1):
    """mamba_simple.py:650-663: the block above followed by out_proj; returns (b, l, d_model)."""
    _no_given_BC(B, C)
    return MambaInnerFn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight, out_proj_bias, A, None,
                              D, delta_bias, B_proj_bias, C_proj_bias, delta_softplus, checkpoint_lvl)


def bimamba_inner_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight, out_proj_bias, A, A_b,
                     B=None, C=None, D=None, delta_bias=None, B_proj_bias=None, C_proj_bias=None, delta_softplus=True, checkpoint_lvl=1):
    """Vim's bidirectional block (mamba_simple.py:431-446): one set of projections, a forward scan with A and a
    scan over the flipped sequence with A_b, summed before out_proj."""
    _no_given_BC(B, C)
    return MambaInnerFn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight, out_proj_bias, A, A_b,
                              D, delta_bias, B_proj_bias, C_proj_bias, delta_softplus, checkpoint_lvl)
