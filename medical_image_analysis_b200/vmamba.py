"""SS2D (VMamba's 2-D selective-scan block) on the H100 kernels.

Mirrors the module surface of R2GenCSR/VMamba/classification/models/vmamba.py: ``CrossScan`` / ``CrossMerge`` (:25-67),
``cross_selective_scan`` (:318-427) and ``SS2D`` with the v2 family of ``forward_type`` strings (:540-584, 662-802,
1092-1129) -- same constructor arguments, same parameter names and shapes (``x_proj_weight (K, R+2N, D)``,
``dt_projs_weight (K, D, R)``, ``dt_projs_bias (K, D)``, ``A_logs (K*D, N)``, ``Ds (K*D)``, ``in_proj``, ``conv2d``,
``out_norm``, ``out_proj``) so published VMamba checkpoints load unchanged.  The four scan orders and their merge run as
single-pass CUDA kernels (csrc/cross_scan.cu) instead of torch copies / Triton; the scan is ``SelectiveScanOflex/Core/Mamba``
from ``selective_scan_interface``; in_proj / out_proj / the MLPs run on the wgmma GEMM (``gemm.linear``) for bf16 / fp16
activations.  Also here: the legacy ``forwardv0`` and experimental ``forwardxv`` families (:1020-1090, 1131-1215), the
1- / 2-direction ablations (:71-131), and the callers ``VSSBlock`` / ``VSSM`` / ``Backbone_VSSM`` (:1218-1725) with the
reference's parameter names, so that its checkpoints and configs (configs/vssm1/*.yaml) apply unchanged.  Parity: every
class is checked against vectors produced by executing the reference's own module (tests/golden/modules_vmamba.npz).
"""
from __future__ import annotations

import ctypes
import math
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn
import torch.nn.functional as F
import torch.utils.checkpoint as checkpoint

from . import _lib
from . import gemm as _gemm
from .selective_scan_interface import SelectiveScanCore, SelectiveScanMamba, SelectiveScanOflex

def _cs_call(name: str, src: torch.Tensor, dst: torch.Tensor, B: int, C: int, H: int, W: int) -> None:
    if not src.is_cuda:
        raise RuntimeError("CrossScan / CrossMerge need CUDA tensors (there is no CPU fallback)")
    if src.dtype not in _lib.DTYPE_CODES:
        raise RuntimeError("CrossScan / CrossMerge support float32, float16 and bfloat16")
    _lib.call(name, "cross scan/merge", src.device, src.data_ptr(), dst.data_ptr(), B, C, H, W, _lib.dtype_code(src.dtype))


class DWConv2dFn(torch.autograd.Function):
    """Depth-wise 3x3 conv2d (+ bias, + SiLU) of SS2D through the C ABI (csrc/dwconv2d.cu); x (B, C, H, W) channel-first,
    weight (C, 1, 3, 3) as held by nn.Conv2d(C, C, 3, padding=1, groups=C) (vmamba.py:574-582, 1120-1122)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, weight, bias, silu):
        if x.dim() != 4 or tuple(weight.shape) != (x.shape[1], 1, 3, 3):
            raise RuntimeError("dwconv2d: x must be (B, C, H, W) and weight (C, 1, 3, 3)")
        if not x.is_cuda:
            raise RuntimeError("dwconv2d: this build has no CPU path (x must be a CUDA tensor)")
        x = x.contiguous()
        w32 = weight.detach().float().reshape(-1, 9).contiguous()
        b32 = None if bias is None else bias.detach().float().contiguous()
        y = torch.empty_like(x)
        B, C, H, W = x.shape
        _lib.call("mia_dwconv2d_fwd", "dwconv2d_fwd", x.device, x.data_ptr(), w32.data_ptr(), 0 if b32 is None else b32.data_ptr(),
                  y.data_ptr(), B, C, H, W, int(silu), _lib.dtype_code(x.dtype))
        ctx.save_for_backward(x, w32, b32 if b32 is not None else w32.new_empty(0))
        ctx.silu, ctx.has_bias, ctx.wdtype, ctx.bdtype = bool(silu), bias is not None, weight.dtype, None if bias is None else bias.dtype
        return y

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, w32, b32 = ctx.saved_tensors
        dy = dy.to(x.dtype).contiguous()
        B, C, H, W = x.shape
        dx = torch.empty_like(x)
        dw = torch.empty_like(w32)
        db = torch.empty(C, device=x.device, dtype=torch.float32) if ctx.has_bias else None
        _lib.call("mia_dwconv2d_bwd", "dwconv2d_bwd", x.device, x.data_ptr(), w32.data_ptr(), b32.data_ptr() if ctx.has_bias else 0,
                  dy.data_ptr(), dx.data_ptr(), dw.data_ptr(), 0 if db is None else db.data_ptr(), B, C, H, W, int(ctx.silu),
                  _lib.dtype_code(x.dtype))
        return dx, dw.view(C, 1, 3, 3).to(ctx.wdtype), (db.to(ctx.bdtype) if db is not None else None), None


def dwconv2d_silu(x, conv: nn.Conv2d, silu: bool = True):
    """`act(conv2d(x))` for SS2D's depth-wise 3x3 conv; anything else (other kernel sizes / strides) is not this op."""
    return DWConv2dFn.apply(x, conv.weight, conv.bias, silu)


def cross_scan_fwd(x: torch.Tensor) -> torch.Tensor:
    """(B, C, H, W) -> (B, 4, C, H*W): row-major, column-major and their reversals (vmamba.py:28-35)."""
    B, C, H, W = x.shape
    x = x.contiguous()
    xs = x.new_empty((B, 4, C, H * W))
    _cs_call("mia_cross_scan", x, xs, B, C, H, W)
    return xs


def cross_merge_fwd(ys: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """(B, 4, C, H*W) -> (B, C, H*W): adjoint of cross_scan_fwd (vmamba.py:51-57), summed in fp32."""
    B, K, C, L = ys.shape
    ys = ys.contiguous()
    y = ys.new_empty((B, C, L))
    _cs_call("mia_cross_merge", ys, y, B, C, H, W)
    return y


class CrossScan(torch.autograd.Function):
    """vmamba.py:25-45."""

    @staticmethod
    def forward(ctx, x: torch.Tensor):
        B, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        return cross_scan_fwd(x)

    @staticmethod
    def backward(ctx, ys: torch.Tensor):
        B, C, H, W = ctx.shape
        return cross_merge_fwd(ys, H, W).view(B, -1, H, W)


class CrossMerge(torch.autograd.Function):
    """vmamba.py:48-67."""

    @staticmethod
    def forward(ctx, ys: torch.Tensor):
        B, K, D, H, W = ys.shape
        ctx.shape = (H, W)
        return cross_merge_fwd(ys.view(B, K, D, -1), H, W)

    @staticmethod
    def backward(ctx, x: torch.Tensor):
        H, W = ctx.shape
        B, C, L = x.shape
        return cross_scan_fwd(x.view(B, C, H, W)).view(B, 4, C, H, W)


class CrossScan_Ab_2direction(torch.autograd.Function):
    """vmamba.py:71-86: the row-major order and its reversal, twice (no column-major scan)."""

    @staticmethod
    def forward(ctx, x):
        B, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        f = x.reshape(B, 1, C, H * W)
        return torch.cat([f, f, f.flip(-1), f.flip(-1)], dim=1)

    @staticmethod
    def backward(ctx, ys):
        B, C, H, W = ctx.shape
        return (ys[:, 0] + ys[:, 1] + (ys[:, 2] + ys[:, 3]).flip(-1)).view(B, -1, H, W)


class CrossMerge_Ab_2direction(torch.autograd.Function):
    """vmamba.py:89-104."""

    @staticmethod
    def forward(ctx, ys):
        B, K, D, H, W = ys.shape
        ctx.shape = (H, W)
        ys = ys.reshape(B, K, D, -1)
        return ys[:, 0] + ys[:, 1] + (ys[:, 2] + ys[:, 3]).flip(-1)

    @staticmethod
    def backward(ctx, x):
        H, W = ctx.shape
        B, C, L = x.shape
        f = x.reshape(B, 1, C, L)
        return torch.cat([f, f, f.flip(-1), f.flip(-1)], dim=1).view(B, 4, C, H, W)


class CrossScan_Ab_1direction(torch.autograd.Function):
    """vmamba.py:107-119: four copies of the row-major order."""

    @staticmethod
    def forward(ctx, x):
        B, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        return x.reshape(B, 1, C, H * W).repeat(1, 4, 1, 1)

    @staticmethod
    def backward(ctx, ys):
        B, C, H, W = ctx.shape
        return ys.reshape(B, 4, -1, H, W).sum(1)


class CrossMerge_Ab_1direction(torch.autograd.Function):
    """vmamba.py:122-131."""

    @staticmethod
    def forward(ctx, ys):
        B, K, C, H, W = ys.shape
        ctx.shape = (B, C, H, W)
        return ys.reshape(B, 4, -1, H * W).sum(1)

    @staticmethod
    def backward(ctx, x):
        B, C, H, W = ctx.shape
        return x.reshape(B, 1, C, H, W).repeat(1, 4, 1, 1, 1)


def cross_scan_1b1_fwd(x: torch.Tensor) -> torch.Tensor:
    """(B, 4, C, H, W) -> (B, 4, C, H*W): direction k's scan order applied to x[:, k] (csm_triton.py:212-235)."""
    B, K, C, H, W = x.shape
    x = x.contiguous()
    xs = x.new_empty((B, 4, C, H * W))
    _cs_call("mia_cross_scan_1b1", x, xs, B, C, H, W)
    return xs


def cross_merge_1b1_fwd(ys: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """(B, 4, C, H*W) -> (B, 4, C, H, W): adjoint of cross_scan_1b1_fwd (each slice back to image order)."""
    B, K, C, L = ys.shape
    ys = ys.contiguous()
    y = ys.new_empty((B, 4, C, H, W))
    _cs_call("mia_cross_merge_1b1", ys, y, B, C, H, W)
    return y


class CrossScan1b1(torch.autograd.Function):
    """csm_triton.py:212-235 (CrossScanTriton1b1): direction k of the scan applied to its own input x[:, k]."""

    @staticmethod
    def forward(ctx, x):
        B, K, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        return cross_scan_1b1_fwd(x)

    @staticmethod
    def backward(ctx, y):
        B, C, H, W = ctx.shape
        return cross_merge_1b1_fwd(y.reshape(B, 4, C, H * W), H, W)


# the reference's Triton classes (csm_triton.py:163-235) are the same maps as the torch ones (its CHECKS.check_csm_triton):
# here both names resolve to the CUDA kernels
CrossScanTriton, CrossMergeTriton, CrossScanTriton1b1 = CrossScan, CrossMerge, CrossScan1b1


# ---------------------------------------------------------------------------------------------------------
# The SS2D core as one autograd op (DESIGN.md 3.12): x_proj on the unscanned map, dt_proj, CrossScan, the scan, and
# CrossMerge + bf16 cast + LayerNorm + z gate in one kernel (csrc/ss2d_core.cu) whose backward also forms the scan's dout.
_GATE_NONE, _GATE_MUL, _GATE_SILU = 0, 1, 2


def _ln_ok(norm, D):
    return isinstance(norm, nn.LayerNorm) and norm.weight is not None and norm.bias is not None and tuple(norm.normalized_shape) == (D,)


def _tok_view(z, H, W):
    """struct mia_bdl of a channel-last (B, H, W, D) view seen as (B, D, H*W) (d stride 1 or any, token stride uniform)."""
    return _lib.MiaBdl(z.data_ptr(), z.stride(0), z.stride(3), z.stride(2))


class SS2DCoreFn(torch.autograd.Function):
    """cross_selective_scan (v2 / v3 / v4 cores, LayerNorm out_norm, channel-last) followed by SS2D's gate, as ONE op.

    x (B, D, H, W) is the conv output, z (B, H, W, D) the gate input (any view with a uniform token stride, e.g. the second
    half of in_proj's output, read in place) or None.  Forward: Z = x_proj_weight (K C, D) @ x -- a per-token projection
    commutes with the cross-scan permutation, so this is each direction's x_dbl in image order, from one plane instead of
    four -- moved into scan order by mia_cross_scan_1b1; delta = dt_projs_weight @ dts as one batched matmul; the scan on
    xs = CrossScan(x); then mia_ss2d_merge_norm_fwd -> the token-major (B, H, W, D) output.  Saved (checkpoint_lvl 1): x, Z
    (scan order), the bf16 pre-norm plane, the LayerNorm statistics, the scan checkpoints / block states and z; level 0 also
    keeps xs and delta, which level 1 recomputes with the forward's kernels (same bits).  for_backward False (no input needs
    a gradient, or grad mode is off): nothing is kept, and the pre-norm plane, the statistics and the scan's block states are
    not written."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, z, x_proj_weight, dt_projs_weight, As, Ds, delta_bias, ln_weight, ln_bias, eps, gate, force_fp32, out_float,
                delta_softplus, checkpoint_lvl, for_backward):
        from .scan_op import scan_fwd
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not x.is_cuda or x.dtype not in _lib.DTYPE_CODES:
            raise RuntimeError("SS2DCoreFn: x must be a float32 / float16 / bfloat16 CUDA tensor")
        B, D, H, W = x.shape
        K, C, _ = x_proj_weight.shape
        R = dt_projs_weight.shape[2]
        N = (C - R) // 2
        if K != 4 or x_proj_weight.shape[2] != D or tuple(dt_projs_weight.shape) != (K, D, R) or C != R + 2 * N:
            raise RuntimeError(f"SS2DCoreFn: x_proj_weight {tuple(x_proj_weight.shape)} / dt_projs_weight {tuple(dt_projs_weight.shape)} "
                               f"do not fit x {tuple(x.shape)} with 4 cross maps")
        if gate != _GATE_NONE and (z is None or tuple(z.shape) != (B, H, W, D) or z.dtype != x.dtype or z.stride(1) != W * z.stride(2)):
            raise RuntimeError(f"SS2DCoreFn: z must be a (B, H, W, D) = {(B, H, W, D)} {x.dtype} view with a uniform token stride")
        T, dev = x.dtype, x.device
        x = x.contiguous()
        ctx.sizes = (B, D, H, W, K, C, R, N, T, gate, force_fp32, bool(delta_softplus), checkpoint_lvl)
        with torch.autocast("cuda", enabled=False):
            wx = x_proj_weight.to(T)
            Z = torch.bmm(wx.view(K * C, D).expand(B, K * C, D), x.view(B, D, H * W))                   # image order
            Zs = cross_scan_1b1_fwd(Z.view(B, K, C, H, W))                                                 # (B, K, C, L)
            del Z
            xs, delta = SS2DCoreFn._xs_delta(x, Zs, dt_projs_weight, ctx.sizes)
            Bs, Cs = SS2DCoreFn._bc(Zs, ctx.sizes)
            ys, xck, _, *hb = scan_fwd(xs, delta, As, Bs, Cs, Ds, None, delta_bias, delta_softplus, out_float,
                                       want_block_states=for_backward)
            hblk = hb[0] if hb else None
            del Bs, Cs
        w32, b32 = ln_weight.float().contiguous(), ln_bias.float().contiguous()
        out = torch.empty((B, H, W, D), dtype=T, device=dev)
        yb = mean = rstd = None
        if for_backward:
            yb = torch.empty((B, H * W, D), dtype=torch.bfloat16, device=dev)
            mean = torch.empty((B, H * W), dtype=torch.float32, device=dev)
            rstd = torch.empty_like(mean)
        ln = _lib.MiaLn(w32.data_ptr(), b32.data_ptr(), float(eps))
        zb = _tok_view(z, H, W) if gate else _lib.MiaBdl(None, 0, 0, 0)
        ptr = lambda t: None if t is None else t.data_ptr()
        _lib.call("mia_ss2d_merge_norm_fwd", "ss2d_merge_norm_fwd", dev, ys.data_ptr(), ctypes.byref(ln), ctypes.byref(zb), gate,
                  out.data_ptr(), ptr(yb), ptr(mean), ptr(rstd), B, D, H, W, _lib.dtype_code(ys.dtype), _lib.dtype_code(T))
        if not for_backward:
            return out
        keep = [xs, delta] if checkpoint_lvl == 0 else []
        ctx.eps = float(eps)
        ctx.dtypes = (x_proj_weight.dtype, dt_projs_weight.dtype, ln_weight.dtype, ln_bias.dtype)
        ctx.save_for_backward(x, Zs, yb, mean, rstd, xck, hblk, z if gate else None, x_proj_weight, dt_projs_weight, As, Ds, delta_bias,
                              w32, b32, *keep)
        return out

    @staticmethod
    def _xs_delta(x, Zs, dt_projs_weight, sizes):
        """xs = CrossScan(x) (B, 4D, L) and delta = dt_projs_weight @ dts (B, 4D, L); fp32 copies under force_fp32."""
        B, D, H, W, K, C, R, N, T, _, force_fp32, _, _ = sizes
        L = H * W
        xs = cross_scan_fwd(x.view(B, D, H, W)).view(B, K * D, L)
        delta = torch.matmul(dt_projs_weight.to(T), Zs[:, :, :R]).view(B, K * D, L)
        if force_fp32:                                                                   # vmamba.py:400-404
            xs, delta = xs.float(), delta.float()
        return xs, delta

    @staticmethod
    def _bc(Zs, sizes):
        """The scan's B / C: views of Zs (fp32 copies under force_fp32)."""
        R, N, force_fp32 = sizes[6], sizes[7], sizes[10]
        Bs, Cs = Zs[:, :, R:R + N], Zs[:, :, R + N:]
        return (Bs.float(), Cs.float()) if force_fp32 else (Bs, Cs)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        from .scan_op import scan_bwd
        B, D, H, W, K, C, R, N, T, gate, force_fp32, softplus, lvl = ctx.sizes
        L, dev = H * W, dy.device
        x, Zs, yb, mean, rstd, xck, hblk, z, x_proj_weight, dt_projs_weight, As, Ds, delta_bias, w32, b32, *keep = ctx.saved_tensors
        dy = dy.to(T).contiguous()
        dout = torch.empty((B, K, D, L), dtype=torch.float32, device=dev)
        dz = torch.empty((B, H, W, D), dtype=T, device=dev) if gate else None
        dw32, db32 = torch.empty_like(w32), torch.empty_like(b32)
        ws = torch.empty((max(1, int(_lib.lib().mia_ss2d_merge_norm_bwd_workspace(B, D, H, W))),), dtype=torch.uint8, device=dev)
        ln = _lib.MiaLn(w32.data_ptr(), b32.data_ptr(), ctx.eps)
        none = _lib.MiaBdl(None, 0, 0, 0)
        _lib.call("mia_ss2d_merge_norm_bwd", "ss2d_merge_norm_bwd", dev, dy.data_ptr(), yb.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                  ctypes.byref(ln), ctypes.byref(_tok_view(z, H, W) if gate else none), gate,
                  ctypes.byref(_tok_view(dz, H, W) if gate else none), dout.data_ptr(), dw32.data_ptr(), db32.data_ptr(), ws.data_ptr(),
                  ws.numel(), B, D, H, W, _lib.dtype_code(T))
        del dy, ws
        with torch.autocast("cuda", enabled=False):
            xs, delta = keep if lvl == 0 else SS2DCoreFn._xs_delta(x, Zs, dt_projs_weight, ctx.sizes)
            Bs, Cs = SS2DCoreFn._bc(Zs, ctx.sizes)
            du, ddelta, dA, dB, dC, dD, ddb, _ = scan_bwd(xs, delta, As, Bs, Cs, Ds, None, delta_bias, dout.view(B, K * D, L), xck, None,
                                                          softplus, hblk=hblk)
            del dout, xs, delta
            # under force_fp32 the casts' backward brings the gradients back to T (vmamba.py:400-404)
            du, ddelta, dB, dC = du.to(T), ddelta.to(T), dB.to(T), dC.to(T)
            wdt = dt_projs_weight.to(T)
            dd = ddelta.view(B, K, D, L)
            dZs = torch.empty((B, K, C, L), dtype=T, device=dev)
            dZs[:, :, :R] = torch.matmul(wdt.transpose(1, 2), dd)
            dZs[:, :, R:R + N] = dB
            dZs[:, :, R + N:] = dC
            f32 = {} if T == torch.float32 else {"out_dtype": torch.float32}
            dts = Zs[:, :, :R].reshape(B * K, R, L)
            d_wdt = torch.bmm(dd.reshape(B * K, D, L), dts.transpose(1, 2), **f32).view(B, K, D, R).sum(0)
            del dd, ddelta
            dZ = cross_merge_1b1_fwd(dZs, H, W).view(B, K * C, L)                       # back to image order
            dx = cross_merge_fwd(du.view(B, K, D, L), H, W)                              # CrossScan's adjoint, (B, D, L)
            del du
            wx = x_proj_weight.to(T)
            dx.baddbmm_(wx.view(K * C, D).t().contiguous().expand(B, D, K * C), dZ)     # + x_proj_weight^T dZ, in place
            d_wx = torch.bmm(dZ, x.view(B, D, L).transpose(1, 2), **f32).sum(0).view(K, C, D)
        xw_dtype, dtw_dtype, lw_dtype, lb_dtype = ctx.dtypes
        return (dx.view(B, D, H, W), dz, d_wx.to(xw_dtype), d_wdt.to(dtw_dtype), dA, dD, ddb, dw32.to(lw_dtype), db32.to(lb_dtype),
                None, None, None, None, None, None, None)


def ss2d_core(x, z, x_proj_weight, dt_projs_weight, dt_projs_bias, A_logs, Ds, out_norm, gate=_GATE_NONE, force_fp32=False,
              out_float=True, delta_softplus=True, checkpoint_lvl=1):
    """SS2DCoreFn on SS2D's parameters: (B, D, H, W) conv output [+ (B, H, W, D) gate input] -> (B, H, W, D) in x's dtype.
    gate: 0 none, 1 y * z (nozact), 2 y * silu(z).  force_fp32: the v2 core's fp32 scan inputs; out_float: the scan's fp32
    ("oflex") output (v3 / v4)."""
    params = (x, z, x_proj_weight, dt_projs_weight, dt_projs_bias, A_logs, Ds, out_norm.weight, out_norm.bias)
    for_backward = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in params)
    return SS2DCoreFn.apply(x, z, x_proj_weight, dt_projs_weight, -torch.exp(A_logs.float()), Ds.float(), dt_projs_bias.view(-1).float(),
                            out_norm.weight, out_norm.bias, out_norm.eps, gate, force_fp32, out_float, delta_softplus, checkpoint_lvl,
                            for_backward)


_CROSS_MAPS = (CrossScan, CrossMerge)


def cross_selective_scan(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus=True,
                         out_norm=None, out_norm_shape="v0", channel_first=False, to_dtype=True, force_fp32=False,
                         nrows=-1, backnrows=-1, ssoflex=True, SelectiveScan=None, CrossScan=CrossScan, CrossMerge=CrossMerge,
                         no_einsum=False, dt_low_rank=True):
    """vmamba.py:318-427 (the low-rank-dt paths; out_norm is whatever fits (B, L, C) or (B, C, H, W)).  Channel-last with a
    LayerNorm out_norm, the four cross maps, the Oflex / Core scan and CUDA tensors: one fused op (SS2DCoreFn), same
    values; any other configuration: the composition of the reference, _cross_selective_scan_composed."""
    SelectiveScan = SelectiveScan or SelectiveScanOflex
    if (x.is_cuda and dt_low_rank and x_proj_bias is None and not channel_first and to_dtype and out_norm_shape == "v0"
            and _ln_ok(out_norm, x.shape[1]) and (CrossScan, CrossMerge) == _CROSS_MAPS and dt_projs_weight.shape[0] == 4
            and (SelectiveScan is SelectiveScanCore or (SelectiveScan is SelectiveScanOflex and not force_fp32))):
        out_float = bool(ssoflex) if SelectiveScan is SelectiveScanOflex else False
        return ss2d_core(x, None, x_proj_weight, dt_projs_weight, dt_projs_bias, A_logs, Ds, out_norm, 0, force_fp32, out_float,
                         delta_softplus=delta_softplus)
    return _cross_selective_scan_composed(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus,
                                          out_norm, out_norm_shape, channel_first, to_dtype, force_fp32, nrows, backnrows, ssoflex,
                                          SelectiveScan, CrossScan, CrossMerge, no_einsum, dt_low_rank)


def _cross_selective_scan_composed(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus=True,
                                   out_norm=None, out_norm_shape="v0", channel_first=False, to_dtype=True, force_fp32=False,
                                   nrows=-1, backnrows=-1, ssoflex=True, SelectiveScan=None, CrossScan=CrossScan, CrossMerge=CrossMerge,
                                   no_einsum=False, dt_low_rank=True):
    """vmamba.py:318-427 as the reference composes it, on the CrossScan / scan / CrossMerge kernels and torch ops."""
    B, D, H, W = x.shape
    D, N = A_logs.shape
    K, D, R = dt_projs_weight.shape
    L = H * W
    SelectiveScan = SelectiveScan or SelectiveScanOflex

    if not dt_low_rank:                                                                # :372-377 (as written there: the grouped
        x_dbl = F.conv1d(x.view(B, -1, L), x_proj_weight.view(-1, D, 1),               # conv needs K * D input channels)
                         bias=(x_proj_bias.view(-1) if x_proj_bias is not None else None), groups=K)
        dts, Bs, Cs = torch.split(x_dbl.view(B, -1, L), [D, 4 * N, 4 * N], dim=1)
        xs = CrossScan.apply(x)
        dts = CrossScan.apply(dts)
    elif no_einsum:                                                                    # :379-383
        xs = CrossScan.apply(x)
        x_dbl = F.conv1d(xs.view(B, -1, L), x_proj_weight.view(-1, D, 1),
                         bias=(x_proj_bias.view(-1) if x_proj_bias is not None else None), groups=K)
        dts, Bs, Cs = torch.split(x_dbl.view(B, K, -1, L), [R, N, N], dim=2)
        dts = F.conv1d(dts.contiguous().view(B, -1, L), dt_projs_weight.view(K * D, -1, 1), groups=K)
    else:                                                                              # :385-390
        xs = CrossScan.apply(x)
        x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, x_proj_weight)
        if x_proj_bias is not None:
            x_dbl = x_dbl + x_proj_bias.view(1, K, -1, 1)
        dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
        dts = torch.einsum("b k r l, k d r -> b k d l", dts, dt_projs_weight)

    xs = xs.view(B, -1, L)
    dts = dts.contiguous().view(B, -1, L)
    As = -torch.exp(A_logs.to(torch.float))                                            # :394
    Bs = Bs.contiguous().view(B, K, N, L)
    Cs = Cs.contiguous().view(B, K, N, L)
    Ds = Ds.to(torch.float)
    delta_bias = dt_projs_bias.view(-1).to(torch.float)
    if force_fp32:                                                                     # :400-404
        xs, dts, Bs, Cs = xs.to(torch.float), dts.to(torch.float), Bs.to(torch.float), Cs.to(torch.float)

    ys = SelectiveScan.apply(xs, dts, As, Bs, Cs, Ds, delta_bias, delta_softplus, nrows, backnrows, ssoflex).view(B, K, -1, H, W)
    y = CrossMerge.apply(ys)                                                           # :410

    if channel_first:                                                                  # :412-419
        y = y.view(B, -1, H, W)
        if out_norm_shape in ["v1"]:
            y = out_norm(y)
        else:
            y = out_norm(y.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
        return y.to(x.dtype) if to_dtype else y
    y = y.to(torch.bfloat16)                                                           # :420 (unconditional in the reference)
    if not torch.is_autocast_enabled() and isinstance(out_norm, nn.LayerNorm) and out_norm.weight is not None:
        y = y.to(out_norm.weight.dtype)   # the reference only runs this under bf16 autocast; keep the rounding, not the dtype clash
    if out_norm_shape in ["v1"]:
        y = out_norm(y.view(B, -1, H, W)).permute(0, 2, 3, 1)
    else:
        y = out_norm(y.transpose(dim0=1, dim1=2).contiguous()).view(B, H, W, -1)
    return y.to(x.dtype) if to_dtype else y


class Linear2d(nn.Linear):
    """vmamba.py:441-448: a 1x1 conv that loads Linear or Conv2d weights."""

    def forward(self, x: torch.Tensor):
        return F.conv2d(x, self.weight[:, :, None, None], self.bias)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        state_dict[prefix + "weight"] = state_dict[prefix + "weight"].view(self.weight.shape)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class LayerNorm2d(nn.LayerNorm):
    """vmamba.py:451-456."""

    def forward(self, x: torch.Tensor):
        x = x.permute(0, 2, 3, 1)
        x = F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps)
        return x.permute(0, 3, 1, 2)


def _lin(mod: nn.Linear, x: torch.Tensor, act: int = 0) -> torch.Tensor:
    """nn.Linear through the wgmma GEMM for bf16 / fp16 CUDA activations (gemm.linear), F.linear otherwise."""
    if type(mod) is nn.Linear:
        return _gemm.linear(x, mod.weight, mod.bias, act)
    y = mod(x)                                                   # Linear2d (channel-first 1x1 conv)
    return {0: lambda t: t, 1: F.relu, 2: F.gelu, 3: F.silu}[act](y)


def _strip(tag: str, value: str):
    """forward_type postfix parsing of the reference (vmamba.py:699-703)."""
    hit = value.endswith(tag)
    return hit, (value[:-len(tag)] if hit else value)


class _SoftmaxSpatial(nn.Softmax):
    def forward(self, x: torch.Tensor):
        B, C, H, W = x.shape
        return super().forward(x.view(B, C, -1)).view(B, C, H, W)


class SS2D(nn.Module):
    """vmamba.py:540-1215.  One class, three families selected by ``forward_type`` exactly like the reference:
    ``v0*`` (legacy, :589-660 + 1020-1090), ``xv*`` (experimental merged projections, :804-962 + 1131-1215), anything
    else the v2 family (:662-802 + 1092-1129) with its postfix flags (no32 / noz / nozact, none / dwconv3 / softmax /
    sigmoid) and cores v01 / v1 / v2 / v3 / v31d / v32d / v4."""

    def __init__(self, d_model=96, d_state=16, ssm_ratio=2.0, dt_rank="auto", act_layer=nn.SiLU, d_conv=3, conv_bias=True,
                 dropout=0.0, bias=False, dt_min=0.001, dt_max=0.1, dt_init="random", dt_scale=1.0, dt_init_floor=1e-4,
                 initialize="v0", forward_type="v2", channel_first=False, **kwargs):
        super().__init__()
        self.d_inner = d_inner = int(ssm_ratio * d_model)
        self.dt_rank = dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.d_state, self.k_group = d_state, 4
        dt_args = (dt_scale, dt_init, dt_min, dt_max, dt_init_floor)
        if forward_type.startswith("v0"):
            self._build_v0(d_model, d_inner, d_state, dt_rank, dropout, forward_type, channel_first, kwargs.get("force_fp32", True))
        elif forward_type.startswith("xv"):
            self._build_xv(d_model, d_inner, d_state, dt_rank, act_layer, d_conv, conv_bias, dropout, bias, dt_args, initialize,
                           forward_type, channel_first)
        else:
            self._build_v2(d_model, d_inner, d_state, dt_rank, act_layer, d_conv, conv_bias, dropout, bias, dt_args, initialize,
                           forward_type, channel_first)

    # ---- parameter groups shared by the families ---------------------------------------------------------------
    def _init_ssm(self, initialize, d_inner, d_state, dt_rank, dt_args):
        K = self.k_group
        if initialize == "v0":                                                                  # :767-779
            dt_projs = [self.dt_init(dt_rank, d_inner, *dt_args) for _ in range(K)]
            self.dt_projs_weight = nn.Parameter(torch.stack([t.weight for t in dt_projs], dim=0))   # (K, inner, rank)
            self.dt_projs_bias = nn.Parameter(torch.stack([t.bias for t in dt_projs], dim=0))       # (K, inner)
            self.A_logs = self.A_log_init(d_state, d_inner, copies=K, merge=True)                     # (K * D, N)
            self.Ds = self.D_init(d_inner, copies=K, merge=True)                                      # (K * D)
        elif initialize == "v1":                                                                # :780-785
            self.Ds = nn.Parameter(torch.ones(K * d_inner))
            self.A_logs = nn.Parameter(torch.randn(K * d_inner, d_state))
            self.dt_projs_weight = nn.Parameter(torch.randn(K, d_inner, dt_rank))
            self.dt_projs_bias = nn.Parameter(torch.randn(K, d_inner))
        elif initialize == "v2":                                                                # :786-791
            self.Ds = nn.Parameter(torch.ones(K * d_inner))
            self.A_logs = nn.Parameter(torch.zeros(K * d_inner, d_state))
            self.dt_projs_weight = nn.Parameter(0.1 * torch.rand(K, d_inner, dt_rank))
            self.dt_projs_bias = nn.Parameter(0.1 * torch.rand(K, d_inner))
        else:
            raise NotImplementedError(initialize)

    def _pick_out_norm(self, forward_type, d_inner, channel_first):
        """postfix -> (out_norm, out_norm_shape, remaining forward_type); :705-727."""
        self.out_norm_shape = "v1"
        for tag, make in (("none", nn.Identity), ("dwconv3", lambda: nn.Conv2d(d_inner, d_inner, 3, padding=1, groups=d_inner, bias=False)),
                          ("softmax", lambda: _SoftmaxSpatial(dim=-1)), ("sigmoid", nn.Sigmoid)):
            hit, forward_type = _strip(tag, forward_type)
            if hit:
                self.out_norm = make()
                return forward_type
        if channel_first:
            self.out_norm = LayerNorm2d(d_inner)
        else:
            self.out_norm_shape = "v0"
            self.out_norm = nn.LayerNorm(d_inner)
        return forward_type

    # ---- v0 ------------------------------------------------------------------------------------------------------
    def _build_v0(self, d_model, d_inner, d_state, dt_rank, dropout, forward_type, channel_first, force_fp32):
        if channel_first:
            raise AssertionError("forward_type v0 is channel-last only")                         # :606-607
        self.channel_first, self.d_conv = False, 3
        self._v0_seq, self._v0_fp32 = "seq" in forward_type, force_fp32
        self.forward = self.forwardv0
        self.in_proj = nn.Linear(d_model, d_inner * 2, bias=False)
        self.act = nn.SiLU()
        self.conv2d = nn.Conv2d(d_inner, d_inner, groups=d_inner, bias=True, kernel_size=3, padding=1)
        x_proj = [nn.Linear(d_inner, dt_rank + d_state * 2, bias=False) for _ in range(self.k_group)]
        self.x_proj_weight = nn.Parameter(torch.stack([t.weight for t in x_proj], dim=0))
        self._init_ssm("v0", d_inner, d_state, dt_rank, (1.0, "random", 0.001, 0.1, 1e-4))
        self.out_norm = nn.LayerNorm(d_inner)
        self.out_proj = nn.Linear(d_inner, d_model, bias=False)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()

    def forwardv0(self, x: torch.Tensor, SelectiveScan=SelectiveScanMamba, **kwargs):
        """vmamba.py:1020-1090: the four directions built with torch ops in the reference; here CrossScan / CrossMerge kernels
        (identical maps), the scan through ``SelectiveScanMamba`` (fp32 inputs by default), LayerNorm, gate, out_proj."""
        seq, force_fp32 = kwargs.get("seq", self._v0_seq), kwargs.get("force_fp32", self._v0_fp32)
        x = _lin(self.in_proj, x)
        x, z = x.chunk(2, dim=-1)
        z = self.act(z)
        x = self._conv_act(x.permute(0, 3, 1, 2).contiguous())
        B, D, H, W = x.shape
        N, (K, _, R), L = self.A_logs.shape[1], self.dt_projs_weight.shape, H * W
        xs = CrossScan.apply(x)                                                                 # :1036-1037
        x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, self.x_proj_weight)
        dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
        dts = torch.einsum("b k r l, k d r -> b k d l", dts, self.dt_projs_weight)
        xs, dts = xs.view(B, -1, L), dts.contiguous().view(B, -1, L)
        Bs, Cs = Bs.contiguous(), Cs.contiguous()
        As, Ds, bias = -torch.exp(self.A_logs.float()), self.Ds.float(), self.dt_projs_bias.float().view(-1)
        if force_fp32:
            xs, dts, Bs, Cs = xs.float(), dts.float(), Bs.float(), Cs.float()
        if seq:                                                                                 # :1061-1071: one direction at a time
            ys = torch.stack([SelectiveScan.apply(xs.view(B, K, -1, L)[:, i], dts.view(B, K, -1, L)[:, i], As.view(K, -1, N)[i],
                                                  Bs[:, i].unsqueeze(1), Cs[:, i].unsqueeze(1), Ds.view(K, -1)[i], bias.view(K, -1)[i],
                                                  True, 1, False).view(B, -1, L) for i in range(4)], dim=1)
        else:
            ys = SelectiveScan.apply(xs, dts, As, Bs, Cs, Ds, bias, True, 1, False).view(B, K, -1, L)
        if ys.dtype != torch.float:
            raise AssertionError("forwardv0 expects an fp32 scan output")                       # :1079
        y = CrossMerge.apply(ys.view(B, K, -1, H, W))                                           # :1081-1084
        y = self.out_norm(y.transpose(1, 2).contiguous()).view(B, H, W, -1)
        return self.dropout(_lin(self.out_proj, y * z))

    # ---- v2 ------------------------------------------------------------------------------------------------------
    def _build_v2(self, d_model, d_inner, d_state, dt_rank, act_layer, d_conv, conv_bias, dropout, bias, dt_args, initialize, forward_type,
                  channel_first):
        self.d_conv, self.channel_first = d_conv, channel_first
        Linear = Linear2d if channel_first else nn.Linear
        self.disable_force32, forward_type = _strip("no32", forward_type)
        self.disable_z, forward_type = _strip("noz", forward_type)
        self.disable_z_act, forward_type = _strip("nozact", forward_type)
        forward_type = self._pick_out_norm(forward_type, d_inner, channel_first)
        core = self.forward_corev2
        cores = dict(                                                                           # :730-743
            v01=partial(core, force_fp32=(not self.disable_force32), SelectiveScan=SelectiveScanMamba),
            v2=partial(core, force_fp32=(not self.disable_force32), SelectiveScan=SelectiveScanCore),
            v3=partial(core, force_fp32=False, SelectiveScan=SelectiveScanOflex),
            v31d=partial(core, force_fp32=False, SelectiveScan=SelectiveScanOflex, CrossScan=CrossScan_Ab_1direction, CrossMerge=CrossMerge_Ab_1direction),
            v32d=partial(core, force_fp32=False, SelectiveScan=SelectiveScanOflex, CrossScan=CrossScan_Ab_2direction, CrossMerge=CrossMerge_Ab_2direction),
            v4=partial(core, force_fp32=False, SelectiveScan=SelectiveScanOflex, no_einsum=True, CrossScan=CrossScanTriton, CrossMerge=CrossMergeTriton),
            v1=partial(core, force_fp32=True, SelectiveScan=SelectiveScanOflex),
        )
        self.forward_core = cores.get(forward_type, None)       # an unknown type fails at the first forward, as in the reference
        self._core_type = forward_type
        self.in_proj = Linear(d_model, d_inner if self.disable_z else d_inner * 2, bias=bias)
        self.act = act_layer()
        if d_conv > 1:
            self.conv2d = nn.Conv2d(d_inner, d_inner, groups=d_inner, bias=conv_bias, kernel_size=d_conv, padding=(d_conv - 1) // 2)
        x_proj = [nn.Linear(d_inner, dt_rank + d_state * 2, bias=False) for _ in range(self.k_group)]
        self.x_proj_weight = nn.Parameter(torch.stack([t.weight for t in x_proj], dim=0))      # (K, R + 2N, inner)
        self.out_proj = Linear(d_inner, d_model, bias=bias)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        self._init_ssm(initialize, d_inner, d_state, dt_rank, dt_args)

    def _conv_act(self, x):
        """`act(conv2d(x))` on a channel-first map: the fused depth-wise 3x3 + SiLU kernel where it applies."""
        if self.d_conv == 3 and isinstance(self.act, nn.SiLU) and x.is_cuda and x.shape[1] == self.conv2d.weight.shape[0]:
            return dwconv2d_silu(x, self.conv2d, True)
        if self.d_conv > 1:
            x = self.conv2d(x)
        return self.act(x)

    def forward_corev2(self, x: torch.Tensor, cross_selective_scan=cross_selective_scan, **kwargs):
        """vmamba.py:1092-1108."""
        return cross_selective_scan(x, self.x_proj_weight, None, self.dt_projs_weight, self.dt_projs_bias, self.A_logs, self.Ds,
                                    delta_softplus=True, out_norm=getattr(self, "out_norm", None), channel_first=self.channel_first,
                                    out_norm_shape=getattr(self, "out_norm_shape", "v0"), **kwargs)

    def _fused_core_args(self, x):
        """(gate, force_fp32, out_float) when this configuration runs as SS2DCoreFn, else None."""
        if (self.channel_first or self.out_norm_shape != "v0" or not _ln_ok(self.out_norm, self.d_inner) or self.k_group != 4
                or self._core_type not in ("v2", "v3", "v4") or not x.is_cuda):
            return None
        if self.disable_z:
            gate = _GATE_NONE
        elif self.disable_z_act:
            gate = _GATE_MUL
        elif isinstance(self.act, nn.SiLU):
            gate = _GATE_SILU
        else:
            return None
        return (gate, not self.disable_force32, False) if self._core_type == "v2" else (gate, False, True)

    def forward(self, x: torch.Tensor, **kwargs):
        """vmamba.py:1110-1129 (forwardv2); eligible configurations (see _fused_core_args) run the core as SS2DCoreFn."""
        fused = self._fused_core_args(x)
        if fused is None:
            return self._forward_composed(x, **kwargs)
        gate, force_fp32, out_float = fused
        x = _lin(self.in_proj, x)
        z = None
        if gate != _GATE_NONE:
            x, z = x.chunk(2, dim=-1)
        x = self._conv_act(x.permute(0, 3, 1, 2).contiguous())
        y = ss2d_core(x, z, self.x_proj_weight, self.dt_projs_weight, self.dt_projs_bias, self.A_logs, self.Ds, self.out_norm, gate,
                      force_fp32, out_float)
        return self.dropout(_lin(self.out_proj, y))

    def _forward_composed(self, x: torch.Tensor, **kwargs):
        """vmamba.py:1110-1129 as the reference composes it (the core through _cross_selective_scan_composed)."""
        x = _lin(self.in_proj, x)
        if not self.disable_z:
            x, z = x.chunk(2, dim=(1 if self.channel_first else -1))
            if not self.disable_z_act:
                z = self.act(z)
        if not self.channel_first:
            x = x.permute(0, 3, 1, 2).contiguous()
        x = self._conv_act(x)
        y = self.forward_core(x, cross_selective_scan=_cross_selective_scan_composed)
        if not self.disable_z:
            y = y * z
        return self.dropout(_lin(self.out_proj, y))

    forwardv2 = forward

    # ---- xv ------------------------------------------------------------------------------------------------------
    def _build_xv(self, d_model, d_inner, d_state, dt_rank, act_layer, d_conv, conv_bias, dropout, bias, dt_args, initialize, forward_type,
                  channel_first):
        self.d_conv, self.channel_first = d_conv, channel_first
        Linear = Linear2d if channel_first else nn.Linear
        self.disable_force32, forward_type = _strip("no32", forward_type)
        forward_type = self._pick_out_norm(forward_type, d_inner, channel_first)
        self.act, self.out_act = act_layer(), nn.Identity()
        conv1 = lambda c: nn.Conv2d(d_model, c, 1, bias=bias)
        mode = "xv1"                                                                            # :873-913, applied in the same order
        if forward_type.startswith("xv1"):
            self.in_proj = conv1(d_inner + dt_rank + 8 * d_state)
        if forward_type.startswith("xv2") or forward_type.startswith("xv5"):
            raise AttributeError("'SS2D' object has no attribute 'dt_projs_weight' (the reference's xv2 / xv5 constructors delete "
                                 "dt_projs_weight before creating it, vmamba.py:888, 903: these types cannot be built there either)")
        if forward_type.startswith("xv3"):
            mode, self.in_proj = "xv3", conv1(d_inner + 4 * dt_rank + 8 * d_state)
        if forward_type.startswith("xv4"):
            mode, self.in_proj, self.out_act = "xv3", conv1(d_inner + 4 * dt_rank + 8 * d_state), nn.GELU()
        if forward_type.startswith("xv6"):
            mode, self.in_proj, self.out_act = "xv1", conv1(d_inner + dt_rank + 8 * d_state), nn.GELU()
        if forward_type.startswith("xv61"):
            mode, self.in_proj, self.out_act = "xv1", Linear2d(d_model, d_inner + dt_rank + 8 * d_state, bias=bias), nn.GELU()
        if forward_type.startswith("xv7"):
            mode, self.in_proj, self.out_act = "xv7", Linear2d(d_model, d_inner + dt_rank + 8 * d_state, bias=bias), nn.GELU()
        self.forward = partial(self.forwardxv, mode=mode)
        if d_conv > 1:                                                                          # on d_model channels, BEFORE in_proj (:916-925)
            self.conv2d = nn.Conv2d(d_model, d_model, groups=d_model, bias=conv_bias, kernel_size=d_conv, padding=(d_conv - 1) // 2)
        self.out_proj = Linear(d_inner, d_model, bias=bias)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        self._init_ssm(initialize, d_inner, d_state, dt_rank, dt_args)

    def forwardxv(self, x: torch.Tensor, mode="xv1", **kwargs):
        """vmamba.py:1131-1215: conv + act on the block input, ONE projection producing u, dt and all four directions' B / C."""
        if not self.channel_first:
            x = x.permute(0, 3, 1, 2).contiguous()
        B, C, H, W = x.shape
        L, K, N, R, Di = H * W, 4, self.d_state, self.dt_rank, self.d_inner
        if self.d_conv > 1:
            x = self._conv_act(x)
        x = self.in_proj(x)
        dtw = getattr(self, "dt_projs_weight", None)
        if mode in ("xv1", "xv7"):
            _us, dts, Bs, Cs = x.split([Di, R, 4 * N, 4 * N], dim=1)
            us = CrossScanTriton.apply(_us.contiguous()).view(B, -1, L)
            dts = CrossScanTriton.apply(dts.contiguous()).view(B, -1, L)
            dts = F.conv1d(dts, dtw.view(K * Di, R, 1), None, groups=K).contiguous().view(B, -1, L)
        elif mode == "xv3":
            _us, dts, Bs, Cs = x.split([Di, 4 * R, 4 * N, 4 * N], dim=1)
            us = CrossScanTriton.apply(_us.contiguous()).view(B, -1, L)
            dts = CrossScanTriton1b1.apply(dts.contiguous().view(B, K, -1, H, W))
            dts = F.conv1d(dts.view(B, -1, L), dtw.view(K * Di, R, 1), None, groups=K).contiguous().view(B, -1, L)
        else:
            raise NotImplementedError(f"forwardxv mode {mode!r}")
        Bs, Cs = Bs.view(B, K, -1, L).contiguous(), Cs.view(B, K, -1, L).contiguous()
        As, Ds, bias = -torch.exp(self.A_logs.to(torch.float)), self.Ds.to(torch.float), self.dt_projs_bias.view(-1).to(torch.float)
        ys = SelectiveScanOflex.apply(us, dts, As, Bs, Cs, Ds, bias, True, 1, 1, True).view(B, K, -1, H, W)
        y = CrossMergeTriton.apply(ys).view(B, -1, H, W)
        if (not self.channel_first) or (self.out_norm_shape == "v0"):                          # :1200-1205
            y = self.out_norm(y.permute(0, 2, 3, 1))
            if self.channel_first:
                y = y.permute(0, 3, 1, 2)
        else:
            y = self.out_norm(y)
        y = self.out_act(y.to(x.dtype))
        if mode == "xv7":
            y = y * (_us.permute(0, 2, 3, 1) if not self.channel_first else _us)
        return self.dropout(self.out_proj(y))

    # ---- initialisers (static, as in the reference) ----------------------------------------------------------------
    @staticmethod
    def dt_init(dt_rank, d_inner, dt_scale=1.0, dt_init="random", dt_min=0.001, dt_max=0.1, dt_init_floor=1e-4):
        """vmamba.py:964-989: dt_proj whose bias is softplus^-1 of a log-uniform dt in [dt_min, dt_max]."""
        dt_proj = nn.Linear(dt_rank, d_inner, bias=True)
        std = dt_rank ** -0.5 * dt_scale
        if dt_init == "constant":
            nn.init.constant_(dt_proj.weight, std)
        elif dt_init == "random":
            nn.init.uniform_(dt_proj.weight, -std, std)
        else:
            raise NotImplementedError(dt_init)
        dt = torch.exp(torch.rand(d_inner) * (math.log(dt_max) - math.log(dt_min)) + math.log(dt_min)).clamp(min=dt_init_floor)
        inv_dt = dt + torch.log(-torch.expm1(-dt))
        with torch.no_grad():
            dt_proj.bias.copy_(inv_dt)
        return dt_proj

    @staticmethod
    def A_log_init(d_state, d_inner, copies=-1, device=None, merge=True):
        """vmamba.py:991-1005: S4D-real, A = -(1..N)."""
        A_log = torch.log(torch.arange(1, d_state + 1, dtype=torch.float32, device=device)).repeat(d_inner, 1)
        if copies > 0:
            A_log = A_log.unsqueeze(0).repeat(copies, 1, 1)
            if merge:
                A_log = A_log.flatten(0, 1)
        A_log = nn.Parameter(A_log.contiguous())
        A_log._no_weight_decay = True
        return A_log

    @staticmethod
    def D_init(d_inner, copies=-1, device=None, merge=True):
        """vmamba.py:1007-1017."""
        D = torch.ones(d_inner, device=device)
        if copies > 0:
            D = D.unsqueeze(0).repeat(copies, 1)
            if merge:
                D = D.flatten(0, 1)
        D = nn.Parameter(D)
        D._no_weight_decay = True
        return D


# ---------------------------------------------------------------------------------------------------------
# Callers of SS2D (vmamba.py:458-537, 1218-1725).  Stock torch modules around the accelerated block; the MLP matmuls go
# through the wgmma GEMM with the activation fused into its epilogue when the activations are bf16 / fp16.
class DropPath(nn.Module):
    """timm.models.layers.DropPath (stochastic depth per sample), which vmamba.py:14 imports."""

    def __init__(self, drop_prob: float = 0.0, scale_by_keep: bool = True):
        super().__init__()
        self.drop_prob, self.scale_by_keep = drop_prob, scale_by_keep

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1.0 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        if keep > 0.0 and self.scale_by_keep:
            mask.div_(keep)
        return x * mask

    def extra_repr(self):
        return f"drop_prob={self.drop_prob}"


class Permute(nn.Module):
    def __init__(self, *args):
        super().__init__()
        self.args = args

    def forward(self, x: torch.Tensor):
        return x.permute(*self.args)


class PatchMerging2D(nn.Module):
    """vmamba.py:458-483: 2x2 neighbourhood concat -> norm -> Linear(4 dim, 2 dim)."""

    def __init__(self, dim, out_dim=-1, norm_layer=nn.LayerNorm):
        super().__init__()
        self.dim = dim
        self.reduction = nn.Linear(4 * dim, (2 * dim) if out_dim < 0 else out_dim, bias=False)
        self.norm = norm_layer(4 * dim)

    @staticmethod
    def _patch_merging_pad(x: torch.Tensor):
        H, W, _ = x.shape[-3:]
        if (W % 2 != 0) or (H % 2 != 0):
            x = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
        return torch.cat([x[..., 0::2, 0::2, :], x[..., 1::2, 0::2, :], x[..., 0::2, 1::2, :], x[..., 1::2, 1::2, :]], -1)

    def forward(self, x):
        return _lin(self.reduction, self.norm(self._patch_merging_pad(x)))


_ACT_CODE = {nn.ReLU: 1, nn.GELU: 2, nn.SiLU: 3}


class Mlp(nn.Module):
    """vmamba.py:495-514.  Channel-last with exact GELU, when a backward follows and no dropout is active, the layer runs as
    one op (gemm.gelu_mlp_fn); every other case runs the composition, _forward_composed (no-grad inference included, which
    already has the GELU in fc1's epilogue)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0, channels_first=False):
        super().__init__()
        out_features, hidden_features = out_features or in_features, hidden_features or in_features
        Linear = Linear2d if channels_first else nn.Linear
        self.fc1 = Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        if _gemm.gelu_mlp_eligible(self, x, self.drop.p == 0 or not self.training):
            return self.drop(_gemm.gelu_mlp_fn(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias))
        return self._forward_composed(x)

    def _forward_composed(self, x):
        code = _ACT_CODE.get(type(self.act), None)
        if code in (1, 2) and type(self.fc1) is nn.Linear:      # activation fused into the GEMM epilogue
            x = _lin(self.fc1, x, code)
        else:
            x = self.act(_lin(self.fc1, x))
        return self.drop(_lin(self.fc2, self.drop(x)))


class gMlp(nn.Module):
    """vmamba.py:517-535."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0, channels_first=False):
        super().__init__()
        self.channel_first = channels_first
        out_features, hidden_features = out_features or in_features, hidden_features or in_features
        Linear = Linear2d if channels_first else nn.Linear
        self.fc1 = Linear(in_features, 2 * hidden_features)
        self.act = act_layer()
        self.fc2 = Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def forward(self, x: torch.Tensor):
        x, z = _lin(self.fc1, x).chunk(2, dim=(1 if self.channel_first else -1))
        return self.drop(_lin(self.fc2, x * self.act(z)))


class VSSBlock(nn.Module):
    """vmamba.py:1218-1302: x + drop_path(SS2D(norm(x))); x + drop_path(mlp(norm2(x))) (or post-norm)."""

    def __init__(self, hidden_dim: int = 0, drop_path: float = 0, norm_layer=nn.LayerNorm, channel_first=False, ssm_d_state: int = 16,
                 ssm_ratio=2.0, ssm_dt_rank="auto", ssm_act_layer=nn.SiLU, ssm_conv: int = 3, ssm_conv_bias=True, ssm_drop_rate: float = 0,
                 ssm_init="v0", forward_type="v2", mlp_ratio=4.0, mlp_act_layer=nn.GELU, mlp_drop_rate: float = 0.0, gmlp=False,
                 use_checkpoint: bool = False, post_norm: bool = False, **kwargs):
        super().__init__()
        self.ssm_branch, self.mlp_branch = ssm_ratio > 0, mlp_ratio > 0
        self.use_checkpoint, self.post_norm = use_checkpoint, post_norm
        if self.ssm_branch:
            self.norm = norm_layer(hidden_dim)
            self.op = SS2D(d_model=hidden_dim, d_state=ssm_d_state, ssm_ratio=ssm_ratio, dt_rank=ssm_dt_rank, act_layer=ssm_act_layer,
                           d_conv=ssm_conv, conv_bias=ssm_conv_bias, dropout=ssm_drop_rate, initialize=ssm_init, forward_type=forward_type,
                           channel_first=channel_first)
        self.drop_path = DropPath(drop_path)
        if self.mlp_branch:
            self.norm2 = norm_layer(hidden_dim)
            self.mlp = (gMlp if gmlp else Mlp)(in_features=hidden_dim, hidden_features=int(hidden_dim * mlp_ratio), act_layer=mlp_act_layer,
                                               drop=mlp_drop_rate, channels_first=channel_first)

    def _forward(self, input: torch.Tensor):
        x = input
        if self.ssm_branch:
            x = input + self.drop_path(self.norm(self.op(input)) if self.post_norm else self.op(self.norm(input)))
        if self.mlp_branch:
            x = x + self.drop_path(self.norm2(self.mlp(x)) if self.post_norm else self.mlp(self.norm2(x)))
        return x

    def forward(self, input: torch.Tensor):
        return checkpoint.checkpoint(self._forward, input, use_reentrant=True) if self.use_checkpoint else self._forward(input)


class VSSM(nn.Module):
    """vmamba.py:1305-1668: patch embed -> stages of VSSBlocks with v3 down-sampling between them -> (optional) pooled features."""

    def __init__(self, patch_size=4, in_chans=3, num_classes=1000, depths=[2, 2, 9, 2], dims=[96, 192, 384, 768], ssm_d_state=16,
                 ssm_ratio=2.0, ssm_dt_rank="auto", ssm_act_layer="silu", ssm_conv=3, ssm_conv_bias=True, ssm_drop_rate=0.0, ssm_init="v0",
                 forward_type="v2", mlp_ratio=4.0, mlp_act_layer="gelu", mlp_drop_rate=0.0, gmlp=False, drop_path_rate=0.1, patch_norm=True,
                 norm_layer="LN", downsample_version: str = "v2", patchembed_version: str = "v1", use_checkpoint=False, **kwargs):
        super().__init__()
        self.channel_first = norm_layer.lower() in ["bn", "ln2d"]
        self.num_classes, self.num_layers = num_classes, len(depths)
        if isinstance(dims, int):
            dims = [int(dims * 2 ** i) for i in range(self.num_layers)]
        self.num_features, self.dims = dims[-1], dims
        dpr = [v.item() for v in torch.linspace(0, drop_path_rate, sum(depths))]
        norm_cls = dict(ln=nn.LayerNorm, ln2d=LayerNorm2d, bn=nn.BatchNorm2d).get(norm_layer.lower(), None)
        acts = dict(silu=nn.SiLU, gelu=nn.GELU, relu=nn.ReLU, sigmoid=nn.Sigmoid)
        ssm_act, mlp_act = acts.get(ssm_act_layer.lower(), None), acts.get(mlp_act_layer.lower(), None)
        make_embed = dict(v1=self._make_patch_embed, v2=self._make_patch_embed_v2).get(patchembed_version, None)
        self.patch_embed = make_embed(in_chans, dims[0], patch_size, patch_norm, norm_cls, channel_first=self.channel_first)
        self.layers = nn.ModuleList()
        for i in range(self.num_layers):
            # the reference resolves `downsample_version` (:1371-1376) but then always builds the v3 module (:1379-1384)
            down = self._make_downsample_v3(dims[i], dims[i + 1], norm_layer=norm_cls, channel_first=self.channel_first) \
                if i < self.num_layers - 1 else nn.Identity()
            self.layers.append(self._make_layer(
                dim=dims[i], drop_path=dpr[sum(depths[:i]):sum(depths[:i + 1])], use_checkpoint=use_checkpoint, norm_layer=norm_cls,
                downsample=down, channel_first=self.channel_first, ssm_d_state=ssm_d_state, ssm_ratio=ssm_ratio, ssm_dt_rank=ssm_dt_rank,
                ssm_act_layer=ssm_act, ssm_conv=ssm_conv, ssm_conv_bias=ssm_conv_bias, ssm_drop_rate=ssm_drop_rate, ssm_init=ssm_init,
                forward_type=forward_type, mlp_ratio=mlp_ratio, mlp_act_layer=mlp_act, mlp_drop_rate=mlp_drop_rate, gmlp=gmlp))
        self.classifier = nn.Sequential(OrderedDict(
            norm=norm_cls(self.num_features), permute=(Permute(0, 3, 1, 2) if not self.channel_first else nn.Identity()),
            avgpool=nn.AdaptiveAvgPool2d(1), flatten=nn.Flatten(1)))     # the reference has no head here (:1412)
        self.apply(self._init_weights)

    def _init_weights(self, m: nn.Module):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @staticmethod
    def _make_patch_embed(in_chans=3, embed_dim=96, patch_size=4, patch_norm=True, norm_layer=nn.LayerNorm, channel_first=False):
        return nn.Sequential(nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size, bias=True),
                             (nn.Identity() if channel_first else Permute(0, 2, 3, 1)),
                             (norm_layer(embed_dim) if patch_norm else nn.Identity()))

    @staticmethod
    def _make_patch_embed_v2(in_chans=3, embed_dim=96, patch_size=4, patch_norm=True, norm_layer=nn.LayerNorm, channel_first=False):
        assert patch_size == 4
        keep = channel_first or (not patch_norm)
        return nn.Sequential(nn.Conv2d(in_chans, embed_dim // 2, kernel_size=3, stride=2, padding=1),
                             (nn.Identity() if keep else Permute(0, 2, 3, 1)),
                             (norm_layer(embed_dim // 2) if patch_norm else nn.Identity()),
                             (nn.Identity() if keep else Permute(0, 3, 1, 2)),
                             nn.GELU(),
                             nn.Conv2d(embed_dim // 2, embed_dim, kernel_size=3, stride=2, padding=1),
                             (nn.Identity() if channel_first else Permute(0, 2, 3, 1)),
                             (norm_layer(embed_dim) if patch_norm else nn.Identity()))

    @staticmethod
    def _make_downsample(dim=96, out_dim=192, norm_layer=nn.LayerNorm, channel_first=False):
        return nn.Sequential((nn.Identity() if channel_first else Permute(0, 3, 1, 2)), nn.Conv2d(dim, out_dim, kernel_size=2, stride=2),
                             (nn.Identity() if channel_first else Permute(0, 2, 3, 1)), norm_layer(out_dim))

    @staticmethod
    def _make_downsample_v3(dim=96, out_dim=192, norm_layer=nn.LayerNorm, channel_first=False):
        return nn.Sequential((nn.Identity() if channel_first else Permute(0, 3, 1, 2)),
                             nn.Conv2d(dim, out_dim, kernel_size=3, stride=2, padding=1),
                             (nn.Identity() if channel_first else Permute(0, 2, 3, 1)), norm_layer(out_dim))

    @staticmethod
    def _make_layer(dim=96, drop_path=[0.1, 0.1], use_checkpoint=False, norm_layer=nn.LayerNorm, downsample=nn.Identity(),
                    channel_first=False, **block_kwargs):
        blocks = [VSSBlock(hidden_dim=dim, drop_path=dp, norm_layer=norm_layer, channel_first=channel_first, use_checkpoint=use_checkpoint,
                           **block_kwargs) for dp in drop_path]
        return nn.Sequential(OrderedDict(blocks=nn.Sequential(*blocks), downsample=downsample))

    def forward(self, x: torch.Tensor, global_features=False, featuremap_folder=None):
        if featuremap_folder is not None:
            raise NotImplementedError("the matplotlib feature-map dump of the reference (vmamba.py:1540-1596) is a debugging aid, not part of the path")
        x = self.patch_embed(x)
        for layer in self.layers:
            x = layer(x)
        return self.classifier(x) if global_features else x

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        """Key renames of older VMamba checkpoints (vmamba.py:1633-1668)."""
        def rename(src, dst):
            key = prefix + src
            for k in list(state_dict.keys()):
                if k.startswith(key):
                    state_dict[prefix + dst + k[len(key):]] = state_dict.pop(k)
        rename("patch_embed.proj", "patch_embed.0")
        rename("patch_embed.norm", "patch_embed.2")
        for i in range(len(self.layers)):
            for j in range(len(self.layers[i].blocks)):
                rename(f"layers.{i}.blocks.{j}.ln_1", f"layers.{i}.blocks.{j}.norm")
                rename(f"layers.{i}.blocks.{j}.self_attention", f"layers.{i}.blocks.{j}.op")
        rename("norm", "classifier.norm")
        rename("head", "classifier.head")
        return super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


class Backbone_VSSM(VSSM):
    """vmamba.py:1672-1725: per-stage normalised feature maps (B, C, H, W) for detection / segmentation heads."""

    def __init__(self, out_indices=(0, 1, 2, 3), pretrained=None, norm_layer="ln", **kwargs):
        kwargs.update(norm_layer=norm_layer)
        super().__init__(**kwargs)
        norm_cls = dict(ln=nn.LayerNorm, ln2d=LayerNorm2d, bn=nn.BatchNorm2d).get(norm_layer.lower(), None)
        self.out_indices = out_indices
        for i in out_indices:
            self.add_module(f"outnorm{i}", norm_cls(self.dims[i]))
        del self.classifier
        self.load_pretrained(pretrained)

    def load_pretrained(self, ckpt=None, key="model"):
        if ckpt is None:
            return
        try:
            state = torch.load(open(ckpt, "rb"), map_location=torch.device("cpu"))
            print(f"Successfully load ckpt {ckpt}")
            print(self.load_state_dict(state[key], strict=False))
        except Exception as e:
            print(f"Failed loading checkpoint form {ckpt}: {e}")

    def forward(self, x):
        x = self.patch_embed(x)
        outs = []
        for i, layer in enumerate(self.layers):
            o = layer.blocks(x)
            x = layer.downsample(o)
            if i in self.out_indices:
                out = getattr(self, f"outnorm{i}")(o)
                outs.append(out if self.channel_first else out.permute(0, 3, 1, 2).contiguous())
        return x if len(self.out_indices) == 0 else outs
