"""ARM / Vim encoders of the MambaXray-VL, EMRRG and AM_MRG sub-projects on the H100 kernels.

Mirrors ``*/arm/Finetuning/mamba_simple.py`` (``Mamba``, :35-804) and ``models_mamba.py`` (``PatchEmbed`` :32-56, ``SwiGLU``
:59-83, ``Block`` :86-129, ``create_block`` :132-164, ``ARM`` :215-394, ``arm_{base,large,huge}_pz16`` :398-436): same
constructor arguments, same parameter names and shapes (``A_log``, ``D``, ``conv1d``, ``x_proj``, ``dt_proj`` and their
``_b`` / ``_c`` / ``_c_b`` / ``_d`` / ``_d_b`` direction copies), so the published MambaXray-VL checkpoints load unchanged.

What runs where: every scan is ``selective_scan_fn`` (CUDA, with the z gate), the depth-wise conv + SiLU is the CUDA
``causal_conv1d_fn``, in_proj / out_proj / the patch embedding go through the wgmma GEMM for bf16 / fp16 activations, and
so does the SwiGLU MLP, as one autograd op (SwiGLUFn: w1 and w2 in one GEMM with the gate in its epilogue); the
four-direction (v3) mixer is one autograd op (MambaV3Fn, the scan orders as index maps in the kernels),
and the six-direction (v4) orchestration is the reference's, stated once over a table of directions.  Parity: tests/golden/modules_arm.npz holds the outputs of the reference's
own modules (its fused ops evaluated by its own slow path, see tests/golden/make_golden_modules.py).
"""
from __future__ import annotations

import ctypes
import math
from functools import partial
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, gemm as _gemm
from .layernorm import RMSNorm, layer_norm_fn, rms_norm_fn
from .selective_scan_interface import (_bdl, _bwd, _fwd, _mm_nn, _mm_tn, _mm_wgrad, _ops, _tm, _tm_buffer, causal_conv1d_fn,
                                       causal_conv1d_update, mamba_inner_fn, mamba_inner_fn_no_out_proj, bimamba_inner_fn, selective_scan_fn,
                                       selective_state_update)
from .vmamba import DropPath

# direction suffixes per bimamba_type: parameter sets created besides the base one (mamba_simple.py:130-389)
_EXTRA_SETS = {"none": (), "None": (), "v1": (), "v2": ("_b",), "v3": ("_b", "_c", "_c_b"), "v4": ("_b", "_c", "_c_b", "_d", "_d_b")}


def _s4d_A_log(d_inner, d_state, device=None):
    return torch.log(torch.arange(1, d_state + 1, dtype=torch.float32, device=device)).repeat(d_inner, 1).contiguous()


# ---------------------------------------------------------------------------------------------------------
# The four-direction (bimamba v3) mixer as one autograd op.  DESIGN.md section 3.13.
_V3_ORDERS = (_lib.MIA_ORDER_SEQ, _lib.MIA_ORDER_SEQ_REV, _lib.MIA_ORDER_COL, _lib.MIA_ORDER_COL_REV)   # "", _b, _c, _c_b


def _square_grid(L):
    """True when the L - 1 tokens around the middle cls token form a square grid (the column orders need one)."""
    side = math.isqrt(max(L - 1, 0))
    return L >= 2 and side * side == L - 1


def _orders(codes):
    return (ctypes.c_int * len(codes))(*codes)


class MambaV3Fn(torch.autograd.Function):
    """ARM's v3 mixer (mamba_simple.py:447-531: four scans over the token orders identity, reversed, column-major with the
    middle cls token kept in place, and its reverse, summed, / 4, out_proj) as ONE op.  The orders are index maps inside
    the conv and gate kernels (csrc/causal_conv1d.cu, mia_*_dirs), so xz is never re-ordered or copied: the conv writes all
    four directions' scan input u (b, 4 d, L) in one launch, ONE scan runs over 4 d rows with 4 B / C groups, and the gate
    sums the four outputs at each token's scan positions, gates with silu(z) and scales by 1/4 in one launch, rounding once.

    Saved (checkpoint_lvl 1): xz, the four x_dbl, the scan's out (b, 4 d, L), B / C, the scan checkpoints and the
    parameters; level 0 also keeps u and delta.  The backward recomputes the rest with the forward's kernels, so both
    levels give the same bits."""

    @staticmethod
    @_fwd
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, dt_proj_weight, dt_proj_bias, A, D, out_proj_weight, out_proj_bias,
                checkpoint_lvl):
        from .scan_op import scan_fwd
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not xz.is_cuda:
            raise RuntimeError("mamba_v3_fn: this build has no CPU path (xz must be a CUDA tensor)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else xz.dtype
        if T not in _lib.DTYPE_CODES:
            raise RuntimeError("mamba_v3_fn: xz must be float32, float16 or bfloat16")
        xz = xz.to(T)
        b, d2, L = xz.shape
        d, n = d2 // 2, len(_V3_ORDERS)
        W = conv1d_weight.shape[-1]
        R, N = dt_proj_weight.shape[-1], A.shape[-1]
        K = R + 2 * N
        if not _square_grid(L):
            raise RuntimeError(f"mamba_v3_fn: the column orders need seqlen - 1 to be a square, got seqlen {L}")
        if (conv1d_weight.shape[0] != n or tuple(x_proj_weight.shape) != (n, K, d) or tuple(dt_proj_weight.shape) != (n, d, R)
                or tuple(A.shape) != (n, d, N) or tuple(D.shape) != (n, d) or tuple(dt_proj_bias.shape) != (n, d)):
            raise RuntimeError(f"mamba_v3_fn: the parameters must be stacked over {n} directions for d_inner {d}: x_proj "
                               f"{tuple(x_proj_weight.shape)}, dt_proj {tuple(dt_proj_weight.shape)}, A {tuple(A.shape)}, D {tuple(D.shape)}")
        dev = xz.device
        w32 = conv1d_weight.detach().reshape(n, d, W).float().contiguous()
        cb32 = None if conv1d_bias is None else conv1d_bias.detach().reshape(n, d).float().contiguous()
        A32 = A.float().reshape(n * d, N).contiguous()
        D32 = D.float().reshape(n * d).contiguous()
        db32 = dt_proj_bias.float().reshape(n * d).contiguous()
        wx, wdt = x_proj_weight.to(T), dt_proj_weight.to(T)
        ctx.sizes = (b, d, L, W, R, N, K, T, n, checkpoint_lvl)

        u = torch.empty((b, n * d, L), dtype=T, device=dev)
        u_tm = [_tm_buffer(b * L, d, T, dev) for _ in range(n)]
        MambaV3Fn._conv(xz, w32, cb32, ctx, _V3_ORDERS, u, u_tm)
        x_dbl = [_mm_tn(u_tm[k], wx[k]) for k in range(n)]                             # (b l, R + 2N) per direction, scan order
        del u_tm
        delta = MambaV3Fn._delta(x_dbl, wdt, ctx)
        Bs = torch.stack([x.view(b, L, K)[:, :, R:R + N].transpose(1, 2) for x in x_dbl], 1)        # (b, 4, N, L): small
        Cs = torch.stack([x.view(b, L, K)[:, :, R + N:].transpose(1, 2) for x in x_dbl], 1)
        out, x_ck, _ = scan_fwd(u, delta, A32, Bs, Cs, D32, None, db32, True)
        y_tm = MambaV3Fn._gate(out, xz, ctx)
        y = _mm_tn(y_tm, out_proj_weight.to(T), out_proj_bias).view(b, L, -1)
        keep = [u, delta] if checkpoint_lvl == 0 else []
        ctx.save_for_backward(xz, out, Bs, Cs, x_ck, w32, cb32, x_proj_weight, dt_proj_weight, out_proj_weight, A32, D32, db32, *x_dbl, *keep)
        ctx.dtypes = (conv1d_weight.dtype, None if conv1d_bias is None else conv1d_bias.dtype, D.dtype, dt_proj_bias.dtype,
                      None if out_proj_bias is None else out_proj_bias.dtype)
        ctx.shapes = (conv1d_weight.shape, A.shape)
        ctx.has_ob = out_proj_bias is not None
        return y

    @staticmethod
    def _conv(xz, w32, cb32, ctx, orders, u, u_tm):
        """conv + SiLU of xz's x half for every direction of `orders` (w32 / cb32 their stacked taps) in one launch -> u
        (b, len(orders) d, L) and / or the token-major u_tm[k], both in scan order."""
        b, d, L, W, *_ = ctx.sizes
        T = ctx.sizes[7]
        tm = None if u_tm is None else _ops(*[_tm(t, L) for t in u_tm])[0]
        _lib.call("mia_causal_conv1d_fwd_dirs", "causal_conv1d_fwd_dirs", xz.device, ctypes.byref(_bdl(xz[:, :d])), _orders(orders),
                  len(orders), w32.data_ptr(), None if cb32 is None else cb32.data_ptr(), None if u is None else u.data_ptr(), tm, b, d, L,
                  W, 1, _lib.dtype_code(T))

    @staticmethod
    def _delta(x_dbl, wdt, ctx):
        """delta (b, 4 d, L) = dt_proj_k @ dt_k of every direction as one batched matmul."""
        b, d, L, W, R, N, K, T, n, _ = ctx.sizes
        dts = torch.stack([x.view(b, L, K)[:, :, :R].transpose(1, 2) for x in x_dbl], 1)          # (b, 4, R, L): small
        return torch.matmul(wdt, dts).view(b, n * d, L)

    @staticmethod
    def _gate(out, xz, ctx):
        """silu(z) (sum of the four outputs at each token's scan positions) / 4, token-major for out_proj."""
        b, d, L, W, R, N, K, T, n, _ = ctx.sizes
        y_tm = _tm_buffer(b * L, d, T, xz.device)
        _lib.call("mia_silu_gate_fwd_dirs", "silu_gate_fwd_dirs", xz.device, out.data_ptr(), _orders(_V3_ORDERS), n, n,
                  ctypes.byref(_bdl(xz[:, d:])), ctypes.byref(_tm(y_tm, L)), b, d, L, _lib.dtype_code(T))
        return y_tm

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        from .scan_op import scan_bwd
        b, d, L, W, R, N, K, T, n, lvl = ctx.sizes
        xz, out, Bs, Cs, x_ck, w32, cb32, x_proj_weight, dt_proj_weight, out_proj_weight, A32, D32, db32, *rest = ctx.saved_tensors
        x_dbl, keep = rest[:n], rest[n:]
        dev = xz.device
        wx, wdt, wout = x_proj_weight.to(T), dt_proj_weight.to(T), out_proj_weight.to(T)
        dy2 = dy.to(T).reshape(b * L, -1).contiguous()                               # (b l, d_model)
        y_tm = MambaV3Fn._gate(out, xz, ctx)
        d_out_w = _mm_wgrad(dy2, y_tm).to(out_proj_weight.dtype)
        d_out_b = dy2.sum(0, dtype=torch.float32).to(ctx.dtypes[4]) if ctx.has_ob else None
        del y_tm
        g_tm = _mm_nn(dy2, wout)                                                     # (b l, d): d of the gate's output
        dxz = torch.empty_like(xz)
        dout = torch.empty((b, n * d, L), dtype=torch.float32, device=dev)          # unrounded, as when the scan gates itself
        _lib.call("mia_silu_gate_bwd_dirs", "silu_gate_bwd_dirs", dev, ctypes.byref(_tm(g_tm, L)), out.data_ptr(), _orders(_V3_ORDERS), n, n,
                  ctypes.byref(_bdl(xz[:, d:])), dout.data_ptr(), ctypes.byref(_bdl(dxz[:, d:])), b, d, L, _lib.dtype_code(T))
        del g_tm
        if lvl == 0:
            u, delta = keep
        else:
            u = torch.empty((b, n * d, L), dtype=T, device=dev)
            MambaV3Fn._conv(xz, w32, cb32, ctx, _V3_ORDERS, u, None)
            delta = MambaV3Fn._delta(x_dbl, wdt, ctx)
        du, dd, dA, dB, dC, dD, ddb, _ = scan_bwd(u, delta, A32, Bs, Cs, D32, None, db32, dout, x_ck, None, True)
        del dout, u, delta
        f32 = {} if T == torch.float32 else {"out_dtype": torch.float32}             # fp32 partials per batch element
        dd3 = dd.view(b * n, d, L)
        dts = torch.stack([x.view(b, L, K)[:, :, :R] for x in x_dbl], 1).view(b * n, L, R)
        d_wdt = torch.bmm(dd3, dts, **f32).view(b, n, d, R).sum(0)                      # (4, d, R)
        ddt = torch.bmm(dd3.transpose(1, 2), wdt.expand(b, n, d, R).reshape(b * n, d, R)).view(b, n, L, R)
        del dd, dd3, dts
        Kp = (K + 7) // 8 * 8
        wx_p = wx if Kp == K else torch.cat([wx, wx.new_zeros(n, Kp - K, d)], 1)
        d_wx, dy_tm = [], []
        u_tm = _tm_buffer(b * L, d, T, dev)
        for k in range(n):
            dx_dbl = torch.zeros((b * L, Kp), dtype=T, device=dev)
            dxd = dx_dbl.view(b, L, Kp)
            dxd[:, :, :R] = ddt[:, k]
            dxd[:, :, R:R + N] = dB[:, k].transpose(1, 2)
            dxd[:, :, R + N:K] = dC[:, k].transpose(1, 2)
            # x_proj's input of this direction, recomputed at both levels (one buffer for the four)
            MambaV3Fn._conv(xz, w32[k], None if cb32 is None else cb32[k], ctx, _V3_ORDERS[k:k + 1], None, [u_tm])
            d_wx.append(_mm_wgrad(dx_dbl[:, :K], u_tm).to(x_proj_weight.dtype))
            dy_tm.append(_mm_nn(dx_dbl, wx_p[k]) if T != torch.float32 else dx_dbl[:, :K] @ wx[k])    # (b l, d)
        del u_tm, ddt, dB, dC
        dw32 = torch.empty_like(w32)
        dcb32 = torch.empty_like(cb32) if cb32 is not None else None
        ws = torch.empty((max(1, int(_lib.lib().mia_causal_conv1d_bwd_dirs_workspace(n, b, d, L, W))),), dtype=torch.uint8, device=dev)
        _lib.call("mia_causal_conv1d_bwd_dirs", "causal_conv1d_bwd_dirs", dev, ctypes.byref(_bdl(xz[:, :d])), _orders(_V3_ORDERS), n,
                  w32.data_ptr(), None if cb32 is None else cb32.data_ptr(), du.data_ptr(), _ops(*[_tm(t, L) for t in dy_tm])[0],
                  ctypes.byref(_bdl(dxz[:, :d])), dw32.data_ptr(), None if dcb32 is None else dcb32.data_ptr(), ws.data_ptr(), ws.numel(),
                  b, d, L, W, 1, _lib.dtype_code(T))
        cw_dtype, cb_dtype, D_dtype, db_dtype, _ = ctx.dtypes
        conv_shape, A_shape = ctx.shapes
        return (dxz, dw32.view(conv_shape).to(cw_dtype), None if dcb32 is None else dcb32.to(cb_dtype), torch.stack(d_wx),
                d_wdt.to(dt_proj_weight.dtype), ddb.view(n, d).to(db_dtype), dA.view(A_shape), dD.view(n, d).to(D_dtype), d_out_w, d_out_b,
                None)


def mamba_v3_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, dt_proj_weight, dt_proj_bias, A, D, out_proj_weight, out_proj_bias=None,
                checkpoint_lvl=1):
    """ARM's four-direction (bimamba_type "v3") mixer after in_proj: xz (b, 2 d_inner, L) -> (b, L, d_model).

    The directions' parameters are stacked on a leading axis in the order "", "_b", "_c", "_c_b": conv1d_weight
    (4, d_inner, 1, width), conv1d_bias (4, d_inner) or None, x_proj_weight (4, dt_rank + 2 d_state, d_inner),
    dt_proj_weight (4, d_inner, dt_rank), dt_proj_bias (4, d_inner), A = -exp(A_log) (4, d_inner, d_state), D (4, d_inner).
    L - 1 must be a square (the image tokens around the middle cls token at L // 2).  checkpoint_lvl 0 keeps the scan's
    input and delta for the backward, 1 (default) recomputes them; both give the same bits."""
    return MambaV3Fn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, dt_proj_weight, dt_proj_bias, A, D, out_proj_weight, out_proj_bias,
                           checkpoint_lvl)


class Mamba(nn.Module):
    """The ARM / Vim mixer (mamba_simple.py:35-715)."""

    def __init__(self, d_model, d_state=16, d_conv=4, expand=2, dt_rank="auto", dt_min=0.001, dt_max=0.1, dt_init="random", dt_scale=1.0,
                 dt_init_floor=1e-4, conv_bias=True, bias=False, use_fast_path=True, layer_idx=None, device=None, dtype=None,
                 bimamba_type="none", if_devide_out=False, init_layer_scale=None):
        fk = {"device": device, "dtype": dtype}
        super().__init__()
        self.d_model, self.d_state, self.d_conv, self.expand = d_model, d_state, d_conv, expand
        self.d_inner = int(expand * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.use_fast_path, self.layer_idx, self.bimamba_type, self.if_devide_out = use_fast_path, layer_idx, bimamba_type, if_devide_out
        self.init_layer_scale = init_layer_scale
        if init_layer_scale is not None:
            self.gamma = nn.Parameter(init_layer_scale * torch.ones(d_model), requires_grad=True)
        self.in_proj = nn.Linear(d_model, self.d_inner * 2, bias=bias, **fk)
        self.activation, self.act = "silu", nn.SiLU()

        def direction(sfx):
            """conv1d / x_proj / dt_proj / A_log / D of one scan direction under the reference's attribute names."""
            setattr(self, "conv1d" + sfx, nn.Conv1d(self.d_inner, self.d_inner, bias=conv_bias, kernel_size=d_conv, groups=self.d_inner,
                                                    padding=d_conv - 1, **fk))
            setattr(self, "x_proj" + sfx, nn.Linear(self.d_inner, self.dt_rank + d_state * 2, bias=False, **fk))
            setattr(self, "dt_proj" + sfx, nn.Linear(self.dt_rank, self.d_inner, bias=True, **fk))
            A = nn.Parameter(_s4d_A_log(self.d_inner, d_state, device))
            A._no_weight_decay = True
            setattr(self, "A" + sfx + "_log", A)
            D = nn.Parameter(torch.ones(self.d_inner, device=device))
            D._no_weight_decay = True
            setattr(self, "D" + sfx, D)

        direction("")
        # only the base dt_proj gets the variance-preserving init and the inverse-softplus bias (mamba_simple.py:97-115)
        std = self.dt_rank ** -0.5 * dt_scale
        if dt_init == "constant":
            nn.init.constant_(self.dt_proj.weight, std)
        elif dt_init == "random":
            nn.init.uniform_(self.dt_proj.weight, -std, std)
        else:
            raise NotImplementedError
        dt = torch.exp(torch.rand(self.d_inner, **fk) * (math.log(dt_max) - math.log(dt_min)) + math.log(dt_min)).clamp(min=dt_init_floor)
        with torch.no_grad():
            self.dt_proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))
        self.dt_proj.bias._no_reinit = True
        if bimamba_type == "v1":                                      # Vim: a second A only (:131-139)
            self.A_b_log = nn.Parameter(_s4d_A_log(self.d_inner, d_state, device))
            self.A_b_log._no_weight_decay = True
        for sfx in _EXTRA_SETS.get(bimamba_type, ()):
            direction(sfx)
        self.out_proj = nn.Linear(self.d_inner, d_model, bias=bias, **fk)

    # ------------------------------------------------------------------------------------------------------------
    def _dir_args(self, sfx):
        """positional arguments of mamba_inner_fn_no_out_proj for direction `sfx` (mamba_simple.py:450-462)."""
        dt_proj = getattr(self, "dt_proj" + sfx)
        return (getattr(self, "conv1d" + sfx).weight, getattr(self, "conv1d" + sfx).bias, getattr(self, "x_proj" + sfx).weight, dt_proj.weight,
                -torch.exp(getattr(self, "A" + sfx + "_log").float()), None, None, getattr(self, "D" + sfx).float()), \
            dict(delta_bias=dt_proj.bias.float(), delta_softplus=True)

    def _scan_dir(self, xz, sfx):
        args, kw = self._dir_args(sfx)
        return mamba_inner_fn_no_out_proj(xz, *args, **kw)

    @staticmethod
    def _col_major(t, pos):
        """(B, D, L) with the cls token at `pos`: re-order the other L - 1 tokens of the square grid column-major, keeping
        the cls token where it is (mamba_simple.py:476-482; its own inverse, :520-524)."""
        B, D, L = t.shape
        side = int(math.sqrt(L))
        cls = t[:, :, pos:pos + 1]
        grid = torch.cat([t[:, :, :pos], t[:, :, pos + 1:]], dim=-1).reshape(B, D, side, side).permute(0, 1, 3, 2).reshape(B, D, -1)
        return torch.cat((grid[:, :, :pos], cls, grid[:, :, pos:]), dim=-1)

    def _in_proj(self, h):
        """`in_proj.weight @ h` laid out (B, 2 d_inner, L) (mamba_simple.py:408-414)."""
        xz = _gemm.linear(h, self.in_proj.weight, None).transpose(1, 2)
        if self.in_proj.bias is not None:
            xz = xz + self.in_proj.bias.to(dtype=xz.dtype).view(1, -1, 1)
        return xz

    def _forward_v3_fused(self, xz, checkpoint_lvl=1):
        """The v3 mixer after in_proj as one op (mamba_v3_fn) on this layer's four parameter sets, stacked under autograd."""
        sfx = ("", "_b", "_c", "_c_b")
        part = lambda name: [getattr(self, name.format(s)) for s in sfx]
        stack = lambda ts: torch.stack(list(ts))
        cb = part("conv1d{}")
        return mamba_v3_fn(xz, stack(c.weight for c in cb), None if cb[0].bias is None else stack(c.bias for c in cb),
                           stack(p.weight for p in part("x_proj{}")), stack(p.weight for p in part("dt_proj{}")),
                           stack(p.bias for p in part("dt_proj{}")), -torch.exp(stack(part("A{}_log")).float()), stack(part("D{}")),
                           self.out_proj.weight, self.out_proj.bias, checkpoint_lvl)

    def _forward_v3_composed(self, xz, xd, seqlen):
        """v3 / v4 (mamba_simple.py:447-531 / :533-648) composed from one mamba_inner_fn_no_out_proj per direction and the
        reference's flips and column-major re-orders -> (out, out_d (v4) | None).  v4 runs here, and so does a v3 layer whose
        L - 1 is not a square, which fails in the re-order's reshape as the reference does."""
        pos = seqlen // 2
        xc = self._col_major(xz, pos)
        out = self._scan_dir(xz, "") + self._scan_dir(xz.flip([-1]), "_b").flip([-1])
        out_c = self._col_major(self._scan_dir(xc, "_c") + self._scan_dir(xc.flip([-1]), "_c_b").flip([-1]), pos)
        if self.bimamba_type == "v3":
            return _gemm.linear(((out + out_c) / 4.0).transpose(1, 2), self.out_proj.weight, self.out_proj.bias), None
        out_dd = self._scan_dir(xd, "_d") + self._scan_dir(xd.flip([-1]), "_d_b").flip([-1])
        out = _gemm.linear(((out + out_c + out_dd) / 6.0).transpose(1, 2), self.out_proj.weight, self.out_proj.bias)
        return out, _gemm.linear((out_dd / 2.0).transpose(1, 2), self.out_proj.weight, self.out_proj.bias)

    def forward(self, hidden_states, segmenttation_features=None, inference_params=None):
        """hidden_states (B, L, D) -> same shape; bimamba v4 returns (out, out_d).  mamba_simple.py:392-715.

        With ``inference_params`` (mamba_ssm.utils.generation.InferenceParams) the call decodes, as the reference does
        (:399-405, 666-707): at ``seqlen_offset == 0`` the un-fused path runs over the prompt, uni-directionally whatever
        ``bimamba_type`` is, and leaves the layer's conv / SSM states in the cache; after that every call is one ``step``."""
        batch, seqlen, _ = hidden_states.shape
        conv_state = ssm_state = None
        if inference_params is not None:
            conv_state, ssm_state = self._get_states_from_cache(inference_params, batch)
            if inference_params.seqlen_offset > 0:
                out, _, _ = self.step(hidden_states, conv_state, ssm_state)     # the states are updated in place
                return out
        xz = self._in_proj(hidden_states)
        xd = self._in_proj(segmenttation_features) if segmenttation_features is not None else None
        out_d = None
        bt = self.bimamba_type
        fast = self.use_fast_path and inference_params is None                       # :428: the fast path outputs no states
        if fast and bt == "v1":                                             # :430-446
            out = bimamba_inner_fn(xz, self.conv1d.weight, self.conv1d.bias, self.x_proj.weight, self.dt_proj.weight, self.out_proj.weight,
                                   self.out_proj.bias, -torch.exp(self.A_log.float()), -torch.exp(self.A_b_log.float()), None, None,
                                   self.D.float(), delta_bias=self.dt_proj.bias.float(), delta_softplus=True)
        elif fast and bt == "v3" and xz.is_cuda and _square_grid(seqlen):   # :447-531 as one op
            out = self._forward_v3_fused(xz)
        elif fast and bt in ("v3", "v4"):                                   # :447-531 / :533-648
            out, out_d = self._forward_v3_composed(xz, xd, seqlen)
        elif fast:                                                                        # :649-663
            args, kw = self._dir_args("")
            out = mamba_inner_fn(xz, args[0], args[1], args[2], args[3], self.out_proj.weight, self.out_proj.bias, *args[4:], **kw)
        else:                                                                             # :664-709: the un-fused statement
            x, z = xz.chunk(2, dim=1)
            if conv_state is not None:                                                    # F.pad also truncates when seqlen > d_conv
                conv_state.copy_(F.pad(x, (self.d_conv - x.shape[-1], 0)))
            x = causal_conv1d_fn(x=x, weight=self.conv1d.weight.squeeze(1), bias=self.conv1d.bias, activation=self.activation)
            x_dbl = self.x_proj(x.transpose(1, 2).reshape(-1, self.d_inner))
            dt, B, C = torch.split(x_dbl, [self.dt_rank, self.d_state, self.d_state], dim=-1)
            dt = (self.dt_proj.weight @ dt.t()).view(self.d_inner, batch, seqlen).transpose(0, 1)
            B = B.view(batch, seqlen, -1).transpose(1, 2).contiguous()
            C = C.view(batch, seqlen, -1).transpose(1, 2).contiguous()
            y = selective_scan_fn(x, dt, -torch.exp(self.A_log.float()), B, C, self.D.float(), z=z, delta_bias=self.dt_proj.bias.float(),
                                  delta_softplus=True, return_last_state=ssm_state is not None)
            if ssm_state is not None:
                y, last_state = y
                ssm_state.copy_(last_state)
            out = self.out_proj(y.transpose(1, 2))
        if self.init_layer_scale is not None:
            out = out * self.gamma
        return (out, out_d) if bt == "v4" else out

    def step(self, hidden_states, conv_state, ssm_state):
        """One decoding token (mamba_simple.py:717-762): hidden_states (B, 1, D) -> (out (B, 1, D), conv_state, ssm_state), the
        states updated in place by the decode-step kernels (causal_conv1d_update, selective_state_update)."""
        assert hidden_states.shape[1] == 1, "Only support decoding with 1 token at a time for now"
        xz = self.in_proj(hidden_states.squeeze(1))                                       # (B, 2 d_inner)
        x, z = xz.chunk(2, dim=-1)
        x = causal_conv1d_update(x, conv_state, self.conv1d.weight.squeeze(1), self.conv1d.bias, self.activation)
        x_db = self.x_proj(x)
        dt, B, C = torch.split(x_db, [self.dt_rank, self.d_state, self.d_state], dim=-1)
        dt = F.linear(dt, self.dt_proj.weight)                                            # dt_bias is added in the kernel
        A = -torch.exp(self.A_log.float())
        y = selective_state_update(ssm_state, x, dt, A, B, C, self.D, z=z, dt_bias=self.dt_proj.bias, dt_softplus=True)
        return self.out_proj(y).unsqueeze(1), conv_state, ssm_state

    def allocate_inference_cache(self, batch_size, max_seqlen, dtype=None, **kwargs):
        """mamba_simple.py:764-776."""
        dev = self.out_proj.weight.device
        conv_state = torch.zeros(batch_size, self.d_model * self.expand, self.d_conv, device=dev, dtype=dtype or self.conv1d.weight.dtype)
        ssm_state = torch.zeros(batch_size, self.d_model * self.expand, self.d_state, device=dev, dtype=dtype or self.dt_proj.weight.dtype)
        return conv_state, ssm_state

    def _get_states_from_cache(self, inference_params, batch_size, initialize_states=False):
        """mamba_simple.py:777-803: this layer's (conv_state, ssm_state) in inference_params.key_value_memory_dict, created
        zeroed on first use in the dtypes of the conv1d / dt_proj weights."""
        assert self.layer_idx is not None
        cache = inference_params.key_value_memory_dict
        if self.layer_idx not in cache:
            conv_state = torch.zeros(batch_size, self.d_model * self.expand, self.d_conv, device=self.conv1d.weight.device,
                                     dtype=self.conv1d.weight.dtype)
            ssm_state = torch.zeros(batch_size, self.d_model * self.expand, self.d_state, device=self.dt_proj.weight.device,
                                    dtype=self.dt_proj.weight.dtype)
            cache[self.layer_idx] = (conv_state, ssm_state)
        else:
            conv_state, ssm_state = cache[self.layer_idx]
            if initialize_states:
                conv_state.zero_()
                ssm_state.zero_()
        return conv_state, ssm_state


# ---------------------------------------------------------------------------------------------------------
class PatchEmbed(nn.Module):
    """models_mamba.py:32-56: kernel == stride patch projection, flattened to (B, N, C).  For bf16 / fp16 inputs with
    stride == patch the conv IS a GEMM over non-overlapping patches and runs on the wgmma kernel."""

    def __init__(self, img_size=224, patch_size=16, stride=16, in_chans=3, embed_dim=768, norm_layer=None, flatten=True):
        super().__init__()
        two = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)
        self.img_size, self.patch_size = two(img_size), two(patch_size)
        self.grid_size = ((self.img_size[0] - self.patch_size[0]) // stride + 1, (self.img_size[1] - self.patch_size[1]) // stride + 1)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.flatten = flatten
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=self.patch_size, stride=stride)
        self.norm = norm_layer(embed_dim) if norm_layer else nn.Identity()

    def forward(self, x):
        B, C, H, W = x.shape
        assert H == self.img_size[0] and W == self.img_size[1], \
            f"Input image size ({H}*{W}) doesn't match model ({self.img_size[0]}*{self.img_size[1]})."
        x = _gemm.conv2d_patch(x, self.proj.weight, self.proj.bias, self.proj.stride)
        if self.flatten:
            x = x.flatten(2).transpose(1, 2)
        return self.norm(x)


# ---------------------------------------------------------------------------------------------------------
# The SwiGLU MLP as one autograd op.  DESIGN.md section 3.14.
def _pad64(n):
    return (n + 63) // 64 * 64


class SwiGLUFn(torch.autograd.Function):
    """w3(silu(w1(x)) * w2(x)) (models_mamba.py:59-83 with subln=False) as ONE op on the wgmma GEMM: w1 and w2 run as one
    GEMM whose tile pairs their rows, so a = w1(x) and b = w2(x) meet in one thread and the epilogue writes the hidden
    h = silu(a) b (mia_gemm_swiglu_fwd); w3 reads h in place.  The backward's w3 dgrad writes da / db and the recomputed h
    from its epilogue (mia_gemm_swiglu_bwd); dx and [dW1; dW2] are one GEMM each over the packed (M, 2 Hp) gradient.

    Saved (checkpoint_lvl 0): x in the activation dtype and the packed a / b (M, 2 Hp); level 1 keeps x only and reruns the
    forward kernel for a / b.  Both give the same bits.  Hp = H rounded up to 64; with nothing to differentiate, nothing is
    saved and a / b are not written."""

    @staticmethod
    @_fwd
    def forward(ctx, x, w1, b1, w2, b2, w3, b3, checkpoint_lvl, train):
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not x.is_cuda:
            raise RuntimeError("swiglu_fn: this build has no CPU path (x must be a CUDA tensor)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else x.dtype
        if T not in (torch.bfloat16, torch.float16):
            raise RuntimeError(f"swiglu_fn: activations must be bfloat16 or float16, directly or under autocast (got {T})")
        H, K = w1.shape
        N = w3.shape[0]
        if tuple(w2.shape) != (H, K) or tuple(w3.shape) != (N, H) or x.shape[-1] != K:
            raise RuntimeError(f"swiglu_fn: shapes do not chain: x {tuple(x.shape)}, w1 {tuple(w1.shape)}, w2 {tuple(w2.shape)}, w3 {tuple(w3.shape)}")
        if K % 8 or N % 8:
            raise RuntimeError(f"swiglu_fn: in_features ({K}) and out_features ({N}) must be multiples of 8")
        lead = x.shape[:-1]
        x2 = x.to(T).reshape(-1, K)
        if not _gemm._mn_ok(x2):
            x2 = x2.contiguous()
        M, Hp = x2.shape[0], _pad64(H)
        if M == 0:
            raise RuntimeError("swiglu_fn: empty input")
        ctx.sizes = (M, H, Hp, K, N, T, checkpoint_lvl)
        ab = torch.empty((M, 2 * Hp), dtype=T, device=x.device) if train else None
        h = torch.empty((M, Hp), dtype=T, device=x.device)
        SwiGLUFn._gate(x2, w1, b1, w2, b2, ab, h, ctx)
        w3p = SwiGLUFn._w3(w3, ctx)
        y = torch.empty((M, N), dtype=T, device=x.device)
        b3f = None if b3 is None else b3.detach().float().contiguous()
        _lib.call("mia_gemm_tn", "swiglu_fn w3", x.device, h.data_ptr(), w3p.data_ptr(), None if b3f is None else b3f.data_ptr(), y.data_ptr(),
                  M, N, H, h.stride(0), w3p.stride(0), y.stride(0), _lib.dtype_code(T), _lib.dtype_code(T), _gemm.ACT_NONE)
        if train:
            ctx.save_for_backward(x2, w1, b1, w2, b2, w3, *([ab] if checkpoint_lvl == 0 else []))
            ctx.bias_dtypes = tuple(None if b is None else b.dtype for b in (b1, b2, b3))
        return y.view(*lead, N)

    @staticmethod
    def _gate(x2, w1, b1, w2, b2, ab, h, ctx):
        """mia_gemm_swiglu_fwd: h = silu(a) b and, when ab is given, the packed a / b."""
        M, H, Hp, K, N, T, _ = ctx.sizes
        w1c, w2c = w1.to(T).contiguous(), w2.to(T).contiguous()
        b1f, b2f = (None if b is None else b.detach().float().contiguous() for b in (b1, b2))
        _lib.call("mia_gemm_swiglu_fwd", "swiglu_fn", x2.device, x2.data_ptr(), w1c.data_ptr(), w2c.data_ptr(),
                  None if b1f is None else b1f.data_ptr(), None if b2f is None else b2f.data_ptr(), h.data_ptr(),
                  None if ab is None else ab.data_ptr(), M, H, K, x2.stride(0), w1c.stride(0), w2c.stride(0), h.stride(0),
                  0 if ab is None else ab.stride(0), _lib.dtype_code(T))

    @staticmethod
    def _w3(w3, ctx):
        """W3 in the activation dtype with a row pitch that is a multiple of 8 (zero-padded to Hp columns when H is not)."""
        M, H, Hp, K, N, T, _ = ctx.sizes
        if H % 8 == 0:
            return w3.to(T).contiguous()
        w3p = torch.zeros((N, Hp), dtype=T, device=w3.device)
        w3p[:, :H] = w3
        return w3p

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        M, H, Hp, K, N, T, lvl = ctx.sizes
        x2, w1, b1, w2, b2, w3, *keep = ctx.saved_tensors
        dev = x2.device
        need_x, need_w1, need_b1, need_w2, need_b2, need_w3, need_b3 = ctx.needs_input_grad[:7]
        dy2 = dy.to(T).reshape(M, N)
        if not _gemm._mn_ok(dy2):
            dy2 = dy2.contiguous()
        h = torch.empty((M, Hp), dtype=T, device=dev) if need_w3 or lvl == 1 else None
        if lvl == 0:
            ab = keep[0]
        else:                                                      # rerun the forward kernel: a / b and h, bit for bit
            ab = torch.empty((M, 2 * Hp), dtype=T, device=dev)
            SwiGLUFn._gate(x2, w1, b1, w2, b2, ab, h, ctx)
        w3p = SwiGLUFn._w3(w3, ctx)
        dab = torch.empty((M, 2 * Hp), dtype=T, device=dev)
        h_bwd = h if lvl == 0 else None
        _lib.call("mia_gemm_swiglu_bwd", "swiglu_fn backward", dev, dy2.data_ptr(), w3p.data_ptr(), ab.data_ptr(), dab.data_ptr(),
                  None if h_bwd is None else h_bwd.data_ptr(), M, H, N, dy2.stride(0), w3p.stride(0), ab.stride(0), dab.stride(0),
                  Hp if h_bwd is None else h_bwd.stride(0), _lib.dtype_code(T))
        del ab
        dx = dw1 = db1 = dw2 = db2 = dw3 = db3 = None
        if need_w3:                                                # dW3 = dy^T h
            dw3 = _gemm.gemm(dy2, h[:, :H], True, True, torch.float32).to(w3.dtype)
        del h
        if need_b3:
            db3 = dy2.sum(0, dtype=torch.float32).to(ctx.bias_dtypes[2])
        if need_x:                                                 # dx = [da, db] . [W1; W2], K = 2 Hp over a zero-padded stack
            wst = torch.zeros((2 * Hp, K), dtype=T, device=dev)
            wst[:H] = w1
            wst[Hp:Hp + H] = w2
            dx = _gemm.gemm(dab, wst, False, True).view(*dy.shape[:-1], K)
        if need_w1 or need_w2:                                     # [dW1; dW2] = [da, db]^T x
            dw12 = _gemm.gemm(dab, x2, True, True, torch.float32)
            dw1, dw2 = dw12[:H].to(w1.dtype), dw12[Hp:Hp + H].to(w2.dtype)
        if need_b1 or need_b2:
            db12 = dab.sum(0, dtype=torch.float32)
            db1 = None if b1 is None else db12[:H].to(ctx.bias_dtypes[0])
            db2 = None if b2 is None else db12[Hp:Hp + H].to(ctx.bias_dtypes[1])
        return dx, dw1, db1, dw2, db2, dw3, db3, None, None


def swiglu_fn(x, w1, b1, w2, b2, w3, b3, checkpoint_lvl=0):
    """w3(silu(w1(x)) * w2(x)) for bf16 / fp16 CUDA activations (directly or under autocast) as one op: x (..., in), w1 / w2
    (H, in), w3 (out, H) with in and out multiples of 8 (any H), biases (H) / (out) or None.  checkpoint_lvl 0 (default) keeps
    the packed w1(x) / w2(x) for the backward, 1 recomputes them; both give the same bits."""
    train = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, w1, b1, w2, b2, w3, b3))
    return SwiGLUFn.apply(x, w1, b1, w2, b2, w3, b3, checkpoint_lvl, train)


class SwiGLU(nn.Module):
    """models_mamba.py:59-83.  For bf16 / fp16 CUDA activations with the SiLU act and no sub-LN (what Block builds) the
    layer runs as one op (swiglu_fn); every other configuration runs the composition, _forward_composed."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.SiLU, drop=0.0, norm_layer=nn.LayerNorm, subln=False):
        super().__init__()
        out_features, hidden_features = out_features or in_features, hidden_features or in_features
        self.w1 = nn.Linear(in_features, hidden_features)
        self.w2 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.ffn_ln = norm_layer(hidden_features) if subln else nn.Identity()
        self.w3 = nn.Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def _fused_ok(self, x):
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() and x.is_cuda else x.dtype
        return (x.is_cuda and T in (torch.bfloat16, torch.float16) and type(self.act) is nn.SiLU and isinstance(self.ffn_ln, nn.Identity)
                and x.numel() > 0 and self.w1.in_features % 8 == 0 and self.w3.out_features % 8 == 0)

    def forward(self, x):
        if self._fused_ok(x):
            return self.drop(swiglu_fn(x, self.w1.weight, self.w1.bias, self.w2.weight, self.w2.bias, self.w3.weight, self.w3.bias))
        return self._forward_composed(x)

    def _forward_composed(self, x):
        hidden = self.act(_gemm.linear(x, self.w1.weight, self.w1.bias)) * _gemm.linear(x, self.w2.weight, self.w2.bias)
        return self.drop(_gemm.linear(self.ffn_ln(hidden), self.w3.weight, self.w3.bias))


class Block(nn.Module):
    """models_mamba.py:86-129: h + drop_path(mixer(LN(h))); h + drop_path(SwiGLU(LN(h))) (norm_cls / fused_add_norm are accepted
    and unused there too)."""

    def __init__(self, dim, mixer_cls, norm_cls=nn.LayerNorm, fused_add_norm=False, residual_in_fp32=False, drop_path=0.0):
        super().__init__()
        self.residual_in_fp32, self.fused_add_norm = residual_in_fp32, fused_add_norm
        self.mixer = mixer_cls(dim)
        self.mlp = SwiGLU(dim, dim * 4 * 2 // 3, subln=False)
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)

    def forward(self, hidden_states, residual: Optional[torch.Tensor] = None, segmentation: Optional[torch.Tensor] = None, inference_params=None):
        if segmentation is None:
            hidden_states = hidden_states + self.drop_path(self.mixer(self.norm1(hidden_states), inference_params=inference_params))
            return hidden_states + self.drop_path(self.mlp(self.norm2(hidden_states)))
        feats = self.mixer(self.norm1(hidden_states), segmenttation_features=self.norm1(segmentation), inference_params=inference_params)
        hidden_states, segmentation = feats[0] + hidden_states, feats[1] + segmentation
        hidden_states = hidden_states + self.drop_path(self.mlp(self.norm2(hidden_states)))
        segmentation = segmentation + self.drop_path(self.mlp(self.norm2(segmentation)))
        return hidden_states, segmentation

    def allocate_inference_cache(self, batch_size, max_seqlen, dtype=None, **kwargs):
        return self.mixer.allocate_inference_cache(batch_size, max_seqlen, dtype=dtype, **kwargs)


def create_block(d_model, ssm_cfg=None, norm_epsilon=1e-5, drop_path=0.0, rms_norm=False, residual_in_fp32=False, fused_add_norm=False,
                 layer_idx=None, device=None, dtype=None, if_bimamba=False, bimamba_type="none", if_devide_out=False, init_layer_scale=None):
    """models_mamba.py:132-164 (note expand=1)."""
    if if_bimamba:
        bimamba_type = "v1"
    fk = {"device": device, "dtype": dtype}
    mixer_cls = partial(Mamba, expand=1, layer_idx=layer_idx, bimamba_type=bimamba_type, if_devide_out=if_devide_out,
                        init_layer_scale=init_layer_scale, **(ssm_cfg or {}), **fk)
    norm_cls = partial(nn.LayerNorm if not rms_norm else RMSNorm, eps=norm_epsilon, **fk)
    block = Block(d_model, mixer_cls, norm_cls=norm_cls, drop_path=drop_path, fused_add_norm=fused_add_norm, residual_in_fp32=residual_in_fp32)
    block.layer_idx = layer_idx
    return block


def _init_weights(module, n_layer, initializer_range=0.02, rescale_prenorm_residual=True, n_residuals_per_layer=1):
    """models_mamba.py:168-198 (GPT-2 style residual rescaling)."""
    if isinstance(module, nn.Linear):
        if module.bias is not None and not getattr(module.bias, "_no_reinit", False):
            nn.init.zeros_(module.bias)
    elif isinstance(module, nn.Embedding):
        nn.init.normal_(module.weight, std=initializer_range)
    if rescale_prenorm_residual:
        for name, p in module.named_parameters():
            if name in ["out_proj.weight", "fc2.weight"]:
                nn.init.kaiming_uniform_(p, a=math.sqrt(5))
                with torch.no_grad():
                    p /= math.sqrt(n_residuals_per_layer * n_layer)


def segm_init_weights(m):
    """models_mamba.py:201-212."""
    if isinstance(m, nn.Linear):
        nn.init.trunc_normal_(m.weight, std=0.02)
        if m.bias is not None:
            nn.init.constant_(m.bias, 0)
    elif isinstance(m, nn.Conv2d):
        fan_in = m.weight[0].numel()                       # timm lecun_normal_: truncated normal, variance 1 / fan_in
        nn.init.trunc_normal_(m.weight, std=math.sqrt(1.0 / fan_in) / 0.87962566103423978)
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, (nn.LayerNorm, nn.GroupNorm, nn.BatchNorm2d)):
        nn.init.zeros_(m.bias)
        nn.init.ones_(m.weight)


class ARM(nn.Module):
    """models_mamba.py:215-394: patch embed -> cls token in the MIDDLE of the sequence -> + pos_embed -> depth x Block -> LayerNorm."""

    def __init__(self, img_size=224, patch_size=16, stride=16, depth=24, embed_dim=192, channels=3, ssm_cfg=None, drop_rate=0.0,
                 drop_path_rate=0.1, norm_epsilon: float = 1e-5, rms_norm: bool = False, initializer_cfg=None, fused_add_norm=False,
                 residual_in_fp32=False, device=None, dtype=None, ft_seq_len=None, pt_hw_seq_len=14, if_bidirectional=False,
                 final_pool_type="none", if_abs_pos_embed=False, if_rope=False, if_rope_residual=False, flip_img_sequences_ratio=-1.0,
                 if_bimamba=False, bimamba_type="none", if_cls_token=False, if_devide_out=False, init_layer_scale=None,
                 use_double_cls_token=False, use_middle_cls_token=False, global_pool=False, **kwargs):
        fk = {"device": device, "dtype": dtype}
        super().__init__()
        self.residual_in_fp32, self.fused_add_norm, self.if_bidirectional = residual_in_fp32, fused_add_norm, if_bidirectional
        self.final_pool_type, self.if_abs_pos_embed, self.if_rope, self.if_rope_residual = final_pool_type, if_abs_pos_embed, if_rope, if_rope_residual
        self.flip_img_sequences_ratio, self.if_cls_token = flip_img_sequences_ratio, if_cls_token
        self.use_double_cls_token, self.use_middle_cls_token = use_double_cls_token, use_middle_cls_token
        self.num_tokens = 1 if if_cls_token else 0
        self.global_pool = global_pool
        self.d_model = self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, stride=stride, in_chans=channels, embed_dim=embed_dim)
        num_patches = self.patch_embed.num_patches
        if if_cls_token:
            if use_double_cls_token:
                self.cls_token_head = nn.Parameter(torch.zeros(1, 1, embed_dim))
                self.cls_token_tail = nn.Parameter(torch.zeros(1, 1, embed_dim))
                self.num_tokens = 2
            else:
                self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        if if_abs_pos_embed:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + self.num_tokens, embed_dim))
            self.pos_drop = nn.Dropout(p=drop_rate)
        inter_dpr = [0.0] + [v.item() for v in torch.linspace(0, drop_path_rate, depth)]
        self.drop_path = DropPath(drop_path_rate) if drop_path_rate > 0.0 else nn.Identity()
        self.layers = nn.ModuleList([
            create_block(embed_dim, ssm_cfg=ssm_cfg, norm_epsilon=norm_epsilon, rms_norm=rms_norm, residual_in_fp32=residual_in_fp32,
                         fused_add_norm=fused_add_norm, layer_idx=i, if_bimamba=if_bimamba, bimamba_type=bimamba_type, drop_path=inter_dpr[i],
                         if_devide_out=if_devide_out, init_layer_scale=init_layer_scale, **fk) for i in range(depth)])
        self.norm_f = nn.LayerNorm(embed_dim)
        self.patch_embed.apply(segm_init_weights)
        if if_abs_pos_embed:
            nn.init.trunc_normal_(self.pos_embed, std=0.02)
        if if_cls_token:
            for t in ((self.cls_token_head, self.cls_token_tail) if use_double_cls_token else (self.cls_token,)):
                nn.init.trunc_normal_(t, std=0.02)
        self.apply(partial(_init_weights, n_layer=depth, **(initializer_cfg or {})))

    def allocate_inference_cache(self, batch_size, max_seqlen, dtype=None, **kwargs):
        return {i: layer.allocate_inference_cache(batch_size, max_seqlen, dtype=dtype, **kwargs) for i, layer in enumerate(self.layers)}

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "cls_token", "dist_token", "cls_token_head", "cls_token_tail"}

    def forward_features(self, x, segmentation=None, inference_params=None, if_random_cls_token_position=False, if_random_token_rank=False):
        """models_mamba.py:355-389."""
        B, M, _ = x.shape
        cls_token = self.cls_token.expand(B, -1, -1)
        pos = M // 2
        if segmentation is not None:
            mask = torch.zeros_like(x)
            for i in range(len(segmentation)):
                mask[i, segmentation[i], :] = 1
            xm = x * mask
            xm = torch.cat((xm[:, :pos, :], cls_token, xm[:, pos:, :]), dim=1)
            segmentation = self.pos_drop(xm + self.pos_embed)
        x = self.pos_drop(torch.cat((x[:, :pos, :], cls_token, x[:, pos:, :]), dim=1) + self.pos_embed)
        hidden = x
        for layer in self.layers:
            if segmentation is None:
                hidden = layer(hidden, inference_params=inference_params)
            else:
                hidden, segmentation = layer(hidden, segmentation=segmentation, inference_params=inference_params)
        return self.norm_f(hidden)

    def forward(self, x, segmentation=None, return_features=False, inference_params=None, if_random_cls_token_position=False,
                if_random_token_rank=False):
        return self.forward_features(self.patch_embed(x), segmentation, inference_params, if_random_cls_token_position=if_random_cls_token_position,
                                     if_random_token_rank=if_random_token_rank)


def _arm(embed_dim, depth, **kwargs):
    return ARM(patch_size=16, embed_dim=embed_dim, depth=depth, rms_norm=True, residual_in_fp32=True, fused_add_norm=True,
               final_pool_type="mean", if_abs_pos_embed=True, if_rope=False, if_rope_residual=False, bimamba_type="v3", if_cls_token=True,
               if_devide_out=True, use_middle_cls_token=True, **kwargs)


def arm_base_pz16(type=None, pretrained=False, **kwargs):
    """models_mamba.py:398-409 (MambaXray-VL-Base encoder; BASELINE configs[1])."""
    return _arm(768, 12, **kwargs)


def arm_large_pz16(type=None, pretrained=False, **kwargs):
    """models_mamba.py:412-423 (BASELINE configs[3])."""
    return _arm(1024, 24, **kwargs)


def arm_huge_pz16(type=None, pretrained=False, **kwargs):
    """models_mamba.py:425-436."""
    return _arm(1536, 24, **kwargs)
