"""Tensor-core GEMM of libmia_scan.so (csrc/gemm_wgmma.cu) behind the reference's ``nn.Linear`` / 1x1-conv surface.

``linear(x, weight, bias)`` is ``F.linear`` for bf16 / fp16 CUDA activations, computed by the hand-written wgmma kernel
(fp32 accumulation in registers, bias / ReLU / GELU / SiLU fused into the epilogue).  It stands where the reference
calls cuBLAS through ``nn.Linear`` / ``torch.einsum`` (vmamba.py:386, 751, 775; mamba_simple.py:408-414, 686-689, 708;
mae.py:64-66, 82-84) or cuDNN through kernel==stride convolutions (patch_embed.py:25-29).

Backward: dX = dY . W and dW = dY^T . X run on the same kernel with MN-major operand descriptors (``gemm(..., a_mn, b_mn)``:
the transposed operand is read in place, no copies); dbias is a column sum.
fp32 activations (no autocast) are NOT silently rounded to bf16: they take ``F.linear`` like in the reference.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU = 0, 1, 2, 3


def gemm_tn(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, act: int = ACT_NONE, out_dtype=None) -> torch.Tensor:
    """``act(a @ w.T + bias)``: a (M, K), w (N, K), both bf16 or fp16 with K contiguous; bias fp32 (N) or None."""
    if not (a.is_cuda and w.is_cuda):
        raise RuntimeError("gemm_tn: CUDA tensors required (this build has no CPU path)")
    if a.dtype not in (torch.bfloat16, torch.float16) or w.dtype != a.dtype:
        raise RuntimeError("gemm_tn: a and w must both be bfloat16 or both float16")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise RuntimeError(f"gemm_tn: shapes {tuple(a.shape)} x {tuple(w.shape)}^T do not contract")
    M, K = a.shape
    N = w.shape[0]
    out_dtype = out_dtype or a.dtype
    if K % 8:                                            # 16-byte rows for the TMA tensor maps: pad the contraction with zeros
        pad = 8 - K % 8
        a, w = F.pad(a, (0, pad)), F.pad(w, (0, pad))
        K += pad
    if a.stride(1) != 1 or a.stride(0) % 8 or a.data_ptr() % 16:
        a = a.contiguous()
    if w.stride(1) != 1 or w.stride(0) % 8 or w.data_ptr() % 16:
        w = w.contiguous()
    if bias is not None:
        bias = bias.detach().float().contiguous()
    c = torch.empty((M, N), dtype=out_dtype, device=a.device)
    if M == 0 or N == 0:
        return c
    _lib.call("mia_gemm_tn", "mia_gemm_tn", a.device, a.data_ptr(), w.data_ptr(), None if bias is None else bias.data_ptr(), c.data_ptr(),
              M, N, K, a.stride(0), w.stride(0), c.stride(0), _lib.dtype_code(a.dtype), _lib.dtype_code(out_dtype), int(act))
    return c


def gemm(a: torch.Tensor, b: torch.Tensor, a_mn: bool = False, b_mn: bool = False, out_dtype=None) -> torch.Tensor:
    """General wgmma contraction without copies: ``C[M, N] = sum_k A(m, k) B(n, k)`` where each operand is either stored
    [rows = M or N][K] (``*_mn=False``) or [K][M or N] (``*_mn=True``: its transpose read in place, MN-major wgmma operand).
    Both must be bf16 / fp16, last dim contiguous, pitches multiples of 8 elements, 16-byte aligned."""
    K = a.shape[0] if a_mn else a.shape[1]
    M = a.shape[1] if a_mn else a.shape[0]
    N = b.shape[1] if b_mn else b.shape[0]
    if (b.shape[0] if b_mn else b.shape[1]) != K:
        raise RuntimeError(f"gemm: operands {tuple(a.shape)} (mn={a_mn}) and {tuple(b.shape)} (mn={b_mn}) do not contract")
    for t in (a, b):
        if t.dtype not in (torch.bfloat16, torch.float16) or t.dtype != a.dtype or not t.is_cuda:
            raise RuntimeError("gemm: bf16 / fp16 CUDA operands of one dtype required")
        if t.stride(1) != 1 or t.stride(0) % 8 or t.data_ptr() % 16:
            raise RuntimeError("gemm: operands need a contiguous last dim, a row pitch that is a multiple of 8 and 16-byte alignment")
    out_dtype = out_dtype or a.dtype
    c = torch.empty((M, N), dtype=out_dtype, device=a.device)
    _lib.call("mia_gemm", "mia_gemm", a.device, a.data_ptr(), b.data_ptr(), None, c.data_ptr(), M, N, K, a.stride(0), b.stride(0),
              c.stride(0), int(a_mn), int(b_mn), _lib.dtype_code(a.dtype), _lib.dtype_code(out_dtype), ACT_NONE)
    return c


def _mn_ok(t: torch.Tensor) -> bool:
    return t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0


def rows_in(x: torch.Tensor, T: torch.dtype, K: int) -> torch.Tensor:
    """x as a (M, K) operand in dtype T that the wgmma GEMM reads in place (copied only when its rows are not)."""
    x2 = x.to(T).reshape(-1, K)
    return x2 if _mn_ok(x2) else x2.contiguous()


def linear_backward(dy2, x2, weight, bias, need_x, need_w, need_b, w_dtype, b_dtype, T):
    """The gradients of y = x W^T + b from dy2 (M, N) and x2 (M, K), both in dtype T: dx = dy . W with W read MN-major,
    dW = dy^T x in fp32 with both operands read in place, db = the fp32 column sum of dy; each None unless asked for."""
    dx = gemm(dy2, weight.to(T).contiguous(), False, True) if need_x else None
    dw = gemm(dy2, x2, True, True, torch.float32).to(w_dtype) if need_w else None
    db = dy2.sum(0, dtype=torch.float32).to(b_dtype) if need_b and bias is not None else None
    return dx, dw, db


def transpose2d(t: torch.Tensor) -> torch.Tensor:
    """(R, C) -> contiguous (C, R)."""
    return t.t().contiguous()


class LinearTC(torch.autograd.Function):
    """y = act(x @ W^T + b) on the wgmma kernel; x (M, K), W (N, K) in the activation dtype."""

    @staticmethod
    def forward(ctx, x, weight, bias, act, out_dtype):
        w = weight.to(x.dtype)
        if act == ACT_GELU and (x.requires_grad or weight.requires_grad):
            pre = gemm_tn(x, w, bias, ACT_NONE, out_dtype)      # the GELU derivative needs the pre-activation
            y = F.gelu(pre)
            ctx.save_for_backward(x, w, pre)
        else:
            y = gemm_tn(x, w, bias, act, out_dtype)
            ctx.save_for_backward(x, w, y if act in (ACT_RELU, ACT_SILU) else x.new_empty(0))
        ctx.act, ctx.has_bias, ctx.wdtype = act, bias is not None, weight.dtype
        ctx.bdtype = None if bias is None else bias.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, aux = ctx.saved_tensors
        dy = dy.to(x.dtype)
        if ctx.act == ACT_RELU:
            dy = dy * (aux > 0).to(dy.dtype)
        elif ctx.act == ACT_GELU:
            p = aux.float()
            cdf = 0.5 * (1.0 + torch.erf(p * 0.7071067811865476))
            dy = (dy.float() * (cdf + p * torch.exp(-0.5 * p * p) * 0.3989422804014327)).to(x.dtype)
        elif ctx.act == ACT_SILU:
            raise NotImplementedError("fused SiLU epilogue is inference-only")
        dy = dy.contiguous()
        dx = dw = db = None
        direct = _mn_ok(dy) and _mn_ok(w) and _mn_ok(x)         # MN-major operands read in place (no transposed copies)
        if ctx.needs_input_grad[0]:                               # dX[tok, in] = dY[tok, out] . W[out, in]
            dx = gemm(dy, w, False, True) if direct else gemm_tn(dy, transpose2d(w))
        if ctx.needs_input_grad[1]:                               # dW[out, in] = dY[tok, out]^T . X[tok, in]
            dw = (gemm(dy, x, True, True, torch.float32) if direct
                  else gemm_tn(transpose2d(dy), transpose2d(x), out_dtype=torch.float32)).to(ctx.wdtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.float().sum(0).to(ctx.bdtype)
        return dx, dw, db, None, None


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, act: int = ACT_NONE, out_dtype=None) -> torch.Tensor:
    """``F.linear`` (+ fused activation) over the last dimension.  bf16 / fp16 CUDA activations -> wgmma kernel."""
    if torch.is_autocast_enabled() and x.is_cuda:
        x = x.to(torch.get_autocast_dtype("cuda"))
    if not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16):
        y = F.linear(x, weight, bias)                            # fp32 path of the reference: library GEMM, no silent rounding
        return {ACT_NONE: lambda t: t, ACT_RELU: F.relu, ACT_GELU: F.gelu, ACT_SILU: F.silu}[act](y)
    lead = x.shape[:-1]
    y = LinearTC.apply(x.reshape(-1, x.shape[-1]), weight, bias, act, out_dtype)
    return y.view(*lead, weight.shape[0])


def _pad8(n):
    return (n + 7) // 8 * 8


class GeluMlpFn(torch.autograd.Function):
    """fc2(gelu(fc1(x))) (VMamba's channel-last ``Mlp``, timm's ``Mlp`` in the MAE) as ONE op on the wgmma GEMM: fc1 writes
    ``pre`` and ``h = gelu(pre)`` from its epilogue (mia_gemm_gelu_fwd) and fc2 reads ``h`` in place.  The backward's fc2
    dgrad writes ``dpre = g gelu'(pre)`` and the recomputed ``h`` from its epilogue (mia_gemm_gelu_bwd); dW2 = dy^T h,
    dx = dpre . W1 and dW1 = dpre^T x follow with no transposed copies.  DESIGN.md section 3.15.

    ``pre``, ``h`` and the output are bit-identical to ``gemm.linear``'s fc1, ``F.gelu`` and fc2 in training mode.  Saved
    (checkpoint_lvl 0): x in the activation dtype and ``pre`` (M, Hp); level 1 keeps x only and reruns the forward kernel.
    Both give the same bits.  Hp = H rounded up to 8; with nothing to differentiate, nothing is saved and ``pre`` is not
    written."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, w1, b1, w2, b2, checkpoint_lvl, train):
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not x.is_cuda:
            raise RuntimeError("gelu_mlp_fn: this build has no CPU path (x must be a CUDA tensor)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else x.dtype
        if T not in (torch.bfloat16, torch.float16):
            raise RuntimeError(f"gelu_mlp_fn: activations must be bfloat16 or float16, directly or under autocast (got {T})")
        H, K = w1.shape
        N = w2.shape[0]
        if tuple(w2.shape) != (N, H) or x.shape[-1] != K:
            raise RuntimeError(f"gelu_mlp_fn: shapes do not chain: x {tuple(x.shape)}, w1 {tuple(w1.shape)}, w2 {tuple(w2.shape)}")
        if K % 8 or N % 8:
            raise RuntimeError(f"gelu_mlp_fn: in_features ({K}) and out_features ({N}) must be multiples of 8")
        lead = x.shape[:-1]
        x2 = x.to(T).reshape(-1, K)
        if not _mn_ok(x2):
            x2 = x2.contiguous()
        M, Hp = x2.shape[0], _pad8(H)
        if M == 0:
            raise RuntimeError("gelu_mlp_fn: empty input")
        ctx.sizes = (M, H, Hp, K, N, T, checkpoint_lvl)
        pre = torch.empty((M, Hp), dtype=T, device=x.device) if train else None
        h = torch.empty((M, Hp), dtype=T, device=x.device)
        GeluMlpFn._fc1(x2, w1, b1, pre, h, ctx)
        w2p = GeluMlpFn._w2(w2, ctx)
        y = torch.empty((M, N), dtype=T, device=x.device)
        b2f = None if b2 is None else b2.detach().float().contiguous()
        _lib.call("mia_gemm_tn", "gelu_mlp_fn fc2", x.device, h.data_ptr(), w2p.data_ptr(), None if b2f is None else b2f.data_ptr(), y.data_ptr(),
                  M, N, H, h.stride(0), w2p.stride(0), y.stride(0), _lib.dtype_code(T), _lib.dtype_code(T), ACT_NONE)
        if train:
            ctx.save_for_backward(x2, w1, b1, w2, b2, *([pre] if checkpoint_lvl == 0 else []))
            ctx.bias_dtypes = tuple(None if b is None else b.dtype for b in (b1, b2))
        return y.view(*lead, N)

    @staticmethod
    def _fc1(x2, w1, b1, pre, h, ctx):
        """mia_gemm_gelu_fwd: h = gelu(pre) and, when pre is given, pre = x W1^T + b1."""
        M, H, Hp, K, N, T, _ = ctx.sizes
        w1c = w1.to(T).contiguous()
        b1f = None if b1 is None else b1.detach().float().contiguous()
        _lib.call("mia_gemm_gelu_fwd", "gelu_mlp_fn", x2.device, x2.data_ptr(), w1c.data_ptr(), None if b1f is None else b1f.data_ptr(),
                  h.data_ptr(), None if pre is None else pre.data_ptr(), M, H, K, x2.stride(0), w1c.stride(0), h.stride(0),
                  0 if pre is None else pre.stride(0), _lib.dtype_code(T))

    @staticmethod
    def _w2(w2, ctx):
        """W2 in the activation dtype with a row pitch that is a multiple of 8 (zero-padded to Hp columns when H is not)."""
        M, H, Hp, K, N, T, _ = ctx.sizes
        if H % 8 == 0:
            return w2.to(T).contiguous()
        w2p = torch.zeros((N, Hp), dtype=T, device=w2.device)
        w2p[:, :H] = w2
        return w2p

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        M, H, Hp, K, N, T, lvl = ctx.sizes
        x2, w1, b1, w2, b2, *keep = ctx.saved_tensors
        dev = x2.device
        need_x, need_w1, need_b1, need_w2, need_b2 = ctx.needs_input_grad[:5]
        dy2 = dy.to(T).reshape(M, N)
        if not _mn_ok(dy2):
            dy2 = dy2.contiguous()
        h = torch.empty((M, Hp), dtype=T, device=dev) if need_w2 or lvl == 1 else None
        if lvl == 0:
            pre = keep[0]
        else:                                                      # rerun the forward kernel: pre and h, bit for bit
            pre = torch.empty((M, Hp), dtype=T, device=dev)
            GeluMlpFn._fc1(x2, w1, b1, pre, h, ctx)
        w2p = GeluMlpFn._w2(w2, ctx)
        dpre = torch.empty((M, Hp), dtype=T, device=dev)
        h_bwd = h if lvl == 0 else None
        _lib.call("mia_gemm_gelu_bwd", "gelu_mlp_fn backward", dev, dy2.data_ptr(), w2p.data_ptr(), pre.data_ptr(), dpre.data_ptr(),
                  None if h_bwd is None else h_bwd.data_ptr(), M, H, N, dy2.stride(0), w2p.stride(0), pre.stride(0), dpre.stride(0),
                  Hp if h_bwd is None else h_bwd.stride(0), _lib.dtype_code(T))
        del pre
        dx = dw1 = db1 = dw2 = db2 = None
        if need_w2:                                                # dW2 = dy^T h
            dw2 = gemm(dy2, h[:, :H], True, True, torch.float32).to(w2.dtype)
        del h
        if need_b2 and b2 is not None:
            db2 = dy2.sum(0, dtype=torch.float32).to(ctx.bias_dtypes[1])
        dpre = dpre[:, :H]
        if need_x:                                                 # dx = dpre . W1 (W1 read MN-major)
            dx = gemm(dpre, w1.to(T).contiguous(), False, True).view(*dy.shape[:-1], K)
        if need_w1:                                                # dW1 = dpre^T x
            dw1 = gemm(dpre, x2, True, True, torch.float32).to(w1.dtype)
        if need_b1 and b1 is not None:
            db1 = dpre.sum(0, dtype=torch.float32).to(ctx.bias_dtypes[0])
        return dx, dw1, db1, dw2, db2, None, None


def gelu_mlp_fn(x, w1, b1, w2, b2, checkpoint_lvl=0):
    """fc2(gelu(fc1(x))) for bf16 / fp16 CUDA activations (directly or under autocast) as one op: x (..., in), w1 (H, in),
    w2 (out, H) with in and out multiples of 8 (any H), biases (H) / (out) or None.  checkpoint_lvl 0 (default) keeps the
    pre-activation for the backward, 1 recomputes it; both give the same bits."""
    train = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, w1, b1, w2, b2))
    return GeluMlpFn.apply(x, w1, b1, w2, b2, checkpoint_lvl, train)


def gelu_mlp_eligible(mlp: nn.Module, x: torch.Tensor, dropout_off: bool) -> bool:
    """Whether an fc1 -> GELU -> fc2 MLP (vmamba / mae ``Mlp``) runs as one op (gelu_mlp_fn): a backward follows (grad
    enabled and an input or parameter requires it), bf16 / fp16 CUDA activations (directly or under autocast), nn.Linear
    layers with in / out features multiples of 8, exact GELU and no active dropout inside."""
    T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() and x.is_cuda else x.dtype
    return (torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in mlp.parameters())) and x.is_cuda
            and T in (torch.bfloat16, torch.float16) and type(mlp.fc1) is nn.Linear and type(mlp.fc2) is nn.Linear
            and type(mlp.act) is nn.GELU and mlp.act.approximate == "none" and dropout_off and x.numel() > 0
            and mlp.fc1.in_features % 8 == 0 and mlp.fc2.out_features % 8 == 0)


def conv2d_patch(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None, stride, act: int = ACT_NONE) -> torch.Tensor:
    """``nn.Conv2d`` with kernel_size == stride and no padding (patch embeddings: models_mamba.py:45, patch_embed.py:25-29) as
    ONE GEMM over the non-overlapping patches: (B hp wp, C kh kw) x (O, C kh kw)^T on the wgmma kernel for bf16 / fp16
    activations; anything else (fp32, overlapping windows) is the library convolution.  Returns (B, O, hp, wp)."""
    kh, kw = weight.shape[2:]
    sh, sw = (stride, stride) if isinstance(stride, int) else tuple(stride)
    if torch.is_autocast_enabled() and x.is_cuda:
        x = x.to(torch.get_autocast_dtype("cuda"))
    if (kh, kw) != (sh, sw) or not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16):
        y = F.conv2d(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype), stride=(sh, sw))
        return {ACT_NONE: lambda t: t, ACT_RELU: F.relu, ACT_GELU: F.gelu, ACT_SILU: F.silu}[act](y)
    B, C, H, W = x.shape
    hp, wp = H // kh, W // kw
    O = weight.shape[0]
    if kh == 1 and kw == 1:
        patches = x.permute(0, 2, 3, 1).reshape(B * hp * wp, C)
    else:
        patches = x[:, :, :hp * kh, :wp * kw].reshape(B, C, hp, kh, wp, kw).permute(0, 2, 4, 1, 3, 5).reshape(B * hp * wp, C * kh * kw)
    y = LinearTC.apply(patches, weight.reshape(O, -1), bias, act, None)
    return y.view(B, hp, wp, O).permute(0, 3, 1, 2)
