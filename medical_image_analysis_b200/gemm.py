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
