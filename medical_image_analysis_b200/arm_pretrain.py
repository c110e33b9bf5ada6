"""ARM autoregressive pre-training model of MambaXray-VL (BASELINE configs[3]) on the library's kernels.

Mirrors ``CXPMRG_Bench_MambaXray_VL/pretrain/models_pretrain.py`` (``Mlp`` :35-51, ``CrossAttention`` :55-83,
``DecoderBlock`` :86-104, ``create_block`` :202-234, ``VisionMamba`` :285-515 and the ``arm_*`` factories :517-547;
``EMRRG/pretrain/`` holds an identical copy): same constructor arguments, buffers and parameter names, so its checkpoints
load strictly.  The factory names collide with ``arm.py``'s (the fine-tuning encoder), hence a module of its own.

What runs where: the encoder is ``arm.Block`` (LN, the one-direction mixer through ``mamba_inner_fn``, LN, the fused
SwiGLU op), the patch embedding / ``enc2dec`` / ``ar_pred`` are the wgmma GEMM, the decoder MLP is ``mae.Mlp`` (the fused
GELU MLP op), and the decoder's segment-causal ``CrossAttention`` is one op, ``CrossAttentionFn``: the q and kv GEMMs,
the wgmma cross-attention kernels that read q / k / v in place and skip the key tiles the mask hides, and the proj GEMM
(DESIGN.md section 3.17).  Parity: tests/golden/modules_arm_pretrain.npz holds the reference's own outputs (see
tests/golden/make_golden_pretrain.py).
"""
from __future__ import annotations

import weakref
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from . import gemm as _gemm
from .arm import PatchEmbed, _init_weights, create_block, segm_init_weights
from .mae import Mlp
from .vmamba import DropPath

__all__ = ["CrossAttention", "CrossAttentionFn", "DecoderBlock", "VisionMamba", "create_block", "cross_attention_fn", "cross_attention_eligible",
           "mask_segment", "arm_base_pz16", "arm_large_pz16", "arm_huge_pz16", "arm_base_pz16_1280"]

XATTN_HEAD_DIM = 64


# ---------------------------------------------------------------------------------------------------------
class CrossAttentionFn(torch.autograd.Function):
    """The decoder's CrossAttention (proj(softmax(q k^T dh^-0.5 + mask) v) with q = q_in W_q^T + b_q and [k, v] = kv_in
    W_kv^T + b_kv, mask segment-causal of segment length seg) as ONE op: the q GEMM writes (B, N, C), the kv GEMM (B, N, 2C),
    mia_xattn_fwd reads both in place and writes o token-major, the layout proj reads.  The backward runs proj's dgrad /
    wgrad, mia_xattn_bwd (no atomics) writing dq (B, N, C) and dk / dv into a packed (B, N, 2C), which are the q and kv
    GEMMs' output gradients, then their dgrad / wgrad with no transposed copies; weight gradients are fp32 GEMMs and bias
    gradients fp32 column sums.  DESIGN.md section 3.17.

    Saved (checkpoint_lvl 0): q_in and kv_in in the activation dtype, q, kv, o and the fp32 logsumexp (B, H, N); level 1
    keeps q_in and kv_in only and reruns the GEMMs and the forward kernel.  Both give the same bits.  With nothing to
    differentiate, nothing is saved and no logsumexp is written."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, q_in, kv_in, q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias, num_heads, seg, checkpoint_lvl, train):
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not (q_in.is_cuda and kv_in.is_cuda):
            raise RuntimeError("cross_attention_fn: this build has no CPU path (q_in and kv_in must be CUDA tensors)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else q_in.dtype
        if T not in (torch.bfloat16, torch.float16):
            raise RuntimeError(f"cross_attention_fn: activations must be bfloat16 or float16, directly or under autocast (got {T})")
        if q_in.dim() != 3 or q_in.numel() == 0 or q_in.shape != kv_in.shape:
            raise RuntimeError(f"cross_attention_fn: q_in and kv_in must be non-empty (B, N, C) tensors of one shape, got "
                               f"{tuple(q_in.shape)} / {tuple(kv_in.shape)}")
        B, N, C = q_in.shape
        if C != num_heads * XATTN_HEAD_DIM:
            raise RuntimeError(f"cross_attention_fn: head dim C / num_heads = {C} / {num_heads} must be {XATTN_HEAD_DIM}")
        if tuple(q_weight.shape) != (C, C) or tuple(kv_weight.shape) != (2 * C, C) or tuple(proj_weight.shape) != (C, C):
            raise RuntimeError(f"cross_attention_fn: weights {tuple(q_weight.shape)} / {tuple(kv_weight.shape)} / {tuple(proj_weight.shape)} "
                               f"do not match C = {C}")
        if not 1 <= seg <= N:
            raise RuntimeError(f"cross_attention_fn: segment length {seg} is not in [1, N = {N}]")
        xq, xkv = _gemm.rows_in(q_in, T, C), _gemm.rows_in(kv_in, T, C)
        ctx.sizes = (B, N, C, num_heads, seg, T, checkpoint_lvl)
        q, kv, o, lse = CrossAttentionFn._attend(xq, xkv, q_weight, q_bias, kv_weight, kv_bias, ctx, train)
        y = _gemm.gemm_tn(o, proj_weight.to(T), proj_bias)
        if train:
            ctx.save_for_backward(xq, xkv, q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias,
                                  *([q, kv, o, lse] if checkpoint_lvl == 0 else []))
            ctx.param_dtypes = tuple(None if t is None else t.dtype for t in (q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias))
        return y.view(B, N, C)

    @staticmethod
    def _attend(xq, xkv, q_weight, q_bias, kv_weight, kv_bias, ctx, train):
        """q and kv (bit-identical to gemm.linear), o and, when training, the logsumexp."""
        B, N, C, H, seg, T, _ = ctx.sizes
        q = _gemm.gemm_tn(xq, q_weight.to(T), q_bias)
        kv = _gemm.gemm_tn(xkv, kv_weight.to(T), kv_bias)
        o = torch.empty((B * N, C), dtype=T, device=xq.device)
        lse = torch.empty((B, H, N), dtype=torch.float32, device=xq.device) if train else None
        _lib.call("mia_xattn_fwd", "cross_attention_fn", xq.device, q.data_ptr(), kv.data_ptr(), o.data_ptr(), None if lse is None else lse.data_ptr(),
                  B, N, H, XATTN_HEAD_DIM, seg, q.stride(0), kv.stride(0), o.stride(0), _lib.dtype_code(T))
        return q, kv, o, lse

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        B, N, C, H, seg, T, lvl = ctx.sizes
        xq, xkv, wq, bq, wkv, bkv, wp, bp, *keep = ctx.saved_tensors
        dev = xq.device
        need_xq, need_xkv, need_wq, need_bq, need_wkv, need_bkv, need_wp, need_bp = ctx.needs_input_grad[:8]
        dt_wq, dt_bq, dt_wkv, dt_bkv, dt_wp, dt_bp = ctx.param_dtypes
        q, kv, o, lse = keep if lvl == 0 else CrossAttentionFn._attend(xq, xkv, wq, bq, wkv, bkv, ctx, True)
        dy2 = _gemm.rows_in(dy, T, C)
        do, dwp, dbp = _gemm.linear_backward(dy2, o, wp, bp, True, need_wp, need_bp, dt_wp, dt_bp, T)     # dO = dy . Wp
        delta = torch.empty((B, H, N), dtype=torch.float32, device=dev)
        dq = torch.empty((B * N, C), dtype=T, device=dev)
        dkv = torch.empty((B * N, 2 * C), dtype=T, device=dev)
        _lib.call("mia_xattn_bwd", "cross_attention_fn backward", dev, q.data_ptr(), kv.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(),
                  delta.data_ptr(), dq.data_ptr(), dkv.data_ptr(), B, N, H, XATTN_HEAD_DIM, seg, q.stride(0), kv.stride(0), o.stride(0), do.stride(0),
                  dq.stride(0), dkv.stride(0), _lib.dtype_code(T))
        del q, kv, o, lse, do, delta
        dxq, dwq, dbq = _gemm.linear_backward(dq, xq, wq, bq, need_xq, need_wq, need_bq, dt_wq, dt_bq, T)
        del dq
        dxkv, dwkv, dbkv = _gemm.linear_backward(dkv, xkv, wkv, bkv, need_xkv, need_wkv, need_bkv, dt_wkv, dt_bkv, T)
        view = lambda t: None if t is None else t.view(B, N, C)
        return view(dxq), view(dxkv), dwq, dbq, dwkv, dbkv, dwp, dbp, None, None, None, None


def cross_attention_fn(q_in, kv_in, q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias, num_heads, seg, checkpoint_lvl=0):
    """The decoder's CrossAttention for bf16 / fp16 CUDA activations (directly or under autocast) as one op: q_in / kv_in
    (B, N, C), q_weight (C, C), kv_weight (2C, C), proj_weight (C, C), biases or None, head dim C / num_heads = 64, and the
    segment-causal mask of segment length seg (key j visible to query i iff j // seg <= i // seg).  checkpoint_lvl 0
    (default) keeps q, kv, o and the logsumexp for the backward, 1 recomputes them; both give the same bits."""
    train = torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                            for t in (q_in, kv_in, q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias))
    return CrossAttentionFn.apply(q_in, kv_in, q_weight, q_bias, kv_weight, kv_bias, proj_weight, proj_bias, num_heads, seg, checkpoint_lvl, train)


_SEGMENTS: dict = {}


def mask_segment(mask: torch.Tensor | None, N: int) -> int | None:
    """seg when ``mask`` is the (N, N) additive segment-causal mask of ``VisionMamba.mask_generate`` (0 where
    key // seg <= query // seg, -inf elsewhere) with seg the count of zeros in row 0; None for any other mask.  The
    comparison runs once on the mask's device and is cached on (data_ptr, _version), so a buffer mutated in place is
    checked again; the entry also holds a weak reference to the tensor, so a new tensor at a reused address is checked too."""
    if mask is None or mask.dim() != 2 or tuple(mask.shape) != (N, N) or not mask.is_floating_point():
        return None
    key = (mask.data_ptr(), mask._version, str(mask.device), mask.dtype, N, mask.stride())
    hit = _SEGMENTS.get(key)
    if hit is None or hit[0]() is not mask:
        with torch.no_grad():
            seg = int((mask[0] == 0).sum())
            ok = 1 <= seg <= N
            if ok:
                i = torch.arange(N, device=mask.device)
                want = torch.zeros((N, N), dtype=mask.dtype, device=mask.device).masked_fill(i[None, :] // seg > i[:, None] // seg, float("-inf"))
                ok = bool(torch.equal(mask, want))
        if len(_SEGMENTS) > 64:
            _SEGMENTS.clear()
        _SEGMENTS[key] = hit = (weakref.ref(mask), seg if ok else None)
    return hit[1]


def cross_attention_eligible(attn: nn.Module, q_in: torch.Tensor, kv_in: torch.Tensor, mask: torch.Tensor | None) -> bool:
    """Whether a CrossAttention runs as one op (cross_attention_fn): CUDA tensors, bf16 / fp16 activations (directly or
    under autocast), head dim 64 with scale dh^-0.5, q_in and kv_in of one (B, N, C), no active attention dropout, and a
    segment-causal mask (mask_segment), with or without grad."""
    T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() and q_in.is_cuda else q_in.dtype
    return (q_in.is_cuda and kv_in.is_cuda and T in (torch.bfloat16, torch.float16) and attn.head_dim == XATTN_HEAD_DIM
            and attn.scale == XATTN_HEAD_DIM ** -0.5 and q_in.dim() == 3 and q_in.shape == kv_in.shape and q_in.numel() > 0
            and not (attn.training and attn.attn_drop.p > 0) and mask is not None and mask.is_cuda
            and mask_segment(mask, q_in.shape[1]) is not None)


class CrossAttention(nn.Module):
    """models_pretrain.py:55-83.  Runs as one op (cross_attention_fn) where cross_attention_eligible says so; every other
    case runs the reference's math on gemm.linear, _forward_composed.  proj_drop stays outside the op."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0.0, proj_drop=0.0):
        super().__init__()
        self.num_heads = num_heads
        self.head_dim = dim // num_heads
        self.scale = qk_scale or self.head_dim ** -0.5
        self.q = nn.Linear(dim, dim, bias=qkv_bias)
        self.kv = nn.Linear(dim, dim * 2, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)

    def forward(self, q, kv, mask):
        if cross_attention_eligible(self, q, kv, mask):
            return self.proj_drop(cross_attention_fn(q, kv, self.q.weight, self.q.bias, self.kv.weight, self.kv.bias, self.proj.weight,
                                                     self.proj.bias, self.num_heads, mask_segment(mask, q.shape[1])))
        return self._forward_composed(q, kv, mask)

    def _forward_composed(self, q, kv, mask):
        B, N, C = q.shape
        q = _gemm.linear(q, self.q.weight, self.q.bias).reshape(B, N, 1, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        kv = _gemm.linear(kv, self.kv.weight, self.kv.bias).reshape(B, N, 2, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = q[0], kv[0], kv[1]
        attn = (q @ k.transpose(-2, -1)) * self.scale
        attn += mask
        attn = self.attn_drop(attn.softmax(dim=-1))
        x = (attn @ v).transpose(1, 2).reshape(B, N, C)
        return self.proj_drop(_gemm.linear(x, self.proj.weight, self.proj.bias))


class DecoderBlock(nn.Module):
    """models_pretrain.py:86-104: q + attn2(LN(q), LN(kv), mask); q + mlp(LN(q)).  The Mlp (:35-51) is mae.Mlp: the same
    fc1 / act / fc2 keys and math with GELU and no dropout, which is what the model builds; drop_path is built and unused,
    as in the reference."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop=0.0, attn_drop=0.0, drop_path=0.0, act_layer=nn.GELU,
                 norm_layer=nn.LayerNorm):
        super().__init__()
        if act_layer is not nn.GELU or drop > 0:
            raise NotImplementedError("DecoderBlock: the decoder MLP is GELU without dropout, as VisionMamba builds it")
        self.attn2 = CrossAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop, proj_drop=drop)
        self.norm2_1 = norm_layer(dim)
        self.norm2_2 = norm_layer(dim)
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))

    def forward(self, q, kv, mask):
        q = q + self.attn2(self.norm2_1(q), self.norm2_2(kv), mask)
        return q + self.mlp(self.norm2(q))


# ---------------------------------------------------------------------------------------------------------
def _sincos_2d(embed_dim, grid_size):
    """The fixed 2-D sine-cosine table of the pretrain utils (no cls token), computed in float32 as there: the first half
    encodes the column index, the second the row index."""
    def one(dim, pos):
        omega = np.arange(dim // 2, dtype=np.float32)
        omega /= dim / 2.0
        omega = 1.0 / 10000 ** omega
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    g = np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(g, g), axis=0).reshape([2, 1, grid_size, grid_size])
    return np.concatenate([one(embed_dim // 2, grid[0]), one(embed_dim // 2, grid[1])], axis=1)


def _clusters(x, side):
    """(B, side * side, C) in row-major token order -> (B, (side / 4)^2, 16, C): the 4 x 4 clusters of the token grid, each
    row-major (``b (h p1) (w p2) c -> b (h w) (p1 p2) c`` with p1 = p2 = 4)."""
    B, _, C = x.shape
    return x.reshape(B, side // 4, 4, side // 4, 4, C).permute(0, 1, 3, 2, 4, 5).reshape(B, (side // 4) ** 2, 16, C)


class VisionMamba(nn.Module):
    """models_pretrain.py:285-515: patch embed + fixed pos embed -> 4 x 4 token clusters, the last dropped -> depth x Block
    -> the hidden states after layers ``skip``, normed and mapped by enc2dec to four decoder streams -> 4 DecoderBlocks whose
    queries are the AR tokens (first cluster dropped) and whose keys / values are those streams, under the segment-causal
    ``mask`` buffer -> ar_norm -> ar_pred -> per-token squared error against the normalised patches."""

    def __init__(self, img_size=224, patch_size=16, stride=16, depth=24, embed_dim=192, dec_embed_dim=192, channels=3, num_classes=1000, ssm_cfg=None,
                 drop_rate=0.0, drop_path_rate=0.1, norm_epsilon: float = 1e-5, rms_norm: bool = False, initializer_cfg=None, fused_add_norm=False,
                 residual_in_fp32=False, device=None, dtype=None, if_bidirectional=False, if_abs_pos_embed=False, bimamba_type="none",
                 if_devide_out=False, init_layer_scale=None, **kwargs):
        fk = {"device": device, "dtype": dtype}
        super().__init__()
        self.residual_in_fp32, self.fused_add_norm = residual_in_fp32, fused_add_norm
        self.if_bidirectional, self.if_abs_pos_embed = if_bidirectional, if_abs_pos_embed
        if depth == 12:
            self.skip = [6, 8, 10, 12]
        elif depth == 24:
            self.skip = [12, 16, 20, 24]
        self.num_classes = num_classes
        self.d_model = self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, stride=stride, in_chans=channels, embed_dim=embed_dim)
        num_patches = self.patch_embed.num_patches
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches, self.embed_dim), requires_grad=False)
        self.drop_path = DropPath(drop_path_rate) if drop_path_rate > 0.0 else nn.Identity()
        self.layers = nn.ModuleList([
            create_block(embed_dim, ssm_cfg=ssm_cfg, norm_epsilon=norm_epsilon, rms_norm=rms_norm, residual_in_fp32=residual_in_fp32,
                         fused_add_norm=fused_add_norm, layer_idx=i, bimamba_type=bimamba_type, drop_path=0.0, if_devide_out=if_devide_out,
                         init_layer_scale=init_layer_scale, **fk) for i in range(depth)])
        self.dec_embed_dim = dec_embed_dim
        self.ar_token = nn.Parameter(torch.zeros(1, 1, self.dec_embed_dim))
        self.dec_pos_embed = nn.Parameter(torch.zeros(1, num_patches, self.dec_embed_dim), requires_grad=False)
        self.pos_drop = nn.Dropout(p=drop_rate)
        self.enc2dec = nn.Linear(embed_dim * 4, self.dec_embed_dim * 4)
        self.dec_block = nn.ModuleList([DecoderBlock(self.dec_embed_dim, self.dec_embed_dim // 64, 4, qkv_bias=True, qk_scale=None,
                                                     norm_layer=nn.LayerNorm) for _ in range(4)])
        self.norm_1, self.norm_2, self.norm_3, self.norm_4 = (nn.LayerNorm(embed_dim) for _ in range(4))
        self.ar_norm = nn.LayerNorm(self.dec_embed_dim)
        self.ar_pred = nn.Linear(self.dec_embed_dim, patch_size ** 2 * 3)

        self.patch_embed.apply(segm_init_weights)
        if if_abs_pos_embed:
            side = int(self.patch_embed.num_patches ** 0.5)
            self.pos_embed.data.copy_(torch.from_numpy(_sincos_2d(self.pos_embed.shape[-1], side)).float().unsqueeze(0))
            self.dec_pos_embed.data.copy_(torch.from_numpy(_sincos_2d(self.dec_pos_embed.shape[-1], side)).float().unsqueeze(0))
        nn.init.trunc_normal_(self.ar_token, std=0.02)
        self.apply(partial(_init_weights, n_layer=depth, **(initializer_cfg or {})))
        self.dec_block.apply(self.atten_init_weights)
        assert patch_size == stride
        self.cluster_num = ((img_size // patch_size) // 4) * ((img_size // patch_size) // 4) - 1
        self.register_buffer("mask", self.mask_generate(self.cluster_num, 16))

    @staticmethod
    def mask_generate(segment, tokens_per_segment):
        """(segment * tokens_per_segment)^2 fp32: 0 where key // tokens_per_segment <= query // tokens_per_segment, else -inf."""
        seg = torch.arange(segment * tokens_per_segment) // tokens_per_segment
        return torch.zeros(seg.numel(), seg.numel()).masked_fill(seg[None, :] > seg[:, None], float("-inf"))

    @staticmethod
    def atten_init_weights(m):
        if isinstance(m, nn.Linear):
            nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def allocate_inference_cache(self, batch_size, max_seqlen, dtype=None, **kwargs):
        return {i: layer.allocate_inference_cache(batch_size, max_seqlen, dtype=dtype, **kwargs) for i, layer in enumerate(self.layers)}

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "cls_token", "dist_token", "cls_token_head", "cls_token_tail"}

    @torch.jit.ignore()
    def load_pretrained(self, checkpoint_path, prefix=""):
        raise NotImplementedError("load_pretrained (timm's npz loader) is not mirrored: load a state_dict instead")

    def forward_features(self, x, inference_params=None):
        """models_pretrain.py:425-460 -> (B, N, D, 4): decoder block i reads [..., i]."""
        x = self.patch_embed(x)
        B, N, C = x.shape
        x = self.pos_drop(x + self.pos_embed)
        hidden_states = _clusters(x, int(np.sqrt(N)))[:, :-1].reshape(B, -1, C)      # the last cluster would leak the targets
        features = []
        for count, layer in enumerate(self.layers, 1):
            hidden_states = layer(hidden_states, inference_params=inference_params)
            if count in self.skip:
                features.append(hidden_states)
        features = [self.norm_1(features[0]), self.norm_2(features[1]), self.norm_3(features[2]), self.norm_4(features[3])]
        features = _gemm.linear(torch.cat(features, dim=-1), self.enc2dec.weight, self.enc2dec.bias)
        B, N, C = features.shape
        assert N == 16 * self.cluster_num
        return features.reshape(B, N, C // 4, 4)

    def forward_decoder(self, latent_ar, decoder_pos_embed):
        """models_pretrain.py:462-479."""
        B, N, C, depth = latent_ar.shape
        ar_token = self.ar_token + decoder_pos_embed
        ar_token = _clusters(ar_token, int(np.sqrt(ar_token.shape[1])))[:, 1:].reshape(1, -1, C).repeat(B, 1, 1)
        for count, blk in enumerate(self.dec_block):
            ar_token = blk(ar_token, latent_ar[:, :, :, count], self.mask)
        ar_token = self.ar_norm(ar_token)
        return _gemm.linear(ar_token, self.ar_pred.weight, self.ar_pred.bias)

    def patchify(self, imgs):
        p = self.patch_embed.patch_size[0]
        assert imgs.shape[2] == imgs.shape[3] and imgs.shape[2] % p == 0
        h = w = imgs.shape[2] // p
        x = torch.einsum("nchpwq->nhwpqc", imgs.reshape(imgs.shape[0], 3, h, p, w, p))
        return x.reshape(imgs.shape[0], h * w, p ** 2 * 3)

    def forward_loss(self, imgs, pred):
        """models_pretrain.py:495-508: the per-patch normalisation is always applied (unbiased var, eps 1e-6)."""
        target = self.patchify(imgs)
        target = (target - target.mean(dim=-1, keepdim=True)) / (target.var(dim=-1, keepdim=True) + 1.0e-6) ** 0.5
        B, N, C = target.shape
        target = _clusters(target, int(np.sqrt(N)))[:, 1:].reshape(B, -1, C)
        return (pred - target) ** 2

    def forward(self, x, inference_params=None):
        labels = x.clone()
        x = self.forward_features(x, inference_params)
        x = self.forward_decoder(x, self.dec_pos_embed)
        return self.forward_loss(labels, x).mean(-1).mean(0)


def _vision_mamba(**kwargs):
    return VisionMamba(dec_embed_dim=512, rms_norm=True, residual_in_fp32=True, fused_add_norm=True, if_abs_pos_embed=True, bimamba_type="None",
                       **kwargs)


def arm_base_pz16(pretrained=False, **kwargs):
    """models_pretrain.py:517-523."""
    return _vision_mamba(patch_size=16, img_size=192, embed_dim=768, depth=12, **kwargs)


def arm_large_pz16(pretrained=False, **kwargs):
    """models_pretrain.py:525-531 (BASELINE configs[3], SURVEY C4)."""
    return _vision_mamba(patch_size=16, img_size=192, embed_dim=1024, depth=24, **kwargs)


def arm_huge_pz16(pretrained=False, **kwargs):
    """models_pretrain.py:533-539."""
    return _vision_mamba(patch_size=16, stride=16, img_size=192, embed_dim=1536, depth=24, **kwargs)


def arm_base_pz16_1280(pretrained=False, **kwargs):
    """models_pretrain.py:541-547."""
    return _vision_mamba(patch_size=64, stride=64, img_size=1280, embed_dim=768, depth=12, **kwargs)
