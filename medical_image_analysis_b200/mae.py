"""ViT-MAE of HD_Xray_Pretrain_MAE on the wgmma GEMM: the high-resolution patch encode and the transformer blocks.

Mirrors ``HD_Xray_Pretrain_MAE/pretrain/patch_embed.py`` (``SmallPatchEmbed``, :21-41), ``models/mae.py``
(``MaskedAutoencoderViT`` :41-387 and the ``mae_vit_*`` factories :389-420) and the ``Block`` / ``Attention`` / ``Mlp`` of
timm 0.9.2 that mae.py:35 imports (third-party, pinned by pretrain/requirements.txt:93, absent from /root/reference:
restated from its published definition -- pre-LN block, qkv bias, no qk-norm, no layer-scale, GELU MLP x4).  Parameter
names and shapes are the reference's (``patch_embed.conv1/conv2/proj``, ``blocks.N.attn.qkv`` ...) so its checkpoints load.

The patch encode is three kernel == stride convolutions, i.e. three GEMMs over non-overlapping patches with ReLU fused
into the epilogue: per 1280 x 1280 image (6400 x 256).(256 x 1024), (400 x 16384).(16384 x 1024), (400 x 1024).(1024 x
1024) = 17.6 GFLOP.  qkv / proj / fc1 (+GELU) / fc2 of the blocks are the same kernel.  The 61- / 401-token attention of
bf16 / fp16 blocks is one op, ``AttentionFn``: the qkv GEMM, wgmma attention kernels that read q / k / v in place, and the
proj GEMM, with a backward free of atomics (DESIGN.md section 3.16).  fp32 blocks run torch's scaled_dot_product_attention.
"""
from __future__ import annotations

import math
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from . import gemm as _gemm


# ---------------------------------------------------------------------------------------------------------
class SmallPatchEmbed(nn.Module):
    """patch_embed.py:21-41: conv 16/16 -> ReLU -> conv 4/4 -> ReLU -> conv 1x1, flattened to (B, tokens, embed_dim)."""

    def __init__(self, in_chans=1, embed_dim=1024, hidden_dim=1024, bias=True):
        super().__init__()
        self.conv1 = nn.Conv2d(in_chans, hidden_dim, kernel_size=16, stride=16, bias=bias)
        self.conv2 = nn.Conv2d(hidden_dim, hidden_dim, kernel_size=4, stride=4, bias=bias)
        self.proj = nn.Conv2d(hidden_dim, embed_dim, kernel_size=1, stride=1, bias=bias)
        self.num_patches = 400                  # hard-wired in the reference (:30-31): 1280 x 1280 inputs
        self.patch_size = (64, 64)

    def forward(self, x):
        x = _gemm.conv2d_patch(x, self.conv1.weight, self.conv1.bias, 16, _gemm.ACT_RELU)
        x = _gemm.conv2d_patch(x, self.conv2.weight, self.conv2.bias, 4, _gemm.ACT_RELU)
        x = _gemm.conv2d_patch(x, self.proj.weight, self.proj.bias, 1)
        return x.flatten(2).transpose(1, 2)


class Attention(nn.Module):
    """timm 0.9.2 ``vision_transformer.Attention`` (qkv_bias, no qk_norm, no dropout).  Runs as one op (attention_fn) where
    attention_eligible says so; every other case runs the composition, _forward_composed."""

    def __init__(self, dim, num_heads=8, qkv_bias=False):
        super().__init__()
        assert dim % num_heads == 0, "dim should be divisible by num_heads"
        self.num_heads, self.head_dim = num_heads, dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x):
        if attention_eligible(self, x):
            return attention_fn(x, self.qkv.weight, self.qkv.bias, self.proj.weight, self.proj.bias, self.num_heads)
        return self._forward_composed(x)

    def _forward_composed(self, x):
        B, N, C = x.shape
        qkv = _gemm.linear(x, self.qkv.weight, self.qkv.bias).reshape(B, N, 3, self.num_heads, self.head_dim).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        x = F.scaled_dot_product_attention(q, k, v)             # softmax(q k^T / sqrt(d)) v
        return _gemm.linear(x.transpose(1, 2).reshape(B, N, C), self.proj.weight, self.proj.bias)


ATTN_HEAD_DIMS = (32, 64, 80)


class AttentionFn(torch.autograd.Function):
    """timm's Attention (proj(softmax(q k^T dh^-0.5) v) with qkv = x W_qkv^T + b_qkv) as ONE op: the qkv GEMM writes
    (B, N, 3, H, dh), mia_attn_fwd reads q / k / v from it in place and writes o token-major (B, N, C), the layout the
    proj GEMM reads.  The backward runs proj's dgrad / wgrad, mia_attn_bwd (two launches, no atomics) writing dq / dk / dv
    into the packed (B, N, 3C) gradient of qkv, then qkv's dgrad / wgrad with no transposed copies; bias gradients are
    fp32 column sums.  DESIGN.md section 3.16.

    Saved (checkpoint_lvl 0): x in the activation dtype, qkv, o and the fp32 logsumexp (B, H, N); level 1 keeps x only and
    reruns the qkv GEMM and the forward kernel.  Both give the same bits.  With nothing to differentiate, nothing is saved
    and no logsumexp is written."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, qkv_weight, qkv_bias, proj_weight, proj_bias, num_heads, checkpoint_lvl, train):
        if checkpoint_lvl not in (0, 1):
            raise ValueError(f"checkpoint_lvl must be 0 or 1, got {checkpoint_lvl!r}")
        if not x.is_cuda:
            raise RuntimeError("attention_fn: this build has no CPU path (x must be a CUDA tensor)")
        T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else x.dtype
        if T not in (torch.bfloat16, torch.float16):
            raise RuntimeError(f"attention_fn: activations must be bfloat16 or float16, directly or under autocast (got {T})")
        if x.dim() != 3 or x.numel() == 0:
            raise RuntimeError(f"attention_fn: x must be a non-empty (B, N, C) tensor, got {tuple(x.shape)}")
        B, N, C = x.shape
        if C % num_heads or C // num_heads not in ATTN_HEAD_DIMS:
            raise RuntimeError(f"attention_fn: head dim C / num_heads = {C} / {num_heads} must be one of {ATTN_HEAD_DIMS}")
        if tuple(qkv_weight.shape) != (3 * C, C) or tuple(proj_weight.shape) != (C, C):
            raise RuntimeError(f"attention_fn: weights {tuple(qkv_weight.shape)} / {tuple(proj_weight.shape)} do not match C = {C}")
        x2 = _gemm.rows_in(x, T, C)
        ctx.sizes = (B, N, C, num_heads, T, checkpoint_lvl)
        qkv, o, lse = AttentionFn._attend(x2, qkv_weight, qkv_bias, ctx, train)
        y = _gemm.gemm_tn(o, proj_weight.to(T), proj_bias)
        if train:
            ctx.save_for_backward(x2, qkv_weight, qkv_bias, proj_weight, proj_bias, *([qkv, o, lse] if checkpoint_lvl == 0 else []))
            ctx.param_dtypes = tuple(None if t is None else t.dtype for t in (qkv_weight, qkv_bias, proj_weight, proj_bias))
        return y.view(B, N, C)

    @staticmethod
    def _attend(x2, qkv_weight, qkv_bias, ctx, train):
        """qkv = x W^T + b (bit-identical to gemm.linear), o and, when training, the logsumexp."""
        B, N, C, H, T, _ = ctx.sizes
        qkv = _gemm.gemm_tn(x2, qkv_weight.to(T), qkv_bias)
        o = torch.empty((B * N, C), dtype=T, device=x2.device)
        lse = torch.empty((B, H, N), dtype=torch.float32, device=x2.device) if train else None
        _lib.call("mia_attn_fwd", "attention_fn", x2.device, qkv.data_ptr(), o.data_ptr(), None if lse is None else lse.data_ptr(), B, N, H,
                  C // H, qkv.stride(0), o.stride(0), _lib.dtype_code(T))
        return qkv, o, lse

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        B, N, C, H, T, lvl = ctx.sizes
        x2, wq, bq, wp, bp, *keep = ctx.saved_tensors
        dev = x2.device
        need_x, need_wq, need_bq, need_wp, need_bp = ctx.needs_input_grad[:5]
        qkv, o, lse = keep if lvl == 0 else AttentionFn._attend(x2, wq, bq, ctx, True)
        dy2 = _gemm.rows_in(dy, T, C)
        do, dwp, dbp = _gemm.linear_backward(dy2, o, wp, bp, True, need_wp, need_bp, *ctx.param_dtypes[2:], T)   # dO = dy . Wp
        delta = torch.empty((B, H, N), dtype=torch.float32, device=dev)
        dqkv = torch.empty((B * N, 3 * C), dtype=T, device=dev)
        _lib.call("mia_attn_bwd", "attention_fn backward", dev, qkv.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                  dqkv.data_ptr(), B, N, H, C // H, qkv.stride(0), o.stride(0), do.stride(0), dqkv.stride(0), _lib.dtype_code(T))
        del qkv, o, lse, do, delta
        dx, dwq, dbq = _gemm.linear_backward(dqkv, x2, wq, bq, need_x, need_wq, need_bq, *ctx.param_dtypes[:2], T)
        return None if dx is None else dx.view(B, N, C), dwq, dbq, dwp, dbp, None, None, None


def attention_fn(x, qkv_weight, qkv_bias, proj_weight, proj_bias, num_heads, checkpoint_lvl=0):
    """timm's Attention for bf16 / fp16 CUDA activations (directly or under autocast) as one op: x (B, N, C), qkv_weight
    (3C, C), proj_weight (C, C), biases (3C) / (C) or None, head dim C / num_heads in ATTN_HEAD_DIMS.  checkpoint_lvl 0
    (default) keeps qkv, o and the logsumexp for the backward, 1 recomputes them; both give the same bits."""
    train = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, qkv_weight, qkv_bias, proj_weight, proj_bias))
    return AttentionFn.apply(x, qkv_weight, qkv_bias, proj_weight, proj_bias, num_heads, checkpoint_lvl, train)


def attention_eligible(attn: nn.Module, x: torch.Tensor) -> bool:
    """Whether an Attention runs as one op (attention_fn): CUDA tensors, bf16 / fp16 activations (directly or under autocast)
    and a head dim in ATTN_HEAD_DIMS, with or without grad."""
    T = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() and x.is_cuda else x.dtype
    return x.is_cuda and T in (torch.bfloat16, torch.float16) and attn.head_dim in ATTN_HEAD_DIMS and x.dim() == 3 and x.numel() > 0


class Mlp(nn.Module):
    """timm 0.9.2 ``layers.Mlp``: fc1 -> GELU -> fc2.  When a backward follows, bf16 / fp16 CUDA activations run it as one op
    (gemm.gelu_mlp_fn); every other case runs the composition, _forward_composed."""

    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features, in_features)

    def forward(self, x):
        if _gemm.gelu_mlp_eligible(self, x, True):
            return _gemm.gelu_mlp_fn(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias)
        return self._forward_composed(x)

    def _forward_composed(self, x):
        return _gemm.linear(_gemm.linear(x, self.fc1.weight, self.fc1.bias, _gemm.ACT_GELU), self.fc2.weight, self.fc2.bias)


class Block(nn.Module):
    """timm 0.9.2 ``vision_transformer.Block`` as mae.py:64-66, 82-84 builds it: x + attn(LN(x)); x + mlp(LN(x))."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, norm_layer=nn.LayerNorm, **_unused):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


# ---------------------------------------------------------------------------------------------------------
def _sincos_1d(dim, pos):
    omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=float) / (dim / 2.0))
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_2d_sincos_pos_embed(embed_dim, grid_size, cls_token=False):
    """pos_embed.py:20-35 (MAE's fixed 2-D sine-cosine table; w varies fastest in the first half)."""
    gh, gw = np.arange(grid_size, dtype=np.float32), np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(gw, gh), axis=0).reshape([2, 1, grid_size, grid_size])
    emb = np.concatenate([_sincos_1d(embed_dim // 2, grid[0]), _sincos_1d(embed_dim // 2, grid[1])], axis=1)
    return np.concatenate([np.zeros([1, embed_dim]), emb], axis=0) if cls_token else emb


class MaskedAutoencoderViT(nn.Module):
    """models/mae.py:41-387.  ``patch_embed_dims`` = (in_chans, embed, hidden) of the patch encoder; the reference hard-wires
    (1, 1024, 1024) (:57), which only matches ``embed_dim=1024`` (mae_vit_large); the default here follows ``embed_dim`` so
    that the other factories are constructible (a documented deviation, pass (1, 1024, 1024) for the literal behaviour)."""

    def __init__(self, img_size=1280, patch_size=64, in_chans=1, embed_dim=768, depth=12, num_heads=16, decoder_embed_dim=512,
                 decoder_depth=8, decoder_num_heads=16, mlp_ratio=4.0, norm_layer=nn.LayerNorm, norm_pix_loss=False, mask_ratio=0.75,
                 use_learnable_pos_emb=True, new_depth=6, patch_embed_dims=None):
        super().__init__()
        pe_in, pe_embed, pe_hidden = patch_embed_dims or (1, embed_dim, 1024)
        self.patch_embed = SmallPatchEmbed(pe_in, pe_embed, pe_hidden)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim), requires_grad=False)
        self.blocks = nn.ModuleList([Block(embed_dim, num_heads, mlp_ratio, qkv_bias=True, norm_layer=norm_layer) for _ in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.decoder_embed = nn.Linear(embed_dim, decoder_embed_dim, bias=True)
        self.apply(self._init_weights)
        self.mask_token = nn.Parameter(torch.zeros(1, 1, decoder_embed_dim))
        self.decoder_pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, decoder_embed_dim), requires_grad=False)
        self.decoder_blocks = nn.ModuleList([Block(decoder_embed_dim, decoder_num_heads, mlp_ratio, qkv_bias=True, norm_layer=norm_layer)
                                             for _ in range(decoder_depth)])
        self.decoder_norm = norm_layer(decoder_embed_dim)
        self.decoder_pred = nn.Linear(decoder_embed_dim, patch_size ** 2 * in_chans, bias=True)
        self.decoder_image = nn.Linear(196, 1, bias=True)       # present (unused) in the reference: kept for its checkpoints
        self.norm_pix_loss, self.use_learnable_pos_emb = norm_pix_loss, use_learnable_pos_emb
        self.initialize_weights()

    def initialize_weights(self):
        side = int(self.patch_embed.num_patches ** 0.5)
        self.pos_embed.data.copy_(torch.from_numpy(get_2d_sincos_pos_embed(self.pos_embed.shape[-1], side, cls_token=True)).float().unsqueeze(0))
        self.decoder_pos_embed.data.copy_(
            torch.from_numpy(get_2d_sincos_pos_embed(self.decoder_pos_embed.shape[-1], side, cls_token=True)).float().unsqueeze(0))
        w = self.patch_embed.proj.weight.data
        torch.nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        torch.nn.init.normal_(self.cls_token, std=0.02)
        torch.nn.init.normal_(self.mask_token, std=0.02)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            torch.nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    # ---- patches <-> image (:129-156) --------------------------------------------------------------------------------
    def patchify(self, imgs):
        p = self.patch_embed.patch_size[0]
        assert imgs.shape[2] == imgs.shape[3] and imgs.shape[2] % p == 0
        h = w = imgs.shape[2] // p
        x = imgs.reshape(imgs.shape[0], 1, h, p, w, p)
        return torch.einsum("nchpwq->nhwpqc", x).reshape(imgs.shape[0], h * w, p ** 2 * 1)

    def unpatchify(self, x):
        p = self.patch_embed.patch_size[0]
        h = w = int(x.shape[1] ** 0.5)
        assert h * w == x.shape[1]
        x = torch.einsum("nhwpqc->nchpwq", x.reshape(x.shape[0], h, w, p, p, 1))
        return x.reshape(x.shape[0], 1, h * p, h * p)

    # ---- masking (:158-253); `noise*` are optional pre-drawn uniforms (tests pin the reference's draws with them) ----------
    @staticmethod
    def _keep_and_mask(x, ids_shuffle, len_keep):
        N, L, D = x.shape
        ids_restore = torch.argsort(ids_shuffle, dim=1)
        x_masked = torch.gather(x, dim=1, index=ids_shuffle[:, :len_keep].unsqueeze(-1).repeat(1, 1, D))
        mask = torch.ones([N, L], device=x.device)
        mask[:, :len_keep] = 0
        return x_masked, torch.gather(mask, dim=1, index=ids_restore), ids_restore

    def random_masking(self, x, mask_ratio, noise=None):
        N, L, _ = x.shape
        noise = torch.rand(N, L, device=x.device) if noise is None else noise
        return self._keep_and_mask(x, torch.argsort(noise, dim=1), int(L * (1 - mask_ratio)))

    def random_masking_yiliao(self, x, mask_ratio_outer, mask_ratio_iner, noise_outer=None, noise_iner=None):
        """Context-aware masking: an inner rectangle of the token grid is masked at `mask_ratio_iner`, the rest at
        `mask_ratio_outer`; kept tokens = kept outer then kept inner (:184-253)."""
        N, L, _ = x.shape
        side = int(math.sqrt(L))
        label = torch.zeros(side, side)
        label[int(side * 0.25) + 1:int(side * 0.75) + 1, int(side * 0.125) + 1:int(side * 0.75) + 1] = 1
        flat = label.flatten()
        idx_out, idx_in = torch.nonzero(flat == 0).flatten().to(x.device), torch.nonzero(flat == 1).flatten().to(x.device)
        keep_out, keep_in = int(idx_out.numel() * (1 - mask_ratio_outer)), int(idx_in.numel() * (1 - mask_ratio_iner))
        noise_outer = torch.rand(N, idx_out.numel(), device=x.device) if noise_outer is None else noise_outer
        noise_iner = torch.rand(N, idx_in.numel(), device=x.device) if noise_iner is None else noise_iner
        sh_out = idx_out[torch.argsort(noise_outer, dim=1)]
        sh_in = idx_in[torch.argsort(noise_iner, dim=1)]
        ids_shuffle = torch.cat((sh_out[:, :keep_out], sh_in[:, :keep_in], sh_out[:, keep_out:], sh_in[:, keep_in:]), dim=1)
        return self._keep_and_mask(x, ids_shuffle, keep_out + keep_in)

    # ---- encoder / decoder / loss (:255-323) ----------------------------------------------------------------------
    def forward_encoder(self, x, mask_type, mask_ratio_outer, mask_ratio_iner, noise=None):
        x = self.patch_embed(x)
        x = x + self.pos_embed[:, 1:, :].to(x.dtype)
        if mask_type == 1:
            no, ni = noise if noise is not None else (None, None)
            x, mask, ids_restore = self.random_masking_yiliao(x, mask_ratio_outer, mask_ratio_iner, no, ni)
        else:
            x, mask, ids_restore = self.random_masking(x, mask_ratio_outer, noise)
        cls = (self.cls_token + self.pos_embed[:, :1, :]).to(x.dtype).expand(x.shape[0], -1, -1)
        x = torch.cat((cls, x), dim=1)
        for blk in self.blocks:
            x = blk(x)
        return self.norm(x), mask, ids_restore

    def forward_decoder(self, x, ids_restore):
        x = _gemm.linear(x, self.decoder_embed.weight, self.decoder_embed.bias)
        mask_tokens = self.mask_token.to(x.dtype).repeat(x.shape[0], ids_restore.shape[1] + 1 - x.shape[1], 1)
        x_ = torch.cat([x[:, 1:, :], mask_tokens], dim=1)
        x_ = torch.gather(x_, dim=1, index=ids_restore.unsqueeze(-1).repeat(1, 1, x.shape[2]))
        x = torch.cat([x[:, :1, :], x_], dim=1) + self.decoder_pos_embed.to(x.dtype)
        for blk in self.decoder_blocks:
            x = blk(x)
        feat = self.decoder_norm(x)
        return _gemm.linear(feat, self.decoder_pred.weight, self.decoder_pred.bias)[:, 1:, :], feat

    def forward_loss(self, imgs, pred, mask):
        target = self.patchify(imgs)
        if self.norm_pix_loss:
            target = (target - target.mean(dim=-1, keepdim=True)) / (target.var(dim=-1, keepdim=True) + 1.0e-6) ** 0.5
        return ((pred - target) ** 2).mean(dim=-1)              # per patch; the reference leaves the mask weighting to the caller (:319-321)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "cls_token", "mask_token"}

    def forward(self, imgs, mask_type, mask_ratio_outer, mask_ratio_iner, noise=None):
        latent, mask, ids_restore = self.forward_encoder(imgs, mask_type, mask_ratio_outer, mask_ratio_iner, noise)
        pred, _ = self.forward_decoder(latent, ids_restore)
        return self.forward_loss(imgs, pred.float(), mask), mask


def mae_vit_base_patch16_dec512d8b(**kwargs):
    return MaskedAutoencoderViT(patch_size=64, embed_dim=768, depth=12, num_heads=12, decoder_embed_dim=512, decoder_num_heads=16, mlp_ratio=4,
                                norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def mae_vit_large_patch16_dec512d8b(**kwargs):
    return MaskedAutoencoderViT(patch_size=64, embed_dim=1024, depth=24, num_heads=16, decoder_embed_dim=512, decoder_depth=8,
                                decoder_num_heads=16, mlp_ratio=4, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def mae_vit_huge_patch14_dec512d8b(**kwargs):
    return MaskedAutoencoderViT(patch_size=64, embed_dim=1280, depth=32, num_heads=16, decoder_embed_dim=512, decoder_depth=8,
                                decoder_num_heads=16, mlp_ratio=4, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


mae_vit_base_patch16 = mae_vit_base_patch16_dec512d8b
mae_vit_large_patch16 = mae_vit_large_patch16_dec512d8b
mae_vit_huge_patch14 = mae_vit_huge_patch14_dec512d8b
