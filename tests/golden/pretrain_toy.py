"""Inputs of the ARM pre-training golden cases, regenerated from seeds rather than stored (tests/golden/make_golden_pretrain.py
writes modules_arm_pretrain.npz; tests/test_arm_pretrain_golden.py reads it).  Parameters are filled by NAME, so the
reference's modules and this repository's mirror, which share every parameter name and shape, get the same values
whatever order they create them in.  Gradients are stored at SAMPLES entries per tensor, chosen the same way."""
import math
import zlib

import torch

TOY = dict(patch_size=16, stride=16, embed_dim=32, depth=12, dec_embed_dim=128, rms_norm=True, residual_in_fp32=True, fused_add_norm=True,
           if_abs_pos_embed=True, bimamba_type="None", drop_path_rate=0.0, ssm_cfg=dict(d_state=4))
SAMPLES = 256


def _gen(name, seed):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()) ^ seed)


def fill_params(m, seed):
    """Generic values for every trainable parameter of m (the fixed sin-cos tables are left as built): A_log in
    log([0.2, 1.7)), LayerNorm weights 1 + 0.2 N(0, 1), other vectors 0.3 N(0, 1), matrices N(0, 1 / fan_in)."""
    with torch.no_grad():
        for n, p in m.named_parameters():
            if not p.requires_grad:
                continue
            g = _gen(n, seed)
            if "A_log" in n:
                p.copy_(torch.log(0.2 + 1.5 * torch.rand(p.shape, generator=g)))
            elif p.dim() == 1 and "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(0.3 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(max(p[0].numel(), 1)))


def param_sum(m):
    """float64 sum of |p| over every parameter: the stored fingerprint of what fill_params produced."""
    return float(sum(p.detach().double().abs().sum() for p in m.parameters()))


def sample(name, t):
    """The flattened entries of t at the SAMPLES positions chosen for `name` (every entry when t is smaller)."""
    flat = t.detach().reshape(-1)
    if flat.numel() <= SAMPLES:
        return flat
    idx = torch.randperm(flat.numel(), generator=_gen(name, 0))[:SAMPLES].sort().values
    return flat[idx.to(flat.device)]


def image(img_size):
    return torch.randn(2, 3, img_size, img_size, generator=torch.Generator().manual_seed(1200 + img_size))


def decoder_inputs(N, dim):
    g = torch.Generator().manual_seed(1402)
    return torch.randn(2, N, dim, generator=g), torch.randn(2, N, dim, generator=g), torch.randn(2, N, dim, generator=g)
