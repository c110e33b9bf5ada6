"""Golden vectors of the ARM pre-training model, produced by EXECUTING THE REFERENCE'S OWN MODULES on CPU.

    python tests/golden/make_golden_pretrain.py       # needs the reference tree; writes tests/golden/modules_arm_pretrain.npz

What runs unchanged from the reference (imported, not copied): CXPMRG_Bench_MambaXray_VL/pretrain/models_pretrain.py
(VisionMamba, DecoderBlock, CrossAttention, Mlp, the arm_* factories), its utils/pos_embed.py and ITS OWN
mamba_simple.py (Mamba with bimamba_type "None": the one-direction mixer through mamba_inner_fn).

Stubs and helpers are make_golden_modules.py's (install_stubs, install_mamba_stubs, to_np), unchanged: timm / einops-free
layers, selective_scan_fn = the reference's selective_scan_ref, and mamba_inner_fn evaluated by running the reference
Mamba's own slow path (use_fast_path=False) -- here pretrain's Mamba rather than the fine-tuning one.

Inputs are not stored: pretrain_toy.py regenerates the image, the DecoderBlock's inputs and every parameter from seeds
(parameters by name), and the file keeps their fingerprints.  Stored, fp32 on CPU:
  vm{img}|...   the toy VisionMamba (embed 32, depth 12, dec 128 = 2 heads of 64, d_state 4, batch 2) at img 128 (N 48) and
                192 (N 128): the image and parameter fingerprints, the loss vector (N,), the weights w of sum(loss * w),
                the reference's sin-cos tables and mask, and the image gradient and every parameter gradient at
                pretrain_toy.SAMPLES seeded entries each (all entries of smaller tensors);
  dec|...       one DecoderBlock (dim 128, 2 heads) with the model's mask at N 48: out, dq and dkv in full, w's seed
                fingerprint, and every parameter gradient sampled as above;
  sd.{factory}  the state_dict of each of the four factories as "name:shape" strings, built on the meta device.
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_modules as mgm  # noqa: E402
import pretrain_toy as toy  # noqa: E402

PRETRAIN = f"{mgm.REF}/CXPMRG_Bench_MambaXray_VL/pretrain"
FACTORIES = ("arm_base_pz16", "arm_large_pz16", "arm_huge_pz16", "arm_base_pz16_1280")


def import_pretrain():
    """The reference's pretrain models_pretrain / mamba_simple, with mamba_inner_fn evaluated by pretrain's own Mamba."""
    ssr = mgm.install_stubs()
    mgm.install_mamba_stubs(ssr)
    for name in ("mamba_simple", "models_mamba", "utils", "utils.pos_embed"):
        sys.modules.pop(name, None)
    sys.path.insert(0, PRETRAIN)
    ms = importlib.import_module("mamba_simple")
    assert os.path.dirname(ms.__file__) == PRETRAIN
    iface = sys.modules["mamba_ssm.ops.selective_scan_interface"]
    state = next(c.cell_contents for c in iface.mamba_inner_fn_no_out_proj.__closure__ if isinstance(c.cell_contents, dict))
    state["Mamba"] = ms.Mamba                    # the stubbed fused op now runs pretrain's slow path
    return importlib.import_module("models_pretrain")


def sampled(res, prefix, m):
    for n, p in m.named_parameters():
        if p.grad is not None:
            res[f"{prefix}{n}"] = mgm.to_np(toy.sample(n, p.grad))


def golden(mp):
    store = {}
    for k, img_size in enumerate((128, 192)):
        torch.manual_seed(1000)
        net = mp.VisionMamba(img_size=img_size, **toy.TOY)
        toy.fill_params(net, 1100)
        img = toy.image(img_size).requires_grad_()
        loss = net(img)
        w = torch.randn(loss.shape, generator=torch.Generator().manual_seed(1300 + k))
        (loss * w).sum().backward()
        res = {"img_sum": np.array([float(img.detach().double().sum())]), "param_sum": np.array([toy.param_sum(net)]), "loss": mgm.to_np(loss),
               "w": mgm.to_np(w), "dimg": mgm.to_np(toy.sample("dimg", img.grad)), "table.pos_embed": mgm.to_np(net.pos_embed),
               "table.dec_pos_embed": mgm.to_np(net.dec_pos_embed), "mask": mgm.to_np(net.mask)}
        sampled(res, "grad.", net)
        mgm.save(store, f"vm{img_size}", res, dict(toy.TOY, img_size=img_size))
        if img_size == 128:
            mask = net.mask
    torch.manual_seed(1400)
    blk = mp.DecoderBlock(128, 2, 4, qkv_bias=True, qk_scale=None)
    toy.fill_params(blk, 1401)
    q, kv, w = toy.decoder_inputs(mask.shape[0], 128)
    q, kv = q.requires_grad_(), kv.requires_grad_()
    out = blk(q, kv, mask)
    (out * w).sum().backward()
    res = {"param_sum": np.array([toy.param_sum(blk)]), "out": mgm.to_np(out), "dq": mgm.to_np(q.grad), "dkv": mgm.to_np(kv.grad)}
    sampled(res, "grad.", blk)
    mgm.save(store, "dec", res, dict(dim=128, num_heads=2, mlp_ratio=4, qkv_bias=True))
    for name in FACTORIES:
        with torch.device("meta"):
            sd = getattr(mp, name)(norm_pix_loss=True).state_dict()
        store[f"sd.{name}"] = np.array([f"{n}:{tuple(t.shape)}" for n, t in sd.items()])
    np.savez_compressed(os.path.join(HERE, "modules_arm_pretrain.npz"), **store)
    print("modules_arm_pretrain:", len(store), "arrays")


if __name__ == "__main__":
    assert os.path.isdir(mgm.REF), "needs the reference tree"
    torch.set_num_threads(8)
    golden(import_pretrain())
