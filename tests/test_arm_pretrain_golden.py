"""The ARM pre-training model (arm_pretrain.VisionMamba) against vectors produced by executing the reference's own
models_pretrain.py (tests/golden/modules_arm_pretrain.npz, generator tests/golden/make_golden_pretrain.py): the toy model at
N 48 and N 128 and one DecoderBlock, in fp32 with the tolerances of the fp32 ARM cases of test_modules_golden.py; and the
state_dict names and shapes of the four factories.  Inputs and parameters come from tests/golden/pretrain_toy.py's seeds
(checked against the stored fingerprints); gradients are compared at its sampled entries."""
import os

import numpy as np
import pytest
import torch

from medical_image_analysis_b200 import arm_pretrain
from tests.golden import pretrain_toy as toy
from tests.test_modules_golden import _close, _t

RAW = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "modules_arm_pretrain.npz"))
KW = dict(rtol=5e-4, atol_rms=5e-4)


def _case(tag):
    return {k[len(tag) + 1:]: RAW[k] for k in RAW.files if k.startswith(tag + "|")}


def _image(img_size):
    return toy.image(img_size)


def _model(img_size):
    """The toy model with the seeded parameters; its fixed sin-cos tables and mask must be the reference's, bit for bit."""
    c = _case(f"vm{img_size}")
    torch.manual_seed(1000)
    m = arm_pretrain.VisionMamba(img_size=img_size, **toy.TOY)
    toy.fill_params(m, 1100)
    for n in ("pos_embed", "dec_pos_embed"):
        assert np.array_equal(getattr(m, n).detach().numpy(), c[f"table.{n}"]), n
    assert np.array_equal(m.mask.numpy(), c["mask"])
    assert abs(toy.param_sum(m) - float(c["param_sum"][0])) <= 1e-9 * float(c["param_sum"][0])
    return m, c


def _close_grads(m, c, tag):
    n_grads = 0
    for n, p in m.named_parameters():
        if p.requires_grad:
            assert p.grad is not None, n
            _close(toy.sample(n, p.grad), c[f"grad.{n}"], f"{tag} grad {n}", **KW)
            n_grads += 1
    assert n_grads == sum(k.startswith("grad.") for k in c)


@pytest.mark.gpu
@pytest.mark.parametrize("img_size", [128, 192])
def test_model_matches_reference(img_size):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m, c = _model(img_size)
    m = m.cuda()
    img = _image(img_size)
    assert abs(float(img.double().sum()) - float(c["img_sum"][0])) < 1e-9
    img = img.cuda().requires_grad_()
    loss = m(img)
    (loss * _t(c["w"]).cuda()).sum().backward()
    _close(loss, c["loss"], f"vm{img_size} loss", **KW)
    _close(toy.sample("dimg", img.grad), c["dimg"], f"vm{img_size} dimg", **KW)
    _close_grads(m, c, f"vm{img_size}")


@pytest.mark.gpu
def test_decoder_block_matches_reference():
    c = _case("dec")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(1400)
    blk = arm_pretrain.DecoderBlock(128, 2, 4, qkv_bias=True, qk_scale=None)
    toy.fill_params(blk, 1401)
    assert abs(toy.param_sum(blk) - float(c["param_sum"][0])) <= 1e-9 * float(c["param_sum"][0])
    blk = blk.cuda()
    q, kv, w = toy.decoder_inputs(48, 128)
    q, kv = q.cuda().requires_grad_(), kv.cuda().requires_grad_()
    out = blk(q, kv, _t(_case("vm128")["mask"]).cuda())
    (out * w.cuda()).sum().backward()
    _close(out, c["out"], "dec out", **KW)
    _close(q.grad, c["dq"], "dec dq", **KW)
    _close(kv.grad, c["dkv"], "dec dkv", **KW)
    _close_grads(blk, c, "dec")


@pytest.mark.parametrize("factory", ["arm_base_pz16", "arm_large_pz16", "arm_huge_pz16", "arm_base_pz16_1280"])
def test_factory_state_dict_matches_reference(factory):
    with torch.device("meta"):
        sd = getattr(arm_pretrain, factory)().state_dict()
    assert [f"{n}:{tuple(t.shape)}" for n, t in sd.items()] == list(RAW[f"sd.{factory}"])


def test_factories_accept_norm_pix_loss():
    with torch.device("meta"):
        m = arm_pretrain.arm_base_pz16(norm_pix_loss=True)
    assert m.mask.shape == (128, 128) and m.cluster_num == 8
    with torch.device("meta"):
        assert arm_pretrain.arm_base_pz16_1280(norm_pix_loss=False).mask.shape == (384, 384)


def test_load_pretrained_is_not_mirrored():
    with torch.device("meta"):
        m = arm_pretrain.arm_base_pz16()
    with pytest.raises(NotImplementedError):
        m.load_pretrained("x.npz")
