#!/usr/bin/env python
"""The GELU MLP: the fused op (gemm.GeluMlpFn, DESIGN.md 3.15) against the composition it replaced (Mlp._forward_composed:
fc1 GEMM, torch gelu, fc2 GEMM, and an eager GELU backward), alternating in one process.

    python tools/gelu_mlp_bench.py [--rounds 5] [--iters 20] [--mae-batch 32] [--json OUT]

Cases (bf16 autocast over fp32 parameters, as in training):
* the vssm1_base (VMamba-B) MLP of each stage at b 32: (C, L) = (128, 3136), (256, 784), (512, 196), (1024, 49), H = 4 C;
* the MAE-L encoder MLP (1024 -> 4096) at 61 tokens and the decoder MLP (512 -> 2048) at 401 tokens, b 64;
* the whole vssm1_base VSSM (vssm_base_224.yaml, drop_path_rate 0) fwd + bwd at 224 x 224, b 32;
* the whole mae_vit_large_patch16_dec512d8b fwd + bwd (1280 x 1280, mask ratio 0.85) at --mae-batch.
Per implementation and case: median / min / max ms of fwd + bwd over `rounds` rounds (each the mean of `iters` steps by CUDA
events, after 3 warm-up steps; L2 not flushed), peak MB = torch.cuda.max_memory_allocated during one fwd + bwd minus what
was allocated before it, and saved MB = the unique storages autograd saves in one forward (saved_tensors_hooks), parameters
excluded.  The card's name, power limit and SM clock are read (nvidia-smi, read-only) in the same call, after each case."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from arm_mixer_bench import card, peak_mb, timed  # noqa: E402


def step_of(model, fwd):
    def step():
        for p in model.parameters():
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = fwd()
        y.float().sum().backward()
    return step


def saved_mb(model, run):
    params = {p.untyped_storage().data_ptr() for p in model.parameters()}
    saved = {}

    def pack(t):
        st = t.untyped_storage()
        if st.data_ptr() not in params:
            saved[st.data_ptr()] = st.nbytes()
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t), torch.autocast("cuda", dtype=torch.bfloat16):
        y = run()
    del y
    return sum(saved.values()) / 2 ** 20


def cases(mae_batch):
    from medical_image_analysis_b200 import mae, vmamba
    dev = torch.device("cuda")
    for C, L in ((128, 3136), (256, 784), (512, 196), (1024, 49)):
        yield f"vssm1_base MLP {C} -> {4 * C}, L {L}, b 32", lambda C=C: vmamba.Mlp(C, 4 * C).to(dev), lambda C=C, L=L: torch.randn(
            32, L, C, device=dev, requires_grad=True)
    yield "MAE-L encoder MLP 1024 -> 4096, 61 tokens, b 64", lambda: mae.Mlp(1024, 4096).to(dev), lambda: torch.randn(
        64, 61, 1024, device=dev, requires_grad=True)
    yield "MAE-L decoder MLP 512 -> 2048, 401 tokens, b 64", lambda: mae.Mlp(512, 2048).to(dev), lambda: torch.randn(
        64, 401, 512, device=dev, requires_grad=True)
    yield "vssm1_base VSSM fwd+bwd, 224x224, b 32", lambda: vmamba.VSSM(
        depths=[2, 2, 15, 2], dims=128, ssm_d_state=1, ssm_ratio=2.0, ssm_dt_rank="auto", ssm_conv=3, ssm_conv_bias=False,
        forward_type="v3noz", mlp_ratio=4.0, downsample_version="v3", patchembed_version="v2", drop_path_rate=0.0).to(dev), lambda: torch.randn(
        32, 3, 224, 224, device=dev)
    yield f"mae_vit_large_patch16_dec512d8b fwd+bwd, 1280x1280, b {mae_batch}", lambda: mae.mae_vit_large_patch16_dec512d8b(
        patch_embed_dims=(1, 1024, 1024)).to(dev), lambda: torch.randn(mae_batch, 1, 1280, 1280, device=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--mae-batch", type=int, default=32)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gelu_mlp_bench.py measures on a CUDA device"
    from medical_image_analysis_b200 import gemm
    eligible = gemm.gelu_mlp_eligible
    impls = {"fused": eligible, "composition": lambda *a: False}          # the composition is what the layer runs without the op
    rows = []
    for name, make_model, make_x in cases(args.mae_batch):
        torch.manual_seed(0)
        model, x = make_model(), make_x()
        if "mae_vit" in name:
            noise = torch.rand(x.shape[0], 400, device=x.device)
            fwd = lambda: model(x, 0, 0.85, 0.95, noise=noise)[0]
        else:
            fwd = lambda: model(x)
        step = step_of(model, fwd)
        res = {"case": name}
        ms = {k: [] for k in impls}
        for impl, fn in impls.items():                              # warm-up, peak and saved bytes
            gemm.gelu_mlp_eligible = fn
            for _ in range(3):
                step()
            res[impl] = {"peak_MB": round(peak_mb(step), 1), "saved_MB": round(saved_mb(model, fwd), 1)}
        for _ in range(args.rounds):                                # alternate the two in every round
            for impl, fn in impls.items():
                gemm.gelu_mlp_eligible = fn
                ms[impl].append(timed(step, args.iters))
        gemm.gelu_mlp_eligible = eligible
        for impl in impls:
            res[impl].update(ms_median=round(statistics.median(ms[impl]), 3), ms_min=round(min(ms[impl]), 3), ms_max=round(max(ms[impl]), 3),
                             ms_rounds=[round(v, 3) for v in ms[impl]])
        del model, x, step, fwd
        torch.cuda.empty_cache()
        res["card"] = card()
        rows.append(res)
        print(json.dumps(res), flush=True)
    out = {"rows": rows, "rounds": args.rounds, "iters": args.iters, "l2": "not flushed", "autocast": "bf16", "torch": torch.__version__}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
