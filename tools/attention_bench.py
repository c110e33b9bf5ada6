#!/usr/bin/env python
"""MAE attention: the fused op (mae.AttentionFn, DESIGN.md 3.16) against Attention._forward_composed on SDPA's default backend,
and against the composition on SDPA's math backend under torch.use_deterministic_algorithms(True) (the reproducible option
without the op), alternating in one process.

    python tools/attention_bench.py [--rounds 5] [--iters 20] [--mae-batch 32] [--json OUT]

Cases (bf16 autocast over fp32 parameters, as in training):
* MAE-L encoder attention (C 1024, 16 heads, dh 64) at N 61 (mask 0.85) and N 101, b 64;
* MAE-L decoder attention (C 512, 16 heads, dh 32) at N 401, b 32;
* MAE-H encoder attention (C 1280, 16 heads, dh 80) at N 61, b 64;
* the whole mae_vit_large_patch16_dec512d8b fwd + bwd (1280 x 1280, mask ratio 0.85) at --mae-batch.
Per implementation and case: median / min / max ms of fwd + bwd over `rounds` rounds (each the mean of `iters` steps by CUDA
events, after 3 warm-up steps; L2 not flushed), peak MB above what was allocated before one fwd + bwd, and saved MB of one
forward (saved_tensors_hooks, parameters excluded).  For the layer cases, the attention kernels alone (mia_attn_fwd, then
mia_attn_bwd) in TFLOP/s of the algorithmic 4 B H N^2 dh forward and 10 B H N^2 dh backward.  The card's name, power limit
and SM clock are read (nvidia-smi, read-only) in the same call, after each case."""
import argparse
import contextlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from arm_mixer_bench import card, peak_mb, timed  # noqa: E402
from gelu_mlp_bench import saved_mb, step_of  # noqa: E402


@contextlib.contextmanager
def mode(impl):
    """The routing and flags of one implementation: the op forced on, SDPA's default backend, or SDPA's math backend under
    the deterministic flag."""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from medical_image_analysis_b200 import mae
    eligible, prev = mae.attention_eligible, torch.are_deterministic_algorithms_enabled()
    mae.attention_eligible = (lambda *a: True) if impl == "op" else (lambda *a: False)   # every case here is eligible
    try:
        if impl == "sdpa_math_deterministic":
            torch.use_deterministic_algorithms(True, warn_only=True)
            with sdpa_kernel(SDPBackend.MATH):
                yield
        else:
            yield
    finally:
        mae.attention_eligible = eligible
        torch.use_deterministic_algorithms(prev)


def kernel_tflops(B, N, H, dh, iters):
    """fwd and bwd TFLOP/s of the attention kernels alone on random bf16 inputs."""
    from medical_image_analysis_b200 import _lib
    C = H * dh
    qkv = torch.randn(B * N, 3 * C, device="cuda").bfloat16()
    do = torch.randn(B * N, C, device="cuda").bfloat16()
    o = torch.empty(B * N, C, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, N, device="cuda")
    delta = torch.empty_like(lse)
    dqkv = torch.empty_like(qkv)
    bf = _lib.MIA_BF16

    def fwd():
        _lib.call("mia_attn_fwd", "fwd", qkv.device, qkv.data_ptr(), o.data_ptr(), lse.data_ptr(), B, N, H, dh, 3 * C, C, bf)

    def bwd():
        _lib.call("mia_attn_bwd", "bwd", qkv.device, qkv.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                  dqkv.data_ptr(), B, N, H, dh, 3 * C, C, C, 3 * C, bf)

    flops = B * H * N * N * dh
    for _ in range(3):
        fwd()
        bwd()
    t_f, t_b = timed(fwd, iters), timed(bwd, iters)
    return {"fwd_ms": round(t_f, 4), "bwd_ms": round(t_b, 4), "fwd_TFLOPs": round(4 * flops / t_f / 1e9, 1),
            "bwd_TFLOPs": round(10 * flops / t_b / 1e9, 1)}


def cases(mae_batch):
    from medical_image_analysis_b200 import mae
    dev = torch.device("cuda")
    for label, C, N, B in (("MAE-L encoder", 1024, 61, 64), ("MAE-L encoder", 1024, 101, 64), ("MAE-L decoder", 512, 401, 32),
                           ("MAE-H encoder", 1280, 61, 64)):
        yield (f"{label} attention C {C}, 16 heads (dh {C // 16}), N {N}, b {B}", (B, N, 16, C // 16),
               lambda C=C: mae.Attention(C, num_heads=16, qkv_bias=True).to(dev), lambda C=C, N=N, B=B: torch.randn(B, N, C, device=dev, requires_grad=True))
    yield (f"mae_vit_large_patch16_dec512d8b fwd+bwd, 1280x1280, b {mae_batch}", None,
           lambda: mae.mae_vit_large_patch16_dec512d8b(patch_embed_dims=(1, 1024, 1024)).to(dev),
           lambda: torch.randn(mae_batch, 1, 1280, 1280, device=dev))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--mae-batch", type=int, default=32)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "attention_bench.py measures on a CUDA device"
    impls = ("op", "sdpa_default", "sdpa_math_deterministic")
    rows = []
    for name, shape, make_model, make_x in cases(args.mae_batch):
        torch.manual_seed(0)
        model, x = make_model(), make_x()
        if shape is None:
            noise = torch.rand(x.shape[0], 400, device=x.device)
            fwd = lambda: model(x, 0, 0.85, 0.95, noise=noise)[0]
        else:
            fwd = lambda: model(x)
        step = step_of(model, fwd)
        res = {"case": name}
        ms = {k: [] for k in impls}
        for impl in impls:                                          # warm-up, peak and saved bytes
            with mode(impl):
                for _ in range(3):
                    step()
                res[impl] = {"peak_MB": round(peak_mb(step), 1), "saved_MB": round(saved_mb(model, fwd), 1)}
        for _ in range(args.rounds):                                # alternate the three in every round
            for impl in impls:
                with mode(impl):
                    ms[impl].append(timed(step, args.iters))
        for impl in impls:
            res[impl].update(ms_median=round(statistics.median(ms[impl]), 3), ms_min=round(min(ms[impl]), 3), ms_max=round(max(ms[impl]), 3),
                             ms_rounds=[round(v, 3) for v in ms[impl]])
        if shape is not None:
            res["kernels"] = kernel_tflops(*shape, args.iters)
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
