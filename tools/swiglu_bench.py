#!/usr/bin/env python
"""ARM's SwiGLU MLP: the fused op (arm.SwiGLUFn, DESIGN.md 3.14) against the composition it replaced (arm.SwiGLU._forward_composed:
two GEMMs, torch silu and mul, the w3 GEMM), alternating in one process.

    python tools/swiglu_bench.py [--rounds 5] [--iters 20] [--json OUT]

Cases (bf16 autocast over fp32 parameters, as in training; L 197):
* the arm_base_pz16 SwiGLU layer (768 -> 2048 -> 768) at b 32 and b 64;
* the arm_large_pz16 SwiGLU layer (1024 -> 2730 -> 1024) at b 32;
* the whole arm_base_pz16 encoder fwd + bwd at b 32, 224 x 224 (bench.py's module_timings case).
Per implementation and case: median / min / max ms of fwd + bwd over `rounds` rounds (each the mean of `iters` steps by CUDA
events, after 3 warm-up steps; L2 not flushed), peak MB = torch.cuda.max_memory_allocated during one fwd + bwd minus what
was allocated before it, and saved MB = the unique storages autograd saves in one forward (saved_tensors_hooks), parameters
excluded.  For the three layer shapes it also times the dual GEMM alone (mia_gemm_swiglu_fwd writing h and the packed
a / b) against two gemm_tn calls with bias at the same shapes, and reports both in TFLOP/s (4 M H K flops).  The card's
name, power limit and SM clock are read (nvidia-smi, read-only) in the same call, after each case."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from arm_mixer_bench import card, peak_mb, saved_mb, step_of, timed  # noqa: E402


def gemm_rates(d, H, b, rounds, iters):
    """TFLOP/s of the dual GEMM (median of rounds) against two gemm_tn calls with bias, bf16."""
    from medical_image_analysis_b200 import _lib, gemm
    from medical_image_analysis_b200.arm import _pad64
    dev = torch.device("cuda")
    M, Hp = b * 197, _pad64(H)
    x = torch.randn(M, d, device=dev).bfloat16()
    w1, w2 = (torch.randn(H, d, device=dev).bfloat16() * d ** -0.5 for _ in range(2))
    b1, b2 = (torch.randn(H, device=dev) * 0.1 for _ in range(2))
    h = torch.empty(M, Hp, device=dev, dtype=torch.bfloat16)
    ab = torch.empty(M, 2 * Hp, device=dev, dtype=torch.bfloat16)

    def dual():
        _lib.call("mia_gemm_swiglu_fwd", "swiglu", dev, x.data_ptr(), w1.data_ptr(), w2.data_ptr(), b1.data_ptr(), b2.data_ptr(), h.data_ptr(),
                  ab.data_ptr(), M, H, d, d, d, d, Hp, 2 * Hp, _lib.MIA_BF16)

    def two():
        gemm.gemm_tn(x, w1, b1)
        gemm.gemm_tn(x, w2, b2)

    flops = 4.0 * M * H * d
    ms = {"dual": [], "2 x gemm_tn": []}
    for f in (dual, two):
        for _ in range(3):
            f()
    for _ in range(rounds):
        for k, f in (("dual", dual), ("2 x gemm_tn", two)):
            ms[k].append(timed(f, iters))
    return {k: {"tflops_median": round(flops / statistics.median(v) / 1e9, 1), "tflops_min": round(flops / max(v) / 1e9, 1),
                "tflops_max": round(flops / min(v) / 1e9, 1)} for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "swiglu_bench.py measures on a CUDA device"
    from medical_image_analysis_b200 import arm
    dev = torch.device("cuda")
    fused_ok = arm.SwiGLU._fused_ok
    impls = {"fused": fused_ok, "composition": lambda self, x: False}      # the composition is what the layer runs without the op
    cases = [("arm_base_pz16 SwiGLU, b 32", "mlp", 768, 2048, 32), ("arm_base_pz16 SwiGLU, b 64", "mlp", 768, 2048, 64),
             ("arm_large_pz16 SwiGLU, b 32", "mlp", 1024, 2730, 32), ("arm_base_pz16 encoder fwd+bwd, b 32, 224x224", "encoder", 768, 2048, 32)]
    rows = []
    for name, kind, d, H, b in cases:
        torch.manual_seed(0)
        if kind == "mlp":
            model = arm.SwiGLU(d, H).to(dev)
            x = torch.randn(b, 197, d, device=dev, requires_grad=True)
        else:
            model = arm.arm_base_pz16(drop_path_rate=0.0).to(dev)
            x = torch.randn(b, 3, 224, 224, device=dev)
        step = step_of(model, x)
        res = {"case": name}
        ms = {k: [] for k in impls}
        for impl, fn in impls.items():                              # warm-up, peak and saved bytes
            arm.SwiGLU._fused_ok = fn
            for _ in range(3):
                step()
            res[impl] = {"peak_MB": round(peak_mb(step), 1), "saved_MB": round(saved_mb(model, x), 1)}
        for _ in range(args.rounds):                                # alternate the two in every round
            for impl, fn in impls.items():
                arm.SwiGLU._fused_ok = fn
                ms[impl].append(timed(step, args.iters))
        arm.SwiGLU._fused_ok = fused_ok
        for impl in impls:
            res[impl].update(ms_median=round(statistics.median(ms[impl]), 3), ms_min=round(min(ms[impl]), 3), ms_max=round(max(ms[impl]), 3),
                             ms_rounds=[round(v, 3) for v in ms[impl]])
        del model, x, step
        torch.cuda.empty_cache()
        if kind == "mlp":
            res["gemm"] = gemm_rates(d, H, b, args.rounds, args.iters)
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
