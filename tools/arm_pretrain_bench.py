#!/usr/bin/env python
"""ARM pre-training model (arm_pretrain, DESIGN.md 3.17): the decoder's segment-causal cross-attention as one op against the
mirror's composition and against SDPA given the same additive mask, and the whole pre-training step with the op routed and
with routing disabled, alternating in one process.

    python tools/arm_pretrain_bench.py [--rounds 5] [--iters 20] [--batch 32] [--json OUT]

Cases (bf16 autocast over fp32 parameters, as in training):
* decoder cross-attention layer, C 512, 8 heads of 64, seg 16: N 128 at b 32 and b 128, N 384 at b 32;
* the whole arm_large_pz16 and arm_base_pz16 step (192 x 192, N 128) at --batch (C4's per-GPU batch: 256 over 8 GPUs).
Per implementation and case: median (min - max) ms of fwd + bwd over `rounds` rounds (each the mean of `iters` steps by CUDA
events after 3 warm-up steps), peak MiB above what was allocated before one fwd + bwd, and saved MiB of one forward.  For
the layer cases, the kernels alone (mia_xattn_fwd, then mia_xattn_bwd) in TFLOP/s counting only the visible (query, key)
pairs V = sum_i (i // seg + 1) seg (capped at N) per image and head: 4 V dh forward and 10 V dh backward.  For the whole
step, the largest difference between the two paths' losses and gradients.  The card's name, power limit and SM clock are
read (nvidia-smi, read-only) in the same call."""
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
import torch.nn.functional as F  # noqa: E402

from arm_mixer_bench import card, peak_mb, timed  # noqa: E402
from gelu_mlp_bench import saved_mb, step_of  # noqa: E402

SEG, DH = 16, 64


@contextlib.contextmanager
def routed(on):
    from medical_image_analysis_b200 import arm_pretrain
    eligible = arm_pretrain.cross_attention_eligible
    if not on:
        arm_pretrain.cross_attention_eligible = lambda *a: False
    try:
        yield
    finally:
        arm_pretrain.cross_attention_eligible = eligible


def visible_pairs(N, seg):
    return sum(min(N, (i // seg + 1) * seg) for i in range(N))


def kernel_tflops(B, N, H, iters):
    from medical_image_analysis_b200 import _lib
    C = H * DH
    q, kv, do = (torch.randn(B * N, c, device="cuda").bfloat16() for c in (C, 2 * C, C))
    o, dq = torch.empty_like(q), torch.empty_like(q)
    dkv = torch.empty_like(kv)
    lse, delta = (torch.empty(B, H, N, device="cuda") for _ in range(2))
    bf = _lib.dtype_code(torch.bfloat16)
    fwd = lambda: _lib.call("mia_xattn_fwd", "bench", q.device, q.data_ptr(), kv.data_ptr(), o.data_ptr(), lse.data_ptr(), B, N, H, DH, SEG, C, 2 * C, C, bf)
    bwd = lambda: _lib.call("mia_xattn_bwd", "bench", q.device, q.data_ptr(), kv.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                            dq.data_ptr(), dkv.data_ptr(), B, N, H, DH, SEG, C, 2 * C, C, C, C, 2 * C, bf)
    for f in (fwd, bwd):
        f()
    V = B * H * visible_pairs(N, SEG)
    return 4 * V * DH / timed(fwd, iters) / 1e9, 10 * V * DH / timed(bwd, iters) / 1e9


class SdpaCross(torch.nn.Module):
    """The layer with F.scaled_dot_product_attention (default backend) given the additive mask."""

    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, q_in, kv_in, mask):
        m = self.m
        B, N, C = q_in.shape
        q = F.linear(q_in, m.q.weight, m.q.bias).view(B, N, m.num_heads, DH).transpose(1, 2)
        k, v = F.linear(kv_in, m.kv.weight, m.kv.bias).view(B, N, 2, m.num_heads, DH).permute(2, 0, 3, 1, 4).unbind(0)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask.to(q.dtype))
        return F.linear(o.transpose(1, 2).reshape(B, N, C), m.proj.weight, m.proj.bias)


def measure(impls, rounds, iters):
    times = {k: [] for k in impls}
    for _, (step, _) in impls.items():
        for _ in range(3):
            step()
    for _ in range(rounds):
        for k, (step, _) in impls.items():
            times[k].append(timed(step, iters))
    out = {}
    for k, (step, saved) in impls.items():
        t = times[k]
        out[k] = dict(ms=statistics.median(t), min=min(t), max=max(t), peak_mib=peak_mb(step), saved_mib=saved())
    return out


def layer_case(B, N, rounds, iters):
    from medical_image_analysis_b200 import arm_pretrain
    C, H = 512, 8
    torch.manual_seed(0)
    m = arm_pretrain.CrossAttention(C, H, qkv_bias=True).cuda()
    sd = SdpaCross(m)
    mask = arm_pretrain.VisionMamba.mask_generate(N // 16, 16).cuda()
    q_in = torch.randn(B, N, C, device="cuda", requires_grad=True)
    kv_in = torch.randn(B, N, C, device="cuda", requires_grad=True)

    def impl(mod, on):
        run = lambda: mod(q_in, kv_in, mask)

        def step():
            with routed(on):
                step_of(m, run)()

        def saved():
            with routed(on):
                return saved_mb(m, run)
        return step, saved
    res = measure({"op": impl(m, True), "composition": impl(m, False), "sdpa": impl(sd, False)}, rounds, iters)
    fw, bw = kernel_tflops(B, N, H, iters)
    return dict(case=f"xattn C512 H8 N{N} b{B}", results=res, kernel_tflops=dict(fwd=fw, bwd=bw), card=card())


def model_case(name, B, rounds, iters):
    from medical_image_analysis_b200 import arm_pretrain
    torch.manual_seed(0)
    m = getattr(arm_pretrain, name)().cuda()
    img = torch.randn(B, 3, 192, 192, device="cuda")
    run = lambda: m(img)

    def impl(on):
        def step():
            with routed(on):
                step_of(m, run)()

        def saved():
            with routed(on):
                return saved_mb(m, run)
        return step, saved
    res = measure({"op": impl(True), "composition": impl(False)}, rounds, iters)
    grads = {}
    for on in (True, False):
        with routed(on):
            m.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = m(img)
            loss.float().mean().backward()
        grads[on] = [loss.detach().float()] + [p.grad.float() for p in m.parameters() if p.requires_grad]
    diff = max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) for a, b in zip(grads[True], grads[False]))
    return dict(case=f"{name} step b{B}", results=res, max_rel_diff_op_vs_composition=diff, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json")
    a = ap.parse_args()
    out = [layer_case(32, 128, a.rounds, a.iters), layer_case(128, 128, a.rounds, a.iters), layer_case(32, 384, a.rounds, a.iters),
           model_case("arm_large_pz16", a.batch, a.rounds, a.iters), model_case("arm_base_pz16", a.batch, a.rounds, a.iters)]
    for c in out:
        print(c["case"], "|", c["card"])
        for k, r in c["results"].items():
            print(f"  {k:12s} {r['ms']:8.3f} ms ({r['min']:.3f} - {r['max']:.3f})  peak {r['peak_mib']:8.1f} MiB  saved {r['saved_mib']:8.1f} MiB")
        if "kernel_tflops" in c:
            print(f"  kernels: fwd {c['kernel_tflops']['fwd']:.1f} TFLOP/s, bwd {c['kernel_tflops']['bwd']:.1f} TFLOP/s (visible pairs only)")
        if "max_rel_diff_op_vs_composition" in c:
            print(f"  largest |op - composition| / max|composition| over loss and gradients: {c['max_rel_diff_op_vs_composition']:.3e}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
