"""Developer tool (GPU, -DMIA_DEBUG library): random shapes through the column-walk kernels against the other kernel families
(resident-row / chunk-parallel / warp-scan forward, backward without block states).  Both sides are CUDA, so the check is a
cross-family consistency check on many geometries (rows per tensor-map row 1 / 2 / 4, split groups, partial windows, groups,
flags), not a parity test -- those are in tests/.

    python tools/bwd_variants.py --build && python tools/fuzz_cw.py [n_cases] [seed] [--regime model]

--regime model draws the inputs from the `model` regime of tests/test_scan_ranges_gpu.py (softplus argument in about [-8, -1],
A = -(1 .. d_state) scaled per row: what SS2D / the ARM mixers initialise) instead of the reference's generators.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def main():
    import torch
    from medical_image_analysis_b200 import _lib
    _lib.LIB_PATH = os.path.join(ROOT, "medical_image_analysis_b200", "libmia_scan_dbg.so")
    from medical_image_analysis_b200 import scan_bwd, scan_fwd
    argv = sys.argv[1:]
    regime = None
    if "--regime" in argv:
        i = argv.index("--regime")
        regime = argv[i + 1]
        del argv[i:i + 2]
        assert regime == "model", "--regime takes: model"
        from tests.test_scan_ranges_gpu import range_inputs, to_gpu
    n_cases = int(argv[0]) if len(argv) > 0 else 60
    rng = random.Random(int(argv[1]) if len(argv) > 1 else 0)
    worst = {}
    bad = 0
    for case in range(n_cases):
        dt = rng.choice([torch.bfloat16, torch.bfloat16, torch.float16, torch.float32])
        G = rng.choice([1, 1, 2, 4])
        rpg = rng.choice([32, 64, 128, 128, 256])
        D = G * rpg
        L = 4 * rng.choice([1, 2, 3, 4, 5, 7, 8, 9, 12, 13, 16, 24, 25, 31, 32, 33, 49, 50, 51, 63, 64, 65, 100, 130])
        B = rng.choice([1, 2, 3, 5])
        of32 = dt != torch.float32 and rng.random() < 0.3
        has_D, has_bias, softplus = rng.random() < 0.8, rng.random() < 0.8, rng.random() < 0.8
        g = torch.Generator(device="cuda").manual_seed(case)
        u = torch.randn(B, D, L, device="cuda", generator=g).to(dt)
        delta = (0.5 * torch.rand(B, D, L, device="cuda", generator=g)).to(dt)
        A = -0.5 * torch.rand(D, 1, device="cuda", generator=g)
        Bm = torch.randn(B, G, 1, L, device="cuda", generator=g).to(dt)
        Cm = torch.randn(B, G, 1, L, device="cuda", generator=g).to(dt)
        Dv = torch.randn(D, device="cuda", generator=g) if has_D else None
        bias = 0.5 * torch.rand(D, device="cuda", generator=g) if has_bias else None
        dout = torch.randn(B, D, L, device="cuda", generator=g).to(torch.float32 if (of32 or dt == torch.float32) else dt)
        if regime == "model":
            softplus = True
            m = to_gpu(range_inputs("model", case, B, D, L, 1, G, D, has_D, False, has_bias, True, dt))
            u, delta, A, Bm, Cm, Dv, bias = m["u"], m["delta"], m["A"], m["B"], m["C"], m["D"], m["delta_bias"]
            dout = m["dout"].to(dout.dtype)
        for k in ("MIA_NO_CW_FWD", "MIA_FORCE_CW_FWD", "MIA_FORCE_CW_BWD", "MIA_NO_CW_BWD"):
            os.environ.pop(k, None)
        os.environ["MIA_FORCE_CW_FWD"] = "1"
        os.environ["MIA_FORCE_CW_BWD"] = "1"
        out, x, _, hblk = scan_fwd(u, delta, A, Bm, Cm, Dv, None, bias, softplus, of32, want_block_states=True)
        desc = dict(case=case, B=B, D=D, G=G, L=L, dtype=str(dt)[6:], of32=of32, D_=has_D, bias=has_bias, softplus=softplus, hblk=hblk is not None)
        if hblk is None:
            print(json.dumps({**desc, "skipped": "the column-walk forward did not take it"}), flush=True)
            continue
        grads = scan_bwd(u, delta, A, Bm, Cm, Dv, None, bias, dout, x, None, softplus, hblk=hblk)
        os.environ.pop("MIA_FORCE_CW_FWD")
        os.environ.pop("MIA_FORCE_CW_BWD")
        os.environ["MIA_NO_CW_FWD"] = "1"
        out2, x2, _, _ = scan_fwd(u, delta, A, Bm, Cm, Dv, None, bias, softplus, of32, want_block_states=True)
        grads2 = scan_bwd(u, delta, A, Bm, Cm, Dv, None, bias, dout, x2, None, softplus, hblk=None)
        torch.cuda.synchronize()
        tol = 2e-5 if (dt == torch.float32) else (1.6e-2 if dt == torch.bfloat16 else 2e-3)       # ~2 ulp of the storage dtype at the tensor's max
        diffs = {"out": rel(out, out2), "last": rel(x[:, :, -1, 1::2], x2[:, :, -1, 1::2])}
        for name, a_, b_ in zip(("du", "ddelta", "dA", "dB", "dC", "dD", "dbias"), grads, grads2):
            if a_ is not None:
                diffs[name] = rel(a_, b_)
        f32_names = {"last", "dA", "dD", "dbias"} | ({"out"} if of32 else set())
        ok = all(v <= (3e-4 if (k in f32_names or dt == torch.float32) else tol) for k, v in diffs.items())
        finite = all(torch.isfinite(t.float()).all().item() for t in [out] + [t for t in grads if t is not None])
        for k, v in diffs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if not ok or not finite:
            bad += 1
            print(json.dumps({**desc, "MISMATCH": True, "finite": finite, "diffs": diffs}), flush=True)
    print(json.dumps({"cases": n_cases, "mismatches": bad, "worst_rel_diff": worst}), flush=True)


if __name__ == "__main__":
    main()
