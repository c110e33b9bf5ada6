"""Developer tool (GPU): time the backward kernel families against each other on the headline shapes and check they agree.

Needs a -DMIA_DEBUG build of the library (the release library reads no environment variable):
    python tools/bwd_variants.py --build     # here (nvcc): writes medical_image_analysis_b200/libmia_scan_dbg.so
    python tools/bwd_variants.py             # on the GPU box: one JSON line per (shape, variant)
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = os.path.join(ROOT, "medical_image_analysis_b200")
DBG = os.path.join(PKG, "libmia_scan_dbg.so")


def build_debug():
    from medical_image_analysis_b200 import _build
    _build.build()
    nvcc = _build._nvcc()
    obj = os.path.join(PKG, "build", "scan_api_dbg.o")
    subprocess.check_call([nvcc, *[f for f in _build.NVCC_FLAGS if f not in ("-Xptxas", "-v")], "-DMIA_DEBUG", "-c",
                           os.path.join(PKG, "csrc", "scan_api.cu"), "-o", obj])
    objs = [os.path.join(PKG, "build", s.replace(".cu", ".o")) for s in _build.SOURCES if s != "scan_api.cu"] + [obj]
    subprocess.check_call([nvcc, "-shared", "-o", DBG, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    print(DBG)


VARIANTS = {
    "default": {},
    "no_cw": {"MIA_NO_CW_BWD": "1"},
    "no_hblk": None,          # backward without block states: resident-row / warp-scan kernels
}
for _ns in (2, 3):
    VARIANTS[f"cw_ns{_ns}_cap8"] = {"MIA_FORCE_CW_BWD": "1", "MIA_CW_STAGES": str(_ns), "MIA_CW_MAXPERSM": "8"}


def main():
    import torch
    from medical_image_analysis_b200 import _lib
    _lib.LIB_PATH = DBG
    from medical_image_analysis_b200 import scan_bwd, scan_fwd
    shapes = [(132, 196, torch.bfloat16, False), (64, 196, torch.bfloat16, False), (16, 6400, torch.bfloat16, False),
              (4, 6400, torch.bfloat16, False), (64, 196, torch.bfloat16, True), (32, 196, torch.float32, False), (8, 1024, torch.bfloat16, False)]
    D, G = 3072, 4
    for arg in sys.argv:
        if arg.startswith("--shape="):                                 # --shape=B,L,D,G  (bf16)
            b_, l_, D, G = (int(v) for v in arg.split("=")[1].split(","))
            shapes = [(b_, l_, torch.bfloat16, False)]
    if "--small" in sys.argv:
        shapes = [(2, 260, torch.bfloat16, False), (2, 196, torch.bfloat16, False), (2, 264, torch.bfloat16, False), (2, 196, torch.float32, False)]
        D, G = 64, 2
    for B, L, dt, of32 in shapes:
        g = torch.Generator(device="cuda").manual_seed(1)
        u = torch.randn(B, D, L, device="cuda", generator=g).to(dt)
        delta = (0.5 * torch.rand(B, D, L, device="cuda", generator=g)).to(dt)
        A = -0.5 * torch.rand(D, 1, device="cuda", generator=g)
        Bm = torch.randn(B, G, 1, L, device="cuda", generator=g).to(dt)
        Cm = torch.randn(B, G, 1, L, device="cuda", generator=g).to(dt)
        Dv = torch.randn(D, device="cuda", generator=g)
        bias = 0.5 * torch.rand(D, device="cuda", generator=g)
        dout = torch.randn(B, D, L, device="cuda", generator=g).to(torch.float32 if of32 else dt)
        fbase = None
        fvars = [("fwd_default", {}), ("fwd_no_cw", {"MIA_NO_CW_FWD": "1"})]
        for _ns in (3, 4):
            for _cap in (8, 12, 16):
                fvars.append((f"fwd_cw_ns{_ns}_cap{_cap}", {"MIA_CW_STAGES": str(_ns), "MIA_CW_MAXPERSM": str(_cap)}))
        for name, env in fvars:
            for k in ("MIA_NO_CW_FWD", "MIA_CW_STAGES", "MIA_FORCE_CW_FWD", "MIA_CW_MAXPERSM"):
                os.environ.pop(k, None)
            os.environ.update(env)
            runf = lambda: scan_fwd(u, delta, A, Bm, Cm, Dv, None, bias, True, of32, want_block_states=True)
            res = runf()
            for _ in range(3):
                runf()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                runf()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            diff = None
            if fbase is None:
                fbase = res[0].float().clone()
            else:
                diff = float((res[0].float() - fbase).abs().max())
            byt = B * D * L * (u.element_size() * 2 + res[0].element_size())
            print(json.dumps({"B": B, "L": L, "dtype": str(dt), "of32": of32, "variant": name, "ms": round(ms, 4),
                              "GBps": round(byt / ms / 1e6, 1), "max_abs_diff_vs_default": diff, "hblk": res[3] is not None}), flush=True)
        for k in ("MIA_NO_CW_FWD", "MIA_CW_STAGES", "MIA_FORCE_CW_FWD", "MIA_CW_MAXPERSM"):
            os.environ.pop(k, None)
        out, x, _, hblk = scan_fwd(u, delta, A, Bm, Cm, Dv, None, bias, True, of32, want_block_states=True)
        base = None
        for name, env in VARIANTS.items():
            for k in ("MIA_FORCE_CW_BWD", "MIA_NO_CW_BWD", "MIA_CW_STAGES", "MIA_CW_MAXPERSM"):
                os.environ.pop(k, None)
            if env:
                os.environ.update(env)
            hb = None if env is None else hblk
            run = lambda: scan_bwd(u, delta, A, Bm, Cm, Dv, None, bias, dout, x, None, True, hblk=hb)
            try:
                res = run()
            except Exception as e:                                    # noqa: BLE001
                print(json.dumps({"B": B, "L": L, "dtype": str(dt), "of32": of32, "variant": name, "error": str(e)[:200]}), flush=True)
                continue
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            diff = None
            if base is None:
                base = [t.float().clone() for t in res if t is not None]
            else:
                diff = max(float((t.float() - b).abs().max() / b.abs().max().clamp_min(1e-20)) for t, b in zip([t for t in res if t is not None], base))
            es = u.element_size()
            byt = B * D * L * (es * 4 + dout.element_size())
            print(json.dumps({"B": B, "L": L, "dtype": str(dt), "of32": of32, "variant": name, "ms": round(ms, 4),
                              "GBps": round(byt / ms / 1e6, 1), "max_rel_diff_vs_default": diff}), flush=True)


if __name__ == "__main__":
    if "--build" in sys.argv:
        build_debug()
    else:
        main()
