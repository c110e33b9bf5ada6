"""Builds libmia_scan.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a.

Used by ``__graft_entry__.build()`` and by developers; the product never JIT-compiles at import time, it
loads the prebuilt in-tree ``.so`` and fails loudly when it is missing (see ``_lib.py``).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
SOURCES = ["scan_fwd_bf16.cu", "scan_fwd_f16.cu", "scan_fwd_f32.cu", "scan_bwd_bf16.cu", "scan_bwd_f16.cu", "scan_bwd_f32.cu",
           "scan_api.cu", "cross_scan.cu", "causal_conv1d.cu", "dwconv2d.cu", "gemm_wgmma.cu", "ssm_step.cu",
           "ss2d_core.cu", "attention.cu", "abi_host.cu"]
HEADERS = sorted(f for f in os.listdir(os.path.join(PKG, "csrc")) if f.endswith((".cuh", ".h"))) + [os.path.join("..", "..", "include", "mia_selective_scan.h"), os.path.join("..", "..", "include", "mia_gemm.h")]
LIB = os.path.join(PKG, "libmia_scan.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libmia_scan.so")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    os.makedirs(os.path.join(PKG, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(PKG, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
    link = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    out = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"link failed:\n{out.stdout}")
    with open(os.path.join(PKG, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(l for l in "\n".join(log).splitlines() if "registers" in l or "spill" in l or "Compiling" in l))
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(LIB)
