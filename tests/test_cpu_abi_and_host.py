"""CPU-only checks: the C-ABI library loads and exports what include/*.h declares, the ctypes mirror matches the C
struct, argument validation fails the way the reference's TORCH_CHECKs do, the drop-in registers the module names."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mia_selective_scan.h")


def _lib():
    from medical_image_analysis_b200 import _build, _lib
    if not os.path.exists(_lib.LIB_PATH):
        _build.build()
    return _lib.lib()


def test_library_exports_every_declared_symbol():
    """Every function any include/*.h declares is exported by libmia_scan.so."""
    import glob
    lib = _lib()
    names = set()
    for hdr in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        text = open(hdr).read()
        body = text[text.index('extern "C"'):]
        names |= set(re.findall(r"\b(mia_[a-z_0-9]+)\s*\(", body))
    names = sorted(names)
    assert {"mia_gemm_tn", "mia_gemm_last_error", "mia_cs_last_error"} <= set(names)
    assert {"mia_selective_scan_fwd", "mia_selective_scan_bwd", "mia_selective_scan_bwd_workspace", "mia_last_error",
            "mia_abi_version", "mia_ss_num_chunks", "mia_ss_chunk_len", "mia_launch_count"} <= set(names)
    for n in names:
        assert hasattr(lib, n), f"libmia_scan.so does not export {n}"


def test_struct_layout_matches_header(tmp_path):
    """Each ctypes mirror (mia_ss_params, mia_ssu_params, mia_bdl) has the C struct's size and every field at the C offset."""
    from medical_image_analysis_b200._lib import MiaBdl, MiaSSParams, MiaSSUParams
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    for mirror, ctype in ((MiaSSParams, "mia_ss_params"), (MiaSSUParams, "mia_ssu_params"), (MiaBdl, "mia_bdl")):
        src = tmp_path / f"{ctype}.c"
        fields = [f for f, _ in mirror._fields_]
        lines = "\n".join(f'printf("{f} %zu\\n", offsetof({ctype}, {f}));' for f in fields)
        src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mia_selective_scan.h"\nint main(){printf("size %zu\\n", '
                       f'sizeof({ctype}));' + lines + "return 0;}")
        exe = tmp_path / ctype
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
        out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
        assert int(out["size"]) == ctypes.sizeof(mirror), ctype
        for f in fields:
            assert int(out[f]) == getattr(mirror, f).offset, (ctype, f)


def _header_prototypes():
    """name -> (parameter types, return type) of every function in the extern "C" blocks of include/*.h."""
    import glob
    protos = {}
    for hdr in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        text = re.sub(r"/\*.*?\*/", "", open(hdr).read(), flags=re.S)
        body = text[text.index('extern "C"'):]
        for ret, name, params in re.findall(r"([A-Za-z_][\w ]*?\**)\s*\b(mia_\w+)\s*\(([^)]*)\)\s*;", body):
            params = [] if params.strip() == "void" else [re.sub(r"\s*\w+$", "", p.strip()) if not p.strip().endswith("*") else p.strip()
                                                          for p in params.split(",")]
            protos[name] = (params, ret.strip())
    return protos


def _ctype_of(decl):
    """The ctypes type a C parameter / return type maps to in the binding."""
    from medical_image_analysis_b200 import _lib
    decl = " ".join(decl.replace("*", " * ").split())
    if decl == "const char *":
        return ctypes.c_char_p
    structs = {"mia_ss_params": _lib.MiaSSParams, "mia_ssu_params": _lib.MiaSSUParams, "mia_bdl": _lib.MiaBdl}
    if decl.endswith("*"):
        base = decl.replace("const", "").replace("*", "").strip()
        return ctypes.POINTER(structs[base]) if base in structs else ctypes.c_void_p
    return {"int": ctypes.c_int, "long long": ctypes.c_longlong, "size_t": ctypes.c_size_t, "uint64_t": ctypes.c_uint64}[decl]


def test_binding_table_matches_header_prototypes():
    """_lib.ABI states, for every function include/*.h declares, the argtypes and restype of its prototype (a c_int where the
    header says long long would truncate silently) and an error getter that the table and the library both have."""
    from medical_image_analysis_b200 import _lib
    lib = _lib.lib()
    protos = _header_prototypes()
    assert len(protos) >= 30 and "mia_causal_conv1d_bwd_ex" in protos and "mia_gemm" in protos
    assert set(protos) == set(_lib.ABI), set(protos) ^ set(_lib.ABI)
    for name, (params, ret) in protos.items():
        argtypes, restype, getter = _lib.ABI[name]
        assert [_ctype_of(p) for p in params] == argtypes, name
        assert _ctype_of(ret) == restype, name
        assert getattr(lib, name).argtypes == argtypes and getattr(lib, name).restype == restype, name
        if getter is not None:
            assert params[-1].endswith("*") and ret == "int", name           # launches: trailing cuda_stream, rc
            assert _lib.ABI[getter] == ([], ctypes.c_char_p, None), name


def test_call_raises_with_the_entry_points_own_channel():
    """_lib.call reports a failure with the message of the entry point's own error channel, under the caller's prefix; these
    failures happen before any CUDA call, so device=None (no device, null stream) reaches them."""
    from medical_image_analysis_b200 import _lib
    _lib.lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p).value
    with pytest.raises(RuntimeError) as e:
        _lib.call("mia_dwconv2d_fwd", "dwconv2d_fwd", None, p, p, None, p, 1, 1, 1, 16384, 1, _lib.MIA_F32)
    assert str(e.value) == ("dwconv2d_fwd: dwconv2d_fwd: a 1 x 16384 float32 plane needs 262224 bytes of shared memory per block, "
                            "more than the 232448-byte (227 KB) limit (code -1)")
    ops = (_lib.MiaBdl * 1)(_lib.MiaBdl(p, 0, 0, 1))
    with pytest.raises(RuntimeError) as e:
        _lib.call("mia_causal_conv1d_fwd_ex", "causal_conv1d_fwd_ex", None, ctypes.byref(ops[0]), p, None, ops, 1, 0, 4, 8, 4, 1,
                  _lib.MIA_BF16)
    assert str(e.value) == "causal_conv1d_fwd_ex: causal_conv1d_fwd_ex: bad sizes (code -1)"
    with pytest.raises(RuntimeError) as e:                                    # the decode step reports on the scan's channel
        _lib.call("mia_selective_state_update", "selective_state_update", None, None)
    assert str(e.value) == "selective_state_update: selective_state_update: null params (code -1)"
    assert _lib.lib().mia_last_error() == b"selective_state_update: null params"
    with pytest.raises(RuntimeError) as e:                                    # ... and the decode conv on the conv channel
        _lib.call("mia_causal_conv1d_update", "causal_conv1d_update", None, None, p, p, None, p, 1, 4, 4, 1, 2, 2, 0, 0,
                  4, 16, 4, 1, 4, 1, 4)
    assert str(e.value) == "causal_conv1d_update: causal_conv1d_update: null x / conv_state / weight / out (code -1)"
    assert _lib.lib().mia_conv_last_error() == b"causal_conv1d_update: null x / conv_state / weight / out"


def test_cross_scan_rejects_unknown_dtype_without_gpu():
    lib = _lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.mia_cross_scan(p, p, 1, 1, 2, 2, 7, None) == -1
    assert lib.mia_cs_last_error() == b"cross scan / merge: dtype must be MIA_F32, MIA_F16 or MIA_BF16"
    assert lib.mia_silu_gate(p, p, p, 4, 7, 7, None) == -1
    assert lib.mia_cs_last_error() == b"silu_gate: dtype must be MIA_F32, MIA_F16 or MIA_BF16"


def test_chunk_geometry():
    lib = _lib()
    assert lib.mia_abi_version() == 2
    for L, (ch, n) in {1: (32, 1), 49: (64, 1), 128: (128, 1), 129: (256, 1), 196: (256, 1), 197: (256, 1), 256: (256, 1),
                       257: (256, 2), 6400: (256, 25)}.items():
        assert lib.mia_ss_chunk_len(L) == ch and lib.mia_ss_num_chunks(L) == n, L


def test_block_state_sizing_without_gpu():
    """ABI 2: mia_ss_block_state_floats is a pure function of the sizes (4 bytes per 16 row-tokens, d_state 1 with 32-row
    groups only); mia_ss_fwd_writes_block_states needs the device (and the buffers) and answers 0 without them."""
    from medical_image_analysis_b200._lib import MiaSSParams
    lib = _lib()
    p = MiaSSParams()
    p.batch, p.dim, p.seqlen, p.dstate, p.n_groups, p.delta_dim = 3, 128, 196, 1, 2, 128
    p.itype = p.otype = 2
    p.n_chunks = 1
    assert lib.mia_ss_block_state_floats(ctypes.byref(p)) == 3 * 128 * 13          # ceil(196 / 16) groups per row
    p.seqlen = 6400
    assert lib.mia_ss_block_state_floats(ctypes.byref(p)) == 3 * 128 * 400
    p.dstate = 16
    assert lib.mia_ss_block_state_floats(ctypes.byref(p)) == 0                      # the d_state 16 kernels do not use them
    p.dstate, p.dim, p.delta_dim, p.n_groups = 1, 96, 96, 2                         # 48 rows per group: not a multiple of 32
    assert lib.mia_ss_block_state_floats(ctypes.byref(p)) == 0
    assert lib.mia_ss_fwd_writes_block_states(ctypes.byref(p)) == 0
    assert lib.mia_ss_fwd_writes_block_states(None) == 0


def test_c_abi_validation_without_gpu():
    """Shape / dtype checks run before any CUDA call, so they are observable on a CPU box."""
    from medical_image_analysis_b200._lib import MiaSSParams
    lib = _lib()
    assert lib.mia_selective_scan_fwd(None, None) == -1
    p = MiaSSParams()
    p.batch, p.dim, p.seqlen, p.dstate, p.n_groups, p.delta_dim = 2, 6, 16, 1, 4, 6     # 6 % 4 != 0
    p.itype = p.otype = 0
    p.n_chunks = 1
    assert lib.mia_selective_scan_fwd(ctypes.byref(p), None) == -1
    assert b"n_groups" in lib.mia_last_error()
    p.n_groups, p.dstate = 2, 300
    assert lib.mia_selective_scan_fwd(ctypes.byref(p), None) == -1
    assert b"state dimension <= 256" in lib.mia_last_error()
    p.dstate, p.itype = 4, 7
    assert lib.mia_selective_scan_bwd(ctypes.byref(p), None) == -1
    assert b"float32, float16 or bfloat16" in lib.mia_last_error()


def test_gemm_validation_without_gpu():
    lib = _lib()
    buf = ctypes.create_string_buffer(64)
    ptr = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.mia_gemm_tn(None, None, None, None, 4, 4, 8, 8, 8, 4, 2, 2, 0, None) == -1
    assert lib.mia_gemm_tn(ptr, ptr, None, ptr, 4, 4, 8, 8, 8, 4, 0, 0, 0, None) == -1           # fp32 inputs
    assert b"bf16 or fp16" in lib.mia_gemm_last_error()
    assert lib.mia_gemm_tn(ptr, ptr, None, ptr, 4, 4, 12, 12, 12, 4, 2, 2, 0, None) == -1        # pitch not a multiple of 8
    assert b"multiples of 8" in lib.mia_gemm_last_error()
    assert lib.mia_gemm_tn(ptr, ptr, None, ptr, 4, 4, 8, 8, 8, 4, 2, 2, 9, None) == -1
    assert b"activation" in lib.mia_gemm_last_error()


def test_host_checks_raise_runtime_error():
    from medical_image_analysis_b200 import scan_fwd
    u = torch.randn(1, 4, 8)
    A = -torch.rand(4, 2)
    B = torch.randn(1, 1, 2, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        scan_fwd(u, u.clone(), A, B, B.clone())
    with pytest.raises(RuntimeError, match="float32"):
        scan_fwd(u.double(), u.clone(), A, B, B.clone())


def test_no_silent_fallback_when_library_missing(monkeypatch, tmp_path):
    from medical_image_analysis_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU / PyTorch fallback"):
        _lib.lib()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "medical_image_analysis_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f
                assert "ss_ref" not in text, f


def test_dropin_registers_reference_module_names():
    code = ("import medical_image_analysis_b200.dropin as d; d.install();"
            "import selective_scan_cuda_oflex as o, selective_scan_cuda_core as c, selective_scan_cuda as m;"
            "from mamba_ssm.ops.selective_scan_interface import selective_scan_fn, mamba_inner_fn, bimamba_inner_fn, mamba_inner_fn_no_out_proj;"
            "from causal_conv1d import causal_conv1d_fn, causal_conv1d_update;"
            "from mamba_ssm.utils.generation import GenerationMixin; from mamba_ssm.utils.hf import load_config_hf, load_state_dict_hf;"
            "assert callable(o.fwd) and callable(o.bwd) and callable(c.fwd) and callable(m.bwd); print('ok')")
    out = subprocess.check_output([sys.executable, "-c", code], cwd=ROOT, text=True)
    assert out.strip().endswith("ok")


def test_causal_conv1d_has_no_cpu_path():
    """causal_conv1d_fn is a CUDA kernel behind the C ABI (parity vs mamba_simple.py:673 in tests/test_causal_conv1d_gpu.py);
    like the scan it must fail loudly, not fall back, when it cannot run on the GPU."""
    import pytest
    from medical_image_analysis_b200.selective_scan_interface import causal_conv1d_fn
    conv = torch.nn.Conv1d(6, 6, 4, groups=6, padding=3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        causal_conv1d_fn(torch.randn(2, 6, 20), conv.weight.squeeze(1), conv.bias, "silu")


def test_dwconv2d_has_no_cpu_path():
    """SS2D's depth-wise conv kernel (csrc/dwconv2d.cu) is CUDA-only as well: a CPU tensor must raise, not fall back."""
    import pytest
    from medical_image_analysis_b200.vmamba import DWConv2dFn
    conv = torch.nn.Conv2d(4, 4, 3, padding=1, groups=4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        DWConv2dFn.apply(torch.randn(1, 4, 5, 5), conv.weight, conv.bias, True)
    with pytest.raises(RuntimeError, match="weight"):
        DWConv2dFn.apply(torch.randn(1, 4, 5, 5), torch.randn(4, 1, 5, 5), None, True)


def test_dwconv2d_rejects_planes_that_do_not_fit_without_gpu():
    """A thin plane whose blocks would need more than the 227 KB of shared memory a block may have is refused by the
    shape check, before any CUDA call (so the refusal names the limit instead of surfacing as a failed launch)."""
    lib = _lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.mia_dwconv2d_fwd(p, p, None, p, 1, 1, 1, 16384, 1, 0, None) == -1               # fp32 1 x 16384 forward
    assert lib.mia_dwconv2d_last_error() == (b"dwconv2d_fwd: a 1 x 16384 float32 plane needs 262224 bytes of shared memory "
                                             b"per block, more than the 232448-byte (227 KB) limit")
    assert lib.mia_dwconv2d_bwd(p, p, None, p, p, p, None, 2, 1, 4, 4096, 1, 0, None) == -1     # fp32 4 x 4096 backward
    assert b"262240 bytes" in lib.mia_dwconv2d_last_error() and b"dwconv2d_bwd" in lib.mia_dwconv2d_last_error()
    assert lib.mia_dwconv2d_bwd(p, p, None, p, p, p, None, 1, 1, 1, 16384, 1, 2, None) == -1    # bf16 1 x 16384 backward
    assert b"16-bit plane" in lib.mia_dwconv2d_last_error()


def test_model_regime_generator_and_oracles_agree():
    """The `model` regime of tests/test_scan_ranges_gpu.py lands where it claims (softplus argument within [-9, 0], A within
    [-32, -0.5]: what SS2D / the ARM mixers initialise), and there the two oracles - the reference's own arithmetic in fp32
    (oracle/selective_scan_ref.py, torch autograd) and the fp64 C restatement (oracle/ss_ref.c) - agree at fp32 level on the
    output, the last state and every gradient: the oracle is pinned in the range before it judges the kernels there."""
    from oracle import ss_ref_c
    from oracle.selective_scan_ref import selective_scan_ref_fwd_bwd
    from tests.parity import cmp_f32
    from tests.test_scan_ranges_gpu import range_inputs
    for has_bias, has_z, N, G, ddim in ((True, False, 1, 2, 8), (False, True, 16, 1, 8), (True, True, 4, 2, 2)):
        c = range_inputs("model", 50, 2, 8, 197, N, G, ddim, True, has_z, has_bias, True, torch.float32)
        x = c["delta"] + (c["delta_bias"].view(1, -1, 1) if has_bias else 0.0)
        q01, q99 = torch.quantile(x.flatten(), torch.tensor([0.01, 0.99])).tolist()
        assert -9.0 <= q01 and q99 <= 0.0, (q01, q99)
        assert c["A"].min() >= -32.0 and c["A"].max() <= -0.5
        args = (c["u"], c["delta"], c["A"], c["B"], c["C"], c["D"], c["z"], c["delta_bias"])
        ref32 = selective_scan_ref_fwd_bwd(*args, True, c["dout"])
        r_out, r_out_z, r_last = ss_ref_c.fwd(*args, True)
        ref64 = ss_ref_c.bwd(*args, c["dout"], True)
        tag = f"[oracles, model regime, bias{int(has_bias)} z{int(has_z)} N{N}] "
        cmp_f32(ref32["out"], r_out_z if has_z else r_out, tag + "out")
        cmp_f32(ref32["last_state"], r_last, tag + "last_state")
        for name in ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz"):
            if ref64[name] is not None:
                cmp_f32(ref32[name], ref64[name], tag + name)
