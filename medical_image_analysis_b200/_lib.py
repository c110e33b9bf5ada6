"""ctypes binding of the C ABI in include/mia_selective_scan.h (libmia_scan.so).

There is deliberately NO fallback: if the CUDA library is missing or fails, every op raises.
"""
from __future__ import annotations

import ctypes
import os

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libmia_scan.so")

MIA_F32, MIA_F16, MIA_BF16 = 0, 1, 2
MIA_ORDER_SEQ, MIA_ORDER_SEQ_REV, MIA_ORDER_COL, MIA_ORDER_COL_REV = 0, 1, 2, 3

_vp, _i32, _i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64


class MiaSSParams(ctypes.Structure):
    """Field-for-field mirror of ``struct mia_ss_params``."""
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "seqlen", "dstate", "n_groups", "delta_dim", "itype", "otype",
                             "delta_softplus", "n_chunks")]
        + [(n, _vp) for n in ("u", "delta", "A", "B", "C", "D", "delta_bias", "z")]
        + [(n, _i64) for n in ("u_batch_stride", "u_d_stride", "delta_batch_stride", "delta_d_stride",
                               "A_d_stride", "A_dstate_stride", "B_batch_stride", "B_group_stride", "B_dstate_stride",
                               "C_batch_stride", "C_group_stride", "C_dstate_stride", "z_batch_stride", "z_d_stride")]
        + [(n, _vp) for n in ("out", "out_z", "x")]
        + [(n, _i64) for n in ("out_batch_stride", "out_d_stride", "out_z_batch_stride", "out_z_d_stride")]
        + [(n, _vp) for n in ("dout", "out_saved")]
        + [(n, _i64) for n in ("dout_batch_stride", "dout_d_stride", "out_saved_batch_stride", "out_saved_d_stride")]
        + [(n, _vp) for n in ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz")]
        + [(n, _i64) for n in ("du_batch_stride", "du_d_stride", "ddelta_batch_stride", "ddelta_d_stride",
                               "dA_d_stride", "dA_dstate_stride", "dB_batch_stride", "dB_group_stride", "dB_dstate_stride",
                               "dC_batch_stride", "dC_group_stride", "dC_dstate_stride", "dz_batch_stride", "dz_d_stride")]
        + [("workspace", _vp), ("workspace_bytes", ctypes.c_size_t), ("hblk", _vp)]
    )


class MiaSSUParams(ctypes.Structure):
    """Field-for-field mirror of ``struct mia_ssu_params`` (the decode step)."""
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "dstate", "state_type", "itype", "D_type", "dt_bias_type", "dt_softplus")]
        + [(n, _vp) for n in ("state", "x", "dt", "z", "B", "C", "A", "D", "dt_bias", "out")]
        + [(n, _i64) for n in ("state_batch_stride", "state_d_stride", "x_batch_stride", "dt_batch_stride", "z_batch_stride",
                               "B_batch_stride", "C_batch_stride", "out_batch_stride", "A_d_stride", "A_dstate_stride")]
    )


class MiaBdl(ctypes.Structure):
    """Mirror of ``struct mia_bdl``: a (batch, dim, seqlen) operand with element strides (the fused inner block's kernels)."""
    _fields_ = [("ptr", _vp), ("batch_stride", _i64), ("d_stride", _i64), ("seq_stride", _i64)]


class MiaLn(ctypes.Structure):
    """Mirror of ``struct mia_ln``: LayerNorm weight / bias (fp32 device pointers) and eps (the SS2D core epilogue)."""
    _fields_ = [("weight", _vp), ("bias", _vp), ("eps", ctypes.c_float)]


_I, _LL, _SZ, _STR = ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t, ctypes.c_char_p
_SS, _SSU, _BDL = ctypes.POINTER(MiaSSParams), ctypes.POINTER(MiaSSUParams), ctypes.POINTER(MiaBdl)
_LN = ctypes.c_void_p          # const mia_ln * (passed as ctypes.byref(MiaLn(...)))
_SCAN, _CONV, _CS, _DW, _GEMM = "mia_last_error", "mia_conv_last_error", "mia_cs_last_error", "mia_dwconv2d_last_error", "mia_gemm_last_error"

# Every function include/*.h declares: name -> (argtypes, restype, the getter of its error message or None).  The argtypes
# of an entry point that launches end with its cuda_stream, which call() supplies.
ABI = {
    "mia_abi_version": ([], _I, None),
    "mia_last_error": ([], _STR, None),
    "mia_conv_last_error": ([], _STR, None),
    "mia_cs_last_error": ([], _STR, None),
    "mia_dwconv2d_last_error": ([], _STR, None),
    "mia_gemm_last_error": ([], _STR, None),
    "mia_launch_count": ([], ctypes.c_uint64, None),
    "mia_ss_chunk_len": ([_I], _I, None),
    "mia_ss_num_chunks": ([_I], _I, None),
    "mia_ss_block_state_floats": ([_SS], _SZ, None),
    "mia_ss_fwd_writes_block_states": ([_SS], _I, None),
    "mia_selective_scan_fwd": ([_SS, _vp], _I, _SCAN),
    "mia_selective_scan_bwd_workspace": ([_SS], _SZ, None),
    "mia_selective_scan_bwd": ([_SS, _vp], _I, _SCAN),
    "mia_selective_scan_bwd_deterministic_workspace": ([_SS], _SZ, None),
    "mia_selective_scan_bwd_deterministic": ([_SS, _vp], _I, _SCAN),
    "mia_cross_scan": ([_vp, _vp] + [_I] * 5 + [_vp], _I, _CS),
    "mia_cross_merge": ([_vp, _vp] + [_I] * 5 + [_vp], _I, _CS),
    "mia_cross_scan_1b1": ([_vp, _vp] + [_I] * 5 + [_vp], _I, _CS),
    "mia_cross_merge_1b1": ([_vp, _vp] + [_I] * 5 + [_vp], _I, _CS),
    "mia_ss2d_merge_norm_fwd": ([_vp, _LN, _BDL, _I] + [_vp] * 4 + [_I] * 6 + [_vp], _I, _CS),
    "mia_ss2d_merge_norm_bwd_workspace": ([_I] * 4, _SZ, None),
    "mia_ss2d_merge_norm_bwd": ([_vp] * 4 + [_LN, _BDL, _I, _BDL] + [_vp] * 4 + [_SZ] + [_I] * 5 + [_vp], _I, _CS),
    "mia_silu_gate": ([_vp, _vp, _vp, _LL, _I, _I, _vp], _I, _CS),
    "mia_causal_conv1d_fwd": ([_vp] * 4 + [_I] * 6 + [_LL] * 4 + [_vp], _I, _CONV),
    "mia_causal_conv1d_bwd": ([_vp] * 7 + [_I] * 6 + [_LL] * 6 + [_vp], _I, _CONV),
    "mia_causal_conv1d_fwd_ex": ([_BDL, _vp, _vp, _BDL] + [_I] * 7 + [_vp], _I, _CONV),
    "mia_causal_conv1d_bwd_ex_workspace": ([_I] * 4, _SZ, None),
    "mia_causal_conv1d_bwd_ex": ([_BDL, _vp, _vp, _BDL, _I, _BDL, _vp, _vp, _vp, _SZ] + [_I] * 6 + [_vp], _I, _CONV),
    "mia_silu_gate_fwd_ex": ([_BDL, _I, _BDL, _BDL] + [_I] * 5 + [_vp], _I, _CONV),
    "mia_silu_gate_bwd_ex": ([_BDL, _BDL, _I, _BDL, _BDL, _I, _BDL] + [_I] * 5 + [_vp], _I, _CONV),
    "mia_causal_conv1d_fwd_dirs": ([_BDL, _vp, _I, _vp, _vp, _vp, _BDL] + [_I] * 6 + [_vp], _I, _CONV),
    "mia_causal_conv1d_bwd_dirs_workspace": ([_I] * 5, _SZ, None),
    "mia_causal_conv1d_bwd_dirs": ([_BDL, _vp, _I, _vp, _vp, _vp, _BDL, _BDL, _vp, _vp, _vp, _SZ] + [_I] * 6 + [_vp], _I, _CONV),
    "mia_silu_gate_fwd_dirs": ([_vp, _vp, _I, _I, _BDL, _BDL] + [_I] * 4 + [_vp], _I, _CONV),
    "mia_silu_gate_bwd_dirs": ([_BDL, _vp, _vp, _I, _I, _BDL, _vp, _BDL] + [_I] * 4 + [_vp], _I, _CONV),
    "mia_dwconv2d_fwd": ([_vp] * 4 + [_I] * 6 + [_vp], _I, _DW),
    "mia_dwconv2d_bwd": ([_vp] * 7 + [_I] * 6 + [_vp], _I, _DW),
    "mia_selective_state_update": ([_SSU, _vp], _I, _SCAN),
    "mia_causal_conv1d_update": ([_vp] * 5 + [_I] * 8 + [_LL] * 7 + [_vp], _I, _CONV),
    "mia_gemm_tn": ([_vp] * 4 + [_I] * 3 + [_LL] * 3 + [_I] * 3 + [_vp], _I, _GEMM),
    "mia_gemm": ([_vp] * 4 + [_I] * 3 + [_LL] * 3 + [_I] * 5 + [_vp], _I, _GEMM),
    "mia_gemm_swiglu_fwd": ([_vp] * 7 + [_I] * 3 + [_LL] * 5 + [_I, _vp], _I, _GEMM),
    "mia_gemm_swiglu_bwd": ([_vp] * 5 + [_I] * 3 + [_LL] * 5 + [_I, _vp], _I, _GEMM),
    "mia_gemm_gelu_fwd": ([_vp] * 5 + [_I] * 3 + [_LL] * 4 + [_I, _vp], _I, _GEMM),
    "mia_gemm_gelu_bwd": ([_vp] * 5 + [_I] * 3 + [_LL] * 5 + [_I, _vp], _I, _GEMM),
    "mia_attn_fwd": ([_vp] * 3 + [_I] * 4 + [_LL] * 2 + [_I, _vp], _I, _GEMM),
    "mia_attn_bwd": ([_vp] * 6 + [_I] * 4 + [_LL] * 4 + [_I, _vp], _I, _GEMM),
    "mia_xattn_fwd": ([_vp] * 4 + [_I] * 5 + [_LL] * 3 + [_I, _vp], _I, _GEMM),
    "mia_xattn_bwd": ([_vp] * 8 + [_I] * 5 + [_LL] * 6 + [_I, _vp], _I, _GEMM),
}

DTYPE_CODES = {torch.float32: MIA_F32, torch.float16: MIA_F16, torch.bfloat16: MIA_BF16}

_lib = None


def lib() -> ctypes.CDLL:
    """Load libmia_scan.so (built in-tree by ``python -m medical_image_analysis_b200._build``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the CUDA library has not been built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (or `python -m medical_image_analysis_b200._build`). "
                "There is no CPU / PyTorch fallback for the selective scan.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (argtypes, restype, _) in ABI.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = argtypes, restype
        if L.mia_abi_version() != 2:
            raise RuntimeError(f"libmia_scan.so ABI version {L.mia_abi_version()} != 2: rebuild it")
        _lib = L
    return _lib


def dtype_code(dtype: torch.dtype) -> int:
    """MIA_F32 / MIA_F16 / MIA_BF16 of a torch dtype (KeyError for any other)."""
    return DTYPE_CODES[dtype]


def call(name: str, what: str, device, *args) -> None:
    """The launch path of every entry point: runs ``name(*args, cuda_stream)`` with ``device`` current and its current stream
    as the trailing cuda_stream, and raises ``RuntimeError(f"{what}: <message> (code <rc>)")`` with the message of the
    entry point's own error channel when it fails.  device=None passes a null stream and switches no device."""
    L = lib()
    if device is None:
        rc = getattr(L, name)(*args, None)
    else:
        with torch.cuda.device(device):
            rc = getattr(L, name)(*args, torch.cuda.current_stream(device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"{what}: {getattr(L, ABI[name][2])().decode()} (code {rc})")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what}: {lib().mia_last_error().decode()} (code {rc})")


def launch_count() -> int:
    return int(lib().mia_launch_count())
