"""Drop-in for mamba_ssm's pybind module ``selective_scan_cuda`` (not vendored by the reference; its call sites are
R2GenCSR/VMamba/classification/models/vmamba.py:255, 266-269 and test_selective_scan.py:60, 105-108):
  fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus) -> [out, x] or [out, x, out_z]
  bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, dz, delta_softplus, recompute_out_z)
        -> [du, ddelta, dA, dB, dC, dD, ddelta_bias] (+ [dz] with z, + [out_z] when recompute_out_z)
"""
from __future__ import annotations

from .scan_op import scan_bwd, scan_fwd


def _bc4(t):
    return t.unsqueeze(1) if t.dim() == 3 else t


def fwd(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False):
    out, x, out_z = scan_fwd(u, delta, A, _bc4(B), _bc4(C), D, z, delta_bias, delta_softplus, False)
    return [out, x] if z is None else [out, x, out_z]


def bwd(u, delta, A, B, C, D=None, z=None, delta_bias=None, dout=None, x=None, out=None, dz=None,
        delta_softplus=False, recompute_out_z=False):
    squeeze = B.dim() == 3
    du, dd, dA, dB, dC, dD, dbias, dz_new = scan_bwd(u, delta, A, _bc4(B), _bc4(C), D, z, delta_bias, dout, x, out, delta_softplus)
    if squeeze:
        dB, dC = dB.squeeze(1), dC.squeeze(1)
    res = [du, dd, dA, dB, dC, dD, dbias]
    if z is not None:
        if dz is not None:          # caller-provided buffer (mamba_ssm fuses the chunk backward this way)
            dz.copy_(dz_new)
            dz_new = dz
        res.append(dz_new)
        if recompute_out_z:
            import torch
            from . import _lib
            o, zc = out.contiguous(), z.contiguous()
            out_z = torch.empty_like(o)
            _lib.call("mia_silu_gate", "silu_gate", o.device, o.data_ptr(), zc.data_ptr(), out_z.data_ptr(), o.numel(),
                      _lib.dtype_code(zc.dtype), _lib.dtype_code(o.dtype))
            res.append(out_z)
    return res
