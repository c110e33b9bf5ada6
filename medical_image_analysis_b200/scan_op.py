"""Host side of the selective scan: tensor checks, allocation and the C-ABI calls.

Mirrors the host functions of the reference's extension
(R2GenCSR/VMamba/kernels/selective_scan/csrc/selective_scan/cusoflex/selective_scan_oflex.cpp:
``selective_scan_fwd`` 143-231, ``selective_scan_bwd`` 233-355): same argument meaning, same output list,
same error behaviour (RuntimeError on a failed check).  PyTorch is used for device memory and the stream only.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib

def _req(cond: bool, msg: str) -> None:
    if not cond:
        raise RuntimeError(msg)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def num_chunks(seqlen: int) -> int:
    return int(_lib.lib().mia_ss_num_chunks(int(seqlen)))


def _check_inputs(u, delta, A, B, C, D, delta_bias, z):
    _req(u.dtype in _lib.DTYPE_CODES, "u must be float32, float16 or bfloat16")          # oflex.cpp:154
    _req(A.dtype == torch.float32, "A must be float32")                                 # :155
    _req(delta.dtype == u.dtype and B.dtype == u.dtype and C.dtype == u.dtype, "delta, B, C must have u's dtype")  # :157-159
    for name, t in (("u", u), ("delta", delta), ("A", A), ("B", B), ("C", C)):
        _req(t.is_cuda, f"{name} must be a CUDA tensor")                                # :161-165
    _req(u.dim() == 3 and delta.dim() == 3 and A.dim() == 2 and B.dim() == 4 and C.dim() == 4, "bad rank")
    batch, dim, L = u.shape
    N, G, ddim = A.shape[1], B.shape[1], delta.shape[1]
    _req(tuple(delta.shape) == (batch, ddim, L), "delta must have shape (batch_size, delta_dim, seqlen)")
    _req(tuple(A.shape) == (dim, N), "A must have shape (dim, dstate)")
    _req(tuple(B.shape) == (batch, G, N, L), "B must have shape (batch_size, n_groups, dstate, seqlen)")
    _req(tuple(C.shape) == (batch, G, N, L), "C must have shape (batch_size, n_groups, dstate, seqlen)")
    for name, t in (("u", u), ("delta", delta), ("B", B), ("C", C)):
        _req(t.stride(-1) == 1 or t.size(-1) == 1, f"{name} must be contiguous in the last dimension")  # :167-168,186,188
    if D is not None:
        _req(D.dtype == torch.float32 and D.is_cuda and tuple(D.shape) == (dim,) and D.is_contiguous(), "D must be float32 (dim)")
    if delta_bias is not None:
        _req(delta_bias.dtype == torch.float32 and delta_bias.is_cuda and tuple(delta_bias.shape) == (ddim,)
             and delta_bias.is_contiguous(), "delta_bias must be float32 (delta_dim)")
    if z is not None:
        _req(z.dtype == u.dtype and z.is_cuda and tuple(z.shape) == (batch, dim, L) and (z.stride(-1) == 1 or L == 1),
             "z must match u")
    return batch, dim, L, N, G, ddim


def _fill_inputs(p, u, delta, A, B, C, D, delta_bias, z, softplus, otype):
    batch, dim, L = u.shape
    p.batch, p.dim, p.seqlen, p.dstate, p.n_groups, p.delta_dim = batch, dim, L, A.shape[1], B.shape[1], delta.shape[1]
    p.itype, p.otype, p.delta_softplus = _lib.dtype_code(u.dtype), _lib.dtype_code(otype), int(bool(softplus))
    p.n_chunks = num_chunks(L)
    p.u, p.delta, p.A, p.B, p.C = u.data_ptr(), delta.data_ptr(), A.data_ptr(), B.data_ptr(), C.data_ptr()
    p.D, p.delta_bias, p.z = _ptr(D), _ptr(delta_bias), _ptr(z)
    p.u_batch_stride, p.u_d_stride = u.stride(0), u.stride(1)
    p.delta_batch_stride, p.delta_d_stride = delta.stride(0), delta.stride(1)
    p.A_d_stride, p.A_dstate_stride = A.stride(0), A.stride(1)
    p.B_batch_stride, p.B_group_stride, p.B_dstate_stride = B.stride(0), B.stride(1), B.stride(2)
    p.C_batch_stride, p.C_group_stride, p.C_dstate_stride = C.stride(0), C.stride(1), C.stride(2)
    if z is not None:
        p.z_batch_stride, p.z_d_stride = z.stride(0), z.stride(1)


def scan_fwd(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, out_float=False, want_block_states=False):
    """-> (out, x, out_z|None) [+ hblk|None when want_block_states].  out = y + D*u (before the gate), x = (batch, dim,
    n_chunks, 2*dstate) f32.  hblk: the d_state == 1 row-serial forward's per-16-token block states (mia_ss_params.hblk);
    pass it to scan_bwd(..., hblk=...) of the same inputs and the backward skips its forward recompute pass."""
    batch, dim, L, N, G, ddim = _check_inputs(u, delta, A, B, C, D, delta_bias, z)
    otype = torch.float32 if out_float else u.dtype
    with torch.cuda.device(u.device):
        out = torch.empty((batch, dim, L), dtype=otype, device=u.device)
        out_z = torch.empty_like(out) if z is not None else None
        x = torch.empty((batch, dim, num_chunks(L), 2 * N), dtype=torch.float32, device=u.device)
        p = _lib.MiaSSParams()
        _fill_inputs(p, u, delta, A, B, C, D, delta_bias, z, delta_softplus, otype)
        p.out, p.x = out.data_ptr(), x.data_ptr()
        p.out_batch_stride, p.out_d_stride = out.stride(0), out.stride(1)
        if out_z is not None:
            p.out_z = out_z.data_ptr()
            p.out_z_batch_stride, p.out_z_d_stride = out_z.stride(0), out_z.stride(1)
        hblk = None
        if want_block_states:
            nfl = int(_lib.lib().mia_ss_block_state_floats(ctypes.byref(p)))
            if nfl > 0:
                hblk = torch.empty((nfl,), dtype=torch.float32, device=u.device)
                p.hblk = hblk.data_ptr()
                if not _lib.lib().mia_ss_fwd_writes_block_states(ctypes.byref(p)):
                    hblk, p.hblk = None, None            # this shape takes a kernel that does not produce them
        _lib.call("mia_selective_scan_fwd", "selective_scan_fwd", u.device, ctypes.byref(p))
    return (out, x, out_z, hblk) if want_block_states else (out, x, out_z)


def scan_bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, delta_softplus, hblk=None):
    """-> (du, ddelta, dA, dB, dC, dD|None, ddelta_bias|None, dz|None); ddelta has delta's shape.  hblk: block states of
    the matching scan_fwd(..., want_block_states=True), or None.  Under torch.use_deterministic_algorithms(True) (read at
    call time) the deterministic backward runs: bit-reproducible gradients at every d_state."""
    batch, dim, L, N, G, ddim = _check_inputs(u, delta, A, B, C, D, delta_bias, z)
    _req(dout.is_cuda and tuple(dout.shape) == (batch, dim, L), "dout must have shape (batch_size, dim, seqlen)")
    _req(dout.dtype == u.dtype or dout.dtype == torch.float32, "dout must have u's dtype or float32")   # oflex.cpp:248
    _req(dout.stride(-1) == 1 or L == 1, "dout must be contiguous in the last dimension")               # :263
    nch = num_chunks(L)
    if nch > 1:
        _req(x is not None, "x is required when the sequence spans more than one chunk")                 # :305
    if x is not None:
        _req(x.dtype == torch.float32 and x.is_cuda and x.is_contiguous() and tuple(x.shape) == (batch, dim, nch, 2 * N),
             "x must be float32 contiguous (batch_size, dim, n_chunks, 2*dstate)")                       # :306-311
    if z is not None:
        _req(out is not None and out.dtype == dout.dtype and tuple(out.shape) == (batch, dim, L) and out.stride(-1) == 1,
             "out (saved from fwd) is required with z and must match dout")
    with torch.cuda.device(u.device):
        dev = u.device
        du = torch.empty((batch, dim, L), dtype=u.dtype, device=dev)
        ddelta = torch.empty((batch, ddim, L), dtype=u.dtype, device=dev)
        dA = torch.empty((dim, N), dtype=torch.float32, device=dev)
        dB = torch.empty((batch, G, N, L), dtype=u.dtype, device=dev)
        dC = torch.empty((batch, G, N, L), dtype=u.dtype, device=dev)
        dD = torch.empty((dim,), dtype=torch.float32, device=dev) if D is not None else None
        dbias = torch.empty((ddim,), dtype=torch.float32, device=dev) if delta_bias is not None else None
        dz = torch.empty((batch, dim, L), dtype=u.dtype, device=dev) if z is not None else None
        p = _lib.MiaSSParams()
        _fill_inputs(p, u, delta, A, B, C, D, delta_bias, z, delta_softplus, dout.dtype)
        p.x = _ptr(x)
        if hblk is not None:
            _req(hblk.dtype == torch.float32 and hblk.is_cuda and hblk.is_contiguous(), "hblk must be the float32 tensor scan_fwd returned")
            p.hblk = hblk.data_ptr()
            _req(hblk.numel() == int(_lib.lib().mia_ss_block_state_floats(ctypes.byref(p))), "hblk does not belong to these sizes")
        p.dout, p.dout_batch_stride, p.dout_d_stride = dout.data_ptr(), dout.stride(0), dout.stride(1)
        if z is not None:
            p.out_saved, p.out_saved_batch_stride, p.out_saved_d_stride = out.data_ptr(), out.stride(0), out.stride(1)
            p.dz, p.dz_batch_stride, p.dz_d_stride = dz.data_ptr(), dz.stride(0), dz.stride(1)
        p.du, p.du_batch_stride, p.du_d_stride = du.data_ptr(), du.stride(0), du.stride(1)
        p.ddelta, p.ddelta_batch_stride, p.ddelta_d_stride = ddelta.data_ptr(), ddelta.stride(0), ddelta.stride(1)
        p.dA, p.dA_d_stride, p.dA_dstate_stride = dA.data_ptr(), dA.stride(0), dA.stride(1)
        p.dB, p.dB_batch_stride, p.dB_group_stride, p.dB_dstate_stride = dB.data_ptr(), dB.stride(0), dB.stride(1), dB.stride(2)
        p.dC, p.dC_batch_stride, p.dC_group_stride, p.dC_dstate_stride = dC.data_ptr(), dC.stride(0), dC.stride(1), dC.stride(2)
        p.dD, p.ddelta_bias = _ptr(dD), _ptr(dbias)
        lib = _lib.lib()
        if torch.are_deterministic_algorithms_enabled():
            ws_fn, what = lib.mia_selective_scan_bwd_deterministic_workspace, "selective_scan_bwd_deterministic"
        else:
            ws_fn, what = lib.mia_selective_scan_bwd_workspace, "selective_scan_bwd"
        ws_bytes = int(ws_fn(ctypes.byref(p)))
        ws = torch.empty((max(ws_bytes, 256),), dtype=torch.uint8, device=dev)
        p.workspace, p.workspace_bytes = ws.data_ptr(), ws_bytes
        _lib.call("mia_" + what, what, dev, ctypes.byref(p))
        ws.record_stream(torch.cuda.current_stream(dev))
    return du, ddelta, dA, dB, dC, dD, dbias, dz
