"""CrossScan / CrossMerge / SS2D: oracle vs the reference's own outputs (CPU), CUDA kernels vs both (GPU)."""
import copy

import pytest
import torch

from oracle.ss2d_ref import cross_merge_ref, cross_scan_ref
from tests.golden_util import cross_scan as golden_cross_scan

G = golden_cross_scan()


@pytest.mark.parametrize("tag", ["sq", "rect"])
def test_oracle_cross_scan_merge_match_reference(tag):
    x, xs, ys, y = G[f"{tag}.x"], G[f"{tag}.xs"], G[f"{tag}.ys"], G[f"{tag}.y"]
    B, C, H, W = x.shape
    assert torch.equal(cross_scan_ref(x), xs)
    assert torch.allclose(cross_merge_ref(ys.view(B, 4, C, -1), H, W), y, atol=1e-6)
    # adjoint pair: the reference's backward of one is the forward of the other (vmamba.py:37-45, 59-67)
    assert torch.allclose(cross_merge_ref(G[f"{tag}.gxs"], H, W).view(B, C, H, W), G[f"{tag}.dx"], atol=1e-6)
    assert torch.equal(cross_scan_ref(G[f"{tag}.gy"].view(B, C, H, W)).view(B, 4, C, H, W), G[f"{tag}.dys"])


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["sq", "rect"])
def test_cuda_cross_scan_merge_match_reference(tag):
    from medical_image_analysis_b200.vmamba import CrossMerge, CrossScan
    x = G[f"{tag}.x"].cuda().requires_grad_()
    xs = CrossScan.apply(x)
    assert torch.equal(xs.cpu(), G[f"{tag}.xs"])
    xs.backward(G[f"{tag}.gxs"].cuda())
    assert torch.allclose(x.grad.cpu(), G[f"{tag}.dx"], atol=1e-6)
    ys = G[f"{tag}.ys"].cuda().requires_grad_()
    y = CrossMerge.apply(ys)
    assert torch.allclose(y.cpu(), G[f"{tag}.y"], atol=1e-6)
    y.backward(G[f"{tag}.gy"].cuda())
    assert torch.equal(ys.grad.cpu(), G[f"{tag}.dys"])


# Launch paths of csrc/cross_scan.cu (launch_cs): "vec" (4-element accesses, L % 4 == 0 and 4-element aligned operands,
# up to 8 planes per block within 200 KB), "staged" (one element per thread, up to 4 planes per block; the merge stages
# fp32) and "direct" (a plane does not fit: gathers from global memory, grid capped at 132 x 16 blocks).
# (B, C, H, W[, storage offset of the input in elements]) -> {op: (fp32 path, bf16 / fp16 path)}
CS_PATHS = {
    (2, 5, 14, 14): dict(scan=("vec", "vec"), merge=("vec", "vec")),                 # 8 planes per block
    (1, 3, 7, 9): dict(scan=("staged", "staged"), merge=("staged", "staged")),
    (1, 2, 80, 80): dict(scan=("vec", "vec"), merge=("vec", "vec")),                 # fp32 merge: 2 planes
    (3, 1, 1, 6): dict(scan=("staged", "staged"), merge=("staged", "staged")),
    (1, 9, 56, 56): dict(scan=("vec", "vec"), merge=("vec", "vec")),                 # fp32 merge: 4 planes
    (1, 3, 7, 7): dict(scan=("staged", "staged"), merge=("staged", "staged")),
    (2, 3, 3, 1): dict(scan=("staged", "staged"), merge=("staged", "staged")),
    (1, 4, 128, 128): dict(scan=("vec", "staged"), merge=("staged", "vec")),         # 16-bit merge: 1 plane
    (2, 12, 256, 256): dict(scan=("direct", "staged"), merge=("direct", "direct")),  # 2.9 grid sweeps
    (1, 12, 227, 227): dict(scan=("direct", "staged"), merge=("direct", "direct")),  # 1.1 grid sweeps
    (2, 5, 14, 14, 1): dict(scan=("staged", "staged"), merge=("staged", "staged")),
    (2, 5, 14, 14, 2): dict(scan=("staged", "staged"), merge=("staged", "staged")),
}
CS_KERNEL = r"\bcross_(scan|merge)_(vec_|direct_)?kernel<"


def _cs_path(names, op):
    assert len(names) == 1 and f"cross_{op}_" in names[0], names
    return "vec" if "_vec_kernel<" in names[0] else "direct" if "_direct_kernel<" in names[0] else "staged"


def _on_gpu(t, offset):
    """``t`` on the GPU, contiguous, its storage starting ``offset`` elements into a buffer."""
    buf = torch.empty(offset + t.numel(), dtype=t.dtype, device="cuda")
    buf[offset:].copy_(t.reshape(-1))
    return buf[offset:].view(t.shape)


def cs_kernel_paths():
    """{case: [scan, merge of CrossScan's gradient, merge, scan of CrossMerge's gradient] kernels} under the profiler, for
    every case and dtype of test_cuda_cross_scan_merge_vs_oracle."""
    from medical_image_analysis_b200.vmamba import CrossMerge, CrossScan
    from tests.kernel_trace import names_of
    out = {}
    for shape in CS_PATHS:
        B, C, H, W, off = (*shape, 0)[:5]
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            rnd = lambda *s: _on_gpu(torch.randn(*s).to(dtype), off)
            x, ys = rnd(B, C, H, W).requires_grad_(True), rnd(B, 4, C, H, W).requires_grad_(True)
            xs, y = CrossScan.apply(x), CrossMerge.apply(ys)
            gxs, gy = rnd(B, 4, C, H * W), rnd(B, C, H * W)
            out[f"{shape}|{dtype}"] = [names_of(lambda: CrossScan.apply(x), CS_KERNEL),
                                       names_of(lambda: torch.autograd.grad(xs, x, gxs, retain_graph=True), CS_KERNEL),
                                       names_of(lambda: CrossMerge.apply(ys), CS_KERNEL),
                                       names_of(lambda: torch.autograd.grad(y, ys, gy, retain_graph=True), CS_KERNEL)]
    return out


@pytest.fixture(scope="module")
def cs_paths():
    from tests.kernel_trace import in_child
    return in_child("tests.test_ss2d:cs_kernel_paths")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", list(CS_PATHS))
def test_cuda_cross_scan_merge_vs_oracle(cs_paths, shape, dtype):
    """CrossScan / CrossMerge forward and backward against the oracle on float64 values: the scan (a permutation) exactly,
    the merge (a sum of four, rounded once) by the parity criteria; each call's kernel (recorded in a child process,
    tests/kernel_trace.py) is the one the path table names."""
    from medical_image_analysis_b200.vmamba import CrossMerge, CrossScan
    from tests.parity import cmp_f32, cmp_stored
    B, C, H, W, off = (*shape, 0)[:5]
    L = H * W
    want = {op: paths[0 if dtype == torch.float32 else 1] for op, paths in CS_PATHS[shape].items()}
    if "direct" in want.values():
        assert B * C * L > 132 * 16 * 256                       # several sweeps of the capped grid
    g = torch.Generator().manual_seed(B * C * L + off)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dtype)

    def merged(got, ys, what):
        ref = cross_merge_ref(ys.double().view(B, 4, C, L), H, W)
        if dtype == torch.float32:
            cmp_f32(got.reshape(B, C, L), ref, what)
        else:
            cmp_stored(got.reshape(B, C, L), ref, dtype, what)

    tag = f"cross {shape} {dtype}"
    x0, gxs0, ys0, gy0 = rnd(B, C, H, W), rnd(B, 4, C, L), rnd(B, 4, C, H, W), rnd(B, C, L)
    k_scan, k_scan_grad, k_merge, k_merge_grad = cs_paths[f"{shape}|{dtype}"]
    for names, op in ((k_scan, "scan"), (k_scan_grad, "merge"), (k_merge, "merge"), (k_merge_grad, "scan")):
        assert _cs_path(names, op) == want[op], names
    x = _on_gpu(x0, off).requires_grad_(True)
    xs = CrossScan.apply(x)
    assert torch.equal(xs.cpu(), cross_scan_ref(x0))
    (dx,) = torch.autograd.grad(xs, x, _on_gpu(gxs0, off))
    merged(dx, gxs0, f"{tag} CrossScan dx")
    ys = _on_gpu(ys0, off).requires_grad_(True)
    y = CrossMerge.apply(ys)
    merged(y, ys0, f"{tag} CrossMerge y")
    (dys,) = torch.autograd.grad(y, ys, _on_gpu(gy0, off))
    assert torch.equal(dys.cpu(), cross_scan_ref(gy0.view(B, C, H, W)).view(B, 4, C, H, W))


@pytest.mark.gpu
@pytest.mark.parametrize("forward_type,d_state", [("v3noz", 1), ("v2", 4), ("v3", 16), ("v4noz", 1)])
def test_ss2d_module_matches_restated_forward(forward_type, d_state):
    """SS2D on the CUDA kernels vs the reference's forwardv2 restated on the CPU oracle (same weights)."""
    from medical_image_analysis_b200.vmamba import SS2D
    from oracle.ss2d_ref import ss2d_forward_ref
    torch.manual_seed(1)
    m = SS2D(d_model=16, d_state=d_state, ssm_ratio=2.0, forward_type=forward_type)
    mc = copy.deepcopy(m)
    m = m.cuda()
    x = torch.randn(2, 6, 5, 16)
    xg = x.cuda().requires_grad_()
    xc = x.clone().requires_grad_()
    out = m(xg)
    ref = ss2d_forward_ref(mc, xc)
    assert out.shape == ref.shape == (2, 6, 5, 16)
    w = torch.randn_like(ref)
    (out * w.cuda()).sum().backward()
    (ref * w).sum().backward()
    # the reference casts the merged scan output to bf16 (vmamba.py:420): compare at bf16 resolution
    assert torch.allclose(out.cpu(), ref, atol=3e-2, rtol=3e-2), (out.cpu() - ref).abs().max()
    assert torch.allclose(xg.grad.cpu(), xc.grad, atol=5e-2, rtol=5e-2), (xg.grad.cpu() - xc.grad).abs().max()
    for (n, p), (_, pc) in zip(m.named_parameters(), mc.named_parameters()):
        scale = max(1.0, pc.grad.abs().max().item())
        assert torch.allclose(p.grad.cpu(), pc.grad, atol=5e-2 * scale, rtol=5e-2), (n, (p.grad.cpu() - pc.grad).abs().max())


def test_ss2d_parameter_names_match_reference_checkpoints():
    """Names / shapes of vmamba.py:767-790 so that published checkpoints load (SURVEY.md 5, checkpoint/resume)."""
    from medical_image_analysis_b200.vmamba import SS2D
    m = SS2D(d_model=96, d_state=16, ssm_ratio=2.0, dt_rank="auto", forward_type="v2")
    sd = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert sd["x_proj_weight"] == (4, 6 + 32, 192) and sd["dt_projs_weight"] == (4, 192, 6) and sd["dt_projs_bias"] == (4, 192)
    assert sd["A_logs"] == (768, 16) and sd["Ds"] == (768,)
    assert sd["in_proj.weight"] == (384, 96) and sd["out_proj.weight"] == (96, 192) and sd["conv2d.weight"] == (192, 1, 3, 3)
    assert sd["out_norm.weight"] == (192,)
    assert torch.allclose(m.A_logs[0].exp(), torch.arange(1, 17, dtype=torch.float32))
