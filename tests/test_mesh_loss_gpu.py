"""GPU parity of the fused mesh regularisers (csrc/mesh_loss_api.cu, SURVEY.md 8f rank 4): value and
gradient against the op-by-op PyTorch mirror (itself pinned to the reference's Python by
tests/test_host_golden.py), against the reference-Python golden values directly, against central differences of the
float64 oracle, and every entry within the summation-order bound of the oracle's emulated float32 terms."""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import workloads as wl

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
VAL_TOL = 2e-5    # sums of 10^2..10^4 fp32 terms accumulated in a different order (warp tree + atomics)
GRAD_TOL = 5e-5   # of max |grad|: fp32 atomics vs the mirror's index_add order; forward-mode vs reverse-mode rounding


def _both(make_loss, v_np, dev):
    out = {}
    for fused in (True, False):
        loss_mod = make_loss().to(dev)
        loss_mod.fused = fused
        v = torch.from_numpy(v_np).to(dev).requires_grad_(True)
        val = loss_mod(v)
        w = torch.linspace(0.5, 1.5, val.numel(), device=dev).view_as(val)
        (val * w).sum().backward()
        out[fused] = (val.detach().cpu().numpy(), v.grad.cpu().numpy())
    return out


@pytest.mark.parametrize("which", ["laplacian", "flatten"])
def test_fused_losses_match_mirror_and_golden(which, cuda_device):
    g = np.load(os.path.join(G, "ref_host_loss_sphere280.npz"))
    f = torch.from_numpy(g["faces"])
    v0 = torch.from_numpy(g["vertices"][0])
    make = (lambda: jr.LaplacianLoss(v0, f)) if which == "laplacian" else (lambda: jr.FlattenLoss(f))
    out = _both(make, g["vertices"], cuda_device)
    ref = g[which]
    assert out[True][0].shape == ref.shape
    assert np.abs(out[True][0] - ref).max() <= VAL_TOL * np.abs(ref).max()          # vs the reference's own Python
    assert np.abs(out[True][0] - out[False][0]).max() <= VAL_TOL * np.abs(ref).max()
    assert np.abs(out[True][1] - out[False][1]).max() <= GRAD_TOL * np.abs(out[False][1]).max()


@pytest.mark.parametrize("which", ["laplacian", "flatten", "flatten_rot"])
def test_fused_loss_gradients_against_numeric_oracle(which, cuda_device):
    """Gradients of the fused kernels against oracle/mesh_loss.py: float64 restatement of the reference's expressions,
    differentiated by central differences (independent of the PyTorch mirror and of any autograd); and every value and
    gradient entry within the summation-order bound of the oracle's float32 emulation of the kernels' terms (the
    emulation is held to float64 in test_geometry_edges_cpu.py)."""
    from oracle import mesh_loss as oml
    from tests.geometry_edge_cases import check_sums
    g = np.load(os.path.join(G, "ref_host_loss_sphere280.npz"))
    vb = g["vertices"]
    faces = g["faces_rot"] if which == "flatten_rot" else g["faces"]
    f = torch.from_numpy(faces)
    if which == "laplacian":
        mod = jr.LaplacianLoss(torch.from_numpy(vb[0]), f)
        lap = oml.laplacian_matrix(vb.shape[1], faces)
        fn = lambda x: oml.laplacian(x, lap)                      # noqa: E731
        s = oml.laplacian_sums(vb, mod.nbr32.numpy(), mod.nbr_w.numpy(), mod.diag.numpy())
    else:
        mod = jr.FlattenLoss(f)
        edges = oml.flatten_edges(faces)
        fn = lambda x: oml.flatten(x, edges)                      # noqa: E731
        s = oml.flatten_sums(vb, edges)
    mod = mod.to(cuda_device)
    v = torch.from_numpy(vb).to(cuda_device).requires_grad_(True)
    val = mod(v)
    val.sum().backward()     # an upstream gradient of 1 leaves the kernel's gradient unrounded
    check_sums(which + " loss", val.detach().cpu().numpy(), s["loss"])
    check_sums(which + " grad", v.grad.cpu().numpy(), s["grad"])
    v.grad = None
    val = mod(v)
    w = np.linspace(0.5, 1.5, val.numel())
    (val * torch.from_numpy(w.astype(np.float32)).to(cuda_device)).sum().backward()
    ref_val = fn(vb)
    ref_grad = oml.numeric_grad(fn, vb, w)
    assert np.abs(val.detach().cpu().numpy() - ref_val).max() <= VAL_TOL * np.abs(ref_val).max()
    assert np.abs(v.grad.cpu().numpy() - ref_grad).max() <= GRAD_TOL * np.abs(ref_grad).max()


def test_fused_loss_buffers_on_another_device_do_not_reach_the_kernel(cuda_device):
    """A loss module left on the CPU with CUDA vertices must raise torch's device error, never hand host pointers to
    the kernel; a mesh smaller than the edge table must raise an index error, never read out of bounds."""
    g = np.load(os.path.join(G, "ref_host_loss_sphere280.npz"))
    f = torch.from_numpy(g["faces"])
    v = torch.from_numpy(g["vertices"]).to(cuda_device)
    for mod in (jr.LaplacianLoss(torch.from_numpy(g["vertices"][0]), f), jr.FlattenLoss(f)):   # buffers stay on the CPU
        with pytest.raises(RuntimeError):
            mod(v)
    with pytest.raises((RuntimeError, IndexError)):
        jr.FlattenLoss(f).to(cuda_device)(v[:, :100].contiguous())
    torch.cuda.synchronize()


def test_fused_losses_large_mesh_average_and_graph(cuda_device):
    v, f = wl.sphere_by_faces(3280)
    rng = np.random.default_rng(9)
    vb = (v[None] + rng.normal(0, 0.01, (4,) + v.shape)).astype(np.float32)
    ft = torch.from_numpy(f)
    for make in (lambda: jr.LaplacianLoss(torch.from_numpy(v), ft, average=True), lambda: jr.FlattenLoss(ft, average=True)):
        out = _both(make, vb, cuda_device)
        assert abs(float(out[True][0]) - float(out[False][0])) <= VAL_TOL * abs(float(out[False][0]))
        assert np.abs(out[True][1] - out[False][1]).max() <= GRAD_TOL * np.abs(out[False][1]).max()
    # capture + replay: the fused ops enqueue on the capturing stream and never synchronise
    lap = jr.LaplacianLoss(torch.from_numpy(v), ft).to(cuda_device)
    flat = jr.FlattenLoss(ft).to(cuda_device)
    x = torch.from_numpy(vb).to(cuda_device).requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            (lap(x).mean() + flat(x).mean()).backward()
    torch.cuda.current_stream().wait_stream(s)
    eager = x.grad.clone()
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        (lap(x).mean() + flat(x).mean()).backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.allclose(x.grad, eager, rtol=1e-4, atol=1e-6 * float(eager.abs().max()))
