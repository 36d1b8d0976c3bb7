"""The G-buffer kernels (csrc/gbuffer_api.cu) on the GPU.

Forward: every recorded kernel call (kernel_calls fixture) bit for bit against oracle/gbuffer.py's float32 emulation,
with the same NaN / +-inf pattern.  Gradients: against float64 autograd of the op-by-op mirror (Lighting.fused = False on
the CPU) within 1e-4 of each gradient's max |finite value|, with the same non-finite pattern, on the edge scenes of
tests/gbuffer_edge_cases.py.  End to end: Renderer(Gbuffer=...) images against the reference pipeline's
(tests/golden/ref_host_gbuffer.npz), within 1e-3 of the max for SoftRas and 1e-4 for NMR.
Launches: at most two forward and two backward.  CUDA graphs: a depth-mode render and
its backward captured and replayed give the eager images bit for bit.
"""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib
from jrender_b200 import workloads as wl
from oracle import gbuffer as OG
from tests import gbuffer_edge_cases as E

pytestmark = pytest.mark.gpu
GRAD_TOL = 1e-4
G = os.path.join(os.path.dirname(__file__), "golden", "ref_host_gbuffer.npz")


@pytest.fixture
def kernel_calls(monkeypatch):
    """Every call of the four G-buffer entry points made while the test runs: (name, arguments after the call)."""
    calls = []
    real = _lib.call

    def record(name, device, *args):
        real(name, device, *args)
        if name in OG.CALLS:
            torch.cuda.synchronize(device)
            calls.append((name, OG.args_from_call(name, args) if "forward" in name else None))
    monkeypatch.setattr(_lib, "call", record)
    return calls


def _same_bits(got, want, what):
    got, want = np.asarray(got), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), "%s: %d of %d entries differ from the emulation, first at %s (%r vs %r)" % (
        what, bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0])


def _hold_forward(calls):
    n = 0
    for name, a in calls:
        if a is None:
            continue
        if name == "b200r_gbuffer_lighting_forward":
            want, M = OG.gbuffer_forward(a)
            _same_bits(a["out"].reshape(want.shape), want, name)
            if M is not None:
                _same_bits(a["depth_max"], [M], name + " depth_max")
        else:
            _same_bits(a["out"], OG.nm_gbuffer_forward(a), name)
        n += 1
    return n


def _close_grad(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, what
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN pattern differs" % what
    assert np.array_equal(np.isinf(got), np.isinf(want)), "%s: inf pattern differs" % what
    if fin.any():
        scale = max(np.abs(want[fin]).max(), 1e-30)
        err = np.abs(got[fin] - want[fin]).max()
        assert err <= GRAD_TOL * scale, "%s: %.3e > %.1e of %.3e" % (what, err, GRAD_TOL, scale)


@pytest.mark.parametrize("name", E.NAMES)
def test_kernels_against_emulation_and_float64_mirror(name, kernel_calls):
    sc = E.scene(name)
    out, grads = E.run(sc, torch.device("cuda"), torch.float32, fused=True)
    assert {n for n, _ in kernel_calls} >= E.expected_calls(sc)
    assert _hold_forward(kernel_calls) >= 1
    ref_out, ref_grads = E.run(sc, torch.device("cpu"), torch.float64, fused=False)
    assert np.array_equal(np.isnan(out), np.isnan(ref_out)), name
    fin = np.isfinite(ref_out)
    assert np.abs(out[fin] - ref_out[fin]).max(initial=0) <= 2e-5, name
    for k, g in ref_grads.items():
        if g is None:
            assert grads[k] is None, (name, k)
        elif any(t in name for t in ("_metallic_", "_roughness_")):
            # Known difference at a non-finite material input: the kernels' forward-mode duals multiply a zero tangent
            # by the non-finite value (0 * NaN), where the mirror's reverse mode never forms that product, so the
            # kernel's gradient may be NaN where the mirror's is finite.  It is NaN wherever the mirror's is, and
            # within the bound wherever both are finite.
            got = np.asarray(grads[k], np.float64)
            assert np.isnan(got[np.isnan(g)]).all(), (name, k)
            fin = np.isfinite(got) & np.isfinite(g)
            scale = max(np.abs(g[np.isfinite(g)]).max(initial=0), 1e-30)
            assert np.abs(got[fin] - g[fin]).max(initial=0) <= GRAD_TOL * scale, (name, k)
        else:
            _close_grad(grads[k], g, "%s: grad %s" % (name, k))


def test_head_sized_normal_map_against_float64_mirror():
    """The normal-map G-buffer at the head's size (66 282 faces x 225 texels, the specular branch on) against float64
    autograd of the mirror, run on the GPU."""
    from tools.time_normal_lighting import scene
    dev = torch.device("cuda")
    h = scene(dev)
    res = {}
    for fused, dt in ((True, torch.float32), (False, torch.float64)):
        nt = h["nt"].to(dt).detach().requires_grad_(True)
        met = h["met"].to(dt).detach().requires_grad_(True)
        mesh = jr.Mesh(h["v"].to(dt), h["f"], textures=h["tex"].to(dt), normal_textures=nt, TBN=h["tbn"].to(dt),
                       metallic_textures=met, roughness_textures=h["rou"].to(dt), texture_res=15)
        light = jr.Lighting(Gbuffer="normal", **E.LIGHT)
        light.fused = fused
        eye = h["eye"].to(dt)
        if fused:
            assert light._fused_normal_mapped_gbuffer(mesh, eye) is not None
        out = light(mesh, eye).textures
        g = torch.randn(out.shape, generator=torch.Generator(dev).manual_seed(3), device=dev).to(dt)
        out.backward(g)
        res[fused] = (out.detach().double().cpu().numpy(), nt.grad.double().cpu().numpy(), met.grad.double().cpu().numpy())
        del out, g, mesh
    assert np.abs(res[True][0] - res[False][0]).max() <= 2e-5
    _close_grad(res[True][1], res[False][1], "head: grad normal_textures")
    _close_grad(res[True][2], res[False][2], "head: grad metallic")


def test_launch_counts():
    for name in ("sphere_depth_spec", "sphere_normal_spec", "normal_map_spec"):
        sc = E.scene(name)
        ts, light, mesh, eyes = E.build(sc, torch.device("cuda"), torch.float32, fused=True)
        torch.cuda.synchronize()
        n0 = _lib.lib().b200r_launch_count()
        out = light(mesh, eyes).textures
        n1 = _lib.lib().b200r_launch_count()
        out.backward(torch.ones_like(out))
        torch.cuda.synchronize()
        n2 = _lib.lib().b200r_launch_count()
        assert 1 <= n1 - n0 <= 2 and 1 <= n2 - n1 <= 2, (name, n1 - n0, n2 - n1)


@pytest.mark.parametrize("dr_type", ["softras", "n3mr"])
@pytest.mark.parametrize("mode", ["normal", "depth"])
def test_renderer_matches_reference_pipeline(dr_type, mode, kernel_calls):
    g = np.load(G)
    dev = torch.device("cuda")
    v, f = torch.from_numpy(g["e2e_vertices"]).to(dev), torch.from_numpy(g["e2e_faces"]).to(dev)
    if dr_type == "softras":
        r = jr.Renderer(image_size=64, sigma_val=1e-4, anti_aliasing=True, dr_type="softras", Gbuffer=mode)
        r.transform.set_eyes_from_angles(2.732, 30.0, 40.0)
        tex = torch.full((1, 280, 4, 3), 0.3, device=dev)
    else:
        r = jr.Renderer(image_size=64, anti_aliasing=True, dr_type="n3mr", Gbuffer=mode)
        r.transform.set_eyes_from_angles(2.732, 20.0, 100.0)
        tex = torch.full((1, 280, 2, 2, 2, 3), 0.3, device=dev)
    mesh = jr.Mesh(v[None], f[None], textures=tex, texture_res=2, dr_type=dr_type)
    img = r.render_mesh(mesh, mode="rgb").detach().cpu().numpy()
    assert any(n == "b200r_gbuffer_lighting_forward" for n, _ in kernel_calls)
    want = g["e2e_%s_%s" % (dr_type, mode)]
    assert img.shape == want.shape
    tol = 1e-3 if dr_type == "softras" else 1e-4   # the SoftRas kernels against the float32 CPU oracle, anti-aliased
    assert np.abs(img - want).max() <= tol * max(np.abs(want).max(), 1e-30), np.abs(img - want).max()


def test_depth_render_and_backward_replay_in_a_cuda_graph():
    """A depth-mode SoftRas render and its backward captured in a CUDA graph (the G-buffer's two launches each way, the
    max reduced on the device, no host synchronisation) and replayed: the same images bit for bit, the gradient up to
    the float atomics' order.  Warm-up and capture run on a side stream with no graph of an earlier step kept alive."""
    dev = torch.device("cuda")
    vv, ff = wl.sphere_by_faces(3280)
    v = torch.from_numpy(vv).to(dev)[None].repeat(3, 1, 1).requires_grad_(True)
    f = torch.from_numpy(ff).to(dev)[None].repeat(3, 1, 1)
    r = jr.Renderer(image_size=64, sigma_val=1e-4, dr_type="softras", Gbuffer="depth", camera_mode="look_at")
    r.transform.set_eyes_from_angles(torch.full((3,), 2.732, device=dev), torch.tensor([10., 30., -20.], device=dev),
                                     torch.tensor([0., 120., 240.], device=dev))
    w = torch.rand((3, 3, 64, 64), device=dev)

    def step():
        tex = torch.ones((3, ff.shape[0], 1, 3), device=dev)
        img = r.render_mesh(jr.Mesh(v, f, textures=tex), mode="rgb")
        v.grad = None
        (img * w).sum().backward()
        return img.detach(), v.grad
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        eager_img, eager_g = step()
        eager_g = eager_g.clone()
        step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_img, static_g = step()
    graph.replay()
    torch.cuda.synchronize()
    assert static_img.abs().sum() > 0
    assert torch.equal(static_img, eager_img)
    assert (static_g - eager_g).abs().max().item() <= 1e-5 * eager_g.abs().max().item()


def test_fit_lowers_its_loss():
    from examples.render_gbuffers import fit
    hist = fit(iters=30, image_size=32, batch=4, verbose=False)
    assert np.isfinite(hist).all() and hist[-1] < hist[0], hist
