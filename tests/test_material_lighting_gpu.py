"""GPU tests of the fused surface-lighting kernel's material gradients (csrc/lighting_api.cu, grad_metallic /
grad_roughness of b200r_surface_lighting_backward) and of the demo 3, 5 and 6 ports built on them.

Tolerances:
- fused float32 vs the op-by-op mirror's float64 autograd: 1e-4 of max |grad|, as tests/test_lighting_gpu.py states for
  the vertex and texture gradients (float32 forward-mode derivatives vs float64 reverse mode);
- whole renderer, fused vs op-by-op: 1e-4 of max |grad|.  Both arms run the SoftRas backward, whose float atomics sum
  in a different order each run, and the two lighting paths' lit textures differ in the last bits.  Measured on an
  NVIDIA H100 80GB HBM3 (700 W): 2.1e-6 (metallic) and 5.9e-6 (roughness) fused vs op-by-op, against a fused run-to-run
  spread of 4e-8;
- every fused call also against the kernels' float32 emulation (test_lighting_edges_gpu.hold_to_emulation): lit
  textures and per-texel gradients bit for bit, vertex gradients within the float atomics' order bound;
- demo convergence: the final loss is at most CONVERGED of the first.  Measured on the same card: 0.0052 (demo 5,
  20 iterations) and 0.0006 (demo 6, 15 iterations); the thresholds leave a margin of about 6x and 15x.
"""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib
from jrender_b200 import workloads as wl

from tests.test_lighting_edges_gpu import hold_to_emulation, kernel_calls  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")

MATERIAL_RENDERER_TOL = 1e-4
CONVERGED = {"demo5": 0.03, "demo6": 0.01}


@pytest.fixture(scope="module")
def spot(tmp_path_factory):
    """The spot cow of the reference's demos (5856 faces, UV-mapped texture; public domain, Keenan Crane), unpacked
    from tests/golden/spot_triangulated.obj.xz + spot_texture.png into a temporary directory as the demos load it:
    .obj, .mtl naming the texture, .png side by side.  Returns the path of the .obj."""
    import lzma
    import shutil
    d = tmp_path_factory.mktemp("spot")
    with lzma.open(os.path.join(G, "spot_triangulated.obj.xz"), "rb") as f:
        (d / "spot_triangulated.obj").write_bytes(f.read())
    (d / "spot_triangulated.mtl").write_text("newmtl material_1\nmap_Kd spot_texture.png\n")
    shutil.copyfile(os.path.join(G, "spot_texture.png"), d / "spot_texture.png")
    return str(d / "spot_triangulated.obj")


def _light():
    return jr.Lighting(intensity_ambient=0.4, color_ambient=[1, 0.9, 0.8], intensity_directionals=0.7,
                       color_directionals=[0.9, 1, 0.7], directions=[0.3, 1, -0.4])


def _scene(tex6, B=3, seed=5):
    rng = np.random.default_rng(seed)
    v, f = wl.sphere_by_faces(280)
    vb = (v[None] + rng.normal(0, 0.03, (B,) + v.shape)).astype(np.float32)
    shape = (B, f.shape[0], 2, 2, 2, 3) if tex6 else (B, f.shape[0], 4, 3)
    tex = rng.uniform(0.0, 2.5, shape).astype(np.float32)     # some texels saturate the clamp, for every eye
    met = rng.uniform(0, 1, shape[:-1] + (1,)).astype(np.float32)
    rou = rng.uniform(0.2, 1, shape[:-1] + (1,)).astype(np.float32)
    gout = rng.uniform(-1, 1, shape).astype(np.float32)
    return vb, f, tex, met, rou, gout


EYES = {"per_batch": [[0.0, 0.0, -2.7], [1.0, 1.5, -2.0], [-2.0, 0.3, 1.0]],
        "shared": [[0.4, 2.2, 1.6]],
        "grazing": [[2.6, 0.05, 0.2]]}


def _lit_grads(dev, scene, eyes, dtype, fused, spec=True, material_grad=True):
    """Lit textures and the gradients of <out, gout> w.r.t. (vertices, textures, metallic, roughness)."""
    vb, f, tex, met, rou, gout = scene
    B = vb.shape[0]
    vt = torch.from_numpy(vb).to(dev, dtype).requires_grad_(True)
    tt = torch.from_numpy(tex).to(dev, dtype).requires_grad_(True)
    mt = torch.from_numpy(met).to(dev, dtype).requires_grad_(material_grad)
    rt = torch.from_numpy(rou).to(dev, dtype).requires_grad_(material_grad)
    m = jr.Mesh(vt, torch.from_numpy(f)[None].repeat(B, 1, 1).to(dev), textures=tt, dr_type='n3mr' if tex.ndim == 6 else 'softras',
                metallic_textures=mt, roughness_textures=rt)
    m.with_specular = spec
    light = _light()
    light.fused = fused
    e = torch.tensor(eyes, device=dev, dtype=dtype)
    if fused:
        assert light._fusable(m, e)
    out = light(m, e).textures
    out.backward(torch.from_numpy(gout).to(dev, dtype))
    grads = [t.grad for t in (vt, tt, mt, rt)]
    return out.detach(), grads


@pytest.mark.parametrize("eyes", sorted(EYES))
@pytest.mark.parametrize("tex6", [False, True])
def test_material_gradients_match_float64_autograd(cuda_device, kernel_calls, tex6, eyes):
    scene = _scene(tex6)
    out, got = _lit_grads(cuda_device, scene, EYES[eyes], torch.float32, True)
    out64, ref = _lit_grads(cuda_device, scene, EYES[eyes], torch.float64, False)
    assert np.abs(out.double().cpu().numpy() - out64.cpu().numpy()).max() <= 2e-5
    assert bool((out64 >= 1).any())   # texels that saturate the output clamp are in the scene
    for name, a, b in zip(("vertices", "textures", "metallic", "roughness"), got, ref):
        a, b = a.double().cpu().numpy(), b.cpu().numpy()
        assert np.abs(b).max() > 0, name
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max(), (name, np.abs(a - b).max() / np.abs(b).max())
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("tex6", [False, True])
def test_material_gradients_without_specular(cuda_device, kernel_calls, tex6):
    """with_specular off: neither path connects the materials to the output (no gradient), the other gradients still
    match; at the C ABI the kernel writes exact zeros into requested material gradients."""
    scene = _scene(tex6)
    _, got = _lit_grads(cuda_device, scene, EYES["per_batch"], torch.float32, True, spec=False)
    _, ref = _lit_grads(cuda_device, scene, EYES["per_batch"], torch.float64, False, spec=False)
    assert got[2] is None and got[3] is None and ref[2] is None and ref[3] is None
    for a, b in zip(got[:2], ref[:2]):
        a, b = a.double().cpu().numpy(), b.cpu().numpy()
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max()

    vb, f, tex, met, rou, gout = scene
    dev = cuda_device
    v, tx, mt, rt, g = (torch.from_numpy(x).to(dev) for x in (vb, tex, met, rou, gout))
    faces = torch.from_numpy(f)[None].repeat(vb.shape[0], 1, 1).to(dev).int().contiguous()
    eye = torch.tensor(EYES["per_batch"], device=dev)
    Tm = met[0, 0].size
    for with_spec, e in ((0, eye), (1, None)):
        gm = torch.full_like(mt, float("nan"))
        gr = torch.full_like(rt, float("nan"))
        gt = torch.empty_like(tx)
        _lib.call("b200r_surface_lighting_backward", dev, v, faces, tx, mt, rt, e, g, gt, None, gm, gr,
                  vb.shape[0], vb.shape[0], vb.shape[0], 0 if e is None else e.shape[0], vb.shape[1], f.shape[0],
                  tex[0, 0].size // 3, Tm, 0.4, _lib._f3([1, 0.9, 0.8]), 0.7, _lib._f3([0.9, 1, 0.7]),
                  _lib._f3([0.3, 1, -0.4]), with_spec)
        torch.cuda.synchronize()
        assert bool((gm == 0).all()) and bool((gr == 0).all()), (with_spec, e is None)
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("tex6", [False, True])
def test_material_gradients_leave_the_other_gradients_unchanged(cuda_device, kernel_calls, tex6):
    """Requesting material gradients changes neither the lit textures nor the texture gradients (bit for bit) nor the
    vertex gradients (beyond the float atomics' summation order)."""
    scene = _scene(tex6)
    out_a, a = _lit_grads(cuda_device, scene, EYES["per_batch"], torch.float32, True, material_grad=True)
    out_b, b = _lit_grads(cuda_device, scene, EYES["per_batch"], torch.float32, True, material_grad=False)
    assert torch.equal(out_a, out_b) and torch.equal(a[1], b[1])
    assert float((a[0] - b[0]).abs().max()) <= 1e-6 * float(b[0].abs().max())
    assert b[2] is None and b[3] is None
    hold_to_emulation(kernel_calls)


def test_material_gradients_take_the_fused_path(cuda_device):
    """metallic / roughness textures that require grad keep the one-launch kernel: one library launch forward, one
    backward."""
    scene = _scene(False)
    vb, f, tex, met, rou, gout = scene
    dev = cuda_device
    mt = torch.from_numpy(met).to(dev).requires_grad_(True)
    rt = torch.from_numpy(rou).to(dev).requires_grad_(True)
    m = jr.Mesh(torch.from_numpy(vb).to(dev), torch.from_numpy(f)[None].repeat(3, 1, 1).to(dev), textures=torch.from_numpy(tex).to(dev),
                metallic_textures=mt, roughness_textures=rt)
    light = _light()
    eye = torch.tensor(EYES["per_batch"], device=dev)
    assert light._fusable(m, eye)
    L = _lib.lib()
    torch.cuda.synchronize()
    n0 = L.b200r_launch_count()
    out = light(m, eye).textures
    n1 = L.b200r_launch_count()
    out.backward(torch.from_numpy(gout).to(dev))
    torch.cuda.synchronize()
    n2 = L.b200r_launch_count()
    assert (n1 - n0, n2 - n1) == (1, 1)
    assert mt.grad is not None and rt.grad is not None and float(mt.grad.abs().max()) > 0


def _renderer_material_grads(spot, dev, fused):
    mesh = jr.Mesh.from_obj(spot, texture_res=4, load_texture=True, dr_type='softras').to(dev)
    nf = mesh.faces.shape[1]
    rng = np.random.default_rng(11)
    p = torch.from_numpy(rng.uniform(0, 1, (1, nf, 16, 1)).astype(np.float32)).to(dev).requires_grad_(True)
    q = torch.from_numpy(rng.uniform(0.2, 1, (1, nf, 16, 1)).astype(np.float32)).to(dev).requires_grad_(True)
    target = torch.from_numpy(rng.uniform(0, 1, (1, 3, 256, 256)).astype(np.float32)).to(dev)
    r = jr.Renderer(dr_type='softras', light_intensity_directionals=1.0, light_intensity_ambient=0.0)
    r.lighting.fused = fused
    r.transform.set_eyes_from_angles(2.732, 30, 140)
    img = r(mesh.vertices, mesh.faces, mesh.textures, metallic_textures=p, roughness_textures=q)
    torch.sum((img - target) ** 2).backward()
    return p.grad.double().cpu().numpy(), q.grad.double().cpu().numpy()


def test_renderer_material_gradients_fused_vs_op_by_op(cuda_device, spot):
    """One step of the demo 5 / 6 workload on the cow: the same material gradients with the fused lighting on and off."""
    fused = _renderer_material_grads(spot, cuda_device, True)
    again = _renderer_material_grads(spot, cuda_device, True)
    mirror = _renderer_material_grads(spot, cuda_device, False)
    for k, name in enumerate(("metallic", "roughness")):
        scale = np.abs(mirror[k]).max()
        assert scale > 0
        noise = np.abs(fused[k] - again[k]).max() / scale
        err = np.abs(fused[k] - mirror[k]).max() / scale
        print("%s: fused vs op-by-op %.3e, fused run to run %.3e (of max |grad| %.3e)" % (name, err, noise, scale))
        assert err <= MATERIAL_RENDERER_TOL, (name, err, noise)


@pytest.mark.parametrize("demo,iters", [("demo5", 20), ("demo6", 15)])
def test_material_demo_converges(cuda_device, spot, demo, iters):
    """The demo 5 / 6 ports fit their material map: the loss falls over the reference's iteration count."""
    if demo == "demo5":
        from examples.demo5_optim_metallic_textures import run
    else:
        from examples.demo6_optim_roughness_textures import run
    model, losses = run(spot, iters=iters, device=str(cuda_device))
    print("%s loss %.4f -> %.4f (ratio %.4f)" % (demo, losses[0], losses[-1], losses[-1] / losses[0]))
    assert len(losses) == iters and np.all(np.isfinite(losses))
    assert losses[-1] <= CONVERGED[demo] * losses[0], losses


def test_specular_render_demo(cuda_device, spot, tmp_path):
    """demo 3: the rotation frames and the sigma / gamma sweep render lit, specular frames, and main() writes them."""
    from examples import demo3_render_specular as d3
    mesh, rotation, blurring = d3.run(spot, step=90, device=str(cuda_device))
    assert len(rotation) == 4 and len(blurring) == 10
    for img in rotation + blurring:
        assert tuple(img.shape) == (3, 256, 256) and float(img.max()) > 0.2 and bool(torch.isfinite(img).all())
    d3.main(["-i", spot, "-o", str(tmp_path), "--step", "120"])
    assert len(list(tmp_path.glob("rotation_*.png"))) == 3 and (tmp_path / "saved_spot.obj").exists()
