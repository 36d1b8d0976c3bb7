"""GPU tests of the normal-map path: the loader (bake on the GPU), the fused kernels b200r_normal_mapped_lighting_* and
the op-by-op mirror they replace.

Tolerances:
- lit textures, fused vs the golden and vs the mirror: 2e-5 of max, as for ref_host_lighting_stage;
- textures and normal textures baked on the GPU vs oracle/bake.py's emulation of the bake kernel on the same image:
  bit for bit; vs the golden's (an older float64-weight oracle bake): 2e-6 and 1e-5 (the normalize(n * 2 - 1) that
  follows scales the bake's difference by at most 2 / |2n - 1|);
- fused float32 gradients vs the mirror's float64 autograd: 1e-4 of max |grad|, as tests/test_lighting_gpu.py states;
- every fused call also against the kernels' float32 emulation (test_lighting_edges_gpu.hold_to_emulation): lit
  textures and per-texel gradients bit for bit, vertex gradients within the float atomics' order bound;
- the normal-map fit: the final loss is at most FIT_FRACTION of the first.  Measured on an NVIDIA H100 80GB HBM3
  (700 W): 0.056 after 40 iterations on the generated sphere; the threshold leaves a margin of about 3.5x.
"""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib
from jrender_b200 import io as jio
from jrender_b200 import workloads as wl
from oracle import bake as obake

from tests.test_lighting_edges_gpu import hold_to_emulation, kernel_calls  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
LIGHT = dict(intensity_ambient=0.45, color_ambient=[1.0, 0.95, 0.9], intensity_directionals=1.0,
             color_directionals=[0.9, 1.0, 0.8], directions=[0.65, -0.2, -1.0])
FIT_FRACTION = 0.2
MAPS = {"normal_rgb8": "normal.png", "bump8": "bump8.png", "bump16": "bump16.png"}


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(G, "ref_host_normal_map.npz"))


def _write_asset(g, d, kind):
    import cv2
    (d / "cow.obj").write_bytes(g["obj_text"].tobytes())
    (d / "cow.mtl").write_bytes(g["mtl_" + kind].tobytes())
    img = g["image_" + kind]
    assert cv2.imwrite(str(d / MAPS[kind]), np.ascontiguousarray(img[:, :, ::-1]) if img.ndim == 3 else img)
    return str(d / "cow.obj")


@pytest.mark.parametrize("kind", sorted(MAPS))
def test_loader_matches_reference(cuda_device, g, tmp_path, kind):
    path = _write_asset(g, tmp_path, kind)
    before = sorted(os.listdir(tmp_path))
    R = int(g["texture_res"])
    v, f, tex, nt, tbn, ftc = jio.load_obj(path, load_texture=True, texture_res=R, with_normal_map=True)
    assert len(jio.load_obj(path, load_texture=True, texture_res=R)) == 3
    assert np.array_equal(v.numpy(), g["vertices"]) and np.array_equal(f.numpy(), g["faces"])
    assert np.abs(tex.numpy() - g["textures"]).max() <= 2e-6
    assert np.abs(nt.numpy() - g["normal_textures_" + kind]).max() <= 1e-5
    assert np.array_equal(tbn.numpy(), g["TBN"]) and np.array_equal(ftc.numpy(), g["face_texcoords"])
    image = jio._imread_native01(os.path.join(str(tmp_path), MAPS[kind]))
    image = jio.bump_to_normal_map(image) if image.ndim == 2 else image
    nf = ftc.shape[0]
    baked = obake.bake_textures_for_softras(np.ascontiguousarray(image[::-1]), ftc.numpy(), np.ones((nf, R * R, 3), np.float32),
                                            np.ones(nf, np.int32))
    want = jio._normalize_np(baked * 2 - 1, 2, 1e-12)
    assert np.array_equal(nt.numpy().view(np.uint32), want.view(np.uint32))
    m = jr.Mesh.from_obj(path, load_texture=True, texture_res=R, normalization=True).to(cuda_device)
    assert tuple(m.normal_textures.shape) == (1,) + g["TBN"].shape[:1] + (R * R, 3)
    assert torch.equal(m.TBN.cpu(), torch.from_numpy(g["TBN"])[None])   # built before the normalization
    assert tuple(m.face_texcoords.shape) == (1,) + g["face_texcoords"].shape and m.face_texcoords.is_cuda
    assert sorted(os.listdir(tmp_path)) == before   # nothing written next to the asset (no normal_high.jpg)


def _golden_mesh(g, dev, spec, dtype=torch.float32):
    t = lambda k: torch.from_numpy(g[k]).to(dev, dtype)
    m = jr.Mesh(t("lit_vertices"), torch.from_numpy(g["lit_faces"]).to(dev), textures=t("lit_textures"),
                metallic_textures=t("lit_metallic"), roughness_textures=t("lit_roughness"),
                normal_textures=t("normal_textures_normal_rgb8"), TBN=t("TBN"))
    m.with_specular = spec
    return m


@pytest.mark.parametrize("tag,spec", [("specular", True), ("diffuse", False)])
def test_fused_forward_matches_golden_and_mirror(cuda_device, kernel_calls, g, tag, spec):
    eyes = torch.from_numpy(g["lit_eyes"]).to(cuda_device)
    light = jr.Lighting(**LIGHT)
    m = _golden_mesh(g, cuda_device, spec)
    L = _lib.lib()
    n0 = L.b200r_launch_count()
    fused = light(m, eyes).textures
    assert L.b200r_launch_count() - n0 == 1
    light.fused = False
    mirror = light(_golden_mesh(g, cuda_device, spec), eyes).textures
    ref = g["lit_" + tag]
    for x in (fused, mirror):
        x = x.cpu().numpy()
        assert np.abs(x - ref).max() <= 2e-5 * np.abs(ref).max()
    assert float((fused - mirror).abs().max()) <= 2e-5
    hold_to_emulation(kernel_calls)


EYES = {"per_batch": [[0.0, 0.3, -2.7], [1.0, 1.5, -2.0], [-2.0, 0.3, 1.0]],
        "shared": [[0.4, 2.2, 1.6]],
        "grazing": [[2.6, 0.05, 0.2]]}


def _scene(nb, B=3, R=3, seed=4):
    """A jittered sphere with random UVs (TBN from create_TBN), random tangent-space normals (one of them zero, where
    normalize takes its eps path), textures up to 1.6 so that texels saturate the clamp, per-texel materials."""
    rng = np.random.default_rng(seed)
    v, f = wl.sphere_by_faces(280)
    nf, T = f.shape[0], R * R
    vb = (v[None] + rng.normal(0, 0.03, (B,) + v.shape)).astype(np.float32)
    tbn = jio.create_TBN(rng.uniform(0, 1, (nf, 3, 2)).astype(np.float32), v[f])[None]
    assert np.isfinite(tbn).all()
    nt = rng.normal(0, 0.5, (nb, nf, T, 3))
    nt[..., 2] += 1
    nt = (nt / np.linalg.norm(nt, axis=-1, keepdims=True)).astype(np.float32)
    nt[:, 7, 4] = 0
    tex = rng.uniform(0, 1.6, (B, nf, T, 3)).astype(np.float32)
    met = rng.uniform(0, 1, (B, nf, T, 1)).astype(np.float32)
    rou = rng.uniform(0.2, 1, (B, nf, T, 1)).astype(np.float32)
    gout = rng.uniform(-1, 1, (B, nf, T, 3)).astype(np.float32)
    return vb, f, tex, nt, tbn, met, rou, gout


NAMES = ("vertices", "textures", "normal_textures", "metallic", "roughness")


def _grads(dev, sc, eyes, dtype, fused, spec=True, need=NAMES):
    vb, f, tex, nt, tbn, met, rou, gout = sc
    B = vb.shape[0]
    ts = [torch.from_numpy(x).to(dev, dtype).requires_grad_(n in need) for n, x in zip(NAMES, (vb, tex, nt, met, rou))]
    m = jr.Mesh(ts[0], torch.from_numpy(f)[None].repeat(B, 1, 1).to(dev), textures=ts[1], normal_textures=ts[2],
                TBN=torch.from_numpy(tbn).to(dev, dtype), metallic_textures=ts[3], roughness_textures=ts[4])
    m.with_specular = spec
    light = jr.Lighting(**LIGHT)
    light.fused = fused
    e = torch.tensor(eyes, device=dev, dtype=dtype)
    if fused:
        assert light._fused_normal_mapped(m, e) is not None
    out = light(m, e).textures
    out.backward(torch.from_numpy(gout).to(dev, dtype))
    return out.detach(), [t.grad for t in ts]


def _compare(got, ref, need=NAMES):
    for name, a, b in zip(NAMES, got, ref):
        if name not in need:
            assert a is None and b is None, name
            continue
        a, b = a.double().cpu().numpy(), b.cpu().numpy()
        assert np.isfinite(a).all() and np.abs(b).max() > 0, name
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max(), (name, np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("eyes", sorted(EYES))
def test_gradients_match_float64_autograd(cuda_device, kernel_calls, eyes, nb):
    sc = _scene(nb)
    out, got = _grads(cuda_device, sc, EYES[eyes], torch.float32, True)
    out64, ref = _grads(cuda_device, sc, EYES[eyes], torch.float64, False)
    assert np.abs(out.double().cpu().numpy() - out64.cpu().numpy()).max() <= 2e-5
    assert bool((out64 >= 1).any())   # texels that saturate the clamp are in the scene
    _compare(got, ref)
    assert float(got[2][:, 7, 4].abs().max()) == 0.0   # the zero normal: every relu is at its kink
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("nb", [1, 3])
def test_gradients_without_specular(cuda_device, kernel_calls, nb):
    """Without the Cook-Torrance branch the vertices reach nothing: autograd has no path to them, the kernel writes 0."""
    sc = _scene(nb)
    need = NAMES[:3]
    _, got = _grads(cuda_device, sc, EYES["per_batch"], torch.float32, True, spec=False, need=need)
    _, ref = _grads(cuda_device, sc, EYES["per_batch"], torch.float64, False, spec=False, need=need)
    assert ref[0] is None and float(got[0].abs().max()) == 0.0
    _compare([None] + got[1:], [None] + ref[1:], need[1:])
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("need", [("textures",), ("normal_textures",), ("vertices",), ("metallic", "roughness"),
                                  ("vertices", "normal_textures")])
def test_gradient_subsets(cuda_device, kernel_calls, need):
    """Each gradient is written only when requested, and requesting fewer changes none of the others: per-texel ones bit
    for bit, the vertex gradient beyond the float atomics' order."""
    sc = _scene(1)
    out_all, full = _grads(cuda_device, sc, EYES["per_batch"], torch.float32, True)
    out, got = _grads(cuda_device, sc, EYES["per_batch"], torch.float32, True, need=need)
    assert torch.equal(out, out_all)
    for name, a, b in zip(NAMES, got, full):
        if name not in need:
            assert a is None
        elif name == "vertices":
            assert float((a - b).abs().max()) <= 1e-6 * float(b.abs().max())
        else:
            assert torch.equal(a, b), name
    _, ref = _grads(cuda_device, sc, EYES["per_batch"], torch.float64, False, need=need)
    _compare(got, ref, need)
    hold_to_emulation(kernel_calls)


def test_grad_requiring_eye_or_tbn_runs_op_by_op(cuda_device):
    sc = _scene(1)
    vb, f, tex, nt, tbn, met, rou, gout = sc
    dev = cuda_device
    light = jr.Lighting(**LIGHT)
    mk = lambda tb: jr.Mesh(torch.from_numpy(vb).to(dev), torch.from_numpy(f)[None].repeat(3, 1, 1).to(dev),
                            textures=torch.from_numpy(tex).to(dev), normal_textures=torch.from_numpy(nt).to(dev), TBN=tb,
                            metallic_textures=torch.from_numpy(met).to(dev), roughness_textures=torch.from_numpy(rou).to(dev))
    eye = torch.tensor(EYES["per_batch"], device=dev)
    fused = light(mk(torch.from_numpy(tbn).to(dev)), eye).textures
    t = torch.from_numpy(tbn).to(dev).requires_grad_(True)
    m = mk(t)
    assert light._fused_normal_mapped(m, eye) is None
    out = light(m, eye).textures
    out.sum().backward()
    assert t.grad is not None and float((out - fused).abs().max()) <= 2e-5
    e = eye.clone().requires_grad_(True)
    m = mk(torch.from_numpy(tbn).to(dev))
    assert light._fused_normal_mapped(m, e) is None
    light(m, e).textures.sum().backward()
    assert e.grad is not None


def test_abi_rejects_bad_arguments(cuda_device):
    L = _lib.lib()
    dev = cuda_device
    B, nf, T, nv = 2, 5, 4, 6
    v = torch.zeros(B, nv, 3, device=dev)
    f = torch.zeros(B, nf, 3, dtype=torch.int32, device=dev)
    tx = torch.zeros(B, nf, T, 3, device=dev)
    nt = torch.zeros(1, nf, T, 3, device=dev)
    tb = torch.zeros(1, nf, 3, 3, device=dev)
    out = torch.empty_like(tx)
    light = (0.5, _lib._f3([1, 1, 1]), 0.5, _lib._f3([1, 1, 1]), _lib._f3([0, 1, 0]), 1)
    P = lambda x: None if x is None else x.data_ptr()

    def fwd(v_=v, nt_=nt, tb_=tb, out_=out, counts=(B, B, B, 0, 1, nf, T, 1, nf, nv, nf, T)):
        return L.b200r_normal_mapped_lighting_forward(P(v_), P(f), P(tx), P(nt_), P(tb_), None, None, None, P(out_), *counts,
                                                      *light, None)

    def bwd(counts=(B, B, B, 0, 1, nf, T, 1, nf, nv, nf, T), g=out):
        return L.b200r_normal_mapped_lighting_backward(P(v), P(f), P(tx), P(nt), P(tb), None, None, None, P(g), None, None,
                                                       None, P(out), None, *counts, *light, None)
    assert fwd() == 0
    torch.cuda.synchronize()
    for kw in (dict(v_=None), dict(nt_=None), dict(tb_=None), dict(out_=None)):
        assert fwd(**kw) == -1 and b"NULL" in L.b200r_last_error(), kw
    for counts in ((B, B, B, 0, 1, nf + 1, T, 1, nf, nv, nf, T), (B, B, B, 0, 1, nf, T - 1, 1, nf, nv, nf, T),
                   (B, B, B, 0, 1, nf, T, 1, nf - 1, nv, nf, T)):
        assert fwd(counts=counts) == -1 and b"do not match" in L.b200r_last_error(), counts
    for counts in ((B, B, B, 0, 3, nf, T, 1, nf, nv, nf, T), (B, B, B, 0, 1, nf, T, 3, nf, nv, nf, T)):
        assert fwd(counts=counts) == -1 and b"batch" in L.b200r_last_error(), counts
    assert bwd(g=None) == -1 and b"NULL" in L.b200r_last_error()
    assert bwd() == -1 and b"material gradients" in L.b200r_last_error()   # grad_metallic without metallic


def test_renderer_fused_vs_op_by_op(cuda_device, g):
    """Renderer.render_mesh on the golden's cow piece: the whole pipeline with the fused lighting and without."""
    imgs = []
    for fused in (True, False):
        m = _golden_mesh(g, cuda_device, True)
        m.vertices = m.vertices[:1] * 2.0
        m.faces, m.textures = m.faces[:1], m.textures[:1]
        m.metallic_textures, m.roughness_textures = m.metallic_textures[:1], m.roughness_textures[:1]
        r = jr.Renderer(image_size=128, dist_func="barycentric", aggr_func_rgb='hard', light_intensity_ambient=0.45,
                        light_intensity_directionals=1, light_directions=[0.65, -0.2, -1])
        r.lighting.fused = fused
        r.transform.set_eyes_from_angles(2.0, 20.0, 200.0)
        imgs.append(r.render_mesh(m, mode='rgb'))
    assert float(imgs[0].max()) > 0.1
    assert float((imgs[0] - imgs[1]).abs().max()) <= 2e-5


def test_normal_map_fit_converges(cuda_device, tmp_path):
    """The demo's --fit on the generated sphere at a small size: the image loss falls to FIT_FRACTION of its start and
    the fitted normals move toward the true ones."""
    from examples import demo1_5_render_normal_map as demo
    path = demo.write_sphere_asset(str(tmp_path), segments=24, rings=12)
    mesh = jr.Mesh.from_obj(path, load_texture=True, texture_res=3, normalization=True).to(cuda_device)
    r = demo.renderer(128)
    az = [0.0, 90.0, 180.0, 270.0]
    with torch.no_grad():
        targets = [t.detach() for t in demo.render_views(r, mesh, mesh.normal_textures, az)]
    losses, angles, start = demo.fit(r, mesh, targets, az, iters=40)
    print("fit loss %.4g -> %.4g (ratio %.4f); angle %.2f -> %.2f deg" % (losses[0], losses[-1], losses[-1] / losses[0],
                                                                            start, angles[-1]))
    assert np.all(np.isfinite(losses)) and losses[-1] <= FIT_FRACTION * losses[0], losses
    assert angles[-1] < start
