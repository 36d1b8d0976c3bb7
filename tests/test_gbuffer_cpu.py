"""Normal and depth G-buffers (Lighting(Gbuffer='normal' | 'depth')) on the CPU: the op-by-op mirror against the
reference's own Lighting.execute and Renderer.render_mesh (tests/golden/ref_host_gbuffer.npz, oracle/
make_ref_host_gbuffer_golden.py) within 2e-5 of each array's max, the tolerance test_host_golden.py uses for the lighting
stage; the float32 emulation of the kernels (oracle/gbuffer.py) against the float64 mirror; and the decisions the
reference leaves open: the max's gradient on ties, NaN through the max, and the error cases."""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200.lighting import Lighting, _normalized_direction, camera_z
from oracle import gbuffer as OG
from oracle.numbers import F32

G = os.path.join(os.path.dirname(__file__), "golden", "ref_host_gbuffer.npz")
LIGHT = dict(intensity_ambient=0.4, color_ambient=[1.0, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1.0, 0.7], directions=[0.3, 0.8, -0.5])
TOL = 2e-5


def _close(a, b, tol=TOL):
    b = np.asarray(b, np.float64)
    return np.abs(np.asarray(a, np.float64) - b).max() <= tol * max(np.abs(b).max(), 1e-30)


def _transform(eyes):
    t = jr.Transform(camera_mode='look_at', viewing_angle=30)
    t.set_eyes(eyes)
    return t


def _golden_case(g, tag, dtype=torch.float32):
    mode, branch, spec = tag.split("_")
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    light_mode = 'vertex' if branch == 'vertex' else 'surface'
    nm = branch == 'normalmap'
    tex = t("in_" + tag) if ("in_" + tag) in g else torch.rand(g["metallic"].shape[:3] + (3,), dtype=dtype)
    mesh = jr.Mesh(t("vertices"), torch.from_numpy(g["faces"]), textures=tex,
                   dr_type='n3mr' if tex.dim() == 6 else 'softras',
                   metallic_textures=t("metallic"), roughness_textures=t("roughness"),
                   normal_textures=t("normal_textures") if nm else None, TBN=t("tbn") if nm else None,
                   texture_res=2)
    mesh.with_specular = spec == "spec1"
    eyes = t("eyes")
    return Lighting(light_mode, Gbuffer=mode, transform=_transform(eyes), **LIGHT), mesh, eyes


def test_mirror_matches_reference_lighting():
    g = np.load(G)
    tags = sorted(k[4:] for k in g.files if k.startswith("out_"))
    assert len(tags) == 10
    for tag in tags:
        light, mesh, eyes = _golden_case(g, tag)
        out = light(mesh, eyes).textures
        assert out.shape == g["out_" + tag].shape, tag
        assert _close(out.numpy(), g["out_" + tag]), tag


@pytest.mark.parametrize("camera_mode", ["look_at", "look", "projection"])
def test_depth_with_normal_map_raises_the_reference_error(camera_mode):
    g = np.load(G)
    assert str(g["err_depth_normalmap_spec1"]) == 'vertices Tensor should have 3 dimensions'
    light, mesh, eyes = _golden_case(g, "depth_normalmap_spec1")
    kw = dict(K=np.eye(3, dtype=np.float32)[None], R=np.eye(3, dtype=np.float32)[None],
              t=np.zeros((1, 3), np.float32)) if camera_mode == 'projection' else {}
    light.directionals[0].transform = light.transform = jr.Transform(camera_mode=camera_mode, **kw)
    with pytest.raises(ValueError, match=str(g["err_depth_normalmap_spec1"])):
        light(mesh, eyes)


def test_depth_without_transform_and_unknown_gbuffer_raise():
    g = np.load(G)
    light, mesh, eyes = _golden_case(g, "depth_surface4_spec1")
    light.directionals[0].transform = light.transform = None
    with pytest.raises(ValueError, match="transform"):
        light(mesh, eyes)
    with pytest.raises(ValueError, match="Gbuffer"):
        Lighting(Gbuffer='depht')
    for ok in ('None', None, 'albedo', 'normal', 'depth'):
        Lighting(Gbuffer=ok)


def test_textures_get_no_gradient():
    g = np.load(G)
    for tag in ("normal_surface4_spec1", "depth_surface4_spec0"):
        light, mesh, eyes = _golden_case(g, tag)
        tex = mesh.textures.clone().requires_grad_(True)
        v = mesh.vertices.clone().requires_grad_(True)
        mesh = jr.Mesh(v, mesh.faces, textures=tex)
        light(mesh, eyes).textures.sum().backward()
        assert tex.grad is None and torch.isfinite(v.grad).all() and v.grad.abs().sum() > 0


def test_max_gradient_goes_in_full_to_every_tie():
    """Two faces mirrored about the view plane of a camera on the z axis have the same depth: both get the max's whole
    gradient (the mask z == max), where torch.max would split it."""
    v = torch.tensor([[[-1., 0., 1.], [0., 1., 1.], [0., -1., 1.], [1., 0., 1.], [0., 0., 0.5]]], dtype=torch.float64,
                     requires_grad=True)
    f = torch.tensor([[[0, 1, 2], [3, 2, 1], [0, 4, 1]]])
    mesh = jr.Mesh(v, f, textures=torch.ones((1, 3, 1, 3), dtype=torch.float64))
    mesh.with_specular = False
    tr = jr.Transform(camera_mode='look_at', eye=[0., 0., -3.])
    light = Lighting(Gbuffer='depth', transform=tr)
    z = camera_z(tr, torch.sum(mesh.face_vertices, dim=2) / 3.0)
    assert z[0, 0] == z[0, 1] == z.max() and z[0, 2] < z[0, 0]
    out = light(mesh, None).textures
    g = torch.zeros_like(out)
    g[0, 2] = 1.0   # only the third face's output: its depth z2 / M reaches the tied faces through M alone
    out.backward(g)
    M, z2 = z.max().item(), z[0, 2].item()
    dM = -3 * z2 / (M * M)
    # the depth's z row is (0, 0, 1) here: each tied face passes dM / 3 to each of its vertices' z
    want = np.zeros((5, 3))
    for fi in (0, 1):
        for k in f[0, fi].tolist():
            want[k, 2] += dM / 3
    for k in f[0, 2].tolist():
        want[k, 2] += 3 / M / 3
    assert np.allclose(v.grad[0].numpy(), want, rtol=1e-12, atol=1e-12)


def test_nan_depth_reaches_the_whole_batch():
    g = np.load(G)
    light, mesh, eyes = _golden_case(g, "depth_surface4_spec0")
    v = mesh.vertices.clone()
    v[1, 0, 0] = float('nan')
    mesh = jr.Mesh(v, mesh.faces, textures=mesh.textures)
    mesh.with_specular = False
    out = light(mesh, eyes).textures
    assert torch.isnan(out).all()


def host_args(mesh, light, eyes, mode):
    """The arguments Lighting hands b200r_gbuffer_lighting_forward, built on the host (no GPU)."""
    d = light.directionals[0]
    spec = bool(mesh.with_specular)
    tx = mesh.textures
    B, nf = tx.shape[:2]
    tr = light.transform
    a = dict(vertices=mesh.vertices.numpy().astype(F32), faces=mesh.faces.numpy().astype(np.int32),
             metallic=mesh.metallic_textures.numpy().reshape(B, nf, -1) if spec else None,
             roughness=mesh.roughness_textures.numpy().reshape(B, nf, -1) if spec else None,
             eye=eyes.numpy().reshape(-1, 3) if spec else None, camera_eye=np.asarray(tr.transformer._eye, F32).reshape(-1, 3),
             mode=mode, B=B, Bv=mesh.vertices.shape[0], Bf=mesh.faces.shape[0], Be=eyes.shape[0], Bc=1, nv=mesh.vertices.shape[1],
             nf=nf, T=tx[0, 0].numel() // 3, Tm=mesh.metallic_textures[0, 0].numel(), at=np.zeros(3, F32),
             up=np.float32([0, 1, 0]), camera_mode=0)
    a["Bc"] = a["camera_eye"].shape[0]
    a["light"] = OG._light(d.light_intensity, d.light_color, _normalized_direction(d.light_direction), spec)
    return a


def test_emulation_agrees_with_float64_mirror():
    g = np.load(G)
    for tag in ("normal_surface4_spec1", "normal_surface6_spec1", "depth_surface4_spec1", "depth_surface4_spec0"):
        light, mesh, eyes = _golden_case(g, tag, torch.float64)
        a = host_args(mesh, light, eyes, 0 if tag.startswith("normal") else 1)
        want = light(mesh, eyes).textures.numpy()
        got, _ = OG.gbuffer_forward(a)
        assert _close(got.reshape(want.shape), want, 1e-6), tag


def test_edge_scenes_reach_nonpositive_max_depth():
    """The 'behind' scenes put every centroid behind the camera (M < 0: every z / M >= 1, only the max face at the
    clamp's equality); 'zero_max' makes the largest depth exactly 0 (M = 0)."""
    from tests import gbuffer_edge_cases as E
    for name, check in (("behind_depth_nospec", lambda M, z: M < 0 and (z < 0).all()),
                        ("behind_depth_spec", lambda M, z: M < 0 and (z < 0).all()),
                        ("zero_max_depth_nospec", lambda M, z: M == 0 and int((z == 0).sum()) == z.shape[0])):
        sc = E.scene(name)
        ts, light, mesh, eyes = E.build(sc, torch.device("cpu"), torch.float64, fused=False)
        z = camera_z(light.transform, torch.sum(mesh.face_vertices, dim=2) / 3.0).detach()
        assert check(z.max().item(), z), name
