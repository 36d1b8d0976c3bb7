"""Lighting's routes on the CPU (the op-by-op chain) over light_mode x Gbuffer x normal map x texture rank x specular x
batch x directional-light count x transform: every combination raises the error pinned here, and no other, or lights
the textures into their own shape.  Where the reference's own Lighting.execute covers a case (tests/golden/
ref_host_gbuffer.npz, ref_host_lighting_stage.npz, ref_host_normal_map.npz: one directional light) the result agrees
with it within 2e-5 of the array's max, the tolerance test_host_golden.py uses for the lighting stage."""
import itertools
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200.lighting import DirectionalLighting, Lighting

G = os.path.join(os.path.dirname(__file__), "golden")
LIGHT = dict(intensity_ambient=0.4, color_ambient=[1.0, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1.0, 0.7], directions=[0.3, 0.8, -0.5])
SECOND = (0.3, [0.5, 0.6, 1.0], [-0.4, 0.2, 0.9])    # intensity, colour, direction of the second directional light
TOL = 2e-5
GBUFFERS = (None, 'albedo', 'normal', 'depth')
GRID = list(itertools.product(('surface', 'vertex'), GBUFFERS, (False, True), (4, 6), (False, True), (1, 2), (1, 2),
                              (False, True)))
NOT_SOFTRAS = "a normal map needs SoftRas surface textures"
DEPTH_OF_TEXELS = "vertices Tensor should have 3 dimensions"
NO_TRANSFORM = "needs the renderer's transform"


def _close(a, b, tol=TOL):
    b = np.asarray(b, np.float64)
    return np.abs(np.asarray(a, np.float64) - b).max() <= tol * max(np.abs(b).max(), 1e-30)


@pytest.fixture(scope="module")
def gb():
    return np.load(os.path.join(G, "ref_host_gbuffer.npz"))


def _golden_tag(light_mode, gbuffer, nm, rank, spec):
    """The ref_host_gbuffer.npz case with these settings, whether or not the golden holds it."""
    branch = 'vertex' if light_mode == 'vertex' else 'normalmap' if nm else 'surface%d' % rank
    return "%s_%s_spec%d" % (gbuffer, branch, spec)


def _case(g, light_mode, gbuffer, nm, rank, spec, B, lights, transform, with_SSS=False):
    """Lighting and a Mesh from ref_host_gbuffer.npz's inputs, the first B of its batch of 2; textures [B, nf, 4, 3] or
    [B, nf, 2, 2, 2, 3] over the faces, [B, nv, 1, 3] or [B, nv, 2, 2, 2, 3] over the vertices in vertex mode, seeded
    where the golden has none; metallic / roughness per face and texel, or per vertex."""
    t = lambda k: torch.from_numpy(g[k][:B])
    n = g["vertices"].shape[1] if light_mode == 'vertex' else g["faces"].shape[1]
    tag = "in_" + _golden_tag(light_mode, gbuffer, nm, rank, spec)
    shape = (B, n) + (((1,) if light_mode == 'vertex' else (4,)) if rank == 4 else (2, 2, 2)) + (3,)
    tex = t(tag) if tag in g and g[tag].shape[1:] == shape[1:] else \
        torch.rand(shape, generator=torch.Generator().manual_seed(rank + 10 * B), dtype=torch.float32)
    material = lambda k: t(k)[:, :n, 0] if light_mode == 'vertex' else t(k)   # [B, nv, 1] per vertex
    mesh = jr.Mesh(t("vertices"), t("faces"), textures=tex, dr_type='n3mr' if rank == 6 else 'softras',
                   metallic_textures=material("metallic"), roughness_textures=material("roughness"),
                   normal_textures=t("normal_textures") if nm else None, TBN=t("tbn") if nm else None, texture_res=2,
                   with_SSS=with_SSS)
    mesh.with_specular = spec
    eyes = t("eyes")
    tr = None
    if transform:
        tr = jr.Transform(camera_mode='look_at', viewing_angle=30)
        tr.set_eyes(eyes)
    light = Lighting(light_mode, Gbuffer=gbuffer, transform=tr, **LIGHT)
    if lights == 2:
        light.directionals.append(DirectionalLighting(*SECOND, Gbuffer=gbuffer, transform=tr))
    return light, mesh, eyes


def _expected_error(light_mode, gbuffer, nm, rank, transform):
    """The message of the ValueError Lighting raises, None where it lights."""
    if gbuffer == 'albedo':
        return None
    if light_mode == 'surface' and nm:   # vertex mode ignores a normal map
        if rank != 4:
            return NOT_SOFTRAS
        if gbuffer == 'depth':            # the texel positions reach look_at's check, with or without a transform
            return DEPTH_OF_TEXELS
    if gbuffer == 'depth' and not transform:
        return NO_TRANSFORM
    return None


@pytest.mark.parametrize("light_mode", ('surface', 'vertex'))
def test_route_outcomes_over_the_grid(gb, light_mode):
    covered = 0
    for case in GRID:
        if case[0] != light_mode:
            continue
        _, gbuffer, nm, rank, spec, B, lights, transform = case
        light, mesh, eyes = _case(gb, *case)
        tex = mesh.textures
        err = _expected_error(light_mode, gbuffer, nm, rank, transform)
        if err is not None:
            with pytest.raises(ValueError, match=err):
                light(mesh, eyes)
            continue
        out = light(mesh, eyes).textures
        if gbuffer == 'albedo':
            assert out is tex, case
            continue
        assert out.shape == tex.shape and out.dtype == tex.dtype, case
        assert torch.isfinite(out).all() and (out >= 0).all() and (out <= 1).all(), case
        ref = gb["out_" + _golden_tag(light_mode, gbuffer, nm, rank, spec)] \
            if gbuffer is not None and "out_" + _golden_tag(light_mode, gbuffer, nm, rank, spec) in gb.files else None
        # one light, and the depth's max over the whole batch of 2 (the normal G-buffer is per batch element)
        if ref is not None and lights == 1 and (B == 2 or gbuffer == 'normal') and ref.shape[1:] == tuple(out.shape[1:]):
            assert _close(out.numpy(), ref[:B]), case
            covered += 1
    assert covered == {'surface': 23, 'vertex': 10}[light_mode]   # vertex mode ignores a normal map


@pytest.mark.parametrize("B", (1, 2))
@pytest.mark.parametrize("spec", (False, True))
def test_lit_routes_match_reference(B, spec):
    """Gbuffer None on the face-normal route (ref_host_lighting_stage.npz, the default lights) and on the normal-map
    route (ref_host_normal_map.npz and its lights); no batch element depends on another."""
    s = np.load(os.path.join(G, "ref_host_lighting_stage.npz"))
    m = jr.Mesh(torch.from_numpy(s["vertices"][:B]), torch.from_numpy(s["faces"][:B]),
                textures=torch.from_numpy(s["textures"][:B].copy()))
    m.with_specular = spec
    out = Lighting()(m, torch.from_numpy(s["eyes"][:B])).textures
    assert _close(out.numpy(), s["lit_" + ("specular" if spec else "diffuse")][:B])
    g = np.load(os.path.join(G, "ref_host_normal_map.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(torch.float64)
    m = jr.Mesh(t("lit_vertices")[:B], torch.from_numpy(g["lit_faces"][:B]), textures=t("lit_textures")[:B],
                metallic_textures=t("lit_metallic")[:B], roughness_textures=t("lit_roughness")[:B],
                normal_textures=t("normal_textures_normal_rgb8"), TBN=t("TBN"))
    m.with_specular = spec
    out = Lighting(intensity_ambient=0.45, color_ambient=[1.0, 0.95, 0.9], intensity_directionals=1.0,
                   color_directionals=[0.9, 1.0, 0.8], directions=[0.65, -0.2, -1.0])(m, t("lit_eyes")[:B]).textures
    assert _close(out.numpy(), g["lit_" + ("specular" if spec else "diffuse")][:B])


@pytest.mark.parametrize("transform", (False, True))
def test_subsurface_depth_with_normal_map_fails_in_the_depth_terms(gb, transform):
    """with_SSS meshes with 4-D textures skip the fused attempt, so depth with a normal map fails where the light terms
    meet camera_z: on the missing transform first, then on the texel positions' rank."""
    light, mesh, eyes = _case(gb, 'surface', 'depth', True, 4, True, 2, 1, transform, with_SSS=True)
    with pytest.raises(ValueError, match=DEPTH_OF_TEXELS if transform else NO_TRANSFORM):
        light(mesh, eyes)


def test_bad_light_mode_and_gbuffer_raise():
    with pytest.raises(ValueError, match="Lighting mode only support surface and vertex"):
        Lighting('face')
    with pytest.raises(ValueError, match="Gbuffer must be 'None', 'albedo', 'normal' or 'depth'"):
        Lighting(Gbuffer='depht')
