"""CPU checks of the normal-map path against tests/golden/ref_host_normal_map.npz (oracle/make_ref_host_normal_map_golden.py,
the reference's own Python through the numpy jittor stand-in): MTL parsing, bump -> normal conversion at 8 and 16 bits,
the TBN (including degenerate UV triangles), the Mesh normal properties and the op-by-op Lighting mirror of the
normal-map branch.  Tolerance of the lit textures: 2e-5 of max, as for ref_host_lighting_stage."""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import io as jio

G = os.path.join(os.path.dirname(__file__), "golden")
LIGHT = dict(intensity_ambient=0.45, color_ambient=[1.0, 0.95, 0.9], intensity_directionals=1.0,
             color_directionals=[0.9, 1.0, 0.8], directions=[0.65, -0.2, -1.0])


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(G, "ref_host_normal_map.npz"))


def test_load_mtl_reads_map_normal(g, tmp_path):
    p = tmp_path / "a.mtl"
    p.write_bytes(g["mtl_bump16"].tobytes())
    assert jio.load_mtl(str(p), with_normal_map=True)[2] == "bump16.png"
    assert len(jio.load_mtl(str(p))) == 2                  # the two-value form is unchanged
    p.write_text("newmtl a\nmap_Kd a.png\nmap_normal 1.0 first.png\nnewmtl b\nmap_normal 2 second.png\n")
    colors, files, normal = jio.load_mtl(str(p), with_normal_map=True)
    assert normal == "second.png" and files == {"a": "a.png"}   # the scale is ignored, the last line wins
    p.write_text("newmtl a\nKd 1 1 1\n")
    assert jio.load_mtl(str(p), with_normal_map=True)[2] == ""
    p.write_text("newmtl a\nmap_normal bump.png\n")
    with pytest.raises(ValueError, match="map_normal bump.png"):
        jio.load_mtl(str(p), with_normal_map=True)


@pytest.mark.parametrize("kind,top", [("bump8", 1.0), ("bump16", 257.0)])
def test_bump_to_normal_map(g, tmp_path, kind, top):
    """Read at the native bit depth and divided by 255 (a 16-bit image reaches 257), then converted exactly as the
    reference converts it."""
    import cv2
    img = g["image_" + kind]
    path = str(tmp_path / (kind + ".png"))
    assert cv2.imwrite(path, img)
    b = jio._imread_native01(path)
    assert b.shape == img.shape and b.dtype == np.float32 and float(b.max()) == top
    n = jio.bump_to_normal_map(b)
    ref = g["bump_to_normal_" + kind]
    assert n.shape == (img.shape[0] - 2, img.shape[1] - 2, 3)
    assert np.array_equal(n, ref)


def test_rgb_normal_map_is_read_as_rgb(g, tmp_path):
    import cv2
    img = g["image_normal_rgb8"]
    path = str(tmp_path / "n.png")
    assert cv2.imwrite(path, np.ascontiguousarray(img[:, :, ::-1]))
    assert np.array_equal(jio._imread_native01(path), img.astype(np.float32) / 255.)


def test_tbn_matches_reference(g):
    fw = g["vertices"][g["faces"]]
    assert np.array_equal(jio.create_TBN(g["face_texcoords"], fw), g["TBN"])
    got = jio.create_TBN(g["tbn_cases_uv"], g["tbn_cases_xyz"])
    ref = g["tbn_cases_out"]
    assert np.array_equal(got, ref, equal_nan=True)
    # degenerate UV triangles (collinear, coincident) divide by zero and leave a non-finite frame, as in the reference;
    # a zero-area triangle gets a zero normal and binormal
    assert not np.isfinite(got[1, :2]).any() and not np.isfinite(got[2, :2]).any()
    assert np.isfinite(got[0]).all() and np.array_equal(got[3, 1:], np.zeros((2, 3), np.float32))


def _mesh(g, dtype=torch.float64, spec=True):
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    m = jr.Mesh(t("lit_vertices"), torch.from_numpy(g["lit_faces"]), textures=t("lit_textures"),
                metallic_textures=t("lit_metallic"), roughness_textures=t("lit_roughness"),
                normal_textures=t("normal_textures_normal_rgb8"), TBN=t("TBN"))
    m.with_specular = spec
    return m


def test_mesh_normal_properties(g):
    m = _mesh(g, torch.float32)
    assert tuple(m.normal_textures.shape) == (1,) + g["normal_textures_normal_rgb8"].shape
    assert tuple(m.TBN.shape) == (1,) + g["TBN"].shape
    for k in ("surface_ResNormals", "surface_normals"):
        got = getattr(m, k).numpy()
        assert got.shape == g[k].shape and np.abs(got - g[k]).max() <= 2e-6, k


@pytest.mark.parametrize("tag,spec", [("specular", True), ("diffuse", False)])
def test_mirror_matches_reference_golden(g, tag, spec):
    ref = g["lit_" + tag]
    for dtype in (torch.float32, torch.float64):
        m = _mesh(g, dtype, spec)
        lit = jr.Lighting(**LIGHT)(m, torch.from_numpy(g["lit_eyes"]).to(dtype)).textures.numpy()
        assert lit.shape == ref.shape
        assert np.abs(lit - ref).max() <= 2e-5 * np.abs(ref).max(), (dtype, np.abs(lit - ref).max())
    assert (ref >= 1).any() and (ref < 1).any()


def test_flat_path_unchanged_without_normal_map():
    """A mesh without a normal map keeps the face-normal branch: ref_host_lighting_stage at its stated tolerance."""
    s = np.load(os.path.join(G, "ref_host_lighting_stage.npz"))
    m = jr.Mesh(torch.from_numpy(s["vertices"]), torch.from_numpy(s["faces"]), textures=torch.from_numpy(s["textures"]))
    assert m.normal_textures is None and m.TBN is None and m.surface_ResNormals is None
    lit = jr.Lighting()(m, torch.from_numpy(s["eyes"])).textures.numpy()
    assert np.abs(lit - s["lit_specular"]).max() <= 2e-5 * np.abs(s["lit_specular"]).max()


def test_normal_map_needs_matching_softras_textures(g):
    m = _mesh(g)
    m.textures = m.textures[:, :, :4]
    with pytest.raises(ValueError, match="do not match"):
        jr.Lighting()(m, torch.from_numpy(g["lit_eyes"]))
    m = _mesh(g)
    m.textures = torch.ones(2, m.faces.shape[1], 2, 2, 2, 3, dtype=torch.float64)
    with pytest.raises(ValueError, match="SoftRas surface textures"):
        jr.Lighting()(m, torch.from_numpy(g["lit_eyes"]))
