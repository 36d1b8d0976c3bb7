"""CPU tests of the texture-atlas export (create_texture_image / save_obj with textures / Mesh.save_obj(save_texture=True)).

- the numpy oracle (oracle/texture_atlas.py) on cases checkable by hand;
- the product's host side (tile layout, vertical flip, clip + uint8, PNG / MTL / OBJ text) with the CUDA kernel replaced
  by the oracle, against the reference's own io/save_obj.py run through the numpy jittor stub
  (tests/golden/ref_host_save_obj.npz, generator oracle/make_ref_host_save_obj_golden.py);
- argument errors.
The kernels themselves are tested on the GPU (tests/test_texture_atlas_gpu.py).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import io as jio
from oracle import texture_atlas as oat
from tests.conftest import ROOT

G = os.path.join(ROOT, "tests", "golden")


def _oracle_atlas(tile_vertices, textures, texture_res_out, tile_width, image_height, image_width, device=None):
    t = textures.detach().cpu().numpy() if isinstance(textures, torch.Tensor) else np.asarray(textures)
    fn = oat.texture_atlas_softras if t.ndim == 3 else oat.texture_atlas_n3mr
    return fn(np.asarray(tile_vertices), t, texture_res_out, tile_width, image_height, image_width)


@pytest.fixture
def oracle_kernel(monkeypatch):
    """The product's create_texture_image / save_obj with the CUDA kernel call replaced by the oracle."""
    monkeypatch.setattr(jio, "texture_atlas", _oracle_atlas)


@pytest.mark.parametrize("nf,R_out", [(1, 2), (7, 4), (10, 16), (26, 5)])
def test_oracle_one_colour_per_face_fills_its_tile(nf, R_out):
    """One texel per face (SoftRas R 1) or a constant volume (NMR ts 2, 3): every pixel of a used tile is that face's
    colour, every pixel of an unused tile is white."""
    rng = np.random.default_rng(nf)
    col = rng.random((nf, 3), dtype=np.float32)
    tri, tw, th = oat.atlas_layout(nf, R_out)
    H, W = th * R_out, tw * R_out
    want = np.ones((th, tw, 3), np.float32).reshape(-1, 3)
    want[:nf] = col
    want = np.repeat(np.repeat(want.reshape(th, tw, 3), R_out, 0), R_out, 1)
    img = oat.texture_atlas_softras(tri, col[:, None, :], R_out, tw, H, W)
    assert np.array_equal(img, want)
    for ts in (2, 3):
        vol = np.ascontiguousarray(np.broadcast_to(col[:, None, None, None, :], (nf, ts, ts, ts, 3)))
        img = oat.texture_atlas_n3mr(tri, vol, R_out, tw, H, W)
        assert np.abs(img - want).max() <= 1e-6


@pytest.mark.parametrize("R,R_out", [(4, 64), (5, 64), (2, 16)])
def test_oracle_paints_each_texel_at_its_bake_sample_point(R, R_out):
    """R > 1: the pixel nearest to the point the bake samples texel t from (load_textures.py:29-37: (w_x + 1/3) / R,
    (w_y + 1/3) / R in the lower half of a cell, (R - 1 - w + 2/3) / R in the upper) holds texel t."""
    nf = 5
    tex = np.arange(nf * R * R * 3, dtype=np.float32).reshape(nf, R * R, 3)
    tri, tw, th = oat.atlas_layout(nf, R_out)
    img = oat.texture_atlas_softras(tri, tex, R_out, tw, th * R_out, tw * R_out)
    for fn in range(nf):
        for t in range(R * R):
            wy, wx = divmod(t, R)
            if wx + wy < R:
                w0, w1 = (wx + 1 / 3) / R, (wy + 1 / 3) / R
            else:
                w0, w1 = (R - 1 - wx + 2 / 3) / R, (R - 1 - wy + 2 / 3) / R
            p = w0 * tri[fn, 0] + w1 * tri[fn, 1] + (1 - w0 - w1) * tri[fn, 2]
            x, y = int(round(p[0])), int(round(p[1]))
            assert np.array_equal(img[y, x], tex[fn, t]), (fn, t, x, y)


def test_oracle_nmr_reads_the_barycentric_slice():
    """NMR: at a tile vertex the weights are one-hot, so the pixel there samples the volume's corner texel of that vertex
    (ts - 1 - 1e-3 along its axis: 0.999 of the corner, 0.001 of its neighbour)."""
    nf, ts, R_out = 3, 3, 16
    rng = np.random.default_rng(4)
    vol = rng.random((nf, ts, ts, ts, 3), dtype=np.float32)
    tri, tw, th = oat.atlas_layout(nf, R_out)
    img = oat.texture_atlas_n3mr(tri, vol, R_out, tw, th * R_out, tw * R_out)
    w = oat.tile_weights(tri, R_out, tw, th * R_out, tw * R_out)[2]
    for fn in range(nf):
        for k in range(3):               # vertex 0 -> texel (ts-1, 0, 0), 1 -> (0, ts-1, 0), 2 -> (0, 0, ts-1)
            x, y = int(tri[fn, k, 0]), int(tri[fn, k, 1])
            assert w[y * tw * R_out + x, k] > 0.999
            corner, near = [0, 0, 0], [0, 0, 0]
            corner[k], near[k] = ts - 1, ts - 2
            want = 0.999 * vol[fn][tuple(corner)] + 0.001 * vol[fn][tuple(near)]
            assert np.abs(img[y, x] - want).max() <= 1e-4


def test_oracle_matches_reference_kernel_golden():
    """The oracle against the reference's own kernel run on a GPU (tests/golden/ref_atlas_gpu_*.npz): at most 1e-3 of the
    pixels may pick another texel (that build contracts a*b+c)."""
    import glob
    files = sorted(glob.glob(os.path.join(G, "ref_atlas_gpu_*.npz")))
    assert len(files) >= 4, "golden fixtures missing"
    for p in files:
        g = np.load(p)
        ref = g["image"]
        got = oat.texture_atlas_softras(g["tile_vertices"], g["textures"], int(g["texture_res_out"]), int(g["tile_width"]),
                                        ref.shape[0], ref.shape[1])
        assert (got != ref).any(axis=-1).mean() <= 1e-3, p
        assert "H100" in json.loads(str(g["provenance"]))["gpu"]


def _golden():
    g = np.load(os.path.join(G, "ref_host_save_obj.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _text(a):
    return bytes(a).decode()


def test_create_texture_image_layout(oracle_kernel):
    """save_obj.py:7-29 with the integer tile row: image [H, W, 3] flipped vertically, UVs = tile triangle / (W-1, H-1)."""
    nf, R_out = 7, 8
    tex = np.random.default_rng(1).random((nf, 4, 3), dtype=np.float32)
    img, uv = jr.create_texture_image(torch.from_numpy(tex).requires_grad_(True), R_out)
    tri, tw, th = oat.atlas_layout(nf, R_out)
    assert (tw, th) == (3, 3) and img.shape == (24, 24, 3) and img.dtype == np.float32 and uv.dtype == np.float32
    assert np.array_equal(img, oat.texture_atlas_softras(tri, tex, R_out, tw, 24, 24)[::-1])
    assert np.array_equal(uv[..., 0], tri[..., 0] / np.float32(23)) and np.array_equal(uv[..., 1], tri[..., 1] / np.float32(23))
    assert np.array_equal(tri[4], np.float32([[12, 9], [9, 14], [14, 14]]))   # face 4: column 1, row 1


def test_save_obj_surface_matches_reference_python(oracle_kernel, tmp_path):
    """The reference's save_obj (through the stub, its CUDA op replaced by the oracle) and the product's give the same PNG
    and MTL, and the same OBJ text except the `vt` lines the reference's fractional tile row moves: faces outside the
    first tile column.  Those lines hold the integer-row layout here."""
    import cv2
    g, meta = _golden()
    for case in ("surface_r1", "surface_single"):
        m = meta[case]
        fn = str(tmp_path / case / m["filename"])
        os.makedirs(os.path.dirname(fn))
        tex = g[case + "_textures"]
        jr.save_obj(fn, torch.from_numpy(g[case + "_vertices"]), torch.from_numpy(g[case + "_faces"]), textures=torch.from_numpy(tex),
                    texture_res=m["texture_res"], texture_type="surface")
        png = cv2.imread(fn[:-4] + ".png", cv2.IMREAD_UNCHANGED)
        assert png.dtype == np.uint8 and np.array_equal(png[:, :, ::-1], g[case + "_png_rgb"])
        assert open(fn[:-4] + ".mtl").read() == _text(g[case + "_mtl"])
        ours, ref = open(fn).read().split("\n"), _text(g[case + "_obj"]).split("\n")
        assert len(ours) == len(ref)
        nf = tex.shape[0]
        tri, tw, th = oat.atlas_layout(nf, m["texture_res"])
        tri[..., 0] /= np.float32(tw * m["texture_res"] - 1)
        tri[..., 1] /= np.float32(th * m["texture_res"] - 1)
        want_vt = ["vt %.8f %.8f" % (p[0], p[1]) for p in tri.reshape(-1, 2)]
        vt = [i for i, line in enumerate(ours) if line.startswith("vt ")]
        assert [ours[i] for i in vt] == want_vt
        moved = 0
        for j, i in enumerate(vt):
            if (j // 3) % tw == 0:
                assert ours[i] == ref[i]
            else:
                moved += ours[i] != ref[i]
        assert moved == (0 if nf == 1 else 3 * sum(1 for f in range(nf) if f % tw))
        assert [line for i, line in enumerate(ours) if i not in vt] == [line for i, line in enumerate(ref) if i not in vt]


def test_save_obj_vertex_colours_match_reference_python(tmp_path):
    """Vertex colours: the reference's file minus its `mtllib` line (which names a .mtl it never writes); no .mtl / .png."""
    g, meta = _golden()
    fn = str(tmp_path / meta["vertex"]["filename"])
    jr.save_obj(fn, torch.from_numpy(g["vertex_vertices"]), torch.from_numpy(g["vertex_faces"]),
                textures=torch.from_numpy(g["vertex_textures"]).requires_grad_(True), texture_type="vertex")
    assert open(fn).read() == _text(g["vertex_obj"]).replace("mtllib mesh.mtl\n\n", "")
    assert sorted(os.listdir(tmp_path)) == ["mesh.obj"]
    v, f, c = jr.load_obj(fn, load_texture=True, texture_type="vertex")
    assert np.abs(c.numpy() - g["vertex_textures"]).max() <= 1e-8 and np.array_equal(f.numpy(), g["vertex_faces"])


def test_save_obj_without_textures_is_unchanged(tmp_path):
    v = np.float32([[0, 0, 0], [1, 0, 0.5], [0, 1, -0.25]])
    f = np.int32([[0, 1, 2]])
    fn = str(tmp_path / "g.obj")
    jr.save_obj(fn, torch.from_numpy(v), torch.from_numpy(f))
    assert open(fn).read() == ("# g.obj\n\nv 0.00000000 0.00000000 0.00000000\nv 1.00000000 0.00000000 0.50000000\n"
                               "v 0.00000000 1.00000000 -0.25000000\n\nf 1 2 3\n")
    jr.Mesh(torch.from_numpy(v), torch.from_numpy(f)).save_obj(fn)
    assert sorted(os.listdir(tmp_path)) == ["g.obj"]


def test_mesh_save_obj_texture_types(oracle_kernel, tmp_path):
    """Mesh.save_obj(save_texture=True) (structures/mesh.py:330-338) hands textures[0], texture_res_out and the mesh's
    texture type to save_obj, for SoftRas and NMR surface textures and for vertex colours."""
    v = torch.rand(5, 3)
    f = torch.tensor([[0, 1, 2], [0, 2, 3], [1, 3, 4]], dtype=torch.int32)
    for kw, tex in ((dict(dr_type='softras'), torch.rand(1, 3, 9, 3)), (dict(dr_type='n3mr'), torch.rand(1, 3, 2, 2, 2, 3)),
                    (dict(texture_type='vertex'), torch.rand(1, 5, 3))):
        d = tmp_path / (kw.get("dr_type") or "vertex")
        d.mkdir()
        jr.Mesh(v, f, tex, **kw).save_obj(str(d / "m.obj"), save_texture=True, texture_res_out=4)
        files = sorted(os.listdir(d))
        if kw.get("texture_type") == "vertex":
            assert files == ["m.obj"] and open(d / "m.obj").read().count("\nv ") == 5
        else:
            assert files == ["m.mtl", "m.obj", "m.png"]
            import cv2
            assert cv2.imread(str(d / "m.png")).shape == (8, 8, 3)       # 3 faces: 2 x 2 tiles of 4 pixels
    with pytest.raises(ValueError):
        jr.Mesh(torch.rand(2, 5, 3), f[None].repeat(2, 1, 1)).save_obj(str(tmp_path / "b.obj"), save_texture=True)


def test_argument_errors(tmp_path):
    tex = np.ones((3, 4, 3), np.float32)
    for bad in (0, 1, 3):
        with pytest.raises(ValueError):
            jr.create_texture_image(tex, bad)
    with pytest.raises(AssertionError):
        jr.save_obj(str(tmp_path / "x.obj"), np.zeros((3, 3), np.float32), np.zeros((1, 3), np.int32), textures=tex, texture_type="uv")
    with pytest.raises(ValueError):
        jr.save_obj(str(tmp_path / "x.obj"), np.zeros((3, 3), np.float32), np.zeros((1, 3), np.int32), textures=np.ones((4, 3), np.float32),
                    texture_type="vertex")
    if not torch.cuda.is_available():   # GPU-only, like the bake: no CPU fallback
        with pytest.raises(jr.B200RasterError):
            jr.create_texture_image(tex, 4)


def test_abi_rejects_null_pointers():
    from jrender_b200 import build, _lib
    build.build()
    L = _lib.lib()
    null = C.c_void_p(0)
    for name in ("b200r_texture_atlas_softras", "b200r_texture_atlas_n3mr"):
        rc = getattr(L, name)(null, null, null, 1, 2, 4, 1, 4, 4, null)
        assert rc == -1 and b"NULL" in L.b200r_last_error()
