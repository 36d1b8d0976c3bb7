"""GPU tests of the texture-atlas export (csrc/texture_atlas_api.cu <- jrender/io/utils/create_texture_image.py; NMR
volumes through the NMR sampler's trilinear fetch) and of the textured OBJ files it feeds.

Tolerances: both atlases are bit-equal to the numpy oracle (oracle/texture_atlas.py: same float32 operations in the
same order, no contraction on either side), and the oracle chains (atlas -> 8-bit PNG -> bake, oracle/bake.py) are
bit-equal to the product's save / load round trips.  Against
the reference's own kernel (tests/golden/ref_atlas_gpu_*.npz) at most 1e-3 of the pixels may pick another texel: that
build contracts a*b+c, which moves pixels on a cell boundary.  Round trips save_obj -> load_obj compare with the 8-bit
PNG's value floor(255 clip(c)) / 255 to 1e-6.
"""
import glob
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import io as jio
from oracle import bake as obake
from oracle import texture_atlas as oat

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def spot(tmp_path_factory):
    """The spot cow (tests/golden/spot_triangulated.obj.xz + spot_texture.png) unpacked as .obj / .mtl / .png."""
    import lzma
    import shutil
    d = tmp_path_factory.mktemp("spot")
    with lzma.open(os.path.join(G, "spot_triangulated.obj.xz"), "rb") as f:
        (d / "spot_triangulated.obj").write_bytes(f.read())
    (d / "spot_triangulated.mtl").write_text("newmtl material_1\nmap_Kd spot_texture.png\n")
    shutil.copyfile(os.path.join(G, "spot_texture.png"), d / "spot_texture.png")
    return str(d / "spot_triangulated.obj")


def _atlas(tri, tex, R_out, tw, H, W, dev):
    return jio.texture_atlas(tri, tex, R_out, tw, H, W, device=dev).cpu().numpy()


@pytest.mark.parametrize("nf,R_out", [(1, 2), (7, 4), (40, 16), (130, 5)])
def test_kernels_match_oracle(cuda_device, nf, R_out):
    rng = np.random.default_rng(nf + R_out)
    tri, tw, th = oat.atlas_layout(nf, R_out)
    jit = (tri + rng.uniform(-0.3, 0.3, tri.shape)).astype(np.float32)   # off-grid vertices exercise the arithmetic
    H, W = th * R_out, tw * R_out
    for t in (tri, jit):
        for R in (1, 2, 4, 5):
            tex = rng.random((nf, R * R, 3), dtype=np.float32)
            got = _atlas(t, tex, R_out, tw, H, W, cuda_device)
            assert np.array_equal(got, oat.texture_atlas_softras(t, tex, R_out, tw, H, W)), (R, "softras")
        for ts in (2, 3, 4):
            tex = rng.random((nf, ts, ts, ts, 3), dtype=np.float32)
            got = _atlas(t, tex, R_out, tw, H, W, cuda_device)
            assert np.array_equal(got, oat.texture_atlas_n3mr(t, tex, R_out, tw, H, W)), (ts, "n3mr")


def test_kernel_matches_reference_kernel_golden(cuda_device):
    files = sorted(glob.glob(os.path.join(G, "ref_atlas_gpu_*.npz")))
    assert len(files) >= 4, "golden fixtures missing"
    for p in files:
        g = np.load(p)
        ref = g["image"]
        got = _atlas(g["tile_vertices"], g["textures"], int(g["texture_res_out"]), int(g["tile_width"]), ref.shape[0], ref.shape[1],
                     cuda_device)
        differ = (got != ref).any(axis=-1)
        assert differ.mean() <= 1e-3, (p, int(differ.sum()))


def test_abi_rejects_bad_sizes(cuda_device):
    """Argument errors come back as B200R_EINVAL with a message; the buffers are real and sized for the call, so even a
    call that got through would stay inside them."""
    from jrender_b200 import _lib
    import ctypes as C
    L = _lib.lib()
    tri = torch.zeros(2, 3, 2, device=cuda_device)
    tex = torch.zeros(2, 4 * 4 * 4 * 3, device=cuda_device)
    img = torch.zeros(8, 8, 3, device=cuda_device)
    P = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    s = C.c_void_p(torch.cuda.current_stream(cuda_device).cuda_stream)
    cases = [("b200r_texture_atlas_softras", (0, 2, 4, 2, 8, 8), b"nf"),
             ("b200r_texture_atlas_softras", (2, 0, 4, 2, 8, 8), b"texture_res"),
             ("b200r_texture_atlas_softras", (2, 2, 3, 2, 6, 6), b"texture_res_out"),
             ("b200r_texture_atlas_softras", (2, 2, 1, 2, 2, 2), b"texture_res_out"),
             ("b200r_texture_atlas_softras", (2, 2, 4, 2, 8, 6), b"tiles"),
             ("b200r_texture_atlas_n3mr", (2, 1, 4, 2, 8, 8), b"texture_size"),
             ("b200r_texture_atlas_n3mr", (2, 4, 3, 2, 6, 6), b"texture_res_out")]
    for name, args, msg in cases:
        rc = getattr(L, name)(P(tri), P(tex), P(img), *args, s)
        assert rc == -1 and msg in L.b200r_last_error(), (name, args, L.b200r_last_error())
    with pytest.raises(ValueError):
        jio.texture_atlas(np.zeros((3, 3, 2), np.float32), np.zeros((2, 4, 3), np.float32), 4, 2, 4, 8, device=cuda_device)
    with pytest.raises(ValueError):
        jio.texture_atlas(np.zeros((2, 3, 2), np.float32), np.zeros((2, 5, 3), np.float32), 4, 2, 4, 8, device=cuda_device)


def _png_value(c):
    return np.floor(np.clip(c, 0, 1).astype(np.float32) * np.float32(255)).astype(np.float32) / np.float32(255)


@pytest.mark.parametrize("R_out", [4, 16])
@pytest.mark.parametrize("kind,res", [("softras", 1), ("softras", 4), ("softras", 5), ("n3mr", 2), ("n3mr", 4)])
def test_save_load_round_trip(cuda_device, tmp_path, kind, res, R_out):
    """save_obj -> load_obj(load_texture=True) with one colour per face: every reloaded texel is the PNG's 8-bit value of
    that colour.  The tile triangle sits at least one pixel inside its tile, so for R_out >= 4 every bilinear tap of the
    bake lands in the face's own tile.  The one exception is the NMR texel (0, 0, 0): its barycentric point is 0 / 0, so
    the bake (load_textures.py:141-146) samples UV (0, 0) for it, a pixel of face 0's tile."""
    from jrender_b200 import workloads as wl
    v, f = wl.sphere_by_faces(280)
    nf = f.shape[0]
    col = np.random.default_rng(res * 100 + R_out).uniform(-0.2, 1.2, (nf, 3)).astype(np.float32)
    shape = (nf, res * res, 3) if kind == "softras" else (nf, res, res, res, 3)
    tex = torch.from_numpy(np.broadcast_to(col.reshape((nf,) + (1,) * (len(shape) - 2) + (3,)), shape).copy())
    fn = str(tmp_path / "m.obj")
    jr.save_obj(fn, torch.from_numpy(v), torch.from_numpy(f), textures=tex.to(cuda_device).requires_grad_(True), texture_res=R_out)
    v2, f2, t2 = jr.load_obj(fn, load_texture=True, dr_type=kind, texture_res=res)
    assert np.abs(v2.numpy() - v).max() <= 1e-7 and np.array_equal(f2.numpy(), f)
    assert tuple(t2.shape) == shape
    want = np.broadcast_to(_png_value(col).reshape((nf,) + (1,) * (len(shape) - 2) + (3,)), shape).copy()
    got = t2.numpy()
    if kind == "n3mr":
        assert np.abs(got[:, 0, 0, 0] - _png_value(col[0])).max() <= 1e-6
        got, want = got.reshape(nf, -1, 3)[:, 1:], want.reshape(nf, -1, 3)[:, 1:]
    assert np.abs(got - want).max() <= 1e-6


def _oracle_chain(textures, obj, R_out, kind):
    """oracle atlas -> clip, 8 bits -> vertical flip -> the loader's reading (/ 255, flip back) -> oracle bake, through the
    UVs as written to the .obj."""
    nf = textures.shape[0]
    tri, tw, th = oat.atlas_layout(nf, R_out)
    atlas = (oat.texture_atlas_softras if kind == "softras" else oat.texture_atlas_n3mr)(tri, textures, R_out, tw, th * R_out, tw * R_out)
    png = (atlas[::-1].clip(0, 1) * 255).astype(np.uint8)
    image = np.ascontiguousarray(png.astype(np.float32) / 255.)[::-1]
    faces_uv, _ = jio._parse_texture_faces(obj)
    if kind == "softras":
        return obake.bake_textures_for_softras(np.ascontiguousarray(image), faces_uv, np.ones_like(textures), np.ones(nf, np.int32))
    return obake.bake_textures_for_n3mr(np.ascontiguousarray(image), faces_uv, np.full_like(textures, 0.5), np.ones(nf, np.int32), 0, True)


def test_spot_cow_round_trip(cuda_device, spot, tmp_path):
    """The textured cow: load (texture_res 4), Mesh.save_obj(save_texture=True), load again.  The reloaded texels equal
    the oracle's chain bit for bit; how far they moved from the loaded ones is printed (not asserted: the atlas holds one
    sample per pixel of a 16-pixel tile and 8 bits per channel)."""
    mesh = jr.Mesh.from_obj(spot, load_texture=True, texture_res=4).to(cuda_device)
    out = str(tmp_path / "cow.obj")
    mesh.save_obj(out, save_texture=True)
    assert sorted(os.listdir(tmp_path)) == ["cow.mtl", "cow.obj", "cow.png"]
    back = jr.Mesh.from_obj(out, load_texture=True, texture_res=4)
    orig = mesh.textures[0].cpu().numpy()
    got = back.textures[0].numpy()
    assert np.abs(back.vertices.numpy() - mesh.vertices.cpu().numpy()).max() <= 1e-7
    assert np.array_equal(got, _oracle_chain(orig, out, 16, "softras"))
    d = np.abs(got - orig)
    print("\nspot cow round trip (texture_res 4, texture_res_out 16): |reloaded - original| mean %.5f max %.5f" % (d.mean(), d.max()))


def test_mesh_save_obj_nmr_and_vertex_colours(cuda_device, spot, tmp_path):
    """Mesh.save_obj(save_texture=True) on an NMR mesh (ts 4 volumes through the trilinear atlas) and on a vertex-coloured
    mesh."""
    mesh = jr.Mesh.from_obj(spot, load_texture=True, texture_res=4, dr_type='n3mr').to(cuda_device)
    out = str(tmp_path / "n3mr" / "cow.obj")
    os.makedirs(os.path.dirname(out))
    mesh.save_obj(out, save_texture=True, texture_res_out=8)
    back = jr.Mesh.from_obj(out, load_texture=True, texture_res=4, dr_type='n3mr')
    assert tuple(back.textures.shape) == (1, 5856, 4, 4, 4, 3)
    assert np.array_equal(back.textures[0].numpy(), _oracle_chain(mesh.textures[0].cpu().numpy(), out, 8, "n3mr"))
    from jrender_b200 import workloads as wl
    v, f = wl.sphere_by_faces(280)
    col = torch.rand(1, v.shape[0], 3, device=cuda_device)
    vm = jr.Mesh(torch.from_numpy(v).to(cuda_device), torch.from_numpy(f).to(cuda_device), col, texture_type='vertex')
    out = str(tmp_path / "vertex" / "s.obj")
    os.makedirs(os.path.dirname(out))
    vm.save_obj(out, save_texture=True)
    assert os.listdir(os.path.dirname(out)) == ["s.obj"]
    back = jr.Mesh.from_obj(out, load_texture=True, texture_type='vertex')
    assert np.abs(back.textures[0].numpy() - col[0].cpu().numpy()).max() <= 1e-8


def test_demo4_save(cuda_device, spot, tmp_path):
    """examples/demo4_optim_textures.py --save: a few iterations, then the fitted cow (tanh of the texture parameter) as
    .obj / .mtl / .png, which Mesh.from_obj(load_texture=True, dr_type='n3mr') reads back as the oracle chain predicts."""
    from examples import demo4_optim_textures as d4
    out = str(tmp_path / "out" / "cow.obj")
    model, losses = d4.run(spot, None, iters=3, device=str(cuda_device))
    d4.save(model, out)
    assert sorted(os.listdir(os.path.dirname(out))) == ["cow.mtl", "cow.obj", "cow.png"]
    back = jr.Mesh.from_obj(out, load_texture=True, texture_res=4, dr_type='n3mr')
    assert tuple(back.textures.shape) == (1, 5856, 4, 4, 4, 3)
    fitted = torch.tanh(model.textures)[0].detach().cpu().numpy()
    assert np.array_equal(back.textures[0].numpy(), _oracle_chain(fitted, out, 16, "n3mr"))
    assert np.abs(back.vertices.numpy() - model.vertices[0].cpu().numpy()).max() <= 1e-7
