"""CPU tests of mesh voxelization: the numpy oracle (oracle/voxelize.py) on hand-checkable cases, against the reference's
own host code (tests/golden/ref_host_voxelize.npz) and kernels (tests/golden/ref_voxel_gpu_*.npz), plus save_voxel's file
format and the argument checks of the C ABI.

The reference kernels were built with nvcc's default a*b+c contraction, the oracle is unfused: a surface voxel on which
they differ must be one a marginal (face, column) pair of the oracle can set.  The fill has no arithmetic, so
fill(reference surface) must equal the reference's final grid exactly.
"""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib
from oracle import voxelize as ov

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")

CUBE_V = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
CUBE_F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                   [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]])


def test_single_triangle():
    # the triangle z = 1.5 with corners (y, x) = (0.5, 0.5), (3.5, 0.5), (0.5, 3.5): along axis 2 the integer columns
    # with y, x >= 1 and y + x <= 4 are inside, each setting the four voxels (y-1..y, x-1..x, 1)
    faces = np.array([[[[0.5, 0.5, 1.5], [3.5, 0.5, 1.5], [0.5, 3.5, 1.5]]]], np.float32)
    s = ov.surface(faces, 4)[0]
    want = np.zeros((4, 4, 4), np.int32)
    for y, x in ((1, 1), (1, 2), (1, 3), (2, 1), (2, 2), (3, 1)):
        want[y - 1:y + 1, x - 1:x + 1, 1] = 1
    want[0, 0, 1] = want[3, 0, 1] = want[0, 3, 1] = 1       # the corner voxels (voxelize_sub2)
    assert np.array_equal(s, want)                          # axes 0 and 1 see the triangle edge-on: det == 0


def test_closed_cube_is_solid():
    fv = (CUBE_V[CUBE_F] * np.float32(2.2) + np.float32(0.9))[None]
    assert ov.surface(fv, 4).sum() < 64
    assert ov.voxelization(fv, 4, normalize=True).sum() == 64


def test_open_cube_is_hollow():
    fv = (CUBE_V[CUBE_F] * np.float32(5) + np.float32(1.5))[None]
    closed = ov.voxelization(fv, 8, normalize=True)
    assert closed.sum() == 6 ** 3
    opened = ov.voxelization(fv[:, 2:], 8, normalize=True)       # the x = 0 side removed
    assert np.array_equal(opened, ov.surface(fv[:, 2:], 8))
    assert opened.sum() < closed.sum()


def test_fill_bfs_matches_labelling():
    from scipy import ndimage
    rng = np.random.default_rng(5)
    for vs, p in ((1, 0.3), (2, 0.5), (9, 0.4), (17, 0.25)):
        g = (rng.random((2, vs, vs, vs)) < p).astype(np.int32)
        for b in range(2):
            lab, _ = ndimage.label(g[b] == 0)
            edge = np.zeros(g[b].shape, bool)
            edge[[0, -1], :, :] = edge[:, [0, -1], :] = edge[:, :, [0, -1]] = True
            outside = np.isin(lab, np.unique(lab[edge & (lab > 0)]))
            assert np.array_equal(ov.fill(g[b:b + 1])[0], 1 - outside)


def test_oracle_matches_reference_host_code():
    g = np.load(os.path.join(G, "ref_host_voxelize.npz"))
    meta = json.loads(bytes(g["meta_json"]).decode())
    assert len(meta) >= 3
    for name, m in meta.items():
        if name + "_faces" in g:
            got = ov.voxelization(g[name + "_faces"], m["size"], m["normalize"])
        else:
            got = ov.voxelization(ov.mesh_voxelize_faces(g[name + "_face_vertices"], m["size"]), m["size"])
        assert np.array_equal(got, g[name + "_voxels"]), name


def ref_kernel_goldens():
    files = sorted(glob.glob(os.path.join(G, "ref_voxel_gpu_*.npz")))
    assert len(files) >= 4, "golden fixtures missing"
    for p in files:
        g = np.load(p)
        vs = int(g["voxel_size"])
        final = np.unpackbits(g["final_packed"])[:g["surface"].size].reshape(g["surface"].shape).astype(np.int32)
        yield os.path.basename(p), g["faces"], vs, g["surface"], final


def test_oracle_matches_reference_kernels():
    for name, faces, vs, surf, final in ref_kernel_goldens():
        got, maybe = ov.surface(faces, vs, marginal=True)
        differ = got != surf
        assert not (differ & (maybe == 0)).any(), (name, int(differ.sum()), int((differ & (maybe == 0)).sum()))
        assert np.array_equal(ov.fill(surf), final), name


def test_save_voxel_format(tmp_path):
    v = np.zeros((3, 4, 5), np.int32)
    v[1, 2, 3] = v[0, 0, 4] = 1
    v[2, 3, 0] = 2                                       # only voxels equal to 1 are written (save_obj.py:91)
    p = tmp_path / "vox.obj"
    jr.save_voxel(str(p), torch.from_numpy(v))
    assert p.read_text() == "# vox.obj\n#\n\nv 0.00000000 0.00000000 0.80000001\nv 0.33333334 0.50000000 0.60000002\n\n"
    jr.save_voxel(str(p), np.zeros((2, 2, 2), np.int32))
    assert p.read_text() == "# vox.obj\n#\n\n\n"
    with pytest.raises(ValueError):
        jr.save_voxel(str(p), np.zeros((2, 2), np.int32))


def test_cpu_tensors_rejected():
    with pytest.raises(jr.B200RasterError):
        jr.voxelization(torch.zeros((1, 2, 3, 3)), 8)
    with pytest.raises(jr.B200RasterError):
        jr.Mesh(CUBE_V, CUBE_F).voxelize(8)


def test_abi_argument_errors():
    L = _lib.lib()
    p = C.c_void_p(16)
    assert L.b200r_voxelize_surface(None, p, 1, 1, 8, None) == -1
    assert L.b200r_voxelize_surface(p, None, 1, 1, 8, None) == -1
    assert L.b200r_voxelize_surface(p, p, 0, 1, 8, None) == -1
    assert L.b200r_voxelize_surface(p, p, 1, 0, 8, None) == -1
    assert L.b200r_voxelize_surface(p, p, 1, 1, 0, None) == -1
    assert L.b200r_voxelize_surface(p, p, 1, 1, 1025, None) == -1
    ws = L.b200r_voxelize_workspace_bytes(2, 40)
    assert ws == 2 * 2 * 40 * 40 * 2 * 4
    assert L.b200r_voxelize_workspace_bytes(0, 8) == 0 and L.b200r_voxelize_workspace_bytes(1, 1025) == 0
    assert L.b200r_voxelize_fill(None, p, ws, 2, 40, None) == -1
    assert L.b200r_voxelize_fill(p, None, ws, 2, 40, None) == -1
    assert L.b200r_voxelize_fill(p, p, ws, 0, 40, None) == -1
    assert L.b200r_voxelize_fill(p, p, ws, 2, 2000, None) == -1
    assert L.b200r_voxelize_fill(p, p, ws - 1, 2, 40, None) == -2
    assert b"workspace" in L.b200r_last_error()
