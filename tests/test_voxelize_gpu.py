"""GPU tests of mesh voxelization (csrc/voxel_api.cu <- jrender/renderer/utils/voxelization.py and its kernels).

The surface kernel and the fill are bit-equal to the numpy oracle (oracle/voxelize.py: the reference's all-columns loop
in unfused float32, and a BFS).  Against the reference's own kernels (tests/golden/ref_voxel_gpu_*.npz, built with a*b+c
contraction) a differing surface voxel must be one a marginal pair can set, as in tests/test_voxelize_cpu.py.
"""
import importlib
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib
from oracle import voxelize as ov
from tests.test_voxelize_cpu import ref_kernel_goldens

pytestmark = pytest.mark.gpu
# the module, not the function jrender_b200.voxelization that the package exports under the same name
jv = importlib.import_module("jrender_b200.voxelization")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _surface(faces, vs, dev):
    return jv.voxelize_surface(torch.from_numpy(np.ascontiguousarray(faces)).to(dev), vs).cpu().numpy()


def _fill(grid, dev):
    return jv.voxelize_fill(torch.from_numpy(np.ascontiguousarray(grid, np.int32)).to(dev)).cpu().numpy()


def hostile_faces(B, vs, seed):
    """det == 0 faces (collinear, repeated corners), slivers (one corner nudged off the line by an ulp or a tiny
    offset), faces partly and wholly outside the grid, and huge faces."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(B):
        fs = []
        for _ in range(24):
            a = rng.uniform(-0.2, 1.2, 3) * vs
            d = rng.normal(0, 1, 3) * vs * rng.uniform(0.05, 0.7)
            t = rng.uniform(0.1, 0.9)
            fs.append([a, a + d, a + t * d])                                          # collinear
            c = (a + t * d).astype(np.float32)
            fs.append([a, a + d, np.nextafter(c, np.float32(np.inf))])                # sliver, an ulp off the line
            fs.append([a, a + d, c + rng.normal(0, 1e-4, 3)])                         # sliver
            fs.append([a, a, a + d])                                                  # repeated corner
            fs.append([a + 3 * vs, a + d + 3 * vs, a + rng.normal(0, 1, 3) * 3 + 3 * vs])   # wholly outside
            fs.append(list(rng.uniform(-2, 3, (3, 3)) * vs))                          # huge, partly outside
        out.append(np.array(fs, np.float64).astype(np.float32))
    return np.stack(out)


def surface_cases(vs, B):
    yield "random", ov.random_faces(B, 120, vs, seed=vs + B)
    yield "small", ov.random_faces(B, 300, vs, seed=7 * vs + B, size=0.02)
    yield "hostile", hostile_faces(B, vs, seed=vs * 10 + B)
    if vs <= 64:
        sph = ov.sphere_faces(3280, radius=0.45, jitter=0.02)
        yield "sphere", np.repeat(ov.mesh_voxelize_faces(sph, vs) * np.float32(vs), B, axis=0)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("vs", [1, 2, 3, 16, 31, 32, 64, 128])
def test_surface_matches_oracle(cuda_device, vs, B):
    for name, faces in surface_cases(vs, B):
        want = ov.surface(faces, vs)
        got = _surface(faces, vs, cuda_device)
        assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_surface_spot_cow(cuda_device):
    fv = ov.spot_faces()
    for vs in (32, 64):
        faces = ov.mesh_voxelize_faces(fv, vs) * np.float32(vs)
        assert np.array_equal(_surface(faces, vs, cuda_device), ov.surface(faces, vs)), vs


@pytest.mark.parametrize("vs", [1, 2, 3, 5, 32, 33, 70])
def test_fill_random_grids(cuda_device, vs):
    rng = np.random.default_rng(vs)
    for p in (0.1, 0.3, 0.45, 0.6):
        g = (rng.random((3, vs, vs, vs)) < p).astype(np.int32)
        g[1] *= rng.integers(1, 5, g[1].shape).astype(np.int32)     # any nonzero value is solid
        assert np.array_equal(_fill(g, cuda_device), ov.fill(g)), p


def serpentine(vs):
    """A solid block with a winding tunnel: along z, then one step in x, back along z, ... across the x-y plane, open to
    the outside at one end only.  Reaching its far end takes thousands of propagation steps."""
    g = np.ones((vs, vs, vs), np.int32)
    rows = list(range(2, vs - 2, 2))
    cells = []
    for yi, y in enumerate(range(2, vs - 2, 4)):
        xs = rows if yi % 2 == 0 else rows[::-1]
        for j, x in enumerate(xs):
            z0, z1 = (2, vs - 3) if j % 2 == 0 else (vs - 3, 2)
            cells.append((y, x, z0, z1))
    prev = None
    for y, x, z0, z1 in cells:
        lo, hi = min(z0, z1), max(z0, z1)
        g[y, x, lo:hi + 1] = 0
        if prev is not None:
            py, px, pz = prev
            g[min(py, y):max(py, y) + 1, min(px, x):max(px, x) + 1, pz] = 0
        prev = (y, x, z1)
    g[2, 2, 0:3] = 0                                           # the one opening, at z = 0
    return g


def test_fill_serpentine(cuda_device):
    g = serpentine(64)[None]
    want = ov.fill(g)
    assert (want == 0).sum() > (g == 0).sum() * 0.99           # the tunnel is reachable from its opening
    assert np.array_equal(_fill(g, cuda_device), want)
    g[0, 2, 2, 0] = 1                                          # closed: the whole tunnel is inside
    assert np.array_equal(_fill(g, cuda_device), np.ones_like(g))


def test_fill_of_reference_surfaces(cuda_device):
    for name, faces, vs, surf, final in ref_kernel_goldens():
        assert np.array_equal(_fill(surf, cuda_device), final), name


def test_end_to_end_matches_goldens(cuda_device):
    for name, faces, vs, surf, final in ref_kernel_goldens():
        got = jr.voxelization(torch.from_numpy(faces).to(cuda_device), vs, normalize=True).cpu().numpy()
        assert np.array_equal(got, ov.fill(ov.surface(faces, vs))), name
        _, maybe = ov.surface(faces, vs, marginal=True)
        differ = _surface(faces, vs, cuda_device) != surf
        assert not (differ & (maybe == 0)).any(), (name, int(differ.sum()))


def test_mesh_voxelize_matches_oracle_chain(cuda_device):
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_host_voxelize.npz"))
    fv = g["mesh_voxelize_face_vertices"]
    mesh_faces = np.arange(fv.shape[1] * 3, dtype=np.int32).reshape(1, -1, 3)
    mesh = jr.Mesh(torch.from_numpy(fv.reshape(1, -1, 3)).to(cuda_device), torch.from_numpy(mesh_faces).to(cuda_device))
    got = mesh.voxelize(16).cpu().numpy()
    assert np.array_equal(got, g["mesh_voxelize_voxels"])
    spot = ov.spot_faces()
    mesh = jr.Mesh(torch.from_numpy(spot.reshape(1, -1, 3)).to(cuda_device),
                   torch.from_numpy(np.arange(spot.shape[1] * 3, dtype=np.int32).reshape(1, -1, 3)).to(cuda_device))
    got = mesh.voxelize(32).cpu().numpy()
    assert np.array_equal(got, ov.voxelization(ov.mesh_voxelize_faces(spot, 32), 32))


def test_no_host_sync_graph_capture_and_determinism(cuda_device):
    faces = torch.from_numpy(ov.mesh_voxelize_faces(ov.sphere_faces(3280, radius=0.45, jitter=0.02), 48)).to(cuda_device)
    faces = faces.repeat(2, 1, 1, 1)
    want = ov.voxelization(faces.cpu().numpy(), 48)
    jr.voxelization(faces, 48)                                 # warm up (library load, allocator)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = jr.voxelization(faces, 48)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    again = jr.voxelization(faces, 48)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        jr.voxelization(faces, 48)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = jr.voxelization(faces, 48)
    captured.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(eager.cpu().numpy(), want)
    assert torch.equal(eager, again)
    assert torch.equal(captured, eager)


def test_no_writes_outside_the_grid(cuda_device):
    vs, B = 16, 2
    faces = torch.from_numpy(hostile_faces(B, vs, seed=3)).to(cuda_device)
    faces[0, :5] = float("nan")
    faces[1, :5, 1] = float("inf")
    n = B * vs ** 3
    big = torch.full((n + 2 * 4096,), -7, dtype=torch.int32, device=cuda_device)
    view = big[4096:4096 + n].view(B, vs, vs, vs)
    _lib.call("b200r_voxelize_surface", cuda_device, faces, view, B, faces.shape[1], vs)
    jv.voxelize_fill(view)
    torch.cuda.synchronize()
    assert (big[:4096] == -7).all() and (big[4096 + n:] == -7).all()
    assert ((view == 0) | (view == 1)).all()
