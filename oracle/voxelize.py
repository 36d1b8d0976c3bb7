"""numpy float32 restatement of mesh voxelization (TEST INFRASTRUCTURE): jrender/renderer/utils/voxelization.py:1-57
and the four kernels of jrender/renderer/utils/cuda/voxelization.py.

surface() runs the reference's all-columns loop (every integer column (y, x), 0 <= y, x < vs, of every axis against
every face), chunked and vectorised; numpy's float32 operations are unfused IEEE ones, like the product kernel built
with -fmad=false, so csrc/voxel_api.cu must match it bit for bit.  With marginal=True it also returns the voxels a
*marginal* (face, column) pair can set: pairs whose accept decision flips in float64 or lies within a few ulps of a
threshold, and depths within a few ulps of an integer.  A build that contracts a*b+c (the reference's, nvcc default) may
differ from this oracle on those voxels only.  fill() is a plain breadth-first search.
"""
import numpy as np

PERMS = ((2, 1, 0), (0, 2, 1), (0, 1, 2))   # voxelization.py:8-11: axis -> the (y, x, z) coordinates of the faces
EPS32 = 2.0 ** -24
_CHUNK = 1 << 22                            # (face, column) pairs per vectorised step


def _set4(grid, y, x, z, vs, perm):
    """The four writes of voxelize_sub1_kernel (:66-85) for columns (y, x) at depth z, into grid [vs, vs, vs] indexed in
    the input's coordinate order."""
    for dy, dx in ((0, 0), (1, 0), (0, 1), (1, 1)):
        yi, xi = y - dy, x - dx
        ok = (yi >= 0) & (xi >= 0)
        c = [None] * 3
        c[perm[0]], c[perm[1]], c[perm[2]] = yi[ok], xi[ok], z[ok]
        grid[c[0], c[1], c[2]] = 1


def _axis(faces, vs, perm, grid, maybe):
    f = faces[:, :, list(perm)].astype(np.float32)                 # [nf, 3 corners, (y, x, z)]
    f0, f1, f2 = f[:, 0, 0], f[:, 0, 1], f[:, 0, 2]
    y1d, x1d, z1d = f[:, 1, 0] - f0, f[:, 1, 1] - f1, f[:, 1, 2] - f2
    y2d, x2d, z2d = f[:, 2, 0] - f0, f[:, 2, 1] - f1, f[:, 2, 2] - f2
    det = x1d * y2d - x2d * y1d
    live = np.nonzero(det != 0)[0]
    cy, cx = np.meshgrid(np.arange(vs), np.arange(vs), indexing="ij")
    cy, cx = cy.ravel(), cx.ravel()
    fy, fx = cy.astype(np.float32), cx.astype(np.float32)
    step = max(1, _CHUNK // (vs * vs))
    vsf = np.float32(vs)
    for s in range(0, len(live), step):
        fi = live[s:s + step][:, None]
        ypd = fy[None] - f0[fi]
        xpd = fx[None] - f1[fi]
        t1 = (y2d[fi] * xpd - x2d[fi] * ypd) / det[fi]
        t2 = (-y1d[fi] * xpd + x1d[fi] * ypd) / det[fi]
        zf = np.floor(t1 * z1d[fi] + t2 * z2d[fi] + f2[fi])
        acc = ~(t1 < 0) & ~(t2 < 0) & ~(np.float32(1) < t1 + t2)
        hit = acc & (zf >= 0) & (zf < vsf)
        k, c = np.nonzero(hit)
        _set4(grid, cy[c], cx[c], zf[k, c].astype(np.int64), vs, perm)
        if maybe is None:
            continue
        # float64 view of the same pair: the decision and depth a differently rounded build could reach
        d = lambda a: a.astype(np.float64)                          # noqa: E731
        ypd64, xpd64 = d(fy)[None] - d(f0[fi]), d(fx)[None] - d(f1[fi])
        det64 = d(x1d[fi]) * d(y2d[fi]) - d(x2d[fi]) * d(y1d[fi])
        n1 = d(y2d[fi]) * xpd64 - d(x2d[fi]) * ypd64
        n2 = -d(y1d[fi]) * xpd64 + d(x1d[fi]) * ypd64
        T1, T2 = n1 / det64, n2 / det64
        scale = (np.abs(d(y2d[fi]) * xpd64) + np.abs(d(x2d[fi]) * ypd64) + np.abs(d(y1d[fi]) * xpd64) + np.abs(d(x1d[fi]) * ypd64)
                 + np.abs(d(x1d[fi]) * d(y2d[fi])) + np.abs(d(x2d[fi]) * d(y1d[fi]))) / np.abs(det64)
        tol = 16 * EPS32 * (scale + 1)
        acc64 = (T1 >= 0) & (T2 >= 0) & (T1 + T2 <= 1)
        near = (np.abs(T1) <= tol) | (np.abs(T2) <= tol) | (np.abs(1 - T1 - T2) <= tol)
        Z = T1 * d(z1d[fi]) + T2 * d(z2d[fi]) + d(f2[fi])
        ztol = 16 * EPS32 * (np.abs(T1 * d(z1d[fi])) + np.abs(T2 * d(z2d[fi])) + np.abs(d(f2[fi])) + 1) \
            + tol * (np.abs(d(z1d[fi])) + np.abs(d(z2d[fi])))
        marginal = (acc != acc64) | (near & (acc | acc64))
        zmarg = (acc | acc64) & (np.floor(Z - ztol) != np.floor(Z + ztol))
        for sel in (marginal, zmarg):
            for zz in (zf, np.floor(Z), np.floor(Z - ztol), np.floor(Z + ztol)):
                m = sel & (zz >= 0) & (zz < vs)
                k, c = np.nonzero(m)
                _set4(maybe, cy[c], cx[c], zz[k, c].astype(np.int64), vs, perm)


def surface(faces, vs, marginal=False):
    """voxelize_sub1 on the three axes + voxelize_sub2, OR'ed (voxelization.py:48-53).  faces [B, nf, 3, 3] float32 in
    voxel units -> int32 [B, vs, vs, vs].  marginal=True: also an int32 grid of the voxels marginal pairs can set."""
    faces = np.asarray(faces, np.float32)
    B = faces.shape[0]
    out = np.zeros((B, vs, vs, vs), np.int32)
    maybe = np.zeros_like(out) if marginal else None
    with np.errstate(all="ignore"):
        for b in range(B):
            for perm in PERMS:
                _axis(faces[b], vs, perm, out[b], None if maybe is None else maybe[b])
            c = faces[b].reshape(-1, 3)                             # voxelize_sub2_kernel, :150-160
            ok = np.all((c >= 0) & (c < np.float32(vs)), axis=1)
            ci = np.floor(c[ok]).astype(np.int64)
            out[b, ci[:, 0], ci[:, 1], ci[:, 2]] = 1
    return (out, maybe) if marginal else out


def fill(voxels):
    """voxelize_sub3 / sub4 and the host loop (voxelization.py:24-38): 1 - visible, visible = empty (== 0) voxels
    6-connected through empty voxels to an empty voxel on the grid boundary.  Breadth-first search from the empty
    boundary voxels, one frontier per step."""
    voxels = np.asarray(voxels)
    out = np.empty(voxels.shape, np.int32)
    for b in range(voxels.shape[0]):
        empty = voxels[b] == 0
        n = empty.shape[0]
        visible = np.zeros_like(empty)
        edge = np.zeros_like(empty)
        edge[[0, -1], :, :] = edge[:, [0, -1], :] = edge[:, :, [0, -1]] = True
        frontier = np.argwhere(empty & edge)
        visible[tuple(frontier.T)] = True
        while len(frontier):
            nxt = []
            for ax in range(3):
                for dlt in (-1, 1):
                    q = frontier.copy()
                    q[:, ax] += dlt
                    q = q[(q[:, ax] >= 0) & (q[:, ax] < n)]
                    q = q[empty[tuple(q.T)] & ~visible[tuple(q.T)]]
                    visible[tuple(q.T)] = True
                    nxt.append(q)
            frontier = np.concatenate(nxt)
        out[b] = 1 - visible
    return out


def voxelization(faces, size, normalize=False):
    """voxelization.py:41-57 on numpy float32 faces [B, nf, 3, 3]."""
    faces = np.array(faces, np.float32)
    if not normalize:
        faces *= np.float32(size)
    return fill(surface(faces, size))


def mesh_voxelize_faces(face_vertices, voxel_size):
    """structures/mesh.py:341: face_vertices * vs / (vs - 1) + 0.5, float32, left to right."""
    fv = np.asarray(face_vertices, np.float32)
    return fv * np.float32(voxel_size) / np.float32(voxel_size - 1) + np.float32(0.5)


# ---- test inputs (shared by the golden generators, the tests and tools/bench_voxel.py)

def random_faces(batch, num_faces, vs, seed=0, lo=-0.1, hi=1.1, size=0.3):
    """Seeded triangles in voxel units: centres uniform in [lo, hi] * vs (some poke out of the grid), corners within
    size * vs of the centre."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(lo, hi, (batch, num_faces, 1, 3)) * vs
    return (c + rng.uniform(-size, size, (batch, num_faces, 3, 3)) * vs).astype(np.float32)


def sphere_faces(num_faces=39200, radius=0.45, jitter=0.0):
    """The workloads' UV sphere (jrender_b200.workloads.sphere_by_faces) as face vertices [1, nf, 3, 3], centred at 0."""
    from jrender_b200 import workloads as wl
    v, f = wl.sphere_by_faces(num_faces, radius=radius, jitter=jitter)
    return np.asarray(v, np.float32)[np.asarray(f)][None]


def spot_faces():
    """The spot cow (tests/golden/spot_triangulated.obj.xz), normalised by load_obj and scaled by 0.45 so that
    Mesh.voxelize's v * vs / (vs - 1) + 0.5 maps it into the unit cube: face vertices [1, nf, 3, 3]."""
    import lzma
    import os
    import tempfile
    from jrender_b200.io import load_obj
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "spot_triangulated.obj.xz")
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "spot.obj")
        with lzma.open(src, "rb") as fh, open(p, "wb") as out:
            out.write(fh.read())
        v, f = load_obj(p, normalization=True)
    v = v.numpy().astype(np.float32) * np.float32(0.45)
    return v[f.numpy().astype(np.int64)][None]


def golden_cases():
    """(name, faces in voxel units [B, nf, 3, 3], vs) of tests/golden/ref_voxel_gpu_*.npz."""
    yield "random_b2_vs16", random_faces(2, 60, 16, seed=1), 16
    yield "random_vs32", random_faces(1, 200, 32, seed=2, size=0.15), 32
    sph = sphere_faces(3280, radius=0.45, jitter=0.01)
    yield "sphere_vs64", mesh_voxelize_faces(sph, 64) * np.float32(64), 64
    yield "spot_vs32", mesh_voxelize_faces(spot_faces(), 32) * np.float32(32), 32
