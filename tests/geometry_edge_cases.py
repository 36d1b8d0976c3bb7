"""Degenerate cameras and meshes for the pre-raster projection and the mesh regularisers (shared by
test_geometry_edges_cpu.py and test_geometry_edges_gpu.py).  Each generator asserts that it built what it claims.

projection_cases() -> list of dict(name, vertices [Bv, nv, 3] f32, faces [Bf, nf, 3] i32, eye [Be, 3] f32,
                                   grad [B, nf, 3, 3] f32, kw = project_faces keyword arguments)
flatten_cases()    -> list of dict(name, vertices [B, nv, 3] f32, edges (v0s, v1s, v2s, v3s), eps, faces or None)
laplacian_cases()  -> list of dict(name, vertices [B, nv, 3] f32, faces [nf, 3])
"""
import os

import numpy as np

from jrender_b200 import workloads as wl
from oracle import preraster as opr

F = np.float32
INT32_MAX = 2 ** 31 - 1


def check_sums(what, got, s):
    """A kernel output `got` (float32) against the term_sums `s` of its emulated terms, shaped like got: every finite
    entry within the summation-order bound, NaN / +-inf exactly where the emulation has them.  Prints the worst ratio."""
    got = np.asarray(got, np.float64)
    ex = s["exact"]
    for pattern in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(pattern(got), pattern(ex)), what
    fin = np.isfinite(ex)
    with np.errstate(invalid="ignore"):
        err, bound = np.abs(got - ex)[fin], s["bound"][fin]
    worst = float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0
    print("%-40s worst |got - exact| / bound = %.3g" % (what, worst))
    assert np.all(err <= bound), (what, worst)


def check_bits(what, got, ref):
    """Bit for bit, NaN where ref is NaN (payloads may differ)."""
    assert got.shape == ref.shape
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), what
    assert np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32)), what


def _grad(rng, B, nf, zero_frac=0.25):
    """Upstream gradient with a quarter of the corners all-zero (the backward skips those)."""
    g = rng.normal(0, 1, (B, nf, 3, 3)).astype(F)
    g[rng.random((B, nf, 3)) < zero_frac] = 0
    return g


def _axes(c):
    e = np.broadcast_to(c["eye"], (max(c["eye"].shape[0], c["grad"].shape[0]), 3))
    kw = {k: c["kw"][k] for k in ("camera_mode", "at", "direction", "up", "coordinate") if k in c["kw"]}
    return opr.camera_axes(e, **kw)


def _fan(n, rng, hub=0):
    """n triangles around vertex `hub` = 0: [0, k, k+1], rim vertices on a jittered circle."""
    t = np.linspace(0, 2 * np.pi, n + 1)[:-1]
    rim = np.stack([np.cos(t), np.sin(t), 0.05 * rng.normal(size=n)], 1)
    v = np.concatenate([np.zeros((1, 3)), rim], 0).astype(F)
    k = np.arange(1, n + 1)
    f = np.stack([np.full(n, hub), k, k % n + 1], 1).astype(np.int32)
    return v, f


def projection_cases():
    rng = np.random.default_rng(20)
    cases = []

    def add(name, v, f, eye, kw, grad=None):
        v, f, eye = np.asarray(v, F), np.asarray(f, np.int32), np.asarray(eye, F).reshape(-1, 3)
        v = v if v.ndim == 3 else v[None]
        f = f if f.ndim == 3 else f[None]
        B = max(v.shape[0], f.shape[0], eye.shape[0])
        c = dict(name=name, vertices=v, faces=f, eye=eye, kw=kw,
                 grad=_grad(rng, B, f.shape[1]) if grad is None else np.asarray(grad, F))
        cases.append(c)
        return c

    # camera at the origin looking down +z with up +y: r is the identity, so camera space is world space exactly
    depths = [0.0, 1e-30, -1e-30, 1e-7, -1e-7, 1e-3, -1e-3, -1.0, 2.0]
    v = [[0.3 * (k % 3 - 1), 0.2 * (k // 3 - 1), z] for k, z in enumerate(depths)] + [[0.0, 0.0, 0.0]]
    f = [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 8, 0], [2, 4, 6], [1, 3, 9]]
    for mode, kw in (("look_at", dict(camera_mode="look_at", at=(0, 0, 1))),
                     ("look", dict(camera_mode="look", direction=(0, 0, 1)))):
        c = add("depth_" + mode, v, f, [0, 0, 0], kw)
        c["grad"][0, 3] = 0   # face [9 (= eye), 8, 0 (Z = 0)] untouched: the backward skips it (autograd would give NaN)
        assert np.array_equal(_axes(c)[0], np.eye(3, dtype=F))
        assert np.array_equal(opr.to_camera(c["vertices"], c["eye"], _axes(c))[0, :, 2], np.float32(depths + [0.0]))
    # eye == at: every axis normalises a zero vector to zero, every vertex maps to 0/0
    c = add("eye_is_at", rng.normal(0, 1, (12, 3)), rng.integers(0, 12, (8, 3)), [0.5, 0.2, -1.0],
            dict(camera_mode="look_at", at=(0.5, 0.2, -1.0)))
    assert not _axes(c).any()
    # up exactly parallel to at - eye: the x and y axes vanish; 1e-6 away: |up x z| < eps, x is not a unit vector
    for name, up in (("up_parallel", (0, 0, 1)), ("up_near_parallel", (1e-6, 0, 1))):
        c = add(name, rng.normal(0, 0.5, (12, 3)), rng.integers(0, 12, (8, 3)), [0, 0, -3],
                dict(camera_mode="look_at", up=up))
        n = np.linalg.norm(_axes(c)[0], axis=1)
        assert (n[0] == 0) if name == "up_parallel" else (0 < n[0] < 0.5)
    # C5's degenerate view: elevation 90 through get_points_from_angles, up = +y
    sv, sf = wl.sphere_by_faces(280)
    c = add("elevation_90", sv, sf, [wl.get_points_from_angles(2.732, 90.0, az) for az in (0.0, 45.0, 180.0)],
            dict(camera_mode="look_at"))
    assert (np.linalg.norm(_axes(c)[:, 0], axis=1) < 1e-3).all()
    # look with the direction just inside the host's |d . up| > 1 - 1e-4 rejection
    th = np.arccos(1 - 1.1e-4)
    up = (0.0, float(np.sin(th)), float(np.cos(th)))
    d = np.float32([0, 0, 1])
    u = np.asarray(up, F) / np.linalg.norm(np.asarray(up, F))
    assert 1 - 1.2e-4 < abs(float((d * u).sum())) <= 1 - 1e-4
    add("look_near_rejection", sv, sf, [0, 0.1, -2.5], dict(camera_mode="look", direction=(0, 0, 1), up=up))
    # viewing angles and orthogonal scales at their edges
    for ang in (1.0, 89.9):
        add("angle_%g" % ang, sv, sf, [0.3, 0.4, -2.7], dict(camera_mode="look_at", viewing_angle=ang))
    for s in (0.0, -1.0):
        add("ortho_scale_%g" % s, sv, sf, [0.3, 0.4, -2.7], dict(camera_mode="look_at", perspective=False, viewing_scale=s))
    add("look_left_ortho", sv, sf, [0.3, 0.4, -2.7],
        dict(camera_mode="look", direction=(0.1, -0.2, 1), up=(0.2, 1, 0), coordinate="left", perspective=False,
             viewing_scale=0.7))
    # every (vertices_batch, faces_batch, eye_batch) in {1, B}^3
    B, nv, nf = 3, 40, 60
    vb = rng.normal(0, 0.5, (B, nv, 3))
    fb = rng.integers(0, nv, (B, nf, 3))
    eb = rng.normal(0, 0.3, (B, 3)) + [0, 0, -3]
    for m in range(8):
        bv, bf, be = (B if m & 1 else 1), (B if m & 2 else 1), (B if m & 4 else 1)
        c = add("batch_v%d_f%d_e%d" % (bv, bf, be), vb[:bv], fb[:bf], eb[:be], dict(camera_mode="look_at"),
                grad=_grad(rng, B if m else 1, nf))
        assert (c["vertices"].shape[0], c["faces"].shape[0], c["eye"].shape[0]) == (bv, bf, be)
    # C5's batch: one 3280-face mesh seen from 120 views
    v5, f5 = wl.sphere_by_faces(3280)
    c = add("c5_shared_120", v5, f5, [wl.get_points_from_angles(2.732, 30.0, 3.0 * b) for b in range(120)],
            dict(camera_mode="look_at"), grad=_grad(rng, 120, 3280, zero_frac=0.6))
    assert c["faces"].shape[1] == 3280 and c["grad"].shape[0] == 120 and c["vertices"].shape[0] == 1
    # a 20 000-face fan: vertex 0 gathers 20 000 corner terms
    vf, ff = _fan(20000, rng)
    c = add("fan_20000", vf, ff, [0.1, 0.2, -2.5], dict(camera_mode="look_at"))
    assert (c["faces"][0] == 0).sum() == 20000
    # non-finite vertices and non-finite upstream gradients
    vn = rng.normal(0, 0.5, (2, 16, 3))
    vn[0, 3] = np.nan
    vn[1, 5, 1] = np.inf
    vn[1, 6, 2] = -np.inf
    fn = rng.integers(0, 16, (1, 24, 3))
    gn = _grad(rng, 2, 24)
    gn[0, 2, 1, 0] = np.nan
    gn[1, 7, 2, 2] = np.inf
    c = add("non_finite", vn, fn, [[0, 0, -3], [0.2, 0.1, -3]], dict(camera_mode="look_at"), grad=gn)
    assert not np.isfinite(c["vertices"]).all() and not np.isfinite(c["grad"]).all()
    # out-of-range indices: the corner is poisoned in the forward and adds nothing in the backward
    fo = rng.integers(0, 16, (1, 12, 3))
    fo[0, 1, 1], fo[0, 4, 0], fo[0, 9, 2] = 16, -1, INT32_MAX
    add("out_of_range", rng.normal(0, 0.5, (1, 16, 3)), fo, [0, 0, -3],
        dict(camera_mode="look_at"))
    return cases


# ---------------------------------------------------------------- flatten
def _dihedral(theta, scale=1.0, offset=(0, 0, 0)):
    """Edge v0 = 0, v1 = 1 along x; v2 at +y, v3 rotated by theta about the edge (theta = pi: flat, 0: fully folded)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.4, 1, 0], [0.6, np.cos(theta), np.sin(theta)]], np.float64)
    return (v * scale + offset).astype(F)


def flatten_cases():
    rng = np.random.default_rng(21)
    cases = []
    one = (np.array([0]), np.array([1]), np.array([2]), np.array([3]))

    def add(name, v, edges=one, eps=1e-6, faces=None):
        v = np.asarray(v, F)
        if edges is None:   # FlattenLoss's own table
            import torch
            import jrender_b200 as jr
            m = jr.FlattenLoss(torch.from_numpy(np.asarray(faces, np.int64)))
            edges = tuple(getattr(m, k).numpy() for k in ("v0s", "v1s", "v2s", "v3s"))
        cases.append(dict(name=name, vertices=v if v.ndim == 3 else v[None],
                          edges=tuple(np.asarray(e, np.int32) for e in edges), eps=eps, faces=faces))

    # flat (cos = -1: cos + 1 cancels) and fully folded (cos = +1) dihedrals, and some in between
    add("flat", _dihedral(np.pi))
    add("folded", _dihedral(0.0))
    add("angles", np.stack([_dihedral(t) for t in (np.pi - 1e-3, np.pi - 1e-2, 2.0, 1.0, 1e-3)]))
    v = _dihedral(2.0)
    v[2] = [0.3, 0, 0]
    add("collinear_v2", v)
    v = _dihedral(2.0)
    v[1] = v[0]
    add("zero_length_edge", v)
    add("coincident", np.zeros((4, 3), F) + F(0.25))
    add("scale_1e-4", np.stack([_dihedral(t, 1e-4, (1e-4, 0, 0)) for t in (np.pi, 2.5, 1.0)]))
    add("scale_1e3", np.stack([_dihedral(t, 1e3, (2e3, 0, 0)) for t in (np.pi, 2.5, 1.0)]))
    add("eps_0", np.stack([_dihedral(t) for t in (2.5, 1.0)]), eps=0.0)
    # through the edge table built from faces
    sv, sf = wl.sphere_by_faces(280)
    x7 = (sv[None] + rng.normal(0, 0.02, (7,) + sv.shape)).astype(F)
    add("sphere_b1", x7[:1], edges=None, faces=sf)
    add("sphere_b7", x7, edges=None, faces=sf)
    add("duplicate_faces", rng.normal(0, 1, (2, 3, 3)), edges=None, faces=np.array([[0, 1, 2], [0, 1, 2]]))
    # a 3-face edge (0, 1) and boundary edges: the table keeps only edges with two faces
    nm = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [2, 1, 5]])
    add("non_manifold", rng.normal(0, 1, (2, 6, 3)), edges=None, faces=nm)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_host_loss_sphere280.npz"))
    add("rotated_fixture", g["vertices"], edges=None, faces=g["faces_rot"])
    add("no_edges", rng.normal(0, 1, (2, 5, 3)), edges=tuple(np.zeros(0, np.int32) for _ in range(4)))
    for c in cases:
        if c["faces"] is not None:
            c["faces"] = np.asarray(c["faces"], np.int64)
    assert cases[0]["vertices"][0, 3, 1] == F(np.cos(np.pi)) and abs(cases[0]["vertices"][0, 3, 2]) < 1e-7
    return cases


# ---------------------------------------------------------------- Laplacian
def tetra_self_pair():
    """The closed tetrahedron plus the face [2, 2, 2]."""
    f = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2], [2, 2, 2]])
    return np.random.default_rng(1).normal(size=(1, 4, 3)).astype(F), f


def fan_self_pair():
    """A 4-face fan around vertex 0 plus the face [1, 1, 5]."""
    f = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 4, 1], [1, 1, 5]])
    return np.random.default_rng(2).normal(size=(1, 6, 3)).astype(F), f


def laplacian_cases():
    rng = np.random.default_rng(22)
    cases = []
    v, f = tetra_self_pair()
    cases.append(dict(name="tetra_self_pair", vertices=v, faces=f))
    v, f = fan_self_pair()
    cases.append(dict(name="fan_self_pair", vertices=v, faces=f))
    v, f = fan_self_pair()
    cases.append(dict(name="self_pair_orders", vertices=v,
                      faces=np.concatenate([f[:4], [[1, 5, 1], [5, 2, 2], [3, 3, 3]]])))
    sv, sf = wl.sphere_by_faces(280)
    iso = np.concatenate([sv, rng.normal(0, 1, (2, 3))]).astype(F)
    cases.append(dict(name="isolated", vertices=np.stack([iso, iso * F(1.5)]), faces=sf))
    vf, ff = _fan(1000, rng)
    cases.append(dict(name="degree_1000", vertices=vf[None], faces=ff))
    xn = (sv[None] + rng.normal(0, 0.02, (3,) + sv.shape)).astype(F)
    xn[0, 0] = np.nan
    xn[1, 7, 2] = np.inf
    cases.append(dict(name="non_finite", vertices=xn, faces=sf))
    cases.append(dict(name="sphere_b4", vertices=(sv[None] + rng.normal(0, 0.02, (4,) + sv.shape)).astype(F), faces=sf))
    for c in cases:
        c["faces"] = np.asarray(c["faces"], np.int64)
    assert len(np.unique(ff[ff[:, 0] == 0][:, 1:])) == 1000   # vertex 0 has 1000 distinct neighbours
    assert (tetra_self_pair()[1] == 2).all(1).any() and (fan_self_pair()[1][:, 0] == fan_self_pair()[1][:, 1]).any()
    return cases
