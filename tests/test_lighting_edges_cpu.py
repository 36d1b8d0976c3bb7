"""The scenes of test_lighting_edges_gpu.py reach the paths they are built for.  No GPU: the geometry is checked in
numpy, the flat backward's normal derivative is restated in numpy float32 (unfused, as the kernel is compiled), and the
non-finite cases run through the op-by-op float32 mirror on the CPU."""
import numpy as np
import pytest
import torch

from tests import lighting_edge_cases as E

F32 = np.float32


# ---- the normal's derivative on slivers, in the kernel's float32 arithmetic -------------------------------------------

class D:
    """Forward-mode dual numbers over the 9 vertex coordinates in numpy float32, op for op as csrc/dual.cuh."""

    def __init__(self, v, d):
        self.v, self.d = F32(v) if np.isscalar(v) else v.astype(F32), d.astype(F32)

    def __sub__(self, o):
        return D(self.v - o.v, self.d - o.d)

    def __add__(self, o):
        return D(self.v + o.v, self.d + o.d)

    def __mul__(self, o):
        return D(self.v * o.v, self.d * o.v[:, None] + self.v[:, None] * o.d)

    def __truediv__(self, o):
        r = self.v / o.v
        ib = F32(1) / o.v
        return D(r, (self.d - r[:, None] * o.d) * ib[:, None])


def _vars(v):
    n = v.shape[0]
    return [D(v[:, k], np.eye(9, dtype=F32)[k][None].repeat(n, 0)) for k in range(9)]


def _cross_duals(v):
    dv = _vars(v)
    a = [dv[0] - dv[3], dv[1] - dv[4], dv[2] - dv[5]]
    b = [dv[6] - dv[3], dv[7] - dv[4], dv[8] - dv[5]]
    return [b[1] * a[2] - b[2] * a[1], b[2] * a[0] - b[0] * a[2], b[0] * a[1] - b[1] * a[0]]


def normal_jacobian_float32(v):
    """d N / d v [n, 3, 9] as the backward formed it before taking the float64 normal: the float32 cross product,
    normalised in float32 duals (sqrt's derivative 0.5 / sqrt)."""
    c = _cross_duals(v)
    dot = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]
    s = np.sqrt(dot.v)
    n = D(s, dot.d * (F32(0.5) / s)[:, None])
    return np.stack([(ck / n).d for ck in c], axis=1)


def normal_jacobian_fixed(v):
    """The kernel's d N / d v now: float32 partials of c through (I - N N^T) / |c| at the float64 N and |c|."""
    c = _cross_duals(v)
    dc = np.stack([ck.d for ck in c], axis=1)                       # [n, 3, 9]
    c64, n = _cross64(v)
    N = (c64 / n[:, None]).astype(F32)
    inv = F32(1) / n.astype(F32)
    Ndc = (N[:, 0, None] * dc[:, 0] + N[:, 1, None] * dc[:, 1]) + N[:, 2, None] * dc[:, 2]
    return (dc - N[:, :, None] * Ndc[:, None, :]) * inv[:, None, None]


def _cross64(v):
    v = v.astype(F32)
    a = (v[:, 0:3] - v[:, 3:6]).astype(np.float64)
    b = (v[:, 6:9] - v[:, 3:6]).astype(np.float64)
    c = np.cross(b, a)
    return c, np.linalg.norm(c, axis=1)


def normal_jacobian_float64(v):
    c, n = _cross64(v)
    N = c / n[:, None]
    a_idx = [(0, 3), (1, 4), (2, 5)]
    b_idx = [(6, 3), (7, 4), (8, 5)]
    da = np.zeros((3, 9)); db = np.zeros((3, 9))
    for k, (p, q) in enumerate(a_idx):
        da[k, p], da[k, q] = 1, -1
    for k, (p, q) in enumerate(b_idx):
        db[k, p], db[k, q] = 1, -1
    a = (v[:, 0:3] - v[:, 3:6]).astype(np.float64)
    b = (v[:, 6:9] - v[:, 3:6]).astype(np.float64)
    dc = np.cross(db.T[None], a[:, None, :]).transpose(0, 2, 1) + np.cross(b[:, None, :], da.T[None]).transpose(0, 2, 1)
    P = np.eye(3)[None] - N[:, :, None] * N[:, None, :]
    return np.einsum("nij,njk->nik", P, dc) / n[:, None, None]


def test_sliver_normal_gradient_needs_the_float64_normal():
    """The diffuse gradient d (N . L) / d v on the slivers, relative to its largest value over the slivers of one
    aspect: the old float32 normalisation misses the suite's 1e-4 bar at aspect 1e-5 (so the GPU test can fail on it);
    the kernel's formula now stays well inside it at every aspect."""
    sc = E.flat_geometry()
    L = np.float64([0, 1, 0])
    tris = sc["v"][0][sc["f"][sc["slivers"]]].reshape(-1, 9)
    ref = np.einsum("nij,i->nj", normal_jacobian_float64(tris), L)
    old = np.einsum("nij,i->nj", normal_jacobian_float32(tris).astype(np.float64), L)
    new = np.einsum("nij,i->nj", normal_jacobian_fixed(tris).astype(np.float64), L)
    for a in E.SLIVER_ASPECTS:
        m = sc["sliver_aspect"] == a
        scale = np.abs(ref[m]).max()
        err_old = np.abs(old[m] - ref[m]).max() / scale
        err_new = np.abs(new[m] - ref[m]).max() / scale
        print("aspect %g: float32 normal %.2e, float64 normal %.2e" % (a, err_old, err_new))
        assert err_new < 1e-6, (a, err_new)
    assert err_old > 1e-4, err_old   # aspect 1e-5: the error grows like 1 / aspect (5e-5 at 1e-4)
    N = E.flat_normals(sc["v"], sc["f"])[0, sc["slivers"]]
    assert (N @ L > 0.05).sum() >= 0.4 * len(N)    # lit slivers: the derivative reaches the output


def test_geometry_edges_hit_their_exact_zeros():
    sc = E.flat_geometry()
    v, f = sc["v"], sc["f"]
    fv = v[0][f].astype(F32)
    c = np.cross((fv[:, 2] - fv[:, 1]).astype(np.float64), (fv[:, 0] - fv[:, 1]).astype(np.float64))
    assert np.all(c[sc["collinear"]] == 0) and np.all(c[sc["coincident"]] == 0)       # normalize's eps path, N = 0
    N = E.flat_normals(v, f)[0]
    assert np.all(N[sc["edge_on"]] @ np.float64([0, 1, 0]) == 0)                       # N . L == 0: relu's kink
    assert np.all(np.abs(N[sc["edge_on"]]).max(axis=1) == 1)
    pos32 = E.centroid(v, f)[0]
    pos64 = fv.astype(np.float64).sum(axis=1) / 3.0
    for face, eye, want in ((sc["eye_face"], sc["eye"][1], [0, 0, 0]), (sc["below_face"], sc["eye"][2], [0, -1, 0])):
        assert np.array_equal(eye - pos32[face], F32(want)) and np.array_equal(eye - pos64[face], np.float64(want))
    assert N[sc["below_face"]] @ np.float64([0, 1, 0]) > 0.1                           # lit: V = -L, H = 0
    assert (sc["v"].shape[0], sc["eye"].shape[0], sc["tex"].shape[0]) == (1, 4, 4)     # one mesh, four eyes


def _mirror32(sc, tex=None):
    sc = dict(sc)
    if tex is not None:
        sc["tex"] = tex
    return E.run(sc, "cpu", torch.float32, False, grads=False)[0]


def test_clamp_bound_texels_are_exactly_0_and_1_before_the_clamp():
    """On the unlit texels diffuse is exactly the ambient colour and specular exactly 0: with textures 1/8 nothing
    clamps and the output is exactly tex * ambient, so tex = 0 and tex = 1 / ambient land exactly on 0 and 1."""
    for sc, sel in ((E.flat_geometry(), None), (E.nm_clamp_bounds(), None)):
        if "bounds" in sc:
            b, f, t = sc["bounds"]
            sel = (b, f, t)
        else:
            sel = (slice(None), sc["unlit"], slice(0, 2))
        assert sc["tex"][sel].size > 0
        out = _mirror32(sc, np.full_like(sc["tex"], 0.125))
        assert np.array_equal(out[sel], np.broadcast_to(0.125 * E.UNLIT_DIFFUSE, out[sel].shape))
        out = _mirror32(sc)
        assert (out[sel] == 0).any() and (out[sel] == 1).any()
        tex = sc["tex"][sel]
        assert set(np.unique(tex * E.UNLIT_DIFFUSE)) == {0.0, 1.0}


def test_shapes_cover_the_launch_edges():
    for T, Tm in ((1, 1), (25, 1), (25, 25), (125, 1), (125, 125)):
        sc = E.flat_shapes(T, Tm)
        B, nf = sc["tex"].shape[:2]
        assert (B * nf) % E.BLOCK != 0
        assert sc["tex"][0, 0].size // 3 == T and sc["met"][0, 0].size == Tm
    for T in (1, 31, 32, 33, 64, 225):
        sc = E.nm_shapes(T, 1, 3)
        assert sc["nt"].shape[2] == T and (3 * sc["f"].shape[0]) % 4 != 0   # warps per block of the backward: 4
    assert -(-225 // 32) == 8   # T = 225: every lane takes 7 or 8 texels


@pytest.mark.parametrize("nm", [False, True])
@pytest.mark.parametrize("site", E.NM_SITES)
@pytest.mark.parametrize("value", sorted(E.NONFINITE))
def test_nonfinite_inputs_make_the_mirror_nonfinite_where_expected(nm, site, value):
    if not nm and site in ("normal", "tbn"):
        pytest.skip("no per-texel normal on the flat path")
    if site == "tbn" and value != "nan":
        pytest.skip("a degenerate UV triangle: one case")
    clean, dirty, (b, fa) = E.nonfinite(site, E.NONFINITE[value], nm=nm)
    base = _mirror32(clean)
    out = _mirror32(dirty)
    assert np.isfinite(base).all()
    N = E.flat_normals(clean["v"], clean["f"])[:, fa]
    assert (N @ np.float64([0.3, 1, -0.4]) > 0.5).all()       # the face is lit: both light branches are live
    bad = ~np.isfinite(out)
    others = np.ones(bad.shape[:2], bool)
    others[b, fa] = False
    assert not bad[others].any()                                # contained in its face and batch element
    assert np.array_equal(out[others], base[others])
    face = bad[b, fa]
    if site == "texel":
        # one channel of one texel; +-inf clamps to a finite bound in torch, NaN stays NaN
        assert face.sum() == (1 if value == "nan" else 0) and (value != "nan" or face[2, 1])
    elif site == "normal":
        assert face[4].all() and face.sum() == 3                # one texel's normal
    elif site in ("metallic", "roughness") and not nm:
        assert face.all()                                       # the face's mean material
    elif site in ("metallic", "roughness"):
        assert face[3].all() and face.sum() == 3                # the texel's own material
    else:
        assert face.all()                                       # vertex: the normal and centroid; tbn: every texel
