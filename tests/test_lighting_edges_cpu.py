"""The scenes of test_lighting_edges_gpu.py reach the paths they are built for, and the kernels' float32 emulation
(oracle/lighting.py) is held to float64 autograd.  No GPU: the geometry is checked in numpy, the flat backward's normal
derivative is restated with oracle.numbers.Dual (float32, unfused, as the kernel is compiled), and the non-finite cases
run through the op-by-op float32 mirror on the CPU.

Tolerance of the emulation test: per entry, the emulated float32 gradient within its EV bound (oracle/numbers.py: the
propagated input error plus one float32 rounding per operation, with the float32 literals' and light parameters'
distance from the mirror's float64 ones) of the float64 mirror's autograd, plus 1e-12 of the terms' magnitudes for
float64's own rounding; grad_vertices entries within the sum of their terms' bounds.  Members within their bound of a
kink are left out, counted and capped (NEAR_CAP, NEAR_CAP_ABS)."""
import numpy as np
import pytest
import torch

from oracle import lighting as OL
from oracle.numbers import EV, Dual
from oracle.numbers import check_terms as _check_terms
from tests import lighting_edge_cases as E

F32 = np.float32


# ---- the normal's derivative on slivers, in the kernel's float32 arithmetic -------------------------------------------

def _vars(v):
    n = v.shape[0]
    zero, one = np.zeros(n, F32), np.ones(n, F32)
    return [Dual(v[:, k], [one if j == k else zero for j in range(9)]) for k in range(9)]


def _cross_duals(v):
    """The float32 cross product's duals over the 9 vertex coordinates, op for op as csrc/dual.cuh (oracle.numbers)."""
    dv = _vars(v)
    a = [dv[0] - dv[3], dv[1] - dv[4], dv[2] - dv[5]]
    b = [dv[6] - dv[3], dv[7] - dv[4], dv[8] - dv[5]]
    return [b[1] * a[2] - b[2] * a[1], b[2] * a[0] - b[0] * a[2], b[0] * a[1] - b[1] * a[0]]


def normal_jacobian_float32(v):
    """d N / d v [n, 3, 9] as the backward formed it before taking the float64 normal: the float32 cross product,
    normalised in float32 duals (sqrt's derivative 0.5 / sqrt)."""
    c = _cross_duals(v)
    n = ((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]).sqrt()
    return np.stack([np.stack((ck / n).d, 1) for ck in c], axis=1)


def normal_jacobian_fixed(v):
    """The kernel's d N / d v now: float32 partials of c through (I - N N^T) / |c| at the float64 N and |c|."""
    c = _cross_duals(v)
    dc = np.stack([np.stack(ck.d, 1) for ck in c], axis=1)          # [n, 3, 9]
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


# ---- the kernels' float32 emulation against float64 autograd ------------------------------------------------------------
#
# oracle/lighting.py restates the four kernels in numpy float32 (the GPU tests hold the kernels to it bit for bit) and,
# with the same code over EV numbers, bounds each float32 term's distance from the float64 value of the same expression.
# Here those bounds are checked against the op-by-op mirror's float64 autograd, entry by entry: per-texel gradients
# within their own term's bound, each grad_vertices entry within the sum of its terms' bounds (the kernels' atomic order
# is bounded separately, on the GPU).  Branches follow the float32 walk; members whose EV value lies within its bound
# of a kink -- relu arguments at 0, the output clamp's 0 and 1, den4 at 0.01, a norm at normalize's 1e-12 -- may take the
# other branch in float64 and are left out, counted by kind, with the counts capped below.

def _scenes():
    s = {"flat_shapes_25_25": lambda: E.flat_shapes(25, 25), "flat_shapes_125_1": lambda: E.flat_shapes(125, 1),
         "flat_shared_be1": lambda: E.flat_shapes(9, 9, B=4, Bv=1, Be=1), "flat_no_eye": lambda: E.flat_shapes(9, 1, Be=0),
         "flat_geometry": E.flat_geometry, "nm_shapes_33_3_3": lambda: E.nm_shapes(33, 3, 3),
         "nm_shapes_33_1_3": lambda: E.nm_shapes(33, 1, 3), "nm_shapes_1_3_1": lambda: E.nm_shapes(1, 3, 1),
         "nm_no_eye": lambda: E.nm_shapes(31, 1, 1, Be=0), "nm_clamp_bounds": E.nm_clamp_bounds,
         "head_2000_faces": lambda: E.head(faces=2000), "shared_vertex": E.shared_vertex,
         "shared_vertex_nm": lambda: E.shared_vertex(nm=True)}
    for nm in (False, True):
        for spec in (True, False):
            s["equality_%s_%s" % ("nm" if nm else "flat", "spec" if spec else "diffuse")] = \
                (lambda nm=nm, spec=spec: E.equality(nm, spec))
    for nm in (False, True):
        for site in (E.NM_SITES if nm else E.FLAT_SITES):
            s["nonfinite_%s_%s" % ("nm" if nm else "flat", site)] = (lambda nm=nm, site=site: E.nonfinite(site, np.nan, nm=nm)[1])
    return s


SCENES = _scenes()
# most members left out, per kind: a share of the scene's members (faces on the flat path, texels on the normal-map
# path), at least 4; and the counts of the scenes built to sit on kinks, as measured.  flat_geometry: its 80 texels on
# the clamp bounds (20 faces x 4 eyes) and one more, the edge-on, collinear and coincident faces' relus, V and H on
# normalize's eps path; the equality scenes: the zero-centroid face under each eye.
NEAR_CAP = {"relu": 0.01, "clamp": 0.01, "den4": 0.005, "norm_eps": 0.005}
NEAR_CAP_ABS = {"flat_geometry": {"clamp": 81, "relu": 18, "norm_eps": 6, "den4": 3},
                "equality_flat_spec": {"relu": 2, "norm_eps": 2, "den4": 1},
                "equality_nm_spec": {"relu": 6, "norm_eps": 10, "den4": 3}, "equality_nm_diffuse": {"norm_eps": 4}}


def _excluded(sc, near, nm):
    """Per-texel and per-vertex-entry masks of what the near-kink members reach."""
    B, nf = sc["tex"].shape[:2]
    T = sc["tex"][0, 0].size // 3
    Bv, nv = sc["v"].shape[:2]
    ex_v = np.zeros((Bv, nv), bool)
    if nm:
        tex = np.zeros((B, nf, T), bool)
        for fl in near.values():
            tex |= fl
        face = tex.any(2)
    else:
        face = np.zeros(B * nf, bool)
        for fl in near.values():
            face |= fl
        face = face.reshape(B, nf)
        tex = np.broadcast_to(face[:, :, None], (B, nf, T)).copy()
    for b, f in zip(*np.nonzero(face)):
        ex_v[0 if Bv == 1 else b, sc["f"][f]] = True
    return tex, ex_v


@pytest.mark.parametrize("name", sorted(SCENES))
def test_emulated_terms_within_their_bound_of_float64_autograd(name):
    sc = SCENES[name]()
    nm = "nt" in sc
    a = E.kernel_args(sc)
    bwd = OL.nm_backward if nm else OL.surface_backward
    g32 = bwd(a)
    gev = bwd(dict(a, light=OL.light_ev(sc["light"], sc["eye"] is not None)), lift=EV, replay=g32)
    _, ref = E.run(sc, "cpu", torch.float64, False)
    near = gev["near"]
    members = (sc["tex"].shape[0] * sc["tex"].shape[1] * (sc["tex"][0, 0].size // 3 if nm else 1))
    counts = {k: int(np.count_nonzero(v)) for k, v in near.items()}
    print("%s: members left out near a kink, by kind: %s of %d" % (name, counts, members))
    for k, n in counts.items():
        cap = NEAR_CAP_ABS.get(name, {}).get(k, max(4, NEAR_CAP[k] * members))
        assert n <= cap, (name, k, n, cap)
    ex_tex, ex_v = _excluded(sc, near, nm)
    rows = []
    for k, r in ref.items():
        if k == "vertices":
            size = a["vertices"].size
            got, err, A = (np.zeros(size) for _ in range(3))
            sl = g32["vertex_slots"].reshape(-1) if "vertex_slots" in g32 else np.zeros(0, np.int64)
            t32 = np.asarray(g32.get("vertex_terms", np.zeros(0)), np.float64).reshape(-1)
            tev = gev.get("vertex_terms")
            if r is None:   # no path in the mirror: the kernel's terms are exact zeros
                assert not t32.any(), name
                continue
            _check_terms(t32, EV(tev.v.reshape(-1), tev.e.reshape(-1)))
            np.add.at(got, sl, t32)
            np.add.at(err, sl, tev.e.reshape(-1))
            np.add.at(A, sl, np.abs(tev.v.reshape(-1)))
            got, err, A = (x.reshape(r.shape) for x in (got, err, A))
            keep = ~np.broadcast_to(ex_v[..., None], r.shape)
        else:
            got, ev = g32[k], gev[k]
            if r is None:
                assert got is None or not np.asarray(got).any(), (name, k)
                continue
            _check_terms(got, ev)
            got = np.asarray(got, np.float64)
            if got.shape != r.shape:    # a flat face's mean material: the same value on each of its Tm texels
                got = got.reshape(r.shape)
            err, A = ev.e.reshape(r.shape), np.abs(ev.v).reshape(r.shape)
            et = ex_tex.any(0)[None] if (k == "normal_textures" and r.shape[0] == 1) else ex_tex
            keep = ~np.broadcast_to(et.reshape(et.shape[:3] + (1,) * (r.ndim - 3)), r.shape) if nm else \
                ~np.broadcast_to(et[:, :, :1].reshape((et.shape[0], et.shape[1]) + (1,) * (r.ndim - 2)), r.shape)
        fin = np.isfinite(r) & np.isfinite(got) & np.isfinite(err)
        keep = keep & fin
        bound = err + 1e-12 * A + 1e-300
        diff = np.abs(got - r)
        ratio = float((diff[keep] / bound[keep]).max(initial=0.0))
        nz = keep & (r != 0)
        old = 1e-4 * np.abs(r[np.isfinite(r)]).max(initial=0.0)
        share_old = float(np.mean(old > 0.01 * np.abs(r[nz]))) if nz.any() else 0.0
        share_new = float(np.mean(bound[nz] > 0.01 * np.abs(r[nz]))) if nz.any() else 0.0
        rows.append("  %-16s worst |f32 - f64| / bound %.3f; allowance > 1%% of |g|: 1e-4 max %5.1f%%, bound %5.1f%%"
                    % (k, ratio, 100 * share_old, 100 * share_new))
        assert ratio <= 1, (name, k, ratio)
    print("\n".join(rows))
