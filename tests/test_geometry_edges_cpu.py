"""The float32 emulations of k_project_faces_bwd, k_flatten_loss and k_laplacian_loss (oracle/preraster.py,
oracle/mesh_loss.py) against float64 references on the cases of geometry_edge_cases.py, and the host-built tables of
LaplacianLoss / FlattenLoss against the reference's dense matrix and edge scan.  No GPU.

Per-entry bound.  Each emulated term is re-evaluated with `EV` numbers (oracle/numbers.py): a float64 value plus a running bound on how far
the float32 evaluation of the same expression can be from the exact one (every operation: propagated input error plus
one rounding u = 2^-24 of the result, 2^-52 for the float64 value's own rounding and 2^-149 for gradual underflow).  The
sum of those per-term bounds is the bound on |exact sum of the emulated terms - float64 reference| for that entry.
Members where the float32 expression is ill-conditioned by construction are left out by stated thresholds; the tests
count them, and they stay in the bit-level GPU check."""
import numpy as np
import pytest
import torch

import jrender_b200 as jr
from oracle import mesh_loss as oml
from oracle import preraster as opr
from oracle.numbers import EV
from oracle.numbers import check_terms as _check_terms
from tests import geometry_edge_cases as gec

def _ev_sums(slots, terms, size):
    """Per entry: float64 sum of the EV values and sum of their error bounds."""
    s, e = np.zeros(size), np.zeros(size)
    np.add.at(s, slots, terms.v.reshape(-1))
    np.add.at(e, slots, terms.e.reshape(-1))
    return s, e


# ---------------------------------------------------------------- projection
PROJ = gec.projection_cases()
Z_MIN = 1e-3   # corners with |camera Z| below this are left out of the float64 comparison (1/Z amplifies Z's rounding)
PROJ_EXCLUDED = {"depth_look_at": 6, "depth_look": 6, "eye_is_at": 12, "non_finite": 3}


@pytest.mark.parametrize("c", PROJ, ids=[c["name"] for c in PROJ])
def test_projection_backward_terms_against_float64_vjp(c):
    v, f, eye, g, kw = c["vertices"], c["faces"], c["eye"], c["grad"], c["kw"]
    rows, t32 = opr.project_faces_bwd_terms(v, f, eye, g, **kw)
    _, tev = opr.project_faces_bwd_terms(v, f, eye, g, lift=EV, **kw)
    for k in range(3):
        _check_terms(t32[k], tev[k])
    size = v.shape[0] * v.shape[1]
    # the float64 reference: the VJP of every corner, the all-zero ones and the out-of-range ones included
    kw64 = dict(kw)
    B = g.shape[0]
    fb = np.broadcast_to(f, (B,) + f.shape[1:])
    bad = (fb < 0) | (fb >= v.shape[1])
    ref = opr.project_faces_vjp(v, np.where(bad, 0, fb), eye, np.where(bad[..., None], 0, g), vertices_batch=v.shape[0], **kw64)
    ref = ref.reshape(size, 3)
    # excluded rows: a corner with |Z| < Z_MIN or a non-finite input, in any image
    e = np.broadcast_to(eye, (B, 3))
    cam = opr.to_camera(np.broadcast_to(v, (B,) + v.shape[1:]), e, opr.camera_axes(e, **{k: kw[k] for k in kw if k in ("camera_mode", "at", "direction", "up", "coordinate")}))
    persp = kw.get("perspective", True)
    with np.errstate(invalid="ignore"):
        degenerate = ~np.isfinite(cam).all(-1) | (persp & (np.abs(cam[..., 2]) < Z_MIN))
    row_of = (np.arange(B)[:, None] * (v.shape[0] > 1)) * v.shape[1] + np.arange(v.shape[1])
    ex_rows = set(row_of[degenerate].tolist())
    for b, fi, ci in zip(*np.nonzero(~bad & ~np.isfinite(g).all(-1))):
        ex_rows.add((b if v.shape[0] > 1 else 0) * v.shape[1] + fb[b, fi, ci])
    assert len(ex_rows) == PROJ_EXCLUDED.get(c["name"], 0)
    keep = np.ones(size, bool)
    keep[list(ex_rows)] = False
    for k in range(3):
        ev = tev[k]
        s, err = _ev_sums(rows, ev, size)
        got = np.zeros(size)
        np.add.at(got, rows, np.asarray(t32[k], np.float64))
        A = np.zeros(size)
        np.add.at(A, rows, np.abs(ev.v))
        bound = err + 1e-13 * A + 1e-300
        diff = np.abs(got - ref[:, k])
        assert np.all(diff[keep] <= bound[keep]), (diff / bound)[keep].max()
        # the bound is not vacuous: the median entry's is a few ulps of its term magnitudes
        m = keep & (A > 0)
        assert not m.any() or np.median(bound[m] / A[m]) < 1e-5


def test_projection_forward_poisons_out_of_range_corners():
    c = next(c for c in PROJ if c["name"] == "out_of_range")
    fv = opr.project_faces(c["vertices"], c["faces"], c["eye"], **c["kw"])
    bad = np.isnan(fv).all(-1)[0]
    assert sorted(zip(*np.nonzero(bad))) == [(1, 1), (4, 0), (9, 2)]
    assert np.isfinite(fv[0][~bad]).all()


def test_mesh_int64_faces_outside_int32_do_not_alias():
    """2^32 + 1 must not wrap to vertex 1: Mesh and project_faces map every index outside [0, 2^31) to -1."""
    from jrender_b200.preraster import int32_faces
    f = np.array([[0, 2 ** 32 + 1, 2], [-(2 ** 32) + 1, 1, 2], [2 ** 31, 1, 2 ** 31 - 1]], np.int64)
    m = jr.Mesh(np.zeros((3, 3), np.float32), f)
    assert m.faces.dtype == torch.int32
    assert m.faces[0].tolist() == [[0, -1, 2], [-1, 1, 2], [-1, 1, 2 ** 31 - 1]]
    assert int32_faces(torch.from_numpy(f), "cpu").tolist() == m.faces[0].tolist()


# ---------------------------------------------------------------- flatten
FLAT = gec.flatten_cases()
SIN2_MIN = 1e-3   # edges with 1 - cos^2 < this in a half-plane (sqrt(1 - cos^2 + eps) cancels) are left out of the float64 comparison
FLAT_EXCLUDED = {"collinear_v2": 1}


def _flatten_float64(x, edges, eps):
    m = jr.FlattenLoss(torch.zeros(0, 3, dtype=torch.int64))
    for k, e in zip(("v0s", "v1s", "v2s", "v3s"), edges):
        setattr(m, k, torch.from_numpy(np.asarray(e, np.int64)))
    m.fused = False
    xt = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    loss = m(xt, eps=eps)
    loss.sum().backward()
    return loss.detach().numpy(), xt.grad.numpy()


def _flatten_cos2(x, edges, eps):
    """float64 cos^2 of both half-plane angles (v2 - v0 and v3 - v0 against the edge), per (batch, edge)."""
    x = np.asarray(x, np.float64)
    p = [x[:, np.asarray(e, np.int64)] for e in edges]
    a = p[1] - p[0]
    out = []
    for q in (p[2], p[3]):
        b = q - p[0]
        al1, bl1 = np.sqrt((a * a).sum(-1) + eps), np.sqrt((b * b).sum(-1) + eps)
        out.append(((a * b).sum(-1) / (al1 * bl1 + eps)) ** 2)
    return np.max(out, 0)


@pytest.mark.parametrize("c", FLAT, ids=[c["name"] for c in FLAT])
def test_flatten_terms_against_float64_autograd(c):
    x, edges, eps = c["vertices"], c["edges"], c["eps"]
    B, nv = x.shape[:2]
    E = len(edges[0])
    val32, d32 = oml.flatten_terms(x, edges, eps)
    val_ev, d_ev = oml.flatten_terms(x, edges, eps, lift=EV)
    _check_terms(val32, val_ev)
    _check_terms(d32, d_ev)
    ref_loss, ref_grad = _flatten_float64(x, edges, eps)
    with np.errstate(invalid="ignore"):
        ill = (1 - _flatten_cos2(x, edges, eps) < SIN2_MIN).reshape(-1) if E else np.zeros(0, bool)
    b = np.repeat(np.arange(B), E)
    assert int(ill.sum()) == FLAT_EXCLUDED.get(c["name"], 0)
    # loss: batch elements without an excluded edge
    s, err = _ev_sums(b, val_ev, B)
    got = np.zeros(B)
    np.add.at(got, b, val32.astype(np.float64))
    okb = np.ones(B, bool)
    okb[b[ill]] = False
    assert np.all(np.abs(got - ref_loss)[okb] <= (err + 1e-13 * np.abs(ref_loss) + 1e-300)[okb])
    # gradient: entries no excluded edge touches
    idx = [np.asarray(e, np.int64)[np.arange(B * E) % E] for e in edges]
    slots = np.stack([(b * nv + idx[k]) * 3 + cc for k in range(4) for cc in range(3)], 1)
    s, err = _ev_sums(slots.reshape(-1), d_ev, B * nv * 3)
    got = np.zeros(B * nv * 3)
    np.add.at(got, slots.reshape(-1), d32.astype(np.float64).reshape(-1))
    A = np.zeros(B * nv * 3)
    np.add.at(A, slots.reshape(-1), np.abs(d_ev.v).reshape(-1))
    ok = np.ones(B * nv * 3, bool)
    ok[slots[ill].reshape(-1)] = False
    diff = np.abs(got - ref_grad.reshape(-1))
    bound = err + 1e-13 * A + 1e-300
    assert np.all(diff[ok] <= bound[ok]), (diff / bound)[ok].max()
    if E >= 100:   # not vacuous on a whole mesh
        assert np.median((bound / np.maximum(A, 1e-300))[ok & (A > 0)]) < 1e-3   # a worst case over ~60 roundings


@pytest.mark.parametrize("c", [c for c in FLAT if c["faces"] is not None and c["name"] != "non_manifold"],
                         ids=lambda c: c["name"])
def test_flatten_table_matches_reference_scan(c):
    """Where every listed edge has exactly two faces (the reference's scan keeps v2s / v3s aligned with v0s there), the
    table FlattenLoss builds is the reference's, as a set of (v0, v1, v2, v3)."""
    ref = oml.flatten_edges(c["faces"])
    assert len(ref[2]) == len(ref[0]) == len(ref[3])
    got = set(zip(*(np.asarray(e).tolist() for e in c["edges"])))
    assert got == set(zip(*(e.tolist() for e in ref)))


def test_flatten_table_skips_non_manifold_and_boundary_edges():
    c = next(c for c in FLAT if c["name"] == "non_manifold")
    got = set(zip(*(np.asarray(e).tolist() for e in c["edges"])))
    assert got == {(0, 1, 2, 3), (1, 2, 0, 5)}   # (0, 1) in three faces: the first two; (1, 2) in two; the rest in one


@pytest.mark.parametrize("face", [[1, 1, 5], [5, 1, 1], [1, 5, 1], [2, 2, 2]])
def test_flatten_rejects_faces_with_a_repeated_index(face):
    f = np.concatenate([gec.fan_self_pair()[1][:4], [face]])
    with pytest.raises(ValueError, match=r"face 4 \[%d, %d, %d\]" % tuple(face)):
        jr.FlattenLoss(torch.from_numpy(f))
    with pytest.raises(IndexError):   # the reference's own scan
        oml.flatten_edges(f)


# ---------------------------------------------------------------- Laplacian
LAP = gec.laplacian_cases()


def _table(mod):
    return mod.nbr32.numpy(), mod.nbr_w.numpy(), mod.diag.numpy()


def _dense_from_table(mod):
    nbr, w, dg = _table(mod)
    L = np.diag(dg.astype(np.float64))
    for i, k in zip(*np.nonzero(w)):
        L[i, nbr[i, k]] += w[i, k]
    return L


@pytest.mark.parametrize("c", LAP, ids=[c["name"] for c in LAP])
def test_laplacian_table_is_the_reference_matrix(c):
    """The padded table of LaplacianLoss, expanded, is the dense float32 matrix laplacian_loss.py:11-27 builds -- a
    self-pair [a, a, b] adds 1 to a's divisor and does not make a its own neighbour (NaN rows compared as NaN)."""
    x = c["vertices"]
    mod = jr.LaplacianLoss(torch.from_numpy(x[0]), torch.from_numpy(c["faces"]))
    ref = oml.laplacian_matrix(x.shape[1], c["faces"])
    got = _dense_from_table(mod)
    iso = np.isnan(np.diag(ref))   # an isolated vertex: the reference's row is 0/0 throughout, the table's diagonal NaN
    assert np.array_equal(got[~iso], ref[~iso]) and np.isnan(np.diag(got)[iso]).all()
    assert not np.isnan(got[iso][:, ~iso]).any() and int(iso.sum()) == (2 if c["name"] == "isolated" else 0)
    nbr, w, _ = _table(mod)
    assert not ((nbr == np.arange(len(nbr))[:, None]) & (w != 0)).any()


def test_laplacian_self_pair_values():
    """The op-by-op mirror on CPU against the dense oracle (the parent's table gave 4.0933 on the tetrahedron)."""
    for (x, f), want in ((gec.tetra_self_pair(), 4.1930), (gec.fan_self_pair(), 28.4769)):
        mod = jr.LaplacianLoss(torch.from_numpy(x[0]), torch.from_numpy(f))
        got = float(mod(torch.from_numpy(x))[0])
        ref = float(oml.laplacian(x, oml.laplacian_matrix(x.shape[1], f))[0])
        assert abs(ref - want) < 1e-4 and abs(got - ref) <= 1e-5 * ref


@pytest.mark.parametrize("c", LAP, ids=[c["name"] for c in LAP])
def test_laplacian_terms_against_dense_float64(c):
    x = c["vertices"]
    B, nv = x.shape[:2]
    mod = jr.LaplacianLoss(torch.from_numpy(x[0]), torch.from_numpy(c["faces"]))
    nbr, w, dg = _table(mod)
    t32, own32, scat32 = oml.laplacian_terms(x, nbr, w, dg)
    tev, own_ev, scat_ev = oml.laplacian_terms(x, nbr, w, dg, lift=EV)
    _check_terms(t32, tev)
    L = oml.laplacian_matrix(nv, c["faces"])
    with np.errstate(invalid="ignore"):
        y = np.einsum("ij,bjk->bik", L, x.astype(np.float64))
        ref_loss = (y ** 2).sum((1, 2))
        ref_grad = 2 * np.einsum("ij,bik->bjk", L, y)
    # batch elements with an isolated or non-finite vertex: the dense reference is NaN everywhere there, the kernel's
    # terms only where that vertex reaches (narrower pattern, DESIGN.md); left out of the float64 comparison
    poisoned = ~np.isfinite(ref_loss)
    assert int(poisoned.sum()) == {"isolated": 2, "non_finite": 2}.get(c["name"], 0)
    keep = ~poisoned
    with np.errstate(invalid="ignore"):
        tsum = np.nansum(np.where(np.isfinite(t32), 0, 1.0), 1)
    assert np.array_equal(tsum > 0, poisoned)    # every poisoned element has a non-finite term, no other does
    got = t32.astype(np.float64).sum(1)
    err = tev.e.sum(1)
    assert np.all(np.abs(got - ref_loss)[keep] <= (err + 1e-13 * np.abs(ref_loss))[keep])
    # gradient entries
    size = B * nv * 3
    base = np.arange(B)[:, None] * nv
    gsum, gerr, A = np.zeros(size), np.zeros(size), np.zeros(size)
    parts = [(((base + np.arange(nv)) * 3 + cc), own32[cc], own_ev[cc]) for cc in range(3)]
    for k, (rows, t) in enumerate(scat32):
        for cc in range(3):
            parts.append((((base + nbr[rows, k].astype(np.int64)[None]) * 3 + cc), t[cc], scat_ev[k][1][cc]))
    for slots, t, ev in parts:
        _check_terms(t, ev)
        np.add.at(gsum, slots.reshape(-1), np.asarray(t, np.float64).reshape(-1))
        np.add.at(gerr, slots.reshape(-1), ev.e.reshape(-1))
        np.add.at(A, slots.reshape(-1), np.abs(ev.v).reshape(-1))
    gsum, gerr, A = (a.reshape(B, nv, 3) for a in (gsum, gerr, A))
    # the kernel's non-finite entries are a subset of the dense reference's
    assert np.all(~np.isfinite(ref_grad)[~np.isfinite(gsum)])
    m = np.isfinite(ref_grad)
    diff = np.abs(gsum - ref_grad)[m]
    bound = (gerr + 1e-13 * A + 1e-300)[m]
    assert np.all(diff <= bound), (diff / bound).max()
