"""GPU parity of the fused surface lighting (b200r_surface_lighting_*, one normal per face) and the normal-mapped
lighting (b200r_normal_mapped_lighting_*, one normal per texel) on the scenes of tests/lighting_edge_cases.py: texel
counts around the warp width, shared geometry and materials across the batch, slivers, degenerate faces, the relu,
normalize and clamp edges (clamp_min's equality included), non-finite inputs, a vertex in a thousand faces and the demo
1.5 head's size.

Tolerances.  Against oracle/lighting.py, the float32 emulation of the kernels (hold_to_emulation, on every kernel call
the kernel_calls fixture records): lit textures and every per-texel gradient (textures, normal textures, metallic,
roughness) bit for bit, with the same NaN / +-inf pattern; each grad_vertices entry within term_sums' bound of the exact
sum of the emulated terms, gamma_{n-1} sum |t| for its n float atomics (oracle/preraster.py).  The emulation itself is
held to float64 autograd entry by entry in tests/test_lighting_edges_cpu.py.  Coarser, end to end: lit textures against
the op-by-op float32 mirror within 2e-5, with the same NaN / +-inf pattern; at millions of texels two allowances come
in: twice the mirror's own distance from its float64 run, and on the Cook-Torrance branch 16 eps32 / roughness^4
(ggx_bound: GGX's sensitivity to N.H times a few ulps of N.H; 1.2e-3 at roughness 0.2, 2.9e-6 at roughness 1).  Every
gradient the kernel writes against the float64 mirror's autograd within 1e-4 of that gradient's max |finite value|,
with the same non-finite pattern.  A non-finite input changes nothing outside its face and batch element: those outputs
and per-texel gradients are bit-identical to the scene without it, the vertex gradients equal up to the float atomics'
summation order (1e-6 of max).
"""
import numpy as np
import pytest
import torch

from jrender_b200 import _lib
from oracle import lighting as OL
from oracle.preraster import term_sums
from tests import lighting_edge_cases as E

pytestmark = pytest.mark.gpu
OUT_TOL = 2e-5
GRAD_TOL = 1e-4
ATOMIC_TOL = 1e-6


@pytest.fixture
def kernel_calls(monkeypatch):
    """Every call of the four lighting entry points made while the test runs, as (name, the kernel's arguments and
    outputs after the call: oracle.lighting.args_from_call)."""
    calls = []
    real = _lib.call

    def record(name, device, *args):
        real(name, device, *args)
        if name in OL.CALLS:
            torch.cuda.synchronize(device)
            calls.append((name, OL.args_from_call(name, args)))
    monkeypatch.setattr(_lib, "call", record)
    return calls


def _same_bits(got, want, what):
    """Equal values with the same NaN / +-inf pattern (signed zeros compare equal)."""
    got, want = np.asarray(got), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), "%s: %d of %d entries differ from the emulation, first at %s (%r vs %r)" % (
        what, bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0])


def hold_to_emulation(calls):
    """Each recorded kernel call against oracle.lighting's float32 emulation of it: lit textures and every per-texel
    gradient bit for bit; each grad_vertices entry within term_sums' order-independent bound of the exact sum of the
    emulated terms (same NaN / +-inf pattern where that sum is not finite).  Returns the worst |error| / bound."""
    assert calls, "no lighting kernel ran"
    worst = 0.0
    for name, a in calls:
        nm = name in OL.NM_PTRS
        if name.endswith("_forward"):
            _same_bits(a["out"], (OL.nm_forward if nm else OL.surface_forward)(a), name + " lit textures")
            continue
        emu = (OL.nm_backward if nm else OL.surface_backward)(a)
        for k in ("textures", "normal_textures", "metallic", "roughness"):
            if a.get("grad_" + k) is not None:
                _same_bits(a["grad_" + k], emu[k], "%s grad_%s" % (name, k))
        gv = a.get("grad_vertices")
        if gv is None:
            continue
        t = np.asarray(emu["vertex_terms"], np.float32).reshape(-1)
        sl = np.asarray(emu["vertex_slots"]).reshape(-1)
        live = t != 0   # the kernels skip zero terms
        s = term_sums(sl[live], t[live], gv.size)
        got = gv.reshape(-1).astype(np.float64)
        fin = np.isfinite(s["exact"])
        _same_bits(np.where(fin, 0, got).astype(np.float32), np.where(fin, 0, s["exact"]).astype(np.float32),
                   name + " grad_vertices non-finite entries")
        err = np.abs(got - s["exact"])[fin]
        assert (err <= s["bound"][fin]).all(), (name, "grad_vertices", (err / np.maximum(s["bound"][fin], 1e-300)).max())
        worst = max(worst, float((err / np.maximum(s["bound"][fin], 1e-300)).max(initial=0.0)))
    print("grad_vertices: worst |kernel - exact sum of emulated terms| / bound = %.3g" % worst)
    return worst


def same_nonfinite(a, b, what):
    """NaN, +inf and -inf in the same places of a and b; returns the mask of b's finite entries."""
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s NaN pattern differs" % what
    assert np.array_equal(np.isposinf(a), np.isposinf(b)) and np.array_equal(np.isneginf(a), np.isneginf(b)), what
    return np.isfinite(b)


def ggx_bound(sc, shape):
    """16 eps32 / a per texel, a = roughness^4 (GGX's a^2): near N.H = 1 the relative sensitivity of GGX to N.H is up
    to 4 / a, and N.H carries a few float32 roundings (the texel normal's product and normalize, H's normalize) that the
    kernels and the mirror make in different orders.  Count 4 ulps."""
    r = sc["rou"].astype(np.float64)
    if "nt" not in sc:   # the flat path uses the face's mean roughness
        r = r.reshape(r.shape[:2] + (-1,)).mean(axis=2).reshape(r.shape[:2] + (1,) * (len(shape) - 2))
    return np.broadcast_to(16 * np.finfo(np.float32).eps / r ** 4, shape)


def check(dev, sc, calls):
    """The fused kernels against their emulation (hold_to_emulation, on the calls recorded by the kernel_calls fixture),
    and, coarsely, against the float32 mirror (lit textures) and the float64 mirror (gradients); returns the fused
    (out, grads) and the float64 gradients."""
    del calls[:]
    out, got = E.run(sc, dev, torch.float32, True)
    assert {n for n, _ in calls} == {n for n in OL.CALLS if ("normal" in n) == ("nt" in sc)}
    hold_to_emulation(calls)
    out32, _ = E.run(sc, dev, torch.float32, False, grads=False)
    out64, ref = E.run(sc, dev, torch.float64, False)
    m = same_nonfinite(out, out32, "lit textures")
    same_nonfinite(out, out64, "lit textures (float64)")
    bound = np.maximum(OUT_TOL, 2 * np.abs(out32 - out64))
    if sc["eye"] is not None:
        bound = np.maximum(bound, ggx_bound(sc, out.shape))
    assert (np.abs(out[m] - out32[m]) <= bound[m]).all(), np.abs(out[m] - out32[m]).max()
    for name, b in ref.items():
        a = got[name]
        if b is None:   # no path from this input in the mirror: the kernel writes nothing or exact zeros
            assert a is None or not a.any(), name
            continue
        m = same_nonfinite(a, b, name)
        scale = np.abs(b[m]).max()
        assert scale > 0, name
        err = np.abs(a[m] - b[m]).max() / scale
        assert err <= GRAD_TOL, (name, err)
    return out, got, ref


@pytest.mark.parametrize("T,Tm", [(1, 1), (25, 1), (25, 25), (125, 1), (125, 125)])
def test_flat_texel_counts(cuda_device, kernel_calls, T, Tm):
    check(cuda_device, E.flat_shapes(T, Tm), kernel_calls)


@pytest.mark.parametrize("Be", [0, 1, 4])
@pytest.mark.parametrize("Tm", [1, 9])
def test_flat_shared_geometry(cuda_device, kernel_calls, Be, Tm):
    """One mesh (vertices and faces batch 1) lit for four texture sets and eyes: every batch element's vertex
    gradient lands in the one row."""
    sc = E.flat_shapes(9, Tm, B=4, Bv=1, Be=Be)
    _, got, ref = check(cuda_device, sc, kernel_calls)
    assert got["vertices"].shape[0] == 1


def test_flat_geometry_edges(cuda_device, kernel_calls):
    """Slivers down to aspect 1e-5, collinear and coincident-vertex faces, faces edge-on to the light, V and H on
    normalize's eps path, texels exactly on the clamp bounds; one mesh for four eyes."""
    sc = E.flat_geometry()
    out, got, ref = check(cuda_device, sc, kernel_calls)
    g = got["vertices"][0]
    for k in ("collinear", "coincident"):   # N = 0: every relu at its kink, no gradient through the normal
        face = sc["f"][sc[k]]
        assert np.isfinite(g[face]).all()
    u = sc["unlit"]
    # the clamp passes the gradient at 0 and 1: d out / d tex = diffuse on those texels
    want = (sc["gout"][:, u, :2] * E.UNLIT_DIFFUSE).astype(np.float32)
    assert np.array_equal(got["textures"][:, u, :2], want)
    sl = sc["f"][sc["slivers"]].ravel()
    assert np.abs(ref["vertices"][0][sl]).max() == np.abs(ref["vertices"]).max()   # the slivers set max |grad|


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 225])
@pytest.mark.parametrize("Bn,Bt", [(1, 1), (3, 3), (1, 3), (3, 1)])
def test_nm_texel_counts(cuda_device, kernel_calls, T, Bn, Bt):
    if T in (1, 225) and (Bn, Bt) in ((1, 3), (3, 1)):
        pytest.skip("mixed batches run at the middle texel counts")
    check(cuda_device, E.nm_shapes(T, Bn, Bt), kernel_calls)


@pytest.mark.parametrize("Be", [0, 1, 4])
@pytest.mark.parametrize("per_face_material", [False, True])
def test_nm_shared_geometry(cuda_device, kernel_calls, Be, per_face_material):
    """One mesh and one normal texture for four texture sets and eyes; per-face materials broadcast over the texels."""
    sc = E.nm_shapes(33, 1, 1, B=4, Bv=1, Be=Be, per_face_material=per_face_material)
    _, got, _ = check(cuda_device, sc, kernel_calls)
    assert got["normal_textures"].shape[0] == 1


def test_nm_clamp_bounds(cuda_device, kernel_calls):
    sc = E.nm_clamp_bounds()
    _, got, _ = check(cuda_device, sc, kernel_calls)
    b, f, t = sc["bounds"]
    assert np.array_equal(got["textures"][b, f, t], (sc["gout"][b, f, t] * E.UNLIT_DIFFUSE).astype(np.float32))


CASES = [(nm, site, value) for nm in (False, True) for site in (E.NM_SITES if nm else E.FLAT_SITES)
         for value in (("nan",) if site == "tbn" else sorted(E.NONFINITE))]


@pytest.mark.parametrize("nm,site,value", CASES)
def test_nonfinite_input_follows_the_mirror_and_stays_in_its_face(cuda_device, kernel_calls, nm, site, value):
    clean, dirty, (b, fa) = E.nonfinite(site, E.NONFINITE[value], nm=nm)
    out, got, _ = check(cuda_device, dirty, kernel_calls)
    out0, got0 = E.run(clean, cuda_device, torch.float32, True)
    keep = np.ones(out.shape[:2], bool)
    keep[b, fa] = False
    assert np.array_equal(out[keep], out0[keep])
    for name in got:
        a, a0 = got[name], got0[name]
        if name == "vertices":
            mine = np.zeros(a.shape[:2], bool)
            mine[b, dirty["f"][fa]] = True
            assert np.isfinite(a[~mine]).all()
            assert np.abs(a[~mine] - a0[~mine]).max() <= ATOMIC_TOL * np.abs(a0).max()
        elif name == "normal_textures" or a.shape[0] == out.shape[0]:
            assert np.array_equal(a[keep], a0[keep]), name


def test_head_sized_normal_map(cuda_device, kernel_calls):
    """The demo 1.5 head's size: 66 282 faces, T = 225 (every lane of the backward takes 7 or 8 texels), all five
    gradients against the float64 mirror."""
    check(cuda_device, E.head(), kernel_calls)


@pytest.mark.parametrize("spec", [True, False])
@pytest.mark.parametrize("nm", [False, True])
def test_clamp_min_passes_at_equality(cuda_device, kernel_calls, nm, spec):
    """|V| == 1e-12f, |H| == 1e-12f, den4 == 0.01f and (normal map) a texel normal of norm exactly 1e-12f: torch's
    clamp_min passes the gradient at equality, and so must the kernels (bit for bit against the emulation, which follows
    that rule; the float64 mirror does not land on these equalities)."""
    sc = E.equality(nm, spec)
    del kernel_calls[:]
    E.run(sc, cuda_device, torch.float32, True)
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("nm", [False, True])
def test_vertex_shared_by_a_thousand_faces(cuda_device, kernel_calls, nm):
    """One apex in 1000 faces, one mesh for four eyes: its grad_vertices entries sum thousands of atomics."""
    check(cuda_device, E.shared_vertex(nm=nm), kernel_calls)
