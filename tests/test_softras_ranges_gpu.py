"""The SoftRas kernels against the oracle on inputs that leave the range of their optimistic divisions.

Under softras_exact_tail = 0 the forward and backward compute every quotient of a (pixel, face) pair without a range
branch and AND the range conditions into one per-pair guard (DivPolicy<false, true>, softras_math.cuh).  When the guard
drops, the pair is re-run through the guarded divisions before anything is committed.  The guard drops

  * for a whole launch when sigma, gamma or far - near is outside [2^-60, 2^61) (DivConst::consts_ok);
  * for the pairs of a face whose vertex z or edge denominator is outside that range (k_face_setup's flag bits);
  * for a single pair whose strict numerator is zero or below 2^-60.

Every case here runs under softras_exact_tail = 0 (optimistic body plus re-run) and 1 (guarded divisions only) against
the oracle, with check()'s tolerances; where the reference's own arithmetic produces NaN or inf, the NaN / inf pattern
must match.  The reachability tests carry no gpu marker: they restate the kernels' range tests in numpy and show, from the
inputs and the oracle's top-K lists, that each case takes its path on at least one shaded pair.
"""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests.test_softras_gpu import GRAD_RTOL, check, same_nonfinite
from tests.util import run_cuda, run_oracle

H = 64   # a power of two: pixel centres (2i + 1 - H) / H are dyadic


def midrange(x):
    """exact_math.cuh midrange(): exponent field in [67, 187], i.e. |x| in [2^-60, 2^61); false for 0, NaN and inf."""
    u = np.asarray(x, np.float32).view(np.uint32)
    with np.errstate(over="ignore"):   # the unsigned wrap-around is the test
        return ((u << np.uint32(1)) - np.uint32(67 << 24)) < np.uint32(121 << 24)


def face_setup_ranges(fv):
    """k_face_setup's range bits (softras_setup.cuh): (z_ok [B,nf,3], den_ok [B,nf,3], den [B,nf,3]).  sym, a0 and den are
    evaluated in float32 in the kernel's order; numpy does not fuse multiply-adds."""
    f = np.asarray(fv, np.float32)
    x, y = f[..., 0], f[..., 1]
    sym = x[..., :, None] * x[..., None, :] + y[..., :, None] * y[..., None, :] + np.float32(1)   # sym[j][k]
    a0 = sym - np.roll(sym, -1, axis=-2)                                                          # sym[k][j] - sym[k+1][j]
    k = np.arange(3)
    den = a0[..., k, k] - a0[..., k, (k + 1) % 3]
    return midrange(f[..., 2]), midrange(den), den


def listed(ref, b, faces):
    """Which of batch element b's faces appear in the oracle's top-K lists, i.e. had at least one pair shaded."""
    ids = ref["faces_id_buffer"][b]
    return np.isin(np.asarray(faces), ids[ids >= 0])


def pixel_centre(i):
    return np.float32((2.0 * i + 1.0 - H) / H)


def edge_parameters(fv, ref):
    """(num, den, face id) of euclidean_p2f_distance's edge parameter num / den (softras_math.cuh) for every edge the
    kernel evaluates on every pair of batch element 0 the oracle listed: all three edges inside the face, the selected
    v0 outside it.  float32, left to right, no fused multiply-add; w from the oracle's faces_info inverse, a0 from its
    sym rows."""
    ids = ref["faces_id_buffer"][0]
    s, row, col = np.nonzero(ids >= 0)
    fn = ids[s, row, col]
    fi = ref["faces_info"][0, fn]
    f = np.asarray(fv, np.float32)[0, fn].reshape(-1, 9)
    xp = ((2.0 * col + 1.0 - H) / H).astype(np.float32)
    yp = ((2.0 * (H - 1 - row) + 1.0 - H) / H).astype(np.float32)
    w = np.stack([fi[:, 3 * k] * xp + fi[:, 3 * k + 1] * yp + fi[:, 3 * k + 2] for k in range(3)], 1)
    sym = fi[:, 9:18].reshape(-1, 3, 3)
    obt = fi[:, 18:21] == 1
    r = np.arange(len(fn))

    def edge(v0):
        v1 = (v0 + 1) % 3
        a = sym[r, v0] - sym[r, v1]
        return w[:, 0] * a[:, 0] + w[:, 1] * a[:, 1] + w[:, 2] * a[:, 2] - a[r, v1], a[r, v0] - a[r, v1]

    def further(p, q):   # (xp - f[p]) . (f[q] - f[p]) > 0, the obtuse-vertex test
        return (xp - f[:, 3 * p]) * (f[:, 3 * q] - f[:, 3 * p]) + (yp - f[:, 3 * p + 1]) * (f[:, 3 * q + 1] - f[:, 3 * p + 1]) > 0

    inside = np.all((w > 0) & (w < 1), 1)
    le = w <= 0
    v0 = np.select([le[:, 1] & le[:, 2], le[:, 2] & le[:, 0], le[:, 0] & le[:, 1], le[:, 0], le[:, 1], le[:, 2]],
                   [np.where(obt[:, 0] & further(0, 2), 2, 0), np.where(obt[:, 1] & further(1, 0), 0, 1),
                    np.where(obt[:, 2] & further(2, 1), 1, 2), 1, 2, 0], 0)
    evals = [(edge(v0), ~inside)] + [(edge(np.full(len(fn), k)), inside) for k in range(3)]
    return tuple(np.concatenate(x) for x in zip(*[(nd[0][m], nd[1][m], fn[m]) for nd, m in evals]))


# ---------------------------------------------------------------------------------------------------------- scenes
def sphere(batch=1):
    return wl.make_scene(280, batch=batch)


def with_faces(fv, tex, extra, seed):
    """fv / tex with the faces `extra` [1, n, 3, 3] appended to batch element 0 (ids nf .. nf + n - 1)."""
    extra = np.asarray(extra, np.float32)
    etex = np.random.default_rng(seed).random((1, extra.shape[1]) + tex.shape[2:], dtype=np.float32)
    return np.concatenate([fv, extra], 1), np.concatenate([tex, etex], 1)


def tiny_z_scene():
    """The sphere plus copies of every 14th face moved in front of it with one, two or three vertex z of 1e-19,
    1e-30, 1e-40 (subnormal) or 0, all below 2^-60 (render with near = 0)."""
    fv, tex = sphere()
    extra = fv[:, ::14].copy()
    for j in range(extra.shape[1]):
        extra[0, j, :1 + j % 3, 2] = (1e-19, 1e-30, 1e-40, 0.0)[j % 4]
    return with_faces(fv, tex, extra, seed=11)


def huge_z_scene():
    """The sphere plus a copy of it at z = 2^62 + q 2^39, q in 0..4 (ulp(2^62) = 2^39); render with near = 2^62 and
    far = 2^62 + 2^41, which keeps far - near in range.  The original sphere is in front of near: its pairs still
    aggregate alpha, then leave at the near test."""
    fv, tex = sphere()
    z = fv[..., 2]
    q = np.round((z - z.min()) / (z.max() - z.min()) * 4.0)
    far_copy = fv.copy()
    far_copy[..., 2] = 2.0 ** 62 + q * 2.0 ** 39
    return with_faces(fv, tex, far_copy, seed=12)


def micro_scene():
    """The sphere plus small faces in front of it, near the image centre, where float32 still resolves their edges:
    twelve with edges of about 1e-10 and twenty-four with edges between 1e-7 and 3e-5.  Their edge denominators,
    differences of sym entries near 1, round to exactly 0.  For the first group the numerators do too (0 / 0); in the
    second some do not, and there the guarded quotient is +-inf while the optimistic one is NaN, which moves the
    clamped edge parameter and with it the distance compared with the threshold."""
    fv, tex = sphere()
    rng = np.random.default_rng(13)
    faces = []
    for j in range(36):
        c = np.float32(rng.uniform(-0.04, 0.04, 2) if j >= 12 else rng.uniform(-2e-3, 2e-3, 2))
        if j < 12:   # float32 spacing is 1.2e-10 at 1e-3
            e = np.float32(rng.uniform(0.5e-10, 2e-10, (2, 2)))
        else:
            e = np.float32(10.0 ** rng.uniform(-7, -4.5, (2, 2)) * rng.choice([-1, 1], (2, 2)))
        v = np.array([c, c + e[0], c + e[1]])
        faces.append(np.concatenate([v, np.full((3, 1), 1.5 + 0.01 * j)], 1))
    return with_faces(fv, tex, np.array(faces)[None], seed=13)


def huge_faces_scene():
    """The sphere plus faces with one, two or three vertices at |x|, |y| of 1e10 .. 1e15 -- where a vertex close to
    the eye plane projects -- whose edges cross the image.  Their Gram-matrix edge denominators are ~|x|^2, beyond 2^61;
    below |x| ~ 1.8e19 the products do not overflow."""
    fv, tex = sphere()
    rng = np.random.default_rng(14)
    faces = []
    for j in range(9):
        n_far = 1 + j % 3
        v = rng.uniform(-0.7, 0.7, (3, 2))
        ang = rng.uniform(0, 2 * np.pi, n_far)
        v[:n_far] = (10.0 ** rng.uniform(10, 15, n_far))[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)
        if n_far == 3:   # keep one edge through the image: opposite far vertices seen from near the centre
            v[1] = -v[0] * rng.uniform(0.5, 2.0) + rng.uniform(-0.5, 0.5, 2)
        faces.append(np.concatenate([v, rng.uniform(1.5, 3.0, (3, 1))], 1))
    return with_faces(fv, tex, np.array(faces)[None], seed=14)


def pixel_aligned_scene():
    """Four faces with every vertex on a pixel centre and twice their area in pixels a power of two, so that w is exact:
    two right triangles at equal depth sharing a 45-degree hypotenuse, a triangle obtuse at its second vertex (the
    inside pixels on the perpendicular through that vertex project onto it: numerator exactly 0) and one with a
    45-degree edge.  Barycentric weights of exactly 0 and 1, zero edge-parameter numerators, depth ties."""
    c = pixel_centre
    faces = [[(c(8), c(8), 2.0), (c(24), c(8), 2.0), (c(24), c(24), 2.0)],
             [(c(8), c(8), 2.0), (c(24), c(24), 2.0), (c(8), c(24), 2.0)],
             [(c(32), c(8), 2.5), (c(48), c(8), 2.5), (c(56), c(24), 3.0)],
             [(c(20), c(40), 1.5), (c(36), c(56), 1.5), (c(20), c(56), 2.0)]]
    fv = np.array(faces, np.float32)[None]
    return fv, np.random.default_rng(15).random((1, 4, 1, 3), dtype=np.float32)


def non_finite_scene():
    """Batch element 1: the sphere, a face with a NaN vertex x and a face with an infinite vertex z, both over the
    sphere.  Batch element 0 (and the clean copy returned second): the sphere with two faces off screen in their place."""
    fv, tex = sphere(batch=2)
    tri = np.array([[-0.2, -0.15, 1.8], [0.2, -0.1, 1.8], [0.0, 0.25, 1.9]], np.float32)
    off = tri + np.float32([5.0, 5.0, 0.0])
    nan_face, inf_face = tri.copy(), tri + np.float32([0.1, 0.1, 0.0])
    nan_face[0, 0] = np.nan
    inf_face[1, 2] = np.inf
    clean = np.concatenate([fv, np.broadcast_to(np.stack([off, off])[None], (2, 2, 3, 3))], 1)
    bad = clean.copy()
    bad[1, 280], bad[1, 281] = nan_face, inf_face
    tex = np.concatenate([tex, np.random.default_rng(16).random((2, 2, 1, 3), dtype=np.float32)], 1)
    return bad, clean, tex


# ----------------------------------------------------------------------------------------------------------- cases
# name: (scene, params, which path the case reaches, depth case: also run with hard rgb)
CASES = {
    "sigma_2^-62": (sphere, dict(sigma_val=2.0 ** -62), "launch", False),
    "sigma_2^62": (sphere, dict(sigma_val=2.0 ** 62), "launch", False),
    # subnormal: rcp.approx.ftz flushes it, so the optimistic quotients by sigma would all be NaN
    "sigma_1e-39": (sphere, dict(sigma_val=1e-39), "launch", False),
    "gamma_2^-62": (sphere, dict(gamma_val=2.0 ** -62), "launch", False),
    "gamma_2^62": (sphere, dict(gamma_val=2.0 ** 62), "launch", False),
    "far_2^62": (sphere, dict(far=2.0 ** 62), "launch", True),
    # far - near = 2^127, whose reciprocal is subnormal: the optimistic quotients by it would all be 0.  With eps = 0
    # the true zp_norm = (far - zp) / 2^127, about 6e-37, becomes softmax_max
    "near_-2^127": (sphere, dict(near=-2.0 ** 127, eps=0.0), "launch", False),
    "z_below_2^-60": (tiny_z_scene, dict(near=0.0), "z", True),
    "z_2^62": (huge_z_scene, dict(near=2.0 ** 62, far=2.0 ** 62 + 2.0 ** 41), "z", True),
    "micro_faces": (micro_scene, dict(sigma_val=1e-4), "den", False),
    "huge_faces": (huge_faces_scene, dict(), "den", False),
    "pixel_aligned": (pixel_aligned_scene, dict(sigma_val=1e-4), "num", True),
}
DISTS = ("euclidean", "barycentric")


def params(name, dist, rgb="softmax"):
    return osr.Params(image_size=H, dist_func=dist, aggr_func_rgb=rgb, aggr_func_alpha="prod", **CASES[name][1])


def applies(name, dist):
    """The edge parameter (den, num) exists in euclidean mode only; launch constants and depths reach both modes."""
    return dist == "euclidean" or CASES[name][2] in ("launch", "z")


# ----------------------------------------------------------------------------------------------- reachability (CPU)
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dist", DISTS)
def test_case_reaches_its_path(name, dist):
    if not applies(name, dist):
        pytest.skip("no edge parameter outside euclidean mode")
    scene, kw, path, _ = CASES[name]
    fv, tex = scene()
    P = params(name, dist)
    ref = run_oracle(fv, tex, P)
    assert (ref["faces_id_buffer"] >= 0).any(), "no pair shaded"
    if path == "launch":
        # DivConst::consts_ok() is false: every pair of the launch re-runs
        near, far, _, sigma, _, _, gamma = P.scalars()[:7]
        assert not (midrange(sigma) and midrange(gamma) and midrange(far - near))
        return
    z_ok, den_ok, den = face_setup_ranges(fv)
    if path == "z":
        out = np.nonzero(~z_ok[0].all(-1))[0]
        assert midrange(np.float32(P["far"]) - np.float32(P["near"]))
        assert listed(ref, 0, out).any(), "no face with a z outside the range was shaded"
        # and faces in range are shaded beside them
        assert listed(ref, 0, np.nonzero(z_ok[0].all(-1))[0]).any() or P["near"] > 1.0
    elif path == "den":
        out = np.nonzero(~den_ok[0].all(-1))[0]
        assert listed(ref, 0, out).any(), "no face with an edge denominator outside the range was shaded"
        num, d, fn = edge_parameters(fv, ref)
        assert (~midrange(d)).any(), "no shaded pair evaluates an edge with an out-of-range denominator"
        if name == "micro_faces":
            assert np.any(d == 0), "den is recomputed, not assumed: no shaded pair has den == 0"
            # num / +0 is +-inf through the guarded division, NaN through the optimistic one
            assert np.any((d == 0) & (num != 0))
    else:
        num, _, _ = edge_parameters(fv, ref)
        assert np.any((num == 0) | (np.abs(num) < 2.0 ** -60)), "no shaded pair with a zero / tiny numerator"


def test_non_finite_faces_reach_the_guarded_path():
    bad, _, tex = non_finite_scene()
    z_ok, den_ok, _ = face_setup_ranges(bad)
    assert not z_ok[1, 281].all() and not den_ok[1, 280].all()
    for dist in DISTS:
        ref = run_oracle(bad, tex, osr.Params(image_size=H, dist_func=dist, sigma_val=1e-4))
        assert listed(ref, 1, [280, 281]).all()


def test_midrange_restates_the_kernel_bounds():
    x = np.float32([2.0 ** -60, 2.0 ** 61 * (1 - 2.0 ** -24), -2.0 ** -60, 2.0 ** 61, np.nextafter(np.float32(2.0 ** -60), 0),
                    0.0, -0.0, np.inf, np.nan, 1e-40, 1.0])
    assert midrange(x).tolist() == [True, True, True, False, False, False, False, False, False, False, True]


# ------------------------------------------------------------------------------------------------------ GPU parity
def both_tails(fv, tex, P, **kw):
    """check() under softras_exact_tail = 0 (optimistic body + re-run) and 1 (guarded divisions only)."""
    from jrender_b200 import _lib
    try:
        for tail in (0, 1):
            _lib.set_option("softras_exact_tail", tail)
            check(fv, tex, P, nan=True, **kw)
    finally:
        _lib.set_option("softras_exact_tail", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name,dist,rgb", [(n, d, r) for n in CASES for d in DISTS for r in ("softmax", "hard")
                                           if r == "softmax" or CASES[n][3]])
def test_out_of_range_inputs_match_oracle(cuda_device, name, dist, rgb):
    fv, tex = CASES[name][0]()
    both_tails(fv, tex, params(name, dist, rgb))


@pytest.mark.gpu
@pytest.mark.parametrize("dist", DISTS)
def test_non_finite_vertices_stay_in_their_batch_element(cuda_device, dist):
    """NaN / inf vertices in batch element 1 must not fault, must not touch element 0 (forward bit-identical to a run
    without them, gradients within the gradient tolerance), and element 1 must match the oracle, NaN pattern included."""
    from jrender_b200 import _lib
    bad, clean, tex = non_finite_scene()
    P = osr.Params(image_size=H, dist_func=dist, sigma_val=1e-4)
    g = np.random.default_rng(7).uniform(-1, 1, (2, 4, H, H)).astype(np.float32)
    try:
        for tail in (0, 1):
            _lib.set_option("softras_exact_tail", tail)
            check(bad, tex, P, nan=True)
            got, base = run_cuda(bad, tex, P, grad=g), run_cuda(clean, tex, P, grad=g)
            for k in ("soft_colors", "aggrs_info", "faces_id_buffer", "faces_info"):
                assert np.array_equal(got[k][0], base[k][0]), k
            for k in ("grad_faces", "grad_textures"):
                a, b = got[k][0], base[k][0]
                m = same_nonfinite(a, b, k)
                assert np.abs(a[m] - b[m]).max() <= GRAD_RTOL * np.abs(b[m]).max(), k
    finally:
        _lib.set_option("softras_exact_tail", 0)
