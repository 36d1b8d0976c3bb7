"""The NMR (dr_type='n3mr') kernels against the CPU oracle at their seams, with per-element gradient bounds.

Scenes (tests/nmr_edge_cases.py; tests/test_nmr_edges_cpu.py asserts each reaches its target path):
long inward scans (the warp-wide OWNER scan, spans 63 / 64 / 65 and hundreds), outward scans of n = 1 .. 97 pixels
toward every border in both flavours, the past-the-end lanes of a scan toward pixel 0 whose dist cancels to exactly 0,
pixel-aligned vertices, image sizes 1, 2, 31, 33 and 4096, negative / mixed-sign / tied / signed-zero depths,
colours that cancel in diff_grad, and partly off-screen faces.  Each runs with rgb, alpha and rgb + alpha (K9's MODE
1, 2, 3), with and without the depth output.

Forward: every map is bit-exact, as in tests/test_nmr_gpu.py.

Gradients are held per face and per slot against oracle.nmr.backward_stats (u = 2^-24):

K9.  The kernel's term for one visited pixel is d_k * rcp(dist_k), the reference's is fl(diff / dist).
  * diff.  The kernel forms A = sum_k map_k g_k (k_nmr_pack, <= 4 FMAs) and then A - sum_k ref_k g_k (k9_diff,
    <= 4 FMAs, in every scan): <= 8 roundings, each below u * S with
    S = sum_k |map_k g_k| + |ref_k g_k|.  The reference rounds (map - ref), the product and <= 3 partial sums: <= 5 u S.
    So |d_k - diff| <= 13 u S, also where one side is <= 0 and its term is skipped.  Summed over the visited pixels
    this is 13 u R, with R = sum S / |dist| (the scale 1 / |dist_k| differs from 1 / |dist| by O(u));
    a = 16 leaves room for that.
  * dist.  Both sides approximate D = (d1 - d1_cross) (p10 - p00) / (p10 - d0) * 2 / is + -eps without cancellation
    (delta * k has eps's sign for every pixel a scan evaluates).  Kernel: span, p10 - d0, rcp.approx (2 u), two
    products, 2 / is, delta (1 rounding; in k9_scan_out at most one rounding per binade that `delta += 64` crosses,
    a geometric series below 4 u, plus one for the `b` half's + 32), delta * k and + eps: <= 15 u; then rcp.approx of
    dist: 2 u.  Reference: span, p10 - d0, the quotient, delta, the product, the cast after * 2 / is, + eps: <= 7 u,
    and the division: u.  So |term_k - term| <= 25 u |term| + 13 u S / |dist|; b = 32.
  * Summation.  A term goes through at most N float additions: its lane's running sums (the pixels of the slot that
    lane visits), <= 3 per 32-sample group into the lane's six slot sums, and the 5-level warp tree
    (k9_chain, computed by the oracle from the kernel's lane assignment).  Each adds u times a partial sum <= T.
  |got - g64| <= u (16 R + (32 + N) T)  with  g64, T = sum |term|, R, N per slot.
K11 adds its terms -- bit-identical to the oracle's: same expression, IEEE division -- by atomics onto K9's result:
  n11 roundings, each u times a partial sum <= T9 + e9 + T11 (e9 the K9 bound above).
K10 (per texel channel): bit-identical terms w * g added by atomics onto 0: |got - g64| <= u n10 T10.
Where the oracle's float result is NaN the kernel's must be NaN too.  The worst ratio to each bound is printed.
"""
import numpy as np
import pytest

from oracle import nmr as onmr
from tests import nmr_edge_cases as E
from tests.util import run_nmr_cuda

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
A_R, B_T = 16.0, 32.0

MODES = {"rgb": (True, False), "alpha": (False, True), "rgba": (True, True)}


def _held(name, got, ref_f32, g64, bound):
    """NaN where the float oracle has NaN, |got - g64| <= bound elsewhere; -> worst ratio."""
    nan = np.isnan(ref_f32)
    assert np.array_equal(np.isnan(got), nan), (name, "NaN pattern", np.argwhere(np.isnan(got) != nan)[:5])
    got, g64, bound = got[~nan].astype(np.float64), g64[~nan], bound[~nan]
    err = np.abs(got - g64)
    bad = err > bound
    assert not bad.any(), (name, np.argwhere(bad)[:5], got[bad][:5], g64[bad][:5], bound[bad][:5])
    return float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0


def check(faces, tex, H, mode, depth, eps=1e-3, near=0.1, far=100.0, bg=(0, 0, 0), seed=0):
    rgb, alpha = MODES[mode]
    flags = (rgb, alpha, depth)
    ref = onmr.forward(faces, tex if rgb else None, H, near, far, eps, bg, *flags)
    B = faces.shape[0]
    rng = np.random.default_rng(seed)
    g = (rng.uniform(-1, 1, (B, H, H, 3)).astype(np.float32), rng.uniform(-1, 1, (B, H, H)).astype(np.float32),
         rng.uniform(-1, 1, (B, H, H)).astype(np.float32))
    st = onmr.backward_stats(faces, tex if rgb else None, ref, H, eps, g[0], g[1], g[2], *flags)
    got = run_nmr_cuda(faces, tex, H, near, far, eps, bg, flags, grads=g)
    for k in ("face_index_map", "weight_map", "depth_map") + (("rgb_map", "sampling_index_map", "sampling_weight_map") if rgb else ()):
        assert np.array_equal(got[k], ref[k]), k
    if alpha:
        assert np.array_equal(got["alpha_map"], ref["alpha_map"])
    if depth:
        assert np.array_equal(got["face_inv_map"].reshape(ref["face_inv_map"].shape), ref["face_inv_map"])
    with np.errstate(invalid="ignore", over="ignore"):
        T9, R9, N9 = st["k9_T"], st["k9_R"], st["k9_chain"].astype(np.float64)
        e9 = U * (A_R * R9 + (B_T + N9) * T9)
        e11 = U * st["k11_cnt"] * (T9 + e9 + st["k11_T"])
        worst = {"faces": _held("grad_faces", got["grad_faces"], st["grad_faces"], st["k9_g64"] + st["k11_g64"], e9 + e11)}
        if rgb:
            worst["textures"] = _held("grad_textures", got["grad_textures"], st["grad_textures"], st["k10_g64"],
                                      U * st["k10_cnt"] * st["k10_T"])
    print("bound ratio %s" % " ".join("%s %.3g" % kv for kv in worst.items()))
    return ref, got, st


def _modes():
    return [pytest.param(m, d, id="%s-%s" % (m, "depth" if d else "nodepth")) for m in MODES for d in (False, True)]


@pytest.mark.parametrize("mode,depth", _modes())
def test_long_inward_scans(cuda_device, mode, depth):
    faces = E.long_inward()
    _, _, st = check(faces, E.textures(faces, seed=1), 256, mode, depth, seed=1)
    assert st["k9_cnt"].max() > 200


@pytest.mark.parametrize("mode,depth", _modes())
def test_outward_trip_seams(cuda_device, mode, depth):
    faces = E.outward_seams()
    check(faces, E.textures(faces, seed=2), 256, mode, depth, seed=2)


@pytest.mark.parametrize("mode,depth", _modes())
def test_past_end_lanes_toward_zero(cuda_device, mode, depth):
    """The lanes past the end of a scan toward pixel 0 sit across the crossing; with eps = 2^-10 the first of them has
    fma(delta, k, e) == 0 exactly.  The oracle's gradients are finite there, and so must the kernel's be."""
    faces = E.past_end()
    ref, got, st = check(faces, E.textures(faces, seed=3), 256, mode, depth, eps=E.PAST_END_EPS, seed=3)
    assert np.isfinite(st["grad_faces"]).all() and np.isfinite(got["grad_faces"]).all()


@pytest.mark.parametrize("mode,depth", _modes())
def test_pixel_aligned_vertices(cuda_device, mode, depth):
    faces = E.pixel_aligned()
    check(faces, E.textures(faces, seed=4), 64, mode, depth, seed=4)


@pytest.mark.parametrize("is_", [1, 2, 31, 33])
@pytest.mark.parametrize("mode,depth", _modes())
def test_small_image_sizes(cuda_device, is_, mode, depth):
    faces = E.tiny(is_)
    check(faces, E.textures(faces, ts=3, seed=5), is_, mode, depth, seed=5)


@pytest.mark.parametrize("mode,depth", [pytest.param("rgba", True, id="rgba-depth"), pytest.param("alpha", False, id="alpha-nodepth")])
def test_image_size_4096(cuda_device, mode, depth):
    """The ABI's largest image: 32-bit per-image offsets at is^2 * FL = 2^27 floats, scans of ~4000 pixels."""
    faces = E.huge()
    ref, _, st = check(faces, E.textures(faces, seed=6), 4096, mode, depth, seed=6)
    assert (ref["face_index_map"] >= 0).mean() > 0.3 and st["k9_cnt"].max() > 3000


@pytest.mark.parametrize("mode,depth", _modes())
def test_depth_order_signs_ties_and_signed_zero(cuda_device, mode, depth):
    """near < 0: negative depths win over positive ones, duplicates tie to the lower id, and a +0 / -0 depth tie goes
    to the lower id in both orders (the oracle's `zp < depth` does not order -0 before +0)."""
    faces = E.depth_order()
    ref, got, _ = check(faces, E.textures(faces, seed=7), 64, mode, depth, near=E.DEPTH_NEAR, far=E.DEPTH_FAR, seed=7)
    fim, d = ref["face_index_map"], ref["depth_map"]
    assert (d[0] < 0).any() and (d[0] > 0).any()
    assert (fim[1] == 0).any() and not (fim[1] == 1).any()                       # duplicates: id 0 keeps every pixel
    assert (fim[1] == 2).any() and not (fim[1] == 3).any()                       # +0 (id 2) before -0 (id 3)
    assert (fim[1] == 4).any() and not (fim[1] == 5).any()                       # -0 (id 4) before +0 (id 5)
    assert np.signbit(d[1][fim[1] == 4]).all() and not np.signbit(d[1][fim[1] == 2]).any()


@pytest.mark.parametrize("per_batch", [False, True], ids=["bg", "bg_per_batch"])
@pytest.mark.parametrize("mode,depth", _modes())
def test_cancelling_colours(cuda_device, mode, depth, per_batch):
    """Constant textures over a background of the same colour: most reference diffs are exactly 0 and the kernel's
    A - sum ref * grad leaves a rounding residual, which the R term bounds.  A [B, 3] background goes through the
    torch mixing path of n3mr.py."""
    faces = E.long_inward()
    cols = np.array([[0.3, 0.55, 0.8], [0.7, 0.1, 0.45]], np.float32)
    tex = np.concatenate([E.textures(faces[:1], const=cols[0]), E.textures(faces[1:], const=cols[1])])
    if not per_batch:
        tex[1] = cols[0]
    bg = cols if per_batch else tuple(float(c) for c in cols[0])
    ref, _, st = check(faces, tex, 256, mode, depth, bg=bg, seed=8)
    if mode == "rgb":   # the reference's terms nearly vanish next to the scale of the kernel's residual
        assert st["k9_R"].sum() > 0 and st["k9_T"].sum() <= 1e-4 * st["k9_R"].sum()


@pytest.mark.parametrize("mode,depth", _modes())
def test_partly_off_screen(cuda_device, mode, depth):
    faces = E.off_screen()
    check(faces, E.textures(faces, seed=9), 128, mode, depth, seed=9)
