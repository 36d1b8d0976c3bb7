"""The SoftRas forward's reach cull is conservative: every (pixel, face) pair it drops is one the per-pair body leaves.

The euclidean forward drops a pair before the per-pair body when k_face_setup gave the face a margin
(softras_setup.cuh reach_margin_q) and the pixel lies outside the face's reach polygon (softras_forward.cuh
reach_lane_mask); DESIGN.md section 4.4 derives why that is safe.  Here both are restated in numpy -- the setup in
float32 and double exactly as k_face_setup evaluates them, the mask in float32 in the kernel's order -- and so is the
body's exit test (sign < 0 and dis >= threshold, euclidean_p2f_distance in float32, no fused multiply-adds).  The
restated exit is first held to the oracle itself, face by face; then over more than 10^7 (face, pixel) pairs of the
C3 and C2 spheres, random triangles, needles and slivers at the gate's conditioning bound, vertices on pixel centres,
huge, tiny and non-finite coordinates, no dropped pair may be one the body would shade.  The mask's two approximate
operations (rsqrtf, __fdividef) are taken at both ends of their error range, and a pair counts as dropped when either
end drops it.
"""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests import test_softras_ranges_gpu as rng_cases
from tests.test_softras_reach_cull_gpu import SCENES

F = np.float32
U = 2.0 ** -24


def pix(i, H):
    return ((2.0 * np.asarray(i, np.float64) + 1.0 - H) / H).astype(F)


def border_of(P):
    thr = F(osr.dist_eps_logit(P["dist_eps"]) * F(P["sigma_val"]))
    return thr, F(np.sqrt(thr))


# ------------------------------------------------------------------------------------------------ k_face_setup
def face_setup(fv, H, border):
    """Per face: inv [n, 9] f32, rect (x0, x1, r0, r1) [n, 4] (empty rect as (1, 0, 1, 0)) and the margin field q."""
    f = np.asarray(fv, F).reshape(-1, 9)
    p00, p01, p10, p11, p20, p21 = f[:, 0], f[:, 1], f[:, 3], f[:, 4], f[:, 6], f[:, 7]
    with np.errstate(all="ignore"):
        star = np.stack([p11 - p21, p20 - p10, p10 * p21 - p20 * p11, p21 - p01, p00 - p20, p20 * p01 - p00 * p21,
                         p01 - p11, p10 - p00, p00 * p11 - p10 * p01], 1)
        det = p20 * (p01 - p11) + p00 * (p11 - p21) + p10 * (p21 - p01)
        det = np.where(det > 0, np.maximum(det, F(1e-10)), np.minimum(det, F(-1e-10)))
        inv = (star / det[:, None]).astype(F)
        z_ok, den_ok, _ = rng_cases.face_setup_ranges(f.reshape(-1, 3, 3))
        bits_ok = z_ok.all(1) & den_ok.all(1) & np.isfinite(inv).all(1)
        # check_border as a pixel rectangle: the pixels whose centre is inside [min - border, max + border]
        x, y = f[:, 0::3], f[:, 1::3]
        xlo, xhi = x.min(1) - border, x.max(1) + border
        ylo, yhi = y.min(1) - border, y.max(1) + border
    c = pix(np.arange(H), H)
    x0 = np.searchsorted(c, xlo, "left")
    x1 = np.searchsorted(c, xhi, "right") - 1
    y0 = np.searchsorted(c, ylo, "left")
    y1 = np.searchsorted(c, yhi, "right") - 1
    for a, lo in ((x0, xlo), (y0, ylo)):   # NaN: nothing rejected
        a[np.isnan(lo)] = 0
    for a, hi in ((x1, xhi), (y1, yhi)):
        a[np.isnan(hi)] = H - 1
    r0, r1 = H - 1 - y1, H - 1 - y0
    empty = (x0 > x1) | (r0 > r1)
    rect = np.stack([x0, x1, r0, r1], 1)
    rect[empty] = (1, 0, 1, 0)
    q = np.zeros(len(f), np.int64)
    for i in np.nonzero(bits_ok & ~empty)[0]:
        x0_, x1_, r0_, r1_ = rect[i]
        q[i] = reach_margin_q(f[i], inv[i], float(pix(x0_, H)), float(pix(x1_, H)), float(pix(H - 1 - r1_, H)),
                              float(pix(H - 1 - r0_, H)), H)
    return inv, rect, q


def reach_margin_q(f, inv, xlo, xhi, ylo, yhi, H):
    """softras_setup.cuh reach_margin_q, line by line."""
    f = f.astype(np.float64)
    inv = inv.astype(np.float64)
    g3, g4 = 3 * U / (1 - 3 * U), 4 * U / (1 - 4 * U)
    if not np.isfinite(f[[0, 1, 3, 4, 6, 7]]).all() or not np.isfinite(inv).all():
        return 0
    M = np.abs(f[[0, 1, 3, 4, 6, 7]]).max()
    Lmax2 = max((f[3 * k1] - f[3 * k]) ** 2 + (f[3 * k1 + 1] - f[3 * k + 1]) ** 2 for k, k1 in ((0, 1), (1, 2), (2, 0)))
    D = (f[3] - f[0]) * (f[7] - f[1]) - (f[4] - f[1]) * (f[6] - f[0])
    if not (M <= 4.0) or not (abs(D) >= 2.0 ** -12 * Lmax2) or not (Lmax2 > 0):
        return 0
    X, Y = max(abs(xlo), abs(xhi)), max(abs(ylo), abs(yhi))
    ex = ey = es = 0.0
    lam_max = np.zeros(3)
    for px, py in ((xlo, ylo), (xhi, ylo), (xlo, yhi), (xhi, yhi)):
        lam = inv[0::3] * px + inv[1::3] * py + inv[2::3]
        ex = max(ex, abs((lam * f[0::3]).sum() - px))
        ey = max(ey, abs((lam * f[1::3]).sum() - py))
        es = max(es, abs(lam.sum() - 1.0))
        lam_max = np.maximum(lam_max, np.abs(lam))
    s = g3 * (np.abs(inv[0::3]) * X + np.abs(inv[1::3]) * Y + np.abs(inv[2::3]))
    mag = (np.abs(inv[0::3]) * X + np.abs(inv[1::3]) * Y + np.abs(inv[2::3])).sum()
    sig, sig_v, W = s.sum(), (s * np.hypot(f[0::3], f[1::3])).sum(), (lam_max + s).sum()
    slop = 2.0 ** -40 * (mag + 1.0) * (M + X + Y + 1.0)
    E, S = np.hypot(ex, ey) + slop, es + sig + slop
    if not S < 0.5:
        return 0
    dA = (np.hypot(X, Y) * S + E + sig_v) / (1.0 - S)
    dB = np.sqrt(2.0) * U * M + E + sig_v + np.sqrt(2.0) * g4 * (1.0 + U + W) * M
    q = np.ceil(max(dA, dB) * 0.5 * H * 16.0)
    return int(max(q, 1.0)) if q <= 63 else 0


# ----------------------------------------------------------------------------------------------- reach_lane_mask
def reach_radius(threshold, H):
    r = F(F(np.sqrt(threshold)) * F(F(0.5) * F(H)) * F(1.0 + 2.0 ** -19)) + F(F(H + 64) * F(2.0 ** -16))
    return r if r <= F(H) else F(-1)


def fma32(a, b, c):
    """fmaf: the float64 product of two float32 is exact; one rounding of the sum to float64, one to float32."""
    return (np.asarray(a, np.float64) * b + c).astype(F)


def kept_by_mask(fv, q, px, row, H, reach, approx):
    """reach_lane_mask's verdict for pixel (px, row) of face fv [n, 9] (one pair per entry), float32 in the kernel's
    order.  approx in {-1, +1}: rsqrtf and __fdividef taken at that end of their error range (2^-21 relative)."""
    e = F(1.0 + approx * 2.0 ** -21)
    f = fv.astype(F)
    tx0, tr0 = (px // 8) * 8, (row // 4) * 4
    c, r = (px - tx0).astype(F), (row - tr0).astype(F)
    xb, yb, hs = pix(tx0, H), pix(H - 1 - tr0, H), F(F(0.5) * F(H))
    R = reach + q.astype(F) * F(0.0625)
    X = [(f[:, 3 * k] - xb) * hs for k in range(3)]
    Y = [(yb - f[:, 3 * k + 1]) * hs for k in range(3)]
    ux, uy = [], []
    for k in range(3):
        k1 = (k + 1) % 3
        ex, ey = X[k1] - X[k], Y[k1] - Y[k]
        rl = F(1) / np.sqrt(fma32(ex, ex, ey * ey)) * e
        ux.append(ex * rl)
        uy.append(ey * rl)
    o = np.where(fma32(ux[0], uy[1], -(uy[0] * ux[1])) > 0, F(1), F(-1))
    lo, hi = np.zeros(len(f), F), np.full(len(f), F(7))
    for k in range(3):
        a, b = o * uy[k], -o * ux[k]
        H_ = np.maximum(np.maximum(fma32(a, X[0], b * Y[0]), fma32(a, X[1], b * Y[1])), fma32(a, X[2], b * Y[2])) + R
        ra = F(1) / a * e
        q0, dq = H_ * ra, -b * ra
        use = np.abs(a) >= F(2.0 ** -20)
        up, dn = use & (a > 0), use & (a < 0)
        h0, hd = np.where(up, q0, F(7)), np.where(up, dq, F(0))
        l0, ld = np.where(dn, q0, F(0)), np.where(dn, dq, F(0))
        hi = np.fmin(hi, fma32(r, hd, h0))
        lo = np.fmax(lo, fma32(r, ld, l0))
    return (np.ceil(lo) <= c) & (c <= np.floor(hi))


# ---------------------------------------------------------------------------------------- the per-pair exit test
def body_exits(fv, inv, px, row, H, threshold):
    """shade_face<2, ...>'s `sign < 0 && dis >= threshold` for each pair, float32 (euclidean_p2f_distance)."""
    f = fv.astype(F)
    xp, yp = pix(px, H), pix(H - 1 - row, H)
    w = np.stack([inv[:, 3 * k] * xp + inv[:, 3 * k + 1] * yp + inv[:, 3 * k + 2] for k in range(3)], 1)
    x, y = f[:, 0::3], f[:, 1::3]
    sym = x[:, :, None] * x[:, None, :] + y[:, :, None] * y[:, None, :] + F(1)
    a0 = sym - np.roll(sym, -1, axis=1)
    fl = np.zeros(len(f), np.int64)   # obtuse flags as k_face_setup sets them (first obtuse vertex only)
    for k in range(3):
        k1, k2 = (k + 1) % 3, (k + 2) % 3
        obt = (x[:, k1] - x[:, k]) * (x[:, k2] - x[:, k]) + (y[:, k1] - y[:, k]) * (y[:, k2] - y[:, k]) < 0
        fl = np.where((fl == 0) & obt, 1 << k, fl)
    inside = np.all((w > 0) & (w < 1), 1)
    le = w <= 0

    def further(p, qq):
        return (xp - x[:, p]) * (x[:, qq] - x[:, p]) + (yp - y[:, p]) * (y[:, qq] - y[:, p]) > 0
    v0 = np.select([le[:, 1] & le[:, 2], le[:, 2] & le[:, 0], le[:, 0] & le[:, 1], le[:, 0], le[:, 1], le[:, 2]],
                   [np.where(((fl & 1) != 0) & further(0, 2), 2, 0), np.where(((fl & 2) != 0) & further(1, 0), 0, 1),
                    np.where(((fl & 4) != 0) & further(2, 1), 1, 2), 1, 2, 0], 0)
    v1 = (v0 + 1) % 3
    n = np.arange(len(f))
    a = a0[n, v0]
    num = w[:, 0] * a[:, 0] + w[:, 1] * a[:, 1] + w[:, 2] * a[:, 2] - a[n, v1]
    den = a[n, v0] - a[n, v1]
    tv0 = num / den
    tv1 = F(1) - tv0
    c0 = np.fmin(np.fmax(tv0, F(0)), F(1))
    c1 = np.fmin(np.fmax(tv1, F(0)), F(1))
    t = np.zeros_like(w)
    t[n, v0] = c0
    t[n, v1] = c1
    t = t - w
    dx = t[:, 0] * x[:, 0] + t[:, 1] * x[:, 1] + t[:, 2] * x[:, 2]
    dy = t[:, 0] * y[:, 0] + t[:, 1] * y[:, 1] + t[:, 2] * y[:, 2]
    dis = dx * dx + dy * dy
    return ~inside & (dis >= threshold)


# --------------------------------------------------------------------------------------------------- the sweep
def pairs(rect, faces):
    """Every (face, pixel) pair of the given faces' rectangles: (face index, px, row)."""
    x0, x1, r0, r1 = rect[faces].T
    nx, nr = np.maximum(x1 - x0 + 1, 0), np.maximum(r1 - r0 + 1, 0)
    cnt = nx * nr
    fi = np.repeat(faces, cnt)
    k = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    nxr = np.repeat(nx, cnt)
    return fi, np.repeat(x0, cnt) + k % nxr, np.repeat(r0, cnt) + k // nxr


def sweep(fv, H, P, chunk=400_000):
    """(pairs walked, pairs the mask drops, faces the gate rejects, faces) over every face of fv [n, 3, 3]; asserts
    that each dropped pair is one the body leaves."""
    thr, border = border_of(P)
    f = np.asarray(fv, F).reshape(-1, 9)
    inv, rect, q = face_setup(f, H, border)
    reach = reach_radius(thr, H)
    gated = np.nonzero(q > 0)[0]
    n_pairs = int(np.prod(np.maximum(rect[:, [1, 3]] - rect[:, [0, 2]] + 1, 0), 1).sum())
    dropped = 0
    if reach >= 0 and len(gated):
        sizes = np.prod(np.maximum(rect[gated][:, [1, 3]] - rect[gated][:, [0, 2]] + 1, 0), 1)
        group = np.cumsum(sizes) // chunk
        for g in np.unique(group):
            sel = gated[group == g]
            fi, px, row = pairs(rect, sel)
            kept = np.ones(len(fi), bool)
            for approx in (-1, 1):
                with np.errstate(all="ignore"):
                    kept &= kept_by_mask(f[fi], q[fi], px, row, H, reach, approx)
            drop = ~kept
            if drop.any():
                ex = body_exits(f[fi[drop]], inv[fi[drop]], px[drop], row[drop], H, thr)
                bad = np.nonzero(~ex)[0]
                assert len(bad) == 0, "dropped pairs the body shades: face %s pixel %s" % (
                    fi[drop][bad[:5]], list(zip(px[drop][bad[:5]], row[drop][bad[:5]])))
            dropped += int(drop.sum())
    bits_rect = np.isfinite(f[:, [0, 1, 3, 4, 6, 7]]).all(1) & (rect[:, 0] <= rect[:, 1])
    return n_pairs, dropped, int((bits_rect & (q == 0)).sum()), len(f)


def test_restated_exit_matches_the_oracle():
    """body_exits() against the oracle's own per-face loop: each face alone in its batch element, alpha ('prod') is
    > 0 exactly on the pixels whose pair the body did not leave (the sigmoid of a kept pair is >= dist_eps)."""
    H = 64
    fv, _ = SCENES["slivers"](H)
    fv = np.concatenate([fv[:, ::40], SCENES["coords"](H)[0][:, 280::4], SCENES["pixel_centres"](H)[0][:, 280::8]], 1)
    one = fv[0][:, None]   # [n, 1, 3, 3]
    tex = np.ones((len(one), 1, 1, 3), F)
    P = osr.Params(image_size=H, sigma_val=1e-4)
    thr, border = border_of(P)
    alpha = osr.forward(one, tex, P)["soft_colors"][:, 3]
    f = one.reshape(-1, 9)
    inv, rect, _ = face_setup(f, H, border)
    fi, px, row = pairs(rect, np.arange(len(f)))
    shaded = alpha[fi, row, px] > 0
    exits = body_exits(f[fi], inv[fi], px, row, H, thr)
    assert len(fi) > 20_000
    assert np.array_equal(shaded, ~exits)


def test_reach_cull_is_conservative_on_c3_and_c2():
    P = osr.Params(image_size=1024)
    tot = drop = 0
    for nf, b in ((39200, 0), (3280, 3)):
        fv, _ = wl.make_scene(nf, batch=4)
        n, d, rejected, faces = sweep(fv[b], 1024, P)
        tot, drop = tot + n, drop + d
        if nf == 39200:
            print("C3 image 0: %d pairs, %d dropped (%.1f %%), gate rejects %d of %d faces"
                  % (n, d, 100.0 * d / n, rejected, faces))
            assert rejected <= faces // 50, "the gate rejects %d of the C3 faces" % rejected
            assert d > 0.15 * n
    assert tot >= 10_000_000


@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("H,sigma", [(128, 3e-5), (512, 1e-5), (1024, 1e-6)])
def test_reach_cull_is_conservative_on_hostile_scenes(name, H, sigma):
    fv, _ = SCENES[name](H)
    n, d, _, _ = sweep(fv[0], H, osr.Params(image_size=H, sigma_val=sigma))
    assert n > 0


@pytest.mark.parametrize("name", ["micro_faces", "huge_faces", "pixel_aligned", "non_finite"])
def test_reach_cull_is_conservative_on_out_of_range_inputs(name):
    if name == "non_finite":
        fv = rng_cases.non_finite_scene()[0][1]
        P = osr.Params(image_size=rng_cases.H, sigma_val=1e-4)
    else:
        fv = rng_cases.CASES[name][0]()[0][0]
        P = rng_cases.params(name, "euclidean")
    sweep(fv, rng_cases.H, P)
