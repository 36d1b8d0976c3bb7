"""The SoftRas forward's per-entry error bound (oracle.softras.forward_bound, softras_oracle.c "rounding sites of the K2
forward") on the oracle alone: no GPU needed.

* Every case of tests/softras_forward_cases.py reaches the sites it targets, under both softras_exact_tail values.
* The bound holds its own perturbation semantics: the oracle forward with every live site moved by its budget (up,
  down, hashed signs; with exact_tail = 0 the kernel's fp32 tails) stays within the plain forward's bound, entry by
  entry, and the bound is exactly 0 wherever no site is live.
* It closes the gap the old blanket tolerances (2e-6 absolute on soft_colors, 2e-6 relative on softmax_sum) left:
  three outputs the oracle computes from subtly perturbed inputs pass those tolerances and fail the bound.
* It is tight: its median is a few ulp of the value in every aggregation mode.
"""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests import softras_forward_cases as fc
from tests.util import hold_to_bound

OLD_COLOR_ATOL = 2e-6   # the blanket tolerances the bound replaces
OLD_SUM_RTOL = 2e-6
NUDGES = (1, -1, 2, 3, 4, 5)


def passes_old(got, ref):
    m = np.isfinite(ref["soft_colors"])
    ok = np.abs(got["soft_colors"][m] - ref["soft_colors"][m]).max(initial=0.0) <= OLD_COLOR_ATOL
    s, r = got["aggrs_info"][:, 0].astype(np.float64), ref["aggrs_info"][:, 0].astype(np.float64)
    return ok and bool(np.all(np.abs(s - r) <= OLD_SUM_RTOL * np.abs(r))) and \
        np.array_equal(got["aggrs_info"][:, 1], ref["aggrs_info"][:, 1])


def fails_bound(got, ref):
    try:
        hold_to_bound(got["soft_colors"], ref["soft_colors"], ref["bound_colors"], "soft_colors")
        hold_to_bound(got["aggrs_info"][:, 0], ref["aggrs_info"][:, 0], ref["bound_sum"], "softmax_sum")
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("exact_tail", [0, 1])
@pytest.mark.parametrize("name", sorted(fc.CASES))
def test_case_reaches_its_sites(name, exact_tail):
    fv, tex, P = fc.build(name)
    ref = osr.forward_bound(fv, tex, P, exact_tail=exact_tail)
    want = set(fc.CASES[name][2]) - (fc.FP32_ONLY if exact_tail else set())
    got = fc.reached(ref)
    assert want <= got, "%s missed %s (reached %s)" % (name, sorted(want - got), sorted(got))
    if exact_tail:
        assert not got & fc.FP32_ONLY, "a site of the fp32 tails is live under softras_exact_tail = 1"
    assert (ref["faces_id_buffer"] >= 0).any()


def test_cases_reach_their_values():
    """What the scenes are for, seen in the oracle's outputs."""
    def run(name, **kw):
        fv, tex, P = fc.build(name, **kw)
        return osr.forward_bound(fv, tex, P)
    sc = run("dark_textures")["soft_colors"][:, :3]
    assert 0 < sc.max() <= 1e-3
    assert run("bright_textures")["soft_colors"][:, :3].max() > 1.0
    # gamma 1e-6: softmax weights of faces behind the front one underflow to exactly 0
    fv, tex, P = fc.build("gamma_1e-6")
    ids = osr.forward(fv, tex, P)["faces_id_buffer"]
    hidden = np.zeros(tex.shape[:2], bool)
    for b in range(ids.shape[0]):
        hidden[b, np.unique(ids[b, 1:][ids[b, 1:] >= 0])] = True
    assert hidden.any()
    # sigma tiny: the sigmoid saturates, every alpha is exactly 0 or 1 and nothing gets a bound
    r = run("sigma_tiny")
    assert set(np.unique(r["soft_colors"][:, 3])) <= {0.0, 1.0}
    # alpha = prod under 72 soft edges: the product stays near 1, the output 1 - alpha at the centre pixel is small,
    # and the 72 fp32 products of softras_exact_tail = 0 give it a bound of many ulp, which nudging reaches
    fv, tex, P = fc.build("stacked_soft_edges")
    c = P["image_size"] // 2
    r = osr.forward_bound(fv, tex, P)
    a, b = r["soft_colors"][:, 3, c, c], r["bound_colors"][:, 3, c, c]
    assert (0 < a).all() and (a < 0.25).all() and (r["live"][:, c, c] >> osr.SITE["prod"] & 1).all()
    assert (b >= 64 * np.spacing(a)).all(), b / np.spacing(a)
    n = osr.forward_bound(fv, tex, P, nudge=1)["soft_colors"][:, 3, c, c]
    assert (np.abs(n.astype(np.float64) - a) >= 0.5 * b).all()
    r = run("alpha_sum")
    assert r["soft_colors"][:, 3].max() > 0 and (r["live"] != 0).any()


@pytest.mark.parametrize("exact_tail", [0, 1])
@pytest.mark.parametrize("variant", sorted(fc.VARIANTS))
@pytest.mark.parametrize("name", sorted(fc.CASES))
def test_nudged_forwards_stay_within_the_bound(name, variant, exact_tail):
    fv, tex, P = fc.build(name, variant)
    plain = osr.forward(fv, tex, P)
    ref = osr.forward_bound(fv, tex, P, exact_tail=exact_tail)
    for k in ("soft_colors", "aggrs_info", "faces_id_buffer", "faces_info"):
        assert np.array_equal(ref[k], plain[k], equal_nan=True), k
    nolive = ref["live"] == 0
    assert (ref["bound_colors"].transpose(1, 0, 2, 3)[:, nolive] == 0).all() and (ref["bound_sum"][nolive] == 0).all()
    for nudge in NUDGES:
        n = osr.forward_bound(fv, tex, P, exact_tail=exact_tail, nudge=nudge)
        assert np.array_equal(n["faces_id_buffer"], ref["faces_id_buffer"])
        hold_to_bound(n["soft_colors"], ref["soft_colors"], ref["bound_colors"], "soft_colors nudge %d" % nudge, ref["live"])
        if P["aggr_func_rgb"] == "softmax":
            hold_to_bound(n["aggrs_info"][:, 0], ref["aggrs_info"][:, 0], ref["bound_sum"], "softmax_sum", ref["live"])
            # softmax_max moves only with a live by_span site
            d = n["aggrs_info"][:, 1] != ref["aggrs_info"][:, 1]
            assert not (d & (ref["live"] >> osr.SITE["div_span"] & 1 == 0)).any()


@pytest.mark.parametrize("image_size", [1000])
def test_nudged_forward_large_odd_image(image_size):
    """Image 1000, batch 3, every 37th row: the bound on the sizes the GPU sweep runs."""
    fv, tex, P = fc.build("gamma_1", image_size=image_size)
    ref = osr.forward_bound(fv, tex, P, row_stride=37)
    n = osr.forward_bound(fv, tex, P, nudge=2, row_stride=37)
    hold_to_bound(n["soft_colors"], ref["soft_colors"], ref["bound_colors"], "soft_colors", ref["live"])
    hold_to_bound(n["aggrs_info"][:, 0], ref["aggrs_info"][:, 0], ref["bound_sum"], "softmax_sum", ref["live"])


@pytest.mark.parametrize("dist,rgb", [("hard", "hard"), ("hard", "none")])
@pytest.mark.parametrize("alpha", ["hard", "sum", "prod"])
def test_exp_free_modes_have_no_site(dist, rgb, alpha):
    """Hard distance with hard or no colour aggregation reaches no expf and no tail: the bound is 0 everywhere, so the
    kernel's soft_colors must be the oracle's bit for bit."""
    fv, tex = wl.make_scene(280, batch=2)
    P = osr.Params(image_size=48, dist_func=dist, aggr_func_rgb=rgb, aggr_func_alpha=alpha)
    for et in (0, 1):
        ref = osr.forward_bound(fv, tex, P, exact_tail=et)
        assert (ref["live"] == 0).all() and (ref["bound_colors"] == 0).all() and (ref["bound_sum"] == 0).all()


# ------------------------------------------------------------------------------------------------ the gap is closed
def scene_with_background():
    return wl.make_scene(280, batch=1)


def test_gamma_one_ulp_off_is_caught():
    """A softmax weight computed from a reciprocal of gamma one ulp off: within the old tolerances, outside the bound."""
    fv, tex = scene_with_background()
    P = osr.Params(image_size=64)
    ref = osr.forward_bound(fv, tex, P)
    P2 = osr.Params(image_size=64, gamma_val=float(np.nextafter(np.float32(P["gamma_val"]), np.float32(1))))
    got = osr.forward(fv, tex, P2)
    assert passes_old(got, ref)
    assert fails_bound(got, ref)


def test_background_term_moved_8_ulp_is_caught():
    """A background term expf(eps / gamma) moved 8 ulp (gamma moved until it is, eps kept, so softmax_max stays put):
    within the old tolerances, outside the bound."""
    fv, tex = scene_with_background()
    P = osr.Params(image_size=64, gamma_val=1e-3)
    ref = osr.forward_bound(fv, tex, P)
    g, eps = np.float32(P["gamma_val"]), np.float32(P["eps"])
    bg = np.exp(eps / g)
    g2 = g
    while abs(int(np.exp(eps / g2).view(np.int32)) - int(bg.view(np.int32))) < 8:
        g2 = np.nextafter(g2, np.float32(0))   # six steps down: 8 ulp
    assert abs(int(np.exp(eps / g2).view(np.int32)) - int(bg.view(np.int32))) == 8
    got = osr.forward(fv, tex, osr.Params(image_size=64, gamma_val=float(g2)))
    assert passes_old(got, ref)
    assert fails_bound(got, ref)


def test_texture_of_a_faint_face_is_caught():
    """One face's texture changed where that face's largest softmax weight is 1e-6 .. 4e-6 of its pixel's sum: the
    colour moves by less than 2e-6 (the old tolerance) but by more than the bound, on at least one pixel."""
    fv, tex = scene_with_background()
    P = osr.Params(image_size=32, gamma_val=3e-4)
    ref = osr.forward_bound(fv, tex, P)
    ids = ref["faces_id_buffer"][0]
    cands = np.unique(ids[ids >= 0])
    # a face's share of a pixel's colour sum, per pixel: the colour change per unit texture change (colour is linear
    # in the texture, weight / sum exactly up to rounding)
    found = None
    for f in cands:
        t2 = tex.copy()
        t2[0, f] += 1.0
        share = np.abs(osr.forward(fv, t2, P)["soft_colors"][0, :3].astype(np.float64) - ref["soft_colors"][0, :3]).max()
        if 1e-6 <= share <= 4e-6:
            found = f
            break
    assert found is not None, "no face whose largest weight share is in [1e-6, 4e-6]"
    t2 = tex.copy()
    t2[0, found] = np.where(t2[0, found] > 0.5, t2[0, found] - 0.5, t2[0, found] + 0.5)
    got = osr.forward(fv, t2, P)
    assert passes_old(got, ref)
    assert fails_bound(got, ref)


# ------------------------------------------------------------------------------------------------------ tightness
MODES = [dict(), dict(aggr_func_alpha="sum"), dict(aggr_func_alpha="hard"), dict(dist_func="barycentric"),
         dict(aggr_func_rgb="hard"), dict(aggr_func_rgb="hard", aggr_func_alpha="sum")]


@pytest.mark.parametrize("exact_tail", [0, 1])
def test_bound_is_tight(exact_tail, capsys):
    """The bound in ulps of the value (entries with a non-zero, finite bound): median and 99th percentile per mode.  The
    median must stay a few ulp, or the bound has quietly become vacuous."""
    fv, tex = wl.make_scene(280, batch=2)
    lines = []
    for mode in MODES:
        P = osr.Params(image_size=64, sigma_val=3e-5, **mode)
        ref = osr.forward_bound(fv, tex, P, exact_tail=exact_tail)
        for what, v, b in (("colors", ref["soft_colors"], ref["bound_colors"]),
                           ("sum", ref["aggrs_info"][:, 0], ref["bound_sum"])):
            m = (b > 0) & np.isfinite(b)
            if not m.any():
                continue
            u = b[m] / np.spacing(np.abs(v[m]).astype(np.float32)).astype(np.float64)
            med, p99 = np.median(u), np.percentile(u, 99)
            lines.append("exact_tail=%d %-40s %-6s n=%6d median %5.1f ulp  p99 %6.1f ulp" % (
                exact_tail, ",".join("%s=%s" % kv for kv in mode.items()) or "default", what, m.sum(), med, p99))
            assert med <= 8, lines[-1]
    with capsys.disabled():
        print("\n" + "\n".join(lines))
