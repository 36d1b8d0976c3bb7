"""The scenes of test_nmr_edges_gpu.py reach the NMR kernel paths they are built for, and stay inside the reference's
defined behaviour (every float -> int conversion of K7 / K9 has a finite, in-range input).  No GPU: the decisions come
from oracle.nmr_paths, the kernels' per-sample set-up restated in numpy float32, over the oracle's face index map."""
import collections

import numpy as np
import pytest

from oracle import nmr as onmr
from oracle import nmr_paths as P
from tests import nmr_edge_cases as E


def paths(faces, is_, eps=1e-3, near=0.1, far=100.0):
    ref = onmr.forward(faces, None, is_, near, far, eps, (0, 0, 0), False, True, False)
    with np.errstate(all="ignore"):
        for b in range(faces.shape[0]):
            for f in faces[b]:
                assert P.zbuffer_path(f, is_)[1], "bounding box not convertible"
        S = P.scene_paths(faces, ref["face_index_map"], is_, eps)   # raises on an undefined conversion
    assert any(s["live"] for s in S) or is_ == 1   # one pixel: every out-pixel is off the image
    return ref, S


def outward(S):
    """{(flavour, axis, toward_zero): set of n}"""
    r = collections.defaultdict(set)
    for s in S:
        if s["out"]:
            r[(s["out"]["flavour"], s["axis"], s["out"]["toward_zero"])].add(s["out"]["n"])
    return r


def test_long_inward_reaches_warp_scan_with_owner_test():
    faces = E.long_inward()
    ref, S = paths(faces, 256)
    inw = [s["inward"] for s in S if s["inward"]]
    for span in (63, 64, 65):   # in_to - in_from: 63 is the serial loop's last width, 64 the warp scan's first
        assert any(i["span"] == span for i in inw), span
    assert all((i["flavour"] == "warp") == (i["span"] >= 64) for i in inw)
    warp = [i for i in inw if i["flavour"] == "warp"]
    assert max(i["span"] for i in warp) >= 200
    assert sum(1 for i in warp if i["unowned"] > 0 and i["owned"] > 0) >= 50   # the owner test drops pixels
    assert {s["axis"] for s in S if s["inward"] and s["inward"]["flavour"] == "warp"} == {0, 1}
    assert {s["b"] for s in S if s["inward"] and s["inward"]["flavour"] == "warp"} == {0, 1}


def test_outward_seams_cover_every_n_direction_axis_and_flavour():
    _, S = paths(E.outward_seams(), 256)
    got = outward(S)
    for flavour in ("out", "generic"):
        for axis in (0, 1):
            for toward_zero in (False, True):
                missing = set(E.SEAM_N) - got[(flavour, axis, toward_zero)]
                assert not missing, (flavour, axis, toward_zero, sorted(missing))


def test_past_end_lanes_cancel_exactly():
    _, S = paths(E.past_end(), 256, eps=E.PAST_END_EPS)
    hits = {(s["axis"], s["out"]["n"], s["out"]["half"]) for s in S if s["out"] and s["out"]["past_end_zero"]}
    assert all(s["out"]["toward_zero"] and s["out"]["flavour"] == "out" for s in S if s["out"] and s["out"]["past_end_zero"])
    assert (0, 110, "b") in hits and (1, 110, "b") in hits                     # the constructed case and its transpose
    for axis in (0, 1):
        assert {h for a, _, h in hits if a == axis} == {"a", "b"}
        assert len({n % 64 for a, n, _ in hits if a == axis}) >= 4
    # at a default eps no lane cancels: the test needs the dyadic eps
    _, S = paths(E.past_end(), 256, eps=1e-3)
    assert not any(s["out"]["past_end_zero"] for s in S if s["out"])


def test_pixel_aligned_vertices_take_generic_scans_and_vertex_crossings():
    faces = E.pixel_aligned()
    _, S = paths(faces, 64)
    assert any(s["live"] and not s["has0"] for s in S) and any(s["live"] and not s["has1"] for s in S)
    assert sum(1 for s in S if s["cross2_zero"]) >= 20
    assert any(s["out"] and s["out"]["flavour"] == "generic" for s in S)
    pix = np.round(0.5 * (faces[..., :2].astype(np.float64) * 64 + 63), 6)
    assert np.all(pix == np.round(pix)) and (pix == 0).any() and (pix == 63).any()


@pytest.mark.parametrize("is_", [1, 2, 31, 33])
def test_small_image_sizes_render(is_):
    ref, S = paths(E.tiny(is_), is_)
    assert (ref["face_index_map"] >= 0).any()
    if is_ > 2:
        assert any(s["out"] for s in S) and any(s["inward"] for s in S)


def test_image_size_4096_scans_span_the_image():
    faces = E.huge()
    ref, S = paths(faces, 4096)
    assert (ref["face_index_map"] >= 0).mean() > 0.3
    assert max(s["out"]["n"] for s in S if s["out"]) > 3900
    assert max(s["inward"]["span"] for s in S if s["inward"]) > 3000
    zp = collections.Counter(P.zbuffer_path(f, 4096)[0] for f in faces[0])
    assert zp["warp"] == 8


def test_depth_order_reaches_negative_and_signed_zero_depths():
    ref, S = paths(E.depth_order(), 64, near=E.DEPTH_NEAR, far=E.DEPTH_FAR)
    d, fim = ref["depth_map"], ref["face_index_map"]
    assert (d < 0).any() and (d > 0).any()                                       # nmr_order_bits' negative branch
    zero = (d == 0) & (fim >= 0)
    assert (zero & np.signbit(d)).any() and (zero & ~np.signbit(d)).any()       # -0 and +0 winners


def test_cancelling_colours_give_exact_zero_diffs():
    faces = E.long_inward()
    tex = E.textures(faces, const=(0.3, 0.55, 0.8))
    ref = onmr.forward(faces, tex, 256, 0.1, 100.0, 1e-3, (0.3, 0.55, 0.8), True, True, False)
    bg = ref["face_index_map"] < 0
    assert bg.mean() > 0.2 and (ref["rgb_map"][bg] == np.float32([0.3, 0.55, 0.8])).all()


def test_off_screen_faces_have_dead_samples_and_clamped_scans():
    faces = E.off_screen()
    assert (np.abs(faces[..., :2]) >= 1.5).any()
    _, S = paths(faces, 128)
    assert sum(1 for s in S if not s["live"]) >= 100
    assert any(s["inward"] and s["inward"]["from_"] == 0 for s in S) and any(s["inward"] and s["inward"]["to"] == 127 for s in S)
    got = outward(S)
    assert all(got[("out", a, t)] >= {1, 64, 65} for a in (0, 1) for t in (False, True))
