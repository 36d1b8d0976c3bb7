"""CPU checks of the subsurface-scattering oracle (oracle/sss.py) and the product's host constants:

- oracle.blur against the reference's own blur kernels run on a GPU (tests/golden/ref_sss_gpu_blur_*.npz, made by
  oracle/make_ref_sss_blur_golden.py from the kernels oracle/build_ref_sss.py builds);
- oracle.stretch and the product's tap weights against the reference's own Python (tests/golden/ref_host_sss.npz, made by
  oracle/make_ref_host_sss_golden.py);
- the C ABI's declarations and the new profiler id;
- when the reference checkout is present, the host golden regenerates array for array.

Tolerance against the reference kernels.  The reference build contracts a*b+c into FMAs (nvcc's default), the oracle
rounds every product.  Per tap, `interpolation = (x - x1) v2 + (x2 - x) v1` and `v += interpolation * tap` each differ by
at most one rounding of a term, i.e. 2^-24 of |term|; summed over the 7 taps that is a few ulp of sum_k |interpolation_k
tap_k| <= max|image| * sum(tap) * 3 (an extrapolating tap has weights up to 2 in magnitude).  The positions x are
computed identically (x += step has no product to contract), so x1, x2, the <= 1e-6 fallback and the zeroed pixels are
the same decisions; the zeroed pixels are compared exactly.  A tap wholly past an edge contributes (x - c) v + (c - x) v,
exactly 0 unfused and the rounding error of a product as large as |x - c| |v| fused: the terms are not bounded by the
image but by the tap's distance from the pixel it reads.  So each pixel is held to
2^-22 max|image| sum_k tap_k (|x_k - x1_k| + |x2_k - x_k|) + 2^-20 max|image| (bound() below): a rounding of each
product in each term, and 16 ulp of the largest input for the accumulation.  The worst measured difference is 0.10 of
that bound.
"""
import glob
import os
import re

import numpy as np
import pytest

from oracle import build_ref
from oracle import sss as osss
from tests.conftest import ROOT

G = os.path.join(ROOT, "tests", "golden")
BLUR_FILES = sorted(glob.glob(os.path.join(G, "ref_sss_gpu_blur_*.npz")))


def bound(img, mod, taps, width, dim):
    """Per-pixel bound on |fused - unfused| for one blur: 2^-22 max|image| sum_k tap_k (|x_k - x1_k| + |x2_k - x_k|) +
    2^-20 max|image| (see the module docstring)."""
    H, W = img.shape
    c = np.broadcast_to(np.arange(W)[None, :] if dim == 1 else np.arange(H)[:, None], (H, W)).astype(np.float32)
    step = np.float32(width) * mod
    x = c - step * np.float32(3)
    s = np.zeros((H, W), np.float64)
    for k in range(7):
        x1 = np.clip(np.trunc(x), 0, W - 1)
        x2 = np.clip(np.trunc(x) + 1, 0, W - 1)
        s += float(taps[k]) * (np.abs(x - x1) + np.abs(x2 - x))
        x = x + step
    m = float(np.abs(img).max())
    return 2.0 ** -22 * m * s + 2.0 ** -20 * m


def test_blur_goldens_cover_the_cases():
    shapes = {os.path.basename(p)[len("ref_sss_gpu_blur_"):-4] for p in BLUR_FILES}
    assert shapes == {"64x64", "48x80", "80x48"}
    keys = set()
    for p in BLUR_FILES:
        keys |= {k.rsplit("_", 1)[0] for k in np.load(p).files if k.endswith("_out")}
    assert {k.split("_")[0] for k in keys} == {"d0", "d1"}
    assert {k.split("_")[1] for k in keys} == {"v25", "v75", "v300"}


@pytest.mark.parametrize("path", BLUR_FILES, ids=lambda p: os.path.basename(p)[:-4])
def test_blur_oracle_matches_reference_kernels(path):
    g = np.load(path)
    cases = sorted(k[:-4] for k in g.files if k.endswith("_out"))
    assert cases
    seen = dict(zero=0, fallback=0, off_left=0, off_right=0, mod0=0, mod1=0)
    for key in cases:
        img, mod, ref = g[key + "_image"], g[key + "_mod"], g[key + "_out"]
        dim = int(key[1])
        got = osss.blur(img, mod, g[key + "_taps"], g[key + "_width"], dim)
        # the decisions: a pixel <= 0 is zeroed on both sides.  Elsewhere a 0 can also come from cancellation: all taps
        # past the edge give exactly 0 unfused and a rounding residue fused, which the tolerance covers
        assert np.all(got[img <= 0] == 0) and np.all(ref[img <= 0] == 0), key
        np.testing.assert_array_less(np.abs(got - ref), bound(img, mod, g[key + "_taps"], g[key + "_width"], dim),
                                     err_msg=key)
        # the cases the golden is meant to hold
        n = img.shape[1] if dim == 1 else img.shape[0]
        c = np.arange(n)[None, :] if dim == 1 else np.arange(n)[:, None]
        reach = 3 * g[key + "_width"] * mod
        live = img > 0
        seen["zero"] += int((~live).sum())
        seen["fallback"] += int(((img > 0) & (img.astype(np.float64) <= 1e-6)).sum())
        seen["off_left"] += int((live & (c - reach < 0)).sum())
        seen["off_right"] += int((live & (c + reach > n - 1)).sum())
        seen["mod0"] += int((live & (mod == 0)).sum())
        seen["mod1"] += int((live & (mod == 1)).sum())
    assert all(v > 0 for v in seen.values()), seen


def test_stretch_oracle_matches_reference_rows():
    """oracle.stretch against computeStretchMap's stretchU, run by the reference's own ToStretchMap.py on the rasterized
    world-coordinate map (stretchU needs only the row itself), clamped as lighting.py:110 does."""
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    u, _ = osss.stretch(g["world_rows"])
    np.testing.assert_array_equal(u, np.clip(g["stretch_u_rows"], 0, 1))
    assert (u == 1).any() and ((u > 0) & (u < 1)).any()   # flat faces give 1, their edges less


def test_product_taps_match_reference():
    from jrender_b200 import lighting
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    variances = [b - a for a, b in zip(lighting.SSS_GAUSSIAN_BASIS, lighting.SSS_GAUSSIAN_BASIS[1:])]
    assert variances == osss.levels() == [25, 75, 300]
    for v in variances:
        taps, width = lighting._sss_taps(v)
        np.testing.assert_array_equal(np.float32(taps), g["taps_v%d" % v])
        assert np.float32(width) == g["width_v%d" % v]
        np.testing.assert_array_equal(osss.taps(v)[0], g["taps_v%d" % v])
    assert lighting.SSS_WEIGHTS == osss.WEIGHTS


def test_header_declares_sss_entry_points():
    from jrender_b200 import _lib
    src = open(os.path.join(ROOT, "include", "b200raster.h")).read()
    sigs = _lib.parse_header(src)
    assert len(sigs["b200r_sss_workspace_bytes"][1]) == 2
    assert len(sigs["b200r_sss_stretch"][1]) == 6
    assert len(sigs["b200r_sss_blur_pyramid"][1]) == 14
    enum = re.search(r"enum \{ (B200R_K_\w+ = 0,[^}]*)\}", src).group(1)
    ids = dict((k, int(v)) for k, v in re.findall(r"(B200R_K_\w+) = (\d+)", enum))
    assert list(ids.values()) == list(range(len(ids))) and ids["B200R_K_SSS"] == 25
    assert enum.rstrip().endswith("B200R_K_SSS = 25, B200R_K_COUNT")
    cu = open(os.path.join(ROOT, "jrender_b200", "csrc", "sss_api.cu")).read()
    assert cu.count("b200r_launch(") == 3   # stretch, x pass, y pass


@pytest.mark.skipif(not os.path.isdir(build_ref.REFERENCE), reason="needs the reference checkout")
def test_host_golden_regenerates_from_reference(tmp_path):
    """About four minutes: twelve 2048^2 oracle rasterizations and 144 oracle blurs."""
    from oracle import make_ref_host_sss_golden as mk
    out = str(tmp_path / "ref_host_sss.npz")
    mk.main(out)
    a, b = np.load(out), np.load(os.path.join(G, "ref_host_sss.npz"))
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
