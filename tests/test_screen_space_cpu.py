"""CPU checks of the render2 screen-space passes: oracle/screen_space.py against the reference goldens
tests/golden/ref_screen_*.npz (made by oracle/make_ref_screen_golden.py from the reference's own kernels), conv_for_image
against a direct loop over the reference's index expression, and the argument errors of jrender_b200.render2.

oracle/screen_space.py emulates every fused multiply-add exactly; its only inexact sites are rsqrtf and the double
cos / sin (named in its docstring).  On these goldens they change no SSAO count and no FXAA bit; SSDO colours, which
carry the rsqrtf of each indirect sample's direction, are held to SSDO_ATOL (measured: at most 1.2e-7, on values up to 1).
"""
import glob
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

from jrender_b200.render2 import FXAA_cuda, SSAO_cuda, SSDO_cuda, conv_for_image
from oracle import screen_space as oss

G = os.path.join(os.path.dirname(__file__), "golden")
GOLDENS = sorted(glob.glob(os.path.join(G, "ref_screen_*.npz")))
SSDO_ATOL = 1e-6


def test_goldens_exist():
    assert len(GOLDENS) == 3


def bits_equal(got, want):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got.view(np.int32)[~nan], want.view(np.int32)[~nan])


@pytest.mark.parametrize("path", GOLDENS, ids=os.path.basename)
def test_oracle_reproduces_reference_goldens(path):
    z = np.load(path)
    args = (z["width"], z["sample_num"], z["sample_range_r"], z["draws"])
    ao = oss.ssao(z["depth"], z["face_ind"], z["normal"], *args)
    assert np.array_equal(ao * z["sample_num"], z["ssao"] * z["sample_num"])   # sample counts, exactly
    assert (z["ssao"] > 0).any() and (z["face_ind"] == -1).any()
    do = oss.ssdo(z["color"], z["depth"], z["face_ind"], z["normal"], *args)
    assert np.abs(do - z["ssdo"]).max() <= SSDO_ATOL
    bg = z["face_ind"] == -1
    assert np.array_equal(z["ssdo"][bg], z["color"][bg])
    for k in ("render", "noise", "const", "nonfinite"):
        bits_equal(oss.fxaa(z["fxaa_in_" + k]), z["fxaa_out_" + k])


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a, b = rng.standard_normal((2, 4000)).astype(np.float32)
    c = (rng.standard_normal(4000) * np.exp2(rng.integers(-30, 30, 4000))).astype(np.float32)
    c[:1000] = -(a[:1000].astype(np.float64) * b[:1000]).astype(np.float32)   # heavy cancellation
    got = oss.fma32(a, b, c)
    for x, y, w, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(w))
        near = np.float32(float(exact))     # within one float32 ulp of the correctly rounded result
        up, dn = np.nextafter(near, np.float32(np.inf)), np.nextafter(near, np.float32(-np.inf))
        want = min((near, up, dn), key=lambda v: (abs(Fraction(float(v)) - exact), int(v.view(np.int32)) & 1))
        assert g == want, (x, y, w)


def loop_conv(x, w, overflow):
    """The reference's reindex: y[i, j] = sum_ab w[a, b] * x[i + a - 1, j + b - 1], overflow outside."""
    H, W = x.shape[:2]
    kh, kw = w.shape
    y = torch.zeros_like(x)
    for i in range(H):
        for j in range(W):
            for a in range(kh):
                for b in range(kw):
                    r, c = i + a - 1, j + b - 1
                    v = x[r, c] if 0 <= r < H and 0 <= c < W else torch.full_like(x[0, 0], overflow)
                    y[i, j] = y[i, j] + w[a, b] * v
    return y


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("overflow", [0, 1])
@pytest.mark.parametrize("channels", [None, 2])
def test_conv_for_image_matches_the_reference_index_expression(k, overflow, channels):
    g = torch.Generator().manual_seed(k * 10 + overflow)
    shape = (9, 9) if channels is None else (9, 9, channels)
    x = torch.rand(shape, generator=g, dtype=torch.float64)
    w = torch.rand((k, k), generator=g, dtype=torch.float64)
    y = conv_for_image(x, w, overflow)
    assert y.shape == x.shape
    torch.testing.assert_close(y, loop_conv(x, w, overflow), rtol=1e-12, atol=1e-12)
    if k == 5 and overflow == 0 and channels is None:   # Render.SSAO's box: the anchor is shifted, not centred
        ones = conv_for_image(torch.ones(9, 9, dtype=torch.float64), torch.ones(5, 5, dtype=torch.float64) / 25)
        assert ones[0, 0] == pytest.approx(16 / 25) and ones[8, 8] == pytest.approx(4 / 25)


@pytest.mark.parametrize("k", [3, 5, 7])
def test_conv_for_image_gradients_match_float64_autograd(k):
    g = torch.Generator().manual_seed(k)
    x = torch.rand((7, 6, 3), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.rand((k, k), generator=g, dtype=torch.float64, requires_grad=True)
    gy = torch.rand((7, 6, 3), generator=g, dtype=torch.float64)
    gx, gw = torch.autograd.grad((conv_for_image(x, w, 1) * gy).sum(), (x, w))
    rx, rw = torch.autograd.grad((loop_conv(x, w, 1) * gy).sum(), (x, w))
    torch.testing.assert_close(gx, rx, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(gw, rw, rtol=1e-12, atol=1e-12)
    assert torch.autograd.gradcheck(lambda a, b: conv_for_image(a, b, 0.5), (x, w))
    # float32 inputs give the float64 result rounded
    y32 = conv_for_image(x.detach().float(), w.detach().float(), 1)
    torch.testing.assert_close(y32.double(), loop_conv(x.detach(), w.detach(), 1), rtol=1e-6, atol=1e-6)


def test_argument_errors():
    d, f, n, c = torch.zeros(4, 4), torch.zeros(4, 4, dtype=torch.int32), torch.zeros(4, 4, 3), torch.zeros(4, 4, 3)
    cases = [
        (lambda: SSAO_cuda(torch.zeros(4, 5), f, n, 0.5, 8, 0.1), "square"),                    # non-square
        (lambda: SSAO_cuda(d, torch.zeros(5, 5, dtype=torch.int32), n, 0.5, 8, 0.1), "match"),  # mismatched shapes
        (lambda: SSAO_cuda(d, f, torch.zeros(4, 4, 4), 0.5, 8, 0.1), "square"),                 # wrong channel count
        (lambda: SSAO_cuda(d, f, n, 0.5, 8, 0.1), "CUDA"),                                       # not on the GPU
        (lambda: SSDO_cuda(torch.zeros(4, 4, 4), d, f, n, 0.5, 8, 0.1), "square"),
        (lambda: SSDO_cuda(torch.zeros(3, 3, 3), d, f, n, 0.5, 8, 0.1), "match"),
        (lambda: SSDO_cuda(c, d, f, torch.zeros(4, 3, 3), 0.5, 8, 0.1), "square"),
        (lambda: SSDO_cuda(c, d, f, n, 0.5, 8, 0.1), "CUDA"),
        (lambda: FXAA_cuda(torch.zeros(4, 4)), "square"),
        (lambda: FXAA_cuda(torch.zeros(4, 5, 3)), "square"),
        (lambda: FXAA_cuda(torch.zeros(4, 4, 1)), "square"),
        (lambda: FXAA_cuda(c), "CUDA"),
        (lambda: FXAA_cuda(np.zeros((4, 4, 3), np.float32)), "Tensor"),
        (lambda: conv_for_image(torch.zeros(4), torch.ones(3, 3)), "conv_for_image"),
    ]
    for fn, words in cases:
        with pytest.raises(ValueError, match=words):
            fn()
