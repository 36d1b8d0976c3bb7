"""numpy restatement of the texture-space subsurface scattering maps (TEST INFRASTRUCTURE, not product code).

  stretch()        computeStretchMap of `7 * Worldcoord_Map` (jrender/renderer/utils/ToStretchMap.py:5-13) and the two
                   clamps to [0, 1] (jrender/renderer/lighting/lighting.py:109-111)
  taps()           gaussian_blur's tap weights and GaussWidth (renderer/utils/gaussian_blur.py:7-13)
  blur()           gaussain_blur_x_Kernel / gaussain_blur_y_Kernel (gaussian_blur.py:33-164) on one single-channel map
  blur_pyramid()   lighting.py:113-150: three levels of blurs on the stretch chains and the irradiance channels, the
                   weighted sum, `* irradiance`, `+ specular` and the vertical flip

Every arithmetic step is one float32 operation in the reference kernels' source order, so this agrees bit for bit with
the product kernels (csrc/sss_api.cu, built with -fmad=false).  The reference's own build contracts a*b+c into FMAs, so
it differs from both by rounding (tests/test_sss_cpu.py, tests/test_sss_gpu.py).

Reference quirks kept: int() truncates toward zero, so a tap in (-1, 0) extrapolates between pixels 0 and 1; a tap wholly
past an edge contributes (x - c) v + (c - x) v = 0; a neighbour <= 1e-6 (compared in double) is replaced by the centre
value; a centre value <= 0 writes 0; the y kernel clamps rows against the width, not the height.
"""
import math

import numpy as np

F32 = np.float32
TAP_NUM = 7                                         # lighting.py:117
GAUSSIAN_BASIS = (0, 25, 100, 400)                  # lighting.py:113: level variances 25, 75, 300
WEIGHTS = ((0.7, 0.2, 0.1), (0.1, 0.2, 0.7), (0.1, 0.2, 0.7))   # lighting.py:123-126, [channel][level]


def taps(v, tap_num=TAP_NUM):
    """(Gauss [tap_num] float32, GaussWidth float32) of gaussian_blur(.., tap_num, v, ..): Python doubles stored as
    float32 (gaussian_blur.py:7-13, 25-26)."""
    width = math.sqrt(v)
    g1 = lambda r: math.exp(-r ** 2 / (2 * v)) / math.sqrt(2 * math.pi * v)
    return np.array([width * g1(-width * ((tap_num - 1) / 2 - i)) for i in range(tap_num)], F32), F32(width)


def levels(basis=GAUSSIAN_BASIS):
    """The incremental variances of lighting.py:137-138."""
    return [basis[i + 1] - basis[i] for i in range(len(basis) - 1)]


def stretch(world):
    """world [H, W, 3] -> (stretchU, stretchV) [H, W] float32, clamped to [0, 1]."""
    w7 = np.asarray(world, F32) * F32(7)
    right = np.concatenate([w7, w7[:, -1:]], axis=1)[:, 1:]
    down = np.concatenate([w7, w7[-1:]], axis=0)[1:]
    out = []
    for nb in (right, down):
        d = w7 - nb
        s = d[..., 0] * d[..., 0]
        s = s + d[..., 1] * d[..., 1]
        s = s + d[..., 2] * d[..., 2]
        with np.errstate(divide="ignore"):
            out.append(np.clip(F32(1) / np.sqrt(s), F32(0), F32(1)).astype(F32))
    return tuple(out)


def _f2i(x):
    """CUDA's float -> int conversion (cvt.rzi.s32.f32): truncation toward zero, saturating, NaN -> 0."""
    x = np.where(np.isnan(x), F32(0), x).astype(np.float64)
    return np.trunc(np.clip(x, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def blur(image, mod, gauss, width, dim):
    """One _blur_for_SSS call on a single-channel map: dim 1 = gaussain_blur_x_Kernel, dim 0 = gaussain_blur_y_Kernel.
    image, mod [H, W]; gauss [7] float32; width = GaussWidth.  Returns [H, W] float32."""
    img = np.asarray(image, F32)
    mod = np.asarray(mod, F32)
    H, W = img.shape
    bound = W - 1                                    # both kernels clamp against w - 1
    c = np.broadcast_to(np.arange(W)[None, :] if dim == 1 else np.arange(H)[:, None], (H, W))
    step = F32(width) * mod
    x = c.astype(F32) - step * F32(TAP_NUM - 1) / F32(2)
    v = np.zeros((H, W), F32)
    for k in range(TAP_NUM):
        t = _f2i(x)
        x1 = np.clip(t, 0, bound)
        x2 = np.clip(t + 1, 0, bound)
        v1 = np.take_along_axis(img, x1, axis=dim)
        v2 = np.take_along_axis(img, x2, axis=dim)
        v1 = np.where(v1.astype(np.float64) > 1e-6, v1, img)
        v2 = np.where(v2.astype(np.float64) > 1e-6, v2, img)
        interpolation = (x - x1.astype(F32)) * v2 + (x2.astype(F32) - x) * v1
        v = v + interpolation * F32(gauss[k])
        x = x + step
    return np.where(img > 0, v, F32(0)).astype(F32)


def blur_pyramid(stretch_u, stretch_v, irradiance, specular, basis=GAUSSIAN_BASIS, weights=WEIGHTS):
    """lighting.py:113-150 from the clamped stretch maps [H, W] and the irradiance / specular maps [H, W, 3]: the final
    map [H, W, 3], already flipped vertically.  The stretch chains are computed once (the reference recomputes them for
    every channel, with the same result)."""
    irradiance = np.asarray(irradiance, F32)
    su, sv = np.asarray(stretch_u, F32), np.asarray(stretch_v, F32)
    irr = [irradiance[..., j].copy() for j in range(3)]
    final = np.zeros(irradiance.shape, F32)
    for i, v in enumerate(levels(basis)):
        g, w = taps(v)
        su = blur(su, su, g, w, 1)
        irr = [blur(x, su, g, w, 1) for x in irr]
        sv = blur(sv, sv, g, w, 0)
        irr = [blur(x, sv, g, w, 0) for x in irr]
        for j in range(3):
            final[..., j] = final[..., j] + F32(weights[j][i]) * irr[j]
    final = final * irradiance
    final = final + np.asarray(specular, F32)
    return np.ascontiguousarray(final[::-1])
