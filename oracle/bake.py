"""CPU oracle of the SoftRas texture bake (TEST INFRASTRUCTURE; product code never imports it).

numpy restatement of load_textures_cuda_kernel, jrender/io/utils/load_textures.py:11-69 (barycentric sample point per
texel :29-37, UV -> image position :42-45, bilinear fetch :46-58, same float / double promotions).  Pinned against the
reference's own kernel compiled by oracle/build_ref.py and run on a GPU (named in the file's provenance):
tests/golden/ref_gpu_bake_random40_R5.npz (generator oracle/make_ref_golden.py --bake-only).
"""
import numpy as np


def bake_textures_for_softras(image, faces_uv, textures, is_update):
    """load_textures.py:11-69.

    image [H,W,3] (already flipped vertically by the caller), faces_uv [nf,3,2],
    textures [nf,R*R,3] (returned updated where is_update != 0)."""
    nf, T = textures.shape[:2]
    R = int(np.sqrt(T))
    H, W = image.shape[:2]
    wy, wx = np.divmod(np.arange(T), R)
    lower = (wx + wy) < R
    w0 = np.where(lower, (wx + 1. / 3.) / R, ((R - 1. - wx) + 2. / 3.) / R).astype(np.float32)
    w1 = np.where(lower, (wy + 1. / 3.) / R, ((R - 1. - wy) + 2. / 3.) / R).astype(np.float32)
    w2 = (1. - w0.astype(np.float64) - w1.astype(np.float64)).astype(np.float32)
    f = faces_uv.astype(np.float32)
    pos_x = ((f[:, None, 0, 0] * w0 + f[:, None, 1, 0] * w1 + f[:, None, 2, 0] * w2) * np.float32(W - 1)).astype(np.float32)
    pos_y = ((f[:, None, 0, 1] * w0 + f[:, None, 1, 1] * w1 + f[:, None, 2, 1] * w2) * np.float32(H - 1)).astype(np.float32)
    ix, iy = pos_x.astype(np.int64), pos_y.astype(np.int64)       # C truncation; UVs are >= 0
    wx1 = pos_x - ix
    wx0 = 1 - wx1
    wy1 = pos_y - iy
    wy0 = 1 - wy1
    flat = image.reshape(-1, 3)
    n = flat.shape[0]
    iy1 = (pos_y + 1).astype(np.int64)

    def px(yy, xx):  # the reference indexes the flat buffer without clamping; keep in-bounds here
        return flat[np.clip(yy * W + xx, 0, n - 1)]
    c = (px(iy, ix) * (wx0 * wy0)[..., None] + px(iy1, ix) * (wx0 * wy1)[..., None] +
         px(iy, ix + 1) * (wx1 * wy0)[..., None] + px(iy1, ix + 1) * (wx1 * wy1)[..., None]).astype(np.float32)
    out = textures.copy()
    m = np.asarray(is_update) != 0
    out[m] = c[m]
    return out




def _ref_mod(x, y):
    """load_textures.py:112-119: x > 0 -> fmod(x, y), else y + fmod(x, y) (float32)."""
    x = x.astype(np.float32)
    y = np.float32(y)
    return np.where(x > 0, np.fmod(x, y), (y + np.fmod(x, y)).astype(np.float32)).astype(np.float32)


def bake_textures_for_n3mr(image, faces_uv, textures, is_update, texture_wrapping=0, use_bilinear=True):
    """load_textures.py:103-246 (load_textures_cuda_kernel of _load_textures_for_n3mr).

    image [H,W,3] (already flipped vertically by the caller), faces_uv [nf,3,2], textures [nf,ts,ts,ts,3] (returned updated
    where is_update != 0).  The reference wraps the face's UVs in place from all of the face's threads (a race); like the
    product, every texel here wraps the original UVs once.  Pinned against the reference's own kernel compiled from
    the reference (oracle/build_ref.py) and run on a GPU (named in each file's provenance): tests/golden/ref_gpu_bake_n3mr_*.npz
    (generator oracle/make_ref_golden.py --bake-only; its UVs avoid the race's non-fixed points)."""
    nf, ts = textures.shape[0], textures.shape[1]
    assert ts >= 2
    H, W = image.shape[:2]
    i = np.arange(ts ** 3)
    d0 = ((i // (ts * ts)) % ts / (ts - 1.)).astype(np.float32)        # :138-140, double division narrowed to float
    d1 = ((i // ts) % ts / (ts - 1.)).astype(np.float32)
    d2 = (i % ts / (ts - 1.)).astype(np.float32)
    s = ((d0 + d1).astype(np.float32) + d2).astype(np.float32)
    pos = s > 0
    sd = np.where(pos, s, np.float32(1))
    d0 = np.where(pos, (d0 / sd).astype(np.float32), d0)
    d1 = np.where(pos, (d1 / sd).astype(np.float32), d1)
    d2 = np.where(pos, (d2 / sd).astype(np.float32), d2)
    f = faces_uv.astype(np.float32).reshape(nf, 6)
    if texture_wrapping == 0:
        f = _ref_mod(f, 1)
    elif texture_wrapping == 1:
        f = np.where(_ref_mod(f, 2) < 1, _ref_mod(f, 1), (np.float32(1) - _ref_mod(f, 1)).astype(np.float32))
    elif texture_wrapping == 2:
        f = np.maximum(np.minimum(f, np.float32(1)), np.float32(0))
    out = textures.astype(np.float32).copy()
    m = np.asarray(is_update) != 0
    if texture_wrapping == 3:
        out[m] = 0
        return out
    f32 = np.float32

    def lin(a, b, c):   # (a*dim0 + b*dim1 + c*dim2), float32 products and sums in source order
        return (((a[:, None] * d0).astype(f32) + (b[:, None] * d1).astype(f32)).astype(f32) + (c[:, None] * d2).astype(f32)).astype(f32)
    pos_x = (lin(f[:, 0], f[:, 2], f[:, 4]) * f32(W - 1)).astype(f32)
    pos_y = (lin(f[:, 1], f[:, 3], f[:, 5]) * f32(H - 1)).astype(f32)
    if use_bilinear:
        ix, iy = pos_x.astype(np.int64), pos_y.astype(np.int64)
        wx1 = (pos_x - ix).astype(f32)
        wx0 = (1 - wx1).astype(f32)
        wy1 = (pos_y - iy).astype(f32)
        wy0 = (1 - wy1).astype(f32)
        x0, y0 = np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)
        x1 = np.minimum(ix + 1, W - 1)
        y1 = np.minimum((pos_y + f32(1)).astype(np.int64), H - 1)
        img = image.astype(f32)
        c = (img[y0, x0] * (wx0 * wy0).astype(f32)[..., None]).astype(f32)
        c = (c + (img[y1, x0] * (wx0 * wy1).astype(f32)[..., None]).astype(f32)).astype(f32)
        c = (c + (img[y0, x1] * (wx1 * wy0).astype(f32)[..., None]).astype(f32)).astype(f32)
        c = (c + (img[y1, x1] * (wx1 * wy1).astype(f32)[..., None]).astype(f32)).astype(f32)
    else:
        def rnd(v):   # C round(): half away from zero, on the double promotion
            v = v.astype(np.float64)
            return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)
        xi, yi = np.clip(rnd(pos_x), 0, W - 1), np.clip(rnd(pos_y), 0, H - 1)
        c = image.astype(f32)[yi, xi]
    c = c.reshape(nf, ts, ts, ts, 3)
    out[m] = c[m]
    return out
