"""CPU oracle of the texture-bake kernels (TEST INFRASTRUCTURE; product code never imports it).

numpy float32 emulation of jrender_b200/csrc/bake_api.cu, operation by operation, so that the kernels' outputs can be
predicted bit for bit (the library is built with -fmad=false and the bake uses no transcendental function):
  bake_textures_for_softras  <- k_bake_textures_softras (load_textures.py:11-69): barycentric sample point per texel
                                (:29-37, double quotients narrowed to float, w2 = (float)(1. - w0 - w1)), UV -> image
                                position in float32 (:42-45), bilinear weights pos - (float)(int)pos in float32, flat tap
                                indices clamped to [0, H*W - 1] at both ends, each colour summed from +0.0 in tap order;
  softras_backward_sums      <- k_bake_textures_softras_bwd: the float32 atomicAdd operands g * w of the same taps;
  bake_textures_for_n3mr     <- k_bake_textures_n3mr (load_textures.py:103-246): every texel wraps the ORIGINAL UVs
                                (ref_mod, fminf / fmaxf), clamps its +1 taps, rounds half away from zero on the double in
                                nearest mode, and writes zeros under CLAMP_TO_BORDER.
Conversions are CUDA's (numbers.cuda_int: truncation, saturation, NaN -> 0), not numpy's.  Each step goes through a
module-level helper, so that tests/test_texture_edges_cpu.py can swap one for a subtly wrong variant and show that the
GPU tests would notice.  `stats` (a dict, optional) counts the edges a call went through.

Pinned against the reference's own kernels compiled by oracle/build_ref.py and run on a GPU (named in each file's
provenance): tests/golden/ref_gpu_bake_random40_R5.npz and ref_gpu_bake_n3mr_*.npz (generator oracle/make_ref_golden.py
--bake-only).  Those builds contract a*b+c, so those comparisons keep a tolerance.
"""
import numpy as np

from oracle.numbers import cuda_int, fmaxf, fminf

F32 = np.float32
CHUNK = 1 << 20     # texels per emulation step (keeps the [texels, 4, 3] temporaries small)
REPEAT, MIRRORED_REPEAT, CLAMP_TO_EDGE, CLAMP_TO_BORDER = range(4)
INT_RANGE = 2.0 ** 31


def _count(stats, key, n):
    if stats is not None:
        stats[key] = stats.get(key, 0) + int(n)


def _frac(pos):
    """The bilinear weight pos - (int)pos: the int converted back to float (rounded once |int| > 2^24) and subtracted
    in float32."""
    return (pos - cuda_int(pos).astype(F32)).astype(F32)


def _clamp_index(j, n):
    """Flat tap index clamped to the image at both ends (a documented deviation: the reference reads out of bounds)."""
    return np.clip(j, 0, n - 1)


def _gather(flat, idx):
    return flat[idx]


def _sum4(p):
    """p [..., 4, 3]: ((((+0 + p0) + p1) + p2) + p3) in float32, the kernel's `float c = 0; c += ...` in tap order."""
    c = F32(0) + p[..., 0, :]
    for j in range(1, 4):
        c = c + p[..., j, :]
    return c


def _conversions(stats, *pos):
    for p in pos:
        _count(stats, "nan_conversions", np.isnan(p).sum())
        _count(stats, "saturated_conversions", (np.abs(p) >= INT_RANGE).sum())


def sample_weights(R):
    """w0, w1, w2 [R*R] float32 of the texels' sample points (load_textures.py:29-37), the kernel's promotions."""
    wy, wx = np.divmod(np.arange(R * R), R)
    lower = (wx + wy) < R
    w0 = np.where(lower, (wx + 1. / 3.) / R, ((R - 1. - wx) + 2. / 3.) / R).astype(F32)
    w1 = np.where(lower, (wy + 1. / 3.) / R, ((R - 1. - wy) + 2. / 3.) / R).astype(F32)
    w2 = (1. - w0.astype(np.float64) - w1.astype(np.float64)).astype(F32)
    return w0, w1, w2


def softras_taps(faces_uv, R, H, W, stats=None):
    """Per texel of [nf, R*R]: the four flat tap indices [nf, T, 4] (i00, i10, i01, i11, clamped) and their float32
    weights [nf, T, 4] (wx0 wy0, wx0 wy1, wx1 wy0, wx1 wy1), as k_bake_textures_softras and its backward form them."""
    w0, w1, w2 = sample_weights(R)
    f = np.asarray(faces_uv, F32).reshape(-1, 3, 2)
    n = H * W
    with np.errstate(all="ignore"):
        pos_x = ((f[:, None, 0, 0] * w0 + f[:, None, 1, 0] * w1) + f[:, None, 2, 0] * w2) * F32(W - 1)
        pos_y = ((f[:, None, 0, 1] * w0 + f[:, None, 1, 1] * w1) + f[:, None, 2, 1] * w2) * F32(H - 1)
        pos_y1 = pos_y + F32(1)
        ix, iy, iy1 = cuda_int(pos_x), cuda_int(pos_y), cuda_int(pos_y1)
        wx1, wy1 = _frac(pos_x), _frac(pos_y)
        wx0, wy0 = F32(1) - wx1, F32(1) - wy1
        wts = np.stack([wx0 * wy0, wx0 * wy1, wx1 * wy0, wx1 * wy1], -1)
    raw = np.stack([iy * W + ix, iy1 * W + ix, iy * W + ix + 1, iy1 * W + ix + 1], -1)
    if stats is not None:
        _conversions(stats, pos_x, pos_y, pos_y1)
        inside = (raw >= 0) & (raw < n)
        _count(stats, "clamped_taps", (~inside).sum())
        col = np.stack([ix, ix, ix + 1, ix + 1], -1)
        _count(stats, "row_wraps", (inside & ((col < 0) | (col >= W))).sum())
        with np.errstate(invalid="ignore"):
            _count(stats, "extrapolating_weights", (np.isfinite(wts) & ((wts < 0) | (wts > 1))).sum())
        _count(stats, "texels", wts.shape[0] * wts.shape[1])
    return _clamp_index(raw, n), wts


def _chunks(is_update, T):
    faces = np.flatnonzero(np.asarray(is_update) != 0)
    step = max(1, CHUNK // T)
    for s in range(0, len(faces), step):
        yield faces[s:s + step]


def bake_textures_for_softras(image, faces_uv, textures, is_update, stats=None):
    """k_bake_textures_softras: image [H, W, 3] (already flipped vertically by the caller), faces_uv [nf, 3, 2],
    textures [nf, R*R, 3] -> a copy of textures with the faces where is_update != 0 baked."""
    out = np.array(textures, F32)
    nf, T = out.shape[:2]
    R = int(round(np.sqrt(T)))
    assert R * R == T
    H, W = image.shape[:2]
    flat = np.asarray(image, F32).reshape(-1, 3)
    uv = np.asarray(faces_uv, F32).reshape(nf, 3, 2)
    for fs in _chunks(is_update, T):
        idx, wts = softras_taps(uv[fs], R, H, W, stats)
        with np.errstate(all="ignore"):
            c = _sum4(_gather(flat, idx) * wts[..., None])
        _count(stats, "nan_texels", np.isnan(c).any(-1).sum())
        _count(stats, "inf_texels", np.isinf(c).any(-1).sum())
        out[fs] = c
    return out


def softras_backward_sums(grad_textures, faces_uv, is_update, H, W):
    """k_bake_textures_softras_bwd's atomicAdd operands, the float32 products g * w, summed per pixel in float64:
    'exact' [H, W, 3] (NaN / +-inf where IEEE addition of those terms in any order gives them), 'nonzero' [H, W, 3]
    (the count of terms that are not +-0) and 'taps' [H, W] (the count of taps landing on the pixel)."""
    g = np.asarray(grad_textures, F32)
    nf, T = g.shape[:2]
    R = int(round(np.sqrt(T)))
    uv = np.asarray(faces_uv, F32).reshape(nf, 3, 2)
    n = H * W
    exact = np.zeros((n, 3))
    nonzero = np.zeros((n, 3), np.int64)
    taps = np.zeros(n, np.int64)
    for fs in _chunks(is_update, T):
        idx, wts = softras_taps(uv[fs], R, H, W)
        with np.errstate(all="ignore"):
            terms = g[fs][:, :, None, :] * wts[..., None]           # [f, T, 4, 3] float32
        i = idx.reshape(-1)
        terms = terms.reshape(-1, 3)
        taps += np.bincount(i, minlength=n)
        for k in range(3):
            with np.errstate(invalid="ignore"):
                exact[:, k] += np.bincount(i, weights=terms[:, k].astype(np.float64), minlength=n)
            nonzero[:, k] += np.bincount(i, weights=(terms[:, k] != 0), minlength=n).astype(np.int64)
    return dict(exact=exact.reshape(H, W, 3), nonzero=nonzero.reshape(H, W, 3), taps=taps.reshape(H, W))


def bake_textures_for_softras_f64(image, faces_uv, textures, is_update):
    """The host goldens' stand-in for the reference's own bake kernel (make_ref_host_sss_golden.py,
    make_ref_host_normal_map_golden.py): the float32 sample positions of bake_textures_for_softras, then the bilinear
    weights and fetch in float64, rounded to float32 once.  Not the product kernel's arithmetic (it differs from
    bake_textures_for_softras by about an ulp on a third of the texels), and not the reference build's bit pattern
    either (that build contracts a*b+c): it is kept so that the committed host goldens regenerate bit for bit."""
    out = np.array(textures, F32)
    nf, T = out.shape[:2]
    R = int(round(np.sqrt(T)))
    H, W = image.shape[:2]
    w0, w1, w2 = sample_weights(R)
    f = np.asarray(faces_uv, F32).reshape(nf, 3, 2)
    pos_x = ((f[:, None, 0, 0] * w0 + f[:, None, 1, 0] * w1) + f[:, None, 2, 0] * w2) * F32(W - 1)
    pos_y = ((f[:, None, 0, 1] * w0 + f[:, None, 1, 1] * w1) + f[:, None, 2, 1] * w2) * F32(H - 1)
    ix, iy, iy1 = cuda_int(pos_x), cuda_int(pos_y), cuda_int(pos_y + F32(1))
    wx1, wy1 = pos_x - ix, pos_y - iy                         # float32 - int64: float64 from here on
    wx0, wy0 = 1 - wx1, 1 - wy1
    flat = np.asarray(image, F32).reshape(-1, 3)
    n = flat.shape[0]

    def px(j):
        return flat[np.clip(j, 0, n - 1)]
    c = (px(iy * W + ix) * (wx0 * wy0)[..., None] + px(iy1 * W + ix) * (wx0 * wy1)[..., None] +
         px(iy * W + ix + 1) * (wx1 * wy0)[..., None] + px(iy1 * W + ix + 1) * (wx1 * wy1)[..., None]).astype(F32)
    m = np.asarray(is_update) != 0
    out[m] = c[m]
    return out


def _ref_mod(x, y):
    """load_textures.py:112-119: x > 0 -> fmod(x, y), else y + fmod(x, y) (float32; -0.0 and 0 give y, NaN and +-inf
    give NaN)."""
    x = np.asarray(x, F32)
    y = F32(y)
    with np.errstate(invalid="ignore"):
        return np.where(x > 0, np.fmod(x, y), (y + np.fmod(x, y)).astype(F32)).astype(F32)


def _wrap(v, mode):
    """The texture_wrapping of load_textures.py:151-173, applied to the face's ORIGINAL UVs."""
    if mode == REPEAT:
        return _ref_mod(v, 1)
    if mode == MIRRORED_REPEAT:
        return np.where(_ref_mod(v, 2) < 1, _ref_mod(v, 1), (F32(1) - _ref_mod(v, 1)).astype(F32))
    if mode == CLAMP_TO_EDGE:
        return fmaxf(fminf(v, F32(1)), F32(0))
    return v


def _round_half_away(v):
    """C round() on the double promotion of a float32 value: half away from zero (exact for float32 inputs)."""
    v = np.asarray(v, np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(v < 0, -np.floor(0.5 - v), np.floor(v + 0.5))


def n3mr_sample_weights(ts):
    """dim0, dim1, dim2 [ts^3] float32 (load_textures.py:138-146): double quotients narrowed, then divided by their
    float32 sum where it is positive."""
    i = np.arange(ts ** 3)
    d0 = ((i // (ts * ts)) % ts / (ts - 1.)).astype(F32)
    d1 = ((i // ts) % ts / (ts - 1.)).astype(F32)
    d2 = (i % ts / (ts - 1.)).astype(F32)
    s = (d0 + d1) + d2
    pos = s > 0
    sd = np.where(pos, s, F32(1))
    return tuple(np.where(pos, d / sd, d).astype(F32) for d in (d0, d1, d2))


def bake_textures_for_n3mr(image, faces_uv, textures, is_update, texture_wrapping=0, use_bilinear=True, stats=None):
    """k_bake_textures_n3mr: image [H, W, 3] (already flipped vertically by the caller), faces_uv [nf, 3, 2], textures
    [nf, ts, ts, ts, 3] -> a copy with the faces where is_update != 0 baked.  The reference wraps the face's UVs in
    place from all of the face's threads (a race); like the product, every texel here wraps the original UVs once."""
    out = np.array(textures, F32)
    nf, ts = out.shape[0], out.shape[1]
    assert ts >= 2
    H, W = image.shape[:2]
    m = np.asarray(is_update) != 0
    if texture_wrapping == CLAMP_TO_BORDER:
        out[m] = 0
        return out
    d0, d1, d2 = n3mr_sample_weights(ts)
    f = _wrap(np.asarray(faces_uv, F32).reshape(nf, 6)[m], texture_wrapping)
    _count(stats, "nan_uvs_after_wrap", np.isnan(f).sum())
    with np.errstate(all="ignore"):
        pos_x = ((f[:, None, 0] * d0 + f[:, None, 2] * d1) + f[:, None, 4] * d2) * F32(W - 1)
        pos_y = ((f[:, None, 1] * d0 + f[:, None, 3] * d1) + f[:, None, 5] * d2) * F32(H - 1)
    img = np.asarray(image, F32)
    if use_bilinear:
        with np.errstate(all="ignore"):
            ix, iy, iy1 = cuda_int(pos_x), cuda_int(pos_y), cuda_int(pos_y + F32(1))
            wx1, wy1 = _frac(pos_x), _frac(pos_y)
            wx0, wy0 = F32(1) - wx1, F32(1) - wy1
            wts = np.stack([wx0 * wy0, wx0 * wy1, wx1 * wy0, wx1 * wy1], -1)
        x0, y0 = np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)
        x1, y1 = np.minimum(ix + 1, W - 1), np.minimum(iy1, H - 1)
        assert (x1 >= 0).all() and (y1 >= 0).all()     # wrapped UVs are in [0, 1] or NaN
        if stats is not None:
            _conversions(stats, pos_x, pos_y)
            _count(stats, "clamped_taps", (ix + 1 > W - 1).sum() + (iy1 > H - 1).sum())
        ys, xs = np.stack([y0, y1, y0, y1], -1), np.stack([x0, x0, x1, x1], -1)
        with np.errstate(all="ignore"):
            c = _sum4(img[ys, xs] * wts[..., None])
    else:
        xi = np.clip(cuda_int(_round_half_away(pos_x)), 0, W - 1)
        yi = np.clip(cuda_int(_round_half_away(pos_y)), 0, H - 1)
        if stats is not None:
            _conversions(stats, pos_x, pos_y)
            _count(stats, "rounded_halves", (np.abs(pos_x - np.trunc(pos_x)) == 0.5).sum())
        c = img[yi, xi]
    _count(stats, "nan_texels", np.isnan(c).any(-1).sum())
    out[m] = c.reshape((-1, ts, ts, ts, 3))
    return out
