"""CPU oracle of the texture-atlas export (TEST INFRASTRUCTURE; product code never imports it).

numpy restatement of both kernels of jrender_b200/csrc/texture_atlas_api.cu:
  texture_atlas_softras  <- create_texture_image_cuda_kernel, jrender/io/utils/create_texture_image.py:13-73 (tile of
                            pixel :25-29, face_inv / (den + eps) :42-51, clamped and normalised weights :53-62 with the
                            double-literal clamp `max(min(w, 1.), 0.)`, texel pick :64-72), texel index clamped to the
                            face's own texels like the product;
  texture_atlas_n3mr     <- the same weights, then the NMR forward sampler's trilinear 8-tap fetch
                            (jrender/renderer/dr/n3mr/cuda/rasterize.py:267-293) at p_k = clamp(w_k (ts-1), 0, ts-1-1e-3).
float32 throughout, every operation in the kernels' order (the product is built with -fmad=false, so there is no
contraction to model).  Pinned against the reference's own kernel compiled by oracle/build_ref_atlas.py and run on a
GPU (named in each file's provenance): tests/golden/ref_atlas_gpu_*.npz (generator oracle/make_ref_atlas_golden.py).

Both functions return the image as the kernel writes it, [H, W, 3] with row 0 at the top; create_texture_image flips it.
"""
import numpy as np

from oracle.numbers import cuda_int, fmaxf, fminf

f32 = np.float32
EPS = f32(1e-5)          # save_obj.py:22
NMR_TEX_EPS = f32(1e-3)  # the NMR sampler's clamp eps at the Renderer's default (renderer.py:12)


def _count(stats, key, n):
    if stats is not None:
        stats[key] = stats.get(key, 0) + int(n)


def tile_weights(tile_vertices, texture_res_out, tile_width, image_height, image_width, stats=None):
    """Per pixel of the [H, W] image: face index fn (>= nf for unused tiles) and the clamped, normalised weights w [H*W, 3]
    of the pixel in its face's tile triangle (pixels of unused tiles get w = 0).  `stats` (a dict, optional) counts
    degenerate tiles (den + eps == 0: the kernel divides by zero), non-finite weights before the clamp and unused
    pixels."""
    nf = tile_vertices.shape[0]
    npix = image_height * image_width
    i = np.arange(npix, dtype=np.int64)
    x, y = i % image_width, i // image_width
    fn = x // texture_res_out + (y // texture_res_out) * tile_width
    used = fn < nf
    w = np.zeros((npix, 3), f32)
    p = np.asarray(tile_vertices, f32).reshape(nf, 3, 2)[fn[used]]
    p0x, p0y, p1x, p1y, p2x, p2y = (p[:, k // 2, k % 2] for k in range(6))
    inv = np.stack([p1y - p2y, p2x - p1x, p1x * p2y - p2x * p1y,
                    p2y - p0y, p0x - p2x, p2x * p0y - p0x * p2y,
                    p0y - p1y, p1x - p0x, p0x * p1y - p1x * p0y], axis=1)
    with np.errstate(all="ignore"):
        den = p2x * (p0y - p1y) + p0x * (p1y - p2y) + p1x * (p2y - p0y)
        inv = inv / (den + EPS)[:, None]
        xf, yf = x[used].astype(f32), y[used].astype(f32)
        wu = np.stack([inv[:, 3 * k + 0] * xf + inv[:, 3 * k + 1] * yf + inv[:, 3 * k + 2] for k in range(3)], axis=1)
    if stats is not None:
        pn = np.asarray(tile_vertices, f32).reshape(nf, 3, 2)
        with np.errstate(all="ignore"):
            dn = pn[:, 2, 0] * (pn[:, 0, 1] - pn[:, 1, 1]) + pn[:, 0, 0] * (pn[:, 1, 1] - pn[:, 2, 1]) + pn[:, 1, 0] * (pn[:, 2, 1] - pn[:, 0, 1])
        _count(stats, "degenerate_tiles", ((dn + EPS) == 0).sum())
        _count(stats, "nonfinite_weights", (~np.isfinite(wu)).sum())
        _count(stats, "unused_pixels", (~used).sum())
    wu = fmaxf(fminf(wu, f32(1)), f32(0))                 # fmin / fmax: NaN -> the other operand, as the GPU's
    w_sum = (wu[:, 0] + wu[:, 1]) + wu[:, 2]
    w[used] = wu / (w_sum + EPS)[:, None]
    return fn, used, w


def texture_atlas_softras(tile_vertices, textures, texture_res_out, tile_width, image_height, image_width, stats=None):
    """create_texture_image_cuda_kernel (create_texture_image.py:13-73): tile_vertices [nf, 3, 2] pixel units,
    textures [nf, R*R, 3] -> image [H, W, 3] float32 (unused tiles 1)."""
    textures = np.asarray(textures, f32)
    nf, T = textures.shape[:2]
    R = int(round(np.sqrt(T)))
    assert R * R == T
    fn, used, w = tile_weights(tile_vertices, texture_res_out, tile_width, image_height, image_width, stats)
    w0, w1 = w[used, 0], w[used, 1]
    w_x, w_y = cuda_int(w0 * f32(R)), cuda_int(w1 * f32(R))
    lower = ((w0 + w1) * f32(R) - w_x.astype(f32)) - w_y.astype(f32) <= f32(1)
    t = np.where(lower, w_y * R + w_x, (R - 1 - w_y) * R + (R - 1 - w_x))
    t = np.clip(t, 0, R * R - 1)
    img = np.ones((image_height * image_width, 3), f32)
    img[used] = textures[fn[used], t]
    return img.reshape(image_height, image_width, 3)


def texture_atlas_n3mr(tile_vertices, textures, texture_res_out, tile_width, image_height, image_width, stats=None):
    """NMR textures [nf, ts, ts, ts, 3]: the same weights, trilinear fetch of rasterize.py:267-293 at depth / z_k = 1."""
    textures = np.asarray(textures, f32)
    nf, ts = textures.shape[0], textures.shape[1]
    assert ts >= 2
    fn, used, w = tile_weights(tile_vertices, texture_res_out, tile_width, image_height, image_width, stats)
    tif = fmaxf(w[used] * f32(ts - 1), f32(0))
    tif = fminf(tif, f32(ts - 1) - NMR_TEX_EPS)
    ti = cuda_int(tif)
    frac = tif - ti.astype(f32)
    tex = textures.reshape(nf, ts ** 3, 3)
    fu = fn[used]
    c = np.zeros((fu.shape[0], 3), f32)
    for pn in range(8):
        wt = np.ones(fu.shape[0], f32)
        idx = np.zeros(fu.shape[0], np.int64)
        for k in range(3):
            if (pn >> k) % 2 == 0:
                wt = wt * (f32(1) - frac[:, k])
                tk = ti[:, k]
            else:
                wt = wt * frac[:, k]
                tk = ti[:, k] + 1
            idx = idx * ts + tk
        c = c + wt[:, None] * tex[fu, idx]
    img = np.ones((image_height * image_width, 3), f32)
    img[used] = c
    return img.reshape(image_height, image_width, 3)


def atlas_layout(num_faces, texture_res):
    """create_texture_image's tile layout (save_obj.py:8-21) with the integer tile row: (tile_vertices [nf, 3, 2] float32
    in pixel units, tile_width, tile_height)."""
    tile_width = int((num_faces - 1.) ** 0.5) + 1
    tile_height = int((num_faces - 1.) / tile_width) + 1
    n = np.arange(num_faces)
    col, row = n % tile_width, n // tile_width
    R = texture_res
    v = np.zeros((num_faces, 3, 2), np.float64)
    v[:, 0, 0], v[:, 0, 1] = col * R + R / 2, row * R + 1
    v[:, 1, 0], v[:, 1, 1] = col * R + 1, (row + 1) * R - 1 - 1
    v[:, 2, 0], v[:, 2, 1] = (col + 1) * R - 1 - 1, (row + 1) * R - 1 - 1
    return v.astype(f32), tile_width, tile_height
