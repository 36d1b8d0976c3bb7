"""Seeded scenes for the SoftRas backward (k_softras_backward_lane), each aimed at a place where a per-lane walk with
warp merges and vector atomics can go wrong.  Every case is (name, face_vertices, textures, Params, upstream gradient);
test_softras_backward_cpu.py checks from the oracle's id lists that each one reaches what it is built for, and
test_softras_backward_gpu.py holds the kernel to the oracle's per-entry bound on all of them.

Geometry is laid out in pixel units: col_edge(c, H) is the x of the boundary between columns c - 1 and c, row_edge(r, H)
the y of the boundary between rows r - 1 and r (row 0 at the top).  The kernel's warps cover 8 x 4 pixels: lanes ^1
are horizontal neighbours (columns 0|1 of a pair), lanes ^8 vertical ones (rows 3|4 lie in different warps)."""
import numpy as np

from jrender_b200 import workloads as wl
from oracle import softras as osr

WARP_SIZES = (1, 7, 8, 9, 31, 33, 100)
LIST_KS = (1, 2, 3, 16, 33, 64)
TEXTURE_RES = (1, 2, 3, 5)   # T = 1, 4, 9, 25


def col_edge(c, H):
    return 2.0 * c / H - 1.0


def row_edge(r, H):
    return 1.0 - 2.0 * r / H


def px_x(c, H):
    return (2.0 * c + 1.0 - H) / H


def px_y(r, H):
    return (2.0 * (H - 1 - r) + 1.0 - H) / H


def rect(x0, x1, y0, y1, z):
    """two triangles covering [x0, x1] x [y0, y1] at depth z"""
    return [[[x0, y0, z], [x1, y0, z], [x1, y1, z]], [[x0, y0, z], [x1, y1, z], [x0, y1, z]]]


def sharp_sigma(H):
    """a sigma whose border sqrt(dist_eps sigma) is 0.7 pixel: coverage ends at the pixel boundary it is drawn on, and
    the pixels next to an edge have 1 - D near 1e-8, under the alpha-prod floor"""
    return 0.49 / (float(osr.dist_eps_logit(1e-4)) * H * H)


def grad(shape, seed):
    B, H = shape[0], shape[1]
    return np.random.default_rng(seed).uniform(-1, 1, (B, 4, H, H)).astype(np.float32)


def _tex(nf, T, seed):
    return np.random.default_rng(seed).random((1, nf, T, 3), dtype=np.float32)


def merge_scene(H):
    """Coverage boundaries between columns 0|1 and 7|8 and between rows 3|4 (and mirrored ones), from faces of
    different ids and depths, so that lanes ^1 and ^8 see the same face, different faces, and a face against an empty
    slot, at several slots."""
    f = []
    f += rect(col_edge(1, H), 1.5, -1.5, row_edge(4, H), 2.0)              # from column 1, from row 4
    f += rect(-1.5, col_edge(8, H), row_edge(H - 4, H), 1.5, 3.0)          # up to column 7, up to row H-5
    f += rect(-1.5, 1.5, -1.5, 1.5, 4.0)                                   # everywhere, behind
    f += rect(col_edge(min(7, H), H), col_edge(min(9, H), H), -1.5, 1.5, 2.5)   # columns 7, 8
    fv = np.array([f], np.float32)
    return fv, _tex(fv.shape[1], 1, H)


def checkerboard_scene(H=16):
    """one small face per pixel, depths alternating like a checkerboard: neighbouring lanes never hold the same face"""
    f = []
    for r in range(H):
        for c in range(H):
            x, y, e = px_x(c, H), px_y(r, H), 0.6 / H
            f.append([[x - e, y - e, 2.0 + (r + c) % 2], [x + e, y - e, 2.0 + (r + c) % 2], [x, y + e, 2.0 + (r + c) % 2]])
    fv = np.array([f], np.float32)
    return fv, _tex(fv.shape[1], 1, 3)


def full_warp_scene(H=16, duplicate=False):
    """one face over the whole image (every lane of every warp holds it: both merge levels fire everywhere); with
    duplicate, a second face with identical vertices and a different id: identical terms that must not merge"""
    f = [[[-1.0, -1.2, 2.0], [3.0, -1.2, 2.0], [-1.0, 3.0, 2.0]]]
    fv = np.array([f + f if duplicate else f], np.float32)
    return fv, np.repeat(_tex(1, 1, 4), fv.shape[1], axis=1)


def stack_scene(H=56, layers=70):
    """`layers` nested triangles of decreasing size: per-pixel list lengths run from 0 to `layers`, so lists end at
    every slot, the central ones are full (no -1 terminator) for K <= layers, and neighbouring lanes end at different
    slots.  A lone one-pixel face in the top-right warp gives a warp with a single non-empty lane."""
    rng = np.random.default_rng(11)
    f = []
    for i in range(layers):
        s = 0.95 * (1.0 - i / (layers + 8.0))
        cx, cy = rng.uniform(-0.03, 0.03, 2)
        z = float(rng.uniform(2.0, 6.0))
        f.append([[cx - s, cy - s, z], [cx + s, cy - 0.8 * s, z], [cx, cy + s, z]])
    x, y, e = px_x(H - 3, H), px_y(1, H), 0.4 / H
    f.append([[x - e, y - e, 2.0], [x + e, y - e, 2.0], [x, y + e, 2.0]])
    fv = np.array([f], np.float32)
    return fv, _tex(fv.shape[1], 1, 5)


def texel_scene(R, H=32):
    """right triangles with vertices on pixel centres and legs of 8 / 16 pixels: the barycentric coordinates of the
    pixels are exact binary fractions, so w * R lands exactly on texel boundaries (R = 2 and 4); R = 3, 5 see the same
    geometry.  Next to them, the sphere's faces."""
    sph, _ = wl.make_scene(280, batch=1, distance=4.0)
    f = []
    for (c0, r0, n, z) in ((2, 29, 16, 1.5), (20, 13, 8, 1.6), (20, 29, 8, 1.7)):
        x0, y0 = px_x(c0, H), px_y(r0, H)
        d = 2.0 * n / H
        f.append([[x0, y0, z], [x0 + d, y0, z], [x0, y0 + d, z]])
    fv = np.concatenate([np.array([f], np.float32), sph], axis=1)
    return fv, _tex(fv.shape[1], R * R, 6 + R)


def batch_scene():
    """B = 3 with different scenes per element and an odd face count; element 2 renders an empty image"""
    a, ta = wl.random_triangles(1, 101, seed=21)
    b, tb = wl.random_triangles(1, 101, seed=22, scale=0.2)
    c, tc = wl.random_triangles(1, 101, seed=23)
    c[..., 0] += 10.0
    return np.concatenate([a, b, c]), np.concatenate([ta, tb, tc])


def cases():
    """[(name, fv, tex, Params, upstream gradient)]"""
    out = []
    for H in WARP_SIZES:
        fv, tex = merge_scene(H)
        out.append(("merge_H%d" % H, fv, tex, osr.Params(image_size=H, sigma_val=sharp_sigma(max(H, 8)))))
    fv, tex = checkerboard_scene()
    out.append(("checkerboard", fv, tex, osr.Params(image_size=16, sigma_val=sharp_sigma(16))))
    for dup in (False, True):
        fv, tex = full_warp_scene(duplicate=dup)
        out.append(("full_warp" + ("_duplicate" if dup else ""), fv, tex, osr.Params(image_size=16, sigma_val=1e-3)))
    fv, tex = stack_scene()
    for K in LIST_KS:
        out.append(("stack_K%d" % K, fv, tex, osr.Params(image_size=56, sigma_val=1e-4, max_faces_per_pixel_for_grad=K)))
    for R in TEXTURE_RES:
        fv, tex = texel_scene(R)
        for rgb in ("softmax", "hard"):
            out.append(("texel_R%d_%s" % (R, rgb), fv, tex, osr.Params(image_size=32, sigma_val=3e-5, aggr_func_rgb=rgb)))
    fv, tex = wl.make_scene(280, batch=1, texture_type="vertex")
    for rgb in ("softmax", "hard"):
        out.append(("vertex_%s" % rgb, fv, tex, osr.Params(image_size=32, texture_type="vertex", aggr_func_rgb=rgb,
                                                            sigma_val=3e-5)))
    fv, tex = wl.make_scene(280, batch=1)
    for dist in ("hard", "barycentric", "euclidean"):
        for rgb in ("hard", "softmax", "none"):
            for alpha in ("hard", "sum", "prod"):
                out.append(("mode_%s_%s_%s" % (dist, rgb, alpha), fv, tex,
                            osr.Params(image_size=32, dist_func=dist, aggr_func_rgb=rgb, aggr_func_alpha=alpha,
                                       sigma_val=3e-5)))
    fv, tex = batch_scene()
    out.append(("batch3_odd_nf_empty", fv, tex, osr.Params(image_size=24, sigma_val=1e-4)))
    return [(n, fv, tex, P, grad((fv.shape[0], P["image_size"]), i)) for i, (n, fv, tex, P) in enumerate(out)]


def case(name):
    return next(c for c in cases() if c[0] == name)
