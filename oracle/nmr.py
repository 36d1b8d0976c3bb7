"""numpy front end of the CPU NMR (n3mr) oracle (TEST INFRASTRUCTURE, not product code).

Mirrors the host side of the reference Function, jrender/renderer/dr/n3mr/n3mr.py:
  :69-123  execute (buffer shapes, sub-op order, background mix :135-143, alpha :145-148)
  :29-67   grad    (backward_pixel_map -> backward_textures -> backward_depth_map in place)
Maps keep the kernels' orientation: [B, yi, xi] with yi up (row 0 = bottom); the flip to image
orientation belongs to rasterize_rgbad (n3mr.py:239-247).
"""
import ctypes as C

import numpy as np

from . import build as _build

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build.build())
        f, i, I, F = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int, C.c_float
        L.nmr_oracle_face_index_map.restype = None
        L.nmr_oracle_face_index_map.argtypes = [f, i, f, f, f, I, I, I, F, F, I]
        L.nmr_oracle_texture_sampling.restype = None
        L.nmr_oracle_texture_sampling.argtypes = [f, f, i, f, f, f, i, f, I, I, I, I, F]
        L.nmr_oracle_backward_pixel_map.restype = None
        L.nmr_oracle_backward_pixel_map.argtypes = [f, i, f, f, f, f, f, I, I, I, F, I, I]
        L.nmr_oracle_backward_textures.restype = None
        L.nmr_oracle_backward_textures.argtypes = [i, f, i, f, f, I, I, I, I]
        L.nmr_oracle_backward_depth_map.restype = None
        L.nmr_oracle_backward_depth_map.argtypes = [f, f, i, f, f, f, f, I, I, I]
        d = C.POINTER(C.c_double)
        L.nmr_oracle_backward_pixel_map_stats.restype = None
        L.nmr_oracle_backward_pixel_map_stats.argtypes = [f, i, f, f, f, f, f, I, I, I, F, I, I, d, d, d, i, i]
        L.nmr_oracle_backward_textures_stats.restype = None
        L.nmr_oracle_backward_textures_stats.argtypes = [i, f, i, f, f, I, I, I, I, d, d, i]
        L.nmr_oracle_backward_depth_map_stats.restype = None
        L.nmr_oracle_backward_depth_map_stats.argtypes = [f, f, i, f, f, f, f, I, I, I, d, d, i]
        _lib = L
    return _lib


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def forward(faces, textures, image_size, near=0.1, far=100.0, eps=1e-4, background_color=(0, 0, 0),
            return_rgb=True, return_alpha=True, return_depth=True):
    """faces [B,nf,3,3], textures [B,nf,ts,ts,ts,3] or None -> dict of maps (kernel orientation)."""
    L = lib()
    fc = np.ascontiguousarray(faces, np.float32)
    B, nf = fc.shape[:2]
    H = int(image_size)
    out = dict(face_index_map=np.empty((B, H, H), np.int32), weight_map=np.empty((B, H, H, 3), np.float32),
               depth_map=np.empty((B, H, H), np.float32),
               face_inv_map=np.zeros((B, H, H, 3, 3), np.float32) if return_depth else None)
    L.nmr_oracle_face_index_map(_f(fc), _i(out["face_index_map"]), _f(out["weight_map"]), _f(out["depth_map"]),
                                _f(out["face_inv_map"]) if return_depth else None, B, nf, H,
                                np.float32(near), np.float32(far), int(return_depth))
    if return_rgb:
        tx = np.ascontiguousarray(textures, np.float32)
        ts = tx.shape[2]
        out["rgb_raw"] = np.empty((B, H, H, 3), np.float32)
        out["sampling_index_map"] = np.empty((B, H, H, 8), np.int32)
        out["sampling_weight_map"] = np.empty((B, H, H, 8), np.float32)
        L.nmr_oracle_texture_sampling(_f(fc), _f(tx), _i(out["face_index_map"]), _f(out["weight_map"]),
                                      _f(out["depth_map"]), _f(out["rgb_raw"]), _i(out["sampling_index_map"]),
                                      _f(out["sampling_weight_map"]), B, nf, H, ts, np.float32(eps))
        mask = (out["face_index_map"] >= 0).astype(np.float32)[..., None]
        bg = np.asarray(background_color, np.float32)
        bg = bg[None, None, None, :] if bg.ndim == 1 else bg[:, None, None, :]
        out["rgb_map"] = (out["rgb_raw"] * mask + (1 - mask) * bg).astype(np.float32)     # n3mr.py:135-143
    if return_alpha:
        out["alpha_map"] = (out["face_index_map"] >= 0).astype(np.float32)                 # :145-148
    return out


def backward(faces, textures, fwd, image_size, eps=1e-4, grad_rgb_map=None, grad_alpha_map=None,
             grad_depth_map=None, return_rgb=True, return_alpha=True, return_depth=True):
    """-> (grad_faces [B,nf,3,3], grad_textures or None), following n3mr.py:29-67."""
    L = lib()
    fc = np.ascontiguousarray(faces, np.float32)
    B, nf = fc.shape[:2]
    H = int(image_size)
    grad_faces = np.zeros((B, nf, 3, 3), np.float32)
    one = np.zeros(1, np.float32)
    g_rgb = np.ascontiguousarray(grad_rgb_map, np.float32) if return_rgb else one
    g_a = np.ascontiguousarray(grad_alpha_map, np.float32) if return_alpha else one
    if return_rgb or return_alpha:
        L.nmr_oracle_backward_pixel_map(_f(fc), _i(fwd["face_index_map"]),
                                        _f(fwd["rgb_map"]) if return_rgb else _f(one),
                                        _f(fwd["alpha_map"]) if return_alpha else _f(one), _f(g_rgb), _f(g_a),
                                        _f(grad_faces), B, nf, H, np.float32(eps), int(return_rgb), int(return_alpha))
    grad_textures = None
    if return_rgb:
        tx = np.ascontiguousarray(textures, np.float32)
        grad_textures = np.zeros_like(tx)
        L.nmr_oracle_backward_textures(_i(fwd["face_index_map"]), _f(fwd["sampling_weight_map"]),
                                       _i(fwd["sampling_index_map"]), _f(g_rgb), _f(grad_textures), B, nf, H, tx.shape[2])
    if return_depth:
        g_d = np.ascontiguousarray(grad_depth_map, np.float32)
        L.nmr_oracle_backward_depth_map(_f(fc), _f(fwd["depth_map"]), _i(fwd["face_index_map"]),
                                        _f(np.ascontiguousarray(fwd["face_inv_map"])), _f(fwd["weight_map"]),
                                        _f(g_d), _f(grad_faces), B, nf, H)
    return grad_faces, grad_textures


def backward_stats(faces, textures, fwd, image_size, eps=1e-4, grad_rgb_map=None, grad_alpha_map=None,
                   grad_depth_map=None, return_rgb=True, return_alpha=True, return_depth=True):
    """backward() plus float64 statistics of every sum, for per-element error bounds (nmr_oracle.c):
    grad_faces / grad_textures (the float results, as backward() returns them) and
      k9_g64, k9_T, k9_R, k9_cnt, k9_chain  [B,nf,3,3]  (K9: see k9_stats; zero without rgb / alpha)
      k10_g64, k10_T, k10_cnt               like textures (K10; None without rgb)
      k11_g64, k11_T, k11_cnt               [B,nf,3,3]   (K11; zero without depth)"""
    L = lib()
    fc = np.ascontiguousarray(faces, np.float32)
    B, nf = fc.shape[:2]
    H = int(image_size)
    z64 = lambda: np.zeros((B, nf, 3, 3), np.float64)
    z32 = lambda: np.zeros((B, nf, 3, 3), np.int32)
    out = dict(k9_g64=z64(), k9_T=z64(), k9_R=z64(), k9_cnt=z32(), k9_chain=z32(),
               k11_g64=z64(), k11_T=z64(), k11_cnt=z32(), k10_g64=None, k10_T=None, k10_cnt=None)
    grad_faces = np.zeros((B, nf, 3, 3), np.float32)
    one = np.zeros(1, np.float32)
    g_rgb = np.ascontiguousarray(grad_rgb_map, np.float32) if return_rgb else one
    g_a = np.ascontiguousarray(grad_alpha_map, np.float32) if return_alpha else one
    if return_rgb or return_alpha:
        L.nmr_oracle_backward_pixel_map_stats(
            _f(fc), _i(fwd["face_index_map"]), _f(fwd["rgb_map"]) if return_rgb else _f(one),
            _f(fwd["alpha_map"]) if return_alpha else _f(one), _f(g_rgb), _f(g_a), _f(grad_faces), B, nf, H,
            np.float32(eps), int(return_rgb), int(return_alpha), _d(out["k9_g64"]), _d(out["k9_T"]), _d(out["k9_R"]),
            _i(out["k9_cnt"]), _i(out["k9_chain"]))
    grad_textures = None
    if return_rgb:
        tx = np.ascontiguousarray(textures, np.float32)
        grad_textures = np.zeros_like(tx)
        out.update(k10_g64=np.zeros(tx.shape, np.float64), k10_T=np.zeros(tx.shape, np.float64),
                   k10_cnt=np.zeros(tx.shape, np.int32))
        L.nmr_oracle_backward_textures_stats(_i(fwd["face_index_map"]), _f(fwd["sampling_weight_map"]),
                                             _i(fwd["sampling_index_map"]), _f(g_rgb), _f(grad_textures), B, nf, H,
                                             tx.shape[2], _d(out["k10_g64"]), _d(out["k10_T"]), _i(out["k10_cnt"]))
    if return_depth:
        g_d = np.ascontiguousarray(grad_depth_map, np.float32)
        L.nmr_oracle_backward_depth_map_stats(_f(fc), _f(fwd["depth_map"]), _i(fwd["face_index_map"]),
                                              _f(np.ascontiguousarray(fwd["face_inv_map"])), _f(fwd["weight_map"]),
                                              _f(g_d), _f(grad_faces), B, nf, H, _d(out["k11_g64"]), _d(out["k11_T"]),
                                              _i(out["k11_cnt"]))
    out.update(grad_faces=grad_faces, grad_textures=grad_textures)
    return out
