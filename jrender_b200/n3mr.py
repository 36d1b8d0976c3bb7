"""Neural Mesh Renderer (dr_type='n3mr'): host-side mirror of the reference's L2 interface.

Mirrors (same names, arguments, defaults, return conventions):
  jrender/renderer/dr/n3mr/n3mr.py:13-166      RasterizeFunction (execute / grad)
  jrender/renderer/dr/n3mr/n3mr.py:168-187     Rasterize
  jrender/renderer/dr/n3mr/n3mr.py:189-346     rasterize_rgbad / rasterize / rasterize_silhouettes / rasterize_depth
  jrender/renderer/dr/n3mr/rasterizer.py:9-105 vertices_to_faces, N3mrRasterizer

Compute: libb200raster.so (b200r_nmr_forward / b200r_nmr_backward, hand-written sm_90a
kernels); PyTorch owns memory, the stream and autograd glue.  CUDA tensors only.
"""
import ctypes as C

import numpy as np
import torch
from torch import nn

from . import _lib

DEFAULT_IMAGE_SIZE = 256
DEFAULT_ANTI_ALIASING = True
DEFAULT_NEAR = 0.1
DEFAULT_FAR = 100
DEFAULT_EPS = 1e-4
DEFAULT_BACKGROUND_COLOR = (0, 0, 0)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class _RasterizeOp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, faces, textures, fn):
        if not faces.is_cuda:
            raise _lib.B200RasterError("n3mr rasterize: tensors must be CUDA tensors (reference: 'Currently "
                                       "implemented only for cuda Tensors', n3mr.py:16-17); no CPU fallback")
        L = _lib.lib()
        fc = faces.contiguous().float()
        B, nf = fc.shape[:2]
        H = int(fn.image_size)
        dev = fc.device
        rgb, alpha, depth_req = bool(fn.return_rgb), bool(fn.return_alpha), bool(fn.return_depth)
        tx = textures.contiguous().float() if rgb else None
        ts = int(tx.shape[2]) if rgb else 0
        bg = fn.background_color
        bg2d = None
        bg_host = (C.c_float * 3)(0.0, 0.0, 0.0)
        if rgb and bg is not None:
            bgt = torch.as_tensor(bg, dtype=torch.float32)
            if bgt.dim() == 1:
                bg_host = (C.c_float * 3)(*[float(x) for x in bgt.tolist()])
            else:
                bg2d = bgt.to(dev)          # per-batch background (n3mr.py:141-142): mixed below
        with torch.cuda.device(dev):
            face_index_map = torch.empty((B, H, H), dtype=torch.int32, device=dev)
            weight_map = torch.empty((B, H, H, 3), dtype=torch.float32, device=dev)
            depth_map = torch.empty((B, H, H), dtype=torch.float32, device=dev)
            rgb_map = torch.empty((B, H, H, 3), dtype=torch.float32, device=dev) if rgb else None
            sidx = torch.empty((B, H, H, 8), dtype=torch.int32, device=dev) if rgb else None
            swgt = torch.empty((B, H, H, 8), dtype=torch.float32, device=dev) if rgb else None
            alpha_map = torch.empty((B, H, H), dtype=torch.float32, device=dev) if alpha else None
            face_inv_map = torch.empty((B, H, H, 3, 3), dtype=torch.float32, device=dev) if depth_req else None
            ws_bytes = L.b200r_nmr_workspace_bytes(B, nf, H)
            workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
            f32 = np.float32
            rc = L.b200r_nmr_forward(
                _ptr(fc), _ptr(tx), _ptr(face_index_map), _ptr(weight_map), _ptr(depth_map), _ptr(rgb_map),
                _ptr(alpha_map), _ptr(sidx), _ptr(swgt), _ptr(face_inv_map), _ptr(workspace), ws_bytes,
                B, nf, ts, H, float(f32(fn.near)), float(f32(fn.far)), float(f32(fn.eps)),
                C.cast(bg_host, C.c_void_p), int(rgb), int(alpha), int(depth_req),
                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        _lib.check(rc, "b200r_nmr_forward")
        if bg2d is not None:
            mask = (face_index_map >= 0).float().unsqueeze(-1)
            rgb_map = rgb_map * mask + (1 - mask) * bg2d[:, None, None, :]
        ctx.dims, ctx.eps = (B, nf, ts, H), float(np.float32(fn.eps))
        ctx.flags = (rgb, alpha, depth_req)
        fn.texture_size = ts if rgb else None
        saved = (fc, tx, face_index_map, weight_map, depth_map, rgb_map, alpha_map, face_inv_map, sidx, swgt)
        ctx.none_mask = [t is None for t in saved]
        ctx.save_for_backward(*[t for t in saved if t is not None])
        # detached aliases on the Function object (n3mr.py:114), never the output tensors themselves:
        # that would close a reference cycle through grad_fn and defer freeing to the cyclic GC
        fn.save_vars = tuple(None if t is None else t.detach() for t in saved)
        empty = torch.empty(0, device=dev)
        outs = (rgb_map if rgb else empty, alpha_map if alpha else empty, depth_map if depth_req else empty)
        ctx.mark_non_differentiable(*[o for o, f in zip(outs, (rgb, alpha, depth_req)) if not f])
        return outs

    @staticmethod
    def backward(ctx, grad_rgb_map, grad_alpha_map, grad_depth_map):
        it = iter(ctx.saved_tensors)
        fc, tx, face_index_map, weight_map, depth_map, rgb_map, alpha_map, face_inv_map, sidx, swgt = \
            [None if is_none else next(it) for is_none in ctx.none_mask]
        B, nf, ts, H = ctx.dims
        rgb, alpha, depth_req = ctx.flags
        L = _lib.lib()
        dev = fc.device

        def prep(g, like):
            if g is None:
                return torch.zeros_like(like)       # n3mr.py:40-52: missing upstream gradients are zeros
            return g.contiguous().float()
        with torch.cuda.device(dev):
            g_rgb = prep(grad_rgb_map, rgb_map) if rgb else None
            g_a = prep(grad_alpha_map, alpha_map) if alpha else None
            g_d = prep(grad_depth_map, depth_map) if depth_req else None
            grad_faces = torch.empty_like(fc)
            grad_textures = torch.empty_like(tx) if rgb else None
            sc_bytes = L.b200r_nmr_backward_scratch_bytes(B, H) if (rgb or alpha) else 0
            scratch = torch.empty((sc_bytes,), dtype=torch.uint8, device=dev) if sc_bytes else None
            rc = L.b200r_nmr_backward(
                _ptr(fc), _ptr(face_index_map), _ptr(weight_map), _ptr(depth_map), _ptr(rgb_map), _ptr(alpha_map),
                _ptr(sidx), _ptr(swgt), _ptr(face_inv_map), _ptr(g_rgb), _ptr(g_a), _ptr(g_d),
                _ptr(grad_faces), _ptr(grad_textures), _ptr(scratch), sc_bytes, B, nf, ts, H, ctx.eps,
                int(rgb), int(alpha), int(depth_req), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        _lib.check(rc, "b200r_nmr_backward")
        return grad_faces, grad_textures, None


class RasterizeFunction(object):
    """n3mr.py:13-166.  Call with (faces [B,nf,3,3], textures [B,nf,ts,ts,ts,3] or None) ->
    (rgb_map [B,H,W,3], alpha_map [B,H,W], depth_map [B,H,W]) in the kernels' orientation
    (row 0 = bottom); outputs that were not requested are empty tensors."""

    def __init__(self, image_size, near, far, eps, background_color, return_rgb=False, return_alpha=False,
                 return_depth=False):
        self.image_size = image_size
        self.near = near
        self.far = far
        self.eps = eps
        self.background_color = background_color
        self.return_rgb = return_rgb
        self.return_alpha = return_alpha
        self.return_depth = return_depth
        self.save_vars = None
        self.texture_size = None

    def __call__(self, faces, textures=None):
        if self.return_rgb and textures is None:
            raise ValueError("return_rgb needs textures")
        if textures is None or not self.return_rgb:
            textures = torch.zeros(1, device=faces.device)
        return _RasterizeOp.apply(faces, textures, self)

    execute = __call__


class Rasterize(nn.Module):
    def __init__(self, image_size, near, far, eps, background_color, return_rgb=False, return_alpha=False,
                 return_depth=False):
        super(Rasterize, self).__init__()
        self.image_size = image_size
        self.near = near
        self.far = far
        self.eps = eps
        self.background_color = background_color
        self.return_rgb = return_rgb
        self.return_alpha = return_alpha
        self.return_depth = return_depth

    def forward(self, faces, textures):
        return RasterizeFunction(self.image_size, self.near, self.far, self.eps, self.background_color,
                                 self.return_rgb, self.return_alpha, self.return_depth)(faces, textures)

    execute = forward


def rasterize_rgbad(faces, textures=None, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING,
                    near=DEFAULT_NEAR, far=DEFAULT_FAR, eps=DEFAULT_EPS, background_color=DEFAULT_BACKGROUND_COLOR,
                    return_rgb=True, return_alpha=True, return_depth=True):
    """n3mr.py:189-264: dict(rgb [B,3,H,W], alpha [B,H,W], depth [B,H,W]) in image orientation."""
    size = image_size * 2 if anti_aliasing else image_size
    rgb, alpha, depth = Rasterize(size, near, far, eps, background_color, return_rgb, return_alpha, return_depth)(faces, textures)
    # transpose & vertical flip (:239-247)
    if return_rgb:
        rgb = rgb.permute((0, 3, 1, 2)).flip(2)
    if return_alpha:
        alpha = alpha.flip(1)
    if return_depth:
        depth = depth.flip(1)
    if anti_aliasing:   # 0.5x down-sampling (:249-256); alpha/depth keep the extra channel dim like the reference
        if return_rgb:
            rgb = torch.nn.functional.avg_pool2d(rgb, 2, stride=2)
        if return_alpha:
            alpha = torch.nn.functional.avg_pool2d(alpha.unsqueeze(1), 2, stride=2)
        if return_depth:
            depth = torch.nn.functional.avg_pool2d(depth.unsqueeze(1), 2, stride=2)
    return {'rgb': rgb if return_rgb else None, 'alpha': alpha if return_alpha else None,
            'depth': depth if return_depth else None}


def rasterize(faces, textures, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
              far=DEFAULT_FAR, eps=DEFAULT_EPS, background_color=DEFAULT_BACKGROUND_COLOR):
    return rasterize_rgbad(faces, textures, image_size, anti_aliasing, near, far, eps, background_color, True, False, False)['rgb']


def rasterize_silhouettes(faces, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
                          far=DEFAULT_FAR, eps=DEFAULT_EPS):
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, True, False)['alpha']


def rasterize_depth(faces, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
                    far=DEFAULT_FAR, eps=DEFAULT_EPS):
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, False, True)['depth']


def vertices_to_faces(vertices, faces):
    """rasterizer.py:9-24."""
    assert vertices.dim() == 3
    assert faces.dim() == 3
    assert vertices.shape[0] == faces.shape[0]
    assert vertices.shape[2] == 3
    assert faces.shape[2] == 3
    bs, nv = vertices.shape[:2]
    faces = faces.long() + (torch.arange(bs, device=vertices.device) * nv)[:, None, None]
    return vertices.reshape((bs * nv, 3))[faces]


class N3mrRasterizer(nn.Module):
    """rasterizer.py:26-105."""

    def __init__(self, image_size=256, anti_aliasing=True, background_color=[0, 0, 0], fill_back=True, near=0.1, far=100):
        super(N3mrRasterizer, self).__init__()
        self.image_size = image_size
        self.anti_aliasing = anti_aliasing
        self.background_color = background_color
        self.fill_back = fill_back
        self.near = near
        self.far = far
        self.rasterizer_eps = 1e-3

    def forward(self, mesh, mode=None):
        vertices, faces, textures = mesh.vertices, mesh.faces, mesh.textures
        if mode is None:
            return self.render(vertices, faces, textures)
        elif mode == 'rgb':
            return self.render_rgb(vertices, faces, textures)
        elif mode == 'silhouettes':
            return self.render_silhouettes(vertices, faces)
        elif mode == 'depth':
            return self.render_depth(vertices, faces)
        else:
            raise ValueError("mode should be one of None, 'silhouettes' or 'depth'")

    execute = forward

    def _fill_back(self, faces, textures=None):
        faces = torch.cat((faces, faces.flip(-1)), dim=1)
        if textures is not None:
            textures = torch.cat((textures, textures.permute((0, 1, 4, 3, 2, 5))), dim=1)
        return faces, textures

    def render_silhouettes(self, vertices, faces):
        if self.fill_back:
            faces, _ = self._fill_back(faces)
        return rasterize_silhouettes(vertices_to_faces(vertices, faces), self.image_size, self.anti_aliasing)

    def render_depth(self, vertices, faces):
        if self.fill_back:
            faces, _ = self._fill_back(faces)
        return rasterize_depth(vertices_to_faces(vertices, faces), self.image_size, self.anti_aliasing)

    def render_rgb(self, vertices, faces, textures):
        if self.fill_back:
            faces, textures = self._fill_back(faces, textures)
        return rasterize(vertices_to_faces(vertices, faces), textures, self.image_size, self.anti_aliasing, self.near,
                         self.far, self.rasterizer_eps, self.background_color)

    def render(self, vertices, faces, textures):
        if self.fill_back:
            faces, textures = self._fill_back(faces, textures)
        out = rasterize_rgbad(vertices_to_faces(vertices, faces), textures, self.image_size, self.anti_aliasing,
                              self.near, self.far, self.rasterizer_eps, self.background_color)
        return out['rgb'], out['depth'], out['alpha']
