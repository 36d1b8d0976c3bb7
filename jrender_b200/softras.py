"""SoftRas rasterizer: host-side mirror of the reference's L2 interface.

Mirrors (same names, argument meaning, defaults and error behaviour):
  jrender/renderer/dr/softras/soft_rasterize.py:9-133   SoftRasterizeFunction
  jrender/renderer/dr/softras/soft_rasterize.py:136-148 soft_rasterize
  jrender/renderer/dr/softras/rasterizer.py:8-61        SoftRasterizer

The compute is done by libb200raster.so (hand-written sm_90a kernels) through the C ABI
in include/b200raster.h; PyTorch only owns device memory, the stream and autograd glue.
There is no CPU path: tensors must live on a CUDA device.
"""
import math

import numpy as np
import torch
from torch import nn

from . import _lib

FUNC_DIST_MAP = {'hard': 0, 'barycentric': 1, 'euclidean': 2}   # soft_rasterize.py:39
FUNC_RGB_MAP = {'hard': 0, 'softmax': 1, 'none': 2}             # :40
FUNC_ALPHA_MAP = {'hard': 0, 'sum': 1, 'prod': 2}               # :41
FUNC_MAP_SAMPLE = {'surface': 0, 'vertex': 1}                   # :42


def _check_inputs(face_vertices, textures):
    if not (face_vertices.is_cuda and textures.is_cuda):
        raise _lib.B200RasterError(
            "soft_rasterize: tensors must be CUDA tensors (the reference op is CUDA-only too, "
            "and this library has no CPU fallback)")
    if face_vertices.dtype != torch.float32 or textures.dtype != torch.float32:
        raise TypeError("soft_rasterize: face_vertices and textures must be float32")
    if face_vertices.dim() != 4 or tuple(face_vertices.shape[2:]) != (3, 3):
        raise ValueError("face_vertices must be [batch, num_faces, 3, 3], got %s" % (tuple(face_vertices.shape),))
    if textures.dim() != 4 or textures.shape[3] != 3 or textures.shape[:2] != face_vertices.shape[:2]:
        raise ValueError("textures must be [batch, num_faces, T, 3], got %s" % (tuple(textures.shape),))


def pad_face_ids(faces_id_buffer):
    """The reference's -1 PADDED `faces_id_buffer` (soft_rasterize.py:470 memsets all of it) from the library's -1
    TERMINATED one: a pixel's top-K list is its slots up to the first -1; the slots behind that terminator are never
    written by the forward kernel (268 MB of stores per launch at C3) and never read by the backward.  [B,K,H,W] int32."""
    alive = (faces_id_buffer >= 0).to(torch.uint8).cummin(dim=1).values.bool()
    return torch.where(alive, faces_id_buffer, torch.full_like(faces_id_buffer, -1))


class _SoftRasterizeOp(torch.autograd.Function):
    """autograd glue around b200r_softras_forward / b200r_softras_backward."""

    @staticmethod
    def forward(ctx, face_vertices, textures, fn):
        _check_inputs(face_vertices, textures)
        L = _lib.lib()
        fv = face_vertices.contiguous()
        tx = textures.contiguous()
        B, nf = fv.shape[:2]
        T = tx.shape[2]
        H = int(fn.image_size)
        K = int(fn.max_faces_id)
        dev = fv.device
        soft_colors = torch.empty((B, 4, H, H), dtype=torch.float32, device=dev)
        aggrs_info = torch.empty((B, 2, H, H), dtype=torch.float32, device=dev)
        faces_id_buffer = torch.empty((B, K, H, H), dtype=torch.int32, device=dev)
        faces_info = torch.empty((B, nf, 27), dtype=torch.float32, device=dev) if fn.return_faces_info else None
        # state: records + gradient accumulator, kept for the backward; workspace: binning scratch, released (back to
        # the caching allocator) as soon as this call returns -- it is not part of the saved state
        st_bytes = L.b200r_softras_state_bytes(B, nf)
        state = torch.empty((st_bytes,), dtype=torch.uint8, device=dev)
        ws_bytes = L.b200r_softras_workspace_bytes(B, nf, H)
        workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        scal = fn._scalars(B, nf, T)
        pooled = None
        if getattr(fn, "pool2x2", False):   # anti-aliasing epilogue: the forward also writes the 2x2 means
            pooled = torch.empty((B, 4, H // 2, H // 2), dtype=torch.float32, device=dev)
        _lib.call("b200r_softras_forward" if pooled is None else "b200r_softras_forward_aa", dev,
                  fv, tx, soft_colors, *(() if pooled is None else (pooled,)), aggrs_info, faces_id_buffer, faces_info,
                  state, st_bytes, workspace, ws_bytes, *scal)
        ctx.pool2x2 = pooled is not None
        ctx.scal = scal
        ctx.st_bytes = st_bytes
        ctx.save_for_backward(fv, tx, soft_colors, aggrs_info, faces_id_buffer, state)
        # The reference keeps these on the Function object (soft_rasterize.py:101; faces_id_buffer here is -1 terminated,
        # pad_face_ids() gives the reference's fully padded form); render2 reads
        # save_vars[4] = aggrs_info (render2/render2.py:306).  Detached aliases only: a strong
        # reference to the OUTPUT tensor from here would close the cycle
        # output -> grad_fn -> ctx -> ... -> output, and ~0.9 GB per call would then wait for
        # Python's cyclic GC instead of being freed (and re-used by the allocator) immediately.
        fn.save_vars = (fv.detach(), tx.detach(), soft_colors.detach(), faces_info, aggrs_info.detach(),
                        faces_id_buffer.detach())
        ctx.mark_non_differentiable(aggrs_info, faces_id_buffer)
        # Without this, autograd hands the backward zero-filled "gradients" for aggrs_info and for the
        # int32 faces_id_buffer: a 268 MB (C3) / 2 GB (C5, 120 views) fill kernel per step for nothing.
        ctx.set_materialize_grads(False)
        if pooled is not None:   # the pooled image is the differentiable output; the supersampled one is saved state
            return pooled, aggrs_info, faces_id_buffer
        return soft_colors, aggrs_info, faces_id_buffer

    @staticmethod
    def backward(ctx, grad_soft_colors, _g1, _g2):
        if grad_soft_colors is None:   # soft_colors did not take part in the loss
            return None, None, None
        fv, tx, soft_colors, aggrs_info, faces_id_buffer, state = ctx.saved_tensors
        g = grad_soft_colors.contiguous()
        if g.dtype != torch.float32:
            g = g.float()
        grad_faces = torch.empty_like(fv)
        grad_textures = torch.empty_like(tx)
        _lib.call("b200r_softras_backward_aa" if ctx.pool2x2 else "b200r_softras_backward", fv.device,   # g: pooled under AA
                  fv, tx, soft_colors, aggrs_info, faces_id_buffer, state, ctx.st_bytes, g, grad_faces, grad_textures,
                  *ctx.scal)
        return grad_faces, grad_textures, None


class SoftRasterizeFunction(object):
    """Drop-in for the reference's jittor.Function of the same name (soft_rasterize.py:9-133).

    Construct with the configuration, call with (face_vertices [B,nf,3,3], textures
    [B,nf,T,3]) -> soft_colors [B,4,H,W].  `bin_size` / `max_elems_per_bin` are accepted for
    signature compatibility; binning is internal, exact and always on, so they have no
    effect on results (the reference's binned path is only an approximation of its naive
    path, SURVEY.md Q12-Q14).
    """

    def __init__(self, image_size=256,
                 background_color=[0, 0, 0], near=1, far=100,
                 fill_back=True, eps=1e-3,
                 sigma_val=1e-5, dist_func='euclidean', dist_eps=1e-4,
                 gamma_val=1e-4, aggr_func_rgb='softmax', aggr_func_alpha='prod',
                 texture_type='surface', bin_size=0, max_elems_per_bin=0, max_faces_per_pixel_for_grad=16):
        self.image_size = image_size
        self.background_color = background_color  # ignored by the reference op as well (SURVEY.md F6)
        self.near = near
        self.far = far
        self.eps = eps
        self.sigma_val = sigma_val
        self.gamma_val = gamma_val
        self.dist_func = dist_func
        self.dist_eps = np.log(1. / dist_eps - 1.)   # soft_rasterize.py:25
        self.aggr_func_rgb = aggr_func_rgb
        self.aggr_func_alpha = aggr_func_alpha
        self.fill_back = fill_back
        self.aggr_texture_type = texture_type
        self.bin_size = bin_size
        self.max_elems_per_bin = max_elems_per_bin
        self.max_faces_id = max_faces_per_pixel_for_grad
        self.return_faces_info = False
        self.pool2x2 = False   # set by SoftRasterizer(anti_aliasing=True): return the 2x2 mean-pooled image (fused epilogue)
        self.save_vars = None

    def _scalars(self, B, nf, T):
        # KeyError on an unknown mode, like the reference's dict lookups (:52-55)
        self.func_dist_type = FUNC_DIST_MAP[self.dist_func]
        self.func_rgb_type = FUNC_RGB_MAP[self.aggr_func_rgb]
        self.func_alpha_type = FUNC_ALPHA_MAP[self.aggr_func_alpha]
        self.texture_type = FUNC_MAP_SAMPLE[self.aggr_texture_type]
        self.batch_size, self.num_faces = B, nf
        f32 = np.float32
        return (B, nf, T, int(self.image_size), int(self.max_faces_id),
                float(f32(self.near)), float(f32(self.far)), float(f32(self.eps)),
                float(f32(self.sigma_val)), float(f32(self.gamma_val)), float(f32(self.dist_eps)),
                self.func_dist_type, self.func_rgb_type, self.func_alpha_type, self.texture_type,
                int(bool(self.fill_back)))

    def __call__(self, face_vertices, textures):
        soft_colors, _, _ = _SoftRasterizeOp.apply(face_vertices, textures, self)
        return soft_colors

    execute = __call__   # jittor spelling

    def raw(self, face_vertices, textures):
        """(soft_colors, aggrs_info, faces_id_buffer); the last two are non-differentiable."""
        return _SoftRasterizeOp.apply(face_vertices, textures, self)


def soft_rasterize(face_vertices, textures, image_size=256,
                   background_color=[0, 0, 0], near=1, far=100,
                   fill_back=True, eps=1e-3,
                   sigma_val=1e-5, dist_func='euclidean', dist_eps=1e-4,
                   gamma_val=1e-4, aggr_func_rgb='softmax', aggr_func_alpha='prod',
                   texture_type='surface', bin_size=0, max_elems_per_bin=0, max_faces_per_pixel_for_grad=16):
    """Functional form, soft_rasterize.py:136-148."""
    return SoftRasterizeFunction(image_size,
                                 background_color, near, far,
                                 fill_back, eps,
                                 sigma_val, dist_func, dist_eps,
                                 gamma_val, aggr_func_rgb, aggr_func_alpha,
                                 texture_type, bin_size, max_elems_per_bin,
                                 max_faces_per_pixel_for_grad)(face_vertices, textures)


class SoftRasterizer(nn.Module):
    """rasterizer.py:8-61: Mesh -> images, with optional 2x supersampling and mode slicing."""

    def __init__(self, image_size=256, background_color=[0, 0, 0], near=1, far=100,
                 anti_aliasing=False, fill_back=False, eps=1e-3,
                 sigma_val=1e-5, dist_func='euclidean', dist_eps=1e-4,
                 gamma_val=1e-4, aggr_func_rgb='softmax', aggr_func_alpha='prod',
                 texture_type='surface',
                 bin_size=0, max_elems_per_bin=0, max_faces_per_pixel_for_grad=16):
        super(SoftRasterizer, self).__init__()

        if dist_func not in ['hard', 'euclidean', 'barycentric']:
            raise ValueError('Distance function only support hard, euclidean and barycentric')
        if aggr_func_rgb not in ['hard', 'softmax']:
            raise ValueError('Aggregate function(rgb) only support hard and softmax')
        if aggr_func_alpha not in ['hard', 'prod', 'sum']:
            raise ValueError('Aggregate function(a) only support hard, prod and sum')
        if texture_type not in ['surface', 'vertex']:
            raise ValueError('Texture type only support surface and vertex')

        self.image_size = image_size
        self.background_color = background_color
        self.near = near
        self.far = far
        self.anti_aliasing = anti_aliasing
        self.eps = eps
        self.fill_back = fill_back
        self.sigma_val = sigma_val
        self.dist_func = dist_func
        self.dist_eps = dist_eps
        self.gamma_val = gamma_val
        self.aggr_func_rgb = aggr_func_rgb
        self.aggr_func_alpha = aggr_func_alpha
        self.texture_type = texture_type
        self.bin_size = bin_size
        self.max_elems_per_bin = max_elems_per_bin
        self.max_faces_per_pixel_for_grad = max_faces_per_pixel_for_grad

    fused_antialiasing = True   # False: the reference's op sequence (full-size image, then avg_pool2d)

    def forward(self, mesh, mode=None):
        image_size = self.image_size * (2 if self.anti_aliasing else 1)
        # mode='silhouettes' returns images[:, 3] only (rasterizer.py:56-57).  Alpha and its gradient
        # do not depend on the colour aggregation (with a zero colour gradient every colour term of
        # the backward is exactly 0), so the kernels run with the colour path compiled out
        # (B200R_RGB_NONE): same alpha, same gradients, no texture sampling / softmax.
        aggr_func_rgb = 'none' if mode == 'silhouettes' else self.aggr_func_rgb
        args = (image_size, self.background_color, self.near, self.far, self.fill_back, self.eps,
                self.sigma_val, self.dist_func, self.dist_eps, self.gamma_val, aggr_func_rgb, self.aggr_func_alpha,
                self.texture_type, self.bin_size, self.max_elems_per_bin, self.max_faces_per_pixel_for_grad)
        if self.anti_aliasing and self.fused_antialiasing and mesh.face_vertices.is_cuda:
            # anti-aliasing (rasterizer.py:45,54-55: render at 2x, 2x2 mean): the forward kernel writes the pooled image
            # from its output staging and the backward reads the pooled gradient (b200r_softras_forward_aa / _backward_aa)
            fn = SoftRasterizeFunction(*args)
            fn.pool2x2 = True
            images = fn(mesh.face_vertices, mesh.face_textures)
        else:
            images = soft_rasterize(mesh.face_vertices, mesh.face_textures, *args)
            if self.anti_aliasing:
                images = torch.nn.functional.avg_pool2d(images, kernel_size=2, stride=2)
        if mode == 'silhouettes':
            return images[:, 3, :, :]
        elif mode == 'rgb':
            return images[:, :3, :, :]
        elif mode is None:
            return images[:, 3, :, :], images[:, :3, :, :]

    execute = forward
