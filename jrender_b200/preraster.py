"""Fused pre-raster geometry stage (SURVEY.md section 8f rank 1).

`project_faces` turns world-space `vertices [B|1, nv, 3]` + `faces [B|1, nf, 3]` + a camera into
the rasterizer's `face_vertices [B, nf, 3, 3]` in ONE kernel launch (and one launch for the
backward), replacing the reference's chain of tensor ops

    jrender/renderer/transform/look_at.py:24-38  or  look.py:23-53     camera axes, v - eye, v @ r^T
    jrender/renderer/transform/perspective.py:11-16 / orthogonal.py:12-15
    jrender/structures/utils/faces_vertices.py:14-19                   gather (backward: scatter-add)

(15 small ops forward, as many again in autograd).  `Transform.forward` (transform.py) routes
here for camera_mode 'look_at' / 'look' on CUDA tensors; everything else keeps the op-by-op
PyTorch mirror.  There is no CPU path: CPU tensors raise.
"""
import math

import numpy as np
import torch

from . import _lib
from ._lib import _f3

CAM_MODES = {'look_at': 0, 'look_right': 1, 'look_left': 2}
PROJECTIONS = {'perspective': 0, 'orthogonal': 1}


def perspective_width(angle):
    """tan(angle) evaluated like perspective.py:11-12 (float32 radians, float32 tan)."""
    return float(np.tan(np.float32(angle / 180 * math.pi), dtype=np.float32))


class _ProjectFacesOp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, faces, eye, cfg):
        v = vertices.contiguous()
        B, nf = cfg["B"], faces.shape[1]
        out = torch.empty((B, nf, 3, 3), dtype=torch.float32, device=v.device)
        _lib.call("b200r_project_faces_forward", v.device,
                  v, faces, eye, out, cfg["at"], cfg["up"], cfg["width"], cfg["mode"], cfg["proj"],
                  B, v.shape[1], nf, v.shape[0], faces.shape[0], eye.shape[0])
        ctx.cfg = cfg
        ctx.save_for_backward(v, faces, eye)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        v, faces, eye = ctx.saved_tensors
        cfg = ctx.cfg
        g = grad_out.contiguous()
        if g.dtype != torch.float32:
            g = g.float()
        gv = torch.empty_like(v)
        _lib.call("b200r_project_faces_backward", v.device,
                  v, faces, eye, g, gv, cfg["at"], cfg["up"], cfg["width"], cfg["mode"],
                  cfg["proj"], cfg["B"], v.shape[1], faces.shape[1], v.shape[0], faces.shape[0], eye.shape[0])
        return gv, None, None, None


def int32_faces(faces, dev):
    """int32 + contiguous, no host synchronisation: the kernel range-checks every index itself (an
    index outside [0, nv) poisons that corner with NaN instead of the reference's out-of-bounds read).
    Wider indices outside [0, 2^31) become -1 on the device first: a plain cast would wrap 2^32 + 1 to 1."""
    f = faces.to(dev)
    if f.dtype != torch.int32:
        if f.dtype == torch.int64:
            f = f.masked_fill((f < 0) | (f > 0x7fffffff), -1)
        f = f.to(torch.int32)
    return f.contiguous()


def project_faces(vertices, faces, eye, camera_mode='look_at', at=(0, 0, 0), direction=(0, 0, 1), up=(0, 1, 0),
                  coordinate='right', perspective=True, viewing_angle=30., viewing_scale=1.0):
    """vertices [B|1, nv, 3] (world), faces [B|1, nf, 3] int, eye [3] | [B, 3] (tensor, list or tuple)
    -> face_vertices [B, nf, 3, 3] = face_vertices(perspective(look_at(vertices, eye)), faces)."""
    if vertices.dim() != 3:
        raise ValueError('vertices Tensor should have 3 dimensions')
    if not vertices.is_cuda:
        raise _lib.B200RasterError("project_faces: tensors must be CUDA tensors (no CPU fallback)")
    if vertices.dtype != torch.float32:
        raise TypeError("project_faces: vertices must be float32")
    if faces.dim() == 2:
        faces = faces[None]
    if faces.dim() != 3 or faces.shape[2] != 3:
        raise ValueError("faces must be [batch, num_faces, 3], got %s" % (tuple(faces.shape),))
    dev = vertices.device
    if isinstance(eye, torch.Tensor):
        e = eye.detach().to(device=dev, dtype=torch.float32)
    else:
        from .transform import _t
        e = _t(list(eye) if isinstance(eye, tuple) else eye, vertices)
    if e.dim() == 1:
        e = e[None]
    e = e.contiguous()
    B = max(vertices.shape[0], faces.shape[0], e.shape[0])
    for name, t in (("vertices", vertices), ("faces", faces), ("eye", e)):
        if t.shape[0] not in (1, B):
            raise ValueError("%s batch %d does not match batch size %d" % (name, t.shape[0], B))
    if e.shape[1:] != (3,):
        raise ValueError("eye must be [3] or [batch, 3]")
    f = int32_faces(faces, dev)
    if camera_mode == 'look_at':
        mode, a = CAM_MODES['look_at'], _f3(at)
    elif camera_mode == 'look':
        if coordinate not in ('right', 'left'):
            raise ValueError("coordinate must be 'right' or 'left'")
        mode, a = CAM_MODES['look_' + coordinate], _f3(direction)
        d = np.asarray(direction, np.float32); u = np.asarray(up, np.float32)
        d = d / max(float(np.linalg.norm(d)), 1e-5); u = u / max(float(np.linalg.norm(u)), 1e-5)
        if abs(float((d * u).sum())) > 1 - 1e-4:   # look.py:26-27
            raise ValueError("camera_direction and camera_up can not be the same")
    else:
        raise ValueError("project_faces supports camera_mode 'look_at' and 'look'")
    cfg = {"B": B, "at": a, "up": _f3(up), "mode": mode,
           "proj": PROJECTIONS['perspective' if perspective else 'orthogonal'],
           "width": perspective_width(viewing_angle) if perspective else float(viewing_scale)}
    return _ProjectFacesOp.apply(vertices, f, e, cfg)
