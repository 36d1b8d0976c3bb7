"""Mesh voxelization: jrender/renderer/utils/voxelization.py:41-57 on the CUDA kernels of csrc/voxel_api.cu.

voxelization(faces, size) scales the faces to voxel units (unless normalize), then b200r_voxelize_surface writes the
surface voxels of all three axes and of the face corners, and b200r_voxelize_fill marks every voxel that is not
6-connected through empty voxels to the grid boundary.  Both run on the caller's current stream with no host
synchronisation, so a call can be captured in a CUDA graph.
"""
import ctypes as C

import torch

from . import _lib


def voxelize_surface(faces, size):
    """The OR of voxelize_sub1 over the three axes and voxelize_sub2: faces [B, nf, 3, 3] float32 CUDA tensor in voxel
    units -> int32 [B, size, size, size] of 0/1."""
    faces = faces.detach().contiguous()
    B, nf = faces.shape[0], faces.shape[1]
    voxels = torch.empty((B, size, size, size), dtype=torch.int32, device=faces.device)
    with torch.cuda.device(faces.device):
        _lib.check(_lib.lib().b200r_voxelize_surface(
            C.c_void_p(faces.data_ptr()), C.c_void_p(voxels.data_ptr()), B, nf, size,
            C.c_void_p(torch.cuda.current_stream(faces.device).cuda_stream)), "b200r_voxelize_surface")
    return voxels


def voxelize_fill(voxels):
    """voxelize_sub3 / voxelize_sub4 and their host loop (voxelization.py:24-38), in place on the int32 CUDA grid
    [B, vs, vs, vs]: every voxel that is not an empty (0) voxel connected to the grid boundary becomes 1, the rest 0.
    Returns voxels."""
    if voxels.dtype != torch.int32 or voxels.dim() != 4 or not voxels.is_cuda or not voxels.is_contiguous():
        raise ValueError("voxelize_fill: voxels must be a contiguous int32 CUDA tensor [B, vs, vs, vs]")
    B, vs = voxels.shape[0], voxels.shape[1]
    if voxels.shape[1:] != (vs, vs, vs):
        raise ValueError("voxelize_fill: voxels must be [B, vs, vs, vs], got %s" % (tuple(voxels.shape),))
    L = _lib.lib()
    nbytes = L.b200r_voxelize_workspace_bytes(B, vs)
    workspace = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=voxels.device)
    with torch.cuda.device(voxels.device):
        _lib.check(L.b200r_voxelize_fill(C.c_void_p(voxels.data_ptr()), C.c_void_p(workspace.data_ptr()), nbytes, B, vs,
                                         C.c_void_p(torch.cuda.current_stream(voxels.device).cuda_stream)),
                   "b200r_voxelize_fill")
    return voxels


def voxelization(faces, size, normalize=False):
    """voxelization.py:41-57: faces [B, nf, 3, 3] (multiplied by size unless normalize) -> int32 [B, size, size, size],
    1 for the surface and the voxels it encloses, indexed [b, c0, c1, c2] in the faces' coordinate order.  CUDA tensors
    only; the result is the reference's with float32 arithmetic left unfused."""
    if not isinstance(faces, torch.Tensor) or not faces.is_cuda:
        raise _lib.B200RasterError("voxelization runs on the GPU (b200r_voxelize_surface / _fill); there is no CPU fallback")
    size = int(size)
    if faces.dim() != 4 or faces.shape[2:] != (3, 3):
        raise ValueError("voxelization: faces must be [B, nf, 3, 3], got %s" % (tuple(faces.shape),))
    faces = faces.detach().float()
    if not normalize:
        faces = faces * size
    return voxelize_fill(voxelize_surface(faces, size))
