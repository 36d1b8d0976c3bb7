"""Mesh-fitting losses (host-side mirror in PyTorch of jrender/loss/*.py; SURVEY.md 8f rank 4).

neg_iou_loss  (iou_loss.py:1-5), LaplacianLoss (laplacian_loss.py:5-36, stored as a padded
neighbour table instead of the reference's dense nv x nv matrix -- same values), FlattenLoss
(flatten_loss.py:5-79, edge table built with a dictionary instead of the O(E*F) scan).
"""
import numpy as np
import torch
from torch import nn

from . import _lib


class _FusedMeshLoss(torch.autograd.Function):
    """loss [B] and d loss / d vertices from ONE launch of csrc/mesh_loss_api.cu; the backward is a scale.
    `name`(vertices, *tables, loss, grad, batch_size, num_vertices, *scalars, stream) is the entry point."""

    @staticmethod
    def forward(ctx, vertices, name, tables, scalars):
        v = vertices.contiguous()
        loss = torch.empty((v.shape[0],), dtype=torch.float32, device=v.device)
        grad = torch.empty_like(v)
        _lib.call(name, v.device, v, *tables, loss, grad, v.shape[0], v.shape[1], *scalars)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        (grad,) = ctx.saved_tensors
        return grad * grad_loss[:, None, None], None, None, None


def _fusable(x):
    return x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == 3 and 0 < x.shape[0] <= 65535


def neg_iou_loss(predict, target):
    dims = tuple(range(predict.dim())[1:])
    intersect = (predict * target).sum(dims)
    union = (predict + target - predict * target).sum(dims) + 1e-6
    return 1. - (intersect / union).sum() / intersect.nelement()


class LaplacianLoss(nn.Module):
    def __init__(self, vertex, faces, average=False):
        super(LaplacianLoss, self).__init__()
        self.nv = vertex.shape[0]
        self.nf = faces.shape[0]
        self.average = average
        f = faces.detach().cpu().numpy().astype(np.int64)
        # laplacian_loss.py:14-27: -1 at (i, j) for every (undirected) edge, diagonal = minus the row sum, rows divided
        # by the diagonal.  A face with a repeated index writes -1 at (a, a) first, which the diagonal then overwrites:
        # the self-pair adds 1 to the divisor but a is not its own neighbour.
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 0]], f[:, [1, 2]], f[:, [2, 1]], f[:, [2, 0]], f[:, [0, 2]]], 0)
        e = np.unique(e, axis=0)
        self_pair = e[:, 0] == e[:, 1]
        div = np.bincount(e[:, 0], minlength=self.nv).astype(np.float32)   # distinct neighbours + has a self-pair
        e = e[~self_pair]
        deg = np.bincount(e[:, 0], minlength=self.nv)
        # Padded neighbour table instead of a sparse matrix: L x = diag * x + sum_k w[:, k] * x[nbr[:, k]].
        # index_select forward / index_add backward are plain kernels (no thrust sort, no host
        # synchronisation), so the loss can be captured in a CUDA graph; torch.sparse.mm cannot.
        maxdeg = int(deg.max()) if e.size else 0
        nbr = np.zeros((self.nv, max(maxdeg, 1)), np.int64)
        w = np.zeros((self.nv, max(maxdeg, 1)), np.float32)
        fill = np.zeros(self.nv, np.int64)
        for a_, b_ in e:
            nbr[a_, fill[a_]] = b_
            w[a_, fill[a_]] = -1.0 / div[a_]
            fill[a_] += 1
        with np.errstate(divide='ignore', invalid='ignore'):
            diag = (div / div).astype(np.float32)     # 1, or NaN for an isolated vertex like the dense 0/0
        self.register_buffer('nbr', torch.from_numpy(nbr.reshape(-1)))
        self.register_buffer('nbr32', torch.from_numpy(nbr.astype(np.int32)))
        self.register_buffer('nbr_w', torch.from_numpy(w))
        self.register_buffer('diag', torch.from_numpy(diag))

    fused = True   # CUDA float32 [B, nv, 3] inputs take the one-launch kernel (b200r_laplacian_loss)

    def forward(self, x):
        batch_size = x.shape[0]
        if self.fused and _fusable(x) and x.shape[1] == self.nv and self.nbr32.device == x.device:
            y = _FusedMeshLoss.apply(x, "b200r_laplacian_loss", (self.nbr32, self.nbr_w, self.diag), (self.nbr_w.shape[1],))
            return y.sum() / batch_size if self.average else y
        xn = torch.index_select(x, 1, self.nbr).view(batch_size, self.nv, -1, x.shape[2])
        y = x * self.diag[None, :, None] + (xn * self.nbr_w[None, :, :, None]).sum(2)
        dims = tuple(range(y.dim())[1:])
        y = y.pow(2).sum(dims)
        if self.average:
            return y.sum() / batch_size
        return y

    execute = forward


class FlattenLoss(nn.Module):
    def __init__(self, faces, average=False):
        super(FlattenLoss, self).__init__()
        self.nf = faces.shape[0]
        self.average = average
        f = faces.detach().cpu().numpy().astype(np.int64)
        self.nv_min = int(f.max()) + 1 if f.size else 0   # smallest vertex count the edge table is valid for
        # a face with a repeated index has an edge with no third vertex (flatten_loss.py:22-24 raises IndexError on it);
        # the table below would pair that face with itself instead
        rep = np.flatnonzero((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 2] == f[:, 0]))
        if rep.size:
            raise ValueError("FlattenLoss: face %d %s repeats a vertex index" % (rep[0], f[rep[0]].tolist()))
        opp = {}
        for tri in f:
            for a, b_, c in ((tri[0], tri[1], tri[2]), (tri[1], tri[2], tri[0]), (tri[2], tri[0], tri[1])):
                opp.setdefault((min(a, b_), max(a, b_)), []).append(c)
        # flatten_loss.py:13 takes the edge set from columns (0,1) and (1,2) of every face ONLY: an edge that is the
        # (v2, v0) edge of both of its faces carries no dihedral term in the reference, so it carries none here.
        # v2 / v3 = third vertex of the first / second face (in face order) containing the edge (:19-30).
        listed = set((min(a, b_), max(a, b_)) for a, b_ in np.concatenate((f[:, 0:2], f[:, 1:3]), axis=0))
        edges = sorted(k for k in listed if len(opp[k]) >= 2)      # the reference assumes a closed manifold
        v0s = np.array([e[0] for e in edges], np.int64)
        v1s = np.array([e[1] for e in edges], np.int64)
        v2s = np.array([opp[e][0] for e in edges], np.int64)
        v3s = np.array([opp[e][1] for e in edges], np.int64)
        for name, v in (('v0s', v0s), ('v1s', v1s), ('v2s', v2s), ('v3s', v3s)):
            self.register_buffer(name, torch.from_numpy(v))
        self.register_buffer('e32', torch.from_numpy(np.stack([v0s, v1s, v2s, v3s]).astype(np.int32)))

    fused = True   # CUDA float32 [B, nv, 3] inputs take the one-launch kernel (b200r_flatten_loss)

    def forward(self, vertices, eps=1e-6):
        batch_size = vertices.shape[0]
        if vertices.shape[1] < self.nv_min:   # checked on the host: a device-side index assert would poison the CUDA context
            raise IndexError("FlattenLoss: the edge table names vertex %d but vertices has only %d" % (self.nv_min - 1, vertices.shape[1]))
        # the kernel dereferences the module's index buffers: they must live on the input's device, otherwise the
        # index_select path below raises torch's own device-mismatch error
        if self.fused and _fusable(vertices) and self.e32.device == vertices.device:
            loss = _FusedMeshLoss.apply(vertices, "b200r_flatten_loss", tuple(self.e32), (int(self.v0s.shape[0]), float(eps)))
            return loss.sum() / batch_size if self.average else loss
        v0s = torch.index_select(vertices, 1, self.v0s)   # backward = index_add (graph-capturable)
        v1s = torch.index_select(vertices, 1, self.v1s)
        v2s = torch.index_select(vertices, 1, self.v2s)
        v3s = torch.index_select(vertices, 1, self.v3s)

        def half(b):
            a = v1s - v0s
            al2 = a.pow(2).sum(-1)
            bl2 = b.pow(2).sum(-1)
            al1 = (al2 + eps).sqrt()
            bl1 = (bl2 + eps).sqrt()
            ab = (a * b).sum(-1)
            cos = ab / (al1 * bl1 + eps)
            sin = (1 - cos.pow(2) + eps).sqrt()
            c = a * (ab / (al2 + eps))[..., None]
            return b - c, bl1 * sin
        cb1, cb1l1 = half(v2s - v0s)
        cb2, cb2l1 = half(v3s - v0s)
        cos = (cb1 * cb2).sum(-1) / (cb1l1 * cb2l1 + eps)
        dims = tuple(range(cos.dim())[1:])
        loss = (cos + 1).pow(2).sum(dims)
        if self.average:
            return loss.sum() / batch_size
        return loss

    execute = forward
