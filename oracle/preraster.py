"""CPU oracle of the pre-raster geometry stage (TEST INFRASTRUCTURE; product code never imports it).

float32 numpy restatement, expression by expression, of
    jrender/renderer/transform/look_at.py:24-38      look_at
    jrender/renderer/transform/look.py:23-53         look
    jrender/renderer/transform/perspective.py:11-16  perspective
    jrender/renderer/transform/orthogonal.py:12-15   orthogonal
    jrender/structures/utils/faces_vertices.py:14-19 face_vertices
and the analytic vector-Jacobian product of that chain (float64) used to check the fused backward.
Pinned against the reference's own Python run through oracle/jittor_numpy_stub.py
(tests/golden/ref_host_transform_*.npz, generator oracle/make_ref_host_golden.py).
"""
import math

import numpy as np

F = np.float32


def _normalize(v, eps=1e-5):
    n = np.sqrt((v * v).sum(-1, keepdims=True, dtype=F)).astype(F)
    return (v / np.maximum(n, F(eps))).astype(F)


def camera_axes(eye, camera_mode="look_at", at=(0, 0, 0), direction=(0, 0, 1), up=(0, 1, 0), coordinate="right"):
    """eye [B,3] -> r [B,3,3] (rows x, y, z axes).  look_at.py:26-32 / look.py:23-46."""
    eye = np.asarray(eye, F)
    B = eye.shape[0]
    up = np.broadcast_to(np.asarray(up, F), (B, 3))
    if camera_mode == "look_at":
        z = _normalize(np.broadcast_to(np.asarray(at, F), (B, 3)) - eye)
    else:
        z = np.broadcast_to(_normalize(np.asarray(direction, F)), (B, 3))
        up = np.broadcast_to(_normalize(np.asarray(up[0], F)), (B, 3))
    if camera_mode == "look" and coordinate == "left":
        x = _normalize(np.cross(z, up).astype(F))
        y = _normalize(np.cross(x, z).astype(F))
    else:
        x = _normalize(np.cross(up, z).astype(F))
        y = _normalize(np.cross(z, x).astype(F))
    return np.stack([x, y, z], axis=1).astype(F)


def to_camera(vertices, eye, r):
    """look_at.py:34-38: (v - eye) @ r^T, accumulated in k order like a plain matmul."""
    d = (np.asarray(vertices, F) - np.asarray(eye, F)[:, None, :]).astype(F)
    out = np.empty(d.shape[:2] + (3,), F)
    for i in range(3):
        acc = (d[:, :, 0] * r[:, None, i, 0]).astype(F)
        acc = (acc + (d[:, :, 1] * r[:, None, i, 1]).astype(F)).astype(F)
        acc = (acc + (d[:, :, 2] * r[:, None, i, 2]).astype(F)).astype(F)
        out[:, :, i] = acc
    return out


def perspective_width(angle):
    return F(np.tan(F(angle / 180 * math.pi)))


def project(cam, perspective=True, viewing_angle=30.0, viewing_scale=1.0):
    z = cam[:, :, 2]
    if perspective:
        w = perspective_width(viewing_angle)
        x = ((cam[:, :, 0] / z).astype(F) / w).astype(F)   # perspective.py:14
        y = ((cam[:, :, 1] / z).astype(F) / w).astype(F)   # :15
    else:
        x = (cam[:, :, 0] * F(viewing_scale)).astype(F)    # orthogonal.py:13-14
        y = (cam[:, :, 1] * F(viewing_scale)).astype(F)
    return np.stack([x, y, z], axis=2).astype(F)


def project_faces(vertices, faces, eye, camera_mode="look_at", at=(0, 0, 0), direction=(0, 0, 1), up=(0, 1, 0),
                  coordinate="right", perspective=True, viewing_angle=30.0, viewing_scale=1.0):
    """vertices [B|1,nv,3], faces [B|1,nf,3], eye [B|1,3] -> face_vertices [B,nf,3,3]."""
    vertices = np.asarray(vertices, F)
    faces = np.asarray(faces)
    eye = np.asarray(eye, F).reshape(-1, 3)
    B = max(vertices.shape[0], faces.shape[0], eye.shape[0])
    vertices = np.broadcast_to(vertices, (B,) + vertices.shape[1:])
    faces = np.broadcast_to(faces, (B,) + faces.shape[1:])
    eye = np.broadcast_to(eye, (B, 3))
    r = camera_axes(eye, camera_mode, at, direction, up, coordinate)
    with np.errstate(all="ignore"):
        pv = project(to_camera(vertices, eye, r), perspective, viewing_angle, viewing_scale)
    nv = pv.shape[1]
    idx = faces.astype(np.int64)
    bad = (idx < 0) | (idx >= nv)   # the kernel poisons such a corner instead of the reference's out-of-bounds read
    out = np.stack([pv[b][np.where(bad[b], 0, idx[b])] for b in range(B)], axis=0).astype(F)   # faces_vertices.py:16-19
    out[bad] = np.nan
    return out


def project_faces_bwd_terms(vertices, faces, eye, grad_face_vertices, lift=None, camera_mode="look_at", at=(0, 0, 0),
                            direction=(0, 0, 1), up=(0, 1, 0), coordinate="right", perspective=True, viewing_angle=30.0,
                            viewing_scale=1.0):
    """k_project_faces_bwd's contribution of every (image, face, corner) to grad_vertices, in the kernel's float32 order:
    cam = (v - eye) r^T; zw = Z*w, dc0 = gx/zw, dc1 = gy/zw, dc2 = gz - (gx*X + gy*Y)/(Z*zw) (orthogonal: gx*s, gy*s, gz);
    term_k = (dc0*r0k + dc1*r1k) + dc2*r2k.  Corners with an out-of-range index or an all-zero upstream gradient add
    nothing, as in the kernel.  -> (rows [n], terms = three arrays [n], one per coordinate k): rows index
    grad_vertices.reshape(-1, 3), one per contributing corner.
    `lift` maps every float32 input array to another number type that supports the same operators (identity: float32)."""
    v = np.asarray(vertices, F)
    Bv, nv = v.shape[:2]
    g = np.asarray(grad_face_vertices, F)
    B, nf = g.shape[:2]
    f = np.broadcast_to(np.asarray(faces).astype(np.int64), (B, nf, 3)).reshape(-1)
    e = np.broadcast_to(np.asarray(eye, F).reshape(-1, 3), (B, 3))
    r = camera_axes(e, camera_mode, at, direction, up, coordinate)
    b = np.repeat(np.arange(B), nf * 3)
    gg = g.reshape(-1, 3)
    keep = (f >= 0) & (f < nv) & (gg != 0).any(1)
    b, f, gg = b[keep], f[keep], gg[keep]
    rows = (b if Bv > 1 else 0) * nv + f
    lift = lift or (lambda x: x)
    vv, ee, rr, G = lift(v.reshape(-1, 3)[rows]), lift(e[b]), lift(r[b]), lift(gg)
    with np.errstate(all="ignore"):
        d = [vv[:, k] - ee[:, k] for k in range(3)]
        cam = [(d[0] * rr[:, i, 0] + d[1] * rr[:, i, 1]) + d[2] * rr[:, i, 2] for i in range(3)]
        gx, gy, gz = G[:, 0], G[:, 1], G[:, 2]
        if perspective:
            zw = cam[2] * perspective_width(viewing_angle)
            dc = [gx / zw, gy / zw, gz - (gx * cam[0] + gy * cam[1]) / (cam[2] * zw)]
        else:
            s = F(viewing_scale)
            dc = [gx * s, gy * s, gz]
        terms = [(dc[0] * rr[:, 0, k] + dc[1] * rr[:, 1, k]) + dc[2] * rr[:, 2, k] for k in range(3)]
    return rows, terms


U = 2.0 ** -24      # fp32 unit roundoff
FTZ = 2.0 ** -125   # the float atomics flush subnormal inputs and results: < 2^-126 lost on each, per add


def term_sums(slots, terms, size):
    """Entries a kernel accumulates from float32 `terms` (one per slot, in [0, size)) in an unspecified order: warp
    shuffles, block partial sums and float atomics, all trees of float additions starting from zero.  Returns dict of
    float64 arrays of length `size`:
        exact  the sum of the terms (float64, within n 2^-53 A of the exact sum),
        A      sum of |t|,  n  the number of terms,
        bound  gamma_{n-1} A + n 2^-52 A + n 2^-125,  gamma_k = k u / (1 - k u),  u = 2^-24:
    any order of float additions is within gamma_{n-1} A of the exact sum (Higham, Accuracy and Stability of Numerical
    Algorithms, 4.2); the second term covers the float64 sum's own error, the third the atomics' subnormal flush.
    Entries whose exact sum is not finite are not bounded: their NaN / +-inf pattern does not depend on the order."""
    slots = np.asarray(slots, np.int64).reshape(-1)
    t = np.asarray(terms, np.float64).reshape(-1)
    exact, A = np.zeros(size), np.zeros(size)
    with np.errstate(invalid="ignore"):
        np.add.at(exact, slots, t)
        np.add.at(A, slots, np.abs(t))
    n = np.bincount(slots, minlength=size).astype(np.float64)
    k = np.maximum(n - 1, 0)
    with np.errstate(invalid="ignore"):
        bound = k * U / (1 - k * U) * A + n * 2.0 ** -52 * A + n * FTZ
    return dict(exact=exact, A=A, n=n, bound=bound)


def project_faces_bwd_sums(vertices, faces, eye, grad_face_vertices, **kw):
    """term_sums of k_project_faces_bwd's corner terms, each array shaped like grad_vertices [Bv, nv, 3]."""
    rows, terms = project_faces_bwd_terms(vertices, faces, eye, grad_face_vertices, **kw)
    shape = np.shape(vertices)
    slots = rows[:, None] * 3 + np.arange(3)
    s = term_sums(slots, np.stack(terms, 1), int(np.prod(shape)))
    return {k: x.reshape(shape) for k, x in s.items()}


def project_faces_vjp(vertices, faces, eye, grad_face_vertices, vertices_batch=None, **kw):
    """float64 vector-Jacobian product: grad_face_vertices [B,nf,3,3] -> grad_vertices [Bv,nv,3]."""
    vertices = np.asarray(vertices, np.float64)
    faces = np.asarray(faces)
    eye = np.asarray(eye, np.float64).reshape(-1, 3)
    g = np.asarray(grad_face_vertices, np.float64)
    B = g.shape[0]
    Bv = vertices.shape[0] if vertices_batch is None else vertices_batch
    nv = vertices.shape[1]
    faces = np.broadcast_to(faces, (B,) + faces.shape[1:])
    eyeb = np.broadcast_to(eye, (B, 3))
    r = camera_axes(eyeb.astype(F), kw.get("camera_mode", "look_at"), kw.get("at", (0, 0, 0)), kw.get("direction", (0, 0, 1)),
                    kw.get("up", (0, 1, 0)), kw.get("coordinate", "right")).astype(np.float64)
    out = np.zeros((Bv, nv, 3), np.float64)
    persp = kw.get("perspective", True)
    w = float(perspective_width(kw.get("viewing_angle", 30.0))) if persp else float(kw.get("viewing_scale", 1.0))
    for b in range(B):
        vb = vertices[b if vertices.shape[0] > 1 else 0]
        cam = (vb - eyeb[b]) @ r[b].T
        gp = np.zeros((nv, 3), np.float64)
        np.add.at(gp, faces[b].reshape(-1).astype(np.int64), g[b].reshape(-1, 3))
        if persp:
            Z = cam[:, 2]
            dc = np.stack([gp[:, 0] / (Z * w), gp[:, 1] / (Z * w),
                           gp[:, 2] - (gp[:, 0] * cam[:, 0] + gp[:, 1] * cam[:, 1]) / (Z * Z * w)], axis=1)
        else:
            dc = np.stack([gp[:, 0] * w, gp[:, 1] * w, gp[:, 2]], axis=1)
        out[b if Bv > 1 else 0] += dc @ r[b]
    return out
