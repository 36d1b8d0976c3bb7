"""Synthetic inputs for tests and bench.py (numpy, deterministic, no files needed).

The reference's README table quotes 280 / 3.3k / 39k-face meshes that are not shipped
(SURVEY.md F7); BASELINE.md section 3 fixes them as UV spheres with 2*S*(R-1) triangles:
280 = (14, 11), 3280 = (40, 42), 39200 = (140, 141).  Cameras follow the reference's
look_at + perspective maths (jrender/renderer/transform/look_at.py:3-39,
perspective.py:4-17, utils/get_points_from_angles.py:4-22) in float32 numpy.
"""
import math

import numpy as np

SPHERES = {280: (14, 11), 3280: (40, 42), 39200: (140, 141)}


def uv_sphere(segments, rings, radius=0.8, jitter=0.0, seed=0):
    """vertices [nv,3] f32, faces [nf,3] i32; nf = 2*segments*(rings-1); outward CCW winding."""
    S, R = int(segments), int(rings)
    verts = [(0.0, radius, 0.0)]
    for r in range(1, R):
        th = math.pi * r / R
        for s in range(S):
            ph = 2.0 * math.pi * s / S
            verts.append((radius * math.sin(th) * math.cos(ph), radius * math.cos(th), radius * math.sin(th) * math.sin(ph)))
    verts.append((0.0, -radius, 0.0))
    bottom = len(verts) - 1
    faces = []
    ring = lambda r, s: 1 + (r - 1) * S + (s % S)
    for s in range(S):
        faces.append((0, ring(1, s + 1), ring(1, s)))
    for r in range(1, R - 1):
        for s in range(S):
            a, b_, c, d = ring(r, s), ring(r, s + 1), ring(r + 1, s), ring(r + 1, s + 1)
            faces.append((a, b_, d))
            faces.append((a, d, c))
    for s in range(S):
        faces.append((bottom, ring(R - 1, s), ring(R - 1, s + 1)))
    v = np.asarray(verts, dtype=np.float32)
    if jitter > 0:
        v = (v + np.random.default_rng(seed).normal(0.0, jitter, v.shape)).astype(np.float32)
    f = np.asarray(faces, dtype=np.int32)
    assert f.shape[0] == 2 * S * (R - 1)
    return v, f


def sphere_by_faces(num_faces, radius=0.8, jitter=0.0):
    return uv_sphere(*SPHERES[num_faces], radius=radius, jitter=jitter)


def get_points_from_angles(distance, elevation, azimuth):
    """Scalar branch of utils/get_points_from_angles.py:5-12 (degrees)."""
    e, a = math.radians(elevation), math.radians(azimuth)
    return (distance * math.cos(e) * math.sin(a), distance * math.sin(e), -distance * math.cos(e) * math.cos(a))


def _normalize(v, eps=1e-5):
    n = np.sqrt((v * v).sum(-1, keepdims=True)).astype(np.float32)
    return (v / np.maximum(n, np.float32(eps))).astype(np.float32)


def look_at(vertices, eye, at=(0, 0, 0), up=(0, 1, 0)):
    """vertices [B,nv,3], eye [B,3] -> camera-space vertices (look_at.py:3-39)."""
    vertices = np.asarray(vertices, np.float32)
    B = vertices.shape[0]
    eye = np.broadcast_to(np.asarray(eye, np.float32), (B, 3))
    at = np.broadcast_to(np.asarray(at, np.float32), (B, 3))
    up = np.broadcast_to(np.asarray(up, np.float32), (B, 3))
    z_axis = _normalize(at - eye)
    x_axis = _normalize(np.cross(up, z_axis).astype(np.float32))
    y_axis = _normalize(np.cross(z_axis, x_axis).astype(np.float32))
    r = np.stack([x_axis, y_axis, z_axis], axis=1)  # [B,3,3]
    v = vertices - eye[:, None, :]
    return np.matmul(v, r.transpose(0, 2, 1)).astype(np.float32)


def perspective(vertices, angle=30.0):
    """perspective.py:4-17: x/(z*tan), y/(z*tan), z."""
    width = np.float32(math.tan(np.float32(angle / 180.0 * math.pi)))
    z = vertices[:, :, 2]
    x = vertices[:, :, 0] / z / width
    y = vertices[:, :, 1] / z / width
    return np.stack([x, y, z], axis=2).astype(np.float32)


def face_vertices(vertices, faces):
    """structures/utils/faces_vertices.py:4-19: [B,nv,3] x [nf,3] -> [B,nf,3,3]."""
    return np.ascontiguousarray(vertices[:, faces.astype(np.int64)], dtype=np.float32)


def make_scene(num_faces=280, batch=1, image_size=None, texture_res=1, texture_type='surface',
               distance=2.732, elevation=30.0, azim0=0.0, radius=0.8, jitter=0.0, seed=1):
    """face_vertices [B,nf,3,3] and textures [B,nf,T,3] for the synthetic sphere family.

    Cameras: azimuth = azim0 + 360*b/B (BASELINE.md section 3), viewing angle 30.
    Textures: U[0,1) rng(seed), T = texture_res**2 (surface) or 3 (vertex).
    """
    v, f = sphere_by_faces(num_faces, radius=radius, jitter=jitter)
    verts = np.broadcast_to(v[None], (batch,) + v.shape).copy()
    eyes = np.asarray([get_points_from_angles(distance, elevation, azim0 + 360.0 * b / batch) for b in range(batch)], np.float32)
    cam = perspective(look_at(verts, eyes), 30.0)
    fv = face_vertices(cam, f)
    rng = np.random.default_rng(seed)
    T = texture_res * texture_res if texture_type == 'surface' else 3
    tex = rng.random((batch, f.shape[0], T, 3), dtype=np.float32)
    return fv, tex


def random_triangles(batch, num_faces, seed=0, zmin=1.5, zmax=4.0, scale=0.5, texture_size=1):
    """Unstructured random triangles covering the screen (edge cases: overlaps, slivers)."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1.0, 1.0, (batch, num_faces, 1, 2))
    d = rng.normal(0.0, scale, (batch, num_faces, 3, 2))
    xy = (c + d).astype(np.float32)
    z = rng.uniform(zmin, zmax, (batch, num_faces, 3, 1)).astype(np.float32)
    fv = np.concatenate([xy, z], axis=3).astype(np.float32)
    tex = rng.random((batch, num_faces, texture_size, 3), dtype=np.float32)
    return np.ascontiguousarray(fv), tex


def nmr_scene(num_faces=280, batch=1, ts=2, fill_back=True, seed=1):
    """faces [B,nf(x2),3,3] and textures [B,nf(x2),ts,ts,ts,3] the way N3mrRasterizer.render_rgb builds
    them (jrender/renderer/dr/n3mr/rasterizer.py:83-88): reversed-winding copies appended, textures permuted."""
    fv, _ = make_scene(num_faces, batch=batch)
    tex = np.random.default_rng(seed).random((batch, fv.shape[1], ts, ts, ts, 3), dtype=np.float32)
    if fill_back:
        fv = np.concatenate([fv, fv[:, :, ::-1]], axis=1)
        tex = np.concatenate([tex, tex.transpose(0, 1, 4, 3, 2, 5)], axis=1)
    return np.ascontiguousarray(fv), np.ascontiguousarray(tex)


def sss_maps(size, seed):
    """Synthetic texture-space SSS maps [size, size, 3] (size a multiple of 16): (world, irradiance, specular).  The
    world coordinates are flat over 16 x 16 patches, as rasterized world coordinates are flat over faces, and some
    patches vary along x, so that the stretch takes values inside (0, 1); all three are zero in background holes."""
    rng = np.random.default_rng(seed)
    n = size // 16
    world = np.kron(rng.uniform(0, 255, (n, n, 3)), np.ones((16, 16, 1))).astype(np.float32)
    world += np.kron(rng.uniform(0, 1, (n, n, 1)), np.ones((16, 16, 3))).astype(np.float32) * np.float32(0.02) \
        * np.arange(size, dtype=np.float32)[None, :, None]
    hole = np.kron(rng.random((n, n)) < 0.3, np.ones((16, 16))).astype(bool)
    hole[:5] = True
    hole[:, -7:] = True
    irr = rng.uniform(0, 1, (size, size, 3)).astype(np.float32)
    spec = rng.uniform(0, 0.3, (size, size, 3)).astype(np.float32)
    for a in (world, irr, spec):
        a[hole] = 0
    return world, irr, spec
