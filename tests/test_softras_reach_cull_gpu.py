"""The SoftRas forward's reach-polygon lane masks against the oracle on scenes built to break them.

In euclidean mode the forward drops a (pixel, face) pair before the per-pair body when the pixel lies outside the
face's reach polygon (softras_forward.cuh reach_lane_mask) and k_face_setup gave the face a margin
(softras_setup.cuh reach_margin_q; DESIGN.md section 4.4).  A dropped pair must be one the body would have left at
its distance threshold, so every output stays exactly what the oracle computes: ids and softmax_max bit-exact, the
colours and gradients within check()'s tolerances, hard-mode aggregates bit-exact.  Each scene runs under
softras_exact_tail = 0 (optimistic body plus re-run) and 1 (guarded divisions only).
"""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests import test_softras_ranges_gpu as rng_cases
from tests.test_softras_gpu import check


def _faces(v, z0=1.6, seed=0):
    """[n, 3, 2] xy -> [1, n, 3, 3] with depths in front of the sphere, and random textures."""
    v = np.asarray(v, np.float64)
    z = z0 + 0.2 * np.random.default_rng(seed).random(v.shape[:2] + (1,))
    fv = np.concatenate([v, z], -1).astype(np.float32)[None]
    return fv, np.random.default_rng(seed + 1).random((1, fv.shape[1], 1, 3), dtype=np.float32)


def _with(base, extra):
    fv, tex = base
    efv, etex = extra
    return np.concatenate([fv, efv], 1), np.concatenate([tex, etex], 1)


def slivers_scene(H):
    """Needles and slivers whose altitude / longest edge ratio straddles k_face_setup's 2^-12 conditioning bound, at
    every orientation, over the 3280-face sphere."""
    r = np.random.default_rng(21)
    faces = []
    for j in range(160):
        c = r.uniform(-0.8, 0.8, 2)
        ang = r.uniform(0, 2 * np.pi)
        L = 10.0 ** r.uniform(-2.5, -0.3)
        d = np.array([np.cos(ang), np.sin(ang)])
        n = np.array([-d[1], d[0]])
        ratio = 2.0 ** r.uniform(-14, -8)
        t = r.uniform(0.05, 0.95) if j % 2 else r.uniform(-0.5, 1.5)   # obtuse needles too
        faces.append([c, c + L * d, c + L * t * d + 2 * ratio * L * n])
    return _with(wl.make_scene(3280), _faces(faces, seed=21))


def pixel_centre_scene(H):
    """Random triangles with every vertex on a pixel centre, and axis-aligned and 45-degree edges."""
    r = np.random.default_rng(22)
    c = lambda i: (2.0 * i + 1.0 - H) / H
    faces = []
    for j in range(200):
        p = r.integers(0, H, (3, 2))
        if j % 3 == 0:
            p[1, 1] = p[0, 1]            # horizontal edge
        elif j % 3 == 1:
            p[1, 0] = p[0, 0]            # vertical edge
            p[2] = p[0] + (p[1, 1] - p[0, 1])   # 45 degrees
        faces.append(c(p.astype(np.float64)))
    return _with(wl.make_scene(280), _faces(faces, seed=22))


def coords_scene(H):
    """Faces with vertices from 2^-20 to 4 (the gate's bound) and beyond, edges crossing the image; and small faces
    far from the origin, where the barycentrics' rounding is largest."""
    r = np.random.default_rng(23)
    faces = []
    for j in range(120):
        s = 2.0 ** r.uniform(-20, 3)
        faces.append(r.uniform(-1, 1, (3, 2)) * s)
    for j in range(120):
        c = r.uniform(-1, 1, 2) * r.choice([0.9, 3.9, 4.1, 40.0])
        faces.append(c + r.uniform(-1, 1, (3, 2)) * 10.0 ** r.uniform(-3, 0))
    return _with(wl.make_scene(280), _faces(faces, seed=23))


def random_scene(H):
    fv, tex = wl.random_triangles(1, 600, seed=24, scale=0.05)
    return fv, tex


SCENES = {"sphere3280": lambda H: wl.make_scene(3280), "slivers": slivers_scene, "pixel_centres": pixel_centre_scene,
          "coords": coords_scene, "random": random_scene}


def both_tails(fv, tex, P, nan=False):
    from jrender_b200 import _lib
    try:
        for tail in (0, 1):
            _lib.set_option("softras_exact_tail", tail)
            check(fv, tex, P, nan=nan, exact_tail=bool(tail))
    finally:
        _lib.set_option("softras_exact_tail", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("name", list(SCENES))
def test_reach_cull_scenes_match_oracle(cuda_device, name, rgb):
    H = 128
    fv, tex = SCENES[name](H)
    both_tails(fv, tex, osr.Params(image_size=H, aggr_func_rgb=rgb, sigma_val=3e-5), nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize("sigma", [1e-7, 1e-5, 1e-3])
def test_reach_cull_border_sizes_match_oracle(cuda_device, sigma):
    """Reach radii from a fraction of a pixel to tens of pixels."""
    fv, tex = wl.make_scene(3280)
    both_tails(fv, tex, osr.Params(image_size=256, sigma_val=sigma))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["micro_faces", "huge_faces", "pixel_aligned"])
def test_reach_cull_out_of_range_inputs_match_oracle(cuda_device, name):
    fv, tex = rng_cases.CASES[name][0]()
    both_tails(fv, tex, rng_cases.params(name, "euclidean"), nan=True)


@pytest.mark.gpu
def test_reach_cull_non_finite_vertices_match_oracle(cuda_device):
    bad, _, tex = rng_cases.non_finite_scene()
    both_tails(bad, tex, osr.Params(image_size=rng_cases.H, sigma_val=1e-4), nan=True)
