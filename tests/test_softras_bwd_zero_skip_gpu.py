"""The SoftRas backward skips the gradient atomics whose values are all +-0 (add_nonzero in softras_backward.cuh).
These scenes make whole classes of terms vanish, and the upstream gradients carry signed zeros, subnormals, NaN and
inf.  Every gradient entry whose oracle terms are all exactly zero must come out +0.0, NaN and inf must sit where the
oracle's are, and every other entry stays within oracle.softras.backward_bound.  An entry counts as all zero when its
terms are (A == 0) and the kernel's terms can differ from them by less than the smallest normal float in all
(E < 2^-126): such terms, and any sum of them, are at most subnormal, and the float atomics flush those to a zero.

What vanishes in zero_class_scene, at sigma 1e-3 and the default gamma 1e-4:
  - a wall covering the lower part of the image, deep inside which D == 1 exactly, so alpha_out == 1 and the alpha
    term of every pair there is 0;
  - a face hidden behind a front face 38 depth units nearer: its zp_softmax underflows to 0 and, with alpha_out == 1,
    every one of its terms is 0;
  - a small face alone in the upper right, whose pixels outside the triangle have a clipped barycentric w_k == 0."""
import numpy as np
import pytest

from oracle import softras as osr
from tests.util import backward_bound_ratio, run_cuda

pytestmark = pytest.mark.gpu

H = 40
HIDDEN = 1   # index of the hidden face


def zero_class_scene(T, texture_type):
    f = [[[-0.8, -0.7, 2.0], [0.8, -0.7, 2.0], [0.0, 0.9, 2.0]],          # front
         [[-0.25, -0.4, 40.0], [0.25, -0.4, 40.0], [0.0, 0.15, 40.0]],     # hidden behind the front face
         [[-1.5, -1.5, 45.0], [1.5, -1.5, 45.0], [1.5, 0.3, 45.0]],        # wall, lower part
         [[-1.5, -1.5, 45.0], [1.5, 0.3, 45.0], [-1.5, 0.3, 45.0]],
         [[0.6, 0.6, 3.0], [0.9, 0.6, 3.0], [0.75, 0.9, 3.0]]]             # alone, upper right
    fv = np.array([f], np.float32)
    tex = np.random.default_rng(T).random((1, fv.shape[1], T, 3), dtype=np.float32)
    return fv, tex


def upstream(kind):
    rng = np.random.default_rng(3)
    g = rng.uniform(-1, 1, (1, 4, H, H)).astype(np.float32)
    if kind == "signed_zeros":
        sub = np.where(rng.random((1, 4, H, H)) < 0.5, -1e-40, 1e-40).astype(np.float32)
        pick = rng.integers(0, 4, (1, 4, H, H))
        g = np.where(pick == 0, np.float32(0.0), g)
        g = np.where(pick == 1, np.float32(-0.0), g)
        g = np.where(pick == 2, sub, g)
        g[:, :, : H // 2, H // 2:] = -0.0            # whole warps of -0
        g[:, :, H // 2:, H // 2:] = sub[:, :, H // 2:, H // 2:]   # and of subnormals
    elif kind == "nonfinite":
        g[0, 0, 5, 5] = np.nan
        g[0, 1, 20, 20] = np.inf
        g[0, 3, 30, 10] = -np.inf
        g[0, 2, 12, 30] = np.inf
    return g


MODES = [("surface", 1, "softmax"), ("surface", 1, "none"), ("surface", 4, "softmax"), ("vertex", 3, "softmax")]


@pytest.mark.parametrize("kind", ["uniform", "signed_zeros", "nonfinite"])
@pytest.mark.parametrize("mode", MODES, ids=["%s_T%d_%s" % m for m in MODES])
def test_zero_terms_leave_positive_zero(cuda_device, mode, kind):
    texture_type, T, rgb = mode
    fv, tex = zero_class_scene(T, texture_type)
    P = osr.Params(image_size=H, sigma_val=1e-3, aggr_func_rgb=rgb, texture_type=texture_type)
    g = upstream(kind)
    got = run_cuda(fv, tex, P, grad=g)
    backward_bound_ratio(got, fv, tex, P, g)
    fwd = dict(soft_colors=got["soft_colors"], aggrs_info=got["aggrs_info"], faces_id_buffer=got["faces_id_buffer"],
               faces_info=got["faces_info"])
    stats = osr.backward(fv, tex, fwd, g, P, stats=True)
    assert (got["soft_colors"][:, 3] == 1.0).any()
    for k, st in zip(("grad_faces", "grad_textures"), stats):
        zero = (st["A"] == 0) & (st["E"] < 2.0 ** -126) & ~np.isnan(st["g64"])
        bits = got[k].view(np.uint32)
        assert (bits[zero] == 0).all(), "%s: %d entries with all-zero terms are not +0.0" % (k, (bits[zero] != 0).sum())
        if k == "grad_faces" and kind != "nonfinite":
            # the hidden face is listed and every one of its terms is exactly 0
            assert (st["N"][0, HIDDEN] > 0).all() and zero[0, HIDDEN].all()
