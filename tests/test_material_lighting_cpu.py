"""CPU checks of the material gradients of surface lighting: the backward's argument validation for grad_metallic /
grad_roughness (b200r_surface_lighting_backward), and float64 gradcheck of the op-by-op mirror w.r.t. metallic and
roughness -- the reference the fused kernel's material gradients are compared against on the GPU
(tests/test_material_lighting_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import jrender_b200 as jr


@pytest.fixture(scope="module")
def lib():
    from jrender_b200 import build, _lib
    build.build()          # nvcc cross-compiles sm_90a without a GPU
    return _lib.lib()


def test_material_gradient_arguments_are_validated(lib):
    """A material gradient without metallic / roughness, or with Tm == 0, is rejected on the host, before any CUDA call
    (the dummy device pointers below are never dereferenced)."""
    null, p = C.c_void_p(0), C.c_void_p(256)
    rgb = (C.c_float * 3)(1.0, 1.0, 1.0)

    def backward(metallic, roughness, grad_metallic, grad_roughness, Tm):
        return lib.b200r_surface_lighting_backward(p, p, p, metallic, roughness, p, p, p, null, grad_metallic, grad_roughness,
                                                   1, 1, 1, 1, 3, 1, 1, Tm, 0.5, rgb, 0.5, rgb, rgb, 1, null)

    for args in ((null, null, p, null, 4),     # grad_metallic, no material inputs
                 (null, null, null, p, 4),     # grad_roughness, no material inputs
                 (p, null, p, p, 4),           # roughness missing
                 (null, p, null, p, 4),        # metallic missing
                 (p, p, p, null, 0),           # Tm == 0
                 (p, p, null, p, 0)):
        assert backward(*args) == -1, args
        msg = lib.b200r_last_error()
        assert b"b200r_surface_lighting_backward" in msg and b"material" in msg, msg


def _gradcheck_scene(tex6, B=2, seed=0):
    rng = np.random.default_rng(seed)
    nv, nf = 9, 7
    v = rng.normal(0, 0.5, (B, nv, 3))
    f = np.stack([rng.choice(nv, 3, replace=False) for _ in range(nf)]).astype(np.int32)
    tail = (2, 2, 2) if tex6 else (4,)
    tex = rng.uniform(0.0, 1.3, (B, nf) + tail + (3,))   # some texels saturate the clamp
    met = rng.uniform(0.0, 1.0, (B, nf) + tail + (1,))
    rou = rng.uniform(0.2, 1.0, (B, nf) + tail + (1,))
    eyes = np.array([[0.3, 0.4, -2.7], [-1.5, 1.0, 1.2]])[:B]
    return v, f, tex, met, rou, eyes


@pytest.mark.parametrize("tex6", [False, True])
def test_mirror_material_gradients_pass_gradcheck(tex6):
    v, f, tex, met, rou, eyes = _gradcheck_scene(tex6)
    dt = torch.float64
    vt = torch.from_numpy(v).to(dt)
    ft = torch.from_numpy(f)[None].repeat(v.shape[0], 1, 1)
    tt, et = torch.from_numpy(tex).to(dt), torch.from_numpy(eyes).to(dt)
    light = jr.Lighting(intensity_ambient=0.4, color_ambient=[1, 0.9, 0.8], intensity_directionals=0.7,
                        color_directionals=[0.9, 1, 0.7], directions=[0.3, 1, -0.4])

    def lit(m, r):
        mesh = jr.Mesh(vt, ft, textures=tt, dr_type='n3mr' if tex6 else 'softras', metallic_textures=m, roughness_textures=r)
        assert mesh.with_specular
        return light(mesh, et).textures

    m = torch.from_numpy(met).to(dt).requires_grad_(True)
    r = torch.from_numpy(rou).to(dt).requires_grad_(True)
    assert torch.autograd.gradcheck(lit, (m, r), eps=1e-6, atol=1e-8, rtol=1e-6)
    gm, gr = torch.autograd.grad(lit(m, r).sum(), (m, r))
    assert gm.abs().max() > 0 and gr.abs().max() > 0   # the check is not vacuous
    # each face's gradient is spread evenly over its texels (the gradient of the mean)
    per_face = gm.reshape(gm.shape[0], gm.shape[1], -1)
    assert torch.equal(per_face, per_face[:, :, :1].expand_as(per_face))


def test_mirror_material_gradients_vanish_without_specular():
    v, f, tex, met, rou, eyes = _gradcheck_scene(False)
    m = torch.from_numpy(met).requires_grad_(True)
    mesh = jr.Mesh(torch.from_numpy(v), torch.from_numpy(f)[None].repeat(2, 1, 1), textures=torch.from_numpy(tex),
                   metallic_textures=m, roughness_textures=torch.from_numpy(rou))
    mesh.with_specular = False
    out = jr.Lighting()(mesh, torch.from_numpy(eyes)).textures
    assert not out.requires_grad or torch.autograd.grad(out.sum(), m, allow_unused=True)[0] is None
