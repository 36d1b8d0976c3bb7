"""GPU parity of the fused surface-lighting kernel (csrc/lighting_api.cu, SURVEY.md 8f rank 1).

Forward against the reference's OWN Python (lighting/lighting.py:159-223 run through the numpy jittor stub,
tests/golden/ref_host_lighting_stage.npz) and against the op-by-op PyTorch mirror; backward (vertices through the face
normals / view vector, textures through the clamp) against the mirror's autograd in float64.
Stated tolerances: lit textures 2e-5 of max (the golden's own tolerance on CPU; GGX ratios amplify ulps), gradients
1e-4 of max |grad| (float32 forward-mode derivatives vs float64 reverse mode).
Every fused call is also held to the kernels' float32 emulation (test_lighting_edges_gpu.hold_to_emulation): lit
textures and per-texel gradients bit for bit, vertex gradients within the float atomics' order bound.
"""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import workloads as wl

from tests.test_lighting_edges_gpu import hold_to_emulation, kernel_calls  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def _mesh(g, dev, spec, dtype=torch.float32):
    m = jr.Mesh(torch.from_numpy(g["vertices"]).to(dev, dtype), torch.from_numpy(g["faces"]).to(dev),
                textures=torch.from_numpy(g["textures"].copy()).to(dev, dtype))
    m.metallic_textures = m.metallic_textures.to(dtype)
    m.roughness_textures = m.roughness_textures.to(dtype)
    m.with_specular = spec
    return m


@pytest.mark.parametrize("spec", [True, False])
def test_fused_lighting_matches_reference_python_golden(cuda_device, kernel_calls, spec):
    g = np.load(os.path.join(G, "ref_host_lighting_stage.npz"))
    eyes = torch.from_numpy(g["eyes"]).to(cuda_device)
    light = jr.Lighting()
    assert light._fusable(_mesh(g, cuda_device, spec), eyes)
    out = light(_mesh(g, cuda_device, spec), eyes).textures.cpu().numpy()
    ref = g["lit_" + ("specular" if spec else "diffuse")]
    assert np.abs(out - ref).max() <= 2e-5 * np.abs(ref).max()
    mirror = jr.Lighting()
    mirror.fused = False
    out2 = mirror(_mesh(g, cuda_device, spec), eyes).textures.cpu().numpy()
    assert np.abs(out - out2).max() <= 2e-5 * np.abs(ref).max()
    hold_to_emulation(kernel_calls)


@pytest.mark.parametrize("spec,tex6", [(True, False), (False, False), (True, True)])
def test_fused_lighting_gradients_match_float64_autograd(cuda_device, kernel_calls, spec, tex6):
    rng = np.random.default_rng(5)
    v, f = wl.sphere_by_faces(280)
    B = 3
    vb = (v[None] + rng.normal(0, 0.03, (B,) + v.shape)).astype(np.float32)
    shape = (B, f.shape[0], 2, 2, 2, 3) if tex6 else (B, f.shape[0], 4, 3)
    tex = rng.uniform(0.0, 1.3, shape).astype(np.float32)     # some texels saturate the clamp
    met = rng.uniform(0, 1, shape[:-1] + (1,)).astype(np.float32)
    rou = rng.uniform(0.2, 1, shape[:-1] + (1,)).astype(np.float32)
    eyes = np.float32([[0.0, 0.0, -2.7], [1.0, 1.5, -2.0], [-2.0, 0.3, 1.0]])
    gout = rng.uniform(-1, 1, shape).astype(np.float32)
    res = {}
    for name, dtype, fused in (("fused", torch.float32, True), ("mirror64", torch.float64, False)):
        vt = torch.from_numpy(vb).to(cuda_device, dtype).requires_grad_(True)
        tt = torch.from_numpy(tex).to(cuda_device, dtype).requires_grad_(True)
        m = jr.Mesh(vt, torch.from_numpy(f)[None].repeat(B, 1, 1).to(cuda_device), textures=tt, dr_type='n3mr' if tex6 else 'softras',
                    metallic_textures=torch.from_numpy(met).to(cuda_device, dtype), roughness_textures=torch.from_numpy(rou).to(cuda_device, dtype))
        m.with_specular = spec
        light = jr.Lighting(intensity_ambient=0.4, color_ambient=[1, 0.9, 0.8], intensity_directionals=0.7,
                            color_directionals=[0.9, 1, 0.7], directions=[0.3, 1, -0.4])
        light.fused = fused
        assert light._fusable(m, torch.from_numpy(eyes).to(cuda_device, dtype)) == fused or not fused
        out = light(m, torch.from_numpy(eyes).to(cuda_device, dtype)).textures
        out.backward(torch.from_numpy(gout).to(cuda_device, dtype))
        res[name] = (out.detach().double().cpu().numpy(), vt.grad.double().cpu().numpy(), tt.grad.double().cpu().numpy())
    a, b = res["fused"], res["mirror64"]
    assert np.abs(a[0] - b[0]).max() <= 2e-5
    assert np.abs(b[1]).max() > 0
    assert np.abs(a[1] - b[1]).max() <= 1e-4 * np.abs(b[1]).max(), np.abs(a[1] - b[1]).max() / np.abs(b[1]).max()
    assert np.abs(a[2] - b[2]).max() <= 1e-4 * np.abs(b[2]).max()
    hold_to_emulation(kernel_calls)


def test_renderer_uses_the_fused_lighting_and_counts_one_launch(cuda_device):
    from jrender_b200 import _lib
    v, f = wl.sphere_by_faces(280)
    r = jr.Renderer(image_size=64, camera_mode='look_at')
    r.transform.set_eyes_from_angles(2.732, 30, 40)
    tex = torch.rand(1, f.shape[0], 1, 3, device=cuda_device)
    L = _lib.lib()
    n0 = L.b200r_launch_count()
    img = r(torch.from_numpy(v)[None].to(cuda_device), torch.from_numpy(f)[None].to(cuda_device), tex)
    torch.cuda.synchronize()
    assert tuple(img.shape) == (1, 3, 64, 64) and float(img.max()) > 0.2
    assert L.b200r_launch_count() - n0 >= 6   # lighting, projection, face setup, binning, tile order, forward: all through the C ABI
