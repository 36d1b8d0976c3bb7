"""The SoftRas backward (k_softras_backward_lane + finalize) against the oracle's per-entry bound
(oracle.softras.backward_bound) on the scenes of softras_backward_cases.py, under both tail settings; the fused
anti-aliased backward; and the headline image on strided rows.  The oracle's backward always runs on the kernel's own
forward outputs (tests.util.backward_bound_ratio), so both sides sum the terms of the same pairs."""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests import softras_backward_cases as SC
from tests.util import backward_bound_ratio, run_cuda

pytestmark = pytest.mark.gpu

CASES = SC.cases()


@pytest.fixture(params=[0, 1], ids=["fp32_tail", "exact_tail"])
def exact_tail(request, cuda_device):
    from jrender_b200 import _lib
    _lib.set_option("softras_exact_tail", request.param)
    yield request.param
    _lib.set_option("softras_exact_tail", 0)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_case_within_per_entry_bound(i, exact_tail):
    name, fv, tex, P, g = CASES[i]
    got = run_cuda(fv, tex, P, grad=g)
    worst = backward_bound_ratio(got, fv, tex, P, g, exact_tail=bool(exact_tail))
    print("%s exact_tail=%d worst |got - g64| / bound: %s" % (name, exact_tail, worst))


@pytest.mark.parametrize("rgb", ["softmax", "hard"])
def test_fused_antialiased_backward_against_oracle_at_2x(cuda_device, rgb):
    """anti_aliasing=True renders at 2H and the fused backward reads the pooled gradient: every 2H pixel gets g / 4
    (exact: a power of two) of its H pixel.  The oracle sums the 2H terms on the kernel's own 2H forward."""
    import torch
    from jrender_b200 import SoftRasterizer

    class M:
        pass
    fv, tex = wl.make_scene(280, batch=2, texture_res=2)
    H = 40
    m = M()
    m.face_vertices = torch.from_numpy(fv).cuda().requires_grad_(True)
    m.face_textures = torch.from_numpy(tex).cuda().requires_grad_(True)
    r = SoftRasterizer(image_size=H, anti_aliasing=True, fill_back=True, sigma_val=3e-5, aggr_func_rgb=rgb)
    assert r.fused_antialiasing
    g = np.random.default_rng(7).uniform(-1, 1, (2, 4, H, H)).astype(np.float32)
    alpha_out, rgb_out = r(m)
    torch.autograd.backward([rgb_out, alpha_out], [torch.from_numpy(g[:, :3]).cuda(), torch.from_numpy(g[:, 3]).cuda()])
    P = osr.Params(image_size=2 * H, sigma_val=3e-5, aggr_func_rgb=rgb)
    g2 = (np.repeat(np.repeat(g, 2, axis=2), 2, axis=3) / np.float32(4)).astype(np.float32)
    full = run_cuda(fv, tex, P)   # the 2H forward the fused op renders (same kernel, same bits)
    got = dict(full, grad_faces=m.face_vertices.grad.cpu().numpy(), grad_textures=m.face_textures.grad.cpu().numpy())
    backward_bound_ratio(got, fv, tex, P, g2)


def test_headline_image_on_strided_rows(cuda_device):
    """C3's image: 39 200 faces at 1024^2.  The upstream gradient is zero outside every 64th row, so the kernel's
    gradients are the oracle's sums over those rows."""
    fv, tex = wl.make_scene(39200, batch=1)
    P = osr.Params(image_size=1024)
    g = np.random.default_rng(2).uniform(-1, 1, (1, 4, 1024, 1024)).astype(np.float32)
    gm = np.zeros_like(g)
    gm[:, :, ::64] = g[:, :, ::64]
    got = run_cuda(fv, tex, P, grad=gm, want_faces_info=False)
    worst = backward_bound_ratio(got, fv, tex, P, gm, row_stride=64)
    assert np.abs(got["grad_faces"]).max() > 0
    print("headline strided rows: %s" % worst)
