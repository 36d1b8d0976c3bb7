"""examples/demo7_nerf.py: its cameras agree with jr's look_at + perspective, a few training steps on the fused kernels
equal those on the op-by-op mirror of oracle/volume.py, and training lowers the loss."""
import numpy as np
import pytest
import torch

import jrender_b200 as jr
from examples import demo7_nerf as demo
from jrender_b200 import vol
from oracle import volume as ov


@pytest.mark.parametrize("elevation,azimuth", [(30., 0.), (-10., 99.), (55., 250.)])
def test_pinhole_rays_land_on_pixel_centres(elevation, azimuth):
    """Points along each pixel's ray, projected by jr.Transform, land on that pixel's NDC centre (row 0 = top)."""
    H = W = 16
    eye = jr.get_points_from_angles(2.732, elevation, azimuth)
    c2w, focal, K = demo.camera(eye, W)
    o, d = vol.pinhole_get_rays(H, W, focal, torch.from_numpy(c2w), torch.from_numpy(K))
    tr = jr.Transform(camera_mode='look_at', viewing_angle=30)
    tr.set_eyes_from_angles(2.732, elevation, azimuth)
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    want = torch.stack([(2 * i + 1 - W) / W, (H - 2 * j - 1) / H], -1)
    for t in (1.5, 2.7, 4.0):
        p = (o + d * t).reshape(1, -1, 3)
        got = tr.transformer(p)[0, :, :2].reshape(H, W, 2)
        assert (got - want).abs().max().item() <= 1e-4


def small_args(**kw):
    a = demo.parser().parse_args([])
    a.netdepth = a.netdepth_fine = 4
    a.netwidth = a.netwidth_fine = 64
    a.N_rand, a.N_samples, a.N_importance = 256, 32, 64
    a.n_views, a.n_test, a.i_print = 8, 1, 0
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.gpu
def test_fused_and_mirror_training_steps_agree(cuda_device, monkeypatch):
    a = small_args(N_iters=3, size=64, precrop_iters=0, raw_noise_std=1.)
    data = demo.make_dataset(a.size, a.n_views, cuda_device)
    fused = demo.train(a, cuda_device, data)["losses"]
    monkeypatch.setattr(vol, "_composite", lambda raw, z, d, noise, white: ov.integrator_mirror(raw, z, d, noise, white))
    monkeypatch.setattr(vol, "_resample", lambda z, w, n, u: ov.fine_stage_mirror(z, w, n, u))
    mirror = demo.train(a, cuda_device, data)["losses"]
    assert len(fused) == 3 and np.allclose(fused, mirror, rtol=1e-4, atol=0), (fused, mirror)


@pytest.mark.gpu
def test_training_halves_the_loss(cuda_device):
    a = small_args(N_iters=300, size=64, precrop_iters=100)
    res = demo.train(a, cuda_device)
    first, last = np.mean(res["losses"][:50]), np.mean(res["losses"][-50:])
    print("demo7 300 iterations: mean loss of the first 50 %.5f, of the last 50 %.5f, held-out PSNR %.2f dB"
          % (first, last, res["psnr"]))
    assert last < 0.5 * first, (first, last)
