"""Albedo fit through subsurface scattering: render target views of the demo1.5 head (or, when it is not staged, the
generated UV sphere of demo1_5_render_normal_map.py) lit with SSS, then fit the albedo textures from flat 0.5 grey with
Adam, with `Lighting.sss_grad = True` so that the gradient flows through the texture-space blur.

    python examples/demo1_5_fit_sss.py [--iters 30] [--views 4] [--size 256] [--lr 0.05]

Prints the image loss before and after, the mean absolute albedo error over the texels the views reach (those that
received a gradient), and the milliseconds per iteration.  The albedo is kept in [0.05, 1]: the gradient of
sqrt(textures * diffuse) is infinite where the product is 0.
"""
import argparse
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from examples.demo1_5_render_normal_map import CAMERA_DISTANCE, ELEVATION, load_mesh, renderer  # noqa: E402


def render(r, mesh, textures, azimuth):
    m = jr.Mesh(mesh.vertices, mesh.faces, textures=textures, texture_res=mesh.texture_res,
                normal_textures=mesh.normal_textures, TBN=mesh.TBN, with_SSS=True, face_texcoords=mesh.face_texcoords)
    r.transform.set_eyes_from_angles(CAMERA_DISTANCE, ELEVATION, azimuth)
    return r.render_mesh(m, mode='rgb')[0]


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--iters", type=int, default=30)
    p.add_argument("--views", type=int, default=4)
    p.add_argument("--size", type=int, default=256)
    p.add_argument("--lr", type=float, default=0.05)
    a = p.parse_args(argv)
    dev = torch.device("cuda")
    with tempfile.TemporaryDirectory() as d:
        mesh, name = load_mesh(dev, texture_res=5, sphere_dir=d)
    print("mesh: %s (%d faces, %d texels per face), SSS" % (name, mesh.faces.shape[1], mesh.textures.shape[2]))
    r = renderer(a.size)
    r.lighting.sss_grad = True
    azimuths = [360.0 * k / a.views for k in range(a.views)]
    truth = mesh.textures.detach().clamp(0.05, 1)
    with torch.no_grad():
        targets = [render(r, mesh, truth, az) for az in azimuths]
    param = torch.full_like(truth, 0.5).requires_grad_(True)
    seen = torch.zeros(truth.shape[:-1], dtype=torch.bool, device=dev)
    opt = torch.optim.Adam([param], lr=a.lr)
    losses, times = [], []
    for _ in range(a.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        opt.zero_grad()
        loss = sum(((render(r, mesh, param, az) - t) ** 2).sum() for az, t in zip(azimuths, targets))
        loss.backward()
        opt.step()
        with torch.no_grad():
            param.clamp_(0.05, 1)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        seen |= param.grad.abs().sum(-1) > 0
        losses.append(float(loss.detach()))
    with torch.no_grad():
        final = float(sum(((render(r, mesh, param, az) - t) ** 2).sum() for az, t in zip(azimuths, targets)))
    err0 = float((0.5 - truth[seen]).abs().mean())
    err1 = float((param.detach()[seen] - truth[seen]).abs().mean())
    ms = 1e3 * sorted(times[1:] or times)[len(times[1:] or times) // 2]
    print("loss %.5g -> %.5g after %d iterations" % (losses[0], final, a.iters))
    print("albedo mean |error| over %d reached texels: %.4f -> %.4f" % (int(seen.sum()), err0, err1))
    print("%.1f ms per iteration (median; %d views at %d^2, forward + backward + Adam)" % (ms, a.views, a.size))
    return 0 if final < losses[0] else 1


if __name__ == "__main__":
    sys.exit(main())
