"""Normal and depth G-buffers of the spot cow through both rasterizers, and a geometry fit to them.

    python examples/render_gbuffers.py [-o out/]            # spot's normal and depth maps, SoftRas and NMR, as PNGs
    python examples/render_gbuffers.py --fit [--iters 200]  # deform demo 2's sphere toward spot's depth + normal maps

Renderer(Gbuffer='normal') renders N * 0.5 + 0.5 of each face, Gbuffer='depth' its camera depth over the largest depth
in the batch; both are differentiable w.r.t. the vertices, so they supervise a geometry fit with more than the
silhouette (the fit uses demo 2's model, losses and optimiser, with the G-buffers added to the silhouette IoU).
"""
import argparse
import lzma
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import neg_iou_loss  # noqa: E402
from examples.demo2_deform import Model  # noqa: E402
from jrender_b200 import workloads as wl  # noqa: E402

SPOT = os.path.join(ROOT, "tests", "golden", "spot_triangulated.obj.xz")


def load_spot(device):
    """spot's vertices [nv, 3] and faces [nf, 3] (5 856 faces), normalised like load_obj(normalization=True)."""
    with tempfile.TemporaryDirectory() as d, lzma.open(SPOT, "rb") as f:
        fn = os.path.join(d, "spot.obj")
        open(fn, "wb").write(f.read())
        v, f = jr.load_obj(fn, normalization=True)
    return v.to(device), f.to(device)


def gbuffer_renderer(mode, dr_type, image_size=256, batch=1):
    r = jr.Renderer(image_size=image_size, dr_type=dr_type, Gbuffer=mode, sigma_val=1e-5, anti_aliasing=False)
    az = torch.arange(batch, dtype=torch.float32) * (360.0 / batch) + 30.0
    r.transform.set_eyes_from_angles(torch.full((batch,), 2.732), torch.full((batch,), 25.0), az)
    return r


def render(v, f, mode, dr_type, image_size=256, batch=1, out='rgb'):
    """The G-buffer images [batch, 3, S, S] (out='rgb'), or (coverage [batch, S, S], G-buffer) with out=None (SoftRas)."""
    r = gbuffer_renderer(mode, dr_type, image_size, batch)
    r.transform.transformer._eye = r.transform.transformer._eye.to(v.device)
    T = 1 if dr_type == 'softras' else 8
    tex = torch.ones((batch, f.shape[0], T, 3) if dr_type == 'softras' else (batch, f.shape[0], 2, 2, 2, 3),
                     device=v.device)
    mesh = jr.Mesh(v[None].expand(batch, -1, -1), f[None].expand(batch, -1, -1), textures=tex, dr_type=dr_type)
    return r.render_mesh(mesh, mode=out)


def fit(iters=200, image_size=64, batch=8, device="cuda", verbose=True):
    """Deform demo 2's sphere toward spot's silhouette, depth and normal G-buffers; returns the loss history."""
    dev = torch.device(device)
    sv, sf = load_spot(dev)
    vv, ff = wl.sphere_by_faces(3280, radius=1.0)
    model = Model(torch.from_numpy(vv).to(dev), torch.from_numpy(ff).to(dev)).to(dev)
    rs = {m: gbuffer_renderer(m, 'softras', image_size, batch) for m in ('normal', 'depth')}
    for r in rs.values():
        r.transform.transformer._eye = r.transform.transformer._eye.to(dev)
    with torch.no_grad():
        targets = {m: render(sv * 0.6, sf, m, 'softras', image_size, batch, out=None) for m in rs}
    optimizer = torch.optim.Adam(model.parameters(), 0.01, betas=(0.5, 0.99))
    hist = []
    for i in range(iters):
        mesh, lap, flat = model(batch)
        loss = 0.03 * lap + 0.0003 * flat
        for m, r in rs.items():
            tex = torch.ones((batch, mesh.faces.shape[1], 1, 3), device=dev)
            alpha, rgb = r.render_mesh(jr.Mesh(mesh.vertices, mesh.faces, textures=tex), mode=None)
            t_alpha, t_rgb = targets[m]
            loss = loss + ((rgb - t_rgb) ** 2 * t_alpha[:, None]).mean() * 10
            if m == 'depth':
                loss = loss + neg_iou_loss(alpha, t_alpha)
        optimizer.zero_grad(set_to_none=True)
        loss.backward()
        optimizer.step()
        hist.append(float(loss.item()))
        if verbose and (i % 20 == 0 or i == iters - 1):
            print("iter %4d  loss %.4f" % (i, hist[-1]), flush=True)
    return hist


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('-o', '--output-dir', default='gbuffers_out')
    ap.add_argument('--fit', action='store_true')
    ap.add_argument('--iters', type=int, default=200)
    a = ap.parse_args()
    if a.fit:
        fit(a.iters)
        return
    from PIL import Image
    os.makedirs(a.output_dir, exist_ok=True)
    v, f = load_spot(torch.device("cuda"))
    for dr in ('softras', 'n3mr'):
        for mode in ('normal', 'depth'):
            img = render(v, f, mode, dr)[0].detach().cpu().numpy()
            rgb = (np.clip(img[:3].transpose(1, 2, 0), 0, 1) * 255).astype(np.uint8)
            fn = os.path.join(a.output_dir, "spot_%s_%s.png" % (dr, mode))
            Image.fromarray(rgb).save(fn)
            print("wrote", fn)


if __name__ == "__main__":
    main()
