"""Normal-mapped rendering: port of the reference's demo1.5-SSS.py WITHOUT subsurface scattering (SSS is not ported;
`with_SSS` is accepted and ignored).  Same settings otherwise: the head at texture_res 15 with its `map_normal` bump map,
SoftRas with dist_func='barycentric' and aggr_func_rgb='hard' at 1024^2, ambient 0.45 and a directional light of 1
from (0.65, -0.2, -1), look_at camera at distance 2, elevation 20, 90 views every 4 degrees of azimuth.  The surface
lighting takes the normal-map branch: one normal per texel from normal_textures and the per-face TBN, shaded by the
fused kernel b200r_normal_mapped_lighting_forward.

The head (data/head/{head.obj, head.mtl, lambertian.jpg, bump.png}) is used when tools/stage_assets.py has staged it;
otherwise a generated UV sphere with a procedural 16-bit bump map stands in, and the script says so.

    python examples/demo1_5_render_normal_map.py [-o DIR] [--size 1024] [--step 4] [--fit [--fit-iters 100]]

--fit then recovers the normal map from those renders: it starts from flat tangent-space normals (0, 0, 1), renders
the same views, and minimises the squared image difference with Adam, through the fused kernel's gradient to the normal
textures.  It prints the image loss and the mean angle between the fitted and the true normals.
"""
import argparse
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import workloads as wl  # noqa: E402

HEAD = os.path.join(ROOT, "baseline", "_ref", "assets", "data", "head", "head.obj")
CAMERA_DISTANCE, ELEVATION = 2, 20


def renderer(image_size=1024):
    """demo1.5-SSS.py:27-29."""
    return jr.Renderer(dr_type='softras', image_size=image_size, light_intensity_ambient=0.45, light_color_ambient=[1, 1, 1],
                       light_intensity_directionals=1, light_color_directionals=[1.0, 1.0, 1.0],
                       light_directions=[0.65, -0.2, -1], dist_func="barycentric", aggr_func_rgb='hard',
                       camera_mode="look_at", eye=[1.1, 0.5, -1.5], camera_direction=[-0.8, -0.2, 1])


def write_sphere_asset(directory, segments=48, rings=24, bump_size=256):
    """A UV sphere (planar UVs from x and y) with a procedural 16-bit grayscale bump map, written as sphere.obj,
    sphere.mtl (`map_normal 1.0 bump.png`) and bump.png.  Returns the .obj path."""
    import cv2
    v, f = wl.uv_sphere(segments, rings)
    uv = np.clip((v[:, :2] / 0.8 + 1) / 2 * 0.98 + 0.01, 0, 1)
    y, x = np.mgrid[0:bump_size, 0:bump_size] / float(bump_size)
    # 16-bit heights reach 257 after / 255, and the reference's z component is 6 per pixel: amplitudes scaled by the
    # image size keep the normals within about 30 degrees of flat
    h = 0.5 + (10.0 / bump_size) * (np.sin(14 * np.pi * x) * np.sin(14 * np.pi * y) + 0.5 * np.sin(6 * np.pi * (x + y)))
    assert cv2.imwrite(os.path.join(directory, "bump.png"), np.round(h * 65535).astype(np.uint16))
    with open(os.path.join(directory, "sphere.mtl"), "w") as fh:
        fh.write("newmtl skin\nKd 0.85 0.7 0.6\nmap_normal 1.0 bump.png\n")
    path = os.path.join(directory, "sphere.obj")
    with open(path, "w") as fh:
        fh.write("mtllib sphere.mtl\n")
        fh.writelines("v %.6f %.6f %.6f\n" % tuple(p) for p in v)
        fh.writelines("vt %.6f %.6f\n" % tuple(t) for t in uv)
        fh.write("usemtl skin\n")
        fh.writelines("f %d/%d %d/%d %d/%d\n" % (a + 1, a + 1, b + 1, b + 1, c + 1, c + 1) for a, b, c in f)
    return path


def load_mesh(device, texture_res=15, sphere_dir=None):
    """(mesh, name): the staged head, else the generated sphere (written into sphere_dir)."""
    if os.path.exists(HEAD):
        path, name = HEAD, "head"
    else:
        path, name = write_sphere_asset(sphere_dir), "generated UV sphere with a procedural bump map"
    mesh = jr.Mesh.from_obj(path, load_texture=True, texture_res=texture_res, texture_type='surface', dr_type='softras',
                            normalization=True, with_SSS=True).to(device)
    return mesh, name


def render_views(r, mesh, normal_textures, azimuths):
    """One [3, H, W] image per azimuth, with `normal_textures` in place of the mesh's."""
    out = []
    for azimuth in azimuths:
        m = jr.Mesh(mesh.vertices, mesh.faces, textures=mesh.textures, normal_textures=normal_textures, TBN=mesh.TBN)
        r.transform.set_eyes_from_angles(CAMERA_DISTANCE, ELEVATION, azimuth)
        out.append(r.render_mesh(m, mode='rgb')[0])
    return out


def mean_angle_deg(a, b):
    a = torch.nn.functional.normalize(a.detach(), dim=-1, eps=1e-12)
    b = torch.nn.functional.normalize(b.detach(), dim=-1, eps=1e-12)
    return float(torch.rad2deg(torch.acos(torch.clamp((a * b).sum(-1), -1, 1))).mean())


def fit(r, mesh, targets, azimuths, iters=100, lr=0.05):
    """Fit the normal textures to `targets` from flat tangent-space normals.  Returns (losses, angles, start angle): the
    loss before each step, and the mean angular error (degrees) to the mesh's own normal textures after each step and
    before the first, over the texels the views reach (those that ever received a gradient)."""
    param = torch.zeros_like(mesh.normal_textures)
    param[..., 2] = 1
    flat = param.clone()
    param.requires_grad_(True)
    seen = torch.zeros(param.shape[:-1], dtype=torch.bool, device=param.device)
    opt = torch.optim.Adam([param], lr=lr)
    losses, angles = [], []
    for _ in range(iters):
        opt.zero_grad()
        loss = sum(torch.sum((img - t) ** 2) for img, t in zip(render_views(r, mesh, param, azimuths), targets))
        loss.backward()
        seen |= param.grad.abs().sum(-1) > 0
        opt.step()
        losses.append(float(loss.detach()))
        angles.append(mean_angle_deg(param[seen], mesh.normal_textures[seen]))
    return losses, angles, mean_angle_deg(flat[seen], mesh.normal_textures[seen])


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("-o", "--output-dir", default="demo1_5_output")
    p.add_argument("--size", type=int, default=1024)
    p.add_argument("--step", type=int, default=4, help="azimuth step in degrees (4: the reference's 90 views)")
    p.add_argument("--fit", action="store_true")
    p.add_argument("--fit-iters", type=int, default=100)
    p.add_argument("--fit-views", type=int, default=8)
    p.add_argument("--fit-size", type=int, default=256)
    a = p.parse_args(argv)
    import cv2
    dev = torch.device("cuda")
    os.makedirs(a.output_dir, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        mesh, name = load_mesh(dev, sphere_dir=d)
    print("mesh: %s (%d faces, %d texels per face); no SSS" % (name, mesh.faces.shape[1], mesh.textures.shape[2]))
    r = renderer(a.size)
    with torch.no_grad():
        for k, azimuth in enumerate(range(0, 360, a.step)):
            img = render_views(r, mesh, mesh.normal_textures, [azimuth])[0]
            frame = (255 * img.permute(1, 2, 0).clamp(0, 1).cpu().numpy()).astype(np.uint8)
            cv2.imwrite(os.path.join(a.output_dir, "rotation_%03d.png" % k), np.ascontiguousarray(frame[:, :, ::-1]))
    print("wrote %d frames to %s" % (len(range(0, 360, a.step)), a.output_dir))
    if a.fit:
        rf = renderer(a.fit_size)
        azimuths = [360.0 * k / a.fit_views for k in range(a.fit_views)]
        with torch.no_grad():
            targets = [t.detach() for t in render_views(rf, mesh, mesh.normal_textures, azimuths)]
        losses, angles, start = fit(rf, mesh, targets, azimuths, a.fit_iters)
        print("fit: flat normals start %.2f deg from the true ones on the texels the views reach" % start)
        for i in sorted({0, len(losses) // 4, len(losses) // 2, len(losses) - 1}):
            print("fit iter %4d  image loss %.5g  mean angular error %.2f deg" % (i, losses[i], angles[i]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
