"""Screen-space ambient occlusion, directional occlusion and FXAA on spot standing on a ground plane.

    python examples/render_ssao.py [-o ssao_out/] [--size 512]

Rasterizes the G-buffers the way render2's Render does (render2.py:343-361): one hard `barycentric` SoftRas raster of
the view-space face normals as vertex textures gives the normal buffer, and its aggrs_info the depth and the face ids;
width = tan(viewing_angle).  Then writes four PNGs:
    spot_plain.png  Lambert shading, no occlusion
    spot_ssao.png   Render.SSAO's composition: (1 - SSAO) blurred by a 5 x 5 / 25 conv_for_image, times the colour
    spot_ssdo.png   SSDO with 1024 samples
    spot_fxaa.png   FXAA of the SSDO image
"""
import argparse
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200.render2 import FXAA_cuda, SSAO_cuda, SSDO_cuda, conv_for_image  # noqa: E402
from examples.render_gbuffers import load_spot  # noqa: E402

EYE = (1.6, 1.1, -2.2)
VIEWING_ANGLE = 30.
LIGHT = (0.5, 0.8, -0.4)


def ground_plane(vertices, faces, n=8, extent=1.6):
    """spot's mesh with an n x n-quad square added under it at its lowest y, facing up."""
    y = float(vertices[:, 1].min())
    s = torch.linspace(-extent, extent, n + 1, device=vertices.device)
    gz, gx = torch.meshgrid(s, s, indexing="ij")
    pv = torch.stack((gx.reshape(-1), torch.full_like(gx.reshape(-1), y), gz.reshape(-1)), 1)
    k = torch.arange(n * (n + 1), device=vertices.device).reshape(n, n + 1)[:, :n].reshape(-1)
    quads = torch.stack((k, k + n + 1, k + 1, k + 1, k + n + 1, k + n + 2), 1).reshape(-1, 3)
    return torch.cat((vertices, pv)), torch.cat((faces, quads.to(faces.dtype) + vertices.shape[0]))


def gbuffers(vertices, faces, image_size, eye=EYE, viewing_angle=VIEWING_ANGLE):
    """(depth [S, S], face ids [S, S] int32, normals [S, S, 3], width) of the mesh seen from `eye`: the view-space
    face normals, turned towards the camera, rasterized as vertex textures by a hard barycentric SoftRas raster."""
    v = jr.look_at(vertices[None].float(), list(eye))[0]
    fv = v[faces.long()]
    n = torch.nn.functional.normalize(torch.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0], dim=1), dim=1)
    n = torch.where(((n * fv.mean(1)).sum(1) > 0)[:, None], -n, n)
    proj = jr.perspective(v[None], viewing_angle)[0][faces.long()]
    rast = jr.SoftRasterizeFunction(image_size=image_size, near=0.1, far=100, dist_func='barycentric',
                                    aggr_func_rgb='hard', texture_type='vertex', fill_back=True)
    colors, aggrs_info, _ = rast.raw(proj[None].contiguous(), n[:, None, :].expand(-1, 3, -1)[None].contiguous())
    normal = colors[0, :3].permute(1, 2, 0).contiguous()
    return aggrs_info[0, 0].contiguous(), aggrs_info[0, 1].int(), normal, math.tan(viewing_angle / 180. * math.pi)


def shade(face_ind, normal):
    """Lambert colour [S, S, 3] of a 0.85-grey surface under one directional light, white background."""
    light = torch.nn.functional.normalize(torch.tensor(LIGHT, device=normal.device), dim=0)
    lit = 0.3 + 0.7 * (normal @ light).clamp(min=0)
    return torch.where((face_ind >= 0)[..., None], 0.85 * lit[..., None].expand(-1, -1, 3), torch.ones_like(normal))


def ssao_composite(color, depth, face_ind, normal, width, sample_num=64, sample_range_r=0.15):
    """Render.SSAO's composition: (1 - occlusion), filtered by a 5 x 5 box of weight 1/25 with 0 outside, times the
    colour."""
    occ = SSAO_cuda(depth, face_ind, normal, width, sample_num, sample_range_r)
    ao = conv_for_image(1 - occ, torch.ones(5, 5, device=occ.device) / 25, 0)
    return color * ao[..., None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('-o', '--output-dir', default='ssao_out')
    ap.add_argument('--size', type=int, default=512)
    a = ap.parse_args()
    from PIL import Image
    os.makedirs(a.output_dir, exist_ok=True)
    v, f = ground_plane(*load_spot(torch.device("cuda")))
    depth, face_ind, normal, width = gbuffers(v, f, a.size)
    color = shade(face_ind, normal)
    ssdo = SSDO_cuda(color, depth, face_ind, normal, width, 1024, 0.15)
    images = {"plain": color, "ssao": ssao_composite(color, depth, face_ind, normal, width),
              "ssdo": ssdo, "fxaa": FXAA_cuda(ssdo)}
    for name, img in images.items():
        fn = os.path.join(a.output_dir, "spot_%s.png" % name)
        Image.fromarray((img.clamp(0, 1) * 255).byte().cpu().numpy()).save(fn)
        print("wrote", fn)


if __name__ == "__main__":
    main()
