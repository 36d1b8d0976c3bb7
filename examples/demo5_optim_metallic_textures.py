"""Metallic-texture optimisation through the SoftRas renderer's Cook-Torrance lighting: port of the reference's
demo5-optim_metallic_textures.py (:19-41 model, :63-68 optimiser loop) to jrender_b200 -- same
model (spot cow at texture_res 4, fixed textures, a [1, nf, 16, 1] metallic parameter starting at 0, roughness fixed at
0.5), renderer (`light_intensity_directionals=1.0, light_intensity_ambient=0.0`), camera (2.732, 30, 140), loss (sum of
squared differences to a reference image) and optimiser (Adam 0.1, betas (0.5, 0.999), 20 iterations).  The metallic
gradient comes from the fused lighting kernel's backward (b200r_surface_lighting_backward).

The reference fits `data/ref/ref_metallic.png`; by default this script fits a render of the cow with a known metallic map
(0.9 on faces whose centroid has x > 0, 0.2 elsewhere), which keeps it self-contained:

    python examples/demo5_optim_metallic_textures.py [--iters 20] [-ir ref_metallic.png]
"""
import argparse
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jrender_b200 as jr  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_OBJ = os.path.join(ROOT, "baseline", "_ref", "assets", "data", "obj", "spot", "spot_triangulated.obj")
TEXTURE_SIZE = 4


def load_image(filename, device):
    """An RGB .png as a [1, 3, H, W] float tensor in [0, 1] (imread(...) / 255., permute(2, 0, 1), unsqueeze(0))."""
    import cv2
    img = cv2.imread(filename, cv2.IMREAD_COLOR)[:, :, ::-1].astype(np.float32) / 255.
    return torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1)[None].to(device)


def split_by_x(vertices, faces, positive, negative):
    """A [1, nf, TEXTURE_SIZE^2, 1] material map: `positive` on faces whose centroid has x > 0, `negative` elsewhere."""
    x = vertices[0][faces[0].long()][:, :, 0].mean(dim=1)
    per_face = torch.where(x > 0, positive, negative).to(vertices.dtype)
    return per_face[None, :, None, None].expand(1, -1, TEXTURE_SIZE * TEXTURE_SIZE, 1).contiguous()


class Model(nn.Module):
    """demo5-optim_metallic_textures.py:19-41."""

    def __init__(self, filename_obj, image_ref, device):
        super(Model, self).__init__()
        self.template_mesh = jr.Mesh.from_obj(filename_obj, texture_res=TEXTURE_SIZE, load_texture=True, dr_type='softras').to(device)
        self.register_buffer('vertices', self.template_mesh.vertices.detach())
        self.register_buffer('faces', self.template_mesh.faces.detach())
        self.register_buffer('textures', self.template_mesh.textures.detach())
        shape = (1, self.faces.shape[1], TEXTURE_SIZE * TEXTURE_SIZE, 1)
        self.metallic_textures = nn.Parameter(torch.zeros(shape, device=device))
        self.register_buffer('roughness_textures', torch.zeros(shape, device=device) + 0.5)
        self.renderer = jr.Renderer(dr_type='softras', light_intensity_directionals=1.0, light_intensity_ambient=0.0)
        if image_ref is None:   # the target: the cow rendered with a known metallic map
            with torch.no_grad():
                image_ref = self.render(split_by_x(self.vertices, self.faces, 0.9, 0.2), self.roughness_textures).detach()
        self.register_buffer('image_ref', image_ref)

    def render(self, metallic_textures, roughness_textures):
        self.renderer.transform.set_eyes_from_angles(2.732, 30, 140)
        return self.renderer(self.vertices, self.faces, self.textures, metallic_textures=metallic_textures,
                             roughness_textures=roughness_textures)

    def forward(self):
        image = self.render(self.metallic_textures, self.roughness_textures)
        return torch.sum((image - self.image_ref) ** 2)


def run(filename_obj=DEFAULT_OBJ, filename_ref=None, iters=20, device='cuda:0', log=None):
    dev = torch.device(device)
    image_ref = None if filename_ref is None else load_image(filename_ref, dev)
    model = Model(filename_obj, image_ref, dev)
    optimizer = torch.optim.Adam([model.metallic_textures], lr=0.1, betas=(0.5, 0.999))
    losses = []
    for it in range(iters):
        optimizer.zero_grad(set_to_none=True)
        loss = model()
        loss.backward()
        optimizer.step()
        losses.append(float(loss.detach()))
        if log is not None and it % log == 0:
            print("iter %4d  loss %.3f" % (it, losses[-1]), flush=True)
    return model, losses


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('-io', '--filename_obj', type=str, default=DEFAULT_OBJ)
    ap.add_argument('-ir', '--filename_ref', type=str, default=None, help="target image, e.g. the reference's ref_metallic.png")
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args(argv)
    model, losses = run(args.filename_obj, args.filename_ref, args.iters, log=5)
    print("loss %.3f -> %.3f" % (losses[0], losses[-1]))


if __name__ == '__main__':
    main()
