"""Roughness-texture optimisation through the SoftRas renderer's Cook-Torrance lighting: port of the reference's
demo6-optim_roughness_textures.py (:19-41 model, :63-68 optimiser loop) to jrender_b200 -- same
model (spot cow at texture_res 4, fixed textures, metallic fixed at 0.4, a [1, nf, 16, 1] roughness parameter starting
at 1), renderer (defaults), camera (2.732, 30, 140), loss (sum of squared differences to a reference image) and optimiser
(Adam 0.1, betas (0.5, 0.999), 15 iterations).  The roughness gradient comes from the fused lighting kernel's backward
(b200r_surface_lighting_backward).

The reference fits `data/ref/ref_roughness.png`; by default this script fits a render of the cow with a known roughness
map (0.3 on faces whose centroid has x > 0, 0.7 elsewhere), which keeps it self-contained:

    python examples/demo6_optim_roughness_textures.py [--iters 15] [-ir ref_roughness.png]
"""
import argparse
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jrender_b200 as jr  # noqa: E402
from examples.demo5_optim_metallic_textures import DEFAULT_OBJ, TEXTURE_SIZE, load_image, split_by_x  # noqa: E402


class Model(nn.Module):
    """demo6-optim_roughness_textures.py:19-41."""

    def __init__(self, filename_obj, image_ref, device):
        super(Model, self).__init__()
        self.template_mesh = jr.Mesh.from_obj(filename_obj, texture_res=TEXTURE_SIZE, load_texture=True, dr_type='softras').to(device)
        self.register_buffer('vertices', self.template_mesh.vertices.detach())
        self.register_buffer('faces', self.template_mesh.faces.detach())
        self.register_buffer('textures', self.template_mesh.textures.detach())
        shape = (1, self.faces.shape[1], TEXTURE_SIZE * TEXTURE_SIZE, 1)
        self.register_buffer('metallic_textures', torch.zeros(shape, device=device) + 0.4)
        self.roughness_textures = nn.Parameter(torch.ones(shape, device=device))
        self.renderer = jr.Renderer(dr_type='softras')
        if image_ref is None:   # the target: the cow rendered with a known roughness map
            with torch.no_grad():
                image_ref = self.render(self.metallic_textures, split_by_x(self.vertices, self.faces, 0.3, 0.7)).detach()
        self.register_buffer('image_ref', image_ref)

    def render(self, metallic_textures, roughness_textures):
        self.renderer.transform.set_eyes_from_angles(2.732, 30, 140)
        return self.renderer(self.vertices, self.faces, self.textures, metallic_textures=metallic_textures,
                             roughness_textures=roughness_textures)

    def forward(self):
        image = self.render(self.metallic_textures, self.roughness_textures)
        return torch.sum((image - self.image_ref) ** 2)


def run(filename_obj=DEFAULT_OBJ, filename_ref=None, iters=15, device='cuda:0', log=None):
    dev = torch.device(device)
    image_ref = None if filename_ref is None else load_image(filename_ref, dev)
    model = Model(filename_obj, image_ref, dev)
    optimizer = torch.optim.Adam([model.roughness_textures], lr=0.1, betas=(0.5, 0.999))
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
    ap.add_argument('-ir', '--filename_ref', type=str, default=None, help="target image, e.g. the reference's ref_roughness.png")
    ap.add_argument('--iters', type=int, default=15)
    args = ap.parse_args(argv)
    model, losses = run(args.filename_obj, args.filename_ref, args.iters, log=5)
    print("loss %.3f -> %.3f" % (losses[0], losses[-1]))


if __name__ == '__main__':
    main()
