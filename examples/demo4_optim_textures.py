"""Texture optimisation through the NMR renderer: port of the reference's demo4-optim_textures.py
(/root/reference/demo4-optim_textures.py:19-92) to jrender_b200 -- same model (vertices * 0.6, [1, nf, 4, 4, 4, 3] texture
parameter squashed by tanh), renderer (`dr_type='n3mr'`, look_at, orthogonal projection, ambient light only), loss (sum of
squared differences to a reference image from a random azimuth) and optimiser (Adam 0.03, betas (0.5, 0.999)).

The reference fits `data/ref/ref_texture.png`; by default this script fits a render of the cow with its own baked texture
from a fixed azimuth, which keeps it self-contained:

    python examples/demo4_optim_textures.py [--iters 200] [-ir ref.png] [--save out/cow.obj]

`--save` writes the fitted cow through Mesh.save_obj(save_texture=True) (.obj + .mtl + texture-atlas .png).
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


class Model(nn.Module):
    """demo4-optim_textures.py:19-45."""

    def __init__(self, filename_obj, image_ref, device):
        super(Model, self).__init__()
        self.template_mesh = jr.Mesh.from_obj(filename_obj, dr_type='n3mr', load_texture=True, texture_res=4).to(device)
        self.register_buffer('vertices', (self.template_mesh.vertices * 0.6).detach())
        self.register_buffer('faces', self.template_mesh.faces.detach())
        texture_size = 4
        self.textures = nn.Parameter(torch.ones((1, self.faces.shape[1], texture_size, texture_size, texture_size, 3), device=device))
        self.renderer = jr.Renderer(camera_mode='look_at', perspective=False, light_intensity_directionals=0.0,
                                    light_intensity_ambient=1.0, dr_type='n3mr')
        self.image_ref = image_ref   # [1,3,H,W] or None: then the template's own texture seen from `ref_azimuth` is the target
        self.ref_azimuth = 40.0
        if self.image_ref is None:
            with torch.no_grad():
                self.renderer.transform.set_eyes_from_angles(2.732, 0, self.ref_azimuth)
                self.image_ref = self.renderer(self.vertices, self.faces, self.template_mesh.textures).detach()
            self.fixed_view = True
        else:
            self.fixed_view = False

    def forward(self):
        num = self.ref_azimuth if self.fixed_view else np.random.uniform(0, 360)
        self.renderer.transform.set_eyes_from_angles(2.732, 0, num)
        image = self.renderer(self.vertices, self.faces, torch.tanh(self.textures))
        return torch.sum((image - self.image_ref) ** 2)


def run(filename_obj=DEFAULT_OBJ, filename_ref=None, iters=200, device='cuda:0', log=None):
    dev = torch.device(device)
    image_ref = None
    if filename_ref is not None:
        import cv2
        img = cv2.imread(filename_ref, cv2.IMREAD_COLOR)[:, :, ::-1].astype(np.float32) / 255.
        image_ref = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1)[None].to(dev)
    np.random.seed(1)
    model = Model(filename_obj, image_ref, dev)
    optimizer = torch.optim.Adam([model.textures], lr=0.03, betas=(0.5, 0.999))
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


def save(model, filename_obj, texture_res_out=16):
    """Write the fitted cow (the model's vertices, tanh of the texture parameter) as .obj + .mtl + .png: the NMR texture
    volumes go through the texture-atlas export (Mesh.save_obj(save_texture=True)), so another tool can open the result
    and Mesh.from_obj(..., load_texture=True, dr_type='n3mr') reads it back."""
    d = os.path.dirname(os.path.abspath(filename_obj))
    os.makedirs(d, exist_ok=True)
    with torch.no_grad():
        mesh = jr.Mesh(model.vertices, model.faces, torch.tanh(model.textures), dr_type='n3mr')
    mesh.save_obj(filename_obj, save_texture=True, texture_res_out=texture_res_out)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('-io', '--filename_obj', type=str, default=DEFAULT_OBJ)
    ap.add_argument('-ir', '--filename_ref', type=str, default=None)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--save', type=str, default=None, metavar='PATH', help='write the fitted textured mesh to PATH (.obj, + .mtl / .png)')
    args = ap.parse_args(argv)
    model, losses = run(args.filename_obj, args.filename_ref, args.iters, log=20)
    print("loss %.3f -> %.3f" % (losses[0], losses[-1]))
    if args.save:
        save(model, args.save)
        print("saved %s" % args.save)


if __name__ == '__main__':
    main()
