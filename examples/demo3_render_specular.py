"""Rendering the textured cow with Cook-Torrance specular lighting from a circle of viewpoints and with a sweep of
sigma / gamma: port of the reference's demo3-render_specular.py (:26-72) to jrender_b200 -- same loader call (texture_res
5), renderer defaults, metallic 0.5 and roughness 0.4 on every texel, camera path and parameter sweep.  Frames are
written as PNG files (the reference writes GIFs through imageio), and the mesh is saved as .obj like the reference's :72.

    python examples/demo3_render_specular.py -i data/obj/spot/spot_triangulated.obj -o out/   # needs the .obj/.mtl/.png
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jrender_b200 as jr  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_OBJ = os.path.join(ROOT, "baseline", "_ref", "assets", "data", "obj", "spot", "spot_triangulated.obj")


def save_png(path, chw):
    import cv2
    img = (255 * chw.detach().clamp(0, 1).cpu().numpy().transpose(1, 2, 0)).astype(np.uint8)
    cv2.imwrite(path, img[:, :, ::-1])


def run(filename_obj=DEFAULT_OBJ, step=4, device='cuda:0'):
    """Returns the mesh and two lists of [3, H, W] frames: the rotation (azimuth 0, step, ... < 360) and the sigma / gamma
    sweep at azimuth 45."""
    camera_distance, elevation = 2.732, 30
    dev = torch.device(device)
    # load from Wavefront .obj file (:27); create renderer with SoftRas (:30)
    mesh = jr.Mesh.from_obj(filename_obj, load_texture=True, texture_res=5, texture_type='surface', dr_type='softras').to(dev)
    renderer = jr.Renderer(dr_type='softras')
    # metallic 0.5, roughness 0.4 (:36-38)
    metallic_textures = torch.zeros((1, mesh.faces.shape[1], 5 * 5, 1), device=dev) + 0.5
    roughness_textures = torch.zeros((1, mesh.faces.shape[1], 5 * 5, 1), device=dev) + 0.4
    rotation, blurring = [], []
    with torch.no_grad():
        # draw object from different views (:41-53)
        for azimuth in range(0, 360, step):
            mesh.reset_()
            renderer.transform.set_eyes_from_angles(camera_distance, elevation, azimuth)
            rgb = renderer(mesh.vertices, mesh.faces, textures=mesh.textures, metallic_textures=metallic_textures,
                           roughness_textures=roughness_textures)
            rotation.append(rgb[0])
        # draw object from different sigma and gamma (:56-68)
        renderer.transform.set_eyes_from_angles(camera_distance, elevation, 45)
        for gamma_pow in np.arange(-4, -2, 0.2):
            mesh.reset_()
            renderer.set_gamma(10 ** gamma_pow)
            renderer.set_sigma(10 ** (gamma_pow - 1))
            images = renderer(mesh.vertices, mesh.faces, textures=mesh.textures, metallic_textures=metallic_textures,
                              roughness_textures=roughness_textures)
            blurring.append(images[0])
    mesh.reset_()
    return mesh, rotation, blurring


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('-i', '--filename-input', type=str, default=DEFAULT_OBJ)
    ap.add_argument('-o', '--output-dir', type=str, default='output_render_specular')
    ap.add_argument('--step', type=int, default=4, help="azimuth step in degrees (demo3: 4)")
    args = ap.parse_args(argv)
    mesh, rotation, blurring = run(args.filename_input, args.step)
    os.makedirs(args.output_dir, exist_ok=True)
    for num, image in enumerate(rotation):
        save_png(os.path.join(args.output_dir, 'rotation_%03d.png' % num), image)
    for num, image in enumerate(blurring):
        save_png(os.path.join(args.output_dir, 'bluring_%03d.png' % num), image)
    mesh.save_obj(os.path.join(args.output_dir, 'saved_spot.obj'))   # save to .obj (:71-72)
    print("wrote %d frames and saved_spot.obj to %s" % (len(rotation) + len(blurring), args.output_dir))


if __name__ == '__main__':
    main()
