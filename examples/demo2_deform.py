"""Silhouette-fitting geometry optimisation, port of the reference's demo2-deform.py
(/root/reference/demo2-deform.py:16-103) to jrender_b200: same model parametrisation, renderer
settings (sigma 1e-4, hard rgb, viewing angle 15), losses and optimiser.

The reference fits `data/source.npy` silhouettes (not available on the GPU box); by default this
script fits silhouettes rendered from a squashed/offset ellipsoid, which keeps it self-contained:

    python examples/demo2_deform.py [--iters 200] [--image-size 64] [--batch-size 24]
    python examples/demo2_deform.py --filename-input data/source.npy --camera-input data/camera.npy \
        --template-mesh data/obj/sphere/sphere_1352.obj          # the reference's inputs
"""
import argparse
import os
import sys
import time

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import neg_iou_loss, LaplacianLoss, FlattenLoss, workloads as wl  # noqa: E402


class Model(nn.Module):
    """demo2-deform.py:16-46."""

    def __init__(self, vertices, faces):
        super(Model, self).__init__()
        self.register_buffer('vertices', vertices[None] * 0.5)
        self.register_buffer('faces', faces[None])
        self.displace = nn.Parameter(torch.zeros_like(self.vertices))
        self.center = nn.Parameter(torch.zeros((1, 1, 3)))
        self.laplacian_loss = LaplacianLoss(self.vertices[0], self.faces[0])
        self.flatten_loss = FlattenLoss(self.faces[0])

    def forward(self, batch_size):
        base = torch.log(self.vertices.abs() / (1 - self.vertices.abs()))
        centroid = torch.tanh(self.center)
        vertices = torch.sigmoid(base + self.displace) * torch.sign(self.vertices)
        vertices = torch.relu(vertices) * (1 - centroid) - torch.relu(-vertices) * (centroid + 1)
        vertices = vertices + centroid
        laplacian_loss = self.laplacian_loss(vertices).mean()
        flatten_loss = self.flatten_loss(vertices).mean()
        return jr.Mesh(vertices.repeat(batch_size, 1, 1), self.faces.repeat(batch_size, 1, 1)), laplacian_loss, flatten_loss


def synthetic_targets(renderer, faces, batch_size, device):
    """Silhouettes of an ellipsoid (sphere template scaled 0.45/0.3/0.38 and shifted) seen from the cameras."""
    v, f = wl.sphere_by_faces(3280, radius=1.0)
    v = v * np.float32([0.45, 0.30, 0.38]) + np.float32([0.05, -0.04, 0.0])
    mesh = jr.Mesh(torch.from_numpy(v).to(device)[None].repeat(batch_size, 1, 1),
                   torch.from_numpy(f).to(device)[None].repeat(batch_size, 1, 1))
    with torch.no_grad():
        return renderer.render_mesh(mesh, mode='silhouettes')


def iou(a, b):
    a, b = (a > 0.5).float(), (b > 0.5).float()
    return float(((a * b).sum((1, 2)) / ((a + b - a * b).sum((1, 2)) + 1e-6)).mean())


def run(iters=200, image_size=64, batch_size=24, filename_input=None, camera_input=None, template_mesh=None,
        output_dir=None, device="cuda", verbose=True, cuda_graph=False):
    dev = torch.device(device)
    if template_mesh:
        v, f = jr.load_obj(template_mesh)
    else:
        vv, ff = wl.sphere_by_faces(3280, radius=1.0)
        v, f = torch.from_numpy(vv), torch.from_numpy(ff)
    model = Model(v.to(dev), f.to(dev)).to(dev)
    renderer = jr.Renderer(image_size=image_size, sigma_val=1e-4, aggr_func_rgb='hard', camera_mode='look_at',
                           viewing_angle=15, dr_type='softras', bin_size=16, max_elems_per_bin=2700,
                           max_faces_per_pixel_for_grad=16)
    if filename_input and camera_input:
        images = np.load(filename_input).astype('float32') / 255.
        cameras = np.load(camera_input).astype('float32')
        batch_size = min(batch_size, images.shape[0])
        target = torch.from_numpy(images[:batch_size, 3]).to(dev)
        if target.shape[-1] != image_size:
            target = torch.nn.functional.interpolate(target[:, None], size=image_size, mode='nearest')[:, 0]
        cams = torch.from_numpy(cameras[:batch_size]).to(dev)
        renderer.transform.set_eyes_from_angles(cams[:, 0], cams[:, 1], cams[:, 2])
    else:
        az = torch.arange(batch_size, device=dev, dtype=torch.float32) * (360.0 / batch_size)
        el = 30.0 * torch.sin(torch.arange(batch_size, device=dev, dtype=torch.float32))
        renderer.transform.set_eyes_from_angles(torch.full((batch_size,), 2.732 * 2, device=dev), el, az)
        target = synthetic_targets(renderer, f, batch_size, dev)
    optimizer = torch.optim.Adam(model.parameters(), 0.01, betas=(0.5, 0.99), capturable=cuda_graph)
    hist = []

    def iteration():
        mesh, laplacian_loss, flatten_loss = model(batch_size)
        images_pred = renderer.render_mesh(mesh, mode='silhouettes')
        loss = neg_iou_loss(images_pred, target) + 0.03 * laplacian_loss + 0.0003 * flatten_loss
        optimizer.zero_grad(set_to_none=True)
        loss.backward()
        optimizer.step()
        return loss, images_pred

    last = {}

    def log(i, loss, images_pred):
        last["images"] = images_pred.detach()
        if i % 20 == 0 or i == iters - 1:
            hist.append((i, float(loss.item()), iou(images_pred.detach(), target)))
            if verbose:
                print("iter %4d  loss %.4f  IoU %.4f" % hist[-1], flush=True)

    if cuda_graph:
        # The whole iteration (model, transform, raster kernels through the C ABI, losses, autograd
        # backward, Adam) is captured once and replayed: at 64^2 the loop is launch-bound, ~400 small
        # kernels per iteration.  The library enqueues everything on the capturing stream and never
        # synchronises, so it is capture-safe.  The warm-up iterations below are part of the fit.
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for i in range(3):
                log(i, *iteration())
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        optimizer.zero_grad(set_to_none=True)
        with torch.cuda.graph(graph):
            static_loss, static_pred = iteration()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for i in range(4, iters):
            graph.replay()
            log(i, static_loss, static_pred)
        e1.record()
        torch.cuda.synchronize()
        timed = max(1, iters - 4)
        dt, dt_dev = (time.time() - t0) * iters / timed, e0.elapsed_time(e1) / 1000.0 * iters / timed
    else:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for i in range(iters):
            log(i, *iteration())
        e1.record()
        torch.cuda.synchronize()
        dt, dt_dev = time.time() - t0, e0.elapsed_time(e1) / 1000.0
    if output_dir:
        os.makedirs(output_dir, exist_ok=True)
        jr.save_obj(os.path.join(output_dir, 'plane.obj'), model(1)[0].vertices[0], model.faces[0])
    with torch.no_grad():
        vertices = model(1)[0].vertices[0].detach()
    return dict(ms_per_iter=1000.0 * dt / iters, device_ms_per_iter=1000.0 * dt_dev / iters, batch_size=batch_size, history=hist, final_iou=hist[-1][2], first_iou=hist[0][2],
                images=last["images"], vertices=vertices)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('-i', '--filename-input', type=str, default=None)
    ap.add_argument('-c', '--camera-input', type=str, default=None)
    ap.add_argument('-t', '--template-mesh', type=str, default=None)
    ap.add_argument('-o', '--output-dir', type=str, default=None)
    ap.add_argument('-b', '--batch-size', type=int, default=24)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--image-size', type=int, default=64)
    ap.add_argument('--cuda-graph', action='store_true', help='capture one iteration in a CUDA graph and replay it')
    a = ap.parse_args()
    r = run(a.iters, a.image_size, a.batch_size, a.filename_input, a.camera_input, a.template_mesh, a.output_dir,
            cuda_graph=a.cuda_graph)
    print("ms/iter %.2f  IoU %.4f -> %.4f" % (r["ms_per_iter"], r["first_iou"], r["final_iou"]))
