"""Training a NeRF: port of the reference's demo7-nerf.py (and nerf_helper/utils.py:13-116) to
jrender_b200.vol -- the same MLP (D=8, W=256, skip at 4, view directions, positional encodings of 10 / 4 octaves), coarse
and fine networks, Adam at 5e-4 with the exponential decay, N_rand rays from one image per step and the centre crop of
the first iterations, with the lego config's sampling (configs/lego.txt: 64 + 128 samples, white background).

The blender / LLFF data cannot be downloaded, so the dataset is synthetic: views of the spot cow
(tests/golden/spot_triangulated.obj.xz + spot_texture.png) rendered by this package's own SoftRas renderer from a ring of
look_at cameras and composited over white.  Each camera becomes the c2w / focal / intrinsic of jrender_vol's pinhole
(pixel (i, j) looks through its centre, as jr's rasteriser samples it).  Dataset loaders, tensorboard, checkpoints and
MPI are left out.  Writes held-out renders and the PSNR under the output directory.

    python examples/demo7_nerf.py [-o demo7_output/] [--N_iters 2000] [--size 64]
"""
import argparse
import lzma
import math
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200.vol import pinhole_get_rays, render  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

img2mse = lambda x, y: torch.mean((x - y) ** 2)
mse2psnr = lambda x: -10. * torch.log(x) / math.log(10.)
to8b = lambda x: (255 * np.clip(x, 0, 1)).astype(np.uint8)


# ---- model (nerf_helper/utils.py:13-116) ---------------------------------------------------------------------------

class Embedder:
    def __init__(self, **kwargs):
        self.kwargs = kwargs
        embed_fns = []
        d = kwargs['input_dims']
        out_dim = 0
        if kwargs['include_input']:
            embed_fns.append(lambda x: x)
            out_dim += d
        max_freq, n_freqs = kwargs['max_freq_log2'], kwargs['num_freqs']
        if kwargs['log_sampling']:
            freq_bands = 2. ** torch.linspace(0., max_freq, steps=n_freqs)
        else:
            freq_bands = torch.linspace(2. ** 0., 2. ** max_freq, steps=n_freqs)
        for freq in freq_bands.tolist():
            for p_fn in kwargs['periodic_fns']:
                embed_fns.append(lambda x, p_fn=p_fn, freq=freq: p_fn(x * freq))
                out_dim += d
        self.embed_fns = embed_fns
        self.out_dim = out_dim

    def embed(self, inputs):
        return torch.cat([fn(inputs) for fn in self.embed_fns], -1)


def get_embedder(multires, i=0, input_dims=3):
    if i == -1:
        return nn.Identity(), 3
    eo = Embedder(include_input=True, input_dims=input_dims, max_freq_log2=multires - 1, num_freqs=multires,
                  log_sampling=True, periodic_fns=[torch.sin, torch.cos])
    return eo.embed, eo.out_dim


class NeRF(nn.Module):
    def __init__(self, D=8, W=256, input_ch=3, input_ch_views=3, output_ch=4, skips=[4], use_viewdirs=False):
        super().__init__()
        self.D, self.W, self.input_ch, self.input_ch_views = D, W, input_ch, input_ch_views
        self.skips, self.use_viewdirs = skips, use_viewdirs
        self.pts_linears = nn.ModuleList(
            [nn.Linear(input_ch, W)] + [nn.Linear(W, W) if i not in skips else nn.Linear(W + input_ch, W)
                                        for i in range(D - 1)])
        self.views_linears = nn.ModuleList([nn.Linear(input_ch_views + W, W // 2)])
        if use_viewdirs:
            self.feature_linear = nn.Linear(W, W)
            self.alpha_linear = nn.Linear(W, 1)
            self.rgb_linear = nn.Linear(W // 2, 3)
        else:
            self.output_linear = nn.Linear(W, output_ch)

    def forward(self, x):
        input_pts, input_views = torch.split(x, [self.input_ch, self.input_ch_views], dim=-1)
        h = input_pts
        for i, l in enumerate(self.pts_linears):
            h = torch.relu(l(h))
            if i in self.skips:
                h = torch.cat([input_pts, h], -1)
        if not self.use_viewdirs:
            return self.output_linear(h)
        alpha = self.alpha_linear(h)
        h = torch.cat([self.feature_linear(h), input_views], -1)
        for l in self.views_linears:
            h = torch.relu(l(h))
        return torch.cat([self.rgb_linear(h), alpha], -1)


def run_network(inputs, viewdirs, fn, embed_fn, embeddirs_fn, netchunk=1024 * 64):
    """demo7-nerf.py:38-52."""
    inputs_flat = torch.reshape(inputs, [-1, inputs.shape[-1]])
    embedded = embed_fn(inputs_flat)
    if viewdirs is not None:
        input_dirs = viewdirs[:, None].expand([*inputs.shape[:-1], viewdirs.shape[-1]])
        embedded = torch.cat([embedded, embeddirs_fn(torch.reshape(input_dirs, [-1, input_dirs.shape[-1]]))], -1)
    outputs_flat = torch.cat([fn(embedded[i:i + netchunk]) for i in range(0, embedded.shape[0], netchunk)], 0)
    return torch.reshape(outputs_flat, list(inputs.shape[:-1]) + [outputs_flat.shape[-1]])


def create_nerf(args, device):
    """demo7-nerf.py:94-182 without checkpoints: (render_kwargs_train, render_kwargs_test, grad_vars, optimizer)."""
    embed_fn, input_ch = get_embedder(args.multires, args.i_embed)
    embeddirs_fn, input_ch_views = get_embedder(args.multires_views, args.i_embed) if args.use_viewdirs else (None, 0)
    output_ch = 5 if args.N_importance > 0 else 4
    model = NeRF(args.netdepth, args.netwidth, input_ch, input_ch_views, output_ch, [4], args.use_viewdirs).to(device)
    grad_vars = list(model.parameters())
    model_fine = None
    if args.N_importance > 0:
        model_fine = NeRF(args.netdepth_fine, args.netwidth_fine, input_ch, input_ch_views, output_ch, [4],
                          args.use_viewdirs).to(device)
        grad_vars += list(model_fine.parameters())
    query = lambda inputs, viewdirs, network_fn: run_network(inputs, viewdirs, network_fn, embed_fn, embeddirs_fn,
                                                             args.netchunk)
    optimizer = torch.optim.Adam(params=grad_vars, lr=args.lrate, betas=(0.9, 0.999))
    train_kw = dict(network_query_fn=query, perturb=args.perturb, N_importance=args.N_importance, network_fine=model_fine,
                    N_samples=args.N_samples, network_fn=model, use_viewdirs=args.use_viewdirs,
                    white_bkgd=args.white_bkgd, raw_noise_std=args.raw_noise_std, ndc=False, lindisp=args.lindisp)
    test_kw = dict(train_kw, perturb=0., raw_noise_std=0.)
    return train_kw, test_kw, grad_vars, optimizer


# ---- synthetic dataset ---------------------------------------------------------------------------------------------

def spot_obj(directory):
    """Unpacks the spot cow next to its .mtl and texture, as the loader expects it."""
    with lzma.open(os.path.join(GOLDEN, "spot_triangulated.obj.xz"), "rb") as f:
        data = f.read()
    with open(os.path.join(directory, "spot_triangulated.obj"), "wb") as f:
        f.write(data)
    with open(os.path.join(directory, "spot_triangulated.mtl"), "w") as f:
        f.write("newmtl material_1\nmap_Kd spot_texture.png\n")
    shutil.copyfile(os.path.join(GOLDEN, "spot_texture.png"), os.path.join(directory, "spot_texture.png"))
    return os.path.join(directory, "spot_triangulated.obj")


def camera(eye, size, viewing_angle=30.):
    """jr's look_at + perspective camera at `eye` (looking at the origin, y up) as jrender_vol's pinhole: (c2w [3, 4],
    focal, intrinsic [3, 3]).  jr's camera frame has x right, y up, z forward and its NDC x = X / (Z tan(angle)); the
    pinhole's pixel (i, j) looks along (-(i + .5 - W/2) / f, -(j + .5 - H/2) / f, 1) through the intrinsic, so with
    f = W / (2 tan(angle)) the pinhole frame is jr's with x negated, and row 0 is the top (NDC y = +1)."""
    eye = np.asarray(eye, np.float64)
    z = -eye / np.linalg.norm(eye)
    x = np.cross([0., 1., 0.], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    y /= np.linalg.norm(y)
    focal = size / (2. * math.tan(math.radians(viewing_angle)))
    c2w = np.concatenate([np.stack([-x, y, z], 1), eye[:, None]], 1).astype(np.float32)
    K = np.array([[-1. / focal, 0., size / (2. * focal)], [0., -1. / focal, size / (2. * focal)], [0., 0., 1.]],
                 np.float32)
    return c2w, focal, K


def make_dataset(size, n_views, device, distance=2.732):
    """Views of the spot cow over white on a ring of cameras at two elevations: (images [V, H, W, 3], poses [V, 3, 4],
    focal, intrinsic [3, 3])."""
    with tempfile.TemporaryDirectory() as d:
        mesh = jr.Mesh.from_obj(spot_obj(d), load_texture=True, texture_res=5, texture_type='surface',
                                dr_type='softras').to(device)
    renderer = jr.Renderer(image_size=size, camera_mode='look_at', viewing_angle=30)
    images, poses = [], []
    for v in range(n_views):
        elevation, azimuth = (30. if v % 2 == 0 else -10.), v * 360. / n_views
        eye = jr.get_points_from_angles(distance, elevation, azimuth)
        mesh.reset_()
        renderer.transform.set_eyes_from_angles(distance, elevation, azimuth)
        with torch.no_grad():
            alpha, rgb = renderer.render_mesh(mesh, mode=None)
        images.append((rgb[0] * alpha[0] + (1. - alpha[0])).permute(1, 2, 0))
        poses.append(torch.from_numpy(camera(eye, size)[0]))
    _, focal, K = camera(eye, size)
    return torch.stack(images).contiguous(), torch.stack(poses).to(device), focal, torch.from_numpy(K).to(device)


# ---- training loop (demo7-nerf.py:503-648, no_batching) -------------------------------------------------------------

def parser():
    p = argparse.ArgumentParser()
    p.add_argument('-o', '--output-dir', type=str, default='demo7_output',
                   help='directory for the held-out renders and psnr.txt (created if missing)')
    p.add_argument('--size', type=int, default=64, help='image height = width')
    p.add_argument('--n_views', type=int, default=40)
    p.add_argument('--n_test', type=int, default=4, help='held-out views (every n_views / n_test-th)')
    p.add_argument('--N_iters', type=int, default=2000)
    p.add_argument('--netdepth', type=int, default=8)
    p.add_argument('--netwidth', type=int, default=256)
    p.add_argument('--netdepth_fine', type=int, default=8)
    p.add_argument('--netwidth_fine', type=int, default=256)
    p.add_argument('--N_rand', type=int, default=1024)
    p.add_argument('--lrate', type=float, default=5e-4)
    p.add_argument('--lrate_decay', type=int, default=500)
    p.add_argument('--chunk', type=int, default=1024 * 8)
    p.add_argument('--netchunk', type=int, default=1024 * 64)
    p.add_argument('--N_samples', type=int, default=64)
    p.add_argument('--N_importance', type=int, default=128)
    p.add_argument('--perturb', type=float, default=1.)
    p.add_argument('--no_viewdirs', dest='use_viewdirs', action='store_false')
    p.add_argument('--i_embed', type=int, default=0)
    p.add_argument('--multires', type=int, default=10)
    p.add_argument('--multires_views', type=int, default=4)
    p.add_argument('--raw_noise_std', type=float, default=0.)
    p.add_argument('--precrop_iters', type=int, default=500)
    p.add_argument('--precrop_frac', type=float, default=.5)
    p.add_argument('--no_white_bkgd', dest='white_bkgd', action='store_false')
    p.add_argument('--lindisp', action='store_true')
    p.add_argument('--near', type=float, default=1.2)
    p.add_argument('--far', type=float, default=4.2)
    p.add_argument('--i_print', type=int, default=100)
    p.add_argument('--seed', type=int, default=0)
    return p


def train(args, device, data=None, log=print):
    """Trains on the synthetic views; returns dict(losses=[...], psnr=held-out PSNR or None, renders=[...])."""
    torch.manual_seed(args.seed)
    images, poses, focal, K = data if data is not None else make_dataset(args.size, args.n_views, device)
    H = W = args.size
    step = max(1, args.n_views // max(args.n_test, 1))
    i_test = list(range(0, args.n_views, step))[:args.n_test]
    i_train = [i for i in range(args.n_views) if i not in i_test]
    train_kw, test_kw, _, optimizer = create_nerf(args, device)
    for kw in (train_kw, test_kw):
        kw.update(near=args.near, far=args.far)
    losses = []
    for i in range(args.N_iters):
        rng = np.random.default_rng(i)
        img_i = int(rng.choice(i_train))
        target = images[img_i]
        rays_o, rays_d = pinhole_get_rays(H, W, focal, poses[img_i], K)
        if i < args.precrop_iters:
            dH, dW = int(H // 2 * args.precrop_frac), int(W // 2 * args.precrop_frac)
            coords = torch.stack(torch.meshgrid(torch.linspace(H // 2 - dH, H // 2 + dH - 1, 2 * dH),
                                                torch.linspace(W // 2 - dW, W // 2 + dW - 1, 2 * dW), indexing='ij'), -1)
        else:
            coords = torch.stack(torch.meshgrid(torch.linspace(0, H - 1, H), torch.linspace(0, W - 1, W),
                                                indexing='ij'), -1)
        coords = torch.reshape(coords, [-1, 2])
        select = rng.choice(coords.shape[0], size=[min(args.N_rand, coords.shape[0])], replace=False)
        sel = coords[select].long().to(device)
        batch_rays = torch.stack([rays_o[sel[:, 0], sel[:, 1]], rays_d[sel[:, 0], sel[:, 1]]], 0)
        target_s = target[sel[:, 0], sel[:, 1]]

        rgb, disp, acc, extras = render(H, W, focal, chunk=args.chunk, rays=batch_rays, retraw=True, **train_kw)
        loss = img2mse(rgb, target_s)
        if 'rgb0' in extras:
            loss = loss + img2mse(extras['rgb0'], target_s)
        optimizer.zero_grad(set_to_none=True)
        loss.backward()
        optimizer.step()
        new_lrate = args.lrate * (0.1 ** (i / (args.lrate_decay * 1000)))
        for g in optimizer.param_groups:
            g['lr'] = new_lrate
        losses.append(loss.detach())
        if args.i_print and i % args.i_print == 0:
            log("[TRAIN] Iter: %d Loss: %.5f" % (i, loss.item()))
    losses = [float(x) for x in torch.stack(losses).cpu()] if losses else []
    renders, mses = [], []
    with torch.no_grad():
        for t in i_test:
            rgb, _, _, _ = render(H, W, focal, chunk=args.chunk, c2w=poses[t], intrinsic=K, **test_kw)
            renders.append(rgb)
            mses.append(img2mse(rgb, images[t]))
    psnr = float(mse2psnr(torch.stack(mses).mean())) if mses else None
    return dict(losses=losses, psnr=psnr, renders=renders, targets=[images[t] for t in i_test])


def main():
    args = parser().parse_args()
    dev = torch.device('cuda:0')
    os.makedirs(args.output_dir, exist_ok=True)
    t0 = time.time()
    res = train(args, dev)
    torch.cuda.synchronize()
    import cv2
    for k, (rgb, tgt) in enumerate(zip(res['renders'], res['targets'])):
        pair = np.concatenate([to8b(rgb.cpu().numpy()), to8b(tgt.cpu().numpy())], 1)
        cv2.imwrite(os.path.join(args.output_dir, 'test_%02d.png' % k), pair[:, :, ::-1])
    msg = "held-out PSNR %.2f dB over %d views after %d iterations (%.0f s, %s)" % (
        res['psnr'], len(res['renders']), args.N_iters, time.time() - t0, torch.cuda.get_device_name(dev))
    with open(os.path.join(args.output_dir, 'psnr.txt'), 'w') as f:
        f.write(msg + "\n")
    print(msg)


if __name__ == '__main__':
    main()
