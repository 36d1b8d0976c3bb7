"""NeRF volume rendering: the reference's jrender_vol package (camera, integrator, rayMarching, renderPass) on the sm_90a
kernels of csrc/vol_api.cu.  A script ports by changing `from jrender_vol.renderPass import render` /
`from jrender_vol.camera import *` to `from jrender_b200.vol import ...`; the names are deliberately not exported from
the top-level package, as the reference keeps jrender_vol separate from jrender.

    integrator()   one fused launch forward (b200r_vol_composite_forward), one backward (b200r_vol_composite_backward)
    sample_pdf()   b200r_vol_resample on explicit bins
    render_rays()  coarse integrator, one b200r_vol_resample for mids + sample_pdf + the sorted merge, fine integrator

Rays, sampling and reshapes are PyTorch.  Every random number (perturb, sample_pdf with det=False, raw_noise_std) is
drawn by _random() from PyTorch's current generator.  Nothing here synchronises with the host, so render_rays with
perturb=0 can be captured in a CUDA graph.  The kernels take CUDA float32 tensors only; there is no CPU fallback.
Gradients flow to the network output `raw` only: z_vals and rays_d must not require grad (in the reference they never
do -- coarse z_vals are constants and fine samples are detached), and a call where they do raises.
"""
import torch

from . import _lib


def _random(shape, device, normal=False):
    """Uniform [0, 1) (jt.random) or standard normal (jt.init.gauss) float32 draws of `shape` from PyTorch's current
    generator: the only source of randomness in this module."""
    if normal:
        return torch.randn(shape, device=device, dtype=torch.float32)
    return torch.rand(shape, device=device, dtype=torch.float32)


def _check(name, **tensors):
    for k, t in tensors.items():
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            raise _lib.B200RasterError("%s: %s must be a CUDA float32 tensor (the kernels have no CPU fallback), got %s"
                                       % (name, k, t.dtype if isinstance(t, torch.Tensor) else type(t).__name__))


def _no_grad_input(name, **tensors):
    for k, t in tensors.items():
        if t is not None and t.requires_grad:
            raise ValueError("%s: %s requires grad, but the volume kernels differentiate with respect to raw only; "
                             "detach it (the reference never differentiates it)" % (name, k))


def _nullable(g):
    return None if g is None else g.contiguous()


class _Composite(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, noise, white_bkgd):
        N, S, C = raw.shape
        dev = raw.device
        rgb = torch.empty(N, 3, device=dev)
        disp, acc, depth = (torch.empty(N, device=dev) for _ in range(3))
        weights = torch.empty(N, S, device=dev)
        _lib.call("b200r_vol_composite_forward", dev, raw, z_vals, rays_d, noise, rgb, disp, acc, weights, depth, N, S, C,
                  int(white_bkgd))
        ctx.save_for_backward(raw, z_vals, rays_d, noise, acc, depth)
        ctx.white_bkgd = white_bkgd
        ctx.set_materialize_grads(False)
        return rgb, disp, acc, weights, depth

    @staticmethod
    def backward(ctx, g_rgb, g_disp, g_acc, g_weights, g_depth):
        raw, z_vals, rays_d, noise, acc, depth = ctx.saved_tensors
        N, S, C = raw.shape
        grad_raw = torch.empty_like(raw)
        if all(g is None for g in (g_rgb, g_disp, g_acc, g_weights, g_depth)):
            return grad_raw.zero_(), None, None, None, None
        _lib.call("b200r_vol_composite_backward", raw.device, raw, z_vals, rays_d, noise, acc, depth, _nullable(g_rgb),
                  _nullable(g_disp), _nullable(g_acc), _nullable(g_weights), _nullable(g_depth), grad_raw, N, S, C,
                  int(ctx.white_bkgd))
        return grad_raw, None, None, None, None


def _composite(raw, z_vals, rays_d, noise, white_bkgd):
    """The fused compositing of integrator(): (rgb_map, disp_map, acc_map, weights, depth_map)."""
    _check("integrator", raw=raw, z_vals=z_vals, rays_d=rays_d, noise=noise)
    return _Composite.apply(raw.contiguous(), z_vals.contiguous(), rays_d.contiguous(),
                            None if noise is None else noise.contiguous(), bool(white_bkgd))


def _resample(z_vals, weights, N_importance, u):
    """rayMarching.py:67-71 in one launch: (z_samples [N, Ni], z_vals_fine [N, S + Ni] sorted); u None = det."""
    _check("render_rays", z_vals=z_vals, weights=weights, u=u)
    N, S = z_vals.shape
    z_samples = torch.empty(N, N_importance, device=z_vals.device)
    z_fine = torch.empty(N, S + N_importance, device=z_vals.device)
    _lib.call("b200r_vol_resample", z_vals.device, z_vals.detach().contiguous(), None, weights.detach().contiguous(),
              None if u is None else u.contiguous(), z_samples, z_fine, N, S, int(N_importance))
    return z_samples, z_fine


def integrator(raw, z_vals, rays_d, raw_noise_std=0, white_bkgd=False):
    """integrator.py:5-39: raw [N, S, C >= 4] network output, z_vals [N, S], rays_d [N, 3] -> rgb_map [N, 3], disp_map
    [N], acc_map [N], weights [N, S], depth_map [N].  Differentiable with respect to raw (all five outputs, weights
    included).  With raw_noise_std > 0 the density is perturbed by _random normal draws times raw_noise_std."""
    _no_grad_input("integrator", z_vals=z_vals, rays_d=rays_d)
    if raw.dim() != 3 or raw.shape[2] < 4 or tuple(z_vals.shape) != tuple(raw.shape[:2]) or \
            tuple(rays_d.shape) != (raw.shape[0], 3):
        raise ValueError("integrator: need raw [N, S, C >= 4], z_vals [N, S], rays_d [N, 3]; got %s, %s, %s"
                         % (tuple(raw.shape), tuple(z_vals.shape), tuple(rays_d.shape)))
    noise = None
    if raw_noise_std > 0.:
        noise = _random(tuple(raw.shape[:2]), raw.device, normal=True) * raw_noise_std
    return _composite(raw, z_vals, rays_d, noise, white_bkgd)


def sample(N_rays, N_samples, lindisp, perturb, near, far):
    """sample.py:6-24: [N_rays, N_samples] depths from near to far (linear in depth, or in disparity with lindisp),
    stratified within their intervals when perturb > 0 (uniform _random draws)."""
    like = near if isinstance(near, torch.Tensor) else far
    dev = like.device if isinstance(like, torch.Tensor) else None
    n = N_samples
    t_vals = torch.arange(n, dtype=torch.float32, device=dev) * 1. / (n - 1) + 0. if n > 1 else \
        torch.zeros(1, device=dev)
    if not lindisp:
        z_vals = near * (1. - t_vals) + far * t_vals
    else:
        z_vals = 1. / (1. / near * (1. - t_vals) + 1. / far * t_vals)
    z_vals = z_vals.expand([N_rays, N_samples])
    if perturb > 0.:
        mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
        upper = torch.cat([mids, z_vals[..., -1:]], -1)
        lower = torch.cat([z_vals[..., :1], mids], -1)
        t_rand = _random(tuple(z_vals.shape), z_vals.device)
        z_vals = lower + (upper - lower) * t_rand
    return z_vals


def sample_pdf(bins, weights, N_samples, det=False):
    """sample.py:28-57: N_samples depths per row drawn from the piecewise-constant pdf of weights [N, nb - 1] over bins
    [N, nb], by inverse transform of linspace(0, 1) (det) or of uniform _random draws.  Runs b200r_vol_resample, the
    kernel of render_rays' fine stage.  The result is detached: every caller in the reference detaches it
    (rayMarching.py:69), and the kernel has no backward."""
    _check("sample_pdf", bins=bins, weights=weights)
    if bins.dim() != 2 or tuple(weights.shape) != (bins.shape[0], bins.shape[1] - 1):
        raise ValueError("sample_pdf: need bins [N, nb] and weights [N, nb - 1]; got %s, %s"
                         % (tuple(bins.shape), tuple(weights.shape)))
    N, nb = bins.shape
    u = None if det else _random((N, int(N_samples)), bins.device)
    out = torch.empty(N, int(N_samples), device=bins.device)
    _lib.call("b200r_vol_resample", bins.device, None, bins.detach().contiguous(), weights.detach().contiguous(), u, out,
              None, N, nb, int(N_samples))
    return out


def render_rays(ray_batch, network_fn, network_query_fn, N_samples, retraw=False, lindisp=False, perturb=0.,
                N_importance=0, network_fine=None, white_bkgd=False, raw_noise_std=0., verbose=False, **kwargs):
    """rayMarching.py:6-88: ray_batch [N, 8 (+3 viewdirs)] = origin, direction, near, far (, viewdir) -> dict rgb_map,
    disp_map, acc_map (+ raw with retraw; + rgb0, disp0, acc0 of the coarse pass with N_importance > 0).  The fine
    samples come from one b200r_vol_resample launch on the coarse weights (det when perturb == 0)."""
    rays_o, rays_d = ray_batch[:, 0:3], ray_batch[:, 3:6]
    _no_grad_input("render_rays", rays_d=rays_d)
    viewdirs = ray_batch[:, -3:] if ray_batch.shape[-1] > 8 else None
    bounds = torch.reshape(ray_batch[..., 6:8], [-1, 1, 2])
    near, far = bounds[..., 0], bounds[..., 1]
    N_rays = ray_batch.shape[0]

    z_vals = sample(N_rays, N_samples, lindisp, perturb, near, far)
    pts = rays_o.unsqueeze(-2) + rays_d.unsqueeze(-2) * z_vals.unsqueeze(-1)
    if kwargs.get('embed_depth', False):
        pts = torch.cat([pts, z_vals.unsqueeze(-1)], dim=-1)
    raw = network_query_fn(pts, viewdirs, network_fn)
    rgb_map, disp_map, acc_map, weights, depth_map = integrator(raw, z_vals, rays_d, raw_noise_std, white_bkgd)

    rgb_map_0, disp_map_0, acc_map_0 = rgb_map, disp_map, acc_map
    if N_importance > 0:
        u = None if perturb == 0. else _random((N_rays, int(N_importance)), z_vals.device)
        _, z_vals = _resample(z_vals, weights, int(N_importance), u)
        pts = rays_o.unsqueeze(-2) + rays_d.unsqueeze(-2) * z_vals.unsqueeze(-1)
        if kwargs.get('embed_depth', False):
            pts = torch.cat([pts, z_vals.unsqueeze(-1)], dim=-1)
        run_fn = network_fn if network_fine is None else network_fine
        raw = network_query_fn(pts, viewdirs, run_fn)
        rgb_map, disp_map, acc_map, weights, depth_map = integrator(raw, z_vals, rays_d, raw_noise_std, white_bkgd)

    ret = {'rgb_map': rgb_map, 'disp_map': disp_map, 'acc_map': acc_map}
    if retraw:
        ret['raw'] = raw
    if N_importance > 0:
        ret['rgb0'] = rgb_map_0
        ret['disp0'] = disp_map_0
        ret['acc0'] = acc_map_0
    return ret


def batchify_rays(rays_flat, chunk=1024 * 32, **kwargs):
    """render.py:7-21: render_rays over chunks of `chunk` rays, outputs concatenated (no host synchronisation)."""
    all_ret = {}
    for i in range(0, rays_flat.shape[0], chunk):
        ret = render_rays(rays_flat[i:i + chunk], **kwargs)
        for k in ret:
            all_ret.setdefault(k, []).append(ret[k])
    return {k: torch.cat(all_ret[k], 0) for k in all_ret}


def pinhole_get_rays(H, W, focal, c2w, intrinsic=None):
    """camera/pinhole.py:6-21: (rays_o, rays_d) [H, W, 3] of a pinhole camera.  Without intrinsic pixel (i, j) looks
    along (-(i - W/2) / focal, -(j - H/2) / focal, 1) in the camera frame; with it, along intrinsic[:3, :3] @
    (i + 0.5, j + 0.5, 1).  Rotated by c2w[:3, :3], from c2w[:3, 3]."""
    dev = c2w.device
    i, j = torch.meshgrid(torch.arange(W, dtype=torch.float32, device=dev),
                          torch.arange(H, dtype=torch.float32, device=dev), indexing='ij')
    i = i.t()
    j = j.t()
    if intrinsic is None:
        dirs = torch.stack([-(i - W * .5) / focal, -(j - H * .5) / focal, torch.ones_like(i)], -1).unsqueeze(-2)
    else:
        i = i + 0.5
        j = j + 0.5
        dirs = torch.stack([i, j, torch.ones_like(i)], -1).unsqueeze(-2)
        dirs = torch.sum(dirs * intrinsic[:3, :3], -1).unsqueeze(-2)
    rays_d = torch.sum(dirs * c2w[:3, :3], -1)
    rays_o = c2w[:3, -1].expand(rays_d.shape)
    return rays_o, rays_d


def ndc_rays(H, W, focal, near, rays_o, rays_d):
    """camera/pinhole.py:25-42: rays shifted to the near plane and mapped to normalised device coordinates."""
    t = -(near + rays_o[..., 2]) / rays_d[..., 2]
    rays_o = rays_o + t.unsqueeze(-1) * rays_d
    o0 = -1. / (W / (2. * focal)) * rays_o[..., 0] / rays_o[..., 2]
    o1 = -1. / (H / (2. * focal)) * rays_o[..., 1] / rays_o[..., 2]
    o2 = 1. + 2. * near / rays_o[..., 2]
    d0 = -1. / (W / (2. * focal)) * (rays_d[..., 0] / rays_d[..., 2] - rays_o[..., 0] / rays_o[..., 2])
    d1 = -1. / (H / (2. * focal)) * (rays_d[..., 1] / rays_d[..., 2] - rays_o[..., 1] / rays_o[..., 2])
    d2 = -2. * near / rays_o[..., 2]
    return torch.stack([o0, o1, o2], -1), torch.stack([d0, d1, d2], -1)


def render(H, W, focal, chunk=1024 * 32, rays=None, c2w=None, intrinsic=None, ndc=True, near=0., far=1.,
           use_viewdirs=False, c2w_staticcam=None, **kwargs):
    """render.py:24-89: renders a whole image (c2w [3, 4]) or a ray batch (rays = (rays_o, rays_d), each [..., 3]) in
    chunks of `chunk` rays; returns [rgb_map, disp_map, acc_map, extras], each shaped like the rays (extras holds the
    remaining render_rays outputs).  kwargs go to render_rays."""
    if c2w is not None:
        rays_o, rays_d = pinhole_get_rays(H, W, focal, c2w, intrinsic)
    else:
        rays_o, rays_d = rays
    if use_viewdirs:
        viewdirs = rays_d
        if c2w_staticcam is not None:
            assert intrinsic is None
            rays_o, rays_d = pinhole_get_rays(H, W, focal, c2w_staticcam)
        viewdirs = viewdirs / torch.norm(viewdirs, p=2, dim=-1, keepdim=True)
        viewdirs = torch.reshape(viewdirs, [-1, 3]).float()
    sh = rays_d.shape
    if ndc:
        rays_o, rays_d = ndc_rays(H, W, focal, 1., rays_o, rays_d)
    rays_o = torch.reshape(rays_o, [-1, 3]).float()
    rays_d = torch.reshape(rays_d, [-1, 3]).float()
    near, far = near * torch.ones_like(rays_d[..., :1]), far * torch.ones_like(rays_d[..., :1])
    rays = torch.cat([rays_o, rays_d, near, far], -1)
    if use_viewdirs:
        rays = torch.cat([rays, viewdirs], -1)
    all_ret = batchify_rays(rays, chunk, **kwargs)
    for k in all_ret:
        all_ret[k] = torch.reshape(all_ret[k], list(sh[:-1]) + list(all_ret[k].shape[1:]))
    k_extract = ['rgb_map', 'disp_map', 'acc_map']
    ret_list = [all_ret[k] for k in k_extract]
    ret_dict = {k: all_ret[k] for k in all_ret if k not in k_extract}
    return ret_list + [ret_dict]
