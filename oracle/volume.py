"""CPU oracles of NeRF volume rendering (TEST INFRASTRUCTURE -- never a product path).

Two restatements of jrender_vol's integrator / sample_pdf / fine stage (jrender_vol/integrator/{integrator,sample}.py,
rayMarching/rayMarching.py:65-71):

  composite(), resample()    numpy float32 in the order csrc/vol_api.cu evaluates: a ray's samples in tiles of 32 lanes,
                             Hillis-Steele scans within a tile times the carry of the tiles before, per-lane partial sums
                             over the tiles closed by an xor butterfly.  Only expf / np.exp may differ (by an ulp).
  integrator_mirror(),       PyTorch, op by op as the reference writes them, in any dtype and device: the float64
  sample_pdf_mirror(),       autograd comparator of the backward kernel, and the op-by-op side of tools/time_nerf_step.py.
  fine_stage_mirror()

jt.maximum(1e-10, q) is read as std::max(1e-10, q) (q when 1e-10 < q, else the constant), so a ray with acc == 0 gets
disp = 1e10 rather than NaN, in both restatements.

Also the analytic radiance field of the volume goldens (soft sphere density, sinusoidal colour), in numpy and torch.
"""
import numpy as np
import torch

F32 = np.float32
LANES = 32


def _tiles(x, fill):
    """[..., n] -> [..., K, 32] padded with fill."""
    n = x.shape[-1]
    K = max(1, -(-n // LANES))
    pad = np.full(x.shape[:-1] + (K * LANES - n,), fill, x.dtype)
    return np.concatenate([x, pad], -1).reshape(x.shape[:-1] + (K, LANES))


def _scan(v, op):
    """Inclusive Hillis-Steele scan over the last axis (32 lanes), as __shfl_up_sync rounds do it."""
    v = v.copy()
    d = 1
    while d < LANES:
        o = v.copy()
        v[..., d:] = op(o[..., d:], o[..., :-d])
        d <<= 1
    return v


def _butterfly(v):
    """xor-shuffle sum over the last axis (32 lanes); every lane ends with the same value."""
    lanes = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def _lane_sum(x_tiles):
    """Per-lane sequential partials over the tiles ([..., K, 32]), then the butterfly."""
    p = np.zeros(x_tiles.shape[:-2] + (LANES,), F32)
    for k in range(x_tiles.shape[-2]):
        p = p + x_tiles[..., k, :]
    return _butterfly(p)


def _sigmoid(x):
    return F32(1) / (F32(1) + np.exp(-x))


def _exclusive_transmittance(t_tiles):
    """T = carry * (exclusive in-tile product), carry_{k+1} = carry_k * (inclusive product at lane 31)."""
    incl = _scan(t_tiles, np.multiply)
    excl = np.concatenate([np.ones(incl.shape[:-1] + (1,), F32), incl[..., :-1]], -1)
    T = np.empty_like(excl)
    carry = np.ones(t_tiles.shape[:-2], F32)
    for k in range(t_tiles.shape[-2]):
        T[..., k, :] = carry[..., None] * excl[..., k, :]
        carry = carry * incl[..., k, -1]
    return T


def composite(raw, z_vals, rays_d, noise=None, white_bkgd=False, trace=None):
    """integrator() in the kernel's order: raw [N, S, C >= 4], z_vals [N, S], rays_d [N, 3], noise [N, S] or None ->
    dict rgb_map [N, 3], disp_map, acc_map, weights [N, S], depth_map.  A dict `trace` receives the per-sample
    intermediates [N, S]: exp_arg (what exp is taken of), alpha, t = (1 - alpha) + 1e-10 and the transmittance T."""
    raw, z, d = (np.asarray(a, F32) for a in (raw, z_vals, rays_d))
    N, S = z.shape
    norm = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    dist = np.concatenate([z[:, 1:] - z[:, :-1], np.full((N, 1), 1e10, F32)], -1) * norm[:, None]
    x = raw[..., 3]
    if noise is not None:
        x = x + np.asarray(noise, F32)
    r = np.where(x > 0, x, F32(0))   # relu(NaN) = 0, as the kernel's x > 0 ? x : 0
    arg = -r * dist
    alpha = F32(1) - np.exp(arg)
    t = (F32(1) - alpha) + F32(1e-10)
    T = _exclusive_transmittance(_tiles(t, F32(1)))
    if trace is not None:
        trace.update(exp_arg=arg, alpha=alpha, t=t, T=T.reshape(N, -1)[:, :S])
    w = (_tiles(alpha, F32(0)) * T)
    sig = _sigmoid(raw[..., :3])
    rgb = np.stack([_lane_sum(w * _tiles(sig[..., c], F32(0))) for c in range(3)], -1)
    acc = _lane_sum(w)
    depth = _lane_sum(w * _tiles(z, F32(0)))
    with np.errstate(invalid="ignore", divide="ignore"):
        q = depth / acc
    disp = F32(1) / np.where(F32(1e-10) < q, q, F32(1e-10))
    if white_bkgd:
        rgb = rgb + (F32(1) - acc)[:, None]
    return dict(rgb_map=rgb, disp_map=disp, acc_map=acc, weights=w.reshape(N, -1)[:, :S], depth_map=depth)


def linspace01(n):
    """jt.linspace(0., 1., steps=n) as the kernel forms it: k * 1 / (n - 1) + 0."""
    if n == 1:
        return np.zeros(1, F32)
    return (np.arange(n, dtype=F32) * F32(1)) / F32(n - 1) + F32(0)


def resample(weights, n_importance, u=None, z_vals=None, bins=None, trace=None):
    """The resampler in the kernel's order.  Fine stage (z_vals [N, S], weights [N, S]): bins = mids, pdf of
    weights[:, 1:-1]; returns (z_samples [N, Ni], z_vals_fine [N, S + Ni]).  sample_pdf (bins [N, nb], weights
    [N, nb - 1]): returns (z_samples, None).  u [N, Ni] or None (det).  A dict `trace` receives cdf [N, nb], and per
    sample [N, Ni] u, the searchsorted count inds and the denominator before the 1e-5 test."""
    w = np.asarray(weights, F32)
    if z_vals is not None:
        z = np.asarray(z_vals, F32)
        bins = F32(.5) * (z[:, 1:] + z[:, :-1])
        w = w[:, 1:-1]
    bins = np.asarray(bins, F32)
    N, nb = bins.shape
    wp = w + F32(1e-5)
    wsum = _lane_sum(_tiles(wp, F32(0))) if wp.shape[1] else np.zeros(N, F32)
    pdf = _tiles(wp / wsum[:, None], F32(0))
    incl = _scan(pdf, np.add)
    cum = np.empty_like(incl)
    carry = np.zeros(N, F32)
    for k in range(pdf.shape[1]):
        cum[:, k] = carry[:, None] + incl[:, k]
        carry = cum[:, k, -1]
    cdf = np.concatenate([np.zeros((N, 1), F32), cum.reshape(N, -1)[:, :nb - 1]], -1)
    u = np.broadcast_to(linspace01(n_importance), (N, n_importance)) if u is None else np.asarray(u, F32)
    inds = (cdf[:, None, :] <= u[:, :, None]).sum(-1)
    below = np.maximum(0, inds - 1)
    above = np.minimum(nb - 1, inds)
    g = lambda a, i: np.take_along_axis(a, i, 1)
    cdf0, cdf1, bin0, bin1 = g(cdf, below), g(cdf, above), g(bins, below), g(bins, above)
    denom = cdf1 - cdf0
    if trace is not None:
        trace.update(cdf=cdf, u=u, inds=inds, denom=denom)
    denom = np.where(denom < F32(1e-5), F32(1), denom)
    samples = bin0 + ((u - cdf0) / denom) * (bin1 - bin0)
    if z_vals is None:
        return samples, None
    return samples, np.sort(np.concatenate([z, samples], -1), -1)


# ---- op-by-op PyTorch mirror of the reference ---------------------------------------------------------------------

def kernel_relu(x):
    """relu as the kernels and composite() read it, x > 0 ? x : 0: NaN gives 0 (and a zero gradient), where
    torch.relu propagates it.  Which of the two Jittor's relu is has not been confirmed (DESIGN.md section 9)."""
    return torch.where(x > 0, x, torch.zeros_like(x))


def integrator_mirror(raw, z_vals, rays_d, noise=None, white_bkgd=False, relu=torch.relu):
    """integrator.py:18-39 op by op; noise is the already scaled gauss draw (or None).  Returns the five outputs.
    relu=kernel_relu gives the kernels' reading of relu(NaN)."""
    dists = z_vals[..., 1:] - z_vals[..., :-1]
    dists = torch.cat([dists, torch.full_like(dists[..., :1], 1e10)], -1)
    dists = dists * torch.norm(rays_d.unsqueeze(-2), p=2, dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    sigma = raw[..., 3] if noise is None else raw[..., 3] + noise
    alpha = 1. - torch.exp(-relu(sigma) * dists)
    ones = torch.ones(alpha.shape[0], 1, dtype=alpha.dtype, device=alpha.device)
    weights = alpha * torch.cumprod(torch.cat([ones, 1. - alpha + 1e-10], -1), -1)[:, :-1]
    rgb_map = torch.sum(weights.unsqueeze(-1) * rgb, -2)
    depth_map = torch.sum(weights * z_vals, -1)
    q = depth_map / torch.sum(weights, -1)
    disp_map = 1. / torch.where(1e-10 < q, q, torch.full_like(q, 1e-10))   # std::max(1e-10, q)
    acc_map = torch.sum(weights, -1)
    if white_bkgd:
        rgb_map = rgb_map + (1. - acc_map.unsqueeze(-1))
    return rgb_map, disp_map, acc_map, weights, depth_map


def sample_pdf_mirror(bins, weights, N_samples, det=False, u=None):
    """sample.py:28-57 op by op; u [N, N_samples] replaces jt.random when det is False."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    if det:
        n = N_samples
        u = torch.arange(n, dtype=bins.dtype, device=bins.device) * 1. / max(n - 1, 1) + 0.
        u = u.expand(list(cdf.shape[:-1]) + [n])
    inds = torch.searchsorted(cdf.contiguous(), u.contiguous(), right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    inds_g = torch.stack([below, above], -1)
    matched_shape = [inds_g.shape[0], inds_g.shape[1], cdf.shape[-1]]
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(matched_shape), 2, inds_g)
    bins_g = torch.gather(bins.unsqueeze(1).expand(matched_shape), 2, inds_g)
    denom = cdf_g[..., 1] - cdf_g[..., 0]
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_g[..., 0]) / denom
    return bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])


def fine_stage_mirror(z_vals, weights, N_importance, u=None):
    """rayMarching.py:67-71: (z_samples, sorted z_vals of the concat); det when u is None."""
    mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
    z_samples = sample_pdf_mirror(mids, weights[..., 1:-1], N_importance, det=u is None, u=u).detach()
    z_fine, _ = torch.sort(torch.cat([z_vals, z_samples], -1), -1)
    return z_samples, z_fine


# ---- the analytic radiance field of the goldens -------------------------------------------------------------------

def field_np(pts, viewdirs=None, channels=4):
    """pts [..., 3] -> raw [..., channels]: density 8 (0.6 - |p|), colour logits sin(3 p + phase) (+ 0.5 viewdir)."""
    p = np.asarray(pts, F32)
    r = np.sqrt(p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1] + p[..., 2] * p[..., 2])
    sigma = F32(8) * (F32(.6) - r)
    col = np.sin(F32(3) * p + np.array([0, 1, 2], F32))
    if viewdirs is not None:
        col = col + F32(.5) * np.broadcast_to(np.asarray(viewdirs, F32)[:, None, :], col.shape)
    out = [col, sigma[..., None]] + [np.zeros_like(sigma[..., None])] * (channels - 4)
    return np.concatenate(out, -1).astype(F32)


def field_torch(pts, viewdirs=None, channels=4):
    """field_np in torch (same float32 expressions)."""
    r = torch.sqrt(pts[..., 0] * pts[..., 0] + pts[..., 1] * pts[..., 1] + pts[..., 2] * pts[..., 2])
    sigma = 8. * (.6 - r)
    col = torch.sin(3. * pts + torch.arange(3, dtype=pts.dtype, device=pts.device))   # no host copy: graph-capturable
    if viewdirs is not None:
        col = col + .5 * viewdirs[:, None, :].expand(col.shape)
    out = [col, sigma[..., None]] + [torch.zeros_like(sigma[..., None])] * (channels - 4)
    return torch.cat(out, -1)
