"""NeRF volume rendering kernels (csrc/vol_api.cu) through jrender_b200.vol on the GPU: the compositing forward against
the float32 oracle, its backward against float64 autograd of the op-by-op mirror, the resampler, the reference's
end-to-end goldens, determinism, CUDA-graph capture, launch accounting and argument errors."""
import numpy as np
import pytest
import torch

from jrender_b200 import _lib
from jrender_b200 import vol
from oracle import volume as ov
from tests import test_vol_cpu as hv
from tests.test_launch_gpu import profiled

pytestmark = pytest.mark.gpu

OUTS = ("rgb_map", "disp_map", "acc_map", "weights", "depth_map")


def scene(N, S, C=4, seed=0, near=2., far=6., empty_and_opaque=True):
    rng = np.random.default_rng(seed)
    z = np.sort(rng.uniform(near, far, (N, S)).astype(np.float32), -1)
    raw = rng.normal(0, 2, (N, S, C)).astype(np.float32)
    d = rng.normal(0, 1, (N, 3)).astype(np.float32)
    if empty_and_opaque and N > 2 and S > 2:
        raw[0, :, 3] = -np.abs(raw[0, :, 3])
        raw[1, S // 2, 3] = 1e4
    return raw, z, d


def cu(*a):
    return [None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def check_forward(got, ref):
    for k, g in zip(OUTS, got):
        g, r = g.cpu().numpy(), ref[k]
        if k in ("depth_map", "disp_map"):
            assert np.all(np.abs(g - r) <= 4e-6 * np.abs(r)), (k, np.abs(g - r).max())
        else:
            assert np.abs(g - r).max() <= 4e-6, (k, np.abs(g - r).max())


@pytest.mark.parametrize("N,S,C,noise,white", [(37, 64, 4, 0., False), (37, 192, 5, 1., True), (9, 1, 4, 0., False),
                                               (5, 33, 4, .5, False), (3, 1024, 4, 0., True), (1000, 96, 4, 0., False)])
def test_composite_forward_matches_oracle(cuda_device, N, S, C, noise, white):
    raw, z, d = scene(N, S, C, seed=S)
    nz = np.random.default_rng(1).normal(0, noise, (N, S)).astype(np.float32) if noise else None
    got = vol._composite(*cu(raw, z, d, nz), white)
    ref = ov.composite(raw, z, d, nz, white)
    check_forward(got, ref)
    if S > 2 and not noise:
        assert got[1][0].item() == np.float32(1e10) and got[2][0].item() == 0   # empty ray: disp = 1e10, not NaN


@pytest.mark.parametrize("name", [n for n in hv.case_names("integrator")])
def test_integrator_reproduces_golden(cuda_device, name, monkeypatch):
    a = hv.META[name]["args"]
    monkeypatch.setattr(vol, "_random", hv.Replay(name, cuda_device))
    raw, z, d = cu(hv.inp(name, "raw"), hv.inp(name, "z_vals"), hv.inp(name, "rays_d"))
    got = vol.integrator(raw, z, d, a["raw_noise_std"], a["white_bkgd"])
    if name == "int_s1":   # the reference degenerates at S = 1 (test_vol_cpu); the kernel matches the oracle there
        check_forward(got, ov.composite(hv.inp(name, "raw"), hv.inp(name, "z_vals"), hv.inp(name, "rays_d")))
        return
    for k, g in zip(OUTS, got):
        hv.close(g.cpu().numpy(), hv.out(name, k))
    if name == "int_plain":
        assert got[1][0].item() == np.float32(1e10)


GRADS = ["rgb_map", "disp_map", "acc_map", "weights", "depth_map", "all"]


@pytest.mark.parametrize("which", GRADS)
@pytest.mark.parametrize("N,S,C,noise,white", [(37, 40, 4, 0., False), (6, 70, 5, .5, True), (11, 1, 4, 0., True),
                                               (4, 300, 4, 0., False)])
def test_composite_backward_matches_float64_autograd(cuda_device, which, N, S, C, noise, white):
    raw, z, d = scene(N, S, C, seed=3 * S + C)
    nz = np.random.default_rng(2).normal(0, noise, (N, S)).astype(np.float32) if noise else None
    rng = np.random.default_rng(5)
    ups = {k: rng.normal(0, 1, s).astype(np.float32) for k, s in
           zip(OUTS, ((N, 3), (N,), (N,), (N, S), (N,)))}
    ups["disp_map"] *= np.float32(1e-2)   # disp is up to 1e10 on empty rays: keep its term comparable
    use = OUTS if which == "all" else (which,)

    r32 = cu(raw)[0].requires_grad_(True)
    zc, dc, nc = cu(z, d, nz)
    outs = vol._composite(r32, zc, dc, nc, white)
    loss = sum((o * cu(ups[k])[0]).sum() for k, o in zip(OUTS, outs) if k in use)
    g32, = torch.autograd.grad(loss, r32)

    def mirror_grad(dtype):
        t = lambda a: None if a is None else torch.from_numpy(a).to(dtype)
        r, zz, nn_ = t(raw).requires_grad_(True), t(z), t(nz)
        if S == 1:   # the reference's dists are empty at S = 1; a second, empty sample 1e10 behind gives the kernel's
            r = torch.cat([r, torch.full_like(r, -1.)], 1)          # single 1e10 * |d| interval
            zz = torch.cat([zz, zz + 1e10], 1)
            nn_ = None if nn_ is None else torch.cat([nn_, torch.zeros_like(nn_)], 1)
        outs = ov.integrator_mirror(r, zz, t(d), nn_, white)
        loss = sum((o[:, :S] if k == "weights" else o).mul(t(ups[k])).sum() for k, o in zip(OUTS, outs) if k in use)
        g, = torch.autograd.grad(loss, r)
        return g[:, :S].numpy().astype(np.float64)
    g64 = mirror_grad(torch.float64)
    assert np.all(np.isfinite(g64))
    g = g32.cpu().numpy()
    assert np.all(np.isfinite(g))
    scale = np.abs(g64).max()
    # Where the true gradient is far below the upstream gradients (acc alone on saturated rays: dL/da_i is the
    # difference of two O(|g_acc|) terms), float32 resolves it only to ~eps32 |g_acc|; the reference's own float32
    # autograd has the same floor, so the kernel must then be within 4x of that op-by-op float32 error.
    floor = 4 * np.abs(mirror_grad(torch.float32) - g64).max()
    assert np.abs(g - g64).max() <= max(1e-5 * scale, floor) + 1e-30, (np.abs(g - g64).max(), scale, floor)
    if C > 4:
        assert np.all(g[..., 4:] == 0)


def test_opaque_sample_leaves_gradients_in_front_finite(cuda_device):
    """A sample with alpha == 1 in float32 mid-ray: the gradient of the samples in front of it is the float64 one."""
    raw, z, d = scene(4, 64, seed=9)
    raw[2, 10, 3] = 1e6
    r = cu(raw)[0].requires_grad_(True)
    rgb = vol._composite(r, *cu(z, d), None, False)[0]
    g, = torch.autograd.grad(rgb.sum(), r)
    r64 = torch.from_numpy(raw).double().requires_grad_(True)
    g64, = torch.autograd.grad(ov.integrator_mirror(r64, *[torch.from_numpy(a).double() for a in (z, d)])[0].sum(), r64)
    g, g64 = g.cpu().numpy()[2, :11], g64.numpy()[2, :11]
    assert np.all(np.isfinite(g)) and np.abs(g - g64).max() <= 1e-5 * np.abs(g64).max()


@pytest.mark.parametrize("N,S,Ni,det", [(37, 64, 128, True), (37, 64, 128, False), (100, 2, 5, True), (9, 17, 1, False),
                                        (3, 500, 524, False), (4, 1000, 24, True)])
def test_resample_matches_oracle_and_sorts(cuda_device, N, S, Ni, det):
    near, far = 2., 6.
    raw, z, d = scene(N, S, seed=S + Ni, near=near, far=far)
    zc, dc = cu(z, d)
    w = vol._composite(cu(raw)[0], zc, dc, None, False)[3]
    u = None if det else torch.rand(N, Ni, device=cuda_device)
    zs, zf = vol._resample(zc, w, Ni, u)
    ref, _ = ov.resample(w.cpu().numpy(), Ni, None if u is None else u.cpu().numpy(), z_vals=z)
    assert np.abs(zs.cpu().numpy() - ref).max() <= 1e-6 * (far - near)
    want, _ = torch.sort(torch.cat([zc, zs], -1), -1)
    assert torch.equal(zf, want)


@pytest.mark.parametrize("name", hv.case_names("sample_pdf"))
def test_sample_pdf_reproduces_golden(cuda_device, name, monkeypatch):
    a = hv.META[name]["args"]
    monkeypatch.setattr(vol, "_random", hv.Replay(name, cuda_device))
    bins, w = cu(hv.inp(name, "bins"), hv.inp(name, "weights"))
    got = vol.sample_pdf(bins, w, a["N_samples"], a["det"]).cpu().numpy()
    b = hv.inp(name, "bins")
    u = hv.G[name + "_draw0"] if hv.META[name]["draws"] else None
    ref, _ = ov.resample(hv.inp(name, "weights"), a["N_samples"], u, bins=b)
    assert np.abs(got - ref).max() <= 1e-6 * (b.max() - b.min())
    assert np.abs(got - hv.out(name, "samples")).max() <= 1e-6 * (b.max() - b.min())


@pytest.mark.parametrize("name", hv.case_names("render"))
def test_render_reproduces_golden(cuda_device, name, monkeypatch):
    run, replay = hv.render_case(name, cuda_device)
    monkeypatch.setattr(vol, "_random", replay)
    rgb, disp, acc, extras = run()
    assert replay.done()
    hv.check_render(name, rgb, disp, acc, extras, rel=2e-5)


def field_query(pts, viewdirs, fn):
    return ov.field_torch(pts, viewdirs, 4)


def ray_batch(N, device, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    o = torch.tensor([0.05, -0.1, -2.2]).expand(N, 3) + 0.05 * torch.randn(N, 3, generator=g)
    dvec = torch.cat([0.2 * torch.randn(N, 2, generator=g), torch.ones(N, 1)], -1)
    vd = dvec / dvec.norm(dim=-1, keepdim=True)
    return torch.cat([o, dvec, torch.full((N, 1), 1.), torch.full((N, 1), 3.4), vd], -1).to(device)


def test_render_rays_is_deterministic(cuda_device):
    rays = ray_batch(333, cuda_device)
    res = []
    for _ in range(2):
        torch.manual_seed(4)
        res.append(vol.render_rays(rays, None, field_query, 64, perturb=1., N_importance=128, raw_noise_std=1.,
                                   white_bkgd=True, retraw=True))
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k


def test_render_rays_captures_in_a_cuda_graph(cuda_device):
    rays = ray_batch(1000, cuda_device, seed=1)
    kw = dict(network_fn=None, network_query_fn=field_query, N_samples=64, perturb=0., N_importance=128)
    eager = vol.render_rays(rays, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        vol.render_rays(rays, **kw)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = vol.render_rays(rays, **kw)
    graph.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k


def test_render_rays_forward_backward_makes_five_launches(cuda_device):
    rays = ray_batch(500, cuda_device, seed=2)
    net = torch.nn.Linear(3, 5).to(cuda_device)
    query = lambda pts, viewdirs, fn: fn(pts)

    def step(dev):
        ret = vol.render_rays(rays, net, query, 64, perturb=1., N_importance=128)
        (ret["rgb_map"].sum() + ret["rgb0"].sum()).backward()
    L = _lib.lib()
    step(cuda_device)
    delta, counts = profiled(L, step, cuda_device)
    assert delta == 5 == sum(counts), (delta, counts)
    assert (counts[22], counts[24], counts[23]) == (2, 1, 2), counts


def test_argument_errors_are_loud(cuda_device):
    raw, z, d = cu(*scene(4, 16))
    with pytest.raises(_lib.B200RasterError, match="CUDA float32"):
        vol.integrator(raw.double(), z, d)
    with pytest.raises(_lib.B200RasterError, match="CUDA float32"):
        vol.integrator(raw.cpu(), z.cpu(), d.cpu())
    with pytest.raises(ValueError, match="z_vals requires grad"):
        vol.integrator(raw, z.clone().requires_grad_(True), d)
    with pytest.raises(ValueError, match="rays_d requires grad"):
        vol.integrator(raw, z, d.clone().requires_grad_(True))
    with pytest.raises(ValueError):
        vol.integrator(raw[..., :3], z, d)
    big = cu(*scene(2, 1025, empty_and_opaque=False))
    with pytest.raises(_lib.B200RasterError, match="1025 samples per ray > 1024"):
        vol.integrator(*big)
    w = torch.rand(2, 1000, device=cuda_device)
    with pytest.raises(_lib.B200RasterError, match="1000 \\+ 25 samples per ray > 1024"):
        vol._resample(torch.sort(torch.rand(2, 1000, device=cuda_device) * 4 + 2)[0], w, 25, None)
    with pytest.raises(_lib.B200RasterError, match="no bins"):
        vol._resample(z[:, :1].contiguous(), z[:, :1].contiguous(), 8, None)


def test_zero_rays_is_a_no_op(cuda_device):
    raw, z, d = cu(*scene(3, 16))
    outs = vol._composite(raw[:0], z[:0], d[:0], None, False)
    assert [tuple(o.shape) for o in outs] == [(0, 3), (0,), (0,), (0, 16), (0,)]
    zs, zf = vol._resample(z[:0], z[:0], 8, None)
    assert zs.shape == (0, 8) and zf.shape == (0, 24)
    ret = vol.render_rays(ray_batch(0, cuda_device), None, field_query, 16, N_importance=8)
    assert ret["rgb_map"].shape == (0, 3)
