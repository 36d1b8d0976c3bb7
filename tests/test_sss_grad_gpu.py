"""GPU tests of the subsurface-scattering gradients (Lighting.sss_grad): b200r_sss_blur_pyramid_backward,
b200r_sss_stretch_backward and b200r_bake_textures_softras_backward against the float64 mirror oracle/sss_grad.py, each
entry within the mirror's own per-entry bound; Lighting's SSS path with sss_grad on (forward bits, gradients against a
composite reference, central differences), its launches and errors, and a short albedo fit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib, lighting
from jrender_b200 import workloads as wl
from oracle import sss as osss
from oracle import sss_grad as sg

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
LIGHT = dict(intensity_ambient=0.45, color_ambient=[1.0, 0.95, 0.9], intensity_directionals=1.0,
             color_directionals=[0.9, 1.0, 0.8], directions=[0.65, -0.2, -1.0])
S = lighting.SSS_IMAGE_SIZE
K_SSS, K_BAKE, K_SOFTRAS_FWD, K_SOFTRAS_BWD = 25, 16, 2, 3


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)


def chw(a, dev):
    return _t(np.transpose(a, (2, 0, 1)), dev)


random_maps = wl.sss_maps   # tests/test_sss_gpu.py's map shape


def stretch(world, dev):
    H, W = world.shape[:2]
    su = torch.empty((H, W), dtype=torch.float32, device=dev)
    sv = torch.empty_like(su)
    _lib.call("b200r_sss_stretch", dev, chw(world, dev), su, sv, H, W)
    return su.cpu().numpy(), sv.cpu().numpy()


def pyramid_backward(su, sv, irr, g, dev, stretch_grads=True, nbytes=None):
    """b200r_sss_blur_pyramid_backward -> dict of numpy gradients (irradiance / specular [H, W, 3])."""
    H, W = su.shape
    taps, widths, weights, L = lighting._sss_levels()
    need = _lib.lib().b200r_sss_backward_workspace_bytes(H, W, L)
    ws = torch.empty((need if nbytes is None else nbytes,), dtype=torch.uint8, device=dev)
    gi = torch.empty((3, H, W), device=dev)
    gs = torch.empty((3, H, W), device=dev)
    gu = torch.empty((H, W), device=dev) if stretch_grads else None
    gv = torch.empty((H, W), device=dev) if stretch_grads else None
    _lib.call("b200r_sss_blur_pyramid_backward", dev, _t(su, dev), _t(sv, dev), chw(irr, dev), _t(g, dev), gi, gs, gu, gv,
              ws, ws.numel(), taps, widths, weights, L, H, W)
    out = dict(irradiance=gi.permute(1, 2, 0).cpu().numpy(), specular=gs.permute(1, 2, 0).cpu().numpy())
    if stretch_grads:
        out.update(stretch_u=gu.cpu().numpy(), stretch_v=gv.cpu().numpy())
    return out


def check_pyramid(su, sv, irr, seed, dev, stretch_grads=True):
    """Kernel against the mirror's adjoint at the float32 forward's intermediates, per entry within sg.bound; returns
    the worst |diff| / bound per gradient."""
    g = np.random.default_rng(seed).normal(size=irr.shape).astype(np.float32)
    got = pyramid_backward(su, sv, irr, g, dev, stretch_grads)
    levels = sg.walk(su, sv, irr)
    irr_t, g_t = torch.from_numpy(irr).to(dev), torch.from_numpy(g).to(dev)
    want = sg.pyramid_vjp(levels, irr_t, g_t, stretch=stretch_grads)
    mag = sg.pyramid_vjp(levels, irr_t, g_t, magnitude=True, stretch=stretch_grads)
    worst = {}
    for k in got:
        w = want[k].cpu().numpy()
        b = sg.bound(mag[k]).cpu().numpy()
        r = np.abs(got[k] - w) / b
        worst[k] = float(r.max())
        assert np.isfinite(got[k]).all(), k
        assert (r <= 1).all(), (k, worst[k], np.abs(w).max())
    return worst


def threshold_maps(n, seed):
    """Maps with neighbours at the 1e-6 replacement threshold (1e-6 is replaced, the next float up is not), zero and
    negative centres, and stretch values up to 1 so that the widest level's taps pass the edges and extrapolate."""
    rng = np.random.default_rng(seed)
    su = np.clip(rng.uniform(-0.1, 1.3, (n, n)), 0, 1).astype(np.float32)
    sv = np.clip(rng.uniform(-0.1, 1.3, (n, n)), 0, 1).astype(np.float32)
    irr = rng.uniform(0.05, 1, (n, n, 3)).astype(np.float32)
    m = rng.random((n, n, 3))
    irr[m < 0.08] = 0
    irr[(m >= 0.08) & (m < 0.12)] = np.float32(1e-6)
    irr[(m >= 0.12) & (m < 0.16)] = np.nextafter(np.float32(1e-6), np.float32(1))
    irr[(m >= 0.16) & (m < 0.18)] = -0.25
    su[rng.random((n, n)) < 0.05] = 0
    sv[rng.random((n, n)) < 0.05] = np.float32(1e-6)
    return su, sv, irr


@pytest.mark.parametrize("stretch_grads", [True, False])
def test_pyramid_backward_64(cuda_device, stretch_grads):
    su, sv, irr = threshold_maps(64, 1)
    levels = sg.walk(su, sv, irr)
    assert any((d["taps"][0][0] == d["taps"][0][1]).any() for d in [levels[2]["dsu"]])   # taps wholly past an edge
    print(check_pyramid(su, sv, irr, 2, cuda_device, stretch_grads))


def test_pyramid_backward_on_golden_maps(cuda_device):
    g = np.load(os.path.join(G, "ref_sss_gpu_blur_64x64.npz"))
    keys = sorted(k[:-6] for k in g.files if k.endswith("_image") and k.startswith("d"))
    imgs = [g[k + "_image"] for k in keys]
    for i in range(0, len(imgs) - 2, 3):
        irr = np.stack([np.maximum(imgs[i + j], 0) for j in range(3)], -1).astype(np.float32)
        su = np.clip(g[keys[i] + "_mod"], 0, 1).astype(np.float32)
        sv = np.clip(g[keys[i + 1] + "_mod"], 0, 1).astype(np.float32)
        print(keys[i], check_pyramid(su, sv, irr, 10 + i, cuda_device))


def test_pyramid_backward_at_2048(cuda_device):
    world, irr, _ = random_maps(S, 11)
    su, sv = stretch(world, cuda_device)
    print(check_pyramid(su, sv, irr, 12, cuda_device))


def test_stretch_backward(cuda_device):
    dev = cuda_device
    for n, seed in ((64, 1), (S, 3)):
        rng = np.random.default_rng(seed)
        world = random_maps(n, seed)[0]
        world[rng.random((n, n)) < 0.01] = rng.uniform(0, 255, 3).astype(np.float32)
        gu, gv = (rng.normal(size=(n, n)).astype(np.float32) for _ in range(2))
        gw = torch.empty((3, n, n), device=dev)
        _lib.call("b200r_sss_stretch_backward", dev, chw(world, dev), _t(gu, dev), _t(gv, dev), gw, n, n)
        got = gw.permute(1, 2, 0).cpu().numpy()
        passes = sg.stretch_pass(world)
        w64 = torch.tensor(world, dtype=torch.float64, device=dev, requires_grad=True)
        u, v = sg.stretch(w64, passes)
        (u * torch.from_numpy(gu).to(dev) + v * torch.from_numpy(gv).to(dev)).sum().backward()
        want = w64.grad.cpu().numpy()
        b = sg.stretch_bound(w64.detach(), passes, torch.from_numpy(gu).to(dev), torch.from_numpy(gv).to(dev)).cpu().numpy()
        r = np.abs(got - want) / b
        print(n, float(r.max()), float(passes[0].mean()))
        assert passes[0].any() and (r <= 1).all(), r.max()


def test_bake_backward(cuda_device):
    dev = cuda_device
    rng = np.random.default_rng(5)
    H = W = 96
    for R in (1, 3, 5):
        nf = 60
        uv = rng.uniform(0, 1, (nf, 3, 2)).astype(np.float32)
        uv[:6] = 1.0                          # UV = 1 reads one past the last row / column: clamped
        uv[6:12, :, 0] = 1.0
        upd = (rng.random(nf) < 0.8).astype(np.int32)
        upd[:3] = 1
        g = rng.normal(size=(nf, R * R, 3)).astype(np.float32)
        gi = torch.empty((H, W, 3), device=dev)
        _lib.call("b200r_bake_textures_softras_backward", dev, _t(g, dev), _t(uv, dev), torch.from_numpy(upd).to(dev), gi,
                  nf, R, H, W)
        got = gi.cpu().numpy()
        gt = torch.from_numpy(g).to(dev)
        want, _ = sg.bake_vjp(gt, uv, R, H, W, upd)
        b = sg.bake_bound(gt, uv, R, H, W, upd).cpu().numpy()
        r = np.abs(got - want.cpu().numpy()) / b
        print(R, float(r.max()))
        assert (r <= 1).all(), r.max()
        # faces with is_update == 0 contribute nothing
        g0 = np.where(upd[:, None, None] != 0, 0, g).astype(np.float32)
        _lib.call("b200r_bake_textures_softras_backward", dev, _t(g0, dev), _t(uv, dev), torch.from_numpy(upd).to(dev), gi,
                  nf, R, H, W)
        assert (gi == 0).all()


# ---------------------------------------------------------------------------------------------- Lighting

def _mesh(g, dev, normal_map, grad=True, **over):
    """The golden mesh; `over` replaces arrays of the file (by key) with tensors."""
    t = lambda k: (over[k] if k in over else _t(g[k], dev)).requires_grad_(grad)
    nt = dict(normal_textures=t("normal_textures"), TBN=_t(g["TBN"], dev)) if normal_map else {}
    return jr.Mesh(t("vertices"), torch.from_numpy(g["faces"]).to(dev), textures=t("textures"),
                   texture_res=int(g["texture_res"]), metallic_textures=t("metallic"), roughness_textures=t("roughness"),
                   with_SSS=True, face_texcoords=_t(g["face_texcoords"], dev), **nt)


def _lit(m, eyes, sss_grad):
    light = jr.Lighting(**LIGHT)
    light.sss_grad = sss_grad
    return light(m, eyes).textures


def _leaves(m, normal_map):
    out = dict(textures=m.textures, vertices=m.vertices, metallic=m.metallic_textures, roughness=m.roughness_textures)
    if normal_map:
        out["normal_textures"] = m.normal_textures
    return out


def _composite(g, dev, normal_map, specular, weight):
    """Lighting's SSS path with the product's SoftRas for the three texture-space rasterizations and the float64
    mirror (oracle/sss_grad.py) for the stretch, the pyramid and the bake; torch autograd for the rest."""
    m = _mesh(g, dev, normal_map)
    m.with_specular = specular
    leaves = _leaves(m, normal_map)
    light = jr.Lighting(**LIGHT)
    captured = {}

    def sss(diffuse, spec, mesh, grad=False):
        world_map, irr_map, spec_map = lighting._sss_maps(diffuse, spec, mesh)
        world = world_map[0, :3].permute(1, 2, 0)
        su32, sv32 = (np.asarray(x, np.float32) for x in osss.stretch(world.detach().cpu().numpy()))
        su, sv = sg.stretch(world.double(), sg.stretch_pass(world.detach().cpu().numpy()))
        irr = irr_map[0, :3].permute(1, 2, 0)
        spc = spec_map[0, :3].permute(1, 2, 0)
        levels = sg.walk(su32, sv32, irr.detach().cpu().numpy())
        final = sg.pyramid(su, sv, irr.double(), spc.double(), levels)
        R = int(mesh.texture_res)
        return sg.bake(final, mesh.face_texcoords[0].cpu().numpy(), R)[None].float()
    orig = lighting.SSS
    lighting.SSS = sss
    try:
        out = light(m, _t(g["eyes"], dev)).textures
    finally:
        lighting.SSS = orig
    (out * weight).sum().backward()
    return _grads(leaves)


def _grads(leaves):
    return {k: (torch.zeros_like(v) if v.grad is None else v.grad).cpu().numpy() for k, v in leaves.items()}


BRANCHES = ["face_specular", "face_diffuse", "normal_specular", "normal_diffuse"]


@pytest.mark.parametrize("tag", BRANCHES)
def test_lighting_forward_bits_and_gradients(cuda_device, tag):
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    dev = cuda_device
    nm, spec = tag.startswith("normal"), tag.endswith("specular")
    eyes = _t(g["eyes"], dev)
    m0 = _mesh(g, dev, nm)
    m0.with_specular = spec
    off = _lit(m0, eyes, False)
    m = _mesh(g, dev, nm)
    m.with_specular = spec
    leaves = _leaves(m, nm)
    on = _lit(m, eyes, True)
    assert not off.requires_grad and on.requires_grad
    assert torch.equal(off, on.detach())
    weight = torch.from_numpy(np.random.default_rng(7).normal(size=tuple(on.shape)).astype(np.float32)).to(dev)
    (on * weight).sum().backward()
    got = _grads(leaves)
    want = _composite(g, dev, nm, spec, weight)
    for k in got:
        top = np.abs(want[k]).max()
        d = np.abs(got[k] - want[k]).max()
        print("%s %s: max |diff| %.3g of max %.3g" % (tag, k, d, top))
        assert np.isfinite(got[k]).all()
        if not spec and k in ("metallic", "roughness"):
            assert top == 0 and d == 0
            continue
        assert top > 0, k
        assert d <= 2e-3 * top, (k, d, top)


def _kink_free(m, eyes, specular):
    """[1, nf, T, 1] mask of the texels whose per-texel normal sits at least 0.05 from every kink of the op-by-op
    lighting: the relu of N.L (the diffuse cosine) and, with the specular term, the relus of N.V and N.H and the clamp
    of 4 (N.V)(N.L) at 0.01."""
    n = m.surface_ResNormals.detach()
    light = torch.nn.functional.normalize(torch.tensor(LIGHT["directions"], device=n.device), dim=0)
    cl = (n * light).sum(-1)
    ok = cl.abs() >= 0.05
    if specular:
        pos = (torch.sum(m.face_vertices.detach(), dim=2) / 3.0)[:, :, None, :]
        v = torch.nn.functional.normalize(eyes.reshape(1, 1, 1, 3) - pos, dim=3, eps=1e-12)
        hv = torch.nn.functional.normalize(v + light, dim=3, eps=1e-12)
        cv, ch = (n * v).sum(-1), (n * hv).sum(-1)
        ok &= (cv.abs() >= 0.05) & (ch.abs() >= 0.05) & ((4 * cv.clamp(min=0) * cl.clamp(min=0) - 0.01).abs() >= 0.01)
    return ok[..., None]


@pytest.mark.parametrize("tag", ["face_specular", "normal_specular", "normal_diffuse"])
def test_lighting_central_differences(cuda_device, tag):
    """Directional derivatives of a weighted sum of the lit textures along random directions of the textures, the
    metallic and roughness textures (with the specular term) and the normal textures (normal-map branch), against
    float32 central differences of step 1e-3.  The loss must be smooth within the step, so:
    - the textures start in [0.2, 1], where sqrt(textures * diffuse) is smooth and no SSS decision changes;
    - the weights skip the lit textures within 0.01 of the final clamp's bounds (Lighting clamps to [0, 1]);
    - a normal-texture direction leaves alone the texels near a kink of the lighting (_kink_free).
    Without the last two, the golden mesh puts a face's nine texels within 0.005 of the diffuse cosine's relu kink, five
    of them change sides at this step, and the central difference misses autograd by 11 % (18 % with the specular
    term); it converges to autograd as the step shrinks (at 1e-4 no texel changes sides, and it agrees to 0.2 %), so
    the gap is the step's, not the gradient's.  Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): textures and
    materials within 0.1 %, the normal textures within 3e-5 without the specular term; with it their derivative is
    small (-0.797) and the central difference 0.017 away, inside the absolute 2e-2, which covers the float32 loss's
    rounding noise over a step of 2e-3."""
    g = dict(np.load(os.path.join(G, "ref_host_sss.npz")))
    g["textures"] = (0.2 + 0.8 * np.clip(g["textures"], 0, 1)).astype(np.float32)
    dev = cuda_device
    nm, specular = tag.startswith("normal"), tag.endswith("specular")
    eyes = _t(g["eyes"], dev)
    weight = torch.from_numpy(np.random.default_rng(8).normal(size=g["textures"].shape).astype(np.float32)).to(dev)
    rng = np.random.default_rng(9)
    m = _mesh(g, dev, nm)
    m.with_specular = specular
    leaves = _leaves(m, nm)
    out = _lit(m, eyes, True)
    weight = weight * ((out.detach() > 0.01) & (out.detach() < 0.99))
    (out * weight).sum().backward()

    def loss(mesh):
        mesh.with_specular = specular
        return float((_lit(mesh, eyes, True) * weight).double().sum())
    names = ["textures"] + (["metallic", "roughness"] if specular else []) + (["normal_textures"] if nm else [])
    for name in names:
        x0 = leaves[name].detach()
        d = torch.from_numpy(rng.normal(size=tuple(x0.shape)).astype(np.float32)).to(dev)
        if name == "normal_textures":
            keep = _kink_free(m, eyes, specular)
            assert keep.float().mean() > 0.5   # measured: all but 91 of the 3240 texels diffuse, 71 % with specular
            d = d * keep
        h = 1e-3
        vals = []
        for s in (1, -1):
            vals.append(loss(_mesh(g, dev, nm, grad=False, **{name: x0 + s * h * d})))
        fd = (vals[0] - vals[1]) / (2 * h)
        an = float((leaves[name].grad.double() * d.double()).sum())
        print("%s %s: analytic %.6g, central difference %.6g" % (tag, name, an, fd))
        assert abs(an - fd) <= 0.02 * abs(an) + 2e-2, (name, an, fd)


def _profiled(run):
    L = _lib.lib()
    torch.cuda.synchronize()
    L.b200r_profile_reset()
    L.b200r_profile_enable(1)
    try:
        n0 = L.b200r_launch_count()
        run()
        torch.cuda.synchronize()
        delta = L.b200r_launch_count() - n0
    finally:
        L.b200r_profile_enable(0)
    counts = []
    for k in range(26):
        n = C.c_longlong(0)
        assert L.b200r_profile_read(k, None, C.byref(n)) == 0
        counts.append(n.value)
    return delta, counts


def test_launch_counts(cuda_device):
    """sss_grad on with nothing requiring grad launches exactly what the forward always did (3 SoftRas forwards, 7 SSS,
    1 bake).  With grad the backward adds, per frame: the pyramid backward's 6 recomputed forward passes and 6
    transposed passes plus the stretch backward (13 more under B200R_K_SSS), one bake backward (under B200R_K_BAKE),
    and one SoftRas backward per texture-space rasterization (3 when the vertices require grad: world, irradiance and
    specular maps)."""
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    dev = cuda_device
    eyes = _t(g["eyes"], dev)
    run = lambda: _lit(_mesh(g, dev, True, grad=False), eyes, True)
    run()
    delta, counts = _profiled(run)
    assert (counts[K_SOFTRAS_FWD], counts[K_SSS], counts[K_BAKE]) == (3, 7, 1), counts
    assert counts[K_SOFTRAS_BWD] == 0, counts
    assert delta == sum(counts)
    # one SoftRas backward's own launches, for the count below
    from jrender_b200.softras import SoftRasterizeFunction
    fv = torch.rand((1, 4, 3, 3), device=dev, requires_grad=True)
    one = lambda: SoftRasterizeFunction(image_size=16)(fv, torch.rand((1, 4, 1, 3), device=dev)).sum().backward()
    one()
    _, c1 = _profiled(one)
    per_bwd = c1[K_SOFTRAS_BWD]

    def step():
        m = _mesh(g, dev, True)
        (_lit(m, eyes, True) * 1.0).sum().backward()
    step()
    delta, counts = _profiled(step)
    assert (counts[K_SOFTRAS_FWD], counts[K_SSS], counts[K_BAKE]) == (3, 7 + 13, 1 + 1), counts
    assert counts[K_SOFTRAS_BWD] == 3 * per_bwd, counts
    assert delta == sum(counts)


def test_errors(cuda_device):
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    dev = cuda_device
    eyes = _t(g["eyes"], dev)
    m = jr.Mesh(_t(g["vertices"], dev), torch.from_numpy(g["faces"]).to(dev), textures=_t(g["textures"], dev).requires_grad_(),
                texture_res=int(g["texture_res"]), with_SSS=True,
                face_texcoords=_t(g["face_texcoords"], dev).requires_grad_())
    with pytest.raises(ValueError, match="face_texcoords"):
        _lit(m, eyes, True)
    n = 64
    su, sv, irr = threshold_maps(n, 3)
    z = np.zeros((n, n, 3), np.float32)
    with pytest.raises(_lib.B200RasterError, match="workspace"):
        pyramid_backward(su, sv, irr, z, dev, nbytes=_lib.lib().b200r_sss_backward_workspace_bytes(n, n, 3) - 4)
    with pytest.raises(_lib.B200RasterError, match="square"):
        pyramid_backward(su[:, :48], sv[:, :48], irr[:, :48], z[:, :48], dev, nbytes=1 << 20)
    taps, widths, weights, L = lighting._sss_levels()
    x = torch.zeros((3, n, n), device=dev)
    with pytest.raises(_lib.B200RasterError, match="NULL"):
        _lib.call("b200r_sss_blur_pyramid_backward", dev, x, x, x, None, x, x, None, None, x, 1 << 30, taps, widths,
                  weights, L, n, n)
    with pytest.raises(_lib.B200RasterError, match="both"):
        _lib.call("b200r_sss_blur_pyramid_backward", dev, x, x, x, x, x, x, x, None, x, 1 << 30, taps, widths,
                  weights, L, n, n)
    with pytest.raises(_lib.B200RasterError, match="NULL"):
        _lib.call("b200r_sss_stretch_backward", dev, x, None, x, x, n, n)
    with pytest.raises(_lib.B200RasterError, match="NULL"):
        _lib.call("b200r_bake_textures_softras_backward", dev, x, None, x, x, 1, 1, n, n)
    assert _lib.lib().b200r_sss_backward_workspace_bytes(n, n, 0) == 0
    assert _lib.lib().b200r_sss_backward_workspace_bytes(S, S, 3) == 34 * S * S * 4


def test_albedo_fit_on_sphere(cuda_device):
    """Fit the albedo of a with_SSS UV sphere (384 faces, R = 3) to renders of a target albedo, from flat 0.5 grey,
    through SSS with sss_grad on: 12 Adam steps at lr 0.05 over 2 views at 64^2.  Measured on an NVIDIA H100 80GB HBM3
    (700 W power limit): the loss falls from 80.0 to 8.7, a ratio of 0.11; the test asks for under 0.5."""
    dev = cuda_device
    v, f = wl.uv_sphere(16, 13)
    uv = np.clip((v[:, :2] / 0.8 + 1) / 2 * 0.98 + 0.01, 0, 1).astype(np.float32)
    R = 3
    rng = np.random.default_rng(0)
    target = _t(rng.uniform(0.2, 0.9, (1, f.shape[0], R * R, 3)), dev)
    r = jr.Renderer(dr_type='softras', image_size=64, light_intensity_ambient=0.45, light_intensity_directionals=1,
                    light_directions=[0.65, -0.2, -1], dist_func="barycentric", aggr_func_rgb='hard',
                    camera_mode="look_at")
    r.lighting.sss_grad = True

    def render(tex, azimuth):
        m = jr.Mesh(_t(v[None], dev), torch.from_numpy(f[None]).to(dev), textures=tex, texture_res=R, with_SSS=True,
                    face_texcoords=_t(uv[f][None], dev))
        r.transform.set_eyes_from_angles(2.0, 20, azimuth)
        return r.render_mesh(m, mode='rgb')[0]
    azimuths = (0, 180)
    with torch.no_grad():
        targets = [render(target, a) for a in azimuths]
    param = torch.full_like(target, 0.5).requires_grad_(True)
    opt = torch.optim.Adam([param], lr=0.05)
    losses = []
    for _ in range(12):
        opt.zero_grad()
        loss = sum(((render(param, a) - t) ** 2).sum() for a, t in zip(azimuths, targets))
        loss.backward()
        assert param.grad.abs().sum() > 0
        opt.step()
        with torch.no_grad():
            param.clamp_(0.05, 1)
        losses.append(float(loss.detach()))
    print("albedo fit: loss %.5g -> %.5g (ratio %.3f)" % (losses[0], losses[-1], losses[-1] / losses[0]))
    assert losses[-1] < 0.5 * losses[0], losses
