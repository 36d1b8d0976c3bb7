"""GPU tests of the texture-space subsurface scattering: the kernels b200r_sss_stretch / b200r_sss_blur_pyramid
(csrc/sss_api.cu), Lighting's SSS path, and its launches and errors.

- stretch and pyramid against oracle/sss.py: bit-identical (both unfused float32 in the reference's order), on the
  golden blur maps and on seeded 2048^2 maps with background holes;
- pyramid against the reference's own blur kernels (oracle/_ref, built by oracle/build_ref_sss.py), chained the
  reference's way: per channel, three levels of four blurs, 36 launches.  The reference build contracts a*b+c into
  FMAs, which moves each blurred value by a few ulp (tests/test_sss_cpu.py bounds one blur).  The chain amplifies that:
  a blurred stretch value is the next blur's tap spacing, and moving a tap by d moves the result by about d times the
  image's jump between neighbouring pixels, up to 1 at face edges, times the tap weight.  A numpy emulation of the fused
  blur gives differences up to about 1.4e-4 after three levels at 512^2.  And a few values are discontinuous in the tap
  position: a tap that crosses x = W - 1 or x = -1 drops from v (or an extrapolation) to the 0 of its clamped pair, so
  where a tap sits within rounding of an edge the two builds can differ by a whole tap weight.  So REF_TOL of the largest
  output holds all but a fraction FLIP_FRACTION of the values, and every value stays within the largest output.
  Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): a maximum difference of 0.036 (of a largest value of 1.23),
  and 3.97e-7 of the values beyond REF_TOL of max (5 of 12.6 million);
- Lighting with a with_SSS mesh against tests/golden/ref_host_sss.npz (the reference's own lighting.py through the
  numpy jittor stand-in and the oracles), both branches, specular on and off.  The diffuse and specular light are
  float32 op by op on both sides, in different reduction orders (torch against numpy), so the inputs of the maps
  differ by a few ulp; held to LIT_TOL absolute on textures in [0, 1].  Measured on the same card: at most 6.8e-6
  (normal map, specular on).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib, lighting
from oracle import build_ref_sss
from oracle import sss as osss

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
LIGHT = dict(intensity_ambient=0.45, color_ambient=[1.0, 0.95, 0.9], intensity_directionals=1.0,
             color_directionals=[0.9, 1.0, 0.8], directions=[0.65, -0.2, -1.0])
REF_TOL = 1e-3
FLIP_FRACTION = 1e-5
LIT_TOL = 2e-5
S = lighting.SSS_IMAGE_SIZE


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)


def stretch(world_chw):
    """b200r_sss_stretch on a [3, H, W] tensor -> (stretch_u, stretch_v) numpy."""
    H, W = world_chw.shape[1:]
    su = torch.empty((H, W), dtype=torch.float32, device=world_chw.device)
    sv = torch.empty_like(su)
    _lib.call("b200r_sss_stretch", world_chw.device, world_chw, su, sv, H, W)
    return su.cpu().numpy(), sv.cpu().numpy()


def pyramid(su, sv, irr_chw, spec_chw):
    """b200r_sss_blur_pyramid with the reference's three levels -> [H, W, 3] numpy (flipped)."""
    dev = irr_chw.device
    H, W = irr_chw.shape[1:]
    variances = osss.levels()
    taps, widths = zip(*[lighting._sss_taps(v) for v in variances])
    L = len(variances)
    nbytes = _lib.lib().b200r_sss_workspace_bytes(H, W)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    out = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
    _lib.call("b200r_sss_blur_pyramid", dev, _t(su, dev), _t(sv, dev), irr_chw, spec_chw, out, ws, nbytes,
              (C.c_float * (7 * L))(*[t for lv in taps for t in lv]), (C.c_float * L)(*widths),
              (C.c_float * (3 * L))(*[w for ch in lighting.SSS_WEIGHTS for w in ch]), L, H, W)
    return out.cpu().numpy()


def random_maps(S_, seed):
    """world [S, S, 3] flat over 16 x 16 patches (as the rasterized world coordinates are flat over faces), irradiance
    and specular [S, S, 3], all zero in background holes."""
    rng = np.random.default_rng(seed)
    n = S_ // 16
    world = np.kron(rng.uniform(0, 255, (n, n, 3)), np.ones((16, 16, 1))).astype(np.float32)
    world += np.kron(rng.uniform(0, 1, (n, n, 1)), np.ones((16, 16, 3))).astype(np.float32) * np.float32(0.02) \
        * np.arange(S_, dtype=np.float32)[None, :, None]   # some patches vary, so stretch takes values inside (0, 1)
    hole = np.kron(rng.random((n, n)) < 0.3, np.ones((16, 16))).astype(bool)
    hole[:5] = True
    hole[:, -7:] = True
    irr = rng.uniform(0, 1, (S_, S_, 3)).astype(np.float32)
    spec = rng.uniform(0, 0.3, (S_, S_, 3)).astype(np.float32)
    for a in (world, irr, spec):
        a[hole] = 0
    return world, irr, spec


def chw(a, dev):
    return _t(np.transpose(a, (2, 0, 1)), dev)


def test_stretch_bit_identical_to_oracle(cuda_device):
    for shape, seed in (((64, 64), 1), ((48, 80), 2), ((S, S), 3)):
        rng = np.random.default_rng(seed)
        world = random_maps(max(shape) // 16 * 16, seed)[0][:shape[0], :shape[1]]
        world[rng.random(shape) < 0.01] = rng.uniform(0, 255, 3).astype(np.float32)   # isolated pixels too
        su, sv = stretch(chw(world, cuda_device))
        ou, ov = osss.stretch(world)
        np.testing.assert_array_equal(su, ou)
        np.testing.assert_array_equal(sv, ov)
        assert (su == 1).any() and ((su > 0) & (su < 1)).any()


def test_pyramid_bit_identical_to_oracle_on_golden_maps(cuda_device):
    g = np.load(os.path.join(G, "ref_sss_gpu_blur_64x64.npz"))
    keys = sorted(k[:-6] for k in g.files if k.endswith("_image") and k.startswith("d"))
    imgs = [g[k + "_image"] for k in keys]
    for i in range(0, len(imgs) - 2, 3):
        irr = np.stack([np.maximum(imgs[i + j], 0) for j in range(3)], -1)
        spec = np.stack([imgs[(i + j + 1) % len(imgs)] for j in range(3)], -1)
        su, sv = np.clip(g[keys[i] + "_mod"], 0, 1), np.clip(g[keys[i + 1] + "_mod"], 0, 1)
        got = pyramid(su, sv, chw(irr, cuda_device), chw(spec, cuda_device))
        np.testing.assert_array_equal(got, osss.blur_pyramid(su, sv, irr, spec))


def test_pyramid_bit_identical_to_oracle_at_2048(cuda_device):
    world, irr, spec = random_maps(S, 11)
    su, sv = stretch(chw(world, cuda_device))
    got = pyramid(su, sv, chw(irr, cuda_device), chw(spec, cuda_device))
    want = osss.blur_pyramid(su, sv, irr, spec)
    np.testing.assert_array_equal(got, want)
    assert (got == 0).any() and (got > 0).mean() > 0.5


@pytest.mark.skipif(build_ref_sss.lib() is None, reason="oracle/_ref/libjrender_ref_sss.so not built")
def test_pyramid_against_reference_kernels_at_2048(cuda_device):
    L = build_ref_sss.lib()
    dev = cuda_device
    world, irr, spec = random_maps(S, 12)
    su, sv = stretch(chw(world, dev))
    got = pyramid(su, sv, chw(irr, dev), chw(spec, dev))
    irr_t, spec_t = _t(irr, dev), _t(spec, dev)
    final = torch.zeros_like(irr_t)
    levels = [(_t(osss.taps(v)[0], dev), osss.taps(v)[1]) for v in osss.levels()]
    for j in range(3):   # lighting.py:133-145
        su_c, sv_c, x = _t(su, dev), _t(sv, dev), irr_t[:, :, j].contiguous()
        basis = []
        for gauss, width in levels:
            su_c = build_ref_sss.blur(L, su_c, su_c, gauss, width, 1)
            x = build_ref_sss.blur(L, x, su_c, gauss, width, 1)
            sv_c = build_ref_sss.blur(L, sv_c, sv_c, gauss, width, 0)
            x = build_ref_sss.blur(L, x, sv_c, gauss, width, 0)
            basis.append(x.clone())
        for k, image in enumerate(basis):
            final[:, :, j] += lighting.SSS_WEIGHTS[j][k] * image
    ref = torch.flip(final * irr_t + spec_t, [0]).cpu().numpy()
    d = np.abs(got - ref)
    top = float(np.abs(ref).max())
    flips = float((d > REF_TOL * top).mean())
    print("SSS pyramid vs the reference kernels: max |diff| %.3g of max %.3g; %.3g of the values beyond %.0e of max"
          % (d.max(), top, flips, REF_TOL))
    hole = irr.sum(-1)[::-1] == 0
    np.testing.assert_array_equal(got[hole], spec[::-1][hole])   # holes keep only the specular map, on both sides
    np.testing.assert_array_equal(ref[hole], spec[::-1][hole])
    assert flips <= FLIP_FRACTION, flips
    assert d.max() <= top, d.max()


def _mesh(g, dev, normal_map, **kw):
    nt = dict(normal_textures=_t(g["normal_textures"], dev), TBN=_t(g["TBN"], dev)) if normal_map else {}
    args = dict(textures=_t(g["textures"], dev), texture_res=int(g["texture_res"]),
                metallic_textures=_t(g["metallic"], dev), roughness_textures=_t(g["roughness"], dev),
                with_SSS=True, face_texcoords=_t(g["face_texcoords"], dev))
    args.update(nt)
    args.update(kw)
    return jr.Mesh(_t(g["vertices"], dev), torch.from_numpy(g["faces"]).to(dev), **args)


@pytest.mark.parametrize("tag", ["face_specular", "face_diffuse", "normal_specular", "normal_diffuse"])
def test_lighting_matches_reference_golden(cuda_device, tag):
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    m = _mesh(g, cuda_device, tag.startswith("normal"))
    m.vertices.requires_grad_(True)
    m.with_specular = tag.endswith("specular")
    out = jr.Lighting(**LIGHT)(m, _t(g["eyes"], cuda_device)).textures
    assert not out.requires_grad and out.grad_fn is None
    got, want = out.detach().cpu().numpy(), g["lit_" + tag]
    diff = np.abs(got - want).max()
    print("%s: max |diff| %.3g" % (tag, diff))
    assert diff <= LIT_TOL, diff


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


def test_sss_launches_are_counted(cuda_device):
    """One SSS frame: three SoftRas forwards, the stretch, 2 x 3 blur passes, one bake."""
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    run = lambda: jr.Lighting(**LIGHT)(_mesh(g, cuda_device, True), _t(g["eyes"], cuda_device))
    run()
    delta, counts = _profiled(run)
    assert counts[25] == 7, counts          # B200R_K_SSS
    assert counts[16] == 1, counts          # B200R_K_BAKE
    assert counts[2] == 3, counts           # B200R_K_SOFTRAS_FWD
    assert counts[15] == 0, counts          # the fused lighting kernels are not used on this path
    assert delta == sum(counts), (delta, counts)


def test_errors(cuda_device):
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    dev = cuda_device
    light = jr.Lighting(**LIGHT)
    eye = _t(g["eyes"], dev)
    two = jr.Mesh(_t(np.concatenate([g["vertices"]] * 2), dev), torch.from_numpy(np.concatenate([g["faces"]] * 2)).to(dev),
                  textures=_t(np.concatenate([g["textures"]] * 2), dev), with_SSS=True,
                  face_texcoords=_t(np.concatenate([g["face_texcoords"]] * 2), dev))
    with pytest.raises(ValueError, match="batch"):
        light(two, eye)
    with pytest.raises(ValueError, match="face_texcoords"):
        light(_mesh(g, dev, False, face_texcoords=None), eye)
    with pytest.raises(ValueError, match="texels"):
        light(_mesh(g, dev, False, textures=_t(g["textures"][:, :, :8], dev), metallic_textures=None,
                    roughness_textures=None), eye)
    # the pyramid takes square maps only (the reference's y kernel clamps rows against the width)
    x = torch.zeros((3, 8, 6), device=dev)
    with pytest.raises(_lib.B200RasterError, match="square"):
        pyramid(np.zeros((8, 6), np.float32), np.zeros((8, 6), np.float32), x, x)


def test_six_d_textures_ignore_with_sss(cuda_device):
    """NMR textures [B, nf, ts, ts, ts, 3] render as they did: with_SSS is ignored there, as in the reference."""
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    dev = cuda_device
    tex = _t(np.random.default_rng(3).uniform(0, 1, (1, g["faces"].shape[1], 2, 2, 2, 3)), dev)
    out = []
    for sss in (True, False):
        m = jr.Mesh(_t(g["vertices"], dev), torch.from_numpy(g["faces"]).to(dev), textures=tex, dr_type='n3mr',
                    texture_res=2, with_SSS=sss, face_texcoords=_t(g["face_texcoords"], dev))
        out.append(jr.Lighting(**LIGHT)(m, _t(g["eyes"], dev)).textures.detach().cpu().numpy())
    np.testing.assert_array_equal(out[0], out[1])
