"""Normal and depth G-buffers (Lighting(Gbuffer='normal' | 'depth')) on the CPU: the op-by-op mirror against the
reference's own Lighting.execute and Renderer.render_mesh (tests/golden/ref_host_gbuffer.npz, oracle/
make_ref_host_gbuffer_golden.py) within 2e-5 of each array's max, the tolerance test_host_golden.py uses for the lighting
stage; the float32 emulation of the kernels (oracle/gbuffer.py) against the float64 mirror; and the decisions the
reference leaves open: the max's gradient on ties, NaN through the max, and the error cases."""
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200.lighting import Lighting, _normalized_direction, camera_z
from oracle import gbuffer as OG
from oracle.numbers import F32

G = os.path.join(os.path.dirname(__file__), "golden", "ref_host_gbuffer.npz")
LIGHT = dict(intensity_ambient=0.4, color_ambient=[1.0, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1.0, 0.7], directions=[0.3, 0.8, -0.5])
TOL = 2e-5


def _close(a, b, tol=TOL):
    b = np.asarray(b, np.float64)
    return np.abs(np.asarray(a, np.float64) - b).max() <= tol * max(np.abs(b).max(), 1e-30)


def _transform(eyes):
    t = jr.Transform(camera_mode='look_at', viewing_angle=30)
    t.set_eyes(eyes)
    return t


def _golden_case(g, tag, dtype=torch.float32):
    mode, branch, spec = tag.split("_")
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    light_mode = 'vertex' if branch == 'vertex' else 'surface'
    nm = branch == 'normalmap'
    tex = t("in_" + tag) if ("in_" + tag) in g else torch.rand(g["metallic"].shape[:3] + (3,), dtype=dtype)
    mesh = jr.Mesh(t("vertices"), torch.from_numpy(g["faces"]), textures=tex,
                   dr_type='n3mr' if tex.dim() == 6 else 'softras',
                   metallic_textures=t("metallic"), roughness_textures=t("roughness"),
                   normal_textures=t("normal_textures") if nm else None, TBN=t("tbn") if nm else None,
                   texture_res=2)
    mesh.with_specular = spec == "spec1"
    eyes = t("eyes")
    return Lighting(light_mode, Gbuffer=mode, transform=_transform(eyes), **LIGHT), mesh, eyes


def test_mirror_matches_reference_lighting():
    g = np.load(G)
    tags = sorted(k[4:] for k in g.files if k.startswith("out_"))
    assert len(tags) == 10
    for tag in tags:
        light, mesh, eyes = _golden_case(g, tag)
        out = light(mesh, eyes).textures
        assert out.shape == g["out_" + tag].shape, tag
        assert _close(out.numpy(), g["out_" + tag]), tag


@pytest.mark.parametrize("camera_mode", ["look_at", "look", "projection"])
def test_depth_with_normal_map_raises_the_reference_error(camera_mode):
    g = np.load(G)
    assert str(g["err_depth_normalmap_spec1"]) == 'vertices Tensor should have 3 dimensions'
    light, mesh, eyes = _golden_case(g, "depth_normalmap_spec1")
    kw = dict(K=np.eye(3, dtype=np.float32)[None], R=np.eye(3, dtype=np.float32)[None],
              t=np.zeros((1, 3), np.float32)) if camera_mode == 'projection' else {}
    light.directionals[0].transform = light.transform = jr.Transform(camera_mode=camera_mode, **kw)
    with pytest.raises(ValueError, match=str(g["err_depth_normalmap_spec1"])):
        light(mesh, eyes)


def test_depth_without_transform_and_unknown_gbuffer_raise():
    g = np.load(G)
    light, mesh, eyes = _golden_case(g, "depth_surface4_spec1")
    light.directionals[0].transform = light.transform = None
    with pytest.raises(ValueError, match="transform"):
        light(mesh, eyes)
    with pytest.raises(ValueError, match="Gbuffer"):
        Lighting(Gbuffer='depht')
    for ok in ('None', None, 'albedo', 'normal', 'depth'):
        Lighting(Gbuffer=ok)


def test_textures_get_no_gradient():
    g = np.load(G)
    for tag in ("normal_surface4_spec1", "depth_surface4_spec0"):
        light, mesh, eyes = _golden_case(g, tag)
        tex = mesh.textures.clone().requires_grad_(True)
        v = mesh.vertices.clone().requires_grad_(True)
        mesh = jr.Mesh(v, mesh.faces, textures=tex)
        light(mesh, eyes).textures.sum().backward()
        assert tex.grad is None and torch.isfinite(v.grad).all() and v.grad.abs().sum() > 0


def test_max_gradient_goes_in_full_to_every_tie():
    """Two faces mirrored about the view plane of a camera on the z axis have the same depth: both get the max's whole
    gradient (the mask z == max), where torch.max would split it."""
    v = torch.tensor([[[-1., 0., 1.], [0., 1., 1.], [0., -1., 1.], [1., 0., 1.], [0., 0., 0.5]]], dtype=torch.float64,
                     requires_grad=True)
    f = torch.tensor([[[0, 1, 2], [3, 2, 1], [0, 4, 1]]])
    mesh = jr.Mesh(v, f, textures=torch.ones((1, 3, 1, 3), dtype=torch.float64))
    mesh.with_specular = False
    tr = jr.Transform(camera_mode='look_at', eye=[0., 0., -3.])
    light = Lighting(Gbuffer='depth', transform=tr)
    z = camera_z(tr, torch.sum(mesh.face_vertices, dim=2) / 3.0)
    assert z[0, 0] == z[0, 1] == z.max() and z[0, 2] < z[0, 0]
    out = light(mesh, None).textures
    g = torch.zeros_like(out)
    g[0, 2] = 1.0   # only the third face's output: its depth z2 / M reaches the tied faces through M alone
    out.backward(g)
    M, z2 = z.max().item(), z[0, 2].item()
    dM = -3 * z2 / (M * M)
    # the depth's z row is (0, 0, 1) here: each tied face passes dM / 3 to each of its vertices' z
    want = np.zeros((5, 3))
    for fi in (0, 1):
        for k in f[0, fi].tolist():
            want[k, 2] += dM / 3
    for k in f[0, 2].tolist():
        want[k, 2] += 3 / M / 3
    assert np.allclose(v.grad[0].numpy(), want, rtol=1e-12, atol=1e-12)


def test_nan_depth_reaches_the_whole_batch():
    g = np.load(G)
    light, mesh, eyes = _golden_case(g, "depth_surface4_spec0")
    v = mesh.vertices.clone()
    v[1, 0, 0] = float('nan')
    mesh = jr.Mesh(v, mesh.faces, textures=mesh.textures)
    mesh.with_specular = False
    out = light(mesh, eyes).textures
    assert torch.isnan(out).all()


def host_args(mesh, light, eyes, mode):
    """The arguments Lighting hands b200r_gbuffer_lighting_forward, built on the host (no GPU)."""
    d = light.directionals[0]
    spec = bool(mesh.with_specular)
    tx = mesh.textures
    B, nf = tx.shape[:2]
    tr = light.transform
    a = dict(vertices=mesh.vertices.numpy().astype(F32), faces=mesh.faces.numpy().astype(np.int32),
             metallic=mesh.metallic_textures.numpy().reshape(B, nf, -1) if spec else None,
             roughness=mesh.roughness_textures.numpy().reshape(B, nf, -1) if spec else None,
             eye=eyes.numpy().reshape(-1, 3) if spec else None, camera_eye=np.asarray(tr.transformer._eye, F32).reshape(-1, 3),
             mode=mode, B=B, Bv=mesh.vertices.shape[0], Bf=mesh.faces.shape[0], Be=eyes.shape[0], Bc=1, nv=mesh.vertices.shape[1],
             nf=nf, T=tx[0, 0].numel() // 3, Tm=mesh.metallic_textures[0, 0].numel(), at=np.zeros(3, F32),
             up=np.float32([0, 1, 0]), camera_mode=0)
    a["Bc"] = a["camera_eye"].shape[0]
    a["light"] = OG._light(d.light_intensity, d.light_color, _normalized_direction(d.light_direction), spec)
    return a


def test_emulation_agrees_with_float64_mirror():
    g = np.load(G)
    for tag in ("normal_surface4_spec1", "normal_surface6_spec1", "depth_surface4_spec1", "depth_surface4_spec0"):
        light, mesh, eyes = _golden_case(g, tag, torch.float64)
        a = host_args(mesh, light, eyes, 0 if tag.startswith("normal") else 1)
        want = light(mesh, eyes).textures.numpy()
        got, _ = OG.gbuffer_forward(a)
        assert _close(got.reshape(want.shape), want, 1e-6), tag


def test_edge_scenes_reach_nonpositive_max_depth():
    """The 'behind' scenes put every centroid behind the camera (M < 0: every z / M >= 1, only the max face at the
    clamp's equality); 'zero_max' makes the largest depth exactly 0 (M = 0)."""
    from tests import gbuffer_edge_cases as E
    for name, check in (("behind_depth_nospec", lambda M, z: M < 0 and (z < 0).all()),
                        ("behind_depth_spec", lambda M, z: M < 0 and (z < 0).all()),
                        ("zero_max_depth_nospec", lambda M, z: M == 0 and int((z == 0).sum()) == z.shape[0])):
        sc = E.scene(name)
        ts, light, mesh, eyes = E.build(sc, torch.device("cpu"), torch.float64, fused=False)
        z = camera_z(light.transform, torch.sum(mesh.face_vertices, dim=2) / 3.0).detach()
        assert check(z.max().item(), z), name


# ---- the backward emulation against float64 autograd -----------------------------------------------------------------
#
# oracle/gbuffer.py restates the backward kernels in numpy float32 (the GPU tests hold the kernels to it bit for bit)
# and, over oracle.numbers.EV, bounds each float32 term's distance from the float64 value of the same expression.  Here
# those bounds are checked against the op-by-op mirror's float64 autograd, entry by entry, as test_lighting_edges_cpu.py
# does for the lighting kernels: per-texel gradients within their own bound, each grad_vertices entry within the sum of
# its terms' bounds.  Members within their bound of a kink -- the clamp at 0 and 1 (every depth scene's max face sits on
# 1), the relus, den4, normalize's eps, a depth within its bound of the max -- may branch the other way in float64 and
# are left out, counted by kind and capped.

from oracle import lighting as OL                      # noqa: E402
from oracle.numbers import EV                          # noqa: E402
from oracle.numbers import check_terms                 # noqa: E402
from tests import gbuffer_edge_cases as E              # noqa: E402

NONFINITE = ("nan_", "pinf_", "ninf_")
NEAR_CAP = 0.01   # most members left out per kind: a share of the scene's members, at least 4
NEAR_CAP_ABS = {"axis_normal_spec": {"relu": 8, "clamp": 16}, "axis_depth_nospec": {"clamp": 8},
                "zero_max_depth_nospec": {"clamp": 8}}


def _excluded(sc, a, near, nm):
    """Per-member masks of what the near-kink members reach: [B, nf, T] texels (nm) or [B, nf] faces, and
    [Bv, nv] vertices."""
    B, nf, T = a["B"], a["nf"], a["T"]
    shape = (B, nf, T) if nm else (B * nf,)
    m = np.zeros(shape, bool)
    for fl in near.values():
        m |= np.asarray(fl, bool).reshape(shape)
    face = m.any(2) if nm else m.reshape(B, nf)
    ex_v = np.zeros(a["vertices"].shape[:2], bool)
    f = a["faces"]
    for b, fc in zip(*np.nonzero(face)):
        ex_v[0 if a["Bv"] == 1 else b, f[0 if a["Bf"] == 1 else b, fc]] = True
    return m, face, ex_v


def _within(got, r, err, A, keep):
    fin = keep & np.isfinite(r) & np.isfinite(got) & np.isfinite(err)
    bound = err + 1e-12 * A + 1e-300
    return float((np.abs(got - r)[fin] / bound[fin]).max(initial=0.0))


@pytest.mark.parametrize("name", [n for n in E.NAMES if n not in E.LARGE] + E.SLIVER_NORMAL + ["grid262145_depth_nospec"])
def test_emulation_within_its_bound_of_float64_autograd(name):
    sc = E.scene(name)
    nm = "nt" in sc
    a = E.kernel_args(sc)
    bwd = OG.nm_gbuffer_backward if nm else OG.gbuffer_backward
    g32 = bwd(a)
    light = dict(OL.light_ev(E.LIGHT, sc["spec"]), amb_i=EV(0.0), amb_c=[EV(0.0)] * 3)
    gev = bwd(dict(a, light=light), lift=EV, replay=g32)
    _, ref = E.run(sc, "cpu", torch.float64, fused=False)
    members = a["B"] * a["nf"] * (a["T"] if nm else 1)
    counts = {k: int(np.count_nonzero(v)) for k, v in gev["near"].items()}
    print("%s: members left out near a kink, by kind: %s of %d" % (name, counts, members))
    for k, n in counts.items():
        # a non-finite input leaves its faces' bounds infinite: each of them counts as near every kink it meets
        cap = NEAR_CAP_ABS.get(name, {}).get(k, max(16 if any(t in name for t in NONFINITE) else 4, NEAR_CAP * members))
        assert n <= cap, (name, k, n, cap)
    ex, face, ex_v = _excluded(sc, a, gev["near"], nm)
    checked = 0
    for k, r in ref.items():
        if k == "textures":
            assert r is None
            continue
        if k == "vertices":
            if r is None:
                assert "vertex_terms" not in g32 or not np.asarray(g32["vertex_terms"]).any(), name
                continue
            t32 = np.asarray(g32["vertex_terms"], np.float64).reshape(-1)
            tev = gev["vertex_terms"]
            check_terms(t32, EV(tev.v.reshape(-1), tev.e.reshape(-1)))
            sl = g32["vertex_slots"].reshape(-1)
            got, err, A = (np.zeros(r.size) for _ in range(3))
            np.add.at(got, sl, t32)
            np.add.at(err, sl, tev.e.reshape(-1))
            np.add.at(A, sl, np.abs(tev.v.reshape(-1)))
            got, err, A = (x.reshape(r.shape) for x in (got, err, A))
            keep = ~np.broadcast_to(ex_v[..., None], r.shape)
        else:
            got, ev = g32[k], gev[k]
            if r is None:
                assert got is None or not np.asarray(got).any(), (name, k)
                continue
            check_terms(got, ev)
            got, err, A = np.asarray(got, np.float64), ev.e, np.abs(ev.v)
            if got.size != r.size:   # a per-face material expanded over the texels: the expand's backward sums them
                got, err, A = (x.reshape(r.shape[:2] + (-1,)).sum(2) for x in (got, err, A))
            got, err, A = (x.reshape(r.shape) for x in (got, err, A))
            if k == "normal_textures":
                keep = ~(ex.any(0, keepdims=True) if r.shape[0] == 1 else ex)
            elif nm:   # per texel, per-face materials summed over the texels by the expand's backward
                keep = ~(ex if r.shape[2] == ex.shape[2] else ex.any(2, keepdims=True))
            else:
                keep = ~face[:, :, None]
            keep = np.broadcast_to(keep.reshape(keep.shape + (1,) * (r.ndim - keep.ndim)), r.shape)
        ratio = _within(got, r, err, A, keep)
        print("  %-16s worst |f32 - f64| / bound %.3f" % (k, ratio))
        assert ratio <= 1, (name, k, ratio)
        checked += 1
    assert checked >= 1, name


def test_large_scenes_reach_the_grid_stride_path():
    """262 145 and 627 200 pairs take more than one grid-stride trip of the 1024 x 256 threads; 262 144 fills every
    partial exactly once; the big scene's max and its exact tie lie past pair 262 144, in different partials; the split
    tie's faces are in different blocks, so different partials."""
    stride = OG.GB_PARTIALS * OG.GB_THREADS
    for n in E.GRID:
        assert E.scene("grid%d_depth_nospec" % n)["f"].shape[0] == n
    assert OG.depth_grid(262144) == OG.depth_grid(262145) == OG.GB_PARTIALS and 262144 == stride
    for name, first in (("big_depth_nospec", stride), ("split_ties_depth_spec", 0)):
        z, partials, M = OG.face_depths(E.kernel_args(E.scene(name)))
        tied = np.flatnonzero(z == M)
        assert len(tied) == 2 and tied.min() >= first, (name, tied)
        part = (tied % stride) // OG.GB_THREADS
        assert part[0] != part[1], (name, part)
        assert OG.depth_grid(len(z)) == len(partials)
    assert len(z) < stride < 627200 == E.BIG_B * E.BIG_NF
    z, _, M = OG.face_depths(E.kernel_args(E.scene("big_nan_depth_nospec")))
    assert np.isnan(M) and (np.flatnonzero(np.isnan(z)) >= stride).all()


def test_zero_max_depth_is_positive_zero():
    """A zero max reached by both zeros: the emulation's fold in the kernels' order, and the float64 mirror's _TiedMax,
    both give +0 (IEEE maximum's +0 > -0), so every other face's z / M is -inf and clamps to 0."""
    sc = E.scene("zero_sign_depth_nospec")
    a = E.kernel_args(sc)
    z, _, M = OG.face_depths(a)
    zeros = z[z == 0]
    assert np.signbit(zeros).any() and not np.signbit(zeros).all()   # both signs in float32
    assert M == 0 and not np.signbit(M)
    assert np.signbit(OG.fold(np.float32([-0.0, 0.0]), 1, OG.nan_max, -np.inf)[0]) == np.False_
    assert not np.signbit(OG.nan_max(np.float32(-0.0), np.float32(0.0))) and \
        not np.signbit(OG.nan_max(np.float32(0.0), np.float32(-0.0)))
    from jrender_b200.lighting import _TiedMax
    for x in ([-0.0, 0.0, -1.0], [0.0, -0.0, -1.0], [-0.0, -2.0]):
        m = _TiedMax.apply(torch.tensor(x, dtype=torch.float64))
        assert m.item() == 0 and bool(torch.signbit(m)) == all(np.signbit(x) | (np.asarray(x) < 0)), x
    ts, light, mesh, eyes = E.build(sc, torch.device("cpu"), torch.float64, fused=False)
    out = light(mesh, eyes).textures.detach().numpy()
    want, _ = OG.gbuffer_forward(dict(a, mode=1))
    assert np.array_equal(np.isnan(out), np.isnan(want)) and (out[np.isfinite(want)] == want[np.isfinite(want)]).all()
    assert (want[np.isfinite(want)] == 0).all()
