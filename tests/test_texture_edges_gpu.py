"""The texture bake and atlas kernels on the hostile inputs of tests/texture_edge_cases.py, against the float32
emulation of their own arithmetic (oracle/bake.py, oracle/texture_atlas.py):
  - b200r_bake_textures_softras, b200r_bake_textures_n3mr (every wrap mode, both samplers) and both atlases: every
    output equal to the emulation as uint32 bit patterns, NaN compared by position; faces with is_update == 0 keep
    their input bits, NaN payloads included;
  - b200r_bake_textures_softras_backward: NaN and +-inf exactly where the emulated float32 terms put them, +0.0 where no
    non-zero term lands, every other entry within oracle/sss_grad.bake_bound of the exact adjoint; and the adjoint
    identity <bake(img), g> = <img, bake_bwd(g)> in float64 within the two sides' summed bounds;
  - the SSS path's bake of a 2048^2 map through the golden mesh's face_texcoords, bit for bit.
Prints the worst |got - exact| / bound per backward case."""
import os

import numpy as np
import pytest
import torch

from jrender_b200 import _lib
from jrender_b200 import io as jio
from oracle import bake as obake
from oracle import sss_grad as sg
from oracle import texture_atlas as oat
from tests import texture_edge_cases as tec

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
U = 2.0 ** -24
SOFTRAS = tec.softras_cases()
N3MR = tec.n3mr_cases()
ATLAS = tec.atlas_cases()


def check_bits(what, got, ref):
    """Bit for bit, NaN where ref is NaN (payloads may differ)."""
    got = np.asarray(got, np.float32)
    assert got.shape == ref.shape, what
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), (what, int((np.isnan(got) != nan).sum()))
    differ = got[~nan].view(np.uint32) != ref[~nan].view(np.uint32)
    assert not differ.any(), (what, int(differ.sum()), got[~nan][differ][:4], ref[~nan][differ][:4])


def _kept(what, got, c):
    keep = c["is_update"] == 0
    assert np.array_equal(got[keep].view(np.uint32), np.asarray(c["textures"], np.float32)[keep].view(np.uint32)), what


@pytest.mark.parametrize("c", SOFTRAS, ids=[c["name"] for c in SOFTRAS])
def test_softras_bake(c, cuda_device):
    got = jio.bake_textures_for_softras(c["image"], c["faces_uv"], c["textures"], c["is_update"], device=cuda_device).cpu().numpy()
    check_bits(c["name"], got, obake.bake_textures_for_softras(c["image"], c["faces_uv"], c["textures"], c["is_update"]))
    _kept(c["name"], got, c)


def _grad(c, seed):
    rng = np.random.default_rng(seed)
    g = rng.normal(size=c["textures"].shape).astype(np.float32)
    m = rng.random(g.shape)
    g[m < 0.1] = 0.0
    g[(m >= 0.1) & (m < 0.15)] = -0.0
    return g


def _backward(c, g, dev):
    nf, T = g.shape[:2]
    H, W = c["image"].shape[:2]
    gi = torch.empty((H, W, 3), device=dev)
    _lib.call("b200r_bake_textures_softras_backward", dev, torch.from_numpy(g).to(dev),
              torch.from_numpy(np.ascontiguousarray(c["faces_uv"])).to(dev), torch.from_numpy(c["is_update"]).to(dev), gi,
              nf, int(round(np.sqrt(T))), H, W)
    return gi.cpu().numpy()


@pytest.mark.parametrize("c", SOFTRAS, ids=[c["name"] for c in SOFTRAS])
def test_softras_bake_backward(c, cuda_device):
    g = _grad(c, 7)
    H, W = c["image"].shape[:2]
    R = int(round(np.sqrt(g.shape[1])))
    got = _backward(c, g, cuda_device)
    s = obake.softras_backward_sums(g, c["faces_uv"], c["is_update"], H, W)
    ex = s["exact"]
    for pattern in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(pattern(got), pattern(ex)), (c["name"], pattern.__name__)
    quiet = s["nonzero"] == 0                                   # no tap, or only +-0 terms: the zeroed +0.0 stays
    assert (got[quiet].view(np.uint32) == 0).all(), c["name"]
    gt = torch.from_numpy(g).to(cuda_device)
    want, _ = sg.bake_vjp(gt, c["faces_uv"], R, H, W, c["is_update"])
    bound = sg.bake_bound(gt, c["faces_uv"], R, H, W, c["is_update"]).cpu().numpy()
    fin = np.isfinite(ex)
    err = np.abs(got.astype(np.float64) - want.cpu().numpy())[fin]
    ratio = float((err / bound[fin]).max()) if err.size else 0.0
    print("%-36s backward worst |got - exact| / bound = %.3g" % (c["name"], ratio))
    assert np.all(err <= bound[fin]), (c["name"], ratio)


FINITE = [c for c in SOFTRAS if np.isfinite(c["image"]).all() and np.isfinite(c["faces_uv"]).all()]


@pytest.mark.parametrize("c", FINITE, ids=[c["name"] for c in FINITE])
def test_softras_adjoint_identity(c, cuda_device):
    """<bake(img), g> = <img, bake_bwd(g)> over the updated faces, both sides in float64 from the kernels' float32
    outputs: within 5 u sum_t |g_t| sum_j |px_j w_j| (four rounded products, three sums per texel) plus
    sum_p |img_p| bake_bound_p."""
    g = _grad(c, 11)
    upd = c["is_update"] != 0
    g[~upd] = 0
    H, W = c["image"].shape[:2]
    R = int(round(np.sqrt(g.shape[1])))
    fwd = jio.bake_textures_for_softras(c["image"], c["faces_uv"], c["textures"], c["is_update"], device=cuda_device).cpu().numpy()
    bwd = _backward(c, g, cuda_device)
    img = c["image"].astype(np.float64)
    lhs = float((fwd[upd].astype(np.float64) * g[upd]).sum())
    rhs = float((img * bwd).sum())
    idx, wts = obake.softras_taps(c["faces_uv"][upd], R, H, W)
    flat = img.reshape(-1, 3)
    fwd_mag = (np.abs(flat[idx]) * np.abs(wts.astype(np.float64))[..., None]).sum(2)
    bound = 5 * U * float((np.abs(g[upd]) * fwd_mag).sum())
    gt = torch.from_numpy(g).to(cuda_device)
    bound += float((np.abs(img) * sg.bake_bound(gt, c["faces_uv"], R, H, W, c["is_update"]).cpu().numpy()).sum())
    bound += 2.0 ** -50 * (abs(lhs) + abs(rhs) + 1)
    print("%-36s adjoint |lhs - rhs| / bound = %.3g" % (c["name"], abs(lhs - rhs) / bound))
    assert abs(lhs - rhs) <= bound, (c["name"], lhs, rhs, bound)


@pytest.mark.parametrize("bilinear", [True, False])
@pytest.mark.parametrize("wrap", range(4))
@pytest.mark.parametrize("c", N3MR, ids=[c["name"] for c in N3MR])
def test_n3mr_bake(c, wrap, bilinear, cuda_device):
    got = jio.bake_textures_for_n3mr(c["image"], c["faces_uv"], c["textures"], c["is_update"], wrap, bilinear,
                                     device=cuda_device).cpu().numpy()
    want = obake.bake_textures_for_n3mr(c["image"], c["faces_uv"], c["textures"], c["is_update"], wrap, bilinear)
    check_bits("%s wrap %d bilinear %s" % (c["name"], wrap, bilinear), got, want)
    _kept(c["name"], got, c)


@pytest.mark.parametrize("kind", ["softras", "n3mr"])
@pytest.mark.parametrize("c", ATLAS, ids=[c["name"] for c in ATLAS])
def test_atlas(c, kind, cuda_device):
    args = (c["tile_vertices"], c[kind], c["texture_res_out"], c["tile_width"], c["H"], c["W"])
    got = jio.texture_atlas(*args, device=cuda_device).cpu().numpy()
    want = (oat.texture_atlas_softras if kind == "softras" else oat.texture_atlas_n3mr)(*args)
    check_bits(c["name"] + " " + kind, got, want)


def test_sss_bake_2048(cuda_device):
    """The bake Lighting's SSS path runs (lighting.py: the 2048^2 final map into textures of ones) on the golden mesh's
    face_texcoords, with UVs of exactly 0 and 1 added."""
    g = np.load(os.path.join(G, "ref_host_sss.npz"))
    ftc = g["face_texcoords"][0].astype(np.float32)
    ftc = np.concatenate([ftc, np.float32([[[0, 0], [1, 1], [1, 0]], [[1, 1], [1, 1], [1, 1]]])])
    R = int(g["texture_res"])
    S = 2048
    img = np.random.default_rng(3).uniform(0, 1.5, (S, S, 3)).astype(np.float32)
    nf = ftc.shape[0]
    ones = np.ones((nf, R * R, 3), np.float32)
    upd = np.ones(nf, np.int32)
    got = jio.bake_textures_for_softras(torch.from_numpy(img).to(cuda_device), torch.from_numpy(ftc).to(cuda_device),
                                        torch.from_numpy(ones).to(cuda_device), torch.from_numpy(upd).to(cuda_device),
                                        device=cuda_device).cpu().numpy()
    check_bits("sss 2048", got, obake.bake_textures_for_softras(img, ftc, ones, upd))
