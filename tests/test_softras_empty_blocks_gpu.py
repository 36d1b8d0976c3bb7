"""Every output pixel of the SoftRas forward is written, whichever path wrote it.

The forward stores the constant outputs of blocks no face rectangle touches on the side of the shaded blocks (a share
of the empty list per shaded queue entry), hands what the shares leave to the atomic queue, and keeps empty blocks in
the shaded path where their constant stores do not apply (image sizes or K not a multiple of 4, the pooled
anti-aliasing epilogue).  Here the output buffers start as NaN / 0x7f7f7f7f instead of whatever the allocator returns,
so a pixel that no path wrote, or that two paths wrote differently, shows against the oracle: ids bit-exact, colours
within 2e-6, the aggregates as tests/test_softras_gpu.py holds them.
"""
import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests.test_softras_gpu import COLOR_ATOL, SUM_RTOL
from tests.util import run_oracle

pytestmark = pytest.mark.gpu

FILL_IDS = 0x7f7f7f7f


def run_prefilled(fv, tex, P, aa=False):
    """The forward through the C ABI into output buffers filled with NaN (floats) and 0x7f7f7f7f (ids)."""
    import torch
    from jrender_b200 import SoftRasterizeFunction, _lib
    from jrender_b200.softras import pad_face_ids
    dev = torch.device("cuda:0")
    fvt = torch.from_numpy(np.ascontiguousarray(fv)).to(dev)
    txt = torch.from_numpy(np.ascontiguousarray(tex)).to(dev)
    B, nf, T, H, K = fv.shape[0], fv.shape[1], tex.shape[2], P["image_size"], P["max_faces_per_pixel_for_grad"]
    fn = SoftRasterizeFunction(
        image_size=H, near=P["near"], far=P["far"], fill_back=P["fill_back"], eps=P["eps"], sigma_val=P["sigma_val"],
        dist_func=P["dist_func"], dist_eps=P["dist_eps"], gamma_val=P["gamma_val"], aggr_func_rgb=P["aggr_func_rgb"],
        aggr_func_alpha=P["aggr_func_alpha"], texture_type=P["texture_type"], max_faces_per_pixel_for_grad=K)
    L = _lib.lib()
    soft_colors = torch.full((B, 4, H, H), float("nan"), dtype=torch.float32, device=dev)
    aggrs_info = torch.full((B, 2, H, H), float("nan"), dtype=torch.float32, device=dev)
    ids = torch.full((B, K, H, H), FILL_IDS, dtype=torch.int32, device=dev)
    st_bytes = L.b200r_softras_state_bytes(B, nf)
    state = torch.empty((st_bytes,), dtype=torch.uint8, device=dev)
    ws_bytes = L.b200r_softras_workspace_bytes(B, nf, H)
    workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    scal = fn._scalars(B, nf, T)
    pooled = torch.full((B, 4, H // 2, H // 2), float("nan"), dtype=torch.float32, device=dev) if aa else None
    _lib.call("b200r_softras_forward_aa" if aa else "b200r_softras_forward", dev,
              fvt, txt, soft_colors, *((pooled,) if aa else ()), aggrs_info, ids, None, state, st_bytes, workspace,
              ws_bytes, *scal)
    torch.cuda.synchronize()
    out = dict(soft_colors=soft_colors.cpu().numpy(), aggrs_info=aggrs_info.cpu().numpy(), ids_raw=ids.cpu().numpy(),
               faces_id_buffer=pad_face_ids(ids).cpu().numpy())
    if aa:
        out["pooled"] = pooled.cpu().numpy()
    return out


def check_prefilled(fv, tex, P, aa=False):
    ref = run_oracle(fv, tex, P)
    got = run_prefilled(fv, tex, P, aa=aa)
    # slot 0 of every pixel is written: a face id or the list's -1 terminator
    assert not (got["ids_raw"][:, 0] == FILL_IDS).any(), "id plane 0 left unwritten"
    assert np.array_equal(got["faces_id_buffer"], ref["faces_id_buffer"]), "top-K ids not bit-exact"
    assert not np.isnan(got["soft_colors"]).any(), "soft_colors left unwritten"
    d = np.abs(got["soft_colors"] - ref["soft_colors"]).max()
    assert d <= COLOR_ATOL, "soft_colors max abs diff %g" % d
    assert not np.isnan(got["aggrs_info"]).any(), "aggrs_info left unwritten"
    if P["aggr_func_rgb"] == "softmax":
        assert np.array_equal(got["aggrs_info"][:, 1], ref["aggrs_info"][:, 1]), "softmax_max not bit-exact"
        assert np.allclose(got["aggrs_info"][:, 0], ref["aggrs_info"][:, 0], rtol=SUM_RTOL, atol=0)
    else:
        assert np.array_equal(got["aggrs_info"], ref["aggrs_info"]), "aggrs_info not bit-exact"
    if aa:   # avg_pool2d's order: window row-major, sum / 4
        s = got["soft_colors"]
        want = (((s[:, :, 0::2, 0::2] + s[:, :, 0::2, 1::2]) + s[:, :, 1::2, 0::2]) + s[:, :, 1::2, 1::2]) / np.float32(4)
        assert np.array_equal(got["pooled"], want), "pooled epilogue differs from the 2x2 mean of soft_colors"
    return got


MODES = {"softmax": dict(), "hard": dict(aggr_func_rgb="hard"), "silhouettes": dict(aggr_func_rgb="none")}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("is_", [1024, 1000, 36, 6])
@pytest.mark.parametrize("K", [16, 6])
def test_every_pixel_written(cuda_device, mode, is_, K):
    """Sizes whose blocks are cut by the image edge (36: 4.5 blocks per row; 6: not a multiple of 4), a K that is not a
    multiple of 4 (ids written per pixel, empty blocks in the shaded path), two cameras of one batch."""
    fv, tex = wl.make_scene(280, batch=2)
    check_prefilled(fv, tex, osr.Params(image_size=is_, max_faces_per_pixel_for_grad=K, sigma_val=3e-5, **MODES[mode]))


@pytest.mark.parametrize("mode", sorted(MODES))
def test_antialiasing_entry_point(cuda_device, mode):
    """b200r_softras_forward_aa: the pooled epilogue needs every block's staged outputs, so empty blocks stay shaded."""
    fv, tex = wl.make_scene(280, batch=2)
    check_prefilled(fv, tex, osr.Params(image_size=128, sigma_val=3e-5, **MODES[mode]), aa=True)


def _out_of_view(fv):
    fv = fv.copy()
    fv[..., 0] += 10.0   # every rectangle right of the image
    return fv


def _screen_quad(nf, z=2.0):
    """Two faces that cover the whole image (NDC [-1.5, 1.5]^2), padded with out-of-view copies to nf faces."""
    q = np.array([[[-1.5, -1.5, z], [1.5, -1.5, z], [1.5, 1.5, z]],
                  [[-1.5, -1.5, z], [1.5, 1.5, z], [-1.5, 1.5, z]]], np.float32)
    fv = np.repeat(q[:1], nf, 0) + np.float32([10.0, 0.0, 0.0])
    fv[:2] = q
    return fv


@pytest.mark.parametrize("mode", sorted(MODES))
def test_image_without_visible_face(cuda_device, mode):
    """Image 1 of the batch has no face in view: all its blocks are empty and stored through the other image's shares."""
    fv, tex = wl.make_scene(280, batch=2)
    fv[1] = _out_of_view(fv[1])
    got = check_prefilled(fv, tex, osr.Params(image_size=256, sigma_val=3e-5, **MODES[mode]))
    assert (got["ids_raw"][1, 0] == -1).all()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_batch_without_visible_face(cuda_device, mode):
    """No block of the batch is shaded: every empty block comes from the queue."""
    fv, tex = wl.make_scene(280, batch=2)
    check_prefilled(_out_of_view(fv), tex, osr.Params(image_size=256, sigma_val=3e-5, **MODES[mode]))


@pytest.mark.parametrize("mode", sorted(MODES))
def test_image_without_empty_block(cuda_device, mode):
    """Image 0 is covered by a full-screen quad (no empty block at all), image 1 is the sphere."""
    fv, tex = wl.make_scene(280, batch=2)
    fv[0] = _screen_quad(fv.shape[1])
    got = check_prefilled(fv, tex, osr.Params(image_size=256, sigma_val=3e-5, **MODES[mode]))
    assert (got["ids_raw"][0, 0] >= 0).all()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_small_object_leaves_empty_blocks_to_the_queue(cuda_device, mode):
    """A sphere ~50 pixels across in a 1024 image: far more empty blocks than the shaded blocks' shares hold, so the
    queue hands out the rest after the shaded blocks."""
    fv, tex = wl.make_scene(280, batch=2, distance=40.0)
    check_prefilled(fv, tex, osr.Params(image_size=1024, sigma_val=3e-5, **MODES[mode]))
