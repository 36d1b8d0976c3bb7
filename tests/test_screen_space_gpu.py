"""GPU tests of the render2 screen-space passes (jrender_b200/render2.py, csrc/screen_space_api.cu): SSAO_cuda, SSDO_cuda
and FXAA_cuda against the reference's own kernels (oracle/_ref, built by oracle/build_ref_screen.py), bit for bit with
the same NaN pattern, or against the committed goldens tests/golden/ref_screen_*.npz where oracle/_ref is absent.

Inputs: spot on a ground plane at 256^2 and 1024^2 and a 39 200-face sphere on the plane at 1024^2 (the G-buffers of
examples/render_ssao.py); 333^2, 1000^2, 1^2 and 2^2; an all-background buffer; random G-buffers whose samples wrap
across rows and project behind the camera; for FXAA hard-edged renders, uniform noise, constant images and NaN / +-inf
pixels.  Also: SSAO -> conv_for_image -> FXAA replays in a CUDA graph, and a call allocates nothing but its output.
"""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

from jrender_b200 import _lib, workloads as wl
from jrender_b200.render2 import FXAA_cuda, SSAO_cuda, SSDO_cuda, conv_for_image
from oracle import build_ref_screen

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ref():
    return build_ref_screen.lib()


def same(got, want):
    """Bit-identical, NaN where the other is NaN (any payload)."""
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype == torch.float32
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), "NaN pattern differs at %d entries" % int((gn != wn).sum())
    gb, wb = got.view(torch.int32), want.view(torch.int32)
    bad = (gb != wb) & ~gn
    assert not bad.any(), "%d of %d entries differ, e.g. %s vs %s" % (
        int(bad.sum()), bad.numel(), got[bad][:4].tolist(), want[bad][:4].tolist())


def check_all(L, depth, face_ind, normal, width, color, samples=(16,), radius=0.15):
    for n in samples:
        same(SSAO_cuda(depth, face_ind, normal, width, n, radius),
             build_ref_screen.ssao(L, depth, face_ind, normal, width, n, radius))
        same(SSDO_cuda(color, depth, face_ind, normal, width, n, radius),
             build_ref_screen.ssdo(L, color, depth, face_ind, normal, width, n, radius))
    same(FXAA_cuda(color), build_ref_screen.fxaa(L, color))


def need(L):
    if L is None:
        pytest.skip("oracle/_ref/libjrender_ref_screen.so not built; the goldens are checked by test_goldens")


def scene(size, mesh="spot"):
    from examples.render_ssao import gbuffers, ground_plane, shade
    from examples.render_gbuffers import load_spot
    dev = torch.device("cuda")
    if mesh == "spot":
        v, f = load_spot(dev)
    else:
        v, f = wl.sphere_by_faces(39200, radius=0.5)
        v, f = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    depth, face_ind, normal, width = gbuffers(*ground_plane(v, f), size)
    return depth, face_ind, normal, width, shade(face_ind, normal)


@pytest.mark.parametrize("size,mesh,samples", [(256, "spot", (1, 64)), (1024, "spot", (256,)), (1024, "sphere", (64,)),
                                               (333, "spot", (32,)), (1000, "spot", (16,)), (2, "spot", (16,)),
                                               (1, "spot", (16,))])
def test_scenes_match_reference(ref, size, mesh, samples):
    need(ref)
    depth, face_ind, normal, width, color = scene(size, mesh)
    check_all(ref, depth, face_ind, normal, width, color, samples)


def test_single_covered_pixel_matches_reference(ref):
    need(ref)
    dev = torch.device("cuda")
    depth = torch.full((1, 1), 2.0, device=dev)
    face_ind = torch.zeros((1, 1), dtype=torch.int32, device=dev)
    normal = torch.tensor([[[0.0, 0.0, -1.0]]], device=dev)
    check_all(ref, depth, face_ind, normal, 0.5, torch.full((1, 1, 3), 0.5, device=dev), (0, 1, 33))


def test_all_background_matches_reference(ref):
    need(ref)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    depth = torch.rand((96, 96), device=dev, generator=g) * 4
    face_ind = torch.full((96, 96), -1, dtype=torch.int32, device=dev)
    normal = torch.rand((96, 96, 3), device=dev, generator=g) - 0.5
    color = torch.rand((96, 96, 3), device=dev, generator=g)
    check_all(ref, depth, face_ind, normal, 0.6, color, (16,))
    assert torch.equal(SSDO_cuda(color, depth, face_ind, normal, 0.6, 16, 0.2), color)
    assert not SSAO_cuda(depth, face_ind, normal, 0.6, 16, 0.2).any()


@pytest.mark.parametrize("size", [64, 333])
def test_wrapping_and_behind_camera_samples_match_reference(ref, size):
    """Random G-buffers with depths near 0 and of both signs and a sample radius of several units, so samples land off
    the left and right edges (and wrap into the neighbouring row), off the top and bottom, and behind the camera
    (projections through z <= 0 that saturate the float-to-int conversion); unnormalised and zero normals."""
    need(ref)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(size)
    depth = (torch.rand((size, size), device=dev, generator=g) - 0.3) * 0.8
    face_ind = torch.randint(-1, 50, (size, size), dtype=torch.int32, device=dev, generator=g)
    normal = (torch.rand((size, size, 3), device=dev, generator=g) - 0.5) * 3
    normal[:3] = 0
    color = torch.rand((size, size, 3), device=dev, generator=g)
    for radius in (0.5, 4.0):
        check_all(ref, depth, face_ind, normal, 1.3, color, (24,), radius)
    occ = SSAO_cuda(depth, face_ind, normal, 1.3, 24, 4.0)
    assert torch.isfinite(occ).all()


@pytest.mark.parametrize("size", [7, 256, 1000])
def test_fxaa_inputs_match_reference(ref, size):
    need(ref)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(size)
    noise = torch.rand((size, size, 3), device=dev, generator=g)
    bad = noise.clone().reshape(-1)
    k = torch.randperm(bad.numel(), device=dev, generator=g)[:max(3, bad.numel() // 50)]
    bad[k[0::3]] = float("nan")
    bad[k[1::3]] = float("inf")
    bad[k[2::3]] = -float("inf")
    yy, xx = torch.meshgrid(torch.arange(size, device=dev), torch.arange(size, device=dev), indexing="ij")
    edges = (((xx // 5 + yy // 3) % 2 == 0) | (xx * 3 > yy * 7)).float()[..., None] * torch.tensor([0.9, 0.2, 0.6], device=dev)
    for img in (noise, bad.reshape(size, size, 3), edges, torch.zeros_like(noise), torch.full_like(noise, 0.73),
                torch.full_like(noise, float("inf"))):
        same(FXAA_cuda(img), build_ref_screen.fxaa(ref, img))


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(G, "ref_screen_*.npz"))), ids=os.path.basename)
def test_goldens(path):
    z = np.load(path)
    dev = torch.device("cuda")
    t = {k: torch.from_numpy(z[k]).to(dev) for k in ("depth", "face_ind", "normal", "color")}
    args = (float(z["width"]), int(z["sample_num"]), float(z["sample_range_r"]))
    same(SSAO_cuda(t["depth"], t["face_ind"], t["normal"], *args), torch.from_numpy(z["ssao"]))
    same(SSDO_cuda(t["color"], t["depth"], t["face_ind"], t["normal"], *args), torch.from_numpy(z["ssdo"]))
    for k in ("render", "noise", "const", "nonfinite"):
        same(FXAA_cuda(torch.from_numpy(z["fxaa_in_" + k]).to(dev)), torch.from_numpy(z["fxaa_out_" + k]))


def test_draws_are_the_reference_streams(ref):
    """The goldens' draws are what the reference's states give; the product draws them in its own kernel."""
    need(ref)
    for path in sorted(glob.glob(os.path.join(G, "ref_screen_*.npz"))):
        z = np.load(path)
        n = z["depth"].shape[0]
        d = build_ref_screen.draws(ref, n, z["draws"].shape[1], torch.device("cuda"))
        assert np.array_equal(d.cpu().numpy(), z["draws"])


def test_graph_replay_and_no_state_allocation():
    """SSAO -> conv_for_image -> FXAA captured in one CUDA graph replays to the eager results; a call allocates its
    output and nothing else (no per-pixel random state), and launches one kernel."""
    depth, face_ind, normal, width, color = scene(256)
    torch.cuda.synchronize()

    def chain():
        occ = SSAO_cuda(depth, face_ind, normal, width, 32, 0.15)
        ao = conv_for_image(1 - occ, torch.ones(5, 5, device=occ.device) / 25, 0)
        return FXAA_cuda(color * ao[..., None])

    eager = chain()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = chain()
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        same(out, eager)

    L = _lib.lib()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    n0 = L.b200r_launch_count()
    occ = SSAO_cuda(depth, face_ind, normal, width, 16, 0.15)
    img = SSDO_cuda(color, depth, face_ind, normal, width, 16, 0.15)
    torch.cuda.synchronize()
    assert L.b200r_launch_count() - n0 == 2
    outputs = occ.untyped_storage().nbytes() + img.untyped_storage().nbytes()
    assert torch.cuda.max_memory_allocated() - base == outputs
    # the entry points themselves, into preallocated outputs (every kernel is loaded by now): device memory unchanged
    d, f, n, c = depth.contiguous(), face_ind.contiguous(), normal.contiguous(), color.contiguous()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    _lib.call("b200r_ssao", d.device, d, f, n, occ, d.shape[0], 64, 0.15, width)
    _lib.call("b200r_ssdo", d.device, c, d, f, n, img, d.shape[0], 64, 0.15, width)
    _lib.call("b200r_fxaa", d.device, c, img, d.shape[0])
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def test_launches_are_profiled_under_one_id(cuda_device):
    L = _lib.lib()
    depth, face_ind, normal, width, color = scene(64)
    torch.cuda.synchronize()
    L.b200r_profile_reset()
    L.b200r_profile_enable(1)
    try:
        SSAO_cuda(depth, face_ind, normal, width, 8, 0.15)
        SSDO_cuda(color, depth, face_ind, normal, width, 8, 0.15)
        FXAA_cuda(color)
        torch.cuda.synchronize()
    finally:
        L.b200r_profile_enable(0)
    n = C.c_longlong(0)
    assert L.b200r_profile_read(25, None, C.byref(n)) == 0 and n.value == 3   # B200R_K_SSS, the image passes
