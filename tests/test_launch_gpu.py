"""Launch accounting of the C ABI: every kernel the library launches goes through one launcher, which counts it in
b200r_launch_count and times it under exactly one profiler id (include/b200raster.h, B200R_K_*).  So over any sequence
of calls the launch-count delta equals the sum of the profiler's per-id launch counts."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib, preraster, workloads as wl
from oracle import softras as osr
from oracle import voxelize as ov
from tests.conftest import ROOT
from tests.util import nmr_scene, run_cuda, run_nmr_cuda

pytestmark = pytest.mark.gpu


def kernel_id_count():
    """B200R_K_COUNT: one past the last B200R_K_* id of the header's enum."""
    src = open(os.path.join(ROOT, "include", "b200raster.h")).read()
    enum = re.search(r"enum \{ (B200R_K_\w+ = 0,[^}]*)\}", src).group(1)
    ids = [int(v) for v in re.findall(r"B200R_K_\w+ = (\d+)", enum)]
    assert enum.rstrip().endswith("B200R_K_COUNT") and ids == list(range(len(ids)))
    return len(ids)


def softras(dev):
    fv, tex = wl.make_scene(280, batch=2)
    g = np.random.default_rng(0).uniform(-1, 1, (2, 4, 64, 64)).astype(np.float32)
    run_cuda(fv, tex, osr.Params(image_size=64), grad=g, want_faces_info=False)


def nmr(dev):
    faces, tex = nmr_scene(280, batch=1, ts=2)
    rng = np.random.default_rng(1)
    g = (rng.uniform(-1, 1, (1, 64, 64, 3)).astype(np.float32), rng.uniform(-1, 1, (1, 64, 64)).astype(np.float32),
         rng.uniform(-1, 1, (1, 64, 64)).astype(np.float32))
    run_nmr_cuda(faces, tex, 64, flags=(True, True, True), grads=g)


def voxelization(dev):
    faces = ov.mesh_voxelize_faces(ov.sphere_faces(280, radius=0.45, jitter=0.02), 16)
    jr.voxelization(torch.from_numpy(faces).to(dev), 16)


def lighting(dev):
    v, f = wl.sphere_by_faces(280)
    vt = torch.from_numpy(v)[None].to(dev).requires_grad_(True)
    tt = torch.rand(1, f.shape[0], 4, 3, device=dev).requires_grad_(True)
    m = jr.Mesh(vt, torch.from_numpy(f)[None].to(dev), textures=tt)
    light = jr.Lighting()
    assert light._fusable(m, None)
    light(m).textures.sum().backward()


def project_faces(dev):
    v, f = wl.sphere_by_faces(280)
    vt = torch.from_numpy(v)[None].to(dev).requires_grad_(True)
    preraster.project_faces(vt, torch.from_numpy(f).to(dev), [0.0, 0.0, -2.732]).sum().backward()


def profiled(L, run, dev):
    """(b200r_launch_count delta, per-id profiler launch counts) over run(dev)."""
    torch.cuda.synchronize()
    L.b200r_profile_reset()
    L.b200r_profile_enable(1)
    try:
        n0 = L.b200r_launch_count()
        run(dev)
        torch.cuda.synchronize()
        delta = L.b200r_launch_count() - n0
    finally:
        L.b200r_profile_enable(0)
    counts = []
    for k in range(kernel_id_count()):
        n = C.c_longlong(0)
        assert L.b200r_profile_read(k, None, C.byref(n)) == 0
        counts.append(n.value)
    assert L.b200r_profile_read(kernel_id_count(), None, None) == -1   # the profiler's table ends where the enum does
    return delta, counts


@pytest.mark.parametrize("run", [softras, nmr, voxelization, lighting, project_faces], ids=lambda f: f.__name__)
def test_every_launch_is_counted_and_profiled_once(cuda_device, run):
    L = _lib.lib()
    run(cuda_device)                       # warm up: library load, one-time kernel attributes
    delta, counts = profiled(L, run, cuda_device)
    assert delta > 0 and delta == sum(counts), (delta, counts)


def test_softras_forward_backward_launches_seven_kernels(cuda_device):
    """face setup, chunk rectangles, coarse binning, tile order, forward; backward lanes, finalize."""
    L = _lib.lib()
    softras(cuda_device)
    delta, counts = profiled(L, softras, cuda_device)
    assert delta == 7
    assert [counts[k] for k in (0, 20, 1, 4, 2, 3, 9)] == [1] * 7, counts


ROUTES = ("_fused_surface", "_fused_normal_mapped", "_fused_gbuffer", "_fused_normal_mapped_gbuffer")


@pytest.mark.parametrize("route,gbuffer,kernel,launches", [
    ("_fused_surface", 'None', "_FusedSurfaceLighting", 1),
    ("_fused_normal_mapped", 'None', "_FusedNormalMappedLighting", 1),
    ("_fused_gbuffer", 'normal', "_FusedGbuffer", 1),
    ("_fused_gbuffer", 'depth', "_FusedGbuffer", 2),   # the depth pass, then the G-buffer
    ("_fused_normal_mapped_gbuffer", 'normal', "_FusedNormalMappedGbuffer", 1)])
def test_each_fused_lighting_route_launches_its_kernel(cuda_device, route, gbuffer, kernel, launches):
    """Lighting's fused dispatcher on each kernel's route: asked by that route's name it returns the kernel's result,
    from `launches` forward and as many backward launches, all under B200R_K_LIGHTING; the other routes' names
    return None on the same inputs."""
    from jrender_b200 import lighting
    dev = cuda_device
    v, f = wl.sphere_by_faces(280)
    nf = f.shape[0]
    g = torch.Generator().manual_seed(0)
    kw = {}
    if "normal_mapped" in route:
        n = torch.nn.functional.normalize(torch.rand(1, nf, 4, 3, generator=g) - 0.5 + torch.tensor([0., 0., 1.]), dim=3)
        tbn = torch.eye(3)[None, None].repeat(1, nf, 1, 1) + 0.1 * torch.rand(1, nf, 3, 3, generator=g)
        kw = dict(normal_textures=n.to(dev).requires_grad_(True), TBN=tbn.to(dev))
    m = jr.Mesh(torch.from_numpy(v)[None].to(dev).requires_grad_(True), torch.from_numpy(f)[None].to(dev),
                textures=torch.rand(1, nf, 4, 3, generator=g).to(dev).requires_grad_(True), texture_res=2, **kw)
    eyes = torch.tensor([[0.3, 0.4, -2.5]], device=dev)
    tr = jr.Transform(camera_mode='look_at')
    tr.set_eyes(eyes)
    light = jr.Lighting(Gbuffer=gbuffer, transform=tr)
    for other in ROUTES:
        if other != route:
            assert getattr(light, other)(m, eyes) is None, other
    L = _lib.lib()
    out = []
    fwd = lambda dev: out.append(getattr(light, route)(m, eyes))
    fwd(dev)                               # warm up
    delta, counts = profiled(L, fwd, dev)
    assert out[-1] is not None and type(out[-1].grad_fn)._forward_cls is getattr(lighting, kernel)
    assert delta == counts[15] == sum(counts) == launches, (delta, counts)   # B200R_K_LIGHTING
    delta, counts = profiled(L, lambda dev: out[-1].sum().backward(), dev)
    assert delta == counts[15] == sum(counts) == launches, (delta, counts)
