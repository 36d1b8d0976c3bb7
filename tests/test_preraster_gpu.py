"""GPU parity tests of the fused pre-raster geometry stage (csrc/preraster_api.cu) through the
C ABI: forward bit for bit against the CPU oracle and within a float tolerance of the reference-Python
goldens, backward within the summation-order bound of the oracle's emulated per-corner terms,
Transform/Renderer fused path against the op-by-op mirror, CUDA graphs."""
import glob
import os

import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import preraster, workloads as wl
from oracle import preraster as opr
from tests.geometry_edge_cases import check_bits, check_sums

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ref_host_transform_*.npz")))
FWD_TOL = 2e-6   # of max |face_vertices| (same bound the oracle holds against the reference's Python)
BWD_TOL = 2e-5   # of max |grad|: fused kernel vs the op-by-op mirror (different operation order)


def _kw(g):
    return dict(camera_mode=str(g["camera_mode"]), direction=[float(x) for x in g["direction"]], up=[float(x) for x in g["up"]],
                coordinate=str(g["coordinate"]), perspective=bool(g["perspective"]), viewing_angle=float(g["viewing_angle"]),
                viewing_scale=float(g["viewing_scale"]))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[19:-4] for p in GOLDEN])
def test_fused_forward_backward_match_oracle_and_golden(path, cuda_device):
    g = np.load(path)
    kw = _kw(g)
    v = torch.from_numpy(g["vertices"]).to(cuda_device).requires_grad_(True)
    f = torch.from_numpy(g["faces"]).to(cuda_device)
    eye = torch.from_numpy(g["eye"]).to(cuda_device)
    fv = preraster.project_faces(v, f, eye, **kw)
    ref = opr.project_faces(g["vertices"], g["faces"], g["eye"], **kw)
    got = fv.detach().cpu().numpy()
    check_bits("forward", got, ref)
    assert np.abs(got - g["face_vertices"]).max() <= FWD_TOL * np.abs(ref).max()
    go = np.random.default_rng(5).normal(0, 1, ref.shape).astype(np.float32)
    fv.backward(torch.from_numpy(go).to(cuda_device))
    check_sums("grad_vertices", v.grad.cpu().numpy(), opr.project_faces_bwd_sums(g["vertices"], g["faces"], g["eye"], go, **kw))


def test_fused_shared_mesh_and_list_eye(cuda_device):
    v, f = wl.sphere_by_faces(3280)
    eyes = np.asarray([wl.get_points_from_angles(2.732, 30.0, 45.0 * b) for b in range(8)], np.float32)
    vt = torch.from_numpy(v)[None].to(cuda_device).requires_grad_(True)          # [1, nv, 3] shared by 8 views
    fv = preraster.project_faces(vt, torch.from_numpy(f).to(cuda_device), torch.from_numpy(eyes).to(cuda_device))
    ref = opr.project_faces(v[None], f[None], eyes)
    assert fv.shape == (8, 3280, 3, 3)
    check_bits("forward", fv.detach().cpu().numpy(), ref)
    go = np.random.default_rng(6).normal(0, 1, ref.shape).astype(np.float32)
    fv.backward(torch.from_numpy(go).to(cuda_device))
    assert vt.grad.shape == (1, v.shape[0], 3)
    check_sums("grad_vertices", vt.grad.cpu().numpy(), opr.project_faces_bwd_sums(v[None], f[None], eyes, go))
    # Python-list eye (Transform's default) broadcast over the batch
    one = preraster.project_faces(vt.detach(), torch.from_numpy(f).to(cuda_device), [0.0, 0.0, -2.732])
    check_bits("list eye", one.cpu().numpy(), opr.project_faces(v[None], f[None], np.float32([[0.0, 0.0, -2.732]])))


def test_out_of_range_index_poisons_only_that_corner(cuda_device):
    v = torch.randn(1, 10, 3, device=cuda_device)
    f = torch.tensor([[[0, 1, 2], [3, 99, 4], [5, -1, 6]]], dtype=torch.int32, device=cuda_device)
    fv = preraster.project_faces(v.requires_grad_(True), f, [0.0, 0.0, -3.0])
    bad = torch.isnan(fv).any(dim=-1)[0].cpu().numpy()
    assert bad.tolist() == [[False, False, False], [False, True, False], [False, True, False]]
    torch.nan_to_num(fv, nan=0.0).sum().backward()
    assert torch.isfinite(v.grad).all()


def test_transform_fused_equals_op_by_op_mirror(cuda_device):
    v, f = wl.sphere_by_faces(280)
    eyes = torch.from_numpy(np.asarray([wl.get_points_from_angles(2.732, 30.0, 120.0 * b) for b in range(3)], np.float32)).to(cuda_device)
    out = {}
    for fused in (True, False):
        jr.Transform.fused = fused
        try:
            vt = torch.from_numpy(v)[None].repeat(3, 1, 1).to(cuda_device).requires_grad_(True)
            mesh = jr.Mesh(vt, torch.from_numpy(f)[None].repeat(3, 1, 1).to(cuda_device))
            r = jr.Renderer(image_size=64, camera_mode='look_at', sigma_val=1e-4)
            r.transform.set_eyes(eyes)
            mesh = r.transform(r.lighting(mesh, r.transform.eyes))
            fv = mesh.face_vertices
            cam = mesh.vertices            # lazily evaluated on the fused path
            (fv * fv).sum().backward()
            out[fused] = (fv.detach().cpu().numpy(), cam.detach().cpu().numpy(), vt.grad.cpu().numpy())
        finally:
            jr.Transform.fused = True
    for a, b, tol in zip(out[True], out[False], (FWD_TOL, FWD_TOL, BWD_TOL)):
        assert np.abs(a - b).max() <= tol * np.abs(b).max()


def test_renderer_end_to_end_fused_vs_mirror_images(cuda_device):
    v, f = wl.sphere_by_faces(280)
    imgs = {}
    for fused in (True, False):
        jr.Transform.fused = fused
        try:
            mesh = jr.Mesh(torch.from_numpy(v)[None].to(cuda_device), torch.from_numpy(f)[None].to(cuda_device))
            r = jr.Renderer(image_size=64, camera_mode='look_at', sigma_val=1e-4)
            r.transform.set_eyes_from_angles(2.732, 30.0, 40.0)
            imgs[fused] = r.render_mesh(mesh, mode='rgb').cpu().numpy()
        finally:
            jr.Transform.fused = True
    # face_vertices differ by <= 1 ulp-ish between the two paths; colours move by ~1e-3 at most where a
    # pixel sits on a soft edge (sigma 1e-4), and not at all in the mean
    assert np.abs(imgs[True] - imgs[False]).max() < 5e-3
    assert abs(float(imgs[True].mean()) - float(imgs[False].mean())) < 1e-5


def test_project_faces_cuda_graph_replay(cuda_device):
    v, f = wl.sphere_by_faces(280)
    vt = torch.from_numpy(v)[None].to(cuda_device).requires_grad_(True)
    ft = torch.from_numpy(f)[None].to(cuda_device)
    eye = torch.tensor([[0.0, 0.0, -2.732]], device=cuda_device)
    go = torch.ones(1, 280, 3, 3, device=cuda_device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            vt.grad = None
            preraster.project_faces(vt, ft, eye).backward(go)
    torch.cuda.current_stream().wait_stream(s)
    eager = vt.grad.clone()
    graph = torch.cuda.CUDAGraph()
    vt.grad = None
    with torch.cuda.graph(graph):
        out = preraster.project_faces(vt, ft, eye)
        out.backward(go)
    with torch.no_grad():
        eye.copy_(torch.tensor([[1.0, 0.5, -2.5]], device=cuda_device))
    graph.replay()
    torch.cuda.synchronize()
    check_bits("replay", out.detach().cpu().numpy(), opr.project_faces(v[None], f[None], np.float32([[1.0, 0.5, -2.5]])))
    assert not torch.equal(vt.grad, eager)


def test_silhouette_render_skips_lighting_without_changing_alpha(cuda_device):
    """Renderer.skip_unused_lighting: mode='silhouettes' never reads a texture value, so leaving the lighting ops
    out must give the same alpha bits and the same vertex gradient as the reference's always-light order."""
    v, f = wl.sphere_by_faces(280)
    res = {}
    for skip in (True, False):
        jr.Renderer.skip_unused_lighting = skip
        try:
            vt = torch.from_numpy(v)[None].to(cuda_device).requires_grad_(True)
            mesh = jr.Mesh(vt, torch.from_numpy(f)[None].to(cuda_device))
            r = jr.Renderer(image_size=64, camera_mode='look_at', sigma_val=1e-4, aggr_func_rgb='hard')
            r.transform.set_eyes_from_angles(2.732, 20.0, 75.0)
            a = r.render_mesh(mesh, mode='silhouettes')
            a.sum().backward()
            res[skip] = (a.detach().cpu().numpy(), vt.grad.cpu().numpy(), mesh.textures.detach().cpu().numpy())
        finally:
            jr.Renderer.skip_unused_lighting = True
    assert np.array_equal(res[True][0], res[False][0])
    assert np.abs(res[True][1] - res[False][1]).max() <= BWD_TOL * np.abs(res[False][1]).max()
    assert np.all(res[True][2] == 1.0) and not np.all(res[False][2] == 1.0)   # the documented side-effect difference
