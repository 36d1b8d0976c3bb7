"""k_project_faces_fwd / _bwd, k_flatten_loss and k_laplacian_loss on the degenerate cameras and meshes of
geometry_edge_cases.py, through the C ABI and through project_faces / FlattenLoss / LaplacianLoss:
  - the forward face_vertices bit for bit equal to oracle/preraster.project_faces;
  - every gradient and loss entry within the summation-order bound of its emulated float32 terms (oracle term_sums);
  - NaN and +-inf exactly where the emulation puts them.
Prints the worst |got - exact| / bound of each tensor."""
import numpy as np
import pytest
import torch

import jrender_b200 as jr
from jrender_b200 import _lib, preraster
from oracle import mesh_loss as oml
from oracle import preraster as opr
from tests import geometry_edge_cases as gec
from tests.geometry_edge_cases import check_bits, check_sums

pytestmark = pytest.mark.gpu
PROJ = gec.projection_cases()
FLAT = gec.flatten_cases()
LAP = gec.laplacian_cases()


def _cam_args(kw):
    if kw.get("camera_mode", "look_at") == "look_at":
        mode, a = preraster.CAM_MODES["look_at"], kw.get("at", (0, 0, 0))
    else:
        mode, a = preraster.CAM_MODES["look_" + kw.get("coordinate", "right")], kw.get("direction", (0, 0, 1))
    persp = kw.get("perspective", True)
    width = preraster.perspective_width(kw.get("viewing_angle", 30.0)) if persp else float(kw.get("viewing_scale", 1.0))
    return (_lib._f3(a), _lib._f3(kw.get("up", (0, 1, 0))), width, mode, preraster.PROJECTIONS["perspective" if persp else "orthogonal"])


@pytest.mark.parametrize("c", PROJ, ids=[c["name"] for c in PROJ])
def test_projection_edges(c, cuda_device):
    v, f, eye, g, kw = c["vertices"], c["faces"], c["eye"], c["grad"], c["kw"]
    B, nf = g.shape[:2]
    ref = opr.project_faces(v, f, eye, **kw)
    sums = opr.project_faces_bwd_sums(v, f, eye, g, **kw)
    vt, ft, et, gt = (torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device) for a in (v, f, eye, g))
    # the C ABI
    out = torch.empty((B, nf, 3, 3), device=cuda_device)
    gv = torch.empty_like(vt)
    dims = (B, v.shape[1], nf, v.shape[0], f.shape[0], eye.shape[0])
    _lib.call("b200r_project_faces_forward", cuda_device, vt, ft, et, out, *_cam_args(kw), *dims)
    _lib.call("b200r_project_faces_backward", cuda_device, vt, ft, et, gt, gv, *_cam_args(kw), *dims)
    check_bits(c["name"] + " abi forward", out.cpu().numpy(), ref)
    check_sums(c["name"] + " abi grad_vertices", gv.cpu().numpy(), sums)
    # project_faces
    vr = vt.clone().requires_grad_(True)
    fv = preraster.project_faces(vr, ft, et, **kw)
    fv.backward(gt)
    check_bits(c["name"] + " api forward", fv.detach().cpu().numpy(), ref)
    check_sums(c["name"] + " api grad_vertices", vr.grad.cpu().numpy(), sums)


def test_int64_indices_outside_int32_poison_their_corner(cuda_device):
    """2^32 + 1 would wrap to vertex 1 in a plain int32 cast: it must poison its corner and add no gradient."""
    v = torch.randn(1, 4, 3, device=cuda_device).requires_grad_(True)
    f = torch.tensor([[[0, 2 ** 32 + 1, 2], [3, 2, 0]]], dtype=torch.int64, device=cuda_device)
    fv = preraster.project_faces(v, f, [0.0, 0.0, -3.0])
    assert torch.isnan(fv[0, 0, 1]).all() and not torch.isnan(fv[0, 0, 0]).any() and not torch.isnan(fv[0, 1]).any()
    torch.nan_to_num(fv, nan=0.0).sum().backward()
    assert (v.grad[0, 1] == 0).all() and (v.grad[0, 0] != 0).all()
    mesh = jr.Mesh(v.detach(), f[0].cpu().numpy())
    assert mesh.faces[0, 0].tolist() == [0, -1, 2]


@pytest.mark.parametrize("c", FLAT, ids=[c["name"] for c in FLAT])
def test_flatten_edges(c, cuda_device):
    x, edges, eps = c["vertices"], c["edges"], c["eps"]
    B, nv = x.shape[:2]
    E = len(edges[0])
    s = oml.flatten_sums(x, edges, eps)
    xt = torch.from_numpy(x).to(cuda_device)
    et = [torch.from_numpy(np.ascontiguousarray(e, np.int32) if E else np.zeros(1, np.int32)).to(cuda_device) for e in edges]
    loss = torch.empty(B, device=cuda_device)
    grad = torch.empty_like(xt)
    _lib.call("b200r_flatten_loss", cuda_device, xt, *et, loss, grad, B, nv, E, float(eps))
    check_sums(c["name"] + " abi loss", loss.cpu().numpy(), s["loss"])
    check_sums(c["name"] + " abi grad", grad.cpu().numpy(), s["grad"])
    if c["faces"] is not None:
        mod = jr.FlattenLoss(torch.from_numpy(c["faces"])).to(cuda_device)
        xr = xt.clone().requires_grad_(True)
        val = mod(xr, eps=eps)
        val.sum().backward()
        check_sums(c["name"] + " api loss", val.detach().cpu().numpy(), s["loss"])
        check_sums(c["name"] + " api grad", xr.grad.cpu().numpy(), s["grad"])


@pytest.mark.parametrize("c", LAP, ids=[c["name"] for c in LAP])
def test_laplacian_edges(c, cuda_device):
    x = c["vertices"]
    B, nv = x.shape[:2]
    mod = jr.LaplacianLoss(torch.from_numpy(x[0]), torch.from_numpy(c["faces"]))
    s = oml.laplacian_sums(x, mod.nbr32.numpy(), mod.nbr_w.numpy(), mod.diag.numpy())
    mod = mod.to(cuda_device)
    xt = torch.from_numpy(x).to(cuda_device)
    loss = torch.empty(B, device=cuda_device)
    grad = torch.empty_like(xt)
    _lib.call("b200r_laplacian_loss", cuda_device, xt, mod.nbr32, mod.nbr_w, mod.diag, loss, grad, B, nv, mod.nbr_w.shape[1])
    check_sums(c["name"] + " abi loss", loss.cpu().numpy(), s["loss"])
    check_sums(c["name"] + " abi grad", grad.cpu().numpy(), s["grad"])
    xr = xt.clone().requires_grad_(True)
    val = mod(xr)
    val.sum().backward()
    check_sums(c["name"] + " api loss", val.detach().cpu().numpy(), s["loss"])
    check_sums(c["name"] + " api grad", xr.grad.cpu().numpy(), s["grad"])
