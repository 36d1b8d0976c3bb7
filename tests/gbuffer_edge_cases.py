"""Scenes for the G-buffer tests (tests/test_gbuffer_gpu.py): both modes with and without the specular branch, 6-D
textures, exact depth ties, axis-aligned faces (a normal component of +-1 puts the clamp at equality), every face behind
the camera (M < 0) and a largest depth of exactly 0 (M = 0), a sliver in depth mode, batches of one, vertices, faces and
eyes shared over a batch of two (batch 1 broadcast), NaN / +-inf at the vertices, the specular eye, the camera eye,
metallic, roughness and the normal textures, and the normal-map path."""
import numpy as np
import torch

import jrender_b200 as jr
from jrender_b200 import workloads as wl

LIGHT = dict(intensity_ambient=0.4, color_ambient=[1.0, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1.0, 0.7], directions=[0.3, 0.8, -0.5])


def _sphere(rng, B=2, nf=280):
    v, f = wl.sphere_by_faces(nf)
    return (v[None] + rng.normal(0, 0.02, (1,) + v.shape)).astype(np.float32).repeat(B, 0), f


def scene(name):
    rng = np.random.default_rng(sum(name.encode()))
    mode = "depth" if "depth" in name else "normal"
    B = 1 if "b1" in name else 2
    cam_eye = np.float32([[0.4, 0.6, -2.6], [1.0, 1.2, -2.2]])[:B]
    if name.startswith("ties"):
        # faces mirrored about the plane x = 0 seen by a camera on the z axis: equal depths, the max tied
        v = np.float32([[[-1, 0, 1], [0, 1, 1], [0, -1, 1], [1, 0, 1], [0.3, 0.2, 0.4], [-0.3, 0.2, 0.4]]]).repeat(B, 0)
        f = np.int32([[0, 1, 2], [3, 2, 1], [4, 5, 1]])
        cam_eye = np.float32([[0, 0, -3]] * B)
    elif name.startswith("axis"):
        v = np.float32([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0]]]).repeat(B, 0)
        f = np.int32([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 4, 2]])
    elif name.startswith("sliver"):
        v, f = _sphere(rng, B)
        v[:, f[:7, 2]] = v[:, f[:7, 0]] + np.float32(1e-3) * (v[:, f[:7, 1]] - v[:, f[:7, 0]])
    else:
        v, f = _sphere(rng, B)
    if name.startswith("behind"):
        cam_eye = np.float32([[0, 0, 3]] * B)
        v = v.copy()
        v[..., 2] += 4.5   # the camera looks at the origin along -z: every centroid behind it, z in [-2.4, -0.6], M < 0
    if name.startswith("zero_max"):
        # a camera on the z axis looking along +z, the sphere behind it and one face through the eye's plane z = -3: that
        # face's depth is exactly 0 and the largest, M = 0 (0 / 0 for it, -inf for every other face)
        cam_eye = np.float32([[0, 0, -3]] * B)
        v = np.concatenate([v + np.float32([0, 0, -4.5]), np.float32([[[0.2, 0, -3], [-0.2, 0.1, -3], [0, -0.2, -3]]]).repeat(B, 0)], 1)
        f = np.concatenate([f, np.int32([[v.shape[1] - 3, v.shape[1] - 2, v.shape[1] - 1]])])
    nf = f.shape[0]
    T = 8 if "tex6" in name else 4
    tex_shape = (B, nf, 2, 2, 2, 3) if "tex6" in name else (B, nf, T, 3)
    sc = dict(mode=mode, v=v.copy(), f=f, tex=rng.random(tex_shape, dtype=np.float32), cam_eye=cam_eye,
              eye=cam_eye + np.float32([0.1, -0.1, 0.05]), spec="nospec" not in name,
              met=(rng.random((B, nf, T, 1), dtype=np.float32) * 0.8),
              rou=(0.3 + 0.7 * rng.random((B, nf, T, 1), dtype=np.float32)).astype(np.float32))
    sc["gout"] = rng.normal(0, 1, tex_shape).astype(np.float32)
    if name.startswith("normal_map"):
        nt = rng.normal(0, 0.3, (1, nf, T, 3)).astype(np.float32)
        nt[..., 2] += 1.0
        sc["nt"] = nt
        sc["tbn"] = np.linalg.qr(rng.normal(0, 1, (nf, 3, 3)))[0].astype(np.float32)[None]
    bad = {"nan": np.nan, "pinf": np.inf, "ninf": -np.inf}
    for tag, x in bad.items():   # <tag>_<site>: one non-finite value at that input site
        if tag + "_vertex" in name:
            sc["v"][-1, f[1, 0], 1] = x
        if tag + "_eye" in name:
            sc["eye"] = sc["eye"].copy()
            sc["eye"][0, 2] = x
        if tag + "_cameye" in name:
            sc["cam_eye"] = sc["cam_eye"].copy()
            sc["cam_eye"][-1, 0] = x
        if tag + "_metallic" in name:
            sc["met"][0, 3, 1, 0] = x
        if tag + "_roughness" in name:
            sc["rou"][-1, 5, 0, 0] = x
        if tag + "_nt" in name:
            sc["nt"][0, 4, 2, 1] = x
    if name.startswith("shared"):   # vertices, faces and the specular eye of batch 1 broadcast over B = 2
        sc["v"], sc["eye"] = sc["v"][:1].copy(), sc["eye"][:1].copy()
        if "cam1" in name:
            sc["cam_eye"] = sc["cam_eye"][:1].copy()
    return sc


NAMES = ["sphere_normal_spec", "sphere_normal_nospec", "sphere_depth_spec", "sphere_depth_nospec", "sphere_normal_tex6",
         "sphere_depth_tex6", "ties_depth_nospec", "ties_depth_spec", "axis_normal_spec", "axis_depth_nospec",
         "behind_depth_nospec", "behind_depth_spec", "zero_max_depth_nospec", "sliver_depth_spec", "sphere_depth_b1",
         "sphere_normal_b1", "shared_depth_spec", "shared_cam1_depth_nospec", "shared_normal_spec",
         "nan_vertex_depth_spec", "nan_vertex_normal_spec", "nan_vertex_normal_nospec", "pinf_vertex_normal_nospec",
         "ninf_vertex_depth_nospec", "pinf_vertex_depth_spec", "nan_eye_normal_spec", "pinf_eye_depth_spec",
         "nan_cameye_depth_nospec", "ninf_cameye_depth_spec", "nan_metallic_normal_spec", "pinf_metallic_depth_spec",
         "nan_roughness_depth_spec", "ninf_roughness_normal_spec", "normal_map_spec", "normal_map_nospec",
         "normal_map_nan_nt_spec", "normal_map_pinf_nt_nospec", "normal_map_nan_vertex_spec", "normal_map_nan_metallic_spec"]


def expected_calls(sc):
    if "nt" in sc:
        return {"b200r_normal_mapped_gbuffer_forward", "b200r_normal_mapped_gbuffer_backward"}
    return {"b200r_gbuffer_lighting_forward", "b200r_gbuffer_lighting_backward"}


def build(sc, dev, dtype, fused):
    names = ["vertices", "textures", "metallic", "roughness"] + (["normal_textures"] if "nt" in sc else [])
    src = dict(vertices=sc["v"], textures=sc["tex"], metallic=sc["met"], roughness=sc["rou"], normal_textures=sc.get("nt"))
    ts = {k: torch.from_numpy(np.ascontiguousarray(src[k])).to(dev, dtype).requires_grad_(True) for k in names}
    faces = torch.from_numpy(sc["f"])[None].repeat(sc["v"].shape[0], 1, 1).to(dev)
    nm = "nt" in sc
    mesh = jr.Mesh(ts["vertices"], faces, textures=ts["textures"], dr_type='n3mr' if sc["tex"].ndim == 6 else 'softras',
                   metallic_textures=ts["metallic"], roughness_textures=ts["roughness"],
                   normal_textures=ts["normal_textures"] if nm else None,
                   TBN=torch.from_numpy(sc["tbn"]).to(dev, dtype) if nm else None, texture_res=2)
    mesh.with_specular = sc["spec"]
    tr = jr.Transform(camera_mode='look_at')
    tr.set_eyes(torch.from_numpy(sc["cam_eye"]).to(dev, dtype))
    light = jr.Lighting(Gbuffer=sc["mode"], transform=tr, **LIGHT)
    light.fused = fused
    return ts, light, mesh, torch.from_numpy(sc["eye"]).to(dev, dtype)


def run(sc, dev, dtype, fused):
    """The G-buffer textures and {name: gradient of <out, gout>} (None where no gradient reaches the leaf)."""
    ts, light, mesh, eyes = build(sc, dev, dtype, fused)
    if fused:
        fn = light._fused_normal_mapped_gbuffer if "nt" in sc else light._fused_gbuffer
        assert fn(mesh, eyes) is not None   # the kernels' path, not a silent fallback
    out = light(mesh, eyes).textures
    out.backward(torch.from_numpy(sc["gout"]).to(dev, dtype))
    g = {k: (None if t.grad is None else t.grad.cpu().double().numpy()) for k, t in ts.items()}
    return out.detach().cpu().double().numpy(), g
