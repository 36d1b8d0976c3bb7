"""Scenes for the G-buffer tests (tests/test_gbuffer_gpu.py): both modes with and without the specular branch, 6-D
textures, exact depth ties, axis-aligned faces (a normal component of +-1 puts the clamp at equality), every face behind
the camera (M < 0) and a largest depth of exactly 0 (M = 0), a sliver in depth mode, batches of one, vertices, faces and
eyes shared over a batch of two (batch 1 broadcast), NaN / +-inf at the vertices, the specular eye, the camera eye,
metallic, roughness and the normal textures, and the normal-map path.  Past one grid of faces: depth at B * nf around
one block (255, 256, 257) and one full grid of the grid-stride passes (262 144 = 256 x 1024, 262 145), and 16 x the
39 200-face sphere (627 200 pairs, three trips) with the max and an exact tie reached only on the second trip; ties
split over blocks and partials; shared batches with ties (vertices, faces and camera batch 1; vertices batch 1 with
per-batch faces); slivers in normal mode; metallic / roughness texel counts Tm other than T; per-batch normal textures
and TBN, per-face metallic on the normal-map path; and a zero max reached by both +0 and -0."""
import numpy as np
import torch

import jrender_b200 as jr
from jrender_b200 import workloads as wl

LIGHT = dict(intensity_ambient=0.4, color_ambient=[1.0, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1.0, 0.7], directions=[0.3, 0.8, -0.5])


def _sphere(rng, B=2, nf=280):
    v, f = wl.sphere_by_faces(nf)
    return (v[None] + rng.normal(0, 0.02, (1,) + v.shape)).astype(np.float32).repeat(B, 0), f


def _small_faces(rng, nf):
    """nf separate random faces of size ~0.01 in the unit cube, one camera-side of z = -3."""
    c = rng.uniform(-1, 1, (nf, 1, 3))
    v = (c + rng.normal(0, 0.01, (nf, 3, 3))).astype(np.float32).reshape(1, -1, 3)
    return v, np.arange(3 * nf, dtype=np.int32).reshape(nf, 3)


GRID = (255, 256, 257, 262144, 262145)   # B * nf of the grid scenes: around one block, one full grid of 1024 blocks
BIG_B, BIG_NF, BIG_MAX, BIG_TIE = 16, 39200, 10, 12   # the max face's batch, and its exact copy's


def scene(name):
    rng = np.random.default_rng(sum(name.encode()))
    mode = "depth" if "depth" in name else "normal"
    B = 1 if "b1" in name or name.startswith(("grid", "split")) else 2
    cam_eye = np.float32([[0.4, 0.6, -2.6], [1.0, 1.2, -2.2]])[:B]
    T = 8 if "tex6" in name else 4
    f3 = None   # per-batch faces [B, nf, 3], where they differ from sc["f"] repeated
    if name.startswith("grid"):
        v, f = _small_faces(rng, int(name[4:name.index("_")]))
        T = 1
    elif name.startswith("split_ties"):
        # 70 000 small faces; face 5 moved to the far side (the max) and its corners copied to face 69 000: an exact tie
        # of faces in blocks 0 and 269, so in different partials
        v, f = _small_faces(rng, 70000)
        v[0, f[5]] += np.float32([0, 0, 2.5])
        v[0, f[69000]] = v[0, f[5]]
    elif name.startswith("big"):
        # 16 jittered 39 200-face spheres: batch 10 scaled up holds the max, batch 12 is its exact copy (a tie); both
        # lie past pair 262 144, reached on the grid-stride passes' second trip
        B, T = BIG_B, 1
        v, f = wl.sphere_by_faces(BIG_NF)
        v = (v[None] + rng.normal(0, 0.002, (B,) + v.shape)).astype(np.float32)
        v[BIG_MAX] *= np.float32(1.5)
        v[BIG_TIE] = v[BIG_MAX]
        cam_eye = np.float32([[0.3, 0.5, -3.5]])
        if "nan" in name:   # one NaN vertex in batch 13, also past pair 262 144
            v[13, f[7, 0], 2] = np.nan
    elif name.startswith("zero_sign"):
        # camera at (1, 1, 1) looking at the origin: the z axis (-a, -a, -a).  Face 0's centroid is exactly the eye
        # (z = -0 from three -0 products), the last face's is the eye + (1, -1, 0) (z = -a + a + -0 = +0); a sphere
        # behind the camera keeps every other z < 0, so the max is a zero reached with both signs
        cam_eye = np.float32([[1, 1, 1]] * B)
        sv, sf = _sphere(rng, B)
        sv = sv * np.float32(0.3) + np.float32(2)
        zero_neg = np.float32([[1.5, 1, 1], [0.5, 1.25, 1], [1, 0.75, 1]])
        zero_pos = np.float32([[2.5, 0, 1.5], [1.5, 0.25, 0.5], [2, -0.25, 1]])
        v = np.concatenate([np.repeat(zero_neg[None], B, 0), sv, np.repeat(zero_pos[None], B, 0)], 1)
        n = sv.shape[1]
        f = np.concatenate([np.int32([[0, 1, 2]]), sf + 3, np.int32([[n + 3, n + 4, n + 5]])])
    elif name.startswith("ties"):
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
    tex_shape = (B, nf, 2, 2, 2, 3) if "tex6" in name else (B, nf, T, 3)
    Tm = 4 if "tm4" in name else 1 if ("tm1" in name or "face_metallic" in name) else T
    sc = dict(mode=mode, v=v.copy(), f=f, tex=rng.random(tex_shape, dtype=np.float32), cam_eye=cam_eye,
              eye=cam_eye + np.float32([0.1, -0.1, 0.05]), spec="nospec" not in name,
              met=(rng.random((B, nf, Tm, 1), dtype=np.float32) * 0.8),
              rou=(0.3 + 0.7 * rng.random((B, nf, Tm, 1), dtype=np.float32)).astype(np.float32))
    sc["gout"] = rng.normal(0, 1, tex_shape).astype(np.float32)
    if name.startswith("normal_map"):
        Bn = B if "_bn" in name else 1
        nt = rng.normal(0, 0.3, (Bn, nf, T, 3)).astype(np.float32)
        nt[..., 2] += 1.0
        sc["nt"] = nt
        sc["tbn"] = np.linalg.qr(rng.normal(0, 1, (Bn, nf, 3, 3)))[0].astype(np.float32)
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
    if "shared" in name:   # vertices, faces and the specular eye of batch 1 broadcast over B = 2
        sc["v"], sc["eye"] = sc["v"][:1].copy(), sc["eye"][:1].copy()
        if "cam1" in name:
            sc["cam_eye"] = sc["cam_eye"][:1].copy()
        if "perbatch_faces" in name:   # batch 1 draws the faces in another order: its depths are a permutation of batch 0's
            sc["f3"] = np.stack([f, f[rng.permutation(nf)]]).astype(np.int32)
    return sc


NAMES = ["sphere_normal_spec", "sphere_normal_nospec", "sphere_depth_spec", "sphere_depth_nospec", "sphere_normal_tex6",
         "sphere_depth_tex6", "ties_depth_nospec", "ties_depth_spec", "axis_normal_spec", "axis_depth_nospec",
         "behind_depth_nospec", "behind_depth_spec", "zero_max_depth_nospec", "sliver_depth_spec", "sphere_depth_b1",
         "sphere_normal_b1", "shared_depth_spec", "shared_cam1_depth_nospec", "shared_normal_spec",
         "nan_vertex_depth_spec", "nan_vertex_normal_spec", "nan_vertex_normal_nospec", "pinf_vertex_normal_nospec",
         "ninf_vertex_depth_nospec", "pinf_vertex_depth_spec", "nan_eye_normal_spec", "pinf_eye_depth_spec",
         "nan_cameye_depth_nospec", "ninf_cameye_depth_spec", "nan_metallic_normal_spec", "pinf_metallic_depth_spec",
         "nan_roughness_depth_spec", "ninf_roughness_normal_spec", "normal_map_spec", "normal_map_nospec",
         "normal_map_nan_nt_spec", "normal_map_pinf_nt_nospec", "normal_map_nan_vertex_spec", "normal_map_nan_metallic_spec",
         "grid255_depth_nospec", "grid256_depth_nospec",
         "grid257_depth_nospec", "grid262144_depth_nospec", "grid262145_depth_nospec", "big_depth_nospec",
         "big_nan_depth_nospec", "split_ties_depth_spec", "ties_shared_cam1_depth_nospec",
         "ties_shared_perbatch_faces_depth_nospec", "sphere_depth_tex6_tm4", "sphere_normal_tm1_spec",
         "normal_map_bn_spec", "normal_map_face_metallic_spec", "zero_sign_depth_nospec"]
# Slivers in normal mode: their normal moves by up to 0.1 under the float32 rounding of the edge vectors the kernels
# take, so no fixed bound against the float64 mirror holds; the kernels are held to the emulation alone, and the
# emulation to float64 per entry within its own error bound.
SLIVER_NORMAL = ["sliver_normal_spec", "sliver_normal_nospec"]
LARGE = {"grid262144_depth_nospec", "grid262145_depth_nospec", "big_depth_nospec", "big_nan_depth_nospec",
         "split_ties_depth_spec"}


def expected_calls(sc):
    if "nt" in sc:
        return {"b200r_normal_mapped_gbuffer_forward", "b200r_normal_mapped_gbuffer_backward"}
    return {"b200r_gbuffer_lighting_forward", "b200r_gbuffer_lighting_backward"}


def faces_of(sc):
    """The faces Lighting gets, [Bf, nf, 3]: per batch where the scene has them, else sc['f'] over the vertex batch."""
    return sc["f3"] if "f3" in sc else np.repeat(sc["f"][None], sc["v"].shape[0], 0)


def kernel_args(sc):
    """The arguments Lighting hands the G-buffer backward for scene sc, as oracle.gbuffer.args_from_call returns them,
    built on the host (no GPU): the eye rows and metallic / roughness only on the specular branch (per-face values
    broadcast over the texels on the normal-map path), the camera of look_at, the light direction normalised in
    float32, and an empty array for each gradient the backward is asked for."""
    from jrender_b200.lighting import _normalized_direction
    from oracle import gbuffer as OG
    F32 = np.float32
    B, nf = sc["tex"].shape[:2]
    T = sc["tex"][0, 0].size // 3
    spec, f = sc["spec"], faces_of(sc)
    eye = sc["eye"].reshape(-1, 3).astype(F32) if spec else None
    a = dict(vertices=sc["v"].astype(F32), faces=f.astype(np.int32), eye=eye, B=B, Bv=sc["v"].shape[0], Bf=f.shape[0],
             Be=eye.shape[0] if spec else 1, nv=sc["v"].shape[1], nf=nf, T=T, grad_out=sc["gout"].astype(F32).reshape(B, nf, T, 3),
             light=OG._light(LIGHT["intensity_directionals"], LIGHT["color_directionals"],
                             _normalized_direction(LIGHT["directions"]), spec))
    empty = lambda x: None if x is None else np.empty_like(x)
    if "nt" in sc:
        met = np.ascontiguousarray(np.broadcast_to(sc["met"], (B, nf, T, 1))) if spec else None
        rou = np.ascontiguousarray(np.broadcast_to(sc["rou"], (B, nf, T, 1))) if spec else None
        a.update(normal_textures=sc["nt"].astype(F32), tbn=sc["tbn"].astype(F32), Bn=sc["nt"].shape[0],
                 Bt=sc["tbn"].shape[0], metallic=met, roughness=rou, grad_normal_textures=np.empty_like(sc["nt"]),
                 grad_vertices=empty(a["vertices"]) if spec else None)
    else:
        met, rou = (sc["met"], sc["rou"]) if spec else (None, None)
        a.update(metallic=met, roughness=rou, Tm=sc["met"][0, 0].size if spec else 0, mode=int(sc["mode"] == "depth"),
                 camera_eye=sc["cam_eye"].astype(F32), Bc=sc["cam_eye"].shape[0], at=np.zeros(3, F32),
                 up=np.float32([0, 1, 0]), camera_mode=0, grad_vertices=empty(a["vertices"]))
    a.update(grad_metallic=empty(met), grad_roughness=empty(rou))
    return a


def build(sc, dev, dtype, fused):
    names = ["vertices", "textures", "metallic", "roughness"] + (["normal_textures"] if "nt" in sc else [])
    src = dict(vertices=sc["v"], textures=sc["tex"], metallic=sc["met"], roughness=sc["rou"], normal_textures=sc.get("nt"))
    ts = {k: torch.from_numpy(np.ascontiguousarray(src[k])).to(dev, dtype).requires_grad_(True) for k in names}
    faces = torch.from_numpy(faces_of(sc)).to(dev)
    nm = "nt" in sc
    v = ts["vertices"]
    if not fused and faces.shape[0] != v.shape[0]:   # the mirror gathers per batch: the one vertex set expanded over B
        v = v.expand(faces.shape[0], -1, -1)
    mesh = jr.Mesh(v, faces, textures=ts["textures"], dr_type='n3mr' if sc["tex"].ndim == 6 else 'softras',
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
