"""Seeded scenes for test_lighting_edges_{cpu,gpu}.py: inputs of the fused surface lighting (b200r_surface_lighting_*,
one normal per face) and the normal-mapped lighting (b200r_normal_mapped_lighting_*, one normal per texel) at the
shapes, batch layouts, geometry and values where those kernels can go wrong.  Every builder returns numpy arrays.

A scene is a dict: v [Bv, nv, 3], f [nf, 3] (int32, shared by the batch), tex [B, nf, T, 3] (or [B, nf, ts, ts, ts, 3]),
met / rou [B, nf, Tm, 1] (or 6-D), eye [Be, 3] (None for Be = 0: no Cook-Torrance branch), gout like tex, light (the
Lighting keyword arguments), and for the normal-map path nt [Bn, nf, T, 3] and tbn [Bt, nf, 3, 3].
"""
import numpy as np

from jrender_b200 import io as jio
from jrender_b200 import workloads as wl

F32 = np.float32
LIGHT = dict(intensity_ambient=0.4, color_ambient=[1, 0.9, 0.8], intensity_directionals=0.7,
             color_directionals=[0.9, 1, 0.7], directions=[0.3, 1, -0.4])
# Axis light and power-of-two ambient colour: N.L is exactly 0 on faces in a vertical plane, and an unlit face's
# diffuse light is exactly (0.5, 0.25, 0.125) with specular exactly 0, so tex = 0 and tex = 1 / diffuse put
# tex * diffuse + specular exactly on the clamp's bounds.
AXIS_LIGHT = dict(intensity_ambient=0.5, color_ambient=[1.0, 0.5, 0.25], intensity_directionals=0.7,
                  color_directionals=[0.9, 1, 0.7], directions=[0, 1, 0])
UNLIT_DIFFUSE = F32([0.5, 0.25, 0.125])
EYES4 = F32([[0.0, 0.3, -2.7], [1.0, 1.5, -2.0], [-2.0, 0.3, 1.0], [0.4, 2.2, 1.6]])
SLIVER_ASPECTS = (1e-2, 1e-3, 1e-4, 1e-5)
Q = 2.0 ** 23   # sliver coordinates lie on this grid
BLOCK = 128   # threads per block of both flat kernels and of the normal-map backward


def sphere(Bv, seed, jitter=0.03):
    rng = np.random.default_rng(seed)
    v, f = wl.sphere_by_faces(280)
    vb = (v[None] + rng.normal(0, jitter, (Bv,) + v.shape)).astype(F32)
    return vb, f.astype(np.int32)


def append(vb, f, tris):
    """Append isolated triangles tris [n, 3, 3] (their own vertices, the same in every batch element); returns the new
    (vb, f) and the indices of the appended faces."""
    n = tris.shape[0]
    nv = vb.shape[1]
    vb = np.concatenate([vb, np.broadcast_to(tris.reshape(1, n * 3, 3), (vb.shape[0], n * 3, 3))], axis=1).astype(F32)
    f = np.concatenate([f, (nv + np.arange(n * 3, dtype=np.int32)).reshape(n, 3)], axis=0)
    return np.ascontiguousarray(vb), f, np.arange(f.shape[0] - n, f.shape[0])


def slivers(rng, per_aspect=12, length=0.4):
    """Thin triangles near the sphere's surface, facing outward (so that most are lit), of height / length = aspect
    (to within the grid below).  Every coordinate is a multiple of 1 / Q, so every edge vector is exact in float32: the
    kernels and the float64 mirror see the same triangle, and only the arithmetic on it differs."""
    out, aspect = [], []
    for a in SLIVER_ASPECTS:
        for _ in range(per_aspect):
            p = rng.normal(0, 1, 3)
            p = 0.8 * p / np.linalg.norm(p)
            n = p / np.linalg.norm(p)
            u = np.cross(n, rng.normal(0, 1, 3))
            u /= np.linalg.norm(u)
            w = np.cross(n, u)
            v0, v1 = p - 0.5 * length * u, p + 0.5 * length * u
            v2 = p + (rng.uniform(-0.3, 0.3) * length) * u + a * length * w
            tri = np.round(np.float64([v0, v2, v1] if np.dot(np.cross(v2 - v1, v0 - v1), n) > 0 else [v0, v1, v2]) * Q) / Q
            out.append(tri)
            aspect.append(a)
    return np.asarray(out, F32), np.asarray(aspect)


# exact geometry (every coordinate dyadic, so every sum and difference below is exact in float32 and float64)
COLLINEAR = F32([[0.25, -0.5, 0.125], [0.375, -0.4375, -0.125], [0.5, -0.375, -0.375]])   # p, p + d, p + 2d
COINCIDENT = F32([[0.125, 0.25, 0.5], [0.125, 0.25, 0.5], [-0.25, 0.375, 0.5]])
EDGE_ON = F32([[[0.5, 0.125, 0.25], [0.5, 0.375, 0.125], [0.5, 0.25, 0.5]],       # in the plane x = 0.5
               [[0.25, 0.125, -0.5], [-0.125, 0.5, -0.5], [0.0, 0.25, -0.5]]])    # in the plane z = -0.5
# centroid q = ((v0 + v1) + v2) / 3 exact: v = q + a, q + b, q - a - b
EYE_Q = F32([0.25, 0.5, -0.75])
EYE_FACE = np.stack([EYE_Q + F32([0.125, 0.0, 0.25]), EYE_Q + F32([-0.25, 0.0, 0.125]), EYE_Q + F32([0.125, 0.0, -0.375])])
BELOW_Q = F32([-0.5, 0.25, 0.375])
BELOW_FACE = np.stack([BELOW_Q + F32([0.25, 0.125, 0.0]), BELOW_Q + F32([-0.125, -0.1875, -0.25]),
                       BELOW_Q + F32([-0.125, 0.0625, 0.25])])


def flat_normals(vb, f):
    """The mirror's face normals (float64 cross product of float32 edges), float64 [Bv, nf, 3]."""
    fv = vb[:, f].astype(F32)
    c = np.cross((fv[:, :, 2] - fv[:, :, 1]).astype(np.float64), (fv[:, :, 0] - fv[:, :, 1]).astype(np.float64))
    return c / np.maximum(np.linalg.norm(c, axis=-1, keepdims=True), 1e-12)


def centroid(vb, f):
    """((v0 + v1) + v2) / 3 in float32, the kernels' order."""
    fv = vb[:, f].astype(F32)
    return ((fv[:, :, 0] + fv[:, :, 1]) + fv[:, :, 2]) / F32(3.0)


def _materials(rng, B, nf, shape_t):
    met = rng.uniform(0, 1, (B, nf) + shape_t + (1,)).astype(F32)
    rou = rng.uniform(0.2, 1, (B, nf) + shape_t + (1,)).astype(F32)
    return met, rou


def flat_shapes(T, Tm, B=3, Bv=None, Be=None, seed=0):
    """Flat path at T texels per face (T = 125 as 6-D n3mr textures, ts = 5) and Tm material texels (1 or T)."""
    rng = np.random.default_rng(seed)
    Bv = B if Bv is None else Bv
    vb, f = sphere(Bv, seed)
    vb, f, _ = append(vb, f, slivers(rng, per_aspect=1)[0][:3])   # 283 faces: B * nf is not a multiple of BLOCK
    nf = f.shape[0]
    tshape = (5, 5, 5) if T == 125 else (T,)
    mshape = tshape if Tm == T else (1,) * len(tshape)
    tex = rng.uniform(0, 2.0, (B, nf) + tshape + (3,)).astype(F32)
    met, rou = _materials(rng, B, nf, mshape)
    Be = B if Be is None else Be
    eye = None if Be == 0 else EYES4[:Be] if Be > 1 else EYES4[3:4]
    return dict(v=vb, f=f, tex=tex, met=met, rou=rou, eye=eye, gout=rng.uniform(-1, 1, tex.shape).astype(F32), light=LIGHT)


def flat_geometry(B=4, Bv=1, seed=1):
    """Flat path on the sphere plus slivers (aspect 1e-2 down to 1e-5), a collinear and a coincident-vertex face, two
    faces edge-on to the light (0, 1, 0), a face whose centroid is eye 1 (V on normalize's eps path) and one whose
    centroid is straight above eye 2 (V = -L: H on its eps path).  Unlit sphere faces carry texels exactly at the clamp
    bounds.  Keys beyond the scene's: the face indices of each group."""
    rng = np.random.default_rng(seed)
    vb, f = sphere(Bv, seed)
    sl, aspect = slivers(rng)
    special = np.concatenate([sl, COLLINEAR[None], COINCIDENT[None], EDGE_ON, EYE_FACE[None], BELOW_FACE[None]]).astype(F32)
    vb, f, idx = append(vb, f, special)
    ns = sl.shape[0]
    nf = f.shape[0]
    T = 4
    tex = rng.uniform(0.05, 1.5, (B, nf, T, 3)).astype(F32)
    met, rou = _materials(rng, B, nf, (T,))
    eye = EYES4.copy()
    eye[1] = EYE_Q
    eye[2] = BELOW_Q - F32([0, 1, 0])
    N = flat_normals(vb, f)
    unlit = np.nonzero((N[:, :, 1] < -0.2).all(axis=0))[0][:20]
    tex[:, unlit, 0] = 0.0                  # tex * diffuse + 0 == 0
    tex[:, unlit, 1] = 1.0 / UNLIT_DIFFUSE  # == 1
    return dict(v=vb, f=f, tex=tex, met=met, rou=rou, eye=eye, gout=rng.uniform(-1, 1, tex.shape).astype(F32),
                light=AXIS_LIGHT, slivers=idx[:ns], sliver_aspect=aspect, collinear=idx[ns], coincident=idx[ns + 1],
                edge_on=idx[ns + 2:ns + 4], eye_face=idx[ns + 4], below_face=idx[ns + 5], unlit=unlit)


def _tbn(rng, vb, f):
    tbn = jio.create_TBN(rng.uniform(0, 1, (f.shape[0], 3, 2)).astype(F32), vb[0][f])
    assert np.isfinite(tbn).all()
    return tbn


def _tangent_normals(rng, shape, spread=0.5):
    nt = rng.normal(0, spread, shape + (3,))
    nt[..., 2] += 1
    return (nt / np.linalg.norm(nt, axis=-1, keepdims=True)).astype(F32)


def nm_shapes(T, Bn, Bt, B=3, Bv=None, Be=None, per_face_material=False, seed=0, base=None):
    """Normal-map path at T texels per face, normal-texture batch Bn and TBN batch Bt (1 or B)."""
    rng = np.random.default_rng(seed)
    Bv = B if Bv is None else Bv
    if base is None:   # 283 faces: Bn * nf is not a multiple of the backward's 4 warps per block
        vb, f, _ = append(*sphere(Bv, seed), _lit_isolated(rng, 3))
    else:
        vb, f = base
    nf = f.shape[0]
    tbn0 = _tbn(rng, vb, f)
    tbn = np.stack([tbn0] + [_tbn(rng, vb, f) for _ in range(Bt - 1)]).astype(F32)
    nt = _tangent_normals(rng, (Bn, nf, T))
    tex = rng.uniform(0, 1.6, (B, nf, T, 3)).astype(F32)
    met, rou = _materials(rng, B, nf, (1,) if per_face_material else (T,))
    Be = B if Be is None else Be
    eye = None if Be == 0 else EYES4[:Be] if Be > 1 else EYES4[3:4]
    return dict(v=vb, f=f, tex=tex, met=met, rou=rou, eye=eye, nt=nt, tbn=tbn,
                gout=rng.uniform(-1, 1, tex.shape).astype(F32), light=LIGHT)


def nm_clamp_bounds(B=2, T=33, seed=2):
    """Normal-map path under the axis light: texels whose normal faces away from it (diffuse exactly the ambient
    colour, specular exactly 0) carry tex = 0 and tex = 1 / diffuse.  Key `bounds`: (b, f, t) of those texels."""
    sc = nm_shapes(T, B, 1, B=B, seed=seed)
    sc["light"] = AXIS_LIGHT
    N = np.einsum("bftk,fkj->bftj", sc["nt"].astype(np.float64), sc["tbn"][0].astype(np.float64))
    b, fi, t = np.nonzero(N[..., 1] < -0.2 * np.linalg.norm(N, axis=-1))
    pick = np.arange(0, b.size, max(1, b.size // 40))[:40]
    b, fi, t = b[pick], fi[pick], t[pick]
    half = pick.size // 2
    sc["tex"][b[:half], fi[:half], t[:half]] = 0.0
    sc["tex"][b[half:], fi[half:], t[half:]] = 1.0 / UNLIT_DIFFUSE
    sc["bounds"] = (b, fi, t)
    return sc


def head(seed=0, faces=66282):
    """The demo 1.5 head's size on the normal-map path: B = 1, 66 282 faces, T = 225 (tools/time_normal_lighting.py's
    synthetic mesh with finite TBNs); `faces` keeps the first that many."""
    rng = np.random.default_rng(seed)
    v, f = wl.uv_sphere(194, 172, jitter=0.002)
    f = f[:faces].astype(np.int32)
    nf, T = f.shape[0], 225
    tbn = jio.create_TBN(rng.uniform(0, 1, (nf, 3, 2)).astype(F32), v[f])
    tbn = np.where(np.isfinite(tbn), tbn, 0).astype(F32)[None]
    nt = _tangent_normals(rng, (1, nf, T), 0.3)
    tex = rng.uniform(0, 1.3, (1, nf, T, 3)).astype(F32)
    met, rou = _materials(rng, 1, nf, (T,))
    return dict(v=v[None].astype(F32), f=f, tex=tex, met=met, rou=rou, eye=F32([[0.3, 0.5, -2.0]]), nt=nt, tbn=tbn,
                gout=rng.uniform(-1, 1, tex.shape).astype(F32), light=LIGHT)


# ---- non-finite inputs ------------------------------------------------------------------------------------------------

NONFINITE = {"nan": np.nan, "posinf": np.inf, "neginf": -np.inf}
FLAT_SITES = ("texel", "vertex", "metallic", "roughness")
NM_SITES = FLAT_SITES + ("normal", "tbn")


def _lit_isolated(rng, n):
    """n isolated triangles facing the light (0.3, 1, -0.4) and the eyes from above, so that both light branches are
    live on them."""
    tris = []
    for k in range(n):
        c = F32([-0.6 + 0.3 * k, 1.2, 0.1 * k])
        tris.append(c + F32([[0.0, 0.0, 0.125], [0.125, 0.0, -0.0625], [-0.125, 0.0, -0.0625]]))
    return np.asarray(tris, F32)


def nonfinite(site, value, nm=False, B=2, T=9, seed=3):
    """A scene with per-batch everything (B = 2) and one non-finite `value` at `site`, always on batch element 1 and on
    an isolated, lit triangle whose vertices no other face shares.  Returns (clean, dirty, (b, f)): the scene without and
    with the value, and the affected (batch element, face).  site 'tbn' gives that face degenerate UVs (create_TBN makes
    its frame non-finite, whatever `value`) and the flat tangent-space normal (0, 0, 1) on all its texels."""
    rng = np.random.default_rng(seed)
    vb, f = sphere(B, seed)
    vb, f, iso = append(vb, f, _lit_isolated(rng, 3))
    if nm:
        clean = nm_shapes(T, B, B, B=B, seed=seed, base=(vb, f))
        uv = rng.uniform(0, 1, (f.shape[0], 3, 2)).astype(F32)
        clean["tbn"] = np.stack([jio.create_TBN(uv, vb[0][f])] * B).astype(F32)
        clean["uv"] = uv
    else:
        clean = flat_shapes(T, T, B=B, seed=seed)
        clean.update(v=vb, f=f)
        nf = f.shape[0]
        clean["tex"] = rng.uniform(0, 1.2, (B, nf, T, 3)).astype(F32)
        clean["met"], clean["rou"] = _materials(rng, B, nf, (T,))
        clean["gout"] = rng.uniform(-1, 1, clean["tex"].shape).astype(F32)
    clean["eye"] = F32([[0.0, 2.5, -1.0], [0.5, 2.0, 1.5]])[:B]
    b, fa = 1, int(iso[1])
    dirty = {k: (x.copy() if isinstance(x, np.ndarray) else x) for k, x in clean.items()}
    if site == "texel":
        dirty["tex"][b, fa, 2, 1] = value
    elif site == "vertex":
        dirty["v"][b, f[fa, 1], 0] = value
    elif site == "metallic":
        dirty["met"][b, fa, 3, 0] = value
    elif site == "roughness":
        dirty["rou"][b, fa, 3, 0] = value
    elif site == "normal":
        dirty["nt"][b, fa, 4, 1] = value
    elif site == "tbn":
        uv = clean["uv"].copy()
        uv[fa] = uv[fa, 0]   # all three UVs equal: a degenerate UV triangle
        tbn = jio.create_TBN(uv, vb[0][f])
        assert not np.isfinite(tbn[fa]).all() and np.isfinite(np.delete(tbn, fa, 0)).all()
        dirty["tbn"][b] = tbn
        clean["nt"][b, fa] = dirty["nt"][b, fa] = F32([0, 0, 1])
    else:
        raise ValueError(site)
    return clean, dirty, (b, fa)


# ---- running a scene ----------------------------------------------------------------------------------------------------

FLAT_GRADS = ("vertices", "textures", "metallic", "roughness")
NM_GRADS = ("vertices", "textures", "normal_textures", "metallic", "roughness")


def run(sc, dev, dtype, fused, grads=True):
    """Lit textures and, with grads, {name: gradient of <out, gout>} through jrender_b200.Lighting: the fused kernels
    (fused=True, float32 CUDA tensors) or the op-by-op mirror (Lighting.fused = False) in `dtype`.  The kernels' path
    is asserted, so a scene cannot silently fall back to the mirror."""
    import torch
    import jrender_b200 as jr
    nm = "nt" in sc
    names = NM_GRADS if nm else FLAT_GRADS
    src = dict(vertices=sc["v"], textures=sc["tex"], normal_textures=sc.get("nt"), metallic=sc["met"], roughness=sc["rou"])
    ts = {k: torch.from_numpy(np.ascontiguousarray(src[k])).to(dev, dtype).requires_grad_(grads) for k in names}
    faces = torch.from_numpy(sc["f"])[None].repeat(sc["v"].shape[0], 1, 1).to(dev)
    extra = dict(normal_textures=ts["normal_textures"], TBN=torch.from_numpy(sc["tbn"]).to(dev, dtype)) if nm else {}
    m = jr.Mesh(ts["vertices"], faces, textures=ts["textures"], dr_type='n3mr' if sc["tex"].ndim == 6 else 'softras',
                metallic_textures=ts["metallic"], roughness_textures=ts["roughness"], **extra)
    light = jr.Lighting(**sc["light"])
    light.fused = fused
    eye = None if sc["eye"] is None else torch.from_numpy(sc["eye"]).to(dev, dtype)
    if fused:
        assert (light._fused_normal_mapped(m, eye) is not None) if nm else (light._fused_surface(m, eye) is not None)
    out = light(m, eye).textures
    if not grads:
        return out.detach().cpu().double().numpy(), None
    out.backward(torch.from_numpy(sc["gout"]).to(dev, dtype))
    g = {k: (None if t.grad is None else t.grad.cpu().double().numpy()) for k, t in ts.items()}
    return out.detach().cpu().double().numpy(), g


def kernel_args(sc, backward=True, grads=None):
    """The arguments Lighting hands the fused kernel for scene sc, as oracle.lighting.args_from_call returns them, built
    on the host (no GPU): faces repeated over the vertex batch, the eye rows, per-face materials broadcast over the
    texels on the normal-map path, the light direction normalised in float32.  grads: the gradients requested (all of
    the path's by default)."""
    import torch
    import torch.nn.functional as F
    nm = "nt" in sc
    B, nf = sc["tex"].shape[:2]
    T = sc["tex"][0, 0].size // 3
    L = sc["light"]
    spec = sc["eye"] is not None
    d = F.normalize(torch.tensor([float(x) for x in L["directions"]], dtype=torch.float32), dim=0, eps=1e-12).numpy()
    a = dict(vertices=sc["v"].astype(F32), faces=np.repeat(sc["f"][None], sc["v"].shape[0], 0).astype(np.int32),
             textures=sc["tex"].astype(F32), eye=None if not spec else sc["eye"].astype(F32),
             light=dict(amb_i=F32(L["intensity_ambient"]), amb_c=np.asarray(L["color_ambient"], F32),
                        dir_i=F32(L["intensity_directionals"]), dir_c=np.asarray(L["color_directionals"], F32),
                        dir=d.astype(F32), with_specular=spec))
    a.update(B=B, Bv=sc["v"].shape[0], Bf=sc["v"].shape[0], Be=0 if not spec else sc["eye"].shape[0], nv=sc["v"].shape[1],
             nf=nf, T=T)
    if nm:
        met = np.broadcast_to(sc["met"], (B, nf, T, 1)).astype(F32) if spec else None
        rou = np.broadcast_to(sc["rou"], (B, nf, T, 1)).astype(F32) if spec else None
        a.update(normal_textures=sc["nt"].astype(F32), tbn=sc["tbn"].astype(F32), metallic=met, roughness=rou,
                 Bn=sc["nt"].shape[0], n_nf=nf, n_T=T, Bt=sc["tbn"].shape[0], t_nf=nf)
    else:
        a.update(metallic=sc["met"].astype(F32) if spec else None, roughness=sc["rou"].astype(F32) if spec else None,
                 Tm=sc["met"][0, 0].size if spec else 0)
    if backward:
        grads = (NM_GRADS if nm else FLAT_GRADS) if grads is None else grads
        a["grad_out"] = sc["gout"].astype(F32)
        for k in grads:
            src = dict(vertices=a["vertices"], textures=a["textures"], normal_textures=a.get("normal_textures"),
                       metallic=a["metallic"], roughness=a["roughness"])[k]
            a["grad_" + k] = None if src is None else np.empty_like(src)
    return a


# ---- equality at the clamp_min kinks ----------------------------------------------------------------------------------

EPS12 = F32(1e-12)
# a face whose centroid is exactly 0 (v, w, -v - w, dyadic): the forward's ((v0 + v1) + v2) / 3 and the flat backward's
# ((v0 + v1) + v2) * (1 / 3) agree on it, so both evaluations see the same V; its normal is (1, 1, 0.5) / 1.5
ZERO_FACE = F32([[0.25, -0.25, 0.0], [0.0, 0.125, -0.25], [-0.25, 0.125, 0.25]])


def eps_texel():
    """A float32 (x, y, 0) near 1e-12 (0.6, 0.8, 0) whose norm as the kernels form it, sqrt((x x + y y) + 0 0), is
    exactly 1e-12f.  Through an identity TBN it is the texel normal itself (products by 1 and 0 are exact); a unit axis
    would be unlit (x, z) or parallel to the axis light (y), where N.L's derivative vanishes."""
    x = (F32(0.6e-12) + np.arange(-300, 300) * np.spacing(F32(0.6e-12))).astype(F32)
    y = np.sqrt(np.float64(EPS12) ** 2 - np.float64(x) ** 2).astype(F32)
    n = np.sqrt((x * x + y * y) + F32(0) * F32(0))
    hit = np.flatnonzero(n == EPS12)
    assert hit.size, "no texel normal of norm 1e-12f"
    return F32([x[hit[0]], y[hit[0]], 0])


def _den4_eye(N, L):
    """An eye over the zero-centroid face for which the kernels' float32 den4 = (N.V * 4) * N.L is exactly 0.01f, with
    N the normal as the kernel forms it: found among small float32 nudges of a grazing eye, with the emulation's own
    normalize3 and dot3."""
    from oracle import lighting as OL
    from oracle.numbers import Walk
    N64 = np.float64(N)
    NdotL = float(N64 @ np.float64(L))
    u = np.cross(N64, [0.0, 0.0, 1.0])
    u /= np.linalg.norm(u)
    want = 0.01 / (4 * NdotL)                      # N.V
    base = 2.0 * (np.sqrt(1 - want ** 2) * u + want * N64)
    k = np.arange(-600, 600)
    w2 = np.cross(N64, u)
    eyes = (base[None, None] + 1e-7 * (k[:, None, None] * N64 + k[None, :, None] * w2)).reshape(-1, 3).astype(F32)
    w = Walk()
    V = OL.normalize3(w, [eyes[:, j] - F32(0) for j in range(3)], F32(1e-12))
    Nc = [np.full(len(eyes), F32(N[j])) for j in range(3)]
    NdotV = np.maximum(OL.dot3(Nc, V), F32(0))
    NdL = np.maximum(OL.dot3(Nc, [F32(x) for x in L]), F32(0))
    den4 = (NdotV * F32(4)) * NdL
    hit = np.flatnonzero(den4 == F32(0.01))
    assert hit.size, "no eye puts den4 on 0.01f"
    return eyes[hit[0]]


def equality(nm, spec, B=4, T=4, seed=7):
    """One mesh (Bv = 1) for four eyes, with a face whose centroid is exactly 0 (key `face`) under the axis light:
        eye 0 = (1e-12f, 0, 0):   V = eye - pos has norm exactly 1e-12f, normalize's eps (sqrt(fl(x^2)) == x);
        eye 1 = (1e-12f, -1, 0):  V = (1e-12f, -1, 0), V + L = (1e-12f, 0, 0): H's norm exactly 1e-12f;
        eye 2: den4 = (N.V * 4) * N.L exactly 0.01f (found by _den4_eye);
        eye 3: an ordinary eye.
    On the normal-map path that face's TBN is the identity, texel 0's tangent-space normal n_t is EPS_TEXEL (norm
    exactly 1e-12f, lit: N.L = 0.8) and its other texels carry the face normal.  spec=False drops the eyes (diffuse branch only)."""
    from oracle import lighting as OL
    rng = np.random.default_rng(seed)
    vb, f = sphere(1, seed)
    vb, f, idx = append(vb, f, ZERO_FACE[None])
    fz = int(idx[0])
    nf = f.shape[0]
    L = F32([0, 1, 0])
    if nm:
        tbn = _tbn(rng, vb, f)[None].astype(F32)
        tbn[0, fz] = np.eye(3, dtype=F32)
        nt = _tangent_normals(rng, (1, nf, T))
        Nf = flat_normals(vb, f)[0, fz].astype(F32)
        nt[0, fz] = Nf
        nt[0, fz, 0] = eps_texel()
        from oracle.numbers import Walk
        N = [x[0] for x in OL._texel_normal(Walk(), F32, [np.atleast_1d(Nf[j]) for j in range(3)],
                                            [np.atleast_1d(F32(x)) for x in np.eye(3, dtype=F32).reshape(-1)])]
    else:
        N, _, _, _ = OL._normal_f64(vb[0][f[fz]].reshape(1, 9).astype(F32), None, F32)
        N = [x[0] for x in N]
    eye = F32([[EPS12, 0, 0], [EPS12, -1, 0], [0, 0, 0], [0.4, 2.2, 1.6]])
    eye[2] = _den4_eye(N, L)
    tex = rng.uniform(0.05, 0.9, (B, nf, T, 3)).astype(F32)
    met, rou = _materials(rng, B, nf, (T,))
    sc = dict(v=vb, f=f, tex=tex, met=met, rou=rou, eye=eye if spec else None,
              gout=rng.uniform(-1, 1, tex.shape).astype(F32), light=AXIS_LIGHT, face=fz)
    if nm:
        sc.update(nt=nt, tbn=tbn)
    return sc


def shared_vertex(n=1000, B=4, nm=False, T=9, seed=8):
    """A fan of n faces around one apex (vertex 0), one mesh (Bv = 1) for B eyes: the apex's grad_vertices entries sum
    3 B n float atomics (the normal-map path: B n), so term_sums' bound carries large n."""
    rng = np.random.default_rng(seed)
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    ring = np.stack([np.cos(ang), 0.3 + 0.05 * np.sin(7 * ang), np.sin(ang)], 1)
    v = np.concatenate([[[0.0, 1.0, 0.0]], ring]).astype(F32)[None]
    f = np.stack([np.zeros(n), 1 + (np.arange(n) + 1) % n, 1 + np.arange(n)], 1).astype(np.int32)
    tex = rng.uniform(0, 1.3, (B, n, T, 3)).astype(F32)
    met, rou = _materials(rng, B, n, (T,))
    sc = dict(v=v, f=f, tex=tex, met=met, rou=rou, eye=EYES4[:B], gout=rng.uniform(-1, 1, tex.shape).astype(F32),
              light=LIGHT)
    if nm:
        sc.update(nt=_tangent_normals(rng, (1, n, T)), tbn=_tbn(rng, v, f)[None].astype(F32))
    return sc
