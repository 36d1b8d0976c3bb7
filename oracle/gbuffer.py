"""Emulation of the G-buffer kernels of csrc/gbuffer_api.cu (TEST INFRASTRUCTURE; product code never imports it):
b200r_gbuffer_lighting_forward (modes normal and depth) and b200r_normal_mapped_gbuffer_forward, in float32, operation
for operation, from the pieces of oracle/lighting.py (face_light, the float64 flat normal, the centroid, the texel
normal) and oracle/preraster.py (camera axes, camera coordinates) that restate the code these kernels share.

    out = clamp01(1 * value + 1 * ((0 + s) * 0)),   value = N * 0.5 + 0.5  or  z / M,   M = max z (NaN if any z is)

Inputs are the kernels' arguments (`args_from_call` turns a recorded `_lib.call` into them).  The backward is held to the
float64 mirror's autograd instead (tests/test_gbuffer_gpu.py).
"""
import numpy as np

from . import lighting as OL
from . import preraster as OP
from .numbers import F32, Walk

FLAT_PTRS = {"b200r_gbuffer_lighting_forward": ("vertices", "faces", "metallic", "roughness", "eye", "camera_eye", "out",
                                                "workspace"),
             "b200r_gbuffer_lighting_backward": ("vertices", "faces", "metallic", "roughness", "eye", "camera_eye",
                                                 "grad_out", "face_depth", "depth_max", "workspace")}
NM_PTRS = {"b200r_normal_mapped_gbuffer_forward": ("vertices", "faces", "normal_textures", "tbn", "metallic", "roughness",
                                                   "eye", "out"),
           "b200r_normal_mapped_gbuffer_backward": ("vertices", "faces", "normal_textures", "tbn", "metallic", "roughness",
                                                    "eye", "grad_out", "grad_normal_textures", "grad_vertices",
                                                    "grad_metallic", "grad_roughness")}
CALLS = tuple(FLAT_PTRS) + tuple(NM_PTRS)
CAMERAS = {0: ("look_at", "right"), 1: ("look", "right"), 2: ("look", "left")}


def _np(x):
    return None if x is None else x.detach().cpu().numpy().copy()


def _light(dir_i, dir_c, d, spec):
    return dict(amb_i=F32(0), amb_c=[F32(0)] * 3, dir_i=F32(dir_i), dir_c=list(np.asarray(list(dir_c), F32)),
                dir=list(np.asarray(list(d), F32)), with_specular=bool(spec))


def args_from_call(name, args):
    """A recorded _lib.call(name, device, *args) of a forward -> dict of the kernel's inputs (numpy copies, None for NULL)
    and its outputs after the call (out; for depth also depth_max)."""
    a = {}
    if name in FLAT_PTRS:
        (v, f, met, rou, eye, ceye, out, ws, nws, dmax, mode, B, Bv, Bf, Be, Bc, nv, nf, T, Tm, dir_i, dir_c, d, spec,
         at, up, cmode) = args
        a.update(vertices=_np(v), faces=_np(f), metallic=_np(met), roughness=_np(rou), eye=_np(eye) if Be else None,
                 camera_eye=_np(ceye), out=_np(out), depth_max=_np(dmax), mode=int(mode), B=B, Bv=Bv, Bf=Bf,
                 Be=Be if Be else 1, Bc=Bc, nv=nv, nf=nf, T=T, Tm=Tm, at=np.asarray(list(at), F32),
                 up=np.asarray(list(up), F32), camera_mode=int(cmode))
    else:
        v, f, nt, tbn, met, rou, eye, out, B, Bv, Bf, Be, Bn, Bt, nv, nf, T, dir_i, dir_c, d, spec = args
        a.update(vertices=_np(v), faces=_np(f), normal_textures=_np(nt), tbn=_np(tbn), metallic=_np(met), roughness=_np(rou),
                 eye=_np(eye) if Be else None, out=_np(out), B=B, Bv=Bv, Bf=Bf, Be=Be if Be else 1, Bn=Bn, Bt=Bt, nv=nv,
                 nf=nf, T=T)
    a["light"] = _light(dir_i, dir_c, d, spec)
    return a


def _compose(value, s):
    """clamp01(1 * value + 1 * ((0 + s) * 0)) per channel."""
    with np.errstate(all="ignore"):
        S = (F32(0) + np.asarray(s, F32)) * F32(0)
        return OL.clamp01(F32(1) * np.asarray(value, F32) + F32(1) * S)


def face_depths(a):
    """k_gb_depth_z: the camera z of every (batch, face) centroid [B, nf], and M = max z (NaN if any z is)."""
    B, nf = a["B"], a["nf"]
    i = np.arange(B * nf)
    b, f = i // nf, i % nf
    v, _ = OL._gather_vertices(a, b, f)
    with np.errstate(all="ignore"):
        pos = np.stack([((v[:, k] + v[:, 3 + k]) + v[:, 6 + k]) / F32(3) for k in range(3)], -1).astype(F32)
        eye = np.broadcast_to(a["camera_eye"].reshape(-1, 3), (B, 3)).astype(F32)
        mode, coord = CAMERAS[a["camera_mode"]]
        r = OP.camera_axes(eye, mode, at=a["at"], direction=a["at"], up=a["up"], coordinate=coord)
        z = OP.to_camera(pos.reshape(B, nf, 3), eye, r)[:, :, 2]
        M = F32(np.max(z))
    return z, M


@OL._quiet
def gbuffer_forward(a):
    """b200r_gbuffer_lighting_forward -> (out [B, nf, T, 3] float32, M or None)."""
    L = a["light"]
    c = OL.const_maker(None)
    B, nf, T = a["B"], a["nf"], a["T"]
    i = np.arange(B * nf)
    _, _, v, _, _, spec, m, r, ey, pos = OL._surface_light_setup(a, i, None, L, c)
    N, _, _, ln = OL._normal_f64(v, None, c)
    N = [np.where(np.isnan(ln), F32(np.nan), x).astype(F32) for x in N]   # a NaN norm makes the whole normal NaN
    _, s = OL.face_light(Walk(), c, N, pos, dict(L, with_specular=spec), ey if spec else None, m, r)
    s = [np.broadcast_to(np.asarray(x, F32), (B * nf,)) for x in s]
    M = None
    if a["mode"] == 0:
        val = [N[k] * F32(0.5) + F32(0.5) for k in range(3)]
    else:
        z, M = face_depths(a)
        val = [(z.reshape(-1) / M).astype(F32)] * 3
    out = np.stack([_compose(val[k], s[k]) for k in range(3)], -1)
    return np.broadcast_to(out[:, None, :], (B * nf, T, 3)).reshape(B, nf, T, 3), M


@OL._quiet
def nm_gbuffer_forward(a):
    """b200r_normal_mapped_gbuffer_forward -> out [B, nf, T, 3] float32."""
    L = a["light"]
    c = OL.const_maker(None)
    B, nf, T = a["B"], a["nf"], a["T"]
    spec = OL._nm_spec(a, L)
    out = np.empty((B, nf, T, 3), F32)
    fc = np.arange(nf)
    for b in range(B):
        bb = np.full(nf, b)
        pos, _ = OL._centroid(a, bb, fc, None, c)
        pos = [OL._per_texel(p, T) for p in pos]
        nt = a["normal_textures"][0 if a["Bn"] == 1 else b].reshape(-1, 3)
        tb = np.repeat(a["tbn"][0 if a["Bt"] == 1 else b].reshape(-1, 9), T, 0)
        w = Walk()
        N = OL._texel_normal(w, c, OL._cols(nt, None), OL._cols(tb, None))
        i = ((b * nf + fc)[:, None] * T + np.arange(T)).reshape(-1)
        m = a["metallic"].reshape(-1)[i] if spec else c(0.0)
        r = a["roughness"].reshape(-1)[i] if spec else c(1.0)
        ey = [OL._per_texel(e, T) for e in OL._eye_rows(a, bb, None)] if spec else None
        _, s = OL.face_light(w, c, N, pos, dict(L, with_specular=spec), ey, m, r)
        s = [np.broadcast_to(np.asarray(x, F32), (nf * T,)) for x in s]
        out[b] = np.stack([_compose(N[k] * F32(0.5) + F32(0.5), s[k]) for k in range(3)], -1).reshape(nf, T, 3)
    return out
