"""Emulation of the G-buffer kernels of csrc/gbuffer_api.cu (TEST INFRASTRUCTURE; product code never imports it):
b200r_gbuffer_lighting_forward (modes normal and depth) and b200r_normal_mapped_gbuffer_forward, in float32, operation
for operation, from the pieces of oracle/lighting.py (face_light, the float64 flat normal, the centroid, the texel
normal) and oracle/preraster.py (camera axes, camera coordinates) that restate the code these kernels share.

    out = clamp01(1 * value + 1 * ((0 + s) * 0)),   value = N * 0.5 + 0.5  or  z / M,   M = max z (NaN if any z is)

Backward (gbuffer_backward, nm_gbuffer_backward), as gb_bwd_face, k_gb_bwd_* and k_nm_gb_bwd form it: the clamp-masked
upstream gradient summed serially over the texels, Gs[c]; the material gradients (Gs * 0) * s' through Dual<2>; the
vertex terms (Gs * 0.5) * dN/dv and (Gs * 0) * ds/dv with their grad_vertices slots; for depth G_f = (Gs0 + Gs1) + Gs2,
dM = -(sum_f G_f z_f) / (M M) and dz_f = G_f / M (+ dM on the faces tied at the max) through z_axis / 3.

The depth reductions are emulated in the kernels' own order, so that face_z, M, face_G, both kernels' partials and dM
come out bit for bit: every thread of the depth_grid(n) blocks folds its grid-stride trips serially, each block folds
its 256 threads in a tree with the stride halving from 128 (block_fold), and fold_partials has thread k take partials
k, k + 256, ... before the same tree.  The max is numpy's (NaN as soon as either is NaN) with +0 > -0.

Every function runs over a number type given by `lift`, as oracle/lighting.py does: None for float32, oracle.numbers.EV
for float64 values with a bound on the float32 evaluation's error (branch decisions replayed from the float32 run).
Inputs are the kernels' arguments (`args_from_call` turns a recorded `_lib.call` into them).
"""
import numpy as np

from . import lighting as OL
from . import preraster as OP
from .numbers import EV, F32, U, Dual, Walk, full, value, where

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
GB_THREADS = 256
GB_PARTIALS = 1024


def _np(x):
    return None if x is None else x.detach().cpu().numpy().copy()


def _light(dir_i, dir_c, d, spec):
    return dict(amb_i=F32(0), amb_c=[F32(0)] * 3, dir_i=F32(dir_i), dir_c=list(np.asarray(list(dir_c), F32)),
                dir=list(np.asarray(list(d), F32)), with_specular=bool(spec))


def args_from_call(name, args):
    """A recorded _lib.call(name, device, *args) -> dict of the kernel's inputs (numpy copies, None for NULL) and what
    it wrote: the forward's out and, for depth, its workspace and depth_max; the backward's requested gradients and,
    for depth, its workspace."""
    a = {}
    if name == "b200r_gbuffer_lighting_forward":
        v, f, met, rou, eye, ceye, out, ws, nws, dmax = args[:10]
        a.update(out=_np(out), workspace=_np(ws), depth_max=_np(dmax))
        rest = args[10:]
    elif name == "b200r_gbuffer_lighting_backward":
        v, f, met, rou, eye, ceye, gout, fz, dmax, ws, nws, gv, gm, gr = args[:14]
        a.update(grad_out=_np(gout), face_depth=_np(fz), depth_max=_np(dmax), workspace=_np(ws), grad_vertices=_np(gv),
                 grad_metallic=_np(gm), grad_roughness=_np(gr))
        rest = args[14:]
    elif name == "b200r_normal_mapped_gbuffer_forward":
        v, f, nt, tbn, met, rou, eye, out = args[:8]
        a.update(out=_np(out))
        rest = args[8:]
    else:
        v, f, nt, tbn, met, rou, eye, gout, gn, gv, gm, gr = args[:12]
        a.update(grad_out=_np(gout), grad_normal_textures=_np(gn), grad_vertices=_np(gv), grad_metallic=_np(gm),
                 grad_roughness=_np(gr))
        rest = args[12:]
    a.update(vertices=_np(v), faces=_np(f), metallic=_np(met), roughness=_np(rou))
    if name in FLAT_PTRS:
        mode, B, Bv, Bf, Be, Bc, nv, nf, T, Tm, dir_i, dir_c, d, spec, at, up, cmode = rest
        a.update(eye=_np(eye) if Be else None, camera_eye=_np(ceye), mode=int(mode), B=B, Bv=Bv, Bf=Bf,
                 Be=Be if Be else 1, Bc=Bc, nv=nv, nf=nf, T=T, Tm=Tm, at=np.asarray(list(at), F32),
                 up=np.asarray(list(up), F32), camera_mode=int(cmode))
    else:
        B, Bv, Bf, Be, Bn, Bt, nv, nf, T, dir_i, dir_c, d, spec = rest
        a.update(normal_textures=_np(nt), tbn=_np(tbn), eye=_np(eye) if Be else None, B=B, Bv=Bv, Bf=Bf,
                 Be=Be if Be else 1, Bn=Bn, Bt=Bt, nv=nv, nf=nf, T=T)
    a["light"] = _light(dir_i, dir_c, d, spec)
    return a


def _compose(value, s):
    """clamp01(1 * value + 1 * ((0 + s) * 0)) per channel."""
    with np.errstate(all="ignore"):
        S = (F32(0) + np.asarray(s, F32)) * F32(0)
        return OL.clamp01(F32(1) * np.asarray(value, F32) + F32(1) * S)


# ---- the depth passes' reductions --------------------------------------------------------------------------------------

def depth_grid(n):
    """Blocks of k_gb_depth_z and k_gb_bwd_depth_fold, and so partials per reduction."""
    return min(n // GB_THREADS + 1, GB_PARTIALS)


def nan_max(a, b):
    """The kernels' nan_max on float32 arrays: a if a is NaN, else b if b is NaN, else the larger, +0 above -0."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    with np.errstate(invalid="ignore"):
        take = ~np.isnan(a) & (np.isnan(b) | (b > a) | ((b == a) & np.signbit(a) & ~np.signbit(b)))
    return np.where(take, b, a)


def _add(a, b):
    return a + b


def _fill(proto, n, x):
    return EV(np.full(n, x)) if isinstance(proto, EV) else np.full(n, F32(x), F32)


def _join(a, b):
    if isinstance(a, EV):
        return EV(np.concatenate([a.v, b.v]), np.concatenate([a.e, b.e]))
    return np.concatenate([a, b])


def _stack(xs, axis=-1):
    if any(isinstance(x, EV) for x in xs):
        xs = [EV.of(x) for x in xs]
        return EV(np.stack([x.v for x in xs], axis), np.stack([x.e for x in xs], axis))
    return np.stack([np.asarray(x, F32) for x in xs], axis)


def _tree(x, op):
    """block_fold over the last axis (256 threads): sh[k] = op(sh[k], sh[k + s]) for s = 128, 64, ..., 1."""
    s = GB_THREADS // 2
    while s:
        x = op(x[..., :s], x[..., s:2 * s])
        s //= 2
    return x[..., 0]


def fold(x, blocks, op, init):
    """Thread t of `blocks` blocks of 256 folds x[t], x[t + 256 blocks], ... in order from init, then each block its
    threads with block_fold's tree -> one value per block.  blocks = depth_grid(n) is the grid-stride pass,
    blocks = 1 is fold_partials."""
    n, stride = x.shape[0], blocks * GB_THREADS
    acc = _fill(x, stride, init)
    for s0 in range(0, n, stride):
        k = min(stride, n - s0)
        acc = _join(op(acc[:k], x[s0:s0 + k]), acc[k:])
    return _tree(OL._reshape(acc, (blocks, GB_THREADS)), op)


def _camera(a):
    """The camera eye rows [B, 3] and the float32 camera axes [B, 3, 3] (rows x, y, z) the kernels form."""
    B = a["B"]
    eye = np.broadcast_to(a["camera_eye"].reshape(-1, 3), (B, 3)).astype(F32)
    mode, coord = CAMERAS[a["camera_mode"]]
    return eye, OP.camera_axes(eye, mode, at=a["at"], direction=a["at"], up=a["up"], coordinate=coord)


def _axis(r, lift):
    """A float32 camera-axis component in the number type: with EV, within 8 ulps of the float64 unit axis (the
    normalize's roundings)."""
    return r if lift is None else EV(np.asarray(r, np.float64), 8 * U)


def face_depths(a, lift=None):
    """k_gb_depth_z and the fold of its partials: the camera z of every (batch, face) centroid [B * nf], the partial
    maxima [depth_grid(n)] and M.  With EV, z is held to the float64 depth and M to the float64 max (the max of
    values each within its bound moves by at most the largest bound); the partials are None."""
    c = OL.const_maker(lift)
    n, nf = a["B"] * a["nf"], a["nf"]
    i = np.arange(n)
    b = i // nf
    v, _ = OL._gather_vertices(a, b, i % nf)
    vl = OL._cols(v, lift)
    eye, r = _camera(a)
    d = [((vl[k] + vl[3 + k]) + vl[6 + k]) / c(3.0) - OL._fl(eye[b, k], lift) for k in range(3)]
    rz = [_axis(r[b, 2, k], lift) for k in range(3)]
    z = (d[0] * rz[0] + d[1] * rz[1]) + d[2] * rz[2]
    if lift is not None:
        return z, None, EV(np.max(z.v), np.max(z.e))
    partials = fold(z, depth_grid(n), nan_max, -np.inf)
    return z, partials, fold(partials, 1, nan_max, -np.inf)[0]


@OL._quiet
def gbuffer_forward(a):
    """b200r_gbuffer_lighting_forward -> (out [B, nf, T, 3] float32, M: depth_max, or None in normal mode).  The
    workspace's used prefix after a depth forward is face_depths(a)'s z and partials."""
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
        z, _, M = face_depths(a)
        val = [(z / M).astype(F32)] * 3
    out = np.stack([_compose(val[k], s[k]) for k in range(3)], -1)
    return np.broadcast_to(out[:, None, :], (B * nf, T, 3)).reshape(B, nf, T, 3), M


def _nan_at(bad, x):
    """x with NaN where bad (float32 or EV)."""
    if isinstance(x, EV):
        return EV(np.where(bad, np.nan, x.v), x.e)
    return np.where(bad, F32(np.nan), x).astype(F32)


def _material_duals(w, c, N, pos, L, ey, m, r, Gs):
    """sum_c (Gs[c] * 0) * ds[c]/d(metallic, roughness), through face_light's Dual<2>."""
    zero = full(m, 0)
    _, sm = OL.face_light(w, c, N, pos, L, ey, Dual(m, [zero + c(1.0), zero]), Dual(r, [zero, zero + c(1.0)]))
    gm, gr = c(0.0), c(0.0)
    for k in range(3):
        gm = gm + (Gs[k] * c(0.0)) * sm[k].d[0]
        gr = gr + (Gs[k] * c(0.0)) * sm[k].d[1]
    return gm, gr


@OL._quiet
def gbuffer_backward(a, lift=None, replay=None):
    """b200r_gbuffer_lighting_backward (k_gb_bwd_normal, or k_gb_bwd_depth_fold then k_gb_bwd_depth_scatter).  Returns
    dict: metallic, roughness (gradients shaped like the inputs, None where not requested); vertex_slots / vertex_terms
    [n, 9] (flat grad_vertices indices and the float atomics' terms, both depth kernels' in depth mode); walks; near
    (kink flags per (batch, face), by kind).  For depth also: face_G [B * nf] and partials [depth_grid(n)] (the
    workspace after the call; float32 only), dM, and tie (the faces dM reaches).  replay: the float32 run's result."""
    c = OL.const_maker(lift)
    L = OL._lift_light(a["light"], lift)
    B, nf, T, Tm, nv = a["B"], a["nf"], a["T"], a["Tm"], a["nv"]
    n = B * nf
    depth = a["mode"] == 1
    go = a["grad_out"].reshape(n, T, 3)
    want_mat = a.get("grad_metallic") is not None or a.get("grad_roughness") is not None
    want_v = a.get("grad_vertices") is not None
    if depth:
        if lift is None and a.get("face_depth") is not None:   # the forward's workspace and max, as the kernels read them
            z, M = a["face_depth"][:n], a["depth_max"].reshape(-1)[0]
        else:
            z, _, M = face_depths(a, lift)
    mats, slots, terms, walks, near, Gf = [], [], [], [], [], []
    sizes = []
    for ci, i in enumerate(OL._chunks(n, T)):
        sizes.append(len(i))
        w = Walk(replay["walks"][ci] if replay is not None else None)
        b, f, v, vl, fi, spec, m, r, ey, pos = OL._surface_light_setup(a, i, lift, L, c)
        Nval, Njac, n32, ln = OL._normal_f64(v, lift, c)
        bad = np.isnan(value(ln))   # the kernel makes the whole normal, and its Jacobian, NaN
        Nval, Njac = [_nan_at(bad, x) for x in Nval], [_nan_at(bad, x) for x in Njac]
        Ls = dict(L, with_specular=spec)
        _, s = OL.face_light(w, c, Nval, pos, Ls, ey if spec else None, m, r)
        Gs = []
        for k in range(3):
            val = z[i] / M if depth else Nval[k] * c(0.5) + c(0.5)
            x = c(1.0) * val + c(1.0) * ((c(0.0) + s[k]) * c(0.0))
            mask = OL._clamp_mask(w, c, x)
            g = c(0.0)
            for t in range(T):
                g = g + where(mask, OL._fl(go[i, t, k], lift), c(0.0))
            Gs.append(g)
        if want_mat:
            gm, gr = c(0.0), c(0.0)
            if spec:
                gm, gr = _material_duals(w, c, Nval, pos, Ls, ey, m, r, Gs)
                gm, gr = gm / c(float(Tm)), gr / c(float(Tm))
            mats.append((gm, gr))
        if want_v and (not depth or spec):
            dv, Nd = OL.normal_duals(w, c, vl, Nval, Njac, n32, ln, lift)
            Nd = [Dual(x.v, [_nan_at(bad, p) for p in x.d]) for x in Nd]
            acc = [c(0.0)] * 9
            if not depth:
                for k in range(9):
                    for cc in range(3):
                        acc[k] = acc[k] + (Gs[cc] * c(0.5)) * Nd[cc].d[k]
            if spec:
                pd = [((dv[k] + dv[3 + k]) + dv[6 + k]) / c(3.0) for k in range(3)]
                _, sd = OL.face_light(w, c, Nd, pd, Ls, ey, m, r)
                for k in range(9):
                    for cc in range(3):
                        acc[k] = acc[k] + (Gs[cc] * c(0.0)) * sd[cc].d[k]
            vbase = np.where(a["Bv"] == 1, 0, b) * nv * 3
            slots.append(np.stack([vbase + fi[:, k // 3] * 3 + k % 3 for k in range(9)], 1))
            terms.append(acc)
        if depth:
            Gf.append((Gs[0] + Gs[1]) + Gs[2])
        walks.append(w)
        near.append(w.near)
    res = dict(walks=walks, near=OL._near(near))
    for j, k in enumerate(("metallic", "roughness")):
        res[k] = None
        if want_mat and a.get("grad_" + k) is not None:
            res[k] = OL._reshape(OL._rep(OL._cat1([p[j] for p in mats], sizes, lift), Tm), a[k].shape)
    if depth:
        G = OL._cat1(Gf, sizes, lift)
        partials = fold(G * z, depth_grid(n), _add, 0.0)
        dM = -fold(partials, 1, _add, 0.0)[0] / (M * M)
        res.update(face_G=G if lift is None else None, partials=partials if lift is None else None, dM=dM)
        if want_v:
            tie = value(z) == value(M) if replay is None else replay["tie"]
            if lift is not None:   # members within their bound of the tie that float64 may decide the other way
                d = z - M
                res["near"]["tie"] = (np.abs(d.v) <= d.e) & ~(tie & (d.v == 0))
            res["tie"] = tie
            bb = np.arange(n) // nf
            shared = a["Bv"] == 1 and a["Bf"] == 1 and a["Bc"] == 1   # one [1, nf] set of depths: each tie once, at b = 0
            once = (bb == 0) | (not shared)
            dz = G / M
            dz = where(once, dz + dM * np.asarray(tie, F32 if lift is None else np.float64), dz)
            _, r = _camera(a)
            fi = a["faces"][np.where(a["Bf"] == 1, 0, bb), np.arange(n) % nf]
            vbase = np.where(a["Bv"] == 1, 0, bb) * nv * 3
            gk = [(dz * _axis(r[bb, 2, k], lift)) / c(3.0) for k in range(3)]
            slots.append(np.stack([vbase + fi[:, j] * 3 + k for k in range(3) for j in range(3)], 1))
            terms.append([gk[k] for k in range(3) for j in range(3)])
    if want_v:
        res["vertex_slots"] = np.concatenate(slots) if slots else np.zeros((0, 9), np.int64)
        res["vertex_terms"] = OL._cat(terms, lift) if terms else np.zeros((0, 9), F32)
    return res


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


@OL._quiet
def nm_gbuffer_backward(a, lift=None, replay=None):
    """b200r_normal_mapped_gbuffer_backward (k_nm_gb_bwd).  Returns dict: normal_textures [Bn, nf, T, 3] (with a batch-1
    normal texture the serial sum over b = 0, 1, ...), metallic, roughness (per texel; None where not requested),
    vertex_slots / vertex_terms [n, 9] (each texel's gk[3 + k] / 3 on its face's three vertices), walks, near (kink
    flags [B, nf, T] by kind).  replay: the float32 run's result."""
    c = OL.const_maker(lift)
    L = OL._lift_light(a["light"], lift)
    B, nf, T, Bn, nv = a["B"], a["nf"], a["T"], a["Bn"], a["nv"]
    spec = OL._nm_spec(a, L)
    Ls = dict(L, with_specular=spec)
    want = {k: a.get("grad_" + k) is not None for k in ("normal_textures", "vertices", "metallic", "roughness")}
    zeros = (lambda *s: np.zeros(s, F32)) if lift is None else (lambda *s: EV(np.zeros(s)))
    gn, gmat = zeros(Bn, nf, T, 3), [zeros(B, nf, T), zeros(B, nf, T)]
    slots, terms, walks, near = [], [], [], {}
    ci = 0
    for b in range(B):
        bn = 0 if Bn == 1 else b
        for fc in OL._chunks(nf, T):
            w = Walk(replay["walks"][ci] if replay is not None else None)
            ci += 1
            nfc = len(fc)
            bb = np.full(nfc, b)
            pos, fi = OL._centroid(a, bb, fc, lift, c)
            post = [OL._per_texel(p, T) for p in pos]
            tb = OL._cols(np.repeat(a["tbn"][0 if a["Bt"] == 1 else b, fc].reshape(-1, 9), T, 0), lift)
            ey = [OL._per_texel(e, T) for e in OL._eye_rows(a, bb, lift)] if spec else None
            i = ((b * nf + fc)[:, None] * T + np.arange(T)).reshape(-1)
            nt = OL._cols(a["normal_textures"][bn, fc].reshape(-1, 3), lift)
            N = OL._texel_normal(w, c, nt, tb)
            m = OL._fl(a["metallic"].reshape(-1)[i], lift) if spec else c(0.0)
            r = OL._fl(a["roughness"].reshape(-1)[i], lift) if spec else c(1.0)
            _, s = OL.face_light(w, c, N, post, Ls, ey, m, r)
            Gs = []
            for k in range(3):
                x = c(1.0) * (N[k] * c(0.5) + c(0.5)) + c(1.0) * ((c(0.0) + s[k]) * c(0.0))
                mask = OL._clamp_mask(w, c, x)
                Gs.append(where(mask, OL._fl(a["grad_out"].reshape(-1, 3)[i, k], lift), c(0.0)))
            if want["metallic"] or want["roughness"]:
                gm, gr = _material_duals(w, c, N, post, Ls, ey, m, r, Gs) if spec else (c(0.0), c(0.0))
                for j, g in enumerate((gm, gr)):
                    gmat[j][b, fc] = OL._reshape(OL._broad(g, nfc * T) if lift is not None else
                                                 np.broadcast_to(np.asarray(g, F32), (nfc * T,)), (nfc, T))
            if want["normal_textures"] or (want["vertices"] and spec):
                zero = full(nt[0], 0)
                one = zero + c(1.0)
                ntd = [Dual(nt[k], [one if j == k else zero for j in range(6)]) for k in range(3)]
                pd = [Dual(post[k] + zero, [one if j == 3 + k else zero for j in range(6)]) for k in range(3)]
                Nd = OL._texel_normal(w, c, ntd, tb)
                gk = []
                for k in range(6):
                    acc = c(0.0)
                    for cc in range(3):
                        acc = acc + (Gs[cc] * c(0.5)) * Nd[cc].d[k]
                    gk.append(acc)
                if spec:
                    _, sd = OL.face_light(w, c, Nd, pd, Ls, ey, m, r)
                    for k in range(6):
                        for cc in range(3):
                            gk[k] = gk[k] + (Gs[cc] * c(0.0)) * sd[cc].d[k]
                if want["normal_textures"]:
                    gn[bn, fc] = gn[bn, fc] + OL._reshape(_stack([OL._broad(x, nfc * T) for x in gk[:3]]), (nfc, T, 3))
                if want["vertices"]:
                    gv = [gk[3 + k] / c(3.0) for k in range(3)]
                    fit = np.repeat(fi, T, 0)
                    vrow = (0 if a["Bv"] == 1 else b) * nv
                    slots.append(np.stack([(vrow + fit[:, j]) * 3 + k for k in range(3) for j in range(3)], 1))
                    terms.append([gv[k] for k in range(3) for j in range(3)])
            walks.append(w)
            for kk, fl in w.near.items():
                near.setdefault(kk, np.zeros((B, nf, T), bool))[b, fc] |= np.broadcast_to(
                    np.asarray(fl, bool), (nfc * T,)).reshape(nfc, T)
    out = dict(walks=walks, near=near, normal_textures=gn if want["normal_textures"] else None)
    for j, k in enumerate(("metallic", "roughness")):
        out[k] = OL._reshape(gmat[j], a[k].shape) if want[k] else None
    if want["vertices"]:
        out["vertex_slots"] = np.concatenate(slots) if slots else np.zeros((0, 9), np.int64)
        out["vertex_terms"] = OL._cat(terms, lift) if terms else np.zeros((0, 9), F32)
    return out
