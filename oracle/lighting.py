"""Emulation of the fused surface-lighting kernels of csrc/lighting_api.cu (TEST INFRASTRUCTURE; product code never
imports it): b200r_surface_lighting_{forward,backward} and b200r_normal_mapped_lighting_{forward,backward}.

The kernels are built with -fmad=false, use no transcendental function beyond IEEE sqrtf and division, and form the flat
normal in double, so every per-thread value is a fixed sequence of float32 operations.  This module restates them
operation for operation -- face_light, normalize3, dot3's order, `acc += a + b` as acc + (a + b), mean_tm's serial sum,
the normal-map backward's lane assignment (t = lane, lane + 32, ...) and its xor butterfly as lane 0 sees it -- over a
number type given by `lift`:
    lift=None  numpy float32: lit textures and per-texel gradients bit for bit, grad_vertices term by term;
    lift=EV    oracle.numbers.EV: float64 values of the same expressions with a bound on the float32 evaluation's error,
               branch decisions replayed from a float32 walk (oracle.numbers.Walk).
Only the float atomics into grad_vertices depend on the order of execution; for them each kernel term is returned with its
slot, for oracle.preraster.term_sums.

Inputs are the arguments the kernels receive (`args_from_call` turns a recorded `_lib.call` into them): numpy arrays for
the device pointers (None for NULL), the counts, and the light parameters with the host-normalised direction.
"""
import numpy as np

from .numbers import EV, F32, Dual, Walk, dclamp_min, dmax, full, sqrt, where

SURFACE_COUNTS = ("B", "Bv", "Bf", "Be", "nv", "nf", "T", "Tm")
NM_COUNTS = ("B", "Bv", "Bf", "Be", "Bn", "n_nf", "n_T", "Bt", "t_nf", "nv", "nf", "T")
SURFACE_PTRS = {"b200r_surface_lighting_forward": ("vertices", "faces", "textures", "metallic", "roughness", "eye", "out"),
                "b200r_surface_lighting_backward": ("vertices", "faces", "textures", "metallic", "roughness", "eye",
                                                    "grad_out", "grad_textures", "grad_vertices", "grad_metallic",
                                                    "grad_roughness")}
NM_PTRS = {"b200r_normal_mapped_lighting_forward": ("vertices", "faces", "textures", "normal_textures", "tbn", "metallic",
                                                    "roughness", "eye", "out"),
           "b200r_normal_mapped_lighting_backward": ("vertices", "faces", "textures", "normal_textures", "tbn", "metallic",
                                                     "roughness", "eye", "grad_out", "grad_textures",
                                                     "grad_normal_textures", "grad_vertices", "grad_metallic",
                                                     "grad_roughness")}
CALLS = tuple(SURFACE_PTRS) + tuple(NM_PTRS)
CHUNK = 1 << 19   # members (faces or texels) per emulated chunk


def args_from_call(name, args):
    """A recorded _lib.call(name, device, *args) -> dict of the kernel's inputs: numpy copies of the tensors (None for
    NULL), ints, and the light (floats as the C ABI receives them: float32)."""
    ptrs = SURFACE_PTRS.get(name) or NM_PTRS[name]
    counts = SURFACE_COUNTS if name in SURFACE_PTRS else NM_COUNTS
    out = {}
    for k, x in zip(ptrs, args):
        out[k] = None if x is None else x.detach().cpu().numpy().copy()
    rest = args[len(ptrs):]
    out.update(zip(counts, (int(x) for x in rest[:len(counts)])))
    amb_i, amb_c, dir_i, dir_c, d, spec = rest[len(counts):]
    out["light"] = dict(amb_i=F32(amb_i), amb_c=np.asarray(list(amb_c), F32), dir_i=F32(dir_i),
                        dir_c=np.asarray(list(dir_c), F32), dir=np.asarray(list(d), F32), with_specular=bool(spec))
    return out


def const_maker(lift):
    """Kernel float constants in the number type: float32, or an EV whose value is the float64 constant the op-by-op
    mirror uses and whose error is the float32 literal's distance from it."""
    if lift is None:
        return F32

    def c(x):
        x = np.float64(x)
        return EV(x, abs(np.float64(F32(x)) - x))
    return c


def light_ev(light, with_specular):
    """The light of a Lighting(**kwargs) as the float64 mirror sees it, as EV constants around the float32 values the
    kernel gets (the direction F.normalize'd in float64)."""
    c = const_maker(EV)
    d = np.asarray(light["directions"], np.float64)
    d = d / max(np.sqrt((d * d).sum()), 1e-12)
    d32 = np.asarray(d, F32)   # bound of the host's float32 normalize: a few ulps
    return dict(amb_i=c(light["intensity_ambient"]), amb_c=[c(x) for x in light["color_ambient"]],
                dir_i=c(light["intensity_directionals"]), dir_c=[c(x) for x in light["color_directionals"]],
                dir=[EV(d[k], abs(np.float64(d32[k]) - d[k]) + 4 * 2.0 ** -24) for k in range(3)],
                with_specular=bool(with_specular))


def _lift_light(light, lift):
    if lift is None:
        return dict(light, amb_c=list(light["amb_c"]), dir_c=list(light["dir_c"]), dir=list(light["dir"]))
    return light


def _is_dual(x):
    return isinstance(x, Dual)


def _lift_to(x, proto):
    """lift<R>(x): a plain value to a Dual with zero partials when R (proto's type) is a Dual."""
    if _is_dual(proto) and not _is_dual(x):
        return Dual(x, [full(x, 0)] * len(proto.d))
    return x


def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def normalize3(w, x, eps):
    n = dclamp_min(w, "norm_eps", sqrt(dot3(x, x)), eps)
    return [x[k] / n for k in range(3)]


def face_light(w, c, N, pos, L, eye, metallic, roughness):
    """face_light: (diffuse[3], specular[3]) of normal N and position pos; eye None for the diffuse-only branch."""
    zero = c(0.0)
    cosine = dmax(w, "relu", dot3(N, L["dir"]), zero)
    R = next((x for x in (N[0], metallic) if _is_dual(x)), None)
    diffuse = [_lift_to(zero + L["amb_i"] * L["amb_c"][k], R) for k in range(3)]
    one = c(1.0)
    if eye is not None:
        V = normalize3(w, [eye[k] - pos[k] for k in range(3)], c(1e-12))
        H = normalize3(w, [V[k] + L["dir"][k] for k in range(3)], c(1e-12))
        a = roughness * roughness
        a2 = a * a
        NdotH = dmax(w, "relu", dot3(N, H), zero)
        den = (NdotH * NdotH) * (a2 - one) + one
        den = (den * c(3.1415)) * den
        NDF = _lift_to(a2, R) / den
        r1 = roughness + one
        k_ = (r1 * r1) / c(8.0)
        NdotV = dmax(w, "relu", dot3(N, V), zero)
        NdotL = dmax(w, "relu", dot3(N, L["dir"]), zero)
        G = (_lift_to(NdotL, R) / (NdotL * (one - k_) + k_)) * (_lift_to(NdotV, R) / (NdotV * (one - k_) + k_))
        hv = one - dmax(w, "relu", dot3(H, V), zero)
        hv2 = hv * hv
        p5 = (hv2 * hv2) * hv
        den4 = dclamp_min(w, "den4", (NdotV * c(4.0)) * NdotL, c(0.01))
        ndf_g = NDF * G
        specular = []
        for k in range(3):
            F0 = c(0.4) * (one - metallic) + one * metallic
            Fr = F0 + (one - F0) * p5
            radiance = (cosine * L["dir_c"][k]) * L["dir_i"]
            KD = (one - Fr) * (one - metallic)
            diffuse[k] = diffuse[k] + KD * radiance
            specular.append(((ndf_g * Fr) / den4) * radiance)
    else:
        for k in range(3):
            diffuse[k] = diffuse[k] + (cosine * L["dir_c"][k]) * L["dir_i"]
        specular = [_lift_to(zero, R)] * 3
    return diffuse, specular


def _clamp_mask(w, c, val):
    """torch.clamp(x, 0, 1) passes the gradient on [0, 1]: (val >= 0) & (val <= 1), NaN false."""
    with np.errstate(invalid="ignore"):
        lo = w.decide("clamp", val, c(0.0), lambda a, lo: np.asarray(a) >= lo)
        hi = w.decide("clamp", val, c(1.0), lambda a, lo: np.asarray(a) <= lo)
    return lo & hi


def clamp01(x):
    with np.errstate(invalid="ignore"):
        return np.where(x != x, x, np.minimum(np.maximum(x, F32(0)), F32(1))).astype(F32)


def _fl(x, lift):
    """A float32 input array in the number type."""
    x = np.asarray(x, F32)
    return x if lift is None else lift(x)


def _cols(x, lift):
    return [_fl(x[..., k], lift) for k in range(x.shape[-1])]


def _normal_f64(v, lift, c):
    """normal_f64: the float32 edge vectors, their float64 cross product normalised and rounded to float32.  Returns
    (N as the value path sees it, N as the Jacobian sees it, n = (float)fmax(len, 1e-12), len).  With EV the value is
    the mirror's (float64 edges, `.float()` of the normal), the Jacobian's normal its unrounded float64 one, and the
    errors bound the kernel's float32 edges and roundings."""
    if lift is None:
        a = [(v[:, k] - v[:, 3 + k]).astype(np.float64) for k in range(3)]
        b = [(v[:, 6 + k] - v[:, 3 + k]).astype(np.float64) for k in range(3)]
        cr = [b[1] * a[2] - b[2] * a[1], b[2] * a[0] - b[0] * a[2], b[0] * a[1] - b[1] * a[0]]
        with np.errstate(invalid="ignore"):
            ln = np.sqrt((cr[0] * cr[0] + cr[1] * cr[1]) + cr[2] * cr[2])
            n = np.fmax(ln, 1e-12)
            N = [(cr[k] / n).astype(F32) for k in range(3)]
        return N, N, n.astype(F32), ln
    x = [EV(np.asarray(v[:, k], np.float64)) for k in range(9)]
    a = [x[k] - x[3 + k] for k in range(3)]
    b = [x[6 + k] - x[3 + k] for k in range(3)]
    av, ae = np.stack([p.v for p in a]), np.stack([p.e for p in a])
    bv, be = np.stack([p.v for p in b]), np.stack([p.e for p in b])
    with np.errstate(all="ignore"):
        cv = np.cross(bv.T, av.T).T
        prods = np.abs(bv)[[1, 2, 0]] * np.abs(av)[[2, 0, 1]] + np.abs(bv)[[2, 0, 1]] * np.abs(av)[[1, 2, 0]]
        ce = (np.abs(bv)[[1, 2, 0]] * ae[[2, 0, 1]] + np.abs(av)[[2, 0, 1]] * be[[1, 2, 0]] + be[[1, 2, 0]] * ae[[2, 0, 1]]
              + np.abs(bv)[[2, 0, 1]] * ae[[1, 2, 0]] + np.abs(av)[[1, 2, 0]] * be[[2, 0, 1]] + be[[2, 0, 1]] * ae[[1, 2, 0]]
              + 4 * 2.0 ** -52 * prods)
        ln = np.sqrt((cv * cv).sum(0))
        le = np.sqrt((ce * ce).sum(0)) + 8 * 2.0 ** -52 * ln
        n = np.fmax(ln, 1e-12)
        lo = np.where(ln > 1e-12, ln - le, 1e-12)
        dirv = np.where(lo > 0, 2 * np.sqrt((ce * ce).sum(0)) / np.maximum(lo, 1e-300), np.inf)
        N64 = cv / n
        N32 = N64.astype(F32).astype(np.float64)
        u = 2.0 ** -24
        Nval = [EV(N32[k], dirv + 2 * u * np.abs(N32[k])) for k in range(3)]
        Njac = [EV(N64[k], dirv + u * np.abs(N64[k])) for k in range(3)]
        n32 = EV(n, le + u * n)
    return Nval, Njac, n32, EV(ln, le)


def normal_duals(w, c, vl, Nval, Njac, n32, ln, lift):
    """normal_duals: the corners as Dual<9> variables dv, and the normal Nd with value Nval and partials of the float32
    cross product's duals through (I - N N^T) / |c| (Njac for N, n32 for |c|), or I / 1e-12 on normalize's eps path
    (decided on ln, the unclamped norm).  Returns (dv, Nd)."""
    zero = full(vl[0], 0)
    one = zero + c(1.0)
    dv = [Dual(vl[k], [one if j == k else zero for j in range(9)]) for k in range(9)]
    ae = [dv[0] - dv[3], dv[1] - dv[4], dv[2] - dv[5]]
    be = [dv[6] - dv[3], dv[7] - dv[4], dv[8] - dv[5]]
    cr = [be[1] * ae[2] - be[2] * ae[1], be[2] * ae[0] - be[0] * ae[2], be[0] * ae[1] - be[1] * ae[0]]
    inv = c(1.0) / n32
    st = w.decide("norm_eps", ln, np.float64(1e-12) if lift is None else EV(1e-12),
                  lambda x, lo: np.where(np.asarray(x) >= lo, 1, 0).astype(np.int8))
    on_eps = st != 1
    Nd = []
    for j in range(3):
        parts = []
        for k in range(9):
            Ndc = where(on_eps, zero, (Njac[0] * cr[0].d[k] + Njac[1] * cr[1].d[k]) + Njac[2] * cr[2].d[k])
            parts.append((cr[j].d[k] - Njac[j] * Ndc) * inv)
        Nd.append(Dual(Nval[j], parts))
    return dv, Nd


def _gather_vertices(a, b, f):
    """The three corners of faces f of batch elements b, [n, 9] float32, and their vertex indices [n, 3]."""
    fi = a["faces"][np.where(a["Bf"] == 1, 0, b), f]
    bv = np.broadcast_to(np.where(a["Bv"] == 1, 0, b), np.shape(b))
    v = np.concatenate([a["vertices"][bv, fi[:, k]] for k in range(3)], axis=1)
    return v, fi


def _mean_tm(p, c):   # serial sum, then / (float)Tm
    s = c(0.0)
    for t in range(p.shape[1]):
        s = s + p[:, t]
    return s / c(float(p.shape[1]))


def _eye_rows(a, b, lift):
    e = a["eye"][np.where(a["Be"] == 1, 0, b)]
    return _cols(e, lift)


def _surface_light_setup(a, i, lift, L, c):
    nf = a["nf"]
    b, f = i // nf, i % nf
    v, fi = _gather_vertices(a, b, f)
    spec = L["with_specular"] and a["metallic"] is not None and a["roughness"] is not None and a["eye"] is not None
    Tm = a["Tm"]
    if spec:
        m = _mean_tm(_fl(a["metallic"].reshape(-1, Tm)[i], lift), c)
        r = _mean_tm(_fl(a["roughness"].reshape(-1, Tm)[i], lift), c)
        ey = _eye_rows(a, b, lift)
    else:
        m, r, ey = c(0.0), c(1.0), None
    vl = _cols(v, lift)
    pos = [((vl[k] + vl[3 + k]) + vl[6 + k]) / c(3.0) for k in range(3)]
    return b, f, v, vl, fi, spec, m, r, ey, pos


def _chunks(n, per):
    step = max(1, CHUNK // max(per, 1))
    for s in range(0, n, step):
        yield np.arange(s, min(n, s + step))


def _quiet(fn):
    """Non-finite inputs and the eps paths divide by zero and make NaNs on purpose, as the kernels do."""
    import functools

    @functools.wraps(fn)
    def run(*args, **kw):
        with np.errstate(all="ignore"):
            return fn(*args, **kw)
    return run


@_quiet
def surface_forward(a, lift=None):
    """k_surface_lighting_fwd -> lit textures shaped like a['textures'] (float32; EV with lift=EV)."""
    c = const_maker(lift)
    L = _lift_light(a["light"], lift)
    nf, B, T = a["nf"], a["B"], a["T"]
    tx = a["textures"].reshape(B * nf, T, 3)
    parts = []
    for i in _chunks(B * nf, T):
        w = Walk()
        _, _, v, _, _, spec, m, r, ey, pos = _surface_light_setup(a, i, lift, L, c)
        N, _, _, _ = _normal_f64(v, lift, c)
        d, s = face_light(w, c, N, pos, L, ey, m, r)
        parts.append(np.stack([clamp01(tx[i, :, k] * d[k][:, None] + np.broadcast_to(s[k], d[k].shape)[:, None])
                               for k in range(3)], -1))
    return np.concatenate(parts).reshape(a["textures"].shape)


@_quiet
def surface_backward(a, lift=None, replay=None):
    """k_surface_lighting_bwd.  Returns dict: textures, metallic, roughness (per-texel gradients shaped like the inputs,
    None where the kernel writes nothing), vertex_slots [n, 9] (flat indices into grad_vertices) and vertex_terms
    [n, 9] (the kernel's `acc`, atomically added where != 0), walks (one per chunk, for replay) and, with EV, near
    (kink flags per face, by kind).  replay: the float32 run's result, whose branch decisions an EV run takes."""
    c = const_maker(lift)
    L = _lift_light(a["light"], lift)
    nf, B, T, Tm, nv = a["nf"], a["B"], a["T"], a["Tm"], a["nv"]
    tx = a["textures"].reshape(B * nf, T, 3)
    go = a["grad_out"].reshape(B * nf, T, 3)
    want_mat = a.get("grad_metallic") is not None or a.get("grad_roughness") is not None
    want_v = a.get("grad_vertices") is not None
    out = dict(textures=[], metallic=[], roughness=[], vertex_slots=[], vertex_terms=[], walks=[], near=[])
    for ci, i in enumerate(_chunks(B * nf, T)):
        w = Walk(replay["walks"][ci] if replay is not None else None)
        b, f, v, vl, fi, spec, m, r, ey, pos = _surface_light_setup(a, i, lift, L, c)
        Nval, Njac, n32, ln = _normal_f64(v, lift, c)
        d, s = face_light(w, c, Nval, pos, L, ey if spec else None, m, r)
        gt = []
        Gd, Gs = [c(0.0)] * 3, [c(0.0)] * 3
        for k in range(3):
            x = _fl(tx[i, :, k], lift)
            dk = d[k][:, None] if np.ndim(getattr(d[k], "v", d[k])) else d[k]
            sk = s[k][:, None] if np.ndim(getattr(s[k], "v", s[k])) else s[k]
            val = x * dk + c(1.0) * sk
            mask = _clamp_mask(w, c, val)
            g = where(mask, _fl(go[i, :, k], lift), c(0.0))
            gt.append(g * dk)
            for t in range(T):
                Gd[k] = Gd[k] + g[:, t] * x[:, t]
                Gs[k] = Gs[k] + g[:, t]
        out["textures"].append(gt)
        if want_mat:
            gm, gr = c(0.0), c(0.0)
            if spec:
                zero = full(m, 0)
                dm, sm = face_light(w, c, Nval, pos, L, ey, Dual(m, [zero + c(1.0), zero]), Dual(r, [zero, zero + c(1.0)]))
                for k in range(3):
                    gm = gm + (Gd[k] * dm[k].d[0] + Gs[k] * sm[k].d[0])
                    gr = gr + Gs[k] * sm[k].d[1]
                gm = gm / c(float(Tm))
                gr = gr / c(float(Tm))
            out["metallic"].append(gm)
            out["roughness"].append(gr)
        if want_v:
            dv, Nd = normal_duals(w, c, vl, Nval, Njac, n32, ln, lift)
            pd = [((dv[k] + dv[3 + k]) + dv[6 + k]) / c(3.0) for k in range(3)]
            dd, sd = face_light(w, c, Nd, pd, L, ey if spec else None, m, r)
            terms = []
            for k in range(9):
                acc = c(0.0)
                for cc in range(3):
                    acc = acc + (Gd[cc] * dd[cc].d[k] + Gs[cc] * sd[cc].d[k])
                terms.append(acc)
            vbase = np.where(a["Bv"] == 1, 0, b) * nv * 3
            out["vertex_slots"].append(np.stack([vbase + fi[:, k // 3] * 3 + k % 3 for k in range(9)], 1))
            out["vertex_terms"].append(terms)
        out["walks"].append(w)
        out["near"].append(w.near)
    return _finish_surface(out, a, lift, want_mat, want_v)


def _cat(parts, lift):
    """Concatenate per-chunk lists of per-channel values."""
    if lift is None:
        return np.concatenate([np.stack([np.broadcast_to(x, np.shape(p[0])) for x in p], -1) for p in parts])
    return EV(np.concatenate([np.stack([np.broadcast_to(x.v, p[0].v.shape) for x in map(EV.of, p)], -1) for p in parts]),
              np.concatenate([np.stack([np.broadcast_to(x.e, p[0].v.shape) for x in map(EV.of, p)], -1) for p in parts]))


def _cat1(parts, n_each, lift):
    """Concatenate per-chunk member values (scalars broadcast to the chunk's members)."""
    if lift is None:
        return np.concatenate([np.broadcast_to(np.asarray(p, F32), (n,)) for p, n in zip(parts, n_each)])
    return EV(np.concatenate([np.broadcast_to(EV.of(p).v, (n,)) for p, n in zip(parts, n_each)]),
              np.concatenate([np.broadcast_to(EV.of(p).e, (n,)) for p, n in zip(parts, n_each)]))


def _near(parts):
    kinds = set(k for p in parts for k in p)
    return {k: np.concatenate([np.asarray(p[k], bool) if k in p else np.zeros(0, bool) for p in parts]) for k in kinds}


def _finish_surface(out, a, lift, want_mat, want_v):
    B, nf, T, Tm = a["B"], a["nf"], a["T"], a["Tm"]
    sizes = [len(x) for x in _chunks(B * nf, T)]
    res = dict(walks=out["walks"], near=out["near"])
    res["textures"] = _cat(out["textures"], lift)
    res["textures"] = _reshape(res["textures"], a["textures"].shape)
    for k in ("metallic", "roughness"):
        if want_mat and a.get("grad_" + k) is not None:
            g = _cat1(out[k], sizes, lift)
            res[k] = _reshape(_rep(g, Tm), a[k].shape)
        else:
            res[k] = None
    if want_v:
        res["vertex_slots"] = np.concatenate(out["vertex_slots"])
        res["vertex_terms"] = _cat(out["vertex_terms"], lift)
    res["near"] = _near(out["near"])
    return res


def _reshape(x, shape):
    return EV(x.v.reshape(shape), x.e.reshape(shape)) if isinstance(x, EV) else np.asarray(x).reshape(shape)


def _rep(g, n):
    if isinstance(g, EV):
        return EV(np.repeat(g.v, n), np.repeat(g.e, n))
    return np.repeat(g, n)


# ---- normal-mapped lighting ------------------------------------------------------------------------------------------

def _centroid(a, b, f, lift, c):
    v, fi = _gather_vertices(a, b, f)
    vl = _cols(v, lift)
    return [((vl[k] + vl[3 + k]) + vl[6 + k]) / c(3.0) for k in range(3)], fi


def _texel_normal(w, c, nt, tb):
    """normalize(n_t . TBN, 1e-12): N_j = (n0 TBN[0][j] + n1 TBN[1][j]) + n2 TBN[2][j]."""
    N = [(nt[0] * tb[j] + nt[1] * tb[3 + j]) + nt[2] * tb[6 + j] for j in range(3)]
    return normalize3(w, N, c(1e-12))


def _nm_spec(a, L):
    return L["with_specular"] and a["metallic"] is not None and a["roughness"] is not None and a["eye"] is not None


def _per_texel(x, T):
    """A per-face value [n] (float32 or EV) repeated over the face's T texels."""
    if isinstance(x, EV):
        return EV(np.repeat(x.v, T), np.repeat(x.e, T))
    return np.repeat(x, T) if np.ndim(x) else x


@_quiet
def nm_forward(a, lift=None):
    """k_nm_lighting_fwd -> lit textures [B, nf, T, 3] float32."""
    c = const_maker(lift)
    L = _lift_light(a["light"], lift)
    B, nf, T = a["B"], a["nf"], a["T"]
    spec = _nm_spec(a, L)
    out = np.empty((B, nf, T, 3), F32)
    for b in range(B):
        for fc in _chunks(nf, T):
            bb = np.full(len(fc), b)
            w = Walk()
            pos, _ = _centroid(a, bb, fc, lift, c)
            pos = [_per_texel(p, T) for p in pos]
            nt = a["normal_textures"][0 if a["Bn"] == 1 else b, fc].reshape(-1, 3)
            tb = np.repeat(a["tbn"][0 if a["Bt"] == 1 else b, fc].reshape(-1, 9), T, 0)
            N = _texel_normal(w, c, _cols(nt, lift), _cols(tb, lift))
            i = ((b * nf + fc)[:, None] * T + np.arange(T)).reshape(-1)
            m = a["metallic"].reshape(-1)[i] if spec else c(0.0)
            r = a["roughness"].reshape(-1)[i] if spec else c(1.0)
            ey = [_per_texel(e, T) for e in _eye_rows(a, bb, lift)] if spec else None
            d, s = face_light(w, c, N, pos, L, ey, m, r)
            tx = a["textures"].reshape(-1, 3)[i]
            out[b, fc] = np.stack([clamp01(tx[:, k] * d[k] + c(1.0) * s[k]) for k in range(3)], -1).reshape(len(fc), T, 3)
    return out


@_quiet
def nm_backward(a, lift=None, replay=None):
    """k_nm_lighting_bwd.  Returns dict: textures, normal_textures, metallic, roughness (per-texel gradients shaped like
    the inputs, None where not requested), vertex_slots / vertex_terms [n, 3] (each (batch, face, coordinate k) term
    gpos_k / 3 as lane 0 holds it after the butterfly, added to the face's three vertices), walks, near (kink flags per
    texel, in (batch, face, texel) order)."""
    c = const_maker(lift)
    L = _lift_light(a["light"], lift)
    B, nf, T, Bn, nv = a["B"], a["nf"], a["T"], a["Bn"], a["nv"]
    spec = _nm_spec(a, L)
    want = {k: a.get("grad_" + k) is not None for k in ("textures", "normal_textures", "vertices", "metallic", "roughness")}
    want_geom = want["normal_textures"] or want["vertices"]
    res = {k: {} for k in ("textures", "normal_textures", "metallic", "roughness")}
    slots, terms, walks, near = [], [], [], {}
    lanes = -(-T // 32)
    ci = 0
    for bn in range(Bn):
        for fc in _chunks(nf, T * (B if Bn == 1 else 1)):
            nfc = len(fc)
            gn = None
            for b in (range(B) if Bn == 1 else [bn]):
                w = Walk(replay["walks"][ci] if replay is not None else None)
                ci += 1
                bb = np.full(nfc, b)
                pos, fi = _centroid(a, bb, fc, lift, c)
                tb = _cols(np.repeat(a["tbn"][0 if a["Bt"] == 1 else b, fc].reshape(-1, 9), T, 0), lift)
                ey = [_per_texel(e, T) for e in _eye_rows(a, bb, lift)] if spec else None
                i = ((b * nf + fc)[:, None] * T + np.arange(T)).reshape(-1)
                nt = _cols(a["normal_textures"][bn, fc].reshape(-1, 3), lift)
                N = _texel_normal(w, c, nt, tb)
                m = _fl(a["metallic"].reshape(-1)[i], lift) if spec else c(0.0)
                r = _fl(a["roughness"].reshape(-1)[i], lift) if spec else c(1.0)
                post = [_per_texel(p, T) for p in pos]
                d, s = face_light(w, c, N, post, L, ey, m, r)
                Gd, Gs, gt = [], [], []
                for k in range(3):
                    x = _fl(a["textures"].reshape(-1, 3)[i, k], lift)
                    val = x * d[k] + c(1.0) * s[k]
                    mask = _clamp_mask(w, c, val)
                    g = where(mask, _fl(a["grad_out"].reshape(-1, 3)[i, k], lift), c(0.0))
                    gt.append(g * d[k])
                    Gd.append(g * x)
                    Gs.append(g)
                key = (b, fc[0], nfc)
                if want["textures"]:
                    res["textures"][key] = gt
                if want["metallic"] or want["roughness"]:
                    gm, gr = c(0.0), c(0.0)
                    if spec:
                        zero = full(m, 0)
                        dm, sm = face_light(w, c, N, post, L, ey, Dual(m, [zero + c(1.0), zero]),
                                            Dual(r, [zero, zero + c(1.0)]))
                        for k in range(3):
                            gm = gm + (Gd[k] * dm[k].d[0] + Gs[k] * sm[k].d[0])
                            gr = gr + Gs[k] * sm[k].d[1]
                    res["metallic"][key], res["roughness"][key] = gm, gr
                if want_geom:
                    zero = full(nt[0], 0)
                    one = zero + c(1.0)
                    ntd = [Dual(nt[k], [one if j == k else zero for j in range(6)]) for k in range(3)]
                    pd = [Dual(post[k] + zero, [one if j == 3 + k else zero for j in range(6)]) for k in range(3)]
                    Nd = _texel_normal(w, c, ntd, tb)
                    dd, sd = face_light(w, c, Nd, pd, L, ey, m, r)
                    gk = []
                    for k in range(6):
                        acc = c(0.0)
                        for cc in range(3):
                            acc = acc + (Gd[cc] * dd[cc].d[k] + Gs[cc] * sd[cc].d[k])
                        gk.append(acc)
                    if want["normal_textures"]:
                        gn = gk[:3] if gn is None else [gn[k] + gk[k] for k in range(3)]
                        res["normal_textures"][(bn, fc[0], nfc)] = gn
                    if want["vertices"]:
                        tm = []
                        for k in range(3):
                            gp = _lanes(gk[3 + k], nfc, T, lanes, lift, c)
                            for o in (16, 8, 4, 2, 1):
                                gp = gp + gp[:, np.arange(32) ^ o]
                            tm.append(gp[:, 0] / c(3.0))
                        vrow = np.where(a["Bv"] == 1, 0, b) * nv
                        slots.append(np.stack([(vrow + fi[:, j]) * 3 + k for k in range(3) for j in range(3)], 1))
                        terms.append([tm[k] for k in range(3) for j in range(3)])
                walks.append(w)
                for kk, fl in w.near.items():
                    near.setdefault(kk, {})[(b, fc[0], nfc)] = fl
    return _finish_nm(a, res, slots, terms, walks, near, want, lift)


def _lanes(x, nfc, T, lanes, lift, c):
    """Per-lane serial sums of x [nfc * T] (texel t on lane t % 32, in increasing t) -> [nfc, 32]."""
    if lift is None:
        xx = np.zeros((nfc, lanes * 32), F32)
        xx[:, :T] = np.asarray(x).reshape(nfc, T)
        gp = np.zeros((nfc, 32), F32)
        for j in range(lanes):
            gp = gp + xx[:, j * 32:(j + 1) * 32]
        return gp
    x = EV.of(x)
    xv, xe = np.zeros((nfc, lanes * 32)), np.zeros((nfc, lanes * 32))
    xv[:, :T], xe[:, :T] = x.v.reshape(nfc, T), x.e.reshape(nfc, T)
    gp = EV(np.zeros((nfc, 32)))
    for j in range(lanes):
        live = (j * 32 + np.arange(32)) < T   # lanes past the last texel add nothing
        nxt = gp + EV(xv[:, j * 32:(j + 1) * 32], xe[:, j * 32:(j + 1) * 32])
        gp = EV(np.where(live, nxt.v, gp.v), np.where(live, nxt.e, gp.e))
    return gp


def _finish_nm(a, res, slots, terms, walks, near, want, lift):
    B, nf, T, Bn = a["B"], a["nf"], a["T"], a["Bn"]
    out = dict(walks=walks)

    def assemble(d, nb, ch):
        shape = (nb, nf, T, ch)
        o = np.zeros(shape, F32) if lift is None else EV(np.zeros(shape))
        for (b, f0, nfc), p in d.items():
            p = p if ch == 3 else [p]
            arr = _reshape(_cat([[_broad(x, nfc * T) for x in p]], lift), (nfc, T, ch))
            if lift is None:
                o[b, f0:f0 + nfc] = arr
            else:
                o.v[b, f0:f0 + nfc], o.e[b, f0:f0 + nfc] = arr.v, arr.e
        return o

    out["textures"] = assemble(res["textures"], B, 3) if want["textures"] else None
    out["normal_textures"] = assemble(res["normal_textures"], Bn, 3) if want["normal_textures"] else None
    for k in ("metallic", "roughness"):
        out[k] = assemble(res[k], B, 1) if want[k] else None
    if want["vertices"]:
        out["vertex_slots"] = np.concatenate(slots) if slots else np.zeros((0, 9), np.int64)
        out["vertex_terms"] = _cat(terms, lift) if terms else np.zeros((0, 9), F32)
    out["near"] = {}
    for kk, parts in near.items():
        fl = np.zeros((B, nf, T), bool)
        for (b, f0, nfc), x in parts.items():
            fl[b, f0:f0 + nfc] |= np.broadcast_to(np.asarray(x, bool), (nfc * T,)).reshape(nfc, T)
        out["near"][kk] = fl
    return out


def _broad(v, n):
    if isinstance(v, EV):
        return EV(np.broadcast_to(v.v, (n,)), np.broadcast_to(v.e, (n,)))
    return np.broadcast_to(np.asarray(v, F32), (n,))
