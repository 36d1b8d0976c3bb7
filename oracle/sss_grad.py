"""float64 mirror of the subsurface-scattering gradients (TEST INFRASTRUCTURE, not product code).

  stretch()        oracle/sss.py's stretch in float64 torch, differentiable; the clamps' pass-through decided in float32
  blur()           one modulated blur in float64 torch, differentiable in the image and the modulation, at decisions
  blur_vjp()       its adjoint, written out the way csrc/sss_api.cu's sss_blur_1d_adjoint runs it
  pyramid()        the blur pyramid and composition in float64 torch, differentiable
  pyramid_vjp()    the pyramid's adjoint at given intermediates, and the same adjoint on magnitudes (the bound)
  bake()           the SoftRas texture bake as a float64 gather with the forward's float32 weights, differentiable

Every decision comes from oracle/sss.py's float32 kernel-order walk (decisions()): the int() tap indices and their
clamps, the <= 1e-6 replacements and the centre test.  So the mirror and the kernels branch identically, and each
function is smooth in its float64 arguments around the point the walk describes: tap k of a pixel c sits at
x_k = c + (k - 3) width mod, a function of the modulation.

Bound.  pyramid_vjp(..., magnitude=True) runs the same adjoint with |g| upstream and every local partial replaced by
the sum of the magnitudes of the float32 operands it is computed from: a tap weight (x - x1) by |x| + |x1|, a
modulation partial (v2 - v1) by |v1| + |v2|.  With u = 2^-24, the kernel's gradient at the forward's float32
intermediates then sits within DEPTH u of that magnitude adjoint (bound()), where DEPTH = 1024 is fixed from the
operation counts of the longest path, as follows.  A blur adjoint evaluates its tap position by at most 9 float32
operations from the centre index and the modulation (width * mod, * 6 / 2, the subtraction and up to six additions),
each rounding by at most u relative to the running position's terms: 10 u of |x| + |x1|.  The products with G and the
tap weight add 3 u.  The sum of a gradient entry's contributions (atomics in any order) adds at most (N - 1) u of the
sum of their magnitudes, N the number of contributions: at most 2 x 7 taps from up to 4 centres per tap and endpoint
in the maps the tests use (4 needs a modulation step below 1/4 pixel over a run of pixels), plus the replaced
neighbours' shares at a centre: N <= 64.  So one adjoint stage contributes at most (10 + 3 + 63) u = 76 u of its
magnitudes.  The longest chain is 13 stages: the composition, six pass adjoints down the irradiance chain and six
more down a stretch chain through the modulation terms.  Errors add along a chain of linear stages (each stage's
error is bounded by the magnitude adjoint of the rest), so 13 x 76 u = 988 u <= DEPTH u.

Stretch and bake bounds are built the same way (stretch_bound(), bake()), with their own, shorter operation counts.
"""
import numpy as np
import torch

from . import sss as osss

F32 = np.float32
U = 2.0 ** -24
DEPTH = 1024
STRETCH_DEPTH = 32     # 3 squares and 2 sums, sqrt, 1 / x, u^3 (3), * g * -7, * d, then 4 terms summed: <= 20 u
TAP = osss.TAP_NUM


# ------------------------------------------------------------------------------------------------- decisions

def decisions(image, mod, gauss, width, dim):
    """The float32 walk of osss.blur on image / mod [H, W] (numpy float32): per tap k the clamped indices x1, x2 on
    the line (int64 [H, W]) and whether each was replaced by the centre; plus `live` (centre > 0) and the float32
    result.  dim 1 = x pass (along rows), dim 0 = y pass (along columns)."""
    img = np.asarray(image, F32)
    mod = np.asarray(mod, F32)
    H, W = img.shape
    bound = W - 1
    c = np.broadcast_to(np.arange(W)[None, :] if dim == 1 else np.arange(H)[:, None], (H, W))
    step = F32(width) * mod
    x = c.astype(F32) - step * F32(TAP - 1) / F32(2)
    taps = []
    v = np.zeros((H, W), F32)
    for k in range(TAP):                              # osss.blur's loop, keeping its decisions
        t = osss._f2i(x)
        x1, x2 = np.clip(t, 0, bound), np.clip(t + 1, 0, bound)
        v1 = np.take_along_axis(img, x1, axis=dim)
        v2 = np.take_along_axis(img, x2, axis=dim)
        r1, r2 = ~(v1.astype(np.float64) > 1e-6), ~(v2.astype(np.float64) > 1e-6)
        v1, v2 = np.where(r1, img, v1), np.where(r2, img, v2)
        v = v + ((x - x1.astype(F32)) * v2 + (x2.astype(F32) - x) * v1) * F32(gauss[k])
        taps.append((x1, x2, r1, r2))
        x = x + step
    return dict(taps=taps, live=img > 0, value=np.where(img > 0, v, F32(0)).astype(F32), dim=dim)


def _t(a, like):
    return torch.as_tensor(np.ascontiguousarray(a), device=like.device)


# ------------------------------------------------------------------------------------------------- one blur

def blur(image, mod, dec, gauss, width):
    """Differentiable in image and mod [H, W] (float64; float32 runs too, for timing): sum_k taps[k] ((x_k - x1) v2 + (x2 - x_k) v1) at the pixels
    live in dec, 0 elsewhere; a replaced v is the centre value; a tap with x1 == x2 contributes 0."""
    dim = dec["dim"]
    H, W = image.shape
    c = torch.arange(W if dim == 1 else H, dtype=image.dtype, device=image.device)
    c = c[None, :].expand(H, W) if dim == 1 else c[:, None].expand(H, W)
    v = torch.zeros_like(image)
    for k, (x1, x2, r1, r2) in enumerate(dec["taps"]):
        x1t, x2t = _t(x1, image), _t(x2, image)
        xk = c + (k - (TAP - 1) // 2) * float(width) * mod
        v1 = torch.where(_t(r1, image), image, torch.gather(image, dim, x1t))
        v2 = torch.where(_t(r2, image), image, torch.gather(image, dim, x2t))
        term = (xk - x1t.to(image.dtype)) * v2 + (x2t.to(image.dtype) - xk) * v1
        v = v + float(gauss[k]) * torch.where(x1t == x2t, torch.zeros_like(term), term)
    return torch.where(_t(dec["live"], image), v, torch.zeros_like(v))


def blur_vjp(image, mod, dec, gauss, width, G, magnitude=False, want_mod=True):
    """Adjoint of blur at (image, mod) given G [H, W]: (grad_image, grad_mod), float64.  With magnitude=True every
    local partial is replaced by its operands' magnitude sum (module docstring) and G should be |G|."""
    dim = dec["dim"]
    H, W = image.shape
    c_line = torch.arange(W if dim == 1 else H, dtype=torch.float64, device=image.device)
    c_line = c_line[None, :].expand(H, W) if dim == 1 else c_line[:, None].expand(H, W)
    ci = c_line.long()
    G = torch.where(_t(dec["live"], image), G, torch.zeros_like(G))
    gi = torch.zeros(H * W, dtype=torch.float64, device=image.device)
    gm = torch.zeros_like(image)
    rows = torch.arange(H, device=image.device)[:, None].expand(H, W)
    cols = torch.arange(W, device=image.device)[None, :].expand(H, W)

    def flat(j):   # line index j -> flat pixel index
        return (rows * W + j) if dim == 1 else (j * W + cols)
    for k, (x1, x2, r1, r2) in enumerate(dec["taps"]):
        x1t, x2t, r1t, r2t = _t(x1, image), _t(x2, image), _t(r1, image), _t(r2, image)
        d = (k - (TAP - 1) // 2) * float(width)
        xk = c_line + d * mod
        same = x1t == x2t
        if magnitude:
            a2, a1 = xk.abs() + x1t.double(), x2t.double() + xk.abs()
        else:
            a2, a1 = xk - x1t.double(), x2t.double() - xk
        gt = torch.where(same, torch.zeros_like(G), G * float(gauss[k]))
        gi.index_add_(0, flat(torch.where(r2t, ci, x2t)).reshape(-1), (gt * a2).reshape(-1))
        gi.index_add_(0, flat(torch.where(r1t, ci, x1t)).reshape(-1), (gt * a1).reshape(-1))
        if want_mod:
            v1 = torch.where(r1t, image, torch.gather(image, dim, x1t))
            v2 = torch.where(r2t, image, torch.gather(image, dim, x2t))
            dv = v2.abs() + v1.abs() if magnitude else v2 - v1
            gm = gm + gt * (abs(d) if magnitude else d) * dv
    return gi.reshape(H, W), gm


# ------------------------------------------------------------------------------------------------- pyramid

def walk(stretch_u, stretch_v, irradiance):
    """oracle/sss.py's float32 pyramid walk from the clamped stretch maps [H, W] and the irradiance [H, W, 3]: for each
    level the decisions of its eight blurs (su, irr x3, sv, irr x3) and the float32 intermediates they produce."""
    su, sv = np.asarray(stretch_u, F32), np.asarray(stretch_v, F32)
    irr = [np.asarray(irradiance, F32)[..., j].copy() for j in range(3)]
    out = []
    for v in osss.levels():
        g, w = osss.taps(v)
        lv = dict(gauss=g, width=w, su_in=su, sv_in=sv, irr_in=irr)
        lv["dsu"] = decisions(su, su, g, w, 1)
        su = lv["dsu"]["value"]
        lv["dirr_x"] = [decisions(x, su, g, w, 1) for x in irr]
        irr_x = [d["value"] for d in lv["dirr_x"]]
        lv["dsv"] = decisions(sv, sv, g, w, 0)
        sv = lv["dsv"]["value"]
        lv["dirr_y"] = [decisions(x, sv, g, w, 0) for x in irr_x]
        irr = [d["value"] for d in lv["dirr_y"]]
        lv.update(su=su, sv=sv, irr_x=irr_x, irr_y=irr)
        out.append(lv)
    return out


def pyramid(stretch_u, stretch_v, irradiance, specular, levels, weights=osss.WEIGHTS):
    """float64, differentiable: osss.blur_pyramid at the decisions of `levels` (walk()).  stretch maps [H, W],
    irradiance / specular [H, W, 3] tensors; returns the composed map [H, W, 3], rows flipped."""
    su, sv = stretch_u, stretch_v
    irr = [irradiance[..., j] for j in range(3)]
    final = [torch.zeros_like(su) for _ in range(3)]
    for i, lv in enumerate(levels):
        g, w = lv["gauss"], lv["width"]
        su = blur(su, su, lv["dsu"], g, w)
        irr = [blur(x, su, d, g, w) for x, d in zip(irr, lv["dirr_x"])]
        sv = blur(sv, sv, lv["dsv"], g, w)
        irr = [blur(x, sv, d, g, w) for x, d in zip(irr, lv["dirr_y"])]
        final = [f + weights[j][i] * irr[j] for j, f in enumerate(final)]
    final = torch.stack(final, -1) * irradiance + specular
    return torch.flip(final, [0])


def pyramid_vjp(levels, irradiance, grad_out, values=None, magnitude=False, stretch=True, weights=osss.WEIGHTS):
    """The pyramid's adjoint, stage by stage as b200r_sss_blur_pyramid_backward runs it, at the intermediates of
    `levels` (the float32 walk; or `values`, a list per level of dicts su_in, sv_in, irr_in, su, sv, irr_x, irr_y of
    float64 tensors, e.g. from pyramid_values()).  irradiance [H, W, 3], grad_out [H, W, 3] flipped.  Returns
    dict(irradiance, specular [H, W, 3], stretch_u, stretch_v [H, W] or None).  magnitude=True: the bound's adjoint."""
    dev = grad_out.device
    g = torch.flip(grad_out, [0]).double()
    if magnitude:
        g = g.abs()
    irr0 = irradiance.double().abs() if magnitude else irradiance.double()
    f64 = lambda a: torch.as_tensor(np.asarray(a, np.float64), device=dev)
    V = values or [{k: (f64(lv[k]) if not isinstance(lv[k], list) else [f64(x) for x in lv[k]])
                    for k in ("su_in", "sv_in", "irr_in", "su", "sv", "irr_x", "irr_y")} for lv in levels]
    ab = (lambda t: t.abs()) if magnitude else (lambda t: t)
    L = len(levels)
    acc = [sum(weights[j][i] * ab(V[i]["irr_y"][j]) for i in range(L)) for j in range(3)]
    g_next = None
    gsu = gsv = None
    for i in range(L - 1, -1, -1):
        lv, v = levels[i], V[i]
        gw, w = lv["gauss"], lv["width"]
        # y pass
        Gy = [weights[j][i] * irr0[..., j] * g[..., j] + (g_next[j] if g_next is not None else 0) for j in range(3)]
        gx, gs = [], torch.zeros_like(g[..., 0])
        for j in range(3):
            a, m = blur_vjp(v["irr_x"][j], v["sv"], lv["dirr_y"][j], gw, w, Gy[j], magnitude, stretch)
            gx.append(a)
            gs = gs + m
        if stretch:
            gs = gs + (gsv if gsv is not None else 0)
            a, m = blur_vjp(v["sv_in"], v["sv_in"], lv["dsv"], gw, w, gs, magnitude)
            gsv = a + m
        # x pass
        gin, gs = [], torch.zeros_like(g[..., 0])
        for j in range(3):
            a, m = blur_vjp(v["irr_in"][j], v["su"], lv["dirr_x"][j], gw, w, gx[j], magnitude, stretch)
            gin.append(a)
            gs = gs + m
        if stretch:
            gs = gs + (gsu if gsu is not None else 0)
            a, m = blur_vjp(v["su_in"], v["su_in"], lv["dsu"], gw, w, gs, magnitude)
            gsu = a + m
        g_next = gin
    girr = torch.stack([g_next[j] + g[..., j] * acc[j] for j in range(3)], -1)
    return dict(irradiance=girr, specular=g.clone(), stretch_u=gsu, stretch_v=gsv)


def pyramid_values(stretch_u, stretch_v, irradiance, levels):
    """The float64 intermediates of pyramid() at the decisions of `levels`, in pyramid_vjp's `values` form."""
    su, sv = stretch_u, stretch_v
    irr = [irradiance[..., j] for j in range(3)]
    out = []
    for lv in levels:
        g, w = lv["gauss"], lv["width"]
        d = dict(su_in=su, sv_in=sv, irr_in=irr)
        su = blur(su, su, lv["dsu"], g, w)
        irr_x = [blur(x, su, dd, g, w) for x, dd in zip(irr, lv["dirr_x"])]
        sv = blur(sv, sv, lv["dsv"], g, w)
        irr = [blur(x, sv, dd, g, w) for x, dd in zip(irr_x, lv["dirr_y"])]
        d.update(su=su, sv=sv, irr_x=irr_x, irr_y=irr)
        out.append(d)
    return out


def bound(magnitude_grad):
    """The per-entry bound on |kernel gradient - mirror gradient| from the magnitude adjoint (module docstring)."""
    return DEPTH * U * magnitude_grad + 2.0 ** -125


# ------------------------------------------------------------------------------------------------- stretch

def stretch_pass(world):
    """float32 decisions of osss.stretch for world [H, W, 3]: masks where each clamp passes u / v through (0 < u < 1)."""
    w7 = np.asarray(world, F32) * F32(7)
    right = np.concatenate([w7, w7[:, -1:]], axis=1)[:, 1:]
    down = np.concatenate([w7, w7[-1:]], axis=0)[1:]
    out = []
    for nb in (right, down):
        d = w7 - nb
        s = d[..., 0] * d[..., 0]
        s = s + d[..., 1] * d[..., 1]
        s = s + d[..., 2] * d[..., 2]
        with np.errstate(divide="ignore"):
            u = F32(1) / np.sqrt(s)
        out.append((u > 0) & (u < 1))
    return tuple(out)


def stretch(world, passes):
    """float64, differentiable: (stretch_u, stretch_v) [H, W] of world [H, W, 3], 1 / |7 (w - w_nb)| where the float32
    clamp passed it through (passes from stretch_pass()), a constant 0 or 1 elsewhere (its float32 value)."""
    w7 = world * 7
    right = torch.cat([w7[:, 1:], w7[:, -1:]], 1)
    down = torch.cat([w7[1:], w7[-1:]], 0)
    out = []
    for nb, p in zip((right, down), passes):
        pt = _t(p, world)
        s = ((w7 - nb) ** 2).sum(-1)
        u = 1 / torch.sqrt(torch.where(pt, s, torch.ones_like(s)))
        const = torch.where(s.detach() > 0, torch.clamp(1 / torch.sqrt(s.detach()), 0, 1), torch.ones_like(s))
        out.append(torch.where(pt, u, const))
    return tuple(out)


def stretch_bound(world, passes, gu, gv):
    """Per-entry bound on the stretch backward's grad_world [H, W, 3]: STRETCH_DEPTH u times the gather of the terms'
    magnitudes 7 |g| u^3 (|7 w| + |7 w_nb|)."""
    w7 = world.double() * 7
    right = torch.cat([w7[:, 1:], w7[:, -1:]], 1)
    down = torch.cat([w7[1:], w7[-1:]], 0)
    out = torch.zeros_like(w7)
    for nb, p, G, shift in zip((right, down), passes, (gu, gv), (1, 0)):
        s = ((w7 - nb) ** 2).sum(-1)
        u = torch.where(_t(p, w7), 1 / torch.sqrt(torch.where(_t(p, w7), s, torch.ones_like(s))), torch.zeros_like(s))
        t = (7 * G.double().abs() * u ** 3)[..., None] * (w7.abs() + nb.abs())
        out = out + t
        if shift == 1:
            out[:, 1:] = out[:, 1:] + t[:, :-1]
        else:
            out[1:] = out[1:] + t[:-1]
    return STRETCH_DEPTH * U * out + 2.0 ** -125


# ------------------------------------------------------------------------------------------------- bake

def bake_weights(faces_uv, R, H, W):
    """The SoftRas bake's per-texel flat indices [nf, T, 4] (clamped as the kernel clamps) and float32 bilinear
    weights [nf, T, 4], in the kernel's promotions (oracle/bake.py)."""
    T = R * R
    wy, wx = np.divmod(np.arange(T), R)
    lower = (wx + wy) < R
    w0 = np.where(lower, (wx + 1. / 3.) / R, ((R - 1. - wx) + 2. / 3.) / R).astype(F32)
    w1 = np.where(lower, (wy + 1. / 3.) / R, ((R - 1. - wy) + 2. / 3.) / R).astype(F32)
    w2 = (1. - w0.astype(np.float64) - w1.astype(np.float64)).astype(F32)
    f = np.asarray(faces_uv, F32)
    pos_x = ((f[:, None, 0, 0] * w0 + f[:, None, 1, 0] * w1 + f[:, None, 2, 0] * w2) * F32(W - 1)).astype(F32)
    pos_y = ((f[:, None, 0, 1] * w0 + f[:, None, 1, 1] * w1 + f[:, None, 2, 1] * w2) * F32(H - 1)).astype(F32)
    ix, iy, iy1 = osss._f2i(pos_x), osss._f2i(pos_y), osss._f2i((pos_y + F32(1)).astype(F32))
    wx1 = (pos_x - ix.astype(F32)).astype(F32)
    wx0 = (F32(1) - wx1).astype(F32)
    wy1 = (pos_y - iy.astype(F32)).astype(F32)
    wy0 = (F32(1) - wy1).astype(F32)
    i00, i10 = iy * W + ix, iy1 * W + ix
    idx = np.clip(np.stack([i00, i10, i00 + 1, i10 + 1], -1), 0, H * W - 1)
    wts = np.stack([wx0 * wy0, wx0 * wy1, wx1 * wy0, wx1 * wy1], -1).astype(F32)
    return idx, wts


def bake(image, faces_uv, R, is_update=None):
    """float64, differentiable in image [H, W, 3]: the baked textures [nf, R*R, 3] (1 where is_update == 0, as the
    product's SSS bake starts from ones)."""
    H, W = image.shape[:2]
    idx, wts = bake_weights(faces_uv, R, H, W)
    flat = image.reshape(-1, 3)
    it, wt = _t(idx, image), _t(wts.astype(np.float64), image)
    out = (flat[it.reshape(-1)].reshape(idx.shape + (3,)) * wt[..., None]).sum(2)
    if is_update is not None:
        keep = _t(np.asarray(is_update) != 0, image)[:, None, None]
        out = torch.where(keep, out, torch.ones_like(out))
    return out


def bake_vjp(grad_textures, faces_uv, R, H, W, is_update=None, magnitude=False):
    """The bake's adjoint [H, W, 3] (magnitude=True: of |g| w), and the count of contributions per pixel [H, W]."""
    idx, wts = bake_weights(faces_uv, R, H, W)
    g = grad_textures.double().abs() if magnitude else grad_textures.double()
    if is_update is not None:
        g = g * _t((np.asarray(is_update) != 0).astype(np.float64), g)[:, None, None]
    it, wt = _t(idx, g).reshape(-1), _t(wts.astype(np.float64), g)
    out = torch.zeros((H * W, 3), dtype=torch.float64, device=g.device)
    out.index_add_(0, it, (g[:, :, None, :] * wt[..., None]).reshape(-1, 3))
    live = torch.ones(idx.shape, dtype=torch.float64, device=g.device)
    if is_update is not None:
        live = live * _t((np.asarray(is_update) != 0).astype(np.float64), g)[:, None, None]
    n = torch.zeros(H * W, dtype=torch.float64, device=g.device).index_add_(0, it, live.reshape(-1))
    return out.reshape(H, W, 3), n.reshape(H, W)


def bake_bound(grad_textures, faces_uv, R, H, W, is_update=None):
    """Per-entry bound on the bake backward: a sum of N products g w in any order is within (N + 1) u of the sum of
    their magnitudes (one rounding per product, N - 1 per sum, one for the double reference)."""
    mag, n = bake_vjp(grad_textures, faces_uv, R, H, W, is_update, magnitude=True)
    return (n[..., None] + 1) * U * mag + 2.0 ** -125
