"""Scenes that stress the SoftRas forward's per-entry error bound (oracle.softras.forward_bound), shared by
tests/test_softras_forward_bound_cpu.py and tests/test_softras_forward_bound_gpu.py.

The everyday scenes put colours near 0.5 and alpha near 0 or 1.  These reach the corners of the forward's arithmetic:
small and large colours, softmax weights that underflow to exactly 0 or stay near 1, long rescale chains of the online
softmax, sigmoids saturated to exactly 0 / 1, 72 soft edges over one pixel, hard alpha's D within an ulp or two of 0.5,
and the relaxed divisions' numerators below 2^-60.  CASES[name] = (scene(batch) -> (fv, tex), Params overrides, the
sites the case must reach (oracle.softras.SITES names; "marginal_alpha" for the hard-alpha decision)).
"""
import numpy as np

from jrender_b200 import workloads as wl
from oracle import softras as osr


def sphere(batch=3, **kw):
    return wl.make_scene(280, batch=batch, **kw)


def scaled(f):
    def scene(batch=3, **kw):
        fv, tex = sphere(batch, **kw)
        return fv, f(tex).astype(np.float32)
    return scene


def quad_stack(n, z0, dz, half=1.5):
    """n screen-filling squares (two faces each) at depths z0, z0 + dz, ... in face-id order."""
    q = np.array([[[-half, -half, 0], [half, -half, 0], [half, half, 0]],
                  [[-half, -half, 0], [half, half, 0], [-half, half, 0]]], np.float32)
    fv = np.concatenate([q + np.float32([0, 0, z0 + i * dz]) for i in range(n)])
    return fv


def layered(front_to_back):
    """34 layers (68 faces) over every pixel: softmax_max set by the first face and never again, or raised by every
    face -- a long exp_z chain or a long exp_delta_zp rescale chain."""
    def scene(batch=3, texture_type="surface", texture_res=1):
        fv = quad_stack(34, 2.0, 0.02) if front_to_back else quad_stack(34, 2.66, -0.02)
        fv = np.repeat(fv[None], batch, 0)
        T = 3 if texture_type == "vertex" else texture_res ** 2
        tex = np.random.default_rng(5).uniform(0, 1, (batch, fv.shape[1], T, 3)).astype(np.float32)
        return fv, tex
    return scene


def stacked_soft_edges(batch=3, texture_type="surface", texture_res=1, n=72, gap=8.3e-3):
    """n copies of a quad whose left edge runs `gap` to the right of the image centre (depths 2 + 0.001 i): the centre
    pixels lie outside all n faces, under n soft edges whose D is a few 1e-3 each.  alpha = prod multiplies n factors
    near 1 and stays near 1, the output 1 - alpha is small, and the n fp32 products alpha * (1.f - D) of
    softras_exact_tail = 0 pile up in it."""
    x0, x1, y0, y1 = gap, 1.5, -1.5, 1.5
    quad = np.array([[[x0, y0, 0], [x1, y0, 0], [x1, y1, 0]], [[x0, y0, 0], [x1, y1, 0], [x0, y1, 0]]], np.float32)
    fv = np.concatenate([quad + np.float32([0, 0, 2.0 + 0.001 * i]) for i in range(n)])
    fv = np.repeat(fv[None], batch, 0)
    T = 3 if texture_type == "vertex" else texture_res ** 2
    tex = np.random.default_rng(6).uniform(0, 1, (batch, fv.shape[1], T, 3)).astype(np.float32)
    return fv, tex


def edge_on_pixel_centres(batch=3, texture_type="surface", texture_res=1, H=17):
    """Faces with a vertical edge exactly on a column of pixel centres, one ulp beside it and 1e-12 beside it (column 8
    of 17 is x = 0): the pixels on it have a distance of 0 or a few ulp, so D is 1/2 to within an ulp or two -- hard
    alpha's `D > 0.5` straddles -- and at x = 0 the sigmoid's numerator -dis is about 1e-24, below 2^-60."""
    xs = [np.float32((2 * c + 1 - H) / H) for c in range(2, H - 2, 3)]
    faces = []
    for x in xs:
        for dx in (np.float32(0), np.spacing(x), np.float32(1e-12)):
            e = x + dx
            faces.append([[e, -0.9, 2.0], [e, 0.9, 2.0], [e + 0.5, 0.0, 2.0]])
            faces.append([[e, 0.9, 2.2], [e, -0.9, 2.2], [e - 0.5, 0.0, 2.2]])
    fv = np.repeat(np.array(faces, np.float32)[None], batch, 0)
    T = 3 if texture_type == "vertex" else texture_res ** 2
    tex = np.random.default_rng(7).uniform(0, 1, (batch, fv.shape[1], T, 3)).astype(np.float32)
    return fv, tex


def at_far(batch=3, texture_type="surface", texture_res=1):
    """The sphere's faces moved to z = far = 2^-50 (near 0): far - zp is a few ulp of 2^-50, below 2^-60, so by_span's
    numerator is tiny; eps 1e-30 puts zp_norm - softmax_max below 2^-60 for faces whose zp_norm is 0."""
    fv, tex = sphere(batch, texture_type=texture_type, texture_res=texture_res)
    fv = fv.copy()
    fv[..., 2] = np.float32(2.0 ** -50) * (1 - np.float32(2.0 ** -22) * (fv[..., 2] > fv[..., 2].mean()))
    return fv, tex


CASES = {
    "dark_textures": (scaled(lambda t: t * 1e-3), dict(), ["exp_soft"]),
    "bright_textures": (scaled(lambda t: 1.0 + 3.0 * t), dict(), ["exp_soft"]),
    "gamma_1e-6": (sphere, dict(gamma_val=1e-6, eps=1e-9), ["exp_soft"]),
    "gamma_1": (sphere, dict(gamma_val=1.0, sigma_val=1e-4), ["exp_soft"]),
    "front_to_back": (layered(True), dict(sigma_val=1e-4, gamma_val=1e-2), ["exp_soft"]),
    "back_to_front": (layered(False), dict(sigma_val=1e-4, gamma_val=1e-2), ["exp_soft"]),
    "sigma_tiny": (sphere, dict(sigma_val=1e-9), ["exp_sig"]),
    "sigma_huge": (sphere, dict(sigma_val=0.5, gamma_val=1e-2), ["exp_sig", "exp_soft"]),
    "stacked_soft_edges": (stacked_soft_edges, dict(sigma_val=1e-5, aggr_func_alpha="prod"), ["exp_sig", "prod"]),
    "alpha_sum": (sphere, dict(sigma_val=3e-3, aggr_func_alpha="sum"), ["exp_sig"]),
    "hard_alpha_half": (edge_on_pixel_centres, dict(sigma_val=1e-5, aggr_func_alpha="hard"),
                        ["exp_sig", "marginal_alpha", "div_sigarg"]),
    "tiny_span": (at_far, dict(near=0.0, far=2.0 ** -50, eps=1e-30), ["div_span", "div_gamma"]),
}
# sites that only the fp32 tails (softras_exact_tail = 0) reach
FP32_ONLY = {"tail_d", "prod", "div_sigarg", "div_span", "div_gamma"}

# the sweep: texture flavour, fill_back, K
VARIANTS = {
    "surface1": dict(scene=dict(), params=dict()),
    "vertex": dict(scene=dict(texture_type="vertex"), params=dict(texture_type="vertex")),
    "res5_back": dict(scene=dict(texture_res=5), params=dict(fill_back=False)),
    "K1": dict(scene=dict(), params=dict(max_faces_per_pixel_for_grad=1)),
    "K64": dict(scene=dict(), params=dict(max_faces_per_pixel_for_grad=64)),
}


def build(name, variant="surface1", image_size=17, batch=3):
    """-> (fv, tex, Params) of a case in a variant."""
    scene, kw, _ = CASES[name]
    v = VARIANTS[variant]
    fv, tex = scene(batch, **v["scene"])
    P = osr.Params(image_size=image_size, **{**kw, **v["params"]})
    return fv, tex, P


def reached(ref):
    """The set of sites (and 'marginal_alpha' / 'marginal_max') one forward_bound result reached."""
    live = np.bitwise_or.reduce(ref["live"].ravel())
    out = set(osr.site_names(live))
    m = np.bitwise_or.reduce(ref["marginal"].ravel())
    if m & osr.MARG_ALPHA:
        out.add("marginal_alpha")
    if m & osr.MARG_MAX:
        out.add("marginal_max")
    return out
