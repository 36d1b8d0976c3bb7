"""numpy front end of the CPU SoftRas oracle (TEST INFRASTRUCTURE, not product code).

Mirrors the host side of the reference op:
  jrender/renderer/dr/softras/soft_rasterize.py:25     dist_eps -> ln(1/dist_eps - 1)
  jrender/renderer/dr/softras/soft_rasterize.py:39-42  enum maps
  jrender/renderer/dr/softras/soft_rasterize.py:59-71  buffer shapes
Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs import this.
"""
import ctypes as C

import numpy as np

from . import build as _build

DIST = {"hard": 0, "barycentric": 1, "euclidean": 2}
RGB = {"hard": 0, "softmax": 1, "none": 2}
ALPHA = {"hard": 0, "sum": 1, "prod": 2}
TEX = {"surface": 0, "vertex": 1}

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_build.build())
        f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        _lib.softras_oracle_forward.restype = None
        _lib.softras_oracle_forward.argtypes = [
            f32p, f32p, f32p, f32p, f32p, i32p,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        _lib.softras_oracle_backward.restype = None
        _lib.softras_oracle_backward.argtypes = [
            f32p, f32p, f32p, f32p, f32p, i32p, f32p, f32p, f32p,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        _lib.softras_oracle_backward_mt.restype = None
        _lib.softras_oracle_backward_mt.argtypes = [
            f32p, f32p, f32p, f32p, f32p, i32p, f32p, f32p, f32p,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        _lib.softras_oracle_backward_stats.restype = C.c_long
        _lib.softras_oracle_backward_stats.argtypes = [
            f32p, f32p, f32p, f32p, f32p, i32p, f32p,
            C.POINTER(C.c_double), C.POINTER(C.c_double), i32p, C.POINTER(C.c_double),
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            f32p, C.POINTER(C.c_int64), C.c_long]
        _lib.softras_oracle_forward_bound.restype = None
        _lib.softras_oracle_forward_bound.argtypes = [
            f32p, f32p, f32p, f32p, f32p, i32p,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
            C.POINTER(C.c_double), C.POINTER(C.c_double), i32p, C.POINTER(C.c_uint32),
            C.c_int, C.c_int, C.c_int, C.c_int]
        _lib.softras_oracle_max_threads.restype = C.c_int
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def dist_eps_logit(dist_eps):
    """soft_rasterize.py:25 -- float64 log, later narrowed to the kernel's float arg."""
    return np.float32(np.log(1.0 / dist_eps - 1.0))


class Params(dict):
    """Scalar parameters of the op with the reference's defaults (soft_rasterize.py:10-16)."""

    def __init__(self, **kw):
        d = dict(image_size=256, near=1.0, far=100.0, fill_back=True, eps=1e-3, sigma_val=1e-5,
                 dist_func="euclidean", dist_eps=1e-4, gamma_val=1e-4, aggr_func_rgb="softmax",
                 aggr_func_alpha="prod", texture_type="surface", max_faces_per_pixel_for_grad=16)
        unknown = set(kw) - set(d)
        if unknown:
            raise TypeError("unknown params %s" % sorted(unknown))
        d.update(kw)
        super().__init__(d)

    def scalars(self):
        return (np.float32(self["near"]), np.float32(self["far"]), np.float32(self["eps"]),
                np.float32(self["sigma_val"]), DIST[self["dist_func"]], dist_eps_logit(self["dist_eps"]),
                np.float32(self["gamma_val"]), RGB[self["aggr_func_rgb"]], ALPHA[self["aggr_func_alpha"]],
                TEX[self["texture_type"]], int(bool(self["fill_back"])))


def forward(face_vertices, textures, params, rows=None, nthreads=0, row_stride=1):
    """face_vertices [B,nf,3,3] f32, textures [B,nf,T,3] f32 ->
    dict(soft_colors [B,4,H,W], faces_info [B,nf,27], aggrs_info [B,2,H,W], faces_id_buffer [B,K,H,W] i32)."""
    fv = np.ascontiguousarray(face_vertices, dtype=np.float32)
    tx = np.ascontiguousarray(textures, dtype=np.float32)
    B, nf = fv.shape[:2]
    T = tx.shape[2]
    H = int(params["image_size"])
    K = int(params["max_faces_per_pixel_for_grad"])
    assert K <= 64, "reference hard limit kMaxPointsPerPixel (cuda/soft_rasterize.py:16)"
    faces_info = np.zeros((B, nf, 27), np.float32)
    aggrs_info = np.zeros((B, 2, H, H), np.float32)
    soft_colors = np.zeros((B, 4, H, H), np.float32)
    ids = np.zeros((B, K, H, H), np.int32)
    r0, r1 = (0, H) if rows is None else rows
    lib().softras_oracle_forward(
        _p(fv, C.c_float), _p(tx, C.c_float), _p(faces_info, C.c_float), _p(aggrs_info, C.c_float),
        _p(soft_colors, C.c_float), _p(ids, C.c_int32), B, nf, T, H, K, *params.scalars(), r0, r1, int(row_stride), nthreads)
    return dict(soft_colors=soft_colors, faces_info=faces_info, aggrs_info=aggrs_info, faces_id_buffer=ids)


# softras_oracle.c's rounding sites, by bit of forward_bound's `live`
SITES = ["exp_sig", "exp_soft", "tail_d", "prod", "div_sigarg", "div_zsoft", "div_cold", "div_gamma", "div_nmf",
         "div_sigma"] + ["div_%s%d" % (n, k) for n in ("z1_", "z2_", "clipw", "clipz", "euc") for k in range(3)] + \
        ["exp_bg", "div_span"]
SITE = {n: i for i, n in enumerate(SITES)}
MARG_ALPHA, MARG_MAX = 1, 2   # forward_bound's `marginal` bits


def site_names(mask):
    return [n for i, n in enumerate(SITES) if int(mask) >> i & 1]


def forward_bound(face_vertices, textures, params, exact_tail=False, nudge=0, rows=None, row_stride=1, nthreads=0):
    """forward() plus the CUDA forward's error bound per output entry (softras_oracle.c, "rounding sites of the K2
    forward").  Adds bound_colors [B,4,H,W] (on |CUDA soft_colors - oracle|), bound_sum [B,H,W] (on the softmax sum,
    aggrs_info[:, 0]; 0 where that channel is not the sum), marginal [B,H,W] (MARG_* bits: a decision the error can
    flip; those entries' bounds are inf) and live [B,H,W] (bit SITE[name]: the site was live in one of the pixel's
    pairs).  exact_tail: the kernel's softras_exact_tail.  nudge = +1 / -1 / >= 2: the outputs are the forward with every
    live site moved by its budget up / down / by a hashed sign, the hash seeded by nudge - 2 for nudge >= 2 (and,
    without exact_tail, the kernel's fp32 tails)."""
    fv = np.ascontiguousarray(face_vertices, dtype=np.float32)
    tx = np.ascontiguousarray(textures, dtype=np.float32)
    B, nf = fv.shape[:2]
    T = tx.shape[2]
    H = int(params["image_size"])
    K = int(params["max_faces_per_pixel_for_grad"])
    assert K <= 64
    out = dict(faces_info=np.zeros((B, nf, 27), np.float32), aggrs_info=np.zeros((B, 2, H, H), np.float32),
               soft_colors=np.zeros((B, 4, H, H), np.float32), faces_id_buffer=np.zeros((B, K, H, H), np.int32),
               bound_colors=np.zeros((B, 4, H, H)), bound_sum=np.zeros((B, H, H)),
               marginal=np.zeros((B, H, H), np.int32), live=np.zeros((B, H, H), np.uint32))
    r0, r1 = (0, H) if rows is None else rows
    lib().softras_oracle_forward_bound(
        _p(fv, C.c_float), _p(tx, C.c_float), _p(out["faces_info"], C.c_float), _p(out["aggrs_info"], C.c_float),
        _p(out["soft_colors"], C.c_float), _p(out["faces_id_buffer"], C.c_int32), B, nf, T, H, K, *params.scalars(),
        int(bool(exact_tail)), int(nudge), _p(out["bound_colors"], C.c_double), _p(out["bound_sum"], C.c_double),
        _p(out["marginal"], C.c_int32), _p(out["live"], C.c_uint32), r0, r1, int(row_stride), nthreads)
    return out


def backward(face_vertices, textures, fwd, grad_soft_colors, params, accumulate_double=True, rows=None, row_stride=1,
             nthreads=1, stats=False, exact_tail=False, nudge=0, terms=False):
    """Top-K backward (K6).  `fwd` is the dict returned by forward().  -> (grad_faces, grad_textures).
    nthreads > 1 (CPU-baseline timing only): rows are dealt to threads with private double accumulators.

    stats=True: -> (faces, textures), each a dict of float64 / int32 arrays shaped like the gradient: g64 (the double
    sum of the reference's float terms, which accumulate_double rounds), A (sum of |term|), N (number of non-zero terms)
    and E (sum over terms of how far the CUDA kernel's term may be from the reference's, see softras_oracle.c's
    rounding sites; exact_tail is the kernel's softras_exact_tail option).  N counts the pairs that write a term into the
    entry, zero or not: at least as many as the float additions the kernel makes into it.  terms=True adds 'terms': (values, slots)
    of every non-zero term in the sequential order, slots indexing the faces then the textures gradient, flattened.
    nudge = +1 / -1 / 2 computes g64 with every rounding site moved by its budget up / down / by a hashed sign."""
    fv = np.ascontiguousarray(face_vertices, dtype=np.float32)
    tx = np.ascontiguousarray(textures, dtype=np.float32)
    g = np.ascontiguousarray(grad_soft_colors, dtype=np.float32)
    B, nf = fv.shape[:2]
    T = tx.shape[2]
    H = int(params["image_size"])
    K = int(params["max_faces_per_pixel_for_grad"])
    gf = np.zeros((B, nf, 3, 3), np.float32)
    gt = np.zeros((B, nf, T, 3), np.float32)
    r0, r1 = (0, H) if rows is None else rows
    if stats:
        return _backward_stats(fv, tx, fwd, g, params, (r0, r1), int(row_stride), exact_tail, nudge, terms)
    if nthreads > 1:
        lib().softras_oracle_backward_mt(
            _p(fv, C.c_float), _p(tx, C.c_float), _p(np.ascontiguousarray(fwd["soft_colors"]), C.c_float),
            _p(np.ascontiguousarray(fwd["faces_info"]), C.c_float), _p(np.ascontiguousarray(fwd["aggrs_info"]), C.c_float),
            _p(np.ascontiguousarray(fwd["faces_id_buffer"]), C.c_int32), _p(g, C.c_float),
            _p(gf, C.c_float), _p(gt, C.c_float), B, nf, T, H, K, *params.scalars(), r0, r1, int(row_stride), int(nthreads))
        return gf, gt
    lib().softras_oracle_backward(
        _p(fv, C.c_float), _p(tx, C.c_float), _p(np.ascontiguousarray(fwd["soft_colors"]), C.c_float),
        _p(np.ascontiguousarray(fwd["faces_info"]), C.c_float), _p(np.ascontiguousarray(fwd["aggrs_info"]), C.c_float),
        _p(np.ascontiguousarray(fwd["faces_id_buffer"]), C.c_int32), _p(g, C.c_float),
        _p(gf, C.c_float), _p(gt, C.c_float), B, nf, T, H, K, *params.scalars(),
        int(bool(accumulate_double)), r0, r1, int(row_stride))
    return gf, gt


def _backward_stats(fv, tx, fwd, g, params, rows, row_stride, exact_tail, nudge, terms):
    B, nf = fv.shape[:2]
    T = tx.shape[2]
    H = int(params["image_size"])
    K = int(params["max_faces_per_pixel_for_grad"])
    ngf, ngt = B * nf * 9, B * nf * T * 3
    g64, A, E = (np.zeros(ngf + ngt) for _ in range(3))
    N = np.zeros(ngf + ngt, np.int32)
    ins = [_p(fv, C.c_float), _p(tx, C.c_float), _p(np.ascontiguousarray(fwd["soft_colors"]), C.c_float),
           _p(np.ascontiguousarray(fwd["faces_info"]), C.c_float), _p(np.ascontiguousarray(fwd["aggrs_info"]), C.c_float),
           _p(np.ascontiguousarray(fwd["faces_id_buffer"]), C.c_int32), _p(g, C.c_float)]
    outs = [_p(g64, C.c_double), _p(A, C.c_double), _p(N, C.c_int32), _p(E, C.c_double)]
    args = [B, nf, T, H, K, *params.scalars(), int(bool(exact_tail)), int(nudge), rows[0], rows[1], row_stride]
    n = lib().softras_oracle_backward_stats(*ins, *outs, *args, None, None, 0)
    res = [dict(g64=x[:ngf].reshape(B, nf, 3, 3), A=a[:ngf].reshape(B, nf, 3, 3), N=c[:ngf].reshape(B, nf, 3, 3),
                E=e[:ngf].reshape(B, nf, 3, 3)) for x, a, c, e in [(g64, A, N, E)]]
    res.append(dict(g64=g64[ngf:].reshape(B, nf, T, 3), A=A[ngf:].reshape(B, nf, T, 3), N=N[ngf:].reshape(B, nf, T, 3),
                    E=E[ngf:].reshape(B, nf, T, 3)))
    if terms:
        val, slot = np.zeros(n, np.float32), np.zeros(n, np.int64)
        lib().softras_oracle_backward_stats(*ins, *outs, *args, _p(val, C.c_float), _p(slot, C.c_int64), n)
        res[0]["terms"] = (val, slot)
    return tuple(res)


U = 2.0 ** -24      # fp32 unit roundoff
FTZ = 2.0 ** -125   # twice the smallest normal fp32


def backward_bound(st):
    """Per-entry bound on |CUDA gradient - g64| for one stats dict of backward(stats=True):

        bound = E * (1 + gamma) + gamma * A + N * 2^-125,   gamma = N u / (1 - N u),  u = 2^-24.

    Derivation.  The kernel's terms t'_i of a slot differ from the reference's float terms t_i by at most the
    per-site budgets, so sum |t'_i - t_i| <= E and sum |t'_i| <= A + E.  The kernel adds the t'_i in float, in some
    binary tree whatever the grouping: the shuffle merges between lanes, the vector and scalar atomics, any
    regrouping.  Starting from the zeroed accumulator, a tree of at most N float additions (adding a zero is exact) is
    within gamma_{N-1} sum |t'_i| of their exact sum (Higham, Accuracy and Stability
    of Numerical Algorithms, 4.2), independent
    of the order.  g64 is the same sum over the t_i in double, within N 2^-53 A of exact; gamma_N - gamma_{N-1} >= u
    covers that and the E gamma term is second order.  So
        |got - g64| <= E + gamma_{N-1} (A + E) + N 2^-53 A <= E (1 + gamma_N) + gamma_N A,
    which in the form 2^-24 (N + c) A has c = N^2 u / (1 - N u), below 1 for N < 4096.  The finalize kernel copies
    the accumulator into grad_faces / grad_textures unchanged, so no rounding follows the sum.  The global float
    atomics flush subnormal inputs and results to zero (PTX red.add.f32): each of at most N atomic adds into the slot
    loses < 2^-126 on its input and < 2^-126 on its result, hence the N 2^-125 floor, which only matters for sums in
    the subnormal range.  Non-finite entries are not bounded: compare their NaN / inf pattern instead."""
    N = st["N"].astype(np.float64)
    gamma = N * U / (1.0 - N * U)
    with np.errstate(invalid="ignore"):
        return st["E"] * (1.0 + gamma) + gamma * st["A"] + N * FTZ


def max_threads():
    return int(lib().softras_oracle_max_threads())
