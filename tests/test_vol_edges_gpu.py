"""NeRF volume rendering kernels (csrc/vol_api.cu) at the edges where their order of arithmetic, their tiling and their
shared-memory bound show: tile seams (samples 32 k - 1, 32 k, 32 k + 1 and S = 1024, the 32-tile limit of the
backward's first pass), transmittances that go subnormal and then 0, the resampler's sort buffer at and past a power
of two, ties in its searchsorted, and NaN / inf inputs.

  forward    bit-exact against oracle.volume.composite where every exp is exactly 0 or 1; elsewhere within a
             per-element bound derived from where expf enters (forward_bound)
  backward   float64 autograd of oracle.volume.integrator_mirror, each ray held to its own largest gradient
  resampler  bit-exact against oracle.volume.resample, NaN-aware, in both modes
  NaN / inf  one bad ray per batch: the oracle's NaN / inf pattern, and every other ray bit-identical to a clean run

The tests without the gpu mark run on the CPU: they check, through the oracle, that each case reaches what it targets.
"""
import numpy as np
import pytest
import torch

from jrender_b200 import vol
from oracle import volume as ov
from tests.test_vol_gpu import GRADS, OUTS, cu, ray_batch, scene

gpu = pytest.mark.gpu
F32 = np.float32
U = 2.0 ** -24                    # unit roundoff of float32
FLT_MIN = np.finfo(F32).tiny
OPAQUE = F32(1e3)                 # sigma of an opaque sample: exp argument <= -1e3 on unit intervals


def nan_equal(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def same_nonfinite(a, b, what):
    """NaN, +inf and -inf in the same places of a and b; returns the mask of b's finite entries."""
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s NaN pattern differs" % what
    assert np.array_equal(np.isposinf(a), np.isposinf(b)) and np.array_equal(np.isneginf(a), np.isneginf(b)), what
    return np.isfinite(b)


# ---- exactness-pinned forward cases ----------------------------------------------------------------------------------

PINNED_S = [31, 32, 33, 63, 64, 65, 1023, 1024]


def pinned_case(S, seed=0):
    """Rays whose every exp argument is 0 (sigma <= 0) or <= -1e3 (sigma = 1e3 on intervals >= 1), so alpha and e
    are exactly 0 or 1, and whose colour logits are 0 or +-inf, so each sigmoid is exactly 0, 1/2 or 1.  z = 2, 3, ...
    and |d| in {1, 2, 5} keep every interval exact.  Opaque samples sit on lanes 0 and 31 and at 32 k - 1, 32 k,
    32 k + 1; ray 10 is opaque throughout (T reaches 1e-10^k, subnormal, then 0)."""
    rng = np.random.default_rng(seed)
    seams = [p for k in range(0, S // 32 + 1) for p in (32 * k - 1, 32 * k, 32 * k + 1) if 0 <= p < S]
    opaque = [[], [0], [min(31, S - 1)], seams, [p for p in seams if p % 32 == 31], [p for p in seams if p % 32 == 0],
              [S - 1], [p for p in (30, 31, 32, 33, 34) if p < S], list(np.flatnonzero(rng.random(S) < .05)),
              [p for p in (1, 63, 64, 65, 1022) if p < S], list(range(S))]
    N = len(opaque)
    raw = rng.choice(np.array([0., np.inf, -np.inf], F32), (N, S, 4))
    raw[..., 3] = rng.choice(np.array([0., -1., -np.inf], F32), (N, S))
    for r, ps in enumerate(opaque):
        raw[r, ps, 3] = OPAQUE
    z = np.broadcast_to(F32(2) + np.arange(S, dtype=F32), (N, S)).copy()
    d = np.array([[1, 0, 0], [0, 3, 4], [0, 0, 2], [0, -4, 3], [-2, 0, 0]], F32)[np.arange(N) % 5]
    return raw, z, d


def opaque_runs_case(S=96):
    """Ray r holds r + 1 consecutive opaque samples (up to 6) over a tile seam, between empty samples: the
    transmittance goes 1, 1e-10, 1e-20, 1e-30, subnormal, 0.  The rows repeat with the run starting at 28, 29, 30."""
    N = 18
    raw = np.zeros((N, S, 4), F32)
    raw[..., 3] = -1
    for r in range(N):
        start = 28 + r // 6
        raw[r, start:start + r % 6 + 1, 3] = OPAQUE
    raw[:, :, :3] = np.array([0, np.inf, -np.inf], F32)
    z = np.broadcast_to(F32(2) + np.arange(S, dtype=F32), (N, S)).copy()
    d = np.tile(np.array([[1, 0, 0]], F32), (N, 1))
    return raw, z, d


def forward_both(raw, z, d, noise=None, white=False):
    got = [o.cpu().numpy() for o in vol._composite(*cu(raw, z, d, noise), white)]
    tr = {}
    ref = ov.composite(raw, z, d, noise, white, trace=tr)
    return dict(zip(OUTS, got)), ref, tr


@gpu
@pytest.mark.parametrize("S", PINNED_S)
def test_forward_is_bit_exact_where_every_exp_is_0_or_1(cuda_device, S):
    raw, z, d = pinned_case(S, seed=S)
    got, ref, _ = forward_both(raw, z, d, white=S % 2 == 1)
    for k in OUTS:
        assert nan_equal(got[k], ref[k]), (k, np.flatnonzero(~((got[k] == ref[k]) | np.isnan(ref[k]))))


@gpu
@pytest.mark.parametrize("S", [96, 1024])
def test_forward_weights_are_bit_exact_through_subnormal_transmittance(cuda_device, S):
    raw, z, d = opaque_runs_case(S)
    got, ref, _ = forward_both(raw, z, d)
    for k in OUTS:
        assert nan_equal(got[k], ref[k]), k


# ---- general forward cases: a per-element bound ------------------------------------------------------------------------

def forward_bound(tr, ref, raw, z, white):
    """Per-element bounds on |kernel - oracle| for the five outputs.

    The kernel and the oracle evaluate the same float32 expressions in the same order, so they differ only because
    expf (CUDA: 2 ulp) and numpy's exp differ on the same argument: |de| <= 3 ulp(e) <= 3 * 2^-24 for e < 1.  Then
    alpha = 1 - e moves by at most |de| plus one rounding of 1 - e, and t = (1 - alpha) + 1e-10 (exact but for its
    own rounding, relative 2u) by at most delta = 2 ulp(1) = 2^-22 absolute.  T_i = prod_{k<i} t_k inherits
    |dT_i| <= T_i sum_{k<i} delta / t_k, and w_i = alpha_i T_i
        |dw_i| <= delta T_i + alpha_i T_i sum_{k<i} delta / t_k + 2u (i + K + 8) w_i + (K + 8) 2^-149,
    the third term the roundings of the t_k and of the <= K + 7 products that form w_i from them (K tiles, 5 scan
    levels), each a relative 2u apart between the two sides, the last the same roundings in the subnormal range.
    T_i / t_k <= prod of the other t_j, so behind an opaque sample (t = 1e-10) the bound shrinks with T, instead of
    the flat 4e-6 that let every weight below it go unchecked.  T is formed in float64 from the oracle's own t.
    A sum of n = K + 5 rounded additions moves by sum |dx| + 2 n u sum |x|.  A sigmoid s = 1 / (1 + E) moves by at
    most 10 u s (3 ulp of E through ds/dE = -s^2 E / E, plus two roundings).  With a white background rgb gains
    (1 - acc): |d acc| and two more roundings."""
    S = z.shape[1]
    K = -(-S // 32)
    n_sum = K + 5
    delta = 2.0 ** -22
    t = tr["t"].astype(np.float64)
    a = tr["alpha"].astype(np.float64)
    T = np.cumprod(np.concatenate([np.ones_like(t[:, :1]), t[:, :-1]], -1), -1)
    inv_excl = np.cumsum(1 / t, -1) - 1 / t
    w = np.abs(ref["weights"].astype(np.float64))
    i = np.arange(S)
    dw = delta * T + a * T * inv_excl * delta + 2 * U * (i + K + 8) * w + (K + 8) * 2.0 ** -149
    bound = dict(weights=dw)
    bound["acc_map"] = dw.sum(-1) + 2 * n_sum * U * w.sum(-1) + (n_sum + 1) * 2.0 ** -149
    s = 1 / (1 + np.exp(-raw[..., :3].astype(np.float64)))
    rgb = (dw[..., None] * s + w[..., None] * 10 * U * s).sum(1) + 2 * (n_sum + 1) * U * (w[..., None] * s).sum(1)
    if white:
        rgb = rgb + bound["acc_map"][:, None] + 4 * U * (1 + np.abs(ref["rgb_map"]))
    bound["rgb_map"] = rgb + (n_sum + 1) * 2.0 ** -149
    za = np.abs(z.astype(np.float64))
    bound["depth_map"] = (dw * za).sum(-1) + 2 * (n_sum + 1) * U * (w * za).sum(-1) + (n_sum + 1) * 2.0 ** -149
    # disp = 1 / (depth / acc) where that quotient is taken: the relative errors of depth and acc plus two divisions;
    # elsewhere the constant 1e10, exactly
    acc, dep, disp = (ref[k].astype(np.float64) for k in ("acc_map", "depth_map", "disp_map"))
    with np.errstate(invalid="ignore", divide="ignore"):
        taken = ref["disp_map"] != F32(1e10)
        rel = bound["depth_map"] / np.abs(dep) + bound["acc_map"] / acc + 4 * U
        bound["disp_map"] = np.where(taken, np.abs(disp) * rel / np.maximum(1 - rel, 0), 0)
    return bound


def check_bounded(got, ref, tr, raw, z, white, rays=slice(None)):
    """Every output within forward_bound on the rays given, with the oracle's NaN / inf pattern; where the bound is
    not finite (the oracle's t is not) the value must be exact.  Returns the largest ratio of error to bound."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        bound = forward_bound(tr, ref, raw, z, white)
    worst = 0.
    for k in OUTS:
        g, r = got[k][rays].astype(np.float64), ref[k][rays].astype(np.float64)
        m = same_nonfinite(g, r, k)
        err = np.abs(g - r)[m]
        b = np.nan_to_num(bound[k][rays], nan=0., posinf=0.)[m]
        assert np.all(err <= b), (k, (err / np.maximum(b, 1e-300)).max())
        with np.errstate(invalid="ignore", divide="ignore"):
            worst = max(worst, np.nan_to_num(err / b).max(initial=0.))
    return worst


@gpu
@pytest.mark.parametrize("N,S,noise,white", [(37, 31, 0., False), (37, 32, .5, True), (37, 33, 0., False),
                                             (37, 64, 1., False), (19, 65, 0., True), (9, 1023, 0., False),
                                             (9, 1024, .5, True), (1000, 96, 0., False)])
def test_forward_within_the_expf_bound(cuda_device, N, S, noise, white):
    raw, z, d = scene(N, S, seed=7 * S)
    raw[2, 31 % S, 3] = raw[3, 32 % S, 3] = raw[4, 33 % S, 3] = 1e4          # opaque on the seams
    raw[5, ::29, 3] = 30.                                                    # dense: T runs down towards 0
    nz = np.random.default_rng(3).normal(0, noise, (N, S)).astype(F32) if noise else None
    got, ref, tr = forward_both(raw, z, d, nz, white)
    ratio = check_bounded(got, ref, tr, raw, z, white)
    print("forward error / bound, N=%d S=%d: %.3g" % (N, S, ratio))


# ---- non-finite inputs, one bad ray per batch ---------------------------------------------------------------------------

BAD = 2   # the bad ray of each batch


def corrupt(case, raw, z, d):
    """Give ray BAD the non-finite input `case`."""
    b = BAD
    if case == "sigma_nan":
        raw[b, [0, 31, 32, 33], 3] = np.nan
    elif case == "sigma_posinf":
        raw[b, [5, 31, 32], 3] = np.inf
    elif case == "sigma_neginf":
        raw[b, [5, 32, 64], 3] = -np.inf
    elif case == "rgb_nan":
        raw[b, 7, 0] = np.nan
    elif case == "rgb_inf":
        raw[b, 7, 1], raw[b, 33, 2] = np.inf, -np.inf
    elif case == "d_nan":
        d[b] = [np.nan, 0., 1.]
    elif case == "d_inf":
        d[b] = [np.inf, 0., 0.]
    elif case == "d_zero":
        d[b] = 0.
    elif case == "d_zero_sigma_inf":
        d[b] = 0.
        raw[b, 10, 3] = np.inf
    elif case == "z_nan":
        z[b, 20] = np.nan
    elif case == "z_repeat_sigma_inf":   # inf * 0 on a zero-length interval
        z[b, 41] = z[b, 40]
        raw[b, 40, 3] = np.inf
    else:
        raise KeyError(case)


NONFINITE = ["sigma_nan", "sigma_posinf", "sigma_neginf", "rgb_nan", "rgb_inf", "d_nan", "d_inf", "d_zero",
             "d_zero_sigma_inf", "z_nan", "z_repeat_sigma_inf"]


def bad_batch(case, S=70):
    raw, z, d = scene(6, S, seed=11)
    clean = [a.copy() for a in (raw, z, d)]
    corrupt(case, raw, z, d)
    return (raw, z, d), clean


@gpu
@pytest.mark.parametrize("case", NONFINITE)
def test_forward_nonfinite_ray_follows_the_oracle_and_leaves_the_others(cuda_device, case):
    (raw, z, d), clean = bad_batch(case)
    with np.errstate(invalid="ignore", over="ignore"):
        got, ref, tr = forward_both(raw, z, d, white=True)
    check_bounded(got, ref, tr, raw, z, True)
    ok, _, _ = forward_both(*clean, white=True)
    others = np.arange(raw.shape[0]) != BAD
    for k in OUTS:
        assert np.array_equal(got[k][others], ok[k][others]), k


def backward(raw, z, d, ups, use, white=False, noise=None):
    r = cu(raw)[0].requires_grad_(True)
    outs = vol._composite(r, *cu(z, d, noise), white)
    loss = sum((o * cu(ups[k])[0]).sum() for k, o in zip(OUTS, outs) if k in use)
    g, = torch.autograd.grad(loss, r)
    return g.cpu().numpy()


def mirror_grad(raw, z, d, ups, use, white, noise, dtype, relu=torch.relu):
    t = lambda a: None if a is None else torch.from_numpy(a).to(dtype)
    r = t(raw).requires_grad_(True)
    outs = ov.integrator_mirror(r, t(z), t(d), t(noise), white, relu=relu)
    loss = sum((o * t(ups[k])).sum() for k, o in zip(OUTS, outs) if k in use)
    g, = torch.autograd.grad(loss, r)
    return g.numpy().astype(np.float64)


def upstream(N, S, seed=5):
    """Upstream gradients scaled per ray by 10^-6 ... 1, so that no ray hides behind another's magnitude."""
    rng = np.random.default_rng(seed)
    scale = (10. ** -np.linspace(6, 0, N)).astype(F32)
    ups = {k: rng.normal(0, 1, s).astype(F32) for k, s in zip(OUTS, ((N, 3), (N,), (N,), (N, S), (N,)))}
    ups["disp_map"] *= F32(1e-2)   # disp is up to 1e10 on empty rays: keep its term comparable
    for k in ups:
        ups[k] *= scale.reshape((N,) + (1,) * (ups[k].ndim - 1))
    return ups


def float32_floor(raw, z, d, ups, use, white, g64):
    """Per ray, what float32 can resolve of dL/dsigma_i = T_i (G_i - R_i) e_i dist_i (DESIGN.md section 9).

    Where the true gradient is far below the upstream gradients (acc alone on a ray whose last sample is opaque: acc
    is 1 whatever sigma_i), it is the difference of the two terms T G e dist and T R e dist.  The kernel forms R by
    a scan of affine maps x -> t x + G a: two roundings per step, over 5 in-tile levels and K tile carries, on terms
    bounded by |G_i| and max_{j>i} |G_j| (the a_j prod t_k after sample i sum to at most 1).  So it resolves the
    gradient to 4 (K + 8) u max_i T_i e_i dist_i (|G_i| + max_{j>i} |G_j|), in float64 from the inputs here.
    Each gradient also carries its T_i's relative error from the forward (forward_bound: delta sum_{k<i} 1 / t_k,
    delta = 2^-22), which over a thin ray of 1024 samples exceeds 1e-5: add max_i |g64_i| delta sum_{k<i} 1 / t_k."""
    r64, z64, d64 = (np.asarray(a, np.float64) for a in (raw, z, d))
    N, S = z64.shape
    K = -(-S // 32)
    dist = np.concatenate([np.diff(z64, axis=-1), np.full((N, 1), 1e10)], -1) * np.sqrt((d64 ** 2).sum(-1))[:, None]
    x = r64[..., 3]
    e = np.exp(-np.where(x > 0, x, 0) * dist)
    t = e + 1e-10
    T = np.cumprod(np.concatenate([np.ones((N, 1)), t[:, :-1]], -1), -1)
    w = (1 - e) * T
    s = 1 / (1 + np.exp(-r64[..., :3]))
    g = {k: np.asarray(ups[k], np.float64) * (k in use) for k in OUTS}
    G = g["acc_map"][:, None] + g["depth_map"][:, None] * z64 + (s * g["rgb_map"][:, None, :]).sum(-1) + g["weights"]
    if white:
        G = G - g["rgb_map"].sum(-1)[:, None]
    acc, dep = w.sum(-1), (w * z64).sum(-1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = dep / acc
        take = q > 1e-10
        gq = np.where(take, -g["disp_map"] / q ** 2, 0)
        G = G + np.where(take, gq / acc, 0)[:, None] * z64 - np.where(take, gq * dep / acc ** 2, 0)[:, None]
    Ga = np.abs(G)
    behind = np.concatenate([np.maximum.accumulate(Ga[:, :0:-1], -1)[:, ::-1], np.zeros((N, 1))], -1)
    cancel = 4 * (K + 8) * U * (np.where(x > 0, T * e * dist, 0) * (Ga + behind)).max(-1)
    drift = 2. ** -22 * (np.abs(g64[..., 3]) * (np.cumsum(1 / t, -1) - 1 / t)).max(-1)
    return cancel + drift


def check_per_ray(g, g64, g32, what, floor64=None):
    """Each ray to 1e-5 of its own largest float64 gradient, or, where float32 cannot resolve the gradient (the
    difference of two O(upstream) terms), to the larger of 4x the op-by-op float32 mirror's error on that ray and
    float32_floor; returns the worst ratio of error to the ray's own largest gradient."""
    worst = 0.
    for r in range(g.shape[0]):
        err = np.abs(g[r] - g64[r]).max()
        scale = np.abs(g64[r]).max()
        floor = np.nan_to_num(4 * np.abs(g32[r] - g64[r]).max(), nan=0., posinf=0.)
        if floor64 is not None:
            floor = max(floor, floor64[r])
        tol = max(1e-5 * scale, floor) + 1e-30
        assert err <= tol, (what, r, err, scale, floor)
        worst = max(worst, err / max(scale, 1e-300))
    return worst


def seam_case(S):
    """12 rays: opaque samples on lane 31 / 0 / 1 of a seam, on the last sample and on several seams at once; ray 7
    sparse (a few dense samples 97 apart) and ray 8 thin, so the last tile still carries weight."""
    raw, z, d = scene(12, S, seed=13 * S)
    raw[2, 31 % S, 3] = raw[3, 32 % S, 3] = raw[4, 33 % S, 3] = raw[5, S - 1, 3] = 1e4
    raw[6, [p for p in (31, 63, 64, 992) if p < S], 3] = 1e4
    raw[7, :, 3] = -np.abs(raw[7, :, 3]) + np.where(np.arange(S) % 97 == 0, F32(3), F32(0))
    raw[8, :, 3] = np.abs(raw[8, :, 3]) * F32(.05)
    return raw, z, d


@gpu
@pytest.mark.parametrize("which", GRADS)
@pytest.mark.parametrize("S", [31, 32, 33, 64, 65, 993, 1024])
def test_backward_per_ray_on_tile_seams(cuda_device, which, S):
    raw, z, d = seam_case(S)
    N = raw.shape[0]
    white = S % 2 == 0
    ups = upstream(N, S)
    use = OUTS if which == "all" else (which,)
    g = backward(raw, z, d, ups, use, white)
    g64 = mirror_grad(raw, z, d, ups, use, white, None, torch.float64)
    g32 = mirror_grad(raw, z, d, ups, use, white, None, torch.float32)
    assert np.all(np.isfinite(g64)) and np.all(np.isfinite(g))
    worst = check_per_ray(g, g64, g32, which, float32_floor(raw, z, d, ups, use, white, g64))
    print("backward worst per-ray error / own max |grad|, S=%d %s: %.3g" % (S, which, worst))


@gpu
@pytest.mark.parametrize("case", NONFINITE)
def test_backward_nonfinite_ray_leaves_the_others(cuda_device, case):
    (raw, z, d), clean = bad_batch(case)
    N, S = z.shape
    ups = upstream(N, S)
    g = backward(raw, z, d, ups, OUTS, white=True)
    ok = backward(*clean, ups, OUTS, white=True)
    others = np.arange(N) != BAD
    assert np.array_equal(g[others], ok[others])
    if case == "sigma_nan":
        # the kernel reads relu(NaN) as 0: the sample is empty, its density gradient 0, and the ray's other
        # gradients are those of float64 autograd under the same reading
        g64 = mirror_grad(raw, z, d, ups, OUTS, True, None, torch.float64, relu=ov.kernel_relu)
        g32 = mirror_grad(raw, z, d, ups, OUTS, True, None, torch.float32, relu=ov.kernel_relu)
        assert np.all(np.isfinite(g[BAD])) and np.all(g[BAD][np.isnan(raw[BAD, :, 3]), 3] == 0)
        check_per_ray(g[BAD:BAD + 1], g64[BAD:BAD + 1], g32[BAD:BAD + 1], case)


# ---- the resampler -------------------------------------------------------------------------------------------------------

FINE_SIZES = [(1023, 1), (513, 511), (512, 512), (2, 1022), (33, 31), (64, 128), (33, 30), (1000, 23)]
PATTERNS = ["random", "zero", "one_hot", "two_hot", "nan", "inf", "z_nan", "spiky"]


def nan_rays(S):
    """The rays of fine_case whose every fine sample is NaN: a NaN or an inf weight in the pdf, or at S = 2 (no pdf
    weights) the NaN z."""
    return [PATTERNS.index("nan"), PATTERNS.index("inf")] if S > 2 else [PATTERNS.index("z_nan")]


def pad_of(S, Ni):
    P = 1
    while P < S + Ni:
        P <<= 1
    return P - (S + Ni)


def pdf_weights(n, rng, z=None):
    """One row of weights per pattern in PATTERNS, each of n entries; z [len(PATTERNS), S] is edited for z_nan."""
    w = np.zeros((len(PATTERNS), n), F32)
    w[0] = rng.exponential(1, n)
    if n > 2:
        w[2, n // 3] = 1.
        w[3, [1, n - 2]] = [.25, 2.]
    w[4:7] = rng.exponential(1, (3, n))
    if n:
        w[4, n // 2], w[5, n // 2] = np.nan, np.inf
    if z is not None:
        z[6, z.shape[1] // 2] = np.nan
    w[7] = np.where(rng.random(n) < .03, rng.exponential(1, n), 0).astype(F32)
    return w


def tie_u(cdf, Ni, rng):
    """Exact cdf entries (searchsorted ties at right=True) that end a plateau, then u = 0, 1 - 2^-24, 1, then the
    other cdf entries; row r starts r entries in, so that with few samples the rows still differ."""
    N = cdf.shape[0]
    u = np.empty((N, Ni), F32)
    for r in range(N):
        c = cdf[r]
        steps = np.diff(c, prepend=c[:1])
        fin = np.isfinite(c)
        flat, rest = np.flatnonzero((steps < 1e-5) & fin)[1:], np.flatnonzero((steps >= 1e-5) & fin)
        vals = np.concatenate([c[rng.permutation(flat)], [0., 1. - 2. ** -24, 1.], c[rng.permutation(rest)]])
        u[r] = np.resize(np.roll(vals.astype(F32), -r), Ni)
    return u


def fine_case(S, Ni, umode, seed=0):
    """(z [N, S], weights [N, S], u [N, Ni] or None) with one ray per pattern of PATTERNS."""
    rng = np.random.default_rng(seed + S * 7 + Ni)
    N = len(PATTERNS)
    z = np.sort(rng.uniform(2, 6, (N, S)).astype(F32), -1)
    w = np.zeros((N, S), F32)
    w[:, 1:S - 1] = pdf_weights(S - 2, rng, z)
    u = None
    if umode == "random":
        u = rng.random((N, Ni)).astype(F32)
    elif umode == "ties":
        tr = {}
        with np.errstate(invalid="ignore"):
            ov.resample(w, 1, None, z_vals=z, trace=tr)
        u = tie_u(tr["cdf"], Ni, rng)
    return z, w, u


def oracle_resample(*a, **k):
    with np.errstate(invalid="ignore"):
        return ov.resample(*a, **k)


@gpu
@pytest.mark.parametrize("umode", ["det", "random", "ties"])
@pytest.mark.parametrize("S,Ni", FINE_SIZES)
def test_fine_stage_is_bit_exact(cuda_device, S, Ni, umode):
    z, w, u = fine_case(S, Ni, umode)
    zs, zf = vol._resample(*cu(z, w), Ni, None if u is None else cu(u)[0])
    zs, zf = zs.cpu().numpy(), zf.cpu().numpy()
    ref_s, ref_f = oracle_resample(w, Ni, u, z_vals=z)
    assert nan_equal(zs, ref_s), np.argwhere(~((zs == ref_s) | (np.isnan(zs) & np.isnan(ref_s))))[:8]
    assert nan_equal(zf, ref_f), np.argwhere(~((zf == ref_f) | (np.isnan(zf) & np.isnan(ref_f))))[:8]
    assert nan_equal(zf, np.sort(np.concatenate([z, zs], -1), -1))   # torch.sort's order, NaN last
    assert np.all(np.isnan(zf[nan_rays(S), S:])) and not np.isinf(zf).any()


@gpu
@pytest.mark.parametrize("umode", ["det", "random", "ties"])
@pytest.mark.parametrize("nb,Ni", [(1023, 1), (512, 512), (2, 5), (40, 64)])
def test_sample_pdf_is_bit_exact(cuda_device, nb, Ni, umode, monkeypatch):
    rng = np.random.default_rng(nb + Ni)
    N = len(PATTERNS)
    bins = np.sort(rng.uniform(-3, 5, (N, nb)).astype(F32), -1)
    bins[6, nb // 2] = np.nan
    w = pdf_weights(nb - 1, rng)
    u = None
    if umode == "random":
        u = rng.random((N, Ni)).astype(F32)
    elif umode == "ties":
        tr = {}
        oracle_resample(w, 1, None, bins=bins, trace=tr)
        u = tie_u(tr["cdf"], Ni, rng)
    if u is not None:
        monkeypatch.setattr(vol, "_random", lambda shape, device, normal=False: cu(u)[0])
    got = vol.sample_pdf(*cu(bins, w), Ni, det=u is None).cpu().numpy()
    ref, _ = oracle_resample(w, Ni, u, bins=bins)
    assert nan_equal(got, ref), np.argwhere(~((got == ref) | (np.isnan(got) & np.isnan(ref))))[:8]


@gpu
def test_render_rays_keeps_nan_rays_to_themselves(cuda_device, monkeypatch):
    """Rays whose density is +inf on zero-length intervals (zero direction, or near == far) get NaN coarse weights.
    Their fine z_vals must hold NaN where the samples were, not inf; every other ray renders exactly as it does in a
    batch without them.  A NaN density (read as empty) and an all-opaque ray ride along."""
    N, S, Ni = 64, 64, 128
    rays = ray_batch(N, cuda_device, seed=3)
    rays[3, 3:6] = 0.
    rays[17, 7] = rays[17, 6]
    nan_rays, odd_rays = [3, 17], [3, 17, 40, 41]
    keep = [i for i in range(N) if i not in odd_rays]
    rec = []
    real_resample = vol._resample

    def resample(z, w, n, u):
        out = real_resample(z, w, n, u)
        rec.append((z.cpu().numpy(), w.cpu().numpy()) + tuple(o.cpu().numpy() for o in out))
        return out
    monkeypatch.setattr(vol, "_resample", resample)

    def query(rows):
        def q(pts, viewdirs, fn):
            raw = ov.field_torch(pts, viewdirs, 4)
            for i, v in ((3, np.inf), (17, np.inf), (40, np.nan), (41, np.inf)):
                if i in rows:
                    raw[rows.index(i), :, 3] = v
            return raw
        return q
    kw = dict(network_fn=None, N_samples=S, perturb=0., N_importance=Ni, white_bkgd=True, retraw=True)
    odd = vol.render_rays(rays, network_query_fn=query(list(range(N))), **kw)
    z, w, zs, zf = rec[-1]
    clean = vol.render_rays(rays[keep], network_query_fn=query(keep), **kw)

    assert np.isnan(w[nan_rays]).any(axis=1).all()
    ref_s, ref_f = oracle_resample(w, Ni, None, z_vals=z)
    assert nan_equal(zs, ref_s) and nan_equal(zf, ref_f)
    assert np.all(np.isnan(zf[nan_rays, S:])) and not np.isinf(zf).any()
    for k in odd:
        assert torch.equal(odd[k][keep], clean[k]), k


# ---- CPU: each case reaches what it targets ------------------------------------------------------------------------------

@pytest.mark.parametrize("S", PINNED_S)
def test_pinned_cases_take_every_exp_at_0_or_below_minus_104(S):
    raw, z, d = pinned_case(S, seed=S)
    tr = {}
    ov.composite(raw, z, d, trace=tr)
    arg = tr["exp_arg"]
    assert np.all((arg == 0) | (arg <= -104))
    assert np.all(np.isin(np.exp(arg), [0, 1])) and np.all(np.isin(tr["alpha"], [0, 1]))
    assert np.all(np.isin(raw[..., :3], [0, np.inf, -np.inf]))
    with np.errstate(over="ignore"):
        assert np.all(np.isin(ov._sigmoid(raw[..., :3]), [0, .5, 1]))
    opaque = tr["alpha"] == 1
    for p in (0, 31, 32, 33, 63, 64, 65, S - 1):
        if p < S:
            assert opaque[:, p].any(), p
    T = tr["T"]
    assert ((T > 0) & (T < FLT_MIN)).any() and (T == 0).any()


@pytest.mark.parametrize("S", [96, 1024])
def test_opaque_runs_take_transmittance_subnormal_then_to_zero(S):
    raw, z, d = opaque_runs_case(S)
    tr = {}
    ref = ov.composite(raw, z, d, trace=tr)
    w, a = ref["weights"], tr["alpha"]
    assert np.array_equal(a == 1, raw[..., 3] == OPAQUE)
    for r in range(raw.shape[0]):
        run = w[r][a[r] == 1]   # the weights of the run are its transmittances
        n = r % 6 + 1
        assert run.size == n and run[0] == 1
        if n >= 5:
            assert 0 < run[4] < FLT_MIN     # 1e-40: subnormal
        if n == 6:
            assert run[5] == 0
        tail = w[r][np.flatnonzero(a[r] == 1)[-1] + 1:]
        assert np.all(tail == 0)


@pytest.mark.parametrize("case", NONFINITE)
def test_nonfinite_cases_reach_nonfinite_arithmetic(case):
    """Each case changes the bad ray's arithmetic where it targets: NaN / inf appear in the oracle's outputs, or (NaN
    density, +-inf colour, zero direction) the outputs stay finite under the kernels' reading."""
    (raw, z, d), _ = bad_batch(case)
    tr = {}
    with np.errstate(invalid="ignore", over="ignore"):
        ref = ov.composite(raw, z, d, white_bkgd=True, trace=tr)
    bad_out = np.concatenate([np.atleast_1d(ref[k][BAD]) for k in OUTS])
    finite_cases = {"sigma_nan", "sigma_posinf", "sigma_neginf", "rgb_inf", "d_zero"}
    assert np.all(np.isfinite(bad_out)) == (case in finite_cases), case
    if case in ("d_zero_sigma_inf", "z_repeat_sigma_inf", "d_inf"):
        assert np.isnan(tr["exp_arg"][BAD]).any()   # inf * 0
    if case == "sigma_posinf":
        assert np.all(tr["alpha"][BAD, [5, 31, 32]] == 1)
    for k in OUTS:
        others = np.delete(np.atleast_2d(ref[k].T).T, BAD, 0)
        assert np.all(np.isfinite(others)), k


def test_seam_backward_cases_hold_alpha_one_on_the_seams():
    for S in (33, 64, 1024):
        raw, z, d = seam_case(S)
        tr = {}
        ov.composite(raw, z, d, trace=tr)
        a = tr["alpha"]
        assert a[2, 31] == 1 and a[3, 32] == 1 and a[4, 33 % S] == 1 and a[5, S - 1] == 1 and a[6, 31] == 1
        assert 0 < tr["T"][7, -1] and tr["T"][7, -1] > 1e-3       # the sparse ray reaches its last tile unshadowed


@pytest.mark.parametrize("S,Ni", FINE_SIZES)
def test_fine_cases_reach_nan_merges_ties_and_plateaus(S, Ni):
    z, w, u = fine_case(S, Ni, "ties")
    tr = {}
    zs, zf = oracle_resample(w, Ni, u, z_vals=z, trace=tr)
    assert np.isnan(zs[nan_rays(S)]).all() and np.isnan(zf[nan_rays(S), S:]).all()
    assert np.isnan(zf[PATTERNS.index("z_nan")]).sum() >= 1
    assert pad_of(S, Ni) == {(1023, 1): 0, (513, 511): 0, (512, 512): 0, (2, 1022): 0, (33, 31): 0, (64, 128): 64,
                             (33, 30): 1, (1000, 23): 1}[(S, Ni)]
    cdf, uu, inds, denom = tr["cdf"], tr["u"], tr["inds"], tr["denom"]
    hits = (cdf[:, None, :] == uu[:, :, None]).any(-1)
    assert hits[[0, 2, 3, 7]].any(axis=1).all()                    # u equal to a cdf entry
    if Ni >= 3:
        assert hits[1].any()
        assert (uu == 0).any() and (uu == F32(1 - 2. ** -24)).any() and (uu == 1).any()
    if S > 3:
        assert (denom[PATTERNS.index("one_hot")] < 1e-5).any() and (denom[PATTERNS.index("two_hot")] < 1e-5).any()
        # counting cdf < u instead of cdf <= u moves some tie to another sample
        strict = (cdf[:, None, :] < uu[:, :, None]).sum(-1)
        assert ((strict != inds) & hits).any()
        moved = strided_samples(tr, z, strict)
        assert not nan_equal(moved, zs)


def strided_samples(tr, z, inds):
    """The fine samples the oracle's formula gives from another searchsorted count."""
    cdf, u = tr["cdf"], tr["u"]
    bins = F32(.5) * (z[:, 1:] + z[:, :-1])
    nb = bins.shape[1]
    below, above = np.maximum(0, inds - 1), np.minimum(nb - 1, inds)
    g = lambda a, i: np.take_along_axis(a, i, 1)
    cdf0, cdf1, bin0, bin1 = g(cdf, below), g(cdf, above), g(bins, below), g(bins, above)
    with np.errstate(invalid="ignore"):
        denom = cdf1 - cdf0
        denom = np.where(denom < F32(1e-5), F32(1), denom)
        return bin0 + ((u - cdf0) / denom) * (bin1 - bin0)


def test_merge_padding_decides_where_nan_samples_land():
    """The sort network of k_vol_resample in numpy: padding with +inf puts +inf where the NaN samples belong once the
    buffer is longer than S + Ni; padding with NaN gives np.sort's result."""
    def network(vals, P, pad):
        buf = np.concatenate([vals, np.full(P - vals.size, pad, F32)])
        size = 2
        while size <= P:
            stride = size >> 1
            while stride > 0:
                for i in range(P // 2):
                    lo = 2 * i - (i & (stride - 1))
                    hi = lo + stride
                    a, b = buf[lo], buf[hi]
                    gt = a > b or (np.isnan(a) and not np.isnan(b))
                    if gt == ((lo & size) == 0):
                        buf[lo], buf[hi] = b, a
                stride >>= 1
            size <<= 1
        return buf[:vals.size]
    vals = np.array([1, np.nan, 2, 3, .5], F32)
    assert nan_equal(network(vals, 8, np.nan), np.sort(vals))
    assert nan_equal(network(vals, 8, np.inf), np.array([.5, 1, 2, 3, np.inf], F32))
    rng = np.random.default_rng(0)
    for n, P in ((63, 64), (192, 256), (64, 64)):
        v = rng.normal(0, 1, n).astype(F32)
        v[rng.random(n) < .2] = np.nan
        assert nan_equal(network(v, P, np.nan), np.sort(v))
