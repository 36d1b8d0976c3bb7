"""Seeded hostile inputs for the texture bake and atlas kernels (csrc/bake_api.cu, csrc/texture_atlas_api.cu), shared by
tests/test_texture_edges_cpu.py (each case reaches the edges it names, the emulation agrees with float64, subtly wrong
emulations are caught) and tests/test_texture_edges_gpu.py (the kernels against the emulation, bit for bit).

UVs sit exactly on 0, 1 and texel centres k / (W - 1), one ulp either side, below 0 (the SoftRas bake extrapolates
there), at +-1e6, +-3e9 (past int range), +-inf, NaN and -0.0, and on integers and half-integers for the NMR wrap modes.
Images are 1 x 1, 1 x W, H x 1, non-square and 2048^2, with NaN and inf pixels in column 0 and in the last pixel (a UV
of 1 reads pixel (y + 1, 0) with weight 0 there) and -0.0 pixels (a sum started from -0.0 would keep the sign).
Atlas tiles hold degenerate triangles (den + 1e-5 == 0), slivers, NaN vertices and vertices on pixel centres.
"""
import numpy as np

from oracle import texture_atlas as oat

F = np.float32
SOFTRAS_R = (1, 2, 5, 16)
N3MR_TS = (2, 3, 4, 8)
SHAPES = ((1, 1), (1, 7), (5, 1), (6, 11), (32, 32), (9, 40))
HUGE = (1e6, -1e6, 3e9, -3e9, np.inf, -np.inf, np.nan, -0.0)


def around(values):
    """Each value and the float32 one ulp below and above it."""
    v = np.asarray(values, F)
    return np.concatenate([np.nextafter(v, F(-np.inf)), v, np.nextafter(v, F(np.inf))])


def seam_uvs(H, W):
    """0 and 1, the texel centres k / (W - 1) and k / (H - 1), and one ulp either side of each."""
    cent = [k / (n - 1) for n in (H, W) if n > 1 for k in range(n)]
    return around([0.0, 1.0] + cent)


def image(rng, H, W, nonfinite=False):
    """Values in [-0.25, 1] with -0.0 and exact zeros; with `nonfinite`, NaN and +-inf in column 0 and inf in the last
    pixel."""
    img = rng.uniform(-0.25, 1.0, (H, W, 3)).astype(F)
    m = rng.random((H, W, 3))
    img[m < 0.05] = -0.0
    img[(m >= 0.05) & (m < 0.08)] = 0.0
    img[0, 0, 1] = -0.0
    if nonfinite:
        rows = rng.random(H) < 0.5
        img[rows, 0, rng.integers(0, 3)] = np.nan
        img[~rows, 0, rng.integers(0, 3)] = np.inf if rng.random() < 0.5 else -np.inf
        img[-1, -1, :] = np.inf
    return img


def _faces(rng, nf, pool):
    """[nf, 3, 2] UVs drawn from `pool`; the first half of the faces have their three vertices on one UV, so every
    texel's position is that UV (up to the sample weights' sum) and lands exactly on the seams in the pool."""
    pool = np.asarray(pool, F)
    uv = rng.choice(pool, (nf, 3, 2))
    h = nf // 2
    uv[:h] = rng.choice(pool, (h, 1, 2))
    return uv.astype(F)


def softras_cases():
    """dicts: name, image [H, W, 3], faces_uv [nf, 3, 2], textures [nf, R*R, 3] (input), is_update [nf]."""
    rng = np.random.default_rng(2024)
    out = []
    k = 0
    for H, W in SHAPES:
        for kind in ("seams", "negative", "huge", "mixed"):
            R = SOFTRAS_R[k % len(SOFTRAS_R)]
            k += 1
            nf = 48
            if kind == "seams":
                pool = seam_uvs(H, W)
            elif kind == "negative":
                pool = np.concatenate([rng.uniform(-1.5, 0, 16), around([-0.0, -1.0, -0.5])])
            elif kind == "huge":
                pool = np.concatenate([np.asarray(HUGE), seam_uvs(H, W)[:6], [0.25, 0.5]])
            else:
                pool = rng.uniform(-0.2, 1.2, 32)
            uv = _faces(rng, nf, pool)
            if kind == "mixed":
                uv[nf // 2:] = rng.uniform(-0.2, 1.2, (nf - nf // 2, 3, 2))
            tex = rng.random((nf, R * R, 3)).astype(F)
            tex[0, 0] = [np.nan, -0.0, np.inf]                 # kept bit for bit where is_update == 0
            upd = (rng.random(nf) < 0.75).astype(np.int32)
            upd[0], upd[1] = 0, 1
            out.append(dict(name="softras_%dx%d_%s_R%d" % (H, W, kind, R), image=image(rng, H, W, nonfinite=(k % 2 == 0)),
                            faces_uv=uv, textures=tex, is_update=upd))
    # one bake of more than 2^24 texels
    nf, R = (1 << 24) // 256 + 37, 16
    uv = rng.uniform(-0.1, 1.1, (nf, 3, 2)).astype(F)
    uv[::97] = 1.0
    out.append(dict(name="softras_large_R16", image=image(rng, 64, 48), faces_uv=uv,
                    textures=np.zeros((nf, R * R, 3), F), is_update=(rng.random(nf) < 0.9).astype(np.int32)))
    return out


def n3mr_cases():
    """dicts: name, image, faces_uv, textures [nf, ts, ts, ts, 3], is_update.  Each runs under every wrap mode and
    both samplers."""
    rng = np.random.default_rng(2025)
    out = []
    ints = np.arange(-3, 4, dtype=F)
    pool = np.concatenate([ints, ints + F(0.5), around([0.0, 1.0, 2.0, -1.0, 0.5]), [-0.0], np.asarray(HUGE, F)])
    for i, (H, W) in enumerate(SHAPES):
        ts = N3MR_TS[i % len(N3MR_TS)]
        nf = 40
        uv = _faces(rng, nf, np.concatenate([pool, seam_uvs(H, W)]))
        uv[-8:] = rng.uniform(-2.3, 3.1, (8, 3, 2))
        tex = rng.random((nf, ts, ts, ts, 3)).astype(F)
        tex[0, 0, 0, 0] = [np.nan, -0.0, np.inf]
        upd = (rng.random(nf) < 0.75).astype(np.int32)
        upd[0], upd[1] = 0, 1
        out.append(dict(name="n3mr_%dx%d_ts%d" % (H, W, ts), image=image(rng, H, W, nonfinite=(i % 2 == 1)),
                        faces_uv=uv, textures=tex, is_update=upd))
    return out


DEGENERATE = np.array([[0, 0], [1, 0], [0, -1e-5]], F)     # den = -1e-5f exactly: den + 1e-5f == 0
COLLINEAR = np.array([[0, 0], [4, 4], [8, 8]], F)          # den == 0: weights scaled by 1e5


def atlas_cases():
    """dicts: name, tile_vertices [nf, 3, 2], texture_res_out, tile_width, H, W, and the textures of both kinds
    (softras [nf, R*R, 3], n3mr [nf, ts, ts, ts, 3])."""
    rng = np.random.default_rng(2026)
    out = []
    for i, (nf, R_out) in enumerate(((1, 2), (7, 4), (10, 5), (26, 16), (130, 8))):
        tri, tw, th = oat.atlas_layout(nf, R_out)
        tri = tri.copy()
        kind = np.arange(nf) % 6
        col, row = (np.arange(nf) % tw) * R_out, (np.arange(nf) // tw) * R_out
        origin = np.stack([col, row], -1)[:, None, :].astype(F)
        jit = (tri + rng.uniform(-0.3, 0.3, tri.shape)).astype(F)
        tri[kind == 1] = jit[kind == 1]                                       # off the pixel centres
        tri[kind == 2] = DEGENERATE                                           # divides by zero
        tri[kind == 3] = (origin + COLLINEAR * F(R_out / 16))[kind == 3]      # sliver: den 0 or nearly
        nanv = tri[kind == 4]
        nanv[:, rng.integers(0, 3), rng.integers(0, 2)] = np.nan
        tri[kind == 4] = nanv                                                 # a NaN vertex
        # kind 0 and 5: the layout's own triangles, vertices on pixel centres
        R, ts = SOFTRAS_R[i % 4], N3MR_TS[i % 4]
        tex = rng.random((nf, R * R, 3)).astype(F)
        vol = rng.random((nf, ts, ts, ts, 3)).astype(F)
        tex[-1, -1, 0] = np.nan
        out.append(dict(name="atlas_nf%d_Rout%d" % (nf, R_out), tile_vertices=tri.astype(F), texture_res_out=R_out,
                        tile_width=tw, H=th * R_out, W=tw * R_out, softras=tex, n3mr=vol))
    return out
