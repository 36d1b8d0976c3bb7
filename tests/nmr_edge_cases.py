"""Scenes that drive the NMR kernels onto specific paths (shared by test_nmr_edges_cpu.py and test_nmr_edges_gpu.py).

Faces are built in pixel coordinates p and converted with x = (2 p + 1 - is) / is, the inverse of the kernels'
p = 0.5 (x is + is - 1): at a power-of-two image size an integer or dyadic p is exact in float32 both ways.  Every
face is front-facing (counter-clockwise); z is given per face or per vertex.
"""
import numpy as np


def ndc(p, is_):
    return (2.0 * np.asarray(p, np.float64) + 1.0 - is_) / is_


def face(pix, is_, z=1.0):
    """pix: three (px, py) pixel-space vertices -> [3, 3] float32 NDC face, reordered counter-clockwise."""
    v = np.asarray(pix, np.float64)
    if (v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[1, 1] - v[0, 1]) * (v[2, 0] - v[0, 0]) < 0:
        v = v[[0, 2, 1]]
    z = np.broadcast_to(np.asarray(z, np.float64), (3,))
    return np.concatenate([ndc(v, is_), z[:, None]], 1).astype(np.float32)


def transpose(f):
    """Swap x and y (the other scan axis), keeping the face front-facing."""
    g = f[:, [1, 0, 2]].copy()
    return g[[0, 2, 1]]


def stack(scenes):
    """list of [nf_b, 3, 3] -> [B, nf, 3, 3], shorter scenes padded with culled (clockwise, off-screen) faces."""
    nf = max(len(s) for s in scenes)
    pad = np.array([[5, 5, 1], [5, 6, 1], [6, 5, 1]], np.float32)   # clockwise: culled, and off-screen
    out = np.empty((len(scenes), nf, 3, 3), np.float32)
    for b, s in enumerate(scenes):
        out[b, :len(s)] = s
        out[b, len(s):] = pad
    return out


def textures(faces, ts=2, seed=0, const=None):
    B, nf = faces.shape[:2]
    if const is not None:
        return np.broadcast_to(np.asarray(const, np.float32), (B, nf, ts, ts, ts, 3)).copy()
    return np.random.default_rng(seed).random((B, nf, ts, ts, ts, 3), dtype=np.float32)


# ---------------------------------------------------------------- long inward scans
def long_inward(is_=256):
    """Large triangles whose rows / columns shrink by less than one pixel per step, so the inward spans take every width
    from 0 to a few hundred (63, 64 and 65 included); small faces in front cover part of each, so the warp-wide scan's
    owner test drops pixels.  Image 1 is image 0 transposed, with its own occluders."""
    rng = np.random.default_rng(11)
    scenes = []
    for b in range(2):
        big = [face([(6.3, 8.6), (249.4, 14.2), (20.7, 246.1)], is_, 2.0),
               face([(250.2, 247.3), (100.6, 250.4), (246.8, 30.9)], is_, 2.5)]
        small = []
        for _ in range(24):
            c = rng.uniform(20, 230, 2)
            r = rng.uniform(2.5, 9.0)
            a = rng.uniform(0, 2 * np.pi)
            small.append(face([c + r * np.array([np.cos(a + t), np.sin(a + t)]) for t in (0, 2.1, 4.2)], is_, 1.0))
        s = np.stack(big + small)
        if b == 1:
            s = np.stack([transpose(f) for f in s])
        scenes.append(s)
    return stack(scenes)


# ---------------------------------------------------------------- outward trip seams
SEAM_N = (1, 31, 32, 33, 63, 64, 65, 96, 97)


def outward_seams(is_=256):
    """Small faces whose outward scans have n in SEAM_N pixels toward each border.  Image 0: faces at x ~ n and at
    x ~ is - n (scans along x, axis 1); image 1: its transpose (scans along y, axis 0).  Each n has a face with
    fractional vertices (k9_scan_out) and one with integer pixel-coordinate vertices (has0 / has1 false: the generic
    scan)."""
    fs = []
    row = 6.0
    for n in SEAM_N:
        for frac in (True, False):
            y = row
            row += 9.0
            # left-facing edge at x in (n - 1, n]: the outward scan toward 0 covers 0 .. n - 1
            if frac:
                fs.append(face([(n - 0.375, y + 0.25), (n + 4.625, y + 2.75), (n + 0.375, y + 6.25)], is_))
                xr = is_ - n
                fs.append(face([(xr - 4.625, y + 0.25), (xr + 0.375, y + 3.25), (xr - 0.625, y + 6.75)], is_))
            else:
                fs.append(face([(n, y), (n + 5, y + 3), (n + 1, y + 7)], is_))
                xr = is_ - n
                fs.append(face([(xr - 6, y + 1), (xr - 1, y + 3), (xr - 2, y + 7)], is_))
    s = np.stack(fs)
    return stack([s, np.stack([transpose(f) for f in s])])


def past_end(is_=256):
    """k9_scan_out scans toward pixel 0 whose first lane past the end sits at d1_in, where fma(delta, k, -eps) is
    exactly 0 for eps = 2^-10: an edge at minor coordinate Y + 0.9375 (delta = 1/16) over a major span of 4 sampled
    at its midpoint (k = 2 / 2 * 2 / 256 = 2^-6).  n = Y + 1 takes residues 70 % 64 = 6 and 20 (the trip pair's `a`
    half), 110 % 64 = 46, 46 and 97 % 64 = 33 (the `b` half).  Image 0 scans along y (axis 0), image 1 is its
    transpose (axis 1).  Use with eps = 2^-10."""
    fs = []
    for x0, Y in ((20, 109), (60, 69), (100, 96), (140, 19), (180, 45)):
        y = Y + 0.9375
        # apex off the integer rows: at an integer apex the sample there takes d0_cross2 through the horizontal
        # edge's zero-length major span, an infinite crossing whose int conversion the reference leaves undefined
        fs.append(face([(x0 - 2, y), (x0 + 2, y), (x0, y + 20.3125)], is_))
    s = np.stack(fs)
    return stack([s, np.stack([transpose(f) for f in s])])


PAST_END_EPS = 2.0 ** -10


# ---------------------------------------------------------------- pixel-aligned vertices
def pixel_aligned(is_=64, nf=14, seed=3):
    """Vertices on integer pixel coordinates (pixel 0 and is - 1 included), no two vertices of a face sharing an x or a
    y: the edges are never axis-aligned on an integer line (reference UB), but samples at a vertex's own major
    coordinate have has0 / has1 false and take the d0_cross2 else-branch with a zero product."""
    rng = np.random.default_rng(seed)
    scenes = []
    for b in range(2):
        fs = [face([(0, 5), (is_ - 1, 0), (20, is_ - 1)], is_, 3.0), face([(is_ - 1, is_ - 3), (3, is_ - 1), (40, 9)], is_, 3.5)]
        while len(fs) < nf:
            v = rng.integers(0, is_, (3, 2))
            if len(set(v[:, 0])) < 3 or len(set(v[:, 1])) < 3:
                continue
            if abs((v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[1, 1] - v[0, 1]) * (v[2, 0] - v[0, 0])) < 20:
                continue
            fs.append(face(v, is_, rng.uniform(1.0, 3.0)))
        scenes.append(np.stack(fs))
    return stack(scenes)


# ---------------------------------------------------------------- image sizes
def tiny(is_, seed=0):
    """A few random faces at image size 1, 2, 31 or 33 (B = 2)."""
    rng = np.random.default_rng(seed + is_)
    scenes = []
    for b in range(2):
        fs = []
        while len(fs) < 5:
            v = rng.uniform(-1.3, 1.3, (3, 2))
            if abs((v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[1, 1] - v[0, 1]) * (v[2, 0] - v[0, 0])) < 0.2:
                continue
            f = np.concatenate([v, rng.uniform(1, 3, (3, 1))], 1).astype(np.float32)
            if (f[1, 0] - f[0, 0]) * (f[2, 1] - f[0, 1]) - (f[1, 1] - f[0, 1]) * (f[2, 0] - f[0, 0]) < 0:
                f = f[[0, 2, 1]]
            fs.append(f)
        scenes.append(np.stack(fs))
    return stack(scenes)


def huge(is_=4096):
    """Eight large faces at the ABI's largest image size: scans of ~4000 pixels (delta += 64 over ~60 trip pairs)."""
    fs = [face([(10.3, 20.6), (4080.7, 60.2), (200.4, 4070.9)], is_, 3.0),
          face([(4085.2, 4090.1), (30.8, 4060.3), (4050.6, 100.4)], is_, 3.5),
          face([(1000.5, 1000.25), (3000.75, 1200.5), (1500.25, 3100.125)], is_, 2.0),
          face([(2500.3, 500.7), (3900.1, 2600.4), (2200.9, 2400.2)], is_, 1.5),
          face([(300.6, 2000.2), (1200.3, 2500.8), (400.1, 3900.5)], is_, 1.0),
          face([(2000.2, 3800.7), (2100.4, 3600.1), (2300.6, 3950.3)], is_, 0.5),
          face([(50.1, 50.2), (90.3, 60.4), (60.5, 95.6)], is_, 0.5),
          face([(3500.7, 3300.2), (4095.0, 3700.5), (3600.4, 4095.0)], is_, 0.8)]
    return np.stack(fs)[None]


# ---------------------------------------------------------------- depth order
def depth_order(is_=64):
    """near < 0.  Image 0: faces at negative depth over faces at positive depth, and faces whose vertices' z have mixed
    signs.  Image 1: duplicate faces with exactly equal depth (lowest id must win), and the signed-zero tie: a face
    with z = +0 and one with z = -0 over the same pixels (depth 1 / (w / z) = +-0), in both id orders."""
    a = [face([(4.5, 3.25), (60.25, 10.5), (12.75, 58.5)], is_, 2.0),
         face([(8.25, 6.5), (50.5, 20.75), (20.5, 50.25)], is_, -1.5),
         face([(30.5, 30.25), (62.25, 40.5), (35.75, 62.5)], is_, -0.5),
         face([(2.5, 40.25), (30.25, 35.5), (10.75, 62.5)], is_, (1.5, -2.0, 0.75)),
         face([(20.5, 2.25), (45.25, 4.5), (40.75, 30.5)], is_, (-3.0, -0.25, -1.0))]
    d = face([(3.5, 2.25), (28.25, 5.5), (8.75, 29.5)], is_, 1.25)
    pz = face([(34.5, 2.25), (61.25, 6.5), (40.75, 29.5)], is_, 0.0)
    nz = pz.copy()
    nz[:, 2] = -0.0
    pz2 = face([(3.5, 34.25), (29.25, 38.5), (9.75, 61.5)], is_, 0.0)
    nz2 = pz2.copy()
    nz2[:, 2] = -0.0
    b = [d, d.copy(), pz, nz, nz2, pz2, face([(36.5, 36.25), (60.25, 40.5), (44.75, 60.5)], is_, -1.0),
         face([(38.5, 34.25), (62.25, 44.5), (40.75, 62.5)], is_, -1.0)]
    return stack([np.stack(a), np.stack(b)])


DEPTH_NEAR, DEPTH_FAR = -5.0, 5.0


# ---------------------------------------------------------------- partly off-screen
def off_screen(is_=128, seed=5):
    """Faces with vertices at NDC +-1.5 .. +-4: samples whose in / out pixel is off the image (live false) and scan
    ranges clamped at the borders."""
    rng = np.random.default_rng(seed)
    scenes = []
    for b in range(2):
        fs = []
        while len(fs) < 8:
            v = rng.uniform(-1.0, 1.0, (3, 2))
            k = rng.integers(0, 3)
            v[k] = rng.choice([-1, 1], 2) * rng.uniform(1.5, 4.0, 2)
            if abs((v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[1, 1] - v[0, 1]) * (v[2, 0] - v[0, 0])) < 0.3:
                continue
            f = np.concatenate([v, rng.uniform(1, 3, (3, 1))], 1).astype(np.float32)
            if (f[1, 0] - f[0, 0]) * (f[2, 1] - f[0, 1]) - (f[1, 1] - f[0, 1]) * (f[2, 0] - f[0, 0]) < 0:
                f = f[[0, 2, 1]]
            fs.append(f)
        scenes.append(np.stack(fs))
    return stack(scenes)
