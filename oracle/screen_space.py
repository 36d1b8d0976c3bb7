"""numpy restatement of the render2 screen-space kernels (csrc/screen_space_api.cu; the reference's SSAO_cuda.py,
SSDO_cuda.py and FXAA_cuda.py), for CPU checks against the reference goldens tests/golden/ref_screen_*.npz.

Float32 operations are numpy float32 operations in the kernels' order.  The reference's contracted a*b+c (FFMA) is
fma32, exact: a*b is exact in float64, the sum is rounded to float64 with round-to-odd and then to float32, which is
the correctly rounded fused result.  Its DFMAs with a double constant (the luma weights) are fma64, exact: the constant
is split so that both partial products are exact in float64, and math.fsum rounds the three-term sum once.

Two sites are not the device's operations bit for bit, and everything downstream of them inherits the difference:
  rsqrtf   MUFU.RSQ, an approximation within 2 ulp of 1/sqrt(x), here 1/sqrt(x) in float64 rounded to float32 (the TBN
           normalisation of SSAO and SSDO, and SSDO's direction to each indirect sample);
  cos, sin CUDA's double cos / sin (within 2 ulp) against numpy's (within 1 ulp), in each sample's direction.
Both move a sample point by an ulp or two of float32, which changes a result only where a sample's projection rounds
within that distance of a pixel boundary or its depth ties the depth buffer's within it.  So SSAO counts agree exactly
except at such pixels (tests/test_screen_space_cpu.py bounds how many), SSDO colours agree to a few ulp, and FXAA, which
has neither site, agrees bit for bit.

SSAO and SSDO take the draws as an input: draws [is * is, 3 * sample_num], pixel i's curand_init(1, i, 0) stream
(x, y, z of each sample in turn), as oracle/make_ref_screen_golden.py records them.
"""
import math

import numpy as np

f32, f64 = np.float32, np.float64
PI = 3.1415926


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c (arrays broadcast)."""
    a, b, c = (np.asarray(x, f32).astype(f64) for x in (a, b, c))
    p = a * b                                    # exact
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bv = s - p
        e = (p - (s - bv)) + (c - bv)            # s + e == p + c exactly (TwoSum)
        bits = s.view(np.int64)
        fix = np.isfinite(s) & np.isfinite(e) & (e != 0) & (bits & 1 == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)   # round to odd
    return s.astype(f32)


def _split(c):
    """c = hi + lo with hi the top 26 significant bits of c and lo (exact) the other 27."""
    hi = float((np.array([c], f64).view(np.int64) & ~np.int64((1 << 27) - 1)).view(f64)[0])
    return hi, c - hi


def fma64(a, c, t):
    """Correctly rounded float64 a * c + t for float32 a, a double constant c and float64 t."""
    hi, lo = _split(c)
    a = np.asarray(a, f32).astype(f64)
    ph, pl = a * hi, a * lo                      # both exact: 24 + 26 and 24 + 27 significant bits
    t = np.broadcast_to(np.asarray(t, f64), a.shape)
    out = np.empty(a.shape, f64)
    for i, (x, y, z) in enumerate(zip(ph.ravel(), pl.ravel(), t.ravel())):
        out.ravel()[i] = math.fsum((x, y, z)) if math.isfinite(x + y + z) else x + y + z
    return out


def roundf(x):
    """CUDA roundf: half away from zero."""
    x = np.asarray(x, f32).astype(f64)
    return np.trunc(x + np.copysign(0.5, x)).astype(f32)


def f2i(x):
    """CUDA's float-to-int conversion: truncation, saturating, NaN -> 0."""
    x = np.asarray(x, f64)
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(x), 0, np.clip(np.trunc(x), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def rsqrt(x):
    return (1.0 / np.sqrt(np.asarray(x, f32).astype(f64))).astype(f32)


def _frame(depth, normals, width, idx, is_):
    fis = f32(is_)
    xp, yp = (idx % is_).astype(f32), (idx // is_).astype(f32)
    xi = (f32(2) * xp + f32(1) - fis) / fis
    yi = (f32(2) * (f32(is_ - 1) - yp) + f32(1) - fis) / fis
    d = depth.reshape(-1)[idx]
    n = normals.reshape(-1, 3)[idx]
    nx, ny, nz = n[:, 0], n[:, 1], n[:, 2]
    w = f32(width)
    wx, wy = xi * w * d, yi * w * d
    first = (np.abs(nx) > f32(0.5)) | (np.abs(ny) > f32(0.5))
    r1 = rsqrt(fma32(nx, nx, ny * ny) + f32(0))
    r2 = rsqrt(fma32(nx, nx, fma32(nz, nz, 0)))
    with np.errstate(invalid="ignore"):
        tx = np.where(first, -ny * r1, nz * r2)
        ty = np.where(first, nx * r1, f32(0) * r2)
        tz = np.where(first, f32(0) * r1, -nx * r2)
    bx = fma32(ty, nz, -(tz * ny))
    by = fma32(tz, nx, -(tx * nz))
    bz = fma32(tx, ny, -(ty * nx))
    return dict(wx=wx, wy=wy, wz=d, nx=nx, ny=ny, nz=nz, tx=tx, ty=ty, tz=tz, bx=bx, by=by, bz=bz)


def _sample(F, u, is_, r, width):
    ux, uy, uz = u[:, 0], u[:, 1], u[:, 2]
    randr = np.sqrt(uz / f32(3))
    a = 2 * PI * ux.astype(f64)
    ry = randr * uy
    lx = (ry.astype(f64) * np.cos(a)).astype(f32)
    ly = randr * np.sqrt(fma32(-uy, uy, 1))
    lz = (ry.astype(f64) * np.sin(a)).astype(f32)
    s = [fma32(F["b" + c], lz, fma32(F["t" + c], lx, F["n" + c] * ly)) for c in "xyz"]
    p = [fma32(s[k], f32(r), F["w" + c]) for k, c in enumerate("xyz")]
    fis, w = f32(is_), f32(width)
    col = f2i(roundf(fis * (p[0] / p[2] / w + f32(1)) * f32(0.5)))
    row = f2i(fis - roundf(fis * (p[1] / p[2] / w + f32(1)) * f32(0.5)))
    j = (row * is_ + col + 2 ** 31) % 2 ** 32 - 2 ** 31     # size_t arithmetic truncated to int
    return p, j


def _samples(depth, face_ind, normals, width, sample_num, sample_range_r, draws):
    is_ = depth.shape[0]
    idx = np.nonzero(face_ind.reshape(-1) != -1)[0]
    F = _frame(depth.astype(f32), normals.astype(f32), width, idx, is_)
    u = np.asarray(draws, f32).reshape(is_ * is_, -1)[idx]
    with np.errstate(all="ignore"):
        for k in range(int(sample_num)):
            p, j = _sample(F, u[:, 3 * k:3 * k + 3], is_, sample_range_r, width)
            ok = (j >= 0) & (j < is_ * is_)
            yield idx, F, p, np.where(ok, j, 0), ok


def ssao(depth, face_ind, normals, width, sample_num, sample_range_r, draws):
    """SSAO_cuda -> occlusion [is, is] float32."""
    is_ = depth.shape[0]
    out = np.zeros(is_ * is_, f32)
    occ = None
    for idx, F, p, j, ok in _samples(depth, face_ind, normals, width, sample_num, sample_range_r, draws):
        occ = np.zeros(idx.size, f32) if occ is None else occ
        occ += (ok & (depth.reshape(-1)[j] < p[2])).astype(f32)
    idx = np.nonzero(face_ind.reshape(-1) != -1)[0]
    with np.errstate(all="ignore"):
        out[idx] = (np.zeros(idx.size, f32) if occ is None else occ) / f32(sample_num)
    return out.reshape(is_, is_)


def ssdo(color, depth, face_ind, normals, width, sample_num, sample_range_r, draws):
    """SSDO_cuda -> image [is, is, 3] float32."""
    is_ = depth.shape[0]
    col = np.asarray(color, f32).reshape(-1, 3)
    nrm = np.asarray(normals, f32).reshape(-1, 3)
    out = col.copy()
    idx = np.nonzero(face_ind.reshape(-1) != -1)[0]
    amb = np.zeros(idx.size, f32)
    ind = np.zeros((idx.size, 3), f32)
    with np.errstate(all="ignore"):
        area = f32(1) / f32(sample_num) * f32(sample_range_r) * f32(sample_range_r)
        for _, F, p, j, ok in _samples(depth, face_ind, normals, width, sample_num, sample_range_r, draws):
            front = ok & (depth.reshape(-1)[j].astype(f64) > p[2].astype(f64) - 0.01)
            amb += front.astype(f32)
            lit = ok & ~front
            d = [p[k] - F["w" + c] for k, c in enumerate("xyz")]
            d2 = fma32(d[2], d[2], fma32(d[0], d[0], d[1] * d[1]))
            dist, rm = np.sqrt(d2), rsqrt(d2)
            d = [x * rm for x in d]
            n = nrm[j]
            cr = np.fmax(-fma32(n[:, 2], d[2], fma32(n[:, 0], d[0], n[:, 1] * d[1])).astype(f64), 0.).astype(f32)
            cn = np.fmax(fma32(F["nz"], d[2], fma32(F["nx"], d[0], F["ny"] * d[1])).astype(f64), 0.).astype(f32)
            w = f32(0.2) * cr * cn * area / (dist * dist)
            for c in range(3):
                ind[:, c] = np.where(lit, fma32(col[j, c], w, ind[:, c]), ind[:, c])
        amb = amb / f32(sample_num)
        for c in range(3):
            out[idx, c] = fma32(amb, col[idx, c], ind[:, c])
    return out.reshape(is_, is_, 3)


def _tex(tex, xp, yp, is_):
    """tex_sample at float32 coordinate arrays -> [n, 3]."""
    hi = f64(f32(is_ - 1))
    xp = np.fmin(np.fmax(np.asarray(xp, f32).astype(f64), 0.), hi).astype(f32)
    yp = np.fmin(np.fmax(np.asarray(yp, f32).astype(f64), 0.), hi).astype(f32)
    yp = f32(is_ - 1) - yp
    x0, y0 = xp.astype(np.int64), yp.astype(np.int64)
    wx1 = xp - x0.astype(f32)
    wx2 = f32(1) - wx1
    wy1 = yp - y0.astype(f32)
    wy2 = f32(1) - wy1
    flat = tex.reshape(-1, 3)
    acc = np.zeros(xp.shape + (3,), f32)
    for p, wa, wb in ((x0 + y0 * is_, wx2, wy2), (x0 + (y0 + 1) * is_, wx2, wy1), (x0 + 1 + y0 * is_, wx1, wy2),
                      (x0 + 1 + (y0 + 1) * is_, wx1, wy1)):
        inside = p < is_ * is_
        v = np.where(inside[:, None], flat[np.where(inside, p, 0)], f32(0))
        with np.errstate(invalid="ignore"):
            acc = fma32(wb[:, None], wa[:, None] * v, acc)
    return acc


def _luma(c):
    s = fma64(c[:, 2], 0.114, fma64(c[:, 0], 0.299, c[:, 1].astype(f64) * 0.587))
    with np.errstate(invalid="ignore"):
        return np.sqrt(s.astype(f32))


def fxaa(texture):
    """FXAA_cuda -> image [is, is, 3] float32."""
    tex = np.asarray(texture, f32)
    is_ = tex.shape[0]
    i = np.arange(is_ * is_)
    ux, uy = (i % is_).astype(f32), f32(is_ - 1) - (i // is_).astype(f32)
    one = f32(1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        centre = _tex(tex, ux, uy, is_)
        lc = _luma(centre)
        ll, lr = _luma(_tex(tex, ux - one, uy, is_)), _luma(_tex(tex, ux + one, uy, is_))
        lu, ld = _luma(_tex(tex, ux, uy + one, is_)), _luma(_tex(tex, ux, uy - one, is_))
        lmin = np.fmin(lc, np.fmin(np.fmin(ld, lu), np.fmin(ll, lr)))
        lmax = np.fmax(lc, np.fmax(np.fmax(ld, lu), np.fmax(ll, lr)))
        rng = lmax - lmin
        keep = rng.astype(f64) < np.fmax(0.0312, lmax.astype(f64) * 0.125)
        lul, lur = _luma(_tex(tex, ux - one, uy + one, is_)), _luma(_tex(tex, ux + one, uy + one, is_))
        ldl, ldr = _luma(_tex(tex, ux - one, uy - one, is_)), _luma(_tex(tex, ux + one, uy - one, is_))
        du, lrs = ld + lu, ll + lr
        lcor, dcor, rcor, ucor = ldl + lul, ldl + ldr, ldr + lur, lur + lul
        D = lambda x: x.astype(f64)  # noqa: E731
        eh = (np.abs(-2.0 * D(ll) + D(lcor)) + np.abs(-2.0 * D(lc) + D(du)) * 2.0 + np.abs(-2.0 * D(lr) + D(rcor))).astype(f32)
        ev = (np.abs(-2.0 * D(lu) + D(ucor)) + np.abs(-2.0 * D(lc) + D(lrs)) * 2.0 + np.abs(-2.0 * D(ld) + D(dcor))).astype(f32)
        horiz = eh >= ev
        g1 = np.where(horiz, ld, ll) - lc
        g2 = np.where(horiz, lu, lr) - lc
        step = np.where(np.abs(g1) >= np.abs(g2), f32(-1), f32(1))
        avg = ((1.0 / 12.0) * (2.0 * D(du + lrs) + D(lcor) + D(rcor))).astype(f32)
        s1 = np.fmin(np.fmax(D(np.abs(avg - lc) / rng), 0.0), 1.0).astype(f32)
        s2 = ((-2.0 * D(s1) + 3.0) * D(s1) * D(s1)).astype(f32)
        off = np.fmax(f32(0), s2 * s2 * f32(0.75))
        fx = np.where(horiz, ux, fma32(step, off, ux))
        fy = np.where(horiz, fma32(step, off, uy), uy)
        final = _tex(tex, fx, fy, is_)
    return np.where(keep[:, None], centre, final).reshape(is_, is_, 3)
