"""Which code paths the NMR kernels take for a scene (TEST INFRASTRUCTURE, not product code).

A numpy float32 restatement of the per-face / per-sample decisions of jrender_b200/csrc/nmr_kernels.cuh, used to
assert that a test scene reaches the path it was built for and stays inside the reference's defined behaviour:

  k_nmr_zbuffer             bounding box <= kNmrSerialBox (32) pixels: the face's own thread; larger: the warp
  k_nmr_backward_pixel_map  per (edge, axis) pass and integer major coordinate d0 ("sample"): k9_pass, d1_cross,
                            in / out pixel, `live`, has0 / has1, the outward and inward scan ranges, and the flavour
                            each scan takes (k9_scan_out / generic k9_scan outwards; the lane-serial loop / the warp-wide
                            OWNER k9_scan inwards)

Every expression that picks a pixel (d0 range, d1_cross, d0_cross2, the bounding box) is evaluated in the kernel's
unfused float32 order, so the decisions match bit for bit.  The distance scales k0 / k1 use an IEEE division where the
kernel uses rcp.approx; they only enter `past_end_zero`, which scenes with power-of-two denominators reach exactly.
"""
import numpy as np

f32 = np.float32
INT_MAX = 2 ** 31 - 1
SERIAL_BOX = 32   # kNmrSerialBox
SERIAL_IN = 64    # kSerialIn


def _int_ok(x):
    """A float -> int conversion the reference defines: finite and inside int's range."""
    x = float(x)
    return np.isfinite(x) and -2.0 ** 31 < x < 2.0 ** 31


def pixel_coords(face, is_):
    """pp[num][dim] = 0.5f * (face * is + is - 1), float32 (the kernels' and the reference's :389-393)."""
    s = f32(is_)
    return [(f32(0.5) * (f32(face[k, 0]) * s + s - f32(1)), f32(0.5) * (f32(face[k, 1]) * s + s - f32(1))) for k in range(3)]


def backside(face):
    f = face.reshape(9).astype(np.float32)
    return bool((f[7] - f[1]) * (f[3] - f[0]) < (f[4] - f[1]) * (f[6] - f[0]))


def zbuffer_path(face, is_):
    """'culled', 'empty', 'serial' (thread walks <= 32 pixels) or 'warp' for k_nmr_zbuffer; also the UB check of the
    bounding-box conversions.  -> (path, defined)"""
    p = pixel_coords(face, is_)
    xs, ys = [q[0] for q in p], [q[1] for q in p]
    x_min, y_min, x_max, y_max = f32(is_), f32(is_), f32(0), f32(0)
    for x, y in zip(xs, ys):
        x_min, x_max = (x if x < x_min else x_min), (x if x > x_max else x_max)
        y_min, y_max = (y if y < y_min else y_min), (y if y > y_max else y_max)
    if backside(face):
        return "culled", True
    defined = all(_int_ok(v) for v in (x_min, x_max, y_min, y_max))
    if not defined:
        return "undefined", False
    ix0, ix1 = max(0, int(x_min)), min(is_ - 1, int(x_max))
    iy0, iy1 = max(0, int(y_min)), min(is_ - 1, int(y_max))
    if ix0 > ix1 or iy0 > iy1:
        return "empty", True
    return ("serial" if (ix1 - ix0 + 1) * (iy1 - iy0 + 1) <= SERIAL_BOX else "warp"), True


def _ceil(x):
    return f32(np.ceil(x))


def _floor(x):
    return f32(np.floor(x))


def k9_samples(face, fn, face_index_map, is_, eps):
    """Every sample K9 sets up for one face of one image (face [3,3] NDC, face_index_map [is, is] of that image, yi up).
    -> list of dicts; empty for a culled face.  Raises ValueError on a conversion the reference leaves undefined."""
    if backside(face):
        return []
    pp = pixel_coords(face, is_)
    eps = f32(eps)
    out = []
    for pass_ in range(6):
        edge, axis = pass_ >> 1, pass_ & 1
        pi = [(edge + n) % 3 for n in range(3)]
        p = [(pp[pi[n]][axis], pp[pi[n]][1 - axis]) for n in range(3)]   # p[num][dim] = pp[num][(dim + axis) % 2]
        if axis == 0:
            direction = -1 if p[0][0] < p[1][0] else 1
        else:
            direction = 1 if p[0][0] < p[1][0] else -1
        lo, hi = float(_ceil(min(p[0][0], p[1][0]))), float(max(p[0][0], p[1][0]))
        lo, hi = max(lo, 0.0), min(hi, is_ - 1.0)
        if not (_int_ok(lo) and _int_ok(hi)):
            raise ValueError("d0 range not convertible")
        for d0 in range(int(lo), int(hi) + 1):
            d0f = f32(d0)
            d1_cross = (p[1][1] - p[0][1]) / (p[1][0] - p[0][0]) * (d0f - p[0][0]) + p[0][1]
            c = _floor(d1_cross) if direction > 0 else _ceil(d1_cross)
            if not _int_ok(c):
                raise ValueError("d1_cross not convertible")
            d1_in = int(c)
            d1_out = d1_in + direction
            live = 0 <= d1_in < is_ and 0 <= d1_out < is_
            has0, has1 = bool(p[1][0] != d0f), bool(p[0][0] != d0f)
            s = dict(pass_=pass_, axis=axis, direction=direction, d0=d0, d1_cross=d1_cross, d1_in=d1_in,
                     d1_out=d1_out, live=live, has0=has0, has1=has1, out=None, inward=None, cross2_zero=False)
            out.append(s)
            if not live:
                continue
            line = face_index_map[:, d0] if axis == 0 else face_index_map[d0, :]   # the scan's pixels, by d1
            prod = (d0f - p[0][0]) * (d0f - p[2][0])
            if prod < 0:
                cross2 = (p[2][1] - p[0][1]) / (p[2][0] - p[0][0]) * (d0f - p[0][0]) + p[0][1]
            else:
                cross2 = (p[1][1] - p[2][1]) / (p[1][0] - p[2][0]) * (d0f - p[2][0]) + p[2][1]
            s["cross2_zero"] = bool(prod == 0)
            c2 = _ceil(cross2) if direction > 0 else _floor(cross2)
            if not _int_ok(c2):
                raise ValueError("d0_cross2 not convertible")
            ilim = int(c2)
            in_from, in_to = max(min(d1_in, ilim), 0), min(max(d1_in, ilim), is_ - 1)
            if in_from <= in_to:
                owned = int((line[in_from:in_to + 1] == fn).sum())
                s["inward"] = dict(from_=in_from, to=in_to, span=in_to - in_from,
                                   flavour="serial" if in_to - in_from < SERIAL_IN else "warp", owned=owned,
                                   unowned=in_to - in_from + 1 - owned)
            if line[d1_in] == fn:
                olim = is_ - 1 if direction > 0 else 0
                o_from, o_to = max(min(d1_out, olim), 0), min(max(d1_out, olim), is_ - 1)
                n = o_to - o_from + 1
                o = dict(from_=o_from, to=o_to, n=n, flavour="out" if (has0 and has1) else "generic",
                         toward_zero=direction < 0, past_end_zero=False, half=None)
                if has0 and has1:
                    # lanes past the end of the last trip pair: pixels o_from + n .. o_from + 64 * ceil(n / 64) - 1
                    span = p[1][0] - p[0][0]
                    scale = f32(2) / f32(is_)
                    k = (span / (p[1][0] - d0f) * scale, span / (d0f - p[0][0]) * scale)
                    side = f32(o_from) - d1_cross
                    for kk in k:
                        e = eps if f32(0) < side * kk else -eps
                        for d1 in range(o_from + n, o_from + 64 * ((n + 63) // 64)):
                            delta = f32(d1) - d1_cross
                            if float(delta) * float(kk) + float(e) == 0.0:   # exact: fma(delta, k, e) == 0
                                o["past_end_zero"] = True
                                o["half"] = "a" if (d1 - o_from) % 64 < 32 else "b"
                o["residue"] = n % 64
                s["out"] = o
    return out


def scene_paths(faces, face_index_map, is_, eps):
    """All samples of a batch: faces [B, nf, 3, 3], face_index_map [B, is, is] (the oracle's)."""
    res = []
    for b in range(faces.shape[0]):
        for fn in range(faces.shape[1]):
            for s in k9_samples(faces[b, fn], fn, face_index_map[b], is_, eps):
                s["b"], s["fn"] = b, fn
                res.append(s)
    return res
