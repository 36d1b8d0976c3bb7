"""CPU oracle of the mesh regularisers (TEST INFRASTRUCTURE; product code never imports it).

float64 numpy restatement, expression by expression, of
    jrender/loss/laplacian_loss.py:5-36   LaplacianLoss (dense nv x nv matrix exactly as :11-26 builds it)
    jrender/loss/flatten_loss.py:5-79     FlattenLoss   (edge table exactly as :12-30 builds it, O(E*F) scan included)
and their gradients by central differences in float64 -- no autograd, no hand-derived formula, so that check of the fused
CUDA kernels' gradients (csrc/mesh_loss_api.cu) is independent of the PyTorch mirror in jrender_b200/loss.py -- plus a
float32 emulation of the kernels' per-thread terms (flatten_terms, laplacian_terms), operation by operation, so the
kernels' outputs can also be held to the sum of those terms within a summation-order bound.
Pinned: tests/test_host_golden.py holds `laplacian()` / `flatten()` to the values the reference's own Python produced
(tests/golden/ref_host_loss_sphere280.npz, generator oracle/make_ref_host_golden.py).
"""
import numpy as np


def laplacian_matrix(nv, faces):
    """laplacian_loss.py:11-26."""
    lap = np.zeros([nv, nv], np.float32)
    f = np.asarray(faces).astype(np.int64)
    lap[f[:, 0], f[:, 1]] = -1
    lap[f[:, 1], f[:, 0]] = -1
    lap[f[:, 1], f[:, 2]] = -1
    lap[f[:, 2], f[:, 1]] = -1
    lap[f[:, 2], f[:, 0]] = -1
    lap[f[:, 0], f[:, 2]] = -1
    r, c = np.diag_indices(nv)
    lap[r, c] = -lap.sum(1)
    for i in range(nv):
        lap[i, :] /= lap[i, i]
    return lap.astype(np.float64)


def laplacian(x, lap):
    """laplacian_loss.py:30-34: x [B,nv,3] -> [B]."""
    y = np.einsum("ij,bjk->bik", lap, np.asarray(x, np.float64))
    return (y ** 2).sum((1, 2))


def flatten_edges(faces):
    """flatten_loss.py:11-30 -> v0s, v1s, v2s, v3s (the reference's own scan; set order replaced by sorted order,
    which only permutes the terms of a sum)."""
    f = np.asarray(faces).astype(np.int64)
    pairs = sorted(set(tuple(v) for v in np.sort(np.concatenate((f[:, 0:2], f[:, 1:3]), axis=0))))
    v0s = np.array([p[0] for p in pairs], np.int64)
    v1s = np.array([p[1] for p in pairs], np.int64)
    v2s, v3s = [], []
    for v0, v1 in zip(v0s, v1s):
        count = 0
        for face in f:
            if v0 in face and v1 in face:
                v = face[(face != v0) & (face != v1)]
                if count == 0:
                    v2s.append(int(v[0]))
                    count += 1
                else:
                    v3s.append(int(v[0]))
    return v0s, v1s, np.array(v2s, np.int64), np.array(v3s, np.int64)


def flatten(vertices, edges, eps=1e-6):
    """flatten_loss.py:38-79: vertices [B,nv,3] -> [B]."""
    x = np.asarray(vertices, np.float64)
    v0s, v1s, v2s, v3s = (x[:, e, :] for e in edges)

    def half(b):
        a = v1s - v0s
        al2 = (a ** 2).sum(-1)
        bl2 = (b ** 2).sum(-1)
        al1 = np.sqrt(al2 + eps)
        bl1 = np.sqrt(bl2 + eps)
        ab = (a * b).sum(-1)
        cos = ab / (al1 * bl1 + eps)
        sin = np.sqrt(1 - cos ** 2 + eps)
        c = a * (ab / (al2 + eps))[..., None]
        return b - c, bl1 * sin
    cb1, cb1l1 = half(v2s - v0s)
    cb2, cb2l1 = half(v3s - v0s)
    cos = (cb1 * cb2).sum(-1) / (cb1l1 * cb2l1 + eps)
    return ((cos + 1) ** 2).sum(1)


def numeric_grad(fn, x, weights, h=1e-6):
    """d (sum_b weights[b] * fn(x)[b]) / d x by central differences in float64 (x [B,nv,3])."""
    x = np.asarray(x, np.float64)
    g = np.zeros_like(x)
    w = np.asarray(weights, np.float64)
    # every batch element's loss depends on its own vertices only: perturb the same coordinate of all of them at once
    for i in range(x.shape[1]):
        for k in range(3):
            xp, xm = x.copy(), x.copy()
            xp[:, i, k] += h
            xm[:, i, k] -= h
            g[:, i, k] = w * (fn(xp) - fn(xm)) / (2 * h)
    return g


F = np.float32


def _sqrt(x):
    return x.sqrt() if hasattr(x, "sqrt") else np.sqrt(x)


# forward-mode rules of csrc/mesh_loss_api.cu's Dual (value [n], partials [n, 12]), one float32 rounding per operation
def _add(a, b):
    return a[0] + b[0], a[1] + b[1]


def _sub(a, b):
    return a[0] - b[0], a[1] - b[1]


def _mul(a, b):
    return a[0] * b[0], a[1] * b[0][:, None] + a[0][:, None] * b[1]


def _div(a, b):
    r = a[0] / b[0]
    ib = F(1) / b[0]
    return r, (a[1] - r[:, None] * b[1]) * ib[:, None]


def _dsqrt(a):
    r = _sqrt(a[0])
    return r, a[1] * (F(0.5) / r)[:, None]


def _dot3(a, b):   # ((xx + yy) + zz), the kernel's dot3
    return _add(_add(_mul(a[0], b[0]), _mul(a[1], b[1])), _mul(a[2], b[2]))


def _half_plane(a, b, eps):   # mesh_loss_api.cu half_plane
    al2, bl2 = _dot3(a, a), _dot3(b, b)
    al1 = _dsqrt((al2[0] + eps, al2[1]))
    bl1 = _dsqrt((bl2[0] + eps, bl2[1]))
    ab = _dot3(a, b)
    m = _mul(al1, bl1)
    cosv = _div(ab, (m[0] + eps, m[1]))
    cc = _mul(cosv, cosv)
    sinv = _dsqrt(((F(1) - cc[0]) + eps, -cc[1]))
    s = _div(ab, (al2[0] + eps, al2[1]))
    cb = [_sub(b[k], _mul(a[k], s)) for k in range(3)]
    return cb, _mul(bl1, sinv)


def flatten_terms(vertices, edges, eps=1e-6, lift=None):
    """k_flatten_loss per (batch, edge), in the kernel's float32 operation order: the loss term (cos + 1)^2 [B, E] and its
    12 forward-mode partials [B, E, 12] (coordinate c of v0s, v1s, v2s, v3s at 3k + c).  `lift` maps every float32 input
    array to another number type with the same operators (identity: float32)."""
    x = np.asarray(vertices, F)
    B = x.shape[0]
    idx = [np.asarray(e, np.int64) for e in edges]
    E = idx[0].shape[0]
    lift = lift or (lambda a: a)
    eps = F(eps)
    p = []
    for k in range(4):
        q = x[:, idx[k], :].reshape(-1, 3)
        comp = []
        for c in range(3):
            seed = np.zeros((B * E, 12), F)
            seed[:, 3 * k + c] = 1
            comp.append((lift(q[:, c]), lift(seed)))
        p.append(comp)
    with np.errstate(all="ignore"):
        a = [_sub(p[1][c], p[0][c]) for c in range(3)]
        cb1, l1 = _half_plane(a, [_sub(p[2][c], p[0][c]) for c in range(3)], eps)
        cb2, l2 = _half_plane(a, [_sub(p[3][c], p[0][c]) for c in range(3)], eps)
        m = _mul(l1, l2)
        cosv = _div(_dot3(cb1, cb2), (m[0] + eps, m[1]))
        c1 = (cosv[0] + F(1), cosv[1])
        t = _mul(c1, c1)
    return t[0], t[1]


def flatten_sums(vertices, edges, eps=1e-6):
    """term_sums of k_flatten_loss: 'loss' (entries [B]) and 'grad' (entries shaped like vertices)."""
    from .preraster import term_sums
    B, nv = np.shape(vertices)[:2]
    val, d = flatten_terms(vertices, edges, eps)
    E = len(edges[0])
    b = np.repeat(np.arange(B), E)
    slots = np.stack([b * nv * 3 + np.asarray(edges[k], np.int64)[np.arange(B * E) % E] * 3 + c
                      for k in range(4) for c in range(3)], 1)
    grad = term_sums(slots, d, B * nv * 3)
    return dict(loss=term_sums(b, val, B), grad={k: g.reshape(B, nv, 3) for k, g in grad.items()})


def laplacian_terms(vertices, nbr, nbr_w, diag, lift=None):
    """k_laplacian_loss per (batch, vertex) in the kernel's float32 order: y = x_i * diag_i, then y += x_nbr * w over the
    table row in slot order, skipping w == 0 (padding); term = (y0 y0 + y1 y1) + y2 y2.  -> (term [B, nv],
    self [B, nv, 3] = (2 y) diag, nbr_terms: list over table slots k of (rows [m] of the vertices with w != 0 there,
    [B, m, 3] = (2 y) w)).  `lift` as in flatten_terms."""
    x = np.asarray(vertices, F)
    nbr = np.asarray(nbr, np.int64)
    w = np.asarray(nbr_w, F)
    dg = np.asarray(diag, F)
    lift = lift or (lambda a: a)
    with np.errstate(all="ignore"):
        y = [lift(x[:, :, c]) * lift(dg[None]) for c in range(3)]
        slots = [np.flatnonzero(w[:, k] != 0) for k in range(w.shape[1])]
        for k, rows in enumerate(slots):
            wk = lift(w[rows, k][None])
            for c in range(3):
                y[c][:, rows] = y[c][:, rows] + lift(x[:, nbr[rows, k], c]) * wk
        term = (y[0] * y[0] + y[1] * y[1]) + y[2] * y[2]
        y2 = [F(2) * y[c] for c in range(3)]
        own = [y2[c] * lift(dg[None]) for c in range(3)]
        scat = [(rows, [y2[c][:, rows] * lift(w[rows, k][None]) for c in range(3)]) for k, rows in enumerate(slots)]
    return term, own, scat


def laplacian_sums(vertices, nbr, nbr_w, diag):
    """term_sums of k_laplacian_loss: 'loss' (entries [B]) and 'grad' (entries shaped like vertices)."""
    from .preraster import term_sums
    B, nv = np.shape(vertices)[:2]
    term, own, scat = laplacian_terms(vertices, nbr, nbr_w, diag)
    nbr = np.asarray(nbr, np.int64)
    base = np.arange(B)[:, None] * nv
    slots, vals = [], []
    for c in range(3):
        slots.append(((base + np.arange(nv)) * 3 + c).reshape(-1))
        vals.append(own[c].reshape(-1))
    for k, (rows, t) in enumerate(scat):
        for c in range(3):
            slots.append(((base + nbr[rows, k][None]) * 3 + c).reshape(-1))
            vals.append(t[c].reshape(-1))
    grad = term_sums(np.concatenate(slots), np.concatenate(vals), B * nv * 3)
    return dict(loss=term_sums(np.repeat(np.arange(B), nv), term.reshape(-1), B),
                grad={k: g.reshape(B, nv, 3) for k, g in grad.items()})
