"""Counts the 16-byte gradient atomics (packets) k_softras_backward_lane issues, on the CPU oracle's per-pair terms.

    python tools/count_softras_bwd_packets.py [--workload c3 c2 c5] [--row-step 16]

For each workload it takes image 0, runs the oracle forward on row pairs (r, r + 1) for r = 0, row_step, ..., and the
oracle backward on the same rows, recovers every (pixel, face) pair's 12 terms (9 vertex, 3 colour), and replays the
kernel's warp walk on them: lanes map to pixels as in k_softras_backward_lane (8 columns x 4 rows per warp, lane & 7 ->
column, lane >> 3 -> row), every slot m the lanes that hold the same face as lane ^ 1 and then lane ^ 8 add their
terms in float32 into the lower lane, and each surviving lane issues its packets.  Row pairs are sampled, not single
rows, so that the vertical (^ 8) merge sees the neighbour it has in the kernel.

Reported per workload: pairs, the packets of the interleaved layout [v0.xyz v1.x] [v1.yz v2.xy] [v2.z t0 t1 t2] issued
unconditionally, the same layout with all-zero packets skipped, and the zero-class layout [v0.xy v1.xy]
[v2.xy v0.z v1.z] [v2.z t0 t1 t2] with all-zero packets skipped.  A packet is all zero when each of its four merged sums
is +0 or -0.  Silhouettes (aggr_func_rgb 'none') have only the first two packets.  The counts are scaled to the whole
step (all rows, all images of the workload) by the row sampling rate and the image count.

The oracle reports only non-zero terms and the gradient slot each one lands in.  To attribute them to pairs, the
backward runs on a face array with one copy of the face per pair, and each pair's id points at its own copy.  The
copies change no term for the softmax and silhouette settings counted here (only aggr_func_alpha 'sum' and
aggr_func_rgb 'hard' read the face count or the face id).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jrender_b200 import workloads as wl  # noqa: E402
from oracle import softras as osr  # noqa: E402

# name: (faces, image size, images per step, scene kwargs, oracle params, upstream gradient channels)
WORKLOADS = {
    "c3": (39200, 1024, 4, {}, {}, 4),
    "c2": (3280, 1024, 8, {}, {}, 4),
    # demo2-deform's silhouette pass: unit sphere, sigma 1e-4, only the alpha gradient; eye distance 2.535 at the
    # scene builder's 30 degree view frames the sphere as demo2's 5.464 at 15 degrees does
    "c5": (3280, 512, 120, dict(radius=1.0, distance=2.535), dict(sigma_val=1e-4, aggr_func_rgb="none"), 1),
}

INTERLEAVED = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10, 11]]   # indices into gv[0..8] ++ gt[0..2]
ZERO_CLASS = [[0, 1, 3, 4], [6, 7, 2, 5], [8, 9, 10, 11]]


def pair_terms(fv, tex, P, g, rows):
    """-> ids [K, len(rows), H] (image 0, sampled rows) and terms [K, len(rows), H, 12] float32 per pair."""
    H, K = int(P["image_size"]), int(P["max_faces_per_pixel_for_grad"])
    assert tex.shape[2] == 1 and P["aggr_func_alpha"] != "sum" and P["aggr_func_rgb"] != "hard"
    fwd = dict(soft_colors=np.zeros((1, 4, H, H), np.float32), aggrs_info=np.zeros((1, 2, H, H), np.float32),
               faces_id_buffer=np.full((1, K, H, H), -1, np.int32))
    step = rows[2] - rows[0]
    for r0 in rows[:2]:
        o = osr.forward(fv, tex, P, rows=(r0, H), row_stride=step, nthreads=osr.max_threads())
        for k in ("soft_colors", "aggrs_info", "faces_id_buffer"):
            fwd[k][:, :, r0::step] = o[k][:, :, r0::step]
    ids = fwd["faces_id_buffer"][0][:, rows]                 # [K, R, H]
    # every pair reads its own copy of its face, so the slot of a term names its pair
    pos = np.argwhere(ids >= 0)                               # (m, r, col) per pair
    fn = ids[ids >= 0]
    npair = len(fn)
    sub = np.full_like(ids, -1)
    sub[ids >= 0] = np.arange(npair, dtype=np.int32)
    pair_ids = np.full_like(fwd["faces_id_buffer"], -1)
    pair_ids[0][:, rows] = sub
    pfwd = dict(fwd, faces_id_buffer=pair_ids, faces_info=o["faces_info"][:, fn])
    gs = np.zeros_like(g)
    gs[0][:, rows] = g[0][:, rows]
    st, _ = osr.backward(fv[:, fn], tex[:, fn], pfwd, gs, P, stats=True, terms=True)
    val, slot = st["terms"]
    ngf = npair * 9
    t = slot >= ngf                                           # T == 1: three texture slots per pair
    pair = np.where(t, (slot - ngf) // 3, slot // 9)
    col = np.where(t, 9 + (slot - ngf) % 3, slot % 9)
    terms = np.zeros(ids.shape + (12,), np.float32)
    m, r, c = pos[pair].T
    terms[m, r, c, col] = val
    return ids, terms


def merge(key, v, d):
    """merge_same_face<d>: lanes L and L ^ d holding the same face add into the lower lane (float32)."""
    lane = np.arange(32)
    pk = key[..., lane ^ d]
    same = (pk == key) & (key >= 0)
    lower = (lane & d) == 0
    add = same & lower
    v = np.where(add[..., None], v + v[..., lane ^ d, :], v)
    key = np.where(same & ~lower, -1, key)
    return key, v


def count(ids, terms, silhouette):
    """Replays the warp walk on the sampled row pairs -> (pairs, interleaved, interleaved skipping, zero-class skipping)."""
    K, R, H = ids.shape
    # warps: 8 columns x (row pair) -- each sampled row pair is the lane >> 3 = 0 / 1 half of a warp; the other half
    # (rows 2, 3 of the 4-row warp) is another sampled pair's, which the vertical merge never pairs with these
    nw = H // 8
    key = ids.reshape(K, R // 2, 2, nw, 8).transpose(0, 1, 3, 2, 4).reshape(K, R // 2, nw, 16)
    v = terms.reshape(K, R // 2, 2, nw, 8, 12).transpose(0, 1, 3, 2, 4, 5).reshape(K, R // 2, nw, 16, 12)
    pad = np.full(key.shape[:-1] + (16,), -1, key.dtype)
    key = np.concatenate([key, pad], -1)
    v = np.concatenate([v, np.zeros(v.shape[:-2] + (16, 12), v.dtype)], -2)
    pairs = int((key >= 0).sum())
    key, v = merge(key, v, 1)
    key, v = merge(key, v, 8)
    live = key >= 0
    npk = 2 if silhouette else 3
    nz = v != 0
    res = [pairs, int(live.sum()) * npk]
    for layout in (INTERLEAVED, ZERO_CLASS):
        res.append(sum(int((live & nz[..., q].any(-1)).sum()) for q in layout[:npk]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["c3", "c2", "c5"], choices=sorted(WORKLOADS))
    ap.add_argument("--row-step", type=int, default=16)
    a = ap.parse_args()
    print("| workload | pairs | interleaved, all | interleaved, zero skipped | zero-class, zero skipped | saved vs today |")
    print("|---|---|---|---|---|---|")
    for name in a.workload:
        nf, H, nimg, skw, pkw, gch = WORKLOADS[name]
        fv, tex = wl.make_scene(nf, batch=1, **skw)
        P = osr.Params(image_size=H, **pkw)
        g = np.zeros((1, 4, H, H), np.float32)
        g[:, 4 - gch:] = np.random.default_rng(2).uniform(-1.0, 1.0, (1, gch, H, H)).astype(np.float32)
        rows = [r + d for r in range(0, H, a.row_step) for d in (0, 1)]
        ids, terms = pair_terms(fv, tex, P, g, rows)
        c = count(ids, terms, pkw.get("aggr_func_rgb") == "none")
        scale = H / len(rows) * nimg
        m = lambda x: "%.2f M" % (x * scale / 1e6)   # noqa: E731
        print("| %s | %s | %s | %s | %s | %.1f %% |" % (name, m(c[0]), m(c[1]), m(c[2]), m(c[3]), 100.0 * (1 - c[3] / c[1])),
              flush=True)


if __name__ == "__main__":
    main()
