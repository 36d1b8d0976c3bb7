"""The SoftRas backward's per-entry bound (oracle.softras.backward_bound) and the scenes of softras_backward_cases.py,
without a GPU: each scene reaches the kernel paths it is built for, the bound holds for every summation order and every
rounding the kernel is allowed, it is far tighter than the per-tensor tolerance it replaces, and the oracle's older
entry points still compute what they did before the per-pair body was shared with the statistics entry point."""
import hashlib
import os

import numpy as np
import pytest

from jrender_b200 import workloads as wl
from oracle import softras as osr
from tests import softras_backward_cases as SC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "softras_oracle_entry_points.npz")

# scenes of the entry-point digests: (make_scene kwargs, Params kwargs); upstream gradient seeded by the index
ENTRY_SCENES = [
    (dict(num_faces=280, batch=1), dict(image_size=24, sigma_val=3e-5)),
    (dict(num_faces=280, batch=2), dict(image_size=20, dist_func="barycentric", aggr_func_alpha="sum", sigma_val=1e-4)),
    (dict(num_faces=280, batch=1), dict(image_size=20, dist_func="hard", aggr_func_rgb="hard", aggr_func_alpha="hard")),
    (dict(num_faces=280, batch=1, texture_type="vertex"), dict(image_size=20, texture_type="vertex",
                                                                max_faces_per_pixel_for_grad=4)),
    (dict(num_faces=280, batch=1, texture_res=3), dict(image_size=20, aggr_func_rgb="hard", sigma_val=1e-3)),
    (dict(num_faces=280, batch=1, texture_res=3), dict(image_size=20, fill_back=False, sigma_val=1e-3, gamma_val=1e-3)),
]


def entry_point_outputs():
    res = {}
    for i, (sk, pk) in enumerate(ENTRY_SCENES):
        fv, tex = wl.make_scene(**sk)
        P = osr.Params(**pk)
        H = P["image_size"]
        g = np.random.default_rng(i).uniform(-1, 1, (fv.shape[0], 4, H, H)).astype(np.float32)
        f = osr.forward(fv, tex, P)
        for k, v in f.items():
            res["%d_%s" % (i, k)] = v
        for acc in (0, 1):
            res["%d_gf%d" % (i, acc)], res["%d_gt%d" % (i, acc)] = osr.backward(fv, tex, f, g, P, accumulate_double=acc)
    return res


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def test_old_entry_points_are_bit_identical():
    """softras_oracle_forward / _backward (both accumulation modes) hash to the bytes the oracle produced before its
    backward got the shared per-pair body (digests in tests/golden/softras_oracle_entry_points.npz)."""
    z = np.load(GOLDEN)
    got = entry_point_outputs()
    assert sorted(z.files) == sorted(got)
    bad = [k for k in z.files if not np.array_equal(z[k], digest(got[k]))]
    assert not bad, bad


@pytest.mark.parametrize("i", range(len(ENTRY_SCENES)))
def test_stats_sum_is_the_double_accumulation(i):
    sk, pk = ENTRY_SCENES[i]
    fv, tex = wl.make_scene(**sk)
    P = osr.Params(**pk)
    H = P["image_size"]
    g = np.random.default_rng(i).uniform(-1, 1, (fv.shape[0], 4, H, H)).astype(np.float32)
    f = osr.forward(fv, tex, P)
    gf, gt = osr.backward(fv, tex, f, g, P)
    sf, st = osr.backward(fv, tex, f, g, P, stats=True)
    assert np.array_equal(gf, sf["g64"].astype(np.float32), equal_nan=True)
    assert np.array_equal(gt, st["g64"].astype(np.float32), equal_nan=True)
    for s in (sf, st):
        fin = np.isfinite(s["g64"])
        assert np.all(s["A"][fin] >= np.abs(s["g64"][fin]) * (1 - 1e-12)) and np.all((s["N"] == 0) <= (s["A"] == 0))


# ---------------------------------------------------------------- each case reaches its target

@pytest.fixture(scope="module")
def oracle_runs():
    out = {}
    for name, fv, tex, P, g in SC.cases():
        f = osr.forward(fv, tex, P)
        out[name] = (fv, tex, P, g, f, osr.backward(fv, tex, f, g, P, stats=True, terms=True))
    return out


def lane_pairs(ids, D):
    """kinds of (lane, lane ^ D) key pairs at every slot, over the kernel's 8 x 4 warps: 'same', 'diff', 'one_empty'"""
    B, K, H, W = ids.shape
    pad = np.full((B, K, (H + 3) // 4 * 4, (W + 7) // 8 * 8), -1, np.int64)
    pad[:, :, :H, :W] = ids
    if D == 1:
        a, b = pad[..., 0::2], pad[..., 1::2]
    else:
        w = pad.reshape(B, K, -1, 4, pad.shape[-1])
        a, b = w[:, :, :, 0::2], w[:, :, :, 1::2]   # lane ^ 8 pairs rows 0|1 and 2|3 of a warp
    kinds = set()
    if np.any((a == b) & (a >= 0)):
        kinds.add("same")
    if np.any((a != b) & (a >= 0) & (b >= 0)):
        kinds.add("diff")
    if np.any((a >= 0) != (b >= 0)):
        kinds.add("one_empty")
    return kinds


def test_warp_geometry_cases_see_every_merge_combination(oracle_runs):
    for H in SC.WARP_SIZES:
        ids = oracle_runs["merge_H%d" % H][4]["faces_id_buffer"]
        cnt = (ids >= 0).sum(1)
        assert cnt.min() >= 1
        if H >= 9:
            for D in (1, 8):
                assert lane_pairs(ids, D) == {"same", "diff", "one_empty"}, (H, D)
            # the boundaries are drawn between columns 0|1, 7|8 and rows 3|4
            assert np.any(cnt[:, :, 0] != cnt[:, :, 1]) and np.any(cnt[:, :, 7] != cnt[:, :, 8])
            assert np.any(cnt[:, 3] != cnt[:, 4])
    ck = oracle_runs["checkerboard"][4]["faces_id_buffer"]
    assert lane_pairs(ck, 1) == {"diff"} and lane_pairs(ck, 8) == {"diff"}
    fw = oracle_runs["full_warp"][4]["faces_id_buffer"]
    assert lane_pairs(fw, 1) == {"same"} and lane_pairs(fw, 8) == {"same"}
    dup = oracle_runs["full_warp_duplicate"]
    assert np.array_equal(dup[0][0, 0], dup[0][0, 1])
    ids = dup[4]["faces_id_buffer"]
    assert np.all(ids[:, 0] == 0) and np.all(ids[:, 1] == 1)
    sf = dup[5][0]
    assert np.array_equal(sf["g64"][0, 0], sf["g64"][0, 1]) and np.abs(sf["g64"]).max() > 0   # same terms, two slots


def test_list_length_cases_end_at_every_slot(oracle_runs):
    for K in SC.LIST_KS:
        ids = oracle_runs["stack_K%d" % K][4]["faces_id_buffer"]
        cnt = (ids >= 0).sum(1)[0]
        assert set(range(K + 1)) <= set(np.unique(cnt).tolist()), K   # lists end at every m, and full lists occur
        H = cnt.shape[0]
        warps = np.full(((H + 3) // 4 * 4, (H + 7) // 8 * 8), 0)
        warps[:H, :H] = cnt
        w = warps.reshape(warps.shape[0] // 4, 4, warps.shape[1] // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 32)
        nonempty = (w > 0).sum(1)
        assert np.any(nonempty == 1), K                                   # a warp with one non-empty lane
        if K > 1:
            assert np.any([len(set(r[r > 0].tolist())) >= min(3, K) for r in w]), K   # lanes ending at different m


def clipped_w(f, fv, H):
    """the backward's clipped barycentric weights of every (pixel, slot) pair, float32 as the oracle computes them"""
    ids = f["faces_id_buffer"][0]
    K = ids.shape[0]
    r, c = np.meshgrid(np.arange(H), np.arange(H), indexing="ij")
    xp = ((2.0 * c + 1 - H) / H).astype(np.float32)
    yp = ((2.0 * (H - 1 - r) + 1 - H) / H).astype(np.float32)
    out = []
    for m in range(K):
        sel = ids[m] >= 0
        inv = f["faces_info"][0][ids[m][sel]][:, :9]
        x, y = xp[sel], yp[sel]
        w = np.stack([inv[:, 3 * k] * x + inv[:, 3 * k + 1] * y + inv[:, 3 * k + 2] for k in range(3)], 1)
        wc = np.clip(w, np.float32(0), np.float32(1))
        s = np.maximum(wc.sum(1, dtype=np.float32), np.float32(1e-5))
        out.append((w, wc / s[:, None]))
    return out


def test_texel_cases_hit_texel_boundaries(oracle_runs):
    for R in (2, 3, 5):
        fv, tex, P, g, f, (sf, st) = oracle_runs["texel_R%d_softmax" % R]
        hit = 0
        for _, wc in clipped_w(f, fv, 32):
            x = wc[:, :2] * np.float32(R)
            hit += int(np.sum((x == np.round(x)) & (wc[:, :2] > 0) & (wc[:, :2] < 1)))
        if R in (2, 4):
            assert hit >= 20, (R, hit)
        used = (st["N"][0] > 0).any(-1)
        assert used.sum(1).max() == R * R or R == 5      # every texel of some face gets a term
    assert oracle_runs["texel_R1_softmax"][5][1]["N"].max() > 0


def test_prod_floor_and_threshold_pairs_occur(oracle_runs):
    """pairs with 1 - D below the alpha-prod floor 1e-6, zero and non-zero, and pairs out towards the distance
    threshold"""
    fv, tex, P, g, f, _ = oracle_runs["mode_barycentric_softmax_prod"]
    sigma = np.float32(P["sigma_val"])
    omd = []
    for w, _ in clipped_w(f, fv, P["image_size"]):
        dis = np.min(w, 1)
        dis = np.where(dis > 0, dis * dis, -dis * dis).astype(np.float32)
        D = (1.0 / (1.0 + np.exp(-(dis / sigma).astype(np.float64)).astype(np.float32))).astype(np.float32)
        omd.append(np.float32(1) - D)
    omd = np.concatenate(omd)
    assert np.sum(omd == 0) > 10 and np.sum((omd > 0) & (omd < 1e-6)) > 0
    assert np.sum(omd > 0.99) > 0     # D < 1e-2: out towards the distance threshold, where D = dist_eps


def test_batch_case_has_an_empty_element(oracle_runs):
    fv, tex, P, g, f, (sf, st) = oracle_runs["batch3_odd_nf_empty"]
    assert fv.shape[:2] == (3, 101)
    ids = f["faces_id_buffer"]
    assert (ids[0] >= 0).any() and (ids[1] >= 0).any() and not (ids[2] >= 0).any()
    assert not np.array_equal(ids[0], ids[1])
    assert np.all(sf["N"][2] == 0) and np.all(sf["N"][:2].sum((1, 2, 3)) > 0)


# ---------------------------------------------------------------- the bound is not too tight

BOUND_CASES = ["merge_H33", "merge_H100", "full_warp_duplicate", "stack_K64", "texel_R3_softmax", "vertex_softmax",
               "mode_barycentric_softmax_prod", "mode_euclidean_softmax_sum", "batch3_odd_nf_empty"]


def within(got_f, got_t, stats):
    for got, st in zip((got_f, got_t), stats):
        m = np.isfinite(st["g64"])
        err = np.abs(got.astype(np.float64)[m] - st["g64"][m])
        assert np.all(err <= osr.backward_bound(st)[m]), (err / np.maximum(osr.backward_bound(st)[m], 1e-300)).max()


@pytest.mark.parametrize("name", BOUND_CASES)
def test_bound_holds_for_serial_float_accumulation(oracle_runs, name):
    fv, tex, P, g, f, stats = oracle_runs[name]
    within(*osr.backward(fv, tex, f, g, P, accumulate_double=False), stats)


@pytest.mark.parametrize("name", BOUND_CASES)
def test_bound_holds_for_float_sums_in_shuffled_order(oracle_runs, name):
    fv, tex, P, g, f, (sf, st) = oracle_runs[name]
    val, slot = sf["terms"]
    ngf = sf["g64"].size
    for seed in range(3):
        p = np.random.default_rng(seed).permutation(len(val))
        acc = np.zeros(ngf + st["g64"].size, np.float32)
        np.add.at(acc, slot[p], val[p])          # unbuffered: one float32 addition per term, in the shuffled order
        within(acc[:ngf].reshape(sf["g64"].shape), acc[ngf:].reshape(st["g64"].shape), (sf, st))


@pytest.mark.parametrize("exact_tail", [False, True])
@pytest.mark.parametrize("name", BOUND_CASES)
def test_bound_holds_with_every_rounding_site_moved_by_its_budget(oracle_runs, name, exact_tail):
    fv, tex, P, g, f, _ = oracle_runs[name]
    stats = osr.backward(fv, tex, f, g, P, stats=True, exact_tail=exact_tail)
    for nudge in (1, -1, 2):
        mf, mt = osr.backward(fv, tex, f, g, P, stats=True, exact_tail=exact_tail, nudge=nudge)
        within(mf["g64"].astype(np.float32), mt["g64"].astype(np.float32), stats)
        if not exact_tail:
            assert not np.array_equal(mf["g64"], stats[0]["g64"])   # the moves reach the sum


# ---------------------------------------------------------------- the bound is not vacuous

def test_bound_is_far_below_the_per_tensor_tolerance(oracle_runs):
    """Against the 2e-5 * max|g| per tensor it replaces: on the suite's own kind of scene (the 280-face sphere in every
    mode) the median entry's bound is below 1e-5 of |g|, and for 90 % of the entries it is a tenth of the old
    tolerance or less."""
    ratios, rel = [], []
    for name, (fv, tex, P, g, f, stats) in oracle_runs.items():
        if not name.startswith(("mode_", "texel_", "vertex_")):
            continue
        for st in stats:
            m = (st["g64"] != 0) & np.isfinite(st["g64"])
            if not m.any():
                continue
            b = osr.backward_bound(st)[m]
            old = 2e-5 * np.abs(st["g64"][m]).max()
            ratios.append(b / old)
            rel.append(b / np.abs(st["g64"][m]))
    ratios, rel = np.concatenate(ratios), np.concatenate(rel)
    assert np.median(rel) < 1e-5, np.median(rel)
    assert np.mean(ratios <= 0.1) >= 0.9, np.mean(ratios <= 0.1)
