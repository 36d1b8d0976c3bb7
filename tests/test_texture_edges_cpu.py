"""CPU checks of the texture bake / atlas emulations (oracle/bake.py, oracle/texture_atlas.py) on the cases of
tests/texture_edge_cases.py, which tests/test_texture_edges_gpu.py holds the kernels to bit for bit:
  - every case family reaches the edges it names (clamped taps, saturated and NaN conversions, row wraps, NaN and inf
    texels, degenerate tiles), counted by the emulations themselves;
  - the float32 bake emulations agree with a float64 restatement of the same formulas within its running error bound
    (oracle.numbers.EV), wherever the float32 walk's integer decisions are well conditioned;
  - mutation checks: each subtly wrong emulation (the old float64 weights, floor for truncation, NaN-propagating min /
    max, no clamp at the last pixel, a sum not started from +0.0, wrapping the already-wrapped UV) changes at least one
    output bit on the case set, so the GPU tests would catch a kernel that did the same."""
import numpy as np
import pytest

from oracle import bake as obake
from oracle import numbers
from oracle import texture_atlas as oat
from oracle.numbers import EV
from tests import texture_edge_cases as tec

F = np.float32
SMALL = [c for c in tec.softras_cases() if not c["name"].startswith("softras_large")]
N3MR = tec.n3mr_cases()
ATLAS = tec.atlas_cases()


def _softras(c, stats=None):
    return obake.bake_textures_for_softras(c["image"], c["faces_uv"], c["textures"], c["is_update"], stats)


def _all_outputs():
    out = [_softras(c) for c in SMALL]
    for c in N3MR:
        for wrap in range(4):
            for bil in (True, False):
                out.append(obake.bake_textures_for_n3mr(c["image"], c["faces_uv"], c["textures"], c["is_update"], wrap, bil))
    for c in ATLAS:
        args = (c["tile_vertices"], c["texture_res_out"], c["tile_width"], c["H"], c["W"])
        out.append(oat.texture_atlas_softras(args[0], c["softras"], *args[1:]))
        out.append(oat.texture_atlas_n3mr(args[0], c["n3mr"], *args[1:]))
    return out


def test_case_set_sizes():
    large = [c for c in tec.softras_cases() if c["name"].startswith("softras_large")]
    assert len(large) == 1 and large[0]["textures"].shape[0] * large[0]["textures"].shape[1] > 1 << 24
    assert {c["textures"].shape[1] for c in SMALL} == {r * r for r in tec.SOFTRAS_R}
    assert {c["textures"].shape[1] for c in N3MR} == set(tec.N3MR_TS)
    assert {c["image"].shape[:2] for c in SMALL} >= {(1, 1), (1, 7), (5, 1)}
    assert all((c["is_update"] == 0).any() and (c["is_update"] != 0).any() for c in SMALL + N3MR)
    texels = sum(c["textures"].size // 3 for c in SMALL + N3MR) + sum(c["H"] * c["W"] for c in ATLAS)
    print("\n%d softras, %d n3mr (x 8 modes), %d atlas cases; %d texels / pixels per mode" % (len(SMALL), len(N3MR), len(ATLAS), texels))


def test_softras_cases_reach_their_edges():
    st = {}
    for c in SMALL:
        _softras(c, st)
    print("\n", st)
    for k in ("clamped_taps", "saturated_conversions", "nan_conversions", "row_wraps", "extrapolating_weights",
              "nan_texels", "inf_texels"):
        assert st.get(k, 0) > 0, k
    # per family: negative UVs extrapolate, huge ones saturate, seams wrap rows
    for fam, key in (("negative", "extrapolating_weights"), ("huge", "saturated_conversions"), ("seams", "row_wraps")):
        s = {}
        for c in SMALL:
            if fam in c["name"]:
                _softras(c, s)
        assert s.get(key, 0) > 0, (fam, key)


def test_n3mr_cases_reach_their_edges():
    for wrap in range(3):
        for bil in (True, False):
            st = {}
            for c in N3MR:
                obake.bake_textures_for_n3mr(c["image"], c["faces_uv"], c["textures"], c["is_update"], wrap, bil, st)
            if wrap < 2:
                assert st["nan_uvs_after_wrap"] > 0 and st["nan_texels"] > 0, (wrap, st)   # inf / NaN UVs stay NaN
            else:
                assert st["nan_uvs_after_wrap"] == 0, st                                   # fminf / fmaxf drop the NaN
            if bil:
                assert st["clamped_taps"] > 0, (wrap, st)
            else:
                assert st["rounded_halves"] > 0, (wrap, st)


def test_atlas_cases_reach_their_edges():
    st = {}
    for c in ATLAS:
        oat.tile_weights(c["tile_vertices"], c["texture_res_out"], c["tile_width"], c["H"], c["W"], st)
    print("\n", st)
    assert st["degenerate_tiles"] > 0 and st["nonfinite_weights"] > 0 and st["unused_pixels"] > 0


def test_ref_mod_signed_zero_and_wrap_modes():
    """REPEAT maps -0.0 and 0 to 1 (x > 0 is false for both) and integers > 0 to 0; MIRRORED_REPEAT reflects odd
    intervals; CLAMP_TO_EDGE takes NaN to 1 as fminf does; NaN and +-inf stay NaN under the fmod wraps."""
    v = F([-0.0, 0.0, 1.0, 2.0, -1.0, 0.25, 1.25, -0.25, np.nan, np.inf, -np.inf])
    rep = obake._wrap(v, obake.REPEAT)
    np.testing.assert_array_equal(rep[:8], F([1, 1, 0, 0, 1, 0.25, 0.25, 0.75]))
    assert np.isnan(rep[8:]).all()
    mir = obake._wrap(v, obake.MIRRORED_REPEAT)
    np.testing.assert_array_equal(mir[:8], F([0, 0, 1, 0, 0, 0.25, 0.75, 0.25]))
    np.testing.assert_array_equal(obake._wrap(v, obake.CLAMP_TO_EDGE), F([0, 0, 1, 1, 0, 0.25, 1, 0, 1, 1, 0]))
    assert list(numbers.cuda_int(F([np.nan, np.inf, -np.inf, 3e9, -3e9, -0.5, 2.99]))) == [0, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31, 0, 2]
    assert list(obake._round_half_away(F([0.5, -0.5, 1.5, 2.5, -2.5, 0.49999997]))) == [1, -1, 2, 3, -3, 0]


def _ev_bake(img, uv, R, H, W, ix, iy, iy1):
    """The SoftRas bake restated over EV (float64 value + float32 error bound), at the float32 walk's integer taps."""
    w0, w1, w2 = obake.sample_weights(R)
    f = uv.astype(np.float64)
    pos_x = ((EV(f[:, None, 0, 0]) * w0 + EV(f[:, None, 1, 0]) * w1) + EV(f[:, None, 2, 0]) * w2) * float(W - 1)
    pos_y = ((EV(f[:, None, 0, 1]) * w0 + EV(f[:, None, 1, 1]) * w1) + EV(f[:, None, 2, 1]) * w2) * float(H - 1)
    # pos - (float)(int)pos is exact in float32 below 2^24 (Sterbenz), so the weights carry the positions' error
    wx1 = EV(pos_x.v - ix, pos_x.e + numbers.U64 * np.abs(pos_x.v))
    wy1 = EV(pos_y.v - iy, pos_y.e + numbers.U64 * np.abs(pos_y.v))
    wx0, wy0 = 1.0 - wx1, 1.0 - wy1
    n = H * W
    flat = img.reshape(-1, 3).astype(np.float64)
    idx = [np.clip(j, 0, n - 1) for j in (iy * W + ix, iy1 * W + ix, iy * W + ix + 1, iy1 * W + ix + 1)]
    wts = [wx0 * wy0, wx0 * wy1, wx1 * wy0, wx1 * wy1]
    c = EV(np.zeros(ix.shape + (3,)))
    for j, w in zip(idx, wts):
        c = c + EV(flat[j]) * EV(w.v[..., None], w.e[..., None])
    return c, pos_x, pos_y


def test_softras_emulation_against_float64():
    """At the float32 walk's integer taps, the bake is linear in the positions, so the restatement holds wherever the
    values are finite and |pos| < 2^24 (above that (float)(int)pos rounds, which the emulation models on purpose).
    The members left out are counted."""
    kept = total = 0
    for c in SMALL:
        H, W = c["image"].shape[:2]
        R = int(round(np.sqrt(c["textures"].shape[1])))
        upd = c["is_update"] != 0
        uv = c["faces_uv"][upd]
        got = _softras(c)[upd]
        w0, w1, w2 = obake.sample_weights(R)
        with np.errstate(all="ignore"):
            px = ((uv[:, None, 0, 0] * w0 + uv[:, None, 1, 0] * w1) + uv[:, None, 2, 0] * w2) * F(W - 1)
            py = ((uv[:, None, 0, 1] * w0 + uv[:, None, 1, 1] * w1) + uv[:, None, 2, 1] * w2) * F(H - 1)
            ix, iy, iy1 = numbers.cuda_int(px), numbers.cuda_int(py), numbers.cuda_int(py + F(1))
            ev, pos_x, pos_y = _ev_bake(c["image"], uv, R, H, W, ix, iy, iy1)
            ok = np.isfinite(ev.v).all(-1) & np.isfinite(ev.e).all(-1) & np.isfinite(got).all(-1)
            ok &= (np.abs(px) < 2.0 ** 24) & (np.abs(py) < 2.0 ** 24)
        total += np.isfinite(got).all(-1).sum()
        kept += ok.sum()
        numbers.check_terms(got[ok], ev[ok])
    print("\nsoftras bake vs float64: %d of the %d finite texels within the bound, the rest past 2^24" % (kept, total))
    assert kept > 0.9 * total


# ---------------------------------------------------------------------------------------------- mutation checks

def _floor_int(a):
    a = np.nan_to_num(np.asarray(a, np.float64), nan=0.0, posinf=2147483647.0, neginf=-2147483648.0)
    return np.clip(np.floor(a), -2147483648.0, 2147483647.0).astype(np.int64)


def _double_frac(pos):          # the old oracle: pos - (int64) pos in float64, so every later product is double
    return pos - numbers.cuda_int(pos)


def _read_past_end(flat, idx):  # taps past the last pixel read something else (here zeros) instead of the last pixel
    return np.concatenate([flat, np.zeros((1, 3), F)])[np.minimum(idx, len(flat))]


def _sum_from_first(p):
    return ((p[..., 0, :] + p[..., 1, :]) + p[..., 2, :]) + p[..., 3, :]


MUTANTS = {
    "double_weights": [(obake, "_frac", _double_frac)],
    "floor_for_truncation": [(obake, "cuda_int", _floor_int), (oat, "cuda_int", _floor_int)],
    "nan_propagating_min_max": [(obake, "fminf", np.minimum), (obake, "fmaxf", np.maximum),
                                (oat, "fminf", np.minimum), (oat, "fmaxf", np.maximum)],
    "no_clamp_at_last_pixel": [(obake, "_clamp_index", lambda j, n: np.maximum(j, 0)), (obake, "_gather", _read_past_end)],
    "sum_without_zero_start": [(obake, "_sum4", _sum_from_first)],
    "wrap_the_wrapped_uv": [(obake, "_wrap", lambda v, mode, w=obake._wrap: w(w(v, mode), mode))],
}


@pytest.fixture(scope="module")
def reference_outputs():
    return _all_outputs()


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutant_changes_an_output_bit(name, monkeypatch, reference_outputs):
    for mod, attr, fn in MUTANTS[name]:
        monkeypatch.setattr(mod, attr, fn)
    changed = 0
    for ref, got in zip(reference_outputs, _all_outputs()):
        got = np.asarray(got, F)
        changed += int(((got.view(np.uint32) != ref.view(np.uint32)) & ~(np.isnan(got) & np.isnan(ref))).sum())
    print("\n%s: %d output values change" % (name, changed))
    assert changed > 0, name
