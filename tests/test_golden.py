"""Pins the CPU oracle to the REAL reference: tests/golden/ref_gpu_*.npz hold outputs of the
reference's own kernel strings (jrender/renderer/dr/softras/cuda/soft_rasterize.py), compiled
by oracle/build_ref.py and run on a GPU by oracle/make_ref_golden.py.  Each file records the GPU and
nvcc flags it was made with in its `provenance` entry: the stored fixtures were made with an sm_100a
build on a B200; regenerated ones (the recipe now builds for sm_90a) record an H100.

The reference build contracts a*b+c into FMAs where nvcc chooses (nvcc defaults), the oracle
and the product never do, and depth enters the colour softmax as exp((z-max)/1e-4): a 1-ulp
difference in z moves a softmax weight by ~6e-4.  Tolerances are therefore statistical
(thresholds ~4x above the measured values):
  * top-K id sets equal on >= 99.8 % of pixels (100 % on all fixtures but the sub-pixel mesh);
  * soft_colors: max |diff| <= 2e-3 (sub-pixel-triangle fixture: <= 2 % of pixels above 2e-3);
  * gradients: sum|diff| / sum|ref| <= 2e-3 (sub-pixel fixture: 5e-2);
  * faces_info (K1): relative 1e-5 (sub-pixel fixture 5e-3: near-degenerate determinants).
"""
import glob
import json
import os

import numpy as np
import pytest

from oracle import softras as osr
from tests.conftest import ROOT

ALL = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ref_gpu_*.npz")))
FILES = [p for p in ALL if "ref_gpu_nmr_" not in p and "ref_gpu_bake_" not in p]        # SoftRas fixtures
NMR_FILES = [p for p in ALL if "ref_gpu_nmr_" in p]        # NMR (dr_type='n3mr') fixtures


def rel_l1(ref, got):
    m = np.isfinite(ref) & np.isfinite(got)
    return float(np.abs(ref[m] - got[m]).sum() / max(np.abs(ref[m]).sum(), 1e-30))


def test_golden_files_present():
    assert len(FILES) >= 8
    prov = json.loads(str(np.load(FILES[0])["provenance"]))
    assert any(g in prov["gpu"] for g in ("B200", "H100")) and "soft_rasterize.py" in prov["source"]


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(p)[8:-4] for p in FILES])
def test_oracle_matches_reference_kernels(path):
    z = np.load(path)
    P = osr.Params(**json.loads(str(z["params"])))
    fv, tex, g = z["face_vertices"], z["textures"], z["grad_soft_colors"]
    cpu = osr.forward(fv, tex, P)
    gf, gt = osr.backward(fv, tex, cpu, g, P)
    subpixel = "3280" in path          # triangles smaller than a pixel: decisions flip with FMA contraction
    ids_ref = z["faces_id_buffer"].astype(np.int32)
    same = (np.sort(ids_ref, 1) == np.sort(cpu["faces_id_buffer"], 1)).all(1).mean()
    assert same >= (0.998 if subpixel else 1.0), same
    d = np.abs(z["soft_colors"] - cpu["soft_colors"]).max(1)
    if subpixel:
        assert (d > 2e-3).mean() <= 0.02 and d.mean() <= 2e-3
    else:
        assert d.max() <= 2e-3, d.max()
    fi_rel = np.abs(z["faces_info"] - cpu["faces_info"]).max() / np.abs(cpu["faces_info"]).max()
    assert fi_rel <= (5e-3 if subpixel else 1e-5)
    assert rel_l1(z["grad_faces"], gf) <= (5e-2 if subpixel else 2e-3)
    T = tex.shape[2]
    if P["texture_type"] == "surface" and T > 1:
        # Reference UB (SURVEY.md Q9): backward_sample_texture returns an uninitialised value for
        # non-hit texels; the nvcc-12.9 build materialises it as "every texel receives the hit
        # texel's gradient".  The oracle defines non-hit texels as 0, so the reference's value at
        # EVERY texel must equal the oracle's per-face total.
        ref_gt = z["grad_textures"]
        assert np.abs(ref_gt - ref_gt[:, :, :1]).max() <= 1e-5 * np.abs(ref_gt).max()   # atomic order only
        assert rel_l1(ref_gt[:, :, 0], gt.sum(2)) <= 2e-3
    else:
        assert rel_l1(z["grad_textures"], gt) <= (5e-2 if subpixel else 2e-3)


# --------------------------------------------------------------------------- NMR (dr_type='n3mr')
# tests/golden/ref_gpu_nmr_*.npz: outputs of the reference's K7-K11 kernel strings
# (jrender/renderer/dr/n3mr/cuda/rasterize.py) compiled by oracle/build_ref.py and run on a GPU (the
# `provenance` entry names it) through oracle/ref_gpu.nmr_run (host semantics of n3mr.py:29-123).  Measured
# differences (the report oracle/make_ref_golden.py writes; FMA contraction in the reference build only): face_index_map
# identical on every pixel of every fixture; weight / rgb / sampling weights <= 5e-5 (9e-4 on the
# sub-pixel mesh), depth <= 3e-5, face_inv <= 9e-4 of values up to 146, grad_faces <= 2.6e-4 of max,
# grad_textures <= 5e-5.  Thresholds are ~4x those.
def test_nmr_golden_files_present():
    assert len(NMR_FILES) >= 4
    prov = json.loads(str(np.load(NMR_FILES[0])["provenance"]))
    assert any(g in prov["gpu"] for g in ("B200", "H100")) and "n3mr/cuda/rasterize.py" in prov["source"]


@pytest.mark.parametrize("path", NMR_FILES, ids=[os.path.basename(p)[12:-4] for p in NMR_FILES])
def test_nmr_oracle_matches_reference_kernels(path):
    from oracle import nmr as onmr
    z = np.load(path)
    kw = json.loads(str(z["params"]))
    faces, tex = z["faces"], z["textures"]
    flags = (kw["return_rgb"], kw["return_alpha"], kw["return_depth"])
    H = kw["image_size"]
    cpu = onmr.forward(faces, tex if flags[0] else None, **kw)
    gf, gt = onmr.backward(faces, tex if flags[0] else None, cpu, H, kw["eps"], z["grad_rgb_map"], z["grad_alpha_map"],
                           z["grad_depth_map"], *flags)
    subpixel = "3280" in path
    assert np.array_equal(z["face_index_map"].astype(np.int32), cpu["face_index_map"])     # every pixel, every fixture
    assert np.abs(z["weight_map"] - cpu["weight_map"]).max() <= (4e-3 if subpixel else 2e-4)
    assert np.abs(z["depth_map"] - cpu["depth_map"]).max() <= 1.2e-4
    if flags[0]:
        assert np.array_equal(z["sampling_index_map"], cpu["sampling_index_map"])
        assert np.abs(z["sampling_weight_map"] - cpu["sampling_weight_map"]).max() <= 2e-4
        assert np.abs(z["rgb_map"] - cpu["rgb_map"]).max() <= 1.2e-4
        assert np.abs(z["grad_textures"] - gt).max() <= 2e-4 * max(1.0, float(np.abs(gt).max()))
    if flags[2]:
        ref_inv = z["face_inv_map"].reshape(cpu["face_inv_map"].shape)
        assert np.abs(ref_inv - cpu["face_inv_map"]).max() <= 4e-5 * np.abs(cpu["face_inv_map"]).max()
    assert np.abs(z["grad_faces"] - gf).max() <= 1e-3 * np.abs(gf).max()


def test_bake_oracle_matches_reference_kernel_golden():
    """oracle/bake.py against the reference's own load_textures_cuda_kernel (io/utils/load_textures.py:3-101) compiled by
    oracle/build_ref.py and run on a GPU (oracle/make_ref_golden.py --bake-only).  The reference build contracts a*b+c."""
    from oracle import bake as obake
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_gpu_bake_random40_R5.npz"))
    out = obake.bake_textures_for_softras(g["image"], g["faces_uv"], g["textures_in"], g["is_update"])
    assert np.abs(out - g["textures"]).max() <= 1e-5
    assert np.array_equal(out[g["is_update"] == 0], g["textures_in"][g["is_update"] == 0])


def test_n3mr_bake_oracle_matches_reference_kernel_golden():
    """oracle/bake.py:bake_textures_for_n3mr against the reference's own kernel (io/utils/load_textures.py:103-246, one build
    per wrapping mode / sampling flavour, oracle/build_ref.py) run on a GPU (oracle/make_ref_golden.py --bake-only).
    Bilinear: 1e-5 (the reference build contracts a*b+c).  Nearest: the same texel except where the sample point lies
    within that rounding of a texel boundary (<= 0.2 % of the texels)."""
    import glob
    from oracle import bake as obake
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ref_gpu_bake_n3mr_*.npz")))
    assert len(files) >= 5
    for p in files:
        g = np.load(p)
        out = obake.bake_textures_for_n3mr(g["image"], g["faces_uv"], g["textures_in"], g["is_update"], int(g["texture_wrapping"]),
                                           bool(int(g["use_bilinear"])))
        d = np.abs(out - g["textures"]).max(axis=-1)
        if int(g["use_bilinear"]):
            assert d.max() <= 1e-5, p
        else:
            assert (d > 1e-5).mean() <= 2e-3, p
        assert np.array_equal(out[g["is_update"] == 0], g["textures_in"][g["is_update"] == 0])
