"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every
symbol include/b200raster.h declares; argument validation fails loudly; no CPU fallback."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200raster.h")).read()
    return sorted(set(re.findall(r"B200R_API\s+[\w\s\*]+?\b(b200r_\w+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from jrender_b200 import build, _lib
    build.build()          # nvcc cross-compiles sm_90a without a GPU
    return _lib.lib()


def test_header_declares_entry_points():
    syms = declared_symbols()
    for s in ["b200r_softras_forward", "b200r_softras_backward", "b200r_softras_workspace_bytes", "b200r_softras_state_bytes",
              "b200r_softras_forward_aa", "b200r_softras_backward_aa", "b200r_surface_lighting_forward", "b200r_bake_textures_softras", "b200r_bake_textures_n3mr",
              "b200r_last_error", "b200r_launch_count", "b200r_profile_read"]:
        assert s in syms


def test_library_exports_every_declared_symbol(lib):
    for s in declared_symbols():
        assert hasattr(lib, s), "libb200raster.so does not export %s" % s


def test_version_and_workspace_size(lib):
    assert b"sm_90a" in lib.b200r_version()
    assert lib.b200r_softras_workspace_bytes(0, 10, 64) == 0
    small = lib.b200r_softras_workspace_bytes(1, 100, 64)
    big = lib.b200r_softras_workspace_bytes(4, 39200, 1024)
    assert 0 < small < big
    assert big >= 4 * 39200 * 8                       # rects (8 B) per face are the floor of the binning scratch
    # what the backward keeps: 160-byte records + 48-byte accumulator rows, independent of the image size
    st = lib.b200r_softras_state_bytes(4, 39200)
    assert 4 * 39200 * 208 <= st <= 4 * 39200 * 208 + 1024 and lib.b200r_softras_state_bytes(0, 5) == 0


def test_argument_validation_is_loud(lib):
    from jrender_b200 import _lib
    null = C.c_void_p(0)
    args_tail = (1.0, 100.0, 1e-3, 1e-5, 1e-4, 9.21, 2, 1, 2, 0, 1, null)
    # K > 64 violates the reference hard limit kMaxPointsPerPixel (cuda/soft_rasterize.py:16)
    rc = lib.b200r_softras_forward(null, null, null, null, null, null, null, 0, null, 0, 1, 10, 1, 64, 65, *args_tail)
    assert rc == -1 and b"max_faces_per_pixel" in lib.b200r_last_error()
    rc = lib.b200r_softras_forward(null, null, null, null, null, null, null, 0, null, 0, 1, 10, 1, 64, 16, *args_tail)
    assert rc == -1 and b"NULL" in lib.b200r_last_error()
    rc = lib.b200r_softras_forward(null, null, null, null, null, null, null, 0, null, 0, 1, 10, 2, 64, 16, *args_tail)
    assert rc == -1 and b"square" in lib.b200r_last_error()
    with pytest.raises(_lib.B200RasterError):
        _lib.check(rc, "b200r_softras_forward")


def test_no_cpu_fallback():
    """CPU tensors are rejected: the product path never routes through the oracle or torch ops."""
    import torch
    from jrender_b200 import B200RasterError, soft_rasterize
    fv = torch.zeros(1, 4, 3, 3)
    tex = torch.zeros(1, 4, 1, 3)
    with pytest.raises(B200RasterError):
        soft_rasterize(fv, tex, image_size=16)


def test_reference_signature_defaults():
    """Same constructor defaults as the reference (soft_rasterize.py:10-16, rasterizer.py:9-15)."""
    from jrender_b200 import SoftRasterizeFunction, SoftRasterizer
    f = SoftRasterizeFunction()
    assert (f.image_size, f.near, f.far, f.eps, f.sigma_val, f.gamma_val) == (256, 1, 100, 1e-3, 1e-5, 1e-4)
    assert (f.dist_func, f.aggr_func_rgb, f.aggr_func_alpha, f.aggr_texture_type, f.max_faces_id) == \
        ("euclidean", "softmax", "prod", "surface", 16)
    assert abs(f.dist_eps - np.log(1.0 / 1e-4 - 1.0)) < 1e-12 and f.fill_back is True
    r = SoftRasterizer()
    assert r.fill_back is False and r.anti_aliasing is False
    with pytest.raises(ValueError):
        SoftRasterizer(dist_func="manhattan")
    with pytest.raises(ValueError):
        SoftRasterizer(aggr_func_rgb="none")
