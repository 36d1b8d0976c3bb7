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


def declared_arg_counts():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200raster.h")).read(), flags=re.S)
    return {name: 0 if params.strip() in ("", "void") else params.count(",") + 1
            for name, params in re.findall(r"B200R_API\s+[\w\s\*]+?\b(b200r_\w+)\s*\(([^)]*)\)", src)}


def test_every_declaration_is_bound_from_the_header(lib):
    counts = declared_arg_counts()
    assert sorted(counts) == declared_symbols() and len(counts) >= 31
    for name, n in counts.items():
        argtypes = getattr(lib, name).argtypes
        assert argtypes is not None and len(argtypes) == n, (name, argtypes, n)


def test_bindings_match_the_c_types(lib):
    P, I, F, Z = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    want = {
        "b200r_voxelize_fill": (I, [P, P, Z, I, I, P]),
        "b200r_nmr_backward": (I, [P] * 15 + [Z, I, I, I, I, F, I, I, I, P]),
        "b200r_softras_workspace_bytes": (Z, [I, I, I]),
        "b200r_profile_enable": (None, [I]),
        "b200r_profile_read": (I, [I, P, P]),
        "b200r_version": (C.c_char_p, []),
        "b200r_launch_count": (C.c_ulonglong, []),
        "b200r_set_option": (I, [C.c_char_p, I]),
    }
    for name, (restype, argtypes) in want.items():
        fn = getattr(lib, name)
        assert (fn.restype, fn.argtypes) == (restype, argtypes), name


def test_every_kernel_launch_goes_through_the_launcher():
    """b200r_launch (csrc/api_util.cuh) is the only place that launches a kernel, times it, counts it and checks the
    launch; a translation unit that launched on its own would drift from b200r_launch_count and the profiler."""
    csrc = os.path.join(ROOT, "jrender_b200", "csrc")
    sources = [f for f in sorted(os.listdir(csrc)) if f.endswith((".cu", ".cuh")) and not f.startswith("api_util.")]
    assert "softras_api.cu" in sources and "nmr_kernels.cuh" in sources
    for f in sources:
        src = open(os.path.join(csrc, f)).read()
        for token in ("<<<", "cudaGetLastError", "B200rProfScope", "b200r_count_launch", "b200r_prof_begin", "b200r_prof_end"):
            assert token not in src, "%s: %s" % (f, token)


def test_retired_scheduling_option_is_unknown(lib):
    """The forward always runs the persistent grid over the cost-ordered block queue; there is no option to turn it off."""
    assert lib.b200r_set_option(b"softras_fwd_persistent", 0) == -1
    assert b"unknown option" in lib.b200r_last_error()


def test_header_parser_rejects_what_it_cannot_bind():
    from jrender_b200 import _lib
    sigs = _lib.parse_header("/* B200R_API int b200r_commented(double x); */\n#define B200R_API\n"
                             "B200R_API const char* b200r_a(void);\n"
                             "B200R_API void b200r_b(const float* p, const int32_t* q, unsigned long long n, void* s);\n")
    assert sigs == {"b200r_a": (C.c_char_p, []),
                    "b200r_b": (None, [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p])}
    for bad in ("B200R_API int b200r_x(double d, void* stream);",      # unknown argument type
                "B200R_API double b200r_x(int n);",                    # unknown return type
                "B200R_API int b200r_x(int (*cb)(int), void* stream);"):   # a declaration the parser cannot read
        with pytest.raises(_lib.B200RasterError):
            _lib.parse_header(bad)


@pytest.mark.gpu
def test_failing_call_names_the_entry_point(cuda_device):
    """The anti-aliased forward rejects an odd supersampled size; the error names the function that was called."""
    import torch
    from jrender_b200 import B200RasterError, SoftRasterizeFunction
    fn = SoftRasterizeFunction(image_size=65)
    fn.pool2x2 = True
    fv = torch.rand(1, 8, 3, 3, device=cuda_device)
    tex = torch.rand(1, 8, 1, 3, device=cuda_device)
    with pytest.raises(B200RasterError) as e:
        fn(fv, tex)
    assert str(e.value).startswith("b200r_softras_forward_aa failed"), str(e.value)


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
