"""ctypes binding of libb200raster.so.

include/b200raster.h is the only statement of the C ABI: lib() binds every `B200R_API` declaration's argument and return
types from it, and call() is the one path through which the package launches work.

The product path has no CPU fallback: if the library is missing or a call fails, an
exception is raised.  The library is never built implicitly at import time on a GPU box --
`__graft_entry__.build()` / `python -m jrender_b200.build` produce it in-tree.
"""
import ctypes as C
import os
import re

import numpy as np
import torch

from . import build as _build

HEADER = os.path.join(_build.HERE, "..", "include", "b200raster.h")

_lib = None


class B200RasterError(RuntimeError):
    pass


# C type -> ctypes type for the non-pointer types the header uses.  Every pointer is c_void_p (tensors pass their
# data_ptr(), host arrays a ctypes array or byref), except `const char*`, which is c_char_p (bytes in, bytes out).
_SCALARS = {"int": C.c_int, "float": C.c_float, "size_t": C.c_size_t, "unsigned long long": C.c_ulonglong,
            "void": None}


def _ctype(decl, where):
    t = " ".join(decl.replace("*", " * ").split())
    if t.endswith("*"):
        return C.c_char_p if t == "const char *" else C.c_void_p
    t = " ".join(w for w in t.split() if w != "const")
    if t not in _SCALARS:
        raise B200RasterError("%s: no ctypes binding for the C type %r" % (where, decl.strip()))
    return _SCALARS[t]


def parse_header(text):
    """{name: (restype, argtypes)} of every B200R_API declaration in the C header source `text`.  Parameters must be
    named.  A type that is neither a pointer nor in _SCALARS, or a declaration of another shape, raises
    B200RasterError: nothing in the header is left unbound or bound by guess."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)   # comments
    text = re.sub(r"^\s*#.*$", " ", text, flags=re.M)              # preprocessor lines, incl. B200R_API's own #define
    sigs = {}
    for ret, name, params in re.findall(r"\bB200R_API\s+([^;(]+?)\s*\b(b200r_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [] if params.strip() in ("", "void") else params.split(",")
        sigs[name] = (_ctype(ret, name), [_ctype(re.sub(r"\w+\s*$", "", p), name) for p in params])
    n = len(re.findall(r"\bB200R_API\b", text))
    if len(sigs) != n:
        raise B200RasterError("%d B200R_API declarations, only %d of them understood" % (n, len(sigs)))
    return sigs


def lib():
    """Load (once) and return the C ABI library; raises B200RasterError when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if not os.path.exists(path):
        raise B200RasterError(
            "libb200raster.so not built (%s). Run `python -m jrender_b200.build` "
            "(needs nvcc); there is no CPU fallback." % path)
    L = C.CDLL(path)
    with open(HEADER) as f:
        sigs = parse_header(f.read())
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        raise B200RasterError("%s failed (rc=%d): %s" % (what, rc, lib().b200r_last_error().decode()))


def call(name, device, *args):
    """Runs the entry point `name` on `device` (the library launches on the current device) and its current stream,
    which is appended to `args`.  Tensors pass their data_ptr(), None passes NULL; a non-zero return raises
    B200RasterError naming `name`."""
    fn = getattr(lib(), name)
    with torch.cuda.device(device):
        rc = fn(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args],
                torch.cuda.current_stream(device).cuda_stream)
    check(rc, name)


def _f3(x):
    """Three host floats as a ctypes array, for the C ABI's host `const float*` vectors (light colours and direction,
    camera `at` / `up`, background colour); x is a list, tuple, numpy array or a tensor on any device."""
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().tolist()
    a = np.asarray(x, dtype=np.float32).reshape(-1)
    if a.shape[0] != 3:
        raise ValueError("expected 3 components, got %r" % (x,))
    return (C.c_float * 3)(*a.tolist())


def set_option(name, value):
    check(lib().b200r_set_option(name.encode(), int(value)), "b200r_set_option(%s)" % name)
