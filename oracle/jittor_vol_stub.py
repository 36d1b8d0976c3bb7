"""The rest of the numpy `jittor` stand-in that the reference's jrender_vol package needs (TEST INFRASTRUCTURE -- never
imported by the product).  install() installs oracle/jittor_numpy_stub.py and adds to it:

  exp, sigmoid, cumprod, cumsum, norm, maximum / minimum, linspace, meshgrid, searchsorted, gather, argsort (returns
  (index, values)), random, init.gauss, reshape, concat, sum with keepdims, flags.no_grad, sync_all, and the Var methods
  t / expand / detach (masked __setitem__ is ndarray's).

jt.maximum(a, b) / jt.minimum(a, b) follow std::max / std::min, which Jittor's binary ops use: max(a, b) = a < b ? b : a
and min(a, b) = b < a ? b : a.  Neither propagates a NaN in b: jt.maximum(1e-10, nan) is 1e-10.  jt.linspace(start, end,
steps) is k * (end - start) / (steps - 1) + start.  random() and init.gauss() draw float32 from one seeded generator and
append ("uniform" | "normal", array) to `draws`, so a golden can hand the same numbers to the code under test.
"""
import sys
import types

import numpy as np

from oracle import jittor_numpy_stub as stub

F32 = np.float32


def _v(a):
    return np.asarray(a).view(stub.Var)


def _expand(self, *shape):
    if len(shape) == 1 and isinstance(shape[0], (tuple, list)):
        shape = tuple(shape[0])
    return np.broadcast_to(np.asarray(self), tuple(shape)).copy().view(stub.Var)


def _t(self):
    return np.asarray(self).T.copy().view(stub.Var)


_VAR_METHODS = dict(expand=_expand, t=_t, detach=lambda self: self)


def install(seed=0):
    """Install the stub as `jittor`; returns (restore, draws)."""
    restore_base = stub.install()
    jt = sys.modules["jittor"]
    rng = np.random.default_rng(seed)
    draws = []
    a32 = lambda x: np.asarray(x)

    def linspace(start, end, steps):
        steps = int(steps)
        if steps == 1:
            return _v(np.full(1, start, F32))
        return _v((np.arange(steps, dtype=F32) * F32(end - start)) / F32(steps - 1) + F32(start))

    def random(shape, dtype="float32", type="uniform"):
        assert type == "uniform"
        x = rng.random(tuple(shape), dtype=np.float32)
        draws.append(("uniform", x.copy()))
        return _v(x)

    def gauss(shape, dtype="float32", mean=0.0, std=1.0):
        x = (rng.standard_normal(tuple(shape), dtype=np.float32) * F32(std) + F32(mean)).astype(F32)
        draws.append(("normal", x.copy()))
        return _v(x)

    def searchsorted(sorted_seq, values, right=False):
        s, v = a32(sorted_seq), a32(values)
        cmp = (s[..., None, :] <= v[..., :, None]) if right else (s[..., None, :] < v[..., :, None])
        return _v(cmp.sum(-1).astype(np.int32))

    def argsort(x, dim=-1, descending=False):
        a = a32(x)
        idx = np.argsort(-a if descending else a, axis=dim, kind="stable").astype(np.int32)
        return _v(idx), _v(np.take_along_axis(a, idx, dim))

    def jsum(a, dim=None, keepdims=False, keepdim=False):
        a = a32(a)
        return _v(np.asarray(np.sum(a, axis=dim, keepdims=keepdims or keepdim, dtype=a.dtype)))

    def norm(x, p=2, dim=-1, keepdim=False, keepdims=False):
        assert p == 2
        a = a32(x)
        return _v(np.sqrt(np.sum(a * a, axis=dim, keepdims=keepdim or keepdims, dtype=a.dtype)))

    jt.exp = lambda a: _v(np.exp(a32(a)))
    jt.sigmoid = lambda a: _v(F32(1) / (F32(1) + np.exp(-a32(a))))
    jt.cumprod = lambda a, dim=-1: _v(np.cumprod(a32(a), axis=dim, dtype=a32(a).dtype))
    jt.cumsum = lambda a, dim=-1: _v(np.cumsum(a32(a), axis=dim, dtype=a32(a).dtype))
    jt.norm = norm
    jt.maximum = lambda a, b: _v(np.where(a32(a) < a32(b), a32(b), a32(a)))
    jt.minimum = lambda a, b: _v(np.where(a32(b) < a32(a), a32(b), a32(a)))
    jt.linspace = linspace
    jt.meshgrid = lambda *xs: [_v(m) for m in np.meshgrid(*[a32(x) for x in xs], indexing="ij")]
    jt.searchsorted = searchsorted
    jt.gather = lambda x, dim, index: _v(np.take_along_axis(a32(x), a32(index).astype(np.int64), dim))
    jt.argsort = argsort
    jt.random = random
    jt.init = types.SimpleNamespace(gauss=gauss)
    jt.reshape = lambda a, shape: _v(np.reshape(a32(a), tuple(shape)))
    jt.concat = stub.concat
    jt.sum = jsum
    jt.zeros_like = lambda a: _v(np.zeros_like(a32(a)))
    jt.flags = types.SimpleNamespace(no_grad=False, use_cuda=0)
    jt.sync_all = lambda *a, **k: None
    jt.nn.relu = lambda a: _v(np.maximum(a32(a), 0))
    saved = {k: stub.Var.__dict__.get(k) for k in _VAR_METHODS}
    for k, f in _VAR_METHODS.items():
        setattr(stub.Var, k, f)

    def restore():
        for k, f in saved.items():
            if f is None:
                delattr(stub.Var, k)
            else:
                setattr(stub.Var, k, f)
        restore_base()
    return restore, draws
