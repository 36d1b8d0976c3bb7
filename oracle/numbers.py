"""Number types the kernel emulations are written over (TEST INFRASTRUCTURE; product code never imports it).

EV     a float64 value and a running bound on how far the float32 evaluation of the same expression can be from it.
Dual   forward-mode dual numbers over any of those number types, operation for operation as csrc/dual.cuh: one
       rounding per value and per partial, Dual-with-float rules distinct from Dual-with-Dual ones.
Walk   the branch decisions of one emulation run: taken on the float32 walk and replayed, unchanged, by a walk in
       another number type, which counts the members whose exact value lies within its bound of the kink.
"""
import numpy as np

F32 = np.float32
U = 2.0 ** -24      # fp32 unit roundoff
U64 = 2.0 ** -52
TINY = 2.0 ** -149  # gradual underflow


def _num(o):
    return isinstance(o, (EV, np.ndarray, np.generic, float, int))


class EV:
    """float64 value `v` and a bound `e` on |float32 evaluation - exact value| of the expression that produced it.
    Every operation adds the propagated input error and one rounding u = 2^-24 of the result, 2^-52 for the float64
    value's own rounding and 2^-149 for gradual underflow."""

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, EV) else EV(x)

    @staticmethod
    def _round(v, prop):
        return EV(v, prop + (U + U64) * (np.abs(v) + prop) + TINY)

    @property
    def shape(self):
        return self.v.shape

    def __getitem__(self, i):
        return EV(self.v[i], self.e[i])

    def __setitem__(self, i, x):
        x = EV.of(x)
        self.v[i], self.e[i] = x.v, x.e

    def __neg__(self):
        return EV(-self.v, self.e)

    def __add__(self, o):
        if not _num(o):
            return NotImplemented
        o = EV.of(o)
        return EV._round(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        if not _num(o):
            return NotImplemented
        o = EV.of(o)
        return EV._round(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return EV.of(o) - self

    def __mul__(self, o):
        if not _num(o):
            return NotImplemented
        o = EV.of(o)
        return EV._round(self.v * o.v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        if not _num(o):
            return NotImplemented
        o = EV.of(o)
        with np.errstate(all="ignore"):
            q = self.v / o.v
            den = np.abs(o.v) - o.e
            prop = np.where(den > 0, (self.e + np.abs(q) * o.e) / den, np.inf)
        return EV._round(q, prop)

    def __rtruediv__(self, o):
        return EV.of(o) / self

    def sqrt(self):
        with np.errstate(all="ignore"):
            r = np.sqrt(np.maximum(self.v, 0))
            prop = np.minimum(np.where(r > 0, self.e / r, np.inf), np.sqrt(self.e))
        return EV._round(r, prop)


def cuda_int(a):
    """C float -> int conversion as the GPU does it (cvt.rzi.s32.f32 / .f64): truncation toward zero, saturating at
    INT_MIN / INT_MAX, NaN -> 0.  Returned as int64 (numpy's own astype gives INT64_MIN for NaN and +-inf on x86)."""
    a = np.nan_to_num(np.asarray(a, np.float64), nan=0.0, posinf=2147483647.0, neginf=-2147483648.0)
    return np.clip(np.trunc(a), -2147483648.0, 2147483647.0).astype(np.int64)


def fminf(a, b):
    """CUDA fminf / fmin: the other operand where one is NaN (np.minimum would propagate the NaN)."""
    return np.fmin(a, b)


def fmaxf(a, b):
    """CUDA fmaxf / fmax: the other operand where one is NaN."""
    return np.fmax(a, b)


def check_terms(f32, ev):
    """Every emulated float32 term is within its EV bound of the float64 value of the same expression (where that bound
    is finite), and NaN wherever that value is NaN."""
    f32 = np.asarray(f32, np.float64)
    ok = np.isfinite(ev.v) & np.isfinite(ev.e)
    assert np.isfinite(f32[ok]).all()
    assert np.all(np.abs(f32 - ev.v)[ok] <= ev.e[ok]), (np.abs(f32 - ev.v)[ok] / ev.e[ok]).max()
    assert np.isnan(f32[np.isnan(ev.v)]).all()


def sqrt(x):
    return x.sqrt() if hasattr(x, "sqrt") else np.sqrt(x)


def full(x, c):
    """c in x's number type and shape (an exact constant: EV error 0)."""
    if isinstance(x, EV):
        return EV(np.full(x.v.shape, c))
    return np.full(np.shape(x), F32(c), F32) if np.ndim(x) else F32(c)


def where(m, a, b):
    """np.where for float32 arrays, EV and Dual (partials component by component)."""
    if isinstance(a, Dual) or isinstance(b, Dual):
        n = len(a.d) if isinstance(a, Dual) else len(b.d)
        a, b = (x if isinstance(x, Dual) else Dual(x, [full(x, 0)] * n) for x in (a, b))
        return Dual(where(m, a.v, b.v), [where(m, p, q) for p, q in zip(a.d, b.d)])
    if isinstance(a, EV) or isinstance(b, EV):
        a, b = EV.of(a), EV.of(b)
        return EV(np.where(m, a.v, b.v), np.where(m, a.e, b.e))
    return np.where(m, a, b)


def value(x):
    """float64 value of a float32 array or an EV."""
    return x.v if isinstance(x, EV) else np.asarray(x, np.float64)


class Dual:
    """Value and N partials, each of the base number type; the rules of csrc/dual.cuh."""
    __array_ufunc__ = None   # numpy array (op) Dual defers to Dual's reflected operator

    def __init__(self, v, d):
        self.v, self.d = v, list(d)

    @staticmethod
    def var(v, i, n, zero):
        return Dual(v, [zero + 1 if k == i else zero for k in range(n)])

    @staticmethod
    def const(v, n, zero):
        return Dual(v, [zero] * n)

    def __add__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v + o.v, [a + b for a, b in zip(self.d, o.d)])
        return Dual(self.v + o, self.d)

    __radd__ = __add__

    def __sub__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v - o.v, [a - b for a, b in zip(self.d, o.d)])
        return Dual(self.v - o, self.d)

    def __rsub__(self, s):   # float - Dual
        return Dual(s - self.v, [-a for a in self.d])

    def __mul__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v * o.v, [a * o.v + self.v * b for a, b in zip(self.d, o.d)])
        return Dual(self.v * o, [a * o for a in self.d])

    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, Dual):
            r = self.v / o.v
            ib = full(o.v, 1) / o.v
            return Dual(r, [(a - r * b) * ib for a, b in zip(self.d, o.d)])
        return self * (full(o, 1) / o)   # a * (1.f / s)

    def sqrt(self):
        r = sqrt(self.v)
        h = full(r, 0.5) / r
        return Dual(r, [a * h for a in self.d])


class Walk:
    """Branch decisions of an emulation run, in call order.  A recording walk (`replay=None`) decides from its own
    float32 values; a replaying walk takes the recorded decisions and flags, per member (first axis), the EV values
    within their bound of the kink, by kind."""

    def __init__(self, replay=None):
        self.decisions = [] if replay is None else replay.decisions
        self.replaying = replay is not None
        self.i = 0
        self.near = {}

    def decide(self, kind, arg, lo, fn):
        """fn(arg value, lo) -> decision array, on the float32 walk; recorded there, replayed here.  With EV, the
        members where |arg - lo| is within its bound are flagged under `kind`."""
        if not self.replaying:
            d = fn(arg, lo)
            self.decisions.append(d)
            return d
        d = self.decisions[self.i]
        self.i += 1
        if isinstance(arg, EV):
            diff = arg - lo
            with np.errstate(invalid="ignore"):
                near = np.abs(diff.v) <= diff.e
            near = np.broadcast_to(near, np.shape(d))
            near = near.reshape(near.shape[0], -1).any(1) if near.ndim > 1 else near
            self.near[kind] = self.near.get(kind, False) | near
        return d


# max-type rules of dual.cuh, over a Walk: state 0 where the value is replaced by lo, 1 where the derivative passes,
# 2 where a is NaN (value NaN, derivative 0)
def _state(strict):
    def fn(a, lo):
        a = value(a)
        with np.errstate(invalid="ignore"):
            passes = a > lo if strict else a >= lo
            return np.where(passes, 1, np.where(a <= lo, 0, 2)).astype(np.int8)
    return fn


def _max(walk, kind, a, lo, strict):
    av = a.v if isinstance(a, Dual) else a
    s = walk.decide(kind, av, lo, _state(strict))
    if isinstance(a, Dual):
        return Dual(where(s == 0, lo, av), [where(s == 1, p, full(p, 0)) for p in a.d])
    return where(s == 0, lo, av)


def dmax(walk, kind, a, lo):
    """max(a, lo) with the derivative passing where a > lo: torch.relu's rule."""
    return _max(walk, kind, a, lo, True)


def dclamp_min(walk, kind, a, lo):
    """max(a, lo) with the derivative passing where a >= lo: torch.clamp(min=) / clamp_min's rule."""
    return _max(walk, kind, a, lo, False)
