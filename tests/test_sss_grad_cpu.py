"""CPU tests of the float64 subsurface-scattering gradient mirror (oracle/sss_grad.py): its forward against the float32
oracle (oracle/sss.py), torch.autograd.gradcheck of its stretch, pyramid and bake, its written-out adjoint against
autograd, and the adjoint identity of one blur pass at fixed decisions."""
import numpy as np
import pytest
import torch

from oracle import bake as obake
from oracle import sss as osss
from oracle import sss_grad as sg


def maps(n, seed, holes=0.1):
    rng = np.random.default_rng(seed)
    su = np.clip(rng.uniform(-0.2, 1.2, (n, n)), 0, 1).astype(np.float32)
    sv = np.clip(rng.uniform(-0.2, 1.2, (n, n)), 0, 1).astype(np.float32)
    irr = rng.uniform(0.1, 1, (n, n, 3)).astype(np.float32)
    irr[rng.random((n, n)) < holes] = 0
    spec = rng.uniform(0, 0.3, (n, n, 3)).astype(np.float32)
    return su, sv, irr, spec


def f64(a, grad=False):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


@pytest.mark.parametrize("n", [16, 24, 64])
def test_pyramid_forward_matches_float32_oracle(n):
    su, sv, irr, spec = maps(n, n)
    levels = sg.walk(su, sv, irr)
    got = sg.pyramid(f64(su), f64(sv), f64(irr), f64(spec), levels).numpy()
    want = osss.blur_pyramid(su, sv, irr, spec)
    for lv, v in zip(levels, osss.levels()):     # the walk's float32 values are the oracle's, bit for bit
        g, w = osss.taps(v)
        np.testing.assert_array_equal(lv["su"], osss.blur(lv["su_in"], lv["su_in"], g, w, 1))
        np.testing.assert_array_equal(lv["irr_y"][1], osss.blur(lv["irr_x"][1], lv["sv"], g, w, 0))
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def test_stretch_forward_matches_float32_oracle():
    rng = np.random.default_rng(2)
    w = np.kron(rng.uniform(0, 1, (4, 4, 3)), np.ones((8, 8, 1))).astype(np.float32)
    w += rng.uniform(0, 0.05, w.shape).astype(np.float32) * (rng.random(w.shape[:2]) < 0.5)[..., None]
    got = sg.stretch(f64(w), sg.stretch_pass(w))
    for g, o in zip(got, osss.stretch(w)):
        assert np.abs(g.numpy() - o).max() <= 1e-6


def test_bake_forward_matches_float32_oracle():
    rng = np.random.default_rng(3)
    img = rng.uniform(0, 1, (40, 40, 3)).astype(np.float32)
    uv = rng.uniform(0, 1, (30, 3, 2)).astype(np.float32)
    uv[:3] = 1
    got = sg.bake(f64(img), uv, 3).numpy()
    want = obake.bake_textures_for_softras(img, uv, np.ones((30, 9, 3), np.float32), np.ones(30, np.int32))
    assert np.abs(got - want).max() <= 1e-6


@pytest.mark.parametrize("n", [16, 24])
def test_pyramid_gradcheck(n):
    """Three real levels; the point is moved off the kinks by construction (the decisions are fixed at the float32
    walk's, and gradcheck's steps of 1e-6 keep every value on the same side of them)."""
    su, sv, irr, spec = maps(n, 5 + n)
    levels = sg.walk(su, sv, irr)
    args = [f64(a, True) for a in (su, sv, irr, spec)]
    assert torch.autograd.gradcheck(lambda *a: sg.pyramid(*a, levels), args, eps=1e-6, atol=1e-6, rtol=1e-5,
                                    fast_mode=True)


def test_stretch_gradcheck():
    rng = np.random.default_rng(6)
    w = rng.uniform(0, 1, (12, 12, 3)).astype(np.float32)
    passes = sg.stretch_pass(w)
    assert passes[0].any() and (~passes[0]).any()
    assert torch.autograd.gradcheck(lambda x: sg.stretch(x, passes), [f64(w, True)], eps=1e-7, atol=1e-6, rtol=1e-5)


def test_bake_gradcheck():
    rng = np.random.default_rng(7)
    uv = rng.uniform(0, 1, (8, 3, 2)).astype(np.float32)
    uv[0] = 1
    assert torch.autograd.gradcheck(lambda x: sg.bake(x, uv, 3, np.array([1, 0, 1, 1, 1, 0, 1, 1])),
                                    [f64(rng.uniform(0, 1, (10, 10, 3)), True)], eps=1e-6, atol=1e-8)


@pytest.mark.parametrize("stretch", [True, False])
def test_written_adjoint_equals_autograd(stretch):
    """pyramid_vjp, the stage-by-stage adjoint the kernels run, at the float64 intermediates: autograd's gradient."""
    su, sv, irr, spec = maps(32, 9)
    levels = sg.walk(su, sv, irr)
    a = [f64(x, True) for x in (su, sv, irr, spec)]
    out = sg.pyramid(*a, levels)
    g = torch.tensor(np.random.default_rng(10).normal(size=tuple(out.shape)))
    out.backward(g)
    vals = sg.pyramid_values(a[0].detach(), a[1].detach(), a[2].detach(), levels)
    r = sg.pyramid_vjp(levels, a[2].detach(), g, values=vals, stretch=stretch)
    for k, x in (("irradiance", a[2]), ("specular", a[3])) + ((("stretch_u", a[0]), ("stretch_v", a[1])) if stretch else ()):
        assert torch.allclose(r[k], x.grad, rtol=1e-12, atol=1e-12 * float(x.grad.abs().max())), k
    m = sg.pyramid_vjp(levels, a[2].detach(), g, values=vals, magnitude=True, stretch=stretch)
    for k in r:
        if r[k] is not None:
            assert (m[k] >= r[k].abs() - 1e-12).all(), k     # term sums bound the sums


@pytest.mark.parametrize("dim", [0, 1])
def test_blur_adjoint_identity(dim):
    """<G, J d> = <J^T G, d> for one blur pass, linear in the image at fixed decisions and modulation."""
    su, _, irr, _ = maps(40, 11)
    img = irr[..., 0]
    g32, w32 = osss.taps(75)
    dec = sg.decisions(img, su, g32, w32, dim)
    rng = np.random.default_rng(12)
    G, d = f64(rng.normal(size=img.shape)), f64(rng.normal(size=img.shape))
    Jd = sg.blur(d, f64(su), dec, g32, w32) - sg.blur(torch.zeros_like(d), f64(su), dec, g32, w32)
    JtG, _ = sg.blur_vjp(f64(img), f64(su), dec, g32, w32, G)
    # blur() replaces neighbours by the centre value of the image it is given: at fixed decisions that is linear too
    assert abs(float((G * Jd).sum()) - float((JtG * d).sum())) <= 1e-10 * float((G.abs() * Jd.abs()).sum() + 1)


def test_mirror_bound_contains_float32_point():
    """At the float32 intermediates the written adjoint sits within the bound of the float64 one."""
    su, sv, irr, spec = maps(32, 13, holes=0.2)
    levels = sg.walk(su, sv, irr)
    g = torch.tensor(np.random.default_rng(14).normal(size=irr.shape))
    vals = sg.pyramid_values(f64(su), f64(sv), f64(irr), levels)
    r64 = sg.pyramid_vjp(levels, f64(irr), g, values=vals)
    r32 = sg.pyramid_vjp(levels, f64(irr), g)
    m = sg.pyramid_vjp(levels, f64(irr), g, magnitude=True)
    for k in ("irradiance", "specular"):
        assert ((r32[k] - r64[k]).abs() <= sg.bound(m[k])).all(), k
