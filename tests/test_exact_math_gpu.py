"""GPU check that csrc/exact_math.cuh reproduces the plain IEEE expressions bit for bit:
fast_div == a / b (nvcc's own division), f2d_mid == (double)x, d2f_mid == (float)d (including
exact round-to-even ties), sigmoid_tail and alpha_prod == the reference's double expressions."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(a, b):
    import torch
    from jrender_b200 import _lib
    ta = torch.from_numpy(a).cuda()
    tb = torch.from_numpy(b).cuda()
    mm = torch.zeros(7, dtype=torch.int32, device="cuda")
    _lib.call("b200r_debug_exact_math", mm.device, ta, tb, a.size, mm)
    return mm.cpu().numpy()


def test_random_bit_patterns(cuda_device):
    rng = np.random.default_rng(0)
    n = 1 << 24
    a = rng.integers(0, 2**32, n, dtype=np.uint32).view(np.float32)   # everything incl. NaN/inf/denormals
    b = rng.integers(0, 2**32, n, dtype=np.uint32).view(np.float32)
    mm = _run(a, b)
    assert mm[:6].tolist() == [0] * 6, mm


def test_rasterizer_value_ranges(cuda_device):
    import torch
    g = torch.Generator(device="cuda").manual_seed(1)
    total_fast = 0
    iters = 8
    for it in range(iters):
        n = 1 << 24

        def rnd(lo, hi):
            e = torch.empty(n, device="cuda").uniform_(lo, hi, generator=g)
            m = torch.empty(n, device="cuda").uniform_(1, 2, generator=g)
            s = (torch.randint(0, 2, (n,), device="cuda", generator=g) * 2 - 1).float()
            return (s * torch.exp2(e) * m).cpu().numpy()
        a, b = rnd(-20, 4), rnd(-20, 7)
        if it == 0:   # special numerators / denominators
            a[:64] = np.float32([0.0, -0.0, 1.0, -1.0] * 16)
            b[64:128] = np.float32([1.0, 3.0, 1e-4, 1e-5] * 16)
            b[128:192] = np.nextafter(np.float32(2.0), np.float32(0.0))   # all-ones mantissa
        mm = _run(a, b)
        assert mm[:6].tolist() == [0] * 6, (it, mm)
        total_fast += int(mm[6])
    assert total_fast > 0.9 * iters * (1 << 24)   # the reciprocal path is the one being exercised


def test_structured_mantissas(cuda_device):
    """All 2^12 x 2^12 combinations of coarse mantissas plus all-ones / one-bit patterns."""
    m = (np.arange(4096, dtype=np.uint32) << 11) | 0x3f800000
    a = np.repeat(m, 4096).view(np.float32)
    b = np.tile(m | 0x7ff, 4096).view(np.float32)
    mm = _run(a.copy(), b.copy())
    assert mm[:6].tolist() == [0] * 6, mm
