"""The SoftRas forward against the oracle's per-entry error bound on the scenes of tests/softras_forward_cases.py.

Each case runs under both softras_exact_tail values, in the texture / fill_back / K variants of the sweep, at image
sizes 17 and 1000 (every 37th row compared) and batch 3.  soft_colors and the softmax sum must be within
oracle.softras.forward_bound entry by entry and bit-equal where it is 0; ids, faces_info, softmax_max and the hard-mode
aggregates bit-exact (tests.util.forward_bound_ratio).  The worst err / bound and the number of entries with a non-zero
bound are printed per case.
"""
import numpy as np
import pytest

from tests import softras_forward_cases as fc
from tests.util import forward_bound_ratio, run_cuda

pytestmark = pytest.mark.gpu


def run(name, variant, image_size, exact_tail, row_stride=1):
    from jrender_b200 import _lib
    fv, tex, P = fc.build(name, variant, image_size=image_size)
    try:
        _lib.set_option("softras_exact_tail", exact_tail)
        got = run_cuda(fv, tex, P, want_faces_info=image_size < 100)
    finally:
        _lib.set_option("softras_exact_tail", 0)
    r = forward_bound_ratio(got, fv, tex, P, exact_tail=bool(exact_tail), row_stride=row_stride)
    ref = r["ref"]
    rows = np.arange(0, image_size, row_stride)
    assert np.array_equal(got["faces_id_buffer"][:, :, rows], ref["faces_id_buffer"][:, :, rows]), "top-K ids not bit-exact"
    if "faces_info" in got:
        assert np.array_equal(got["faces_info"], ref["faces_info"], equal_nan=True), "faces_info not bit-exact"
    print("\n%s/%s/%d exact_tail=%d colors worst %.3f (%d bounded) sum %s" % (
        name, variant, image_size, exact_tail, r["colors"][0], r["colors"][1],
        "worst %.3f (%d bounded)" % r["sum"] if "sum" in r else "-"))
    return r


@pytest.mark.parametrize("exact_tail", [0, 1])
@pytest.mark.parametrize("variant", sorted(fc.VARIANTS))
@pytest.mark.parametrize("name", sorted(fc.CASES))
def test_forward_within_bound_17(cuda_device, name, variant, exact_tail):
    run(name, variant, 17, exact_tail)


@pytest.mark.parametrize("exact_tail", [0, 1])
@pytest.mark.parametrize("name", sorted(fc.CASES))
def test_forward_within_bound_1000(cuda_device, name, exact_tail):
    run(name, "surface1", 1000, exact_tail, row_stride=37)
