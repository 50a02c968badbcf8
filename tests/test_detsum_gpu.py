"""The fixed-order finishing sum of every cross-CTA reduction (csrc/detsum.cuh), run over caller-provided rows through
mcb_det_sum_f32 and compared bit for bit with a float32 re-summation in the documented order
(oracle/elementwise_checks.py reference_sum).  The BatchNorm statistics, the split-K weight gradients, the classifier
and loss sums of the train step all end in this sum, so its order is what keeps their last bits the same from build to
build.  Up to 32 rows the kernel runs one thread per element, above that one warp per element; row counts cover both:
one row, fewer than a warp, exactly a warp, and several lanes' worth (133 rows: more than the 132 SMs of an H100, the
most CTAs a persistent producer launches)."""
import numpy as np
import pytest

from oracle.elementwise_checks import reference_sum, run_det_sum, wide_range_rows

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nrows", [1, 7, 32, 33, 70, 133])
def test_det_sum_matches_fixed_order_bitwise(mcb, cuda, nrows):
    rng = np.random.default_rng(nrows)
    n = 1000                                  # not a multiple of the 256-thread CTA
    rows = wide_range_rows(rng, nrows, n)
    out0 = rng.standard_normal(n).astype(np.float32)
    got = run_det_sum(rows, n, n, 0, out0)
    want = (out0 + reference_sum(rows)).astype(np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), \
        "%d of %d elements differ" % (int((got.view(np.int32) != want.view(np.int32)).sum()), n)
    if nrows >= 33:
        # the order matters at these magnitudes: plain row order gives other bits, so the check above is a real one
        plain = out0.copy()
        acc = np.zeros(n, np.float32)
        for r in rows:
            acc = (acc + r).astype(np.float32)
        plain = (plain + acc).astype(np.float32)
        assert not np.array_equal(plain.view(np.int32), want.view(np.int32))


def test_det_sum_wide_output_and_strided_destination(mcb, cuda):
    """a weight-gradient-sized output written into a wider destination (concat slice: inner columns of every
    out_stride), with the rows of a split-K launch"""
    rng = np.random.default_rng(7)
    inner, groups, out_stride = 192, 1500, 320
    n = inner * groups
    rows = wide_range_rows(rng, 9, n)
    dest = rng.standard_normal(groups * out_stride).astype(np.float32)
    got = run_det_sum(rows, n, inner, out_stride, dest)
    want = dest.copy()
    idx = (np.arange(n) // inner) * out_stride + np.arange(n) % inner
    want[idx] = (dest[idx] + reference_sum(rows)).astype(np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
