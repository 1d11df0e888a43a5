"""The host model of the statistics' summation order (tests/statistics_order_reference.py) on the CPU.

The GPU tests hold the device to this model bit for bit, so the model itself must be right: here its totals are compared with
math.fsum of the pixel terms of each label, within the recursive-summation bound gamma_n * sum |t| (n terms: a term passes through
at most n - 1 additions of the run, warp and label sums, and the last rounding), and its order is checked on inputs small enough to
write out by hand.
"""
import math

import numpy as np
import pytest

import statistics_order_reference as ref

U = 2.0 ** -53


def gamma(n):
    return n * U / (1 - n * U)


def _wide(shape, rng):
    """float32 values from 1e-44 to 1e38 in magnitude, both signs: the order of their additions shows in the bits"""
    mag = 10.0 ** rng.uniform(-44, 38, shape)
    return (mag * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _check_fsum(terms, seg, nb, what):
    """model totals against math.fsum per label within gamma_n sum |t|"""
    labels, parts = ref.colour_partials(terms, seg) if terms.ndim == 3 else ref.gray_partials(terms, seg)
    got = ref.label_totals(labels, parts, nb)
    flat, s = terms.reshape(-1, terms.shape[-1]), seg.ravel()
    for lb in range(nb):
        members = flat[s == lb]
        for k in range(flat.shape[1]):
            want = math.fsum(members[:, k].tolist())
            bound = gamma(len(members)) * np.abs(members[:, k]).sum()
            assert abs(got[lb, k] - want) <= bound, '%s: label %d column %d: %r vs fsum %r, bound %g' % (what, lb, k, got[lb, k], want, bound)


@pytest.mark.parametrize('W', [31, 32, 33, 257, 300])
@pytest.mark.parametrize('H', [1, 15, 16, 17, 40])
def test_colour_model_within_fsum_bound(H, W):
    rng = np.random.RandomState(H * 1000 + W)
    yy, xx = np.mgrid[:H, :W]
    for kind, seg in (('one', np.zeros((H, W), np.int64)), ('stripes', (yy // 5) * 3 + (xx // 3) % 3),
                      ('random', rng.randint(0, 7, (H, W)))):
        v = _wide((H, W, 3), rng).astype(np.float64)
        _check_fsum(v, seg, int(seg.max()) + 1, '%dx%d %s' % (H, W, kind))


@pytest.mark.parametrize('n', [1, 15, 16, 17, 1000])
def test_gray_model_within_fsum_bound(n):
    rng = np.random.RandomState(n)
    seg = np.sort(rng.randint(0, 5, n))                    # runs that cross the 16-voxel strips
    v = _wide((n, 1), rng).astype(np.float64)
    _check_fsum(v, seg, 5, 'gray %d' % n)


def test_seg_sum_tree_order():
    """one row, one warp: lanes 0..4 end runs of label 3, lane 5 does not flush, lanes 6..31 end runs of label 4.  Lane 0 heads
    [0, 5): ((t0 + t1) + (t2 + t3)) + t4 by the shuffle-down steps; lane 6 heads [6, 32)"""
    t = np.array([1.0, 2.0 ** -60, 2.0 ** -60, 2.0 ** -60, 2.0 ** -60] + [0.0] + [1.0] * 26)
    flush = np.array([True] * 5 + [False] + [True] * 26)
    key = np.array([3] * 5 + [9] + [4] * 26)
    head, v = ref._seg_sum(t[None, :, None], flush[None], key[None])
    assert list(np.flatnonzero(head[0])) == [0, 6]
    assert v[0, 0, 0] == ((1.0 + 2.0 ** -60) + (2.0 ** -60 + 2.0 ** -60)) + 2.0 ** -60 == 1.0
    assert v[0, 6, 0] == 26.0


def test_column_runs_flush_at_label_changes_and_strip_ends():
    """a single column over 40 rows: runs end where the label changes and at the ends of the 16-row strips"""
    seg = np.array([0] * 10 + [1] * 20 + [0] * 10)[:, None]
    terms = np.arange(40, dtype=np.float64)[:, None, None]
    labels, parts = ref.colour_partials(terms, seg)
    runs = [(0, 0, 10), (1, 10, 16), (1, 16, 30), (0, 30, 32), (0, 32, 40)]
    assert sorted(zip(labels.tolist(), parts[:, 0].tolist())) == sorted((lb, float(sum(range(a, b)))) for lb, a, b in runs)


def test_exact_total_specials_and_rounding():
    assert math.isnan(ref.exact_total([1.0, np.nan]))
    assert math.isnan(ref.exact_total([np.inf, -np.inf, 1.0]))
    assert ref.exact_total([np.inf, 1.0, 1e300]) == np.inf
    assert ref.exact_total([-np.inf, 1.0]) == -np.inf
    s = ref.exact_total([-0.0])
    assert s == 0.0 and math.copysign(1.0, s) == 1.0
    assert ref.exact_total([1e30, 1.0, -1e30]) == 1.0                   # a recursive sum gives 0
    assert ref.exact_total([1.0, 2.0 ** -53, 2.0 ** -53]) == 1.0 + 2.0 ** -52


def test_banded_model_adds_band_totals():
    """two bands: each band's rounded totals added in band order, not the whole image's"""
    rng = np.random.RandomState(7)
    H, W = 40, 33
    seg = np.zeros((H, W), np.int64)
    img = _wide((H, W, 3), rng)
    mean_b = ref.colour_stats(img, seg, 1, bands=[(0, 17), (17, H)])[0]
    t = ref.f32_terms(img).astype(np.float64)
    lab0, par0 = ref.colour_partials(t[:17], seg[:17])
    lab1, par1 = ref.colour_partials(t[17:], seg[17:])
    a0, a1 = ref.label_totals(lab0, par0, 1), ref.label_totals(lab1, par1, 1)
    np.testing.assert_array_equal(mean_b[0], ((a0 + a1) / (H * W))[0, :3])
