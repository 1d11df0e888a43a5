"""GPU tests of imsegm.classification: the device contingency table against np.unique + np.add.at for every pair of label dtypes,
with drop lists, negative values, a single value, every pixel dropped, value ranges on both sides of 2^26, tables on both sides of the
shared-memory limit, constant runs and white noise, lengths that are not a multiple of a warp's chunk and one 8192 x 8192 map; then
every public function against the oracle bit for bit on 2048 x 2048 class maps, the reference's goldens through the device, the
per-image frame and the error types."""
import logging
import warnings

import numpy as np
import pytest

from oracle import classification as oc

from conftest import synth_regions
from test_classification_host import assert_same, assert_same_outcome, check_golden, plain

pytestmark = pytest.mark.gpu

DTYPES = [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.int32, np.uint32, np.int64]
SMEM_CELLS = 16384


@pytest.fixture(scope='module')
def clf():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import classification
    return classification


@pytest.fixture
def quiet():
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        logging.disable(logging.CRITICAL)
        try:
            yield
        finally:
            logging.disable(logging.NOTSET)


def numpy_table(t, p, drop=()):
    keep = ~(np.isin(t, drop) | np.isin(p, drop))
    t, p = t[keep].astype(np.int64), p[keep].astype(np.int64)
    vt, it = np.unique(t, return_inverse=True)
    vp, ip = np.unique(p, return_inverse=True)
    counts = np.zeros((len(vt), len(vp)), np.int64)
    np.add.at(counts, (it.ravel(), ip.ravel()), 1)
    return vt, vp, counts


def device_table(clf, t, p, drop=()):
    (t, _), (p, _) = clf._labels(t), clf._labels(p)
    return clf._contingency(t, p, np.asarray(sorted(drop), dtype=np.int64))


def assert_table(clf, t, p, drop=()):
    got, want = device_table(clf, t, p, drop), numpy_table(t.ravel(), p.ravel(), drop)
    for g, w in zip(got, want):
        assert g.dtype == np.int64 and np.array_equal(g, w), (g, w)


def random_map(rng, dtype, n, k):
    if dtype == np.bool_:
        return rng.rand(n) < 0.5
    info = np.iinfo(dtype)
    lo = max(int(info.min), -k // 2)
    return rng.randint(lo, min(int(info.max), lo + k) + 1, n).astype(dtype)


@pytest.mark.parametrize('dt_true', DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize('dt_pred', DTYPES, ids=lambda d: np.dtype(d).name)
def test_table_every_dtype_pair(clf, dt_true, dt_pred):
    rng = np.random.RandomState(0)
    n = 100003                                   # not a multiple of a warp's chunk (512 pixels)
    t, p = random_map(rng, dt_true, n, 7), random_map(rng, dt_pred, n, 300)
    assert_table(clf, t, p)
    assert_table(clf, t, p, drop=[-1, 0, 5])
    runs = np.repeat(random_map(rng, dt_pred, n // 997 + 1, 50), 997)[:n]
    assert_table(clf, t, runs, drop=[1])


def test_table_edges(clf):
    rng = np.random.RandomState(1)
    for n in (1, 31, 32, 511, 512, 513, 4097):
        assert_table(clf, rng.randint(-3, 3, n), rng.randint(-3, 3, n).astype(np.int32))
    assert_table(clf, np.full(10000, 7, np.int64), np.full(10000, -2, np.int32))                   # single value, constant runs
    vt, vp, counts = device_table(clf, np.arange(1000), np.arange(1000), drop=list(range(1000)))   # every pixel dropped
    assert counts.shape == (0, 0) and len(vt) == len(vp) == 0
    big = np.array([0, (1 << 26) - 1, 5], np.int64)                                                # range of exactly 2^26 values
    assert_table(clf, big, big.astype(np.uint32))
    with pytest.raises(NotImplementedError):
        device_table(clf, np.array([0, 1 << 26], np.int64), np.zeros(2, np.int64))
    with pytest.raises(NotImplementedError):
        device_table(clf, np.zeros(2, np.int32), np.array([-(1 << 25), 1 << 25], np.int32))
    a = np.array([0, 1 << 27, 3], np.int64)                                                         # wide value dropped: fits
    assert_table(clf, a, np.zeros(3, np.int64), drop=[1 << 27])


def test_table_shared_memory_limit_and_noise(clf):
    rng = np.random.RandomState(2)
    n = 1 << 20
    for kt, kp in ((128, SMEM_CELLS // 128), (128, SMEM_CELLS // 128 + 1), (1, 1), (4096, 4096)):
        t = rng.randint(0, kt, n).astype(np.int32)
        p = rng.randint(0, kp, n).astype(np.int64)
        t[:kt], p[:kp] = np.arange(kt), np.arange(kp)        # every value present: the table is exactly kt x kp
        assert_table(clf, t, p)
    with pytest.raises(MemoryError):
        device_table(clf, np.arange(20000, dtype=np.int32), np.arange(20000, dtype=np.int32)[::-1].copy())


def test_table_8192(clf):
    _, annot = synth_regions(8192, 8192, n_classes=4, seed=3, cell=256)
    _, segm = synth_regions(8192, 8192, n_classes=5, seed=4, cell=128)
    assert_table(clf, annot.astype(np.uint8), segm.astype(np.int32), drop=[2])


def pair_2048(seed):
    _, annot = synth_regions(2048, 2048, n_classes=4, seed=seed)
    _, segm = synth_regions(2048, 2048, n_classes=3, seed=seed + 10, cell=32)
    return annot.astype(np.uint8), segm.astype(np.int64)


@pytest.mark.parametrize('relabel', [False, True])
@pytest.mark.parametrize('drop', [None, [0], [2, 7]])
def test_functions_equal_oracle_2048(clf, quiet, relabel, drop):
    annot, segm = pair_2048(5)
    assert_same_outcome(clf.compute_classif_stat_segm_annot, oc.compute_classif_stat_segm_annot, (annot, segm, 'img'),
                        drop_labels=drop, relabel=relabel)
    if drop is None and not relabel:
        assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, annot.ravel(), segm.ravel(),
                            tuple(clf.METRIC_AVERAGES) + ('micro', 'binary', 'samples'))
        assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, annot[:64, :64], segm[:64, :64])   # 2-D
        for func in ('compute_tp_tn_fp_fn', 'compute_metric_fpfn_tpfn', 'compute_metric_tpfp_tpfn'):
            assert_same_outcome(getattr(clf, func), getattr(oc, func), annot > 1, (segm > 0) * 3)


def test_goldens_through_device(clf):
    check_golden(clf)


def test_stat_per_image_frame(clf, quiet):
    import pandas as pd
    pairs = [pair_2048(s) for s in (6, 7, 8)]
    annots, segms = [a for a, _ in pairs], [s for _, s in pairs]
    for relabel in (False, True):
        got = clf.compute_stat_per_image(segms, annots, names=['a', 'b', 'c'], nb_workers=4, drop_labels=[0], relabel=relabel)
        want = oc.compute_stat_per_image(segms, annots, names=['a', 'b', 'c'], drop_labels=[0], relabel=relabel)
        pd.testing.assert_frame_equal(got, want, check_exact=True)


def test_error_types(clf, quiet):
    a = np.zeros((3, 3), int)
    for args in (((a, np.zeros((3, 4), int), 'x'), ), ((a, a, 'x'), [0])):
        assert_same_outcome(clf.compute_classif_stat_segm_annot, oc.compute_classif_stat_segm_annot, *args)
    assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.zeros(3), np.zeros(4))
    assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.arange(5) * .5, np.arange(5.))
    assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.ones(5), np.zeros(5))
    assert_same_outcome(clf.compute_stat_per_image, oc.compute_stat_per_image, [a], [])
    assert plain(clf.compute_classif_metrics([-1, 0, 0, -1, 0], [0, 0, -1, -1, 0])['confusion']) == [[5]]
    assert_same(plain(clf.compute_tp_tn_fp_fn(a, np.ones((3, 3)))), plain(oc.compute_tp_tn_fp_fn(a, np.ones((3, 3)))))
