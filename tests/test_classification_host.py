"""CPU tests of imsegm.classification: the oracle (oracle/classification.py) against the reference's own outputs
(tests/golden/classification_reference.npz, made by make_classification_goldens.py); the sparse look-up table of the ``relabel`` step
against labeling.max_overlap_unique_lut on expanded overlap matrices; and the host metric code, fed a contingency table counted by
numpy, against the oracle on the pixel arrays -- every dict entry with ``==`` (NaN where NaN) and every exception type."""
import json
import logging
import os
import warnings

import numpy as np
import pytest

from oracle import classification as oc
from pyimsegm_b200 import classification as clf
from pyimsegm_b200.labeling import max_overlap_unique_lut
from pyimsegm_b200.utilities import ImageDimensionError

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
AVERAGES = tuple(clf.METRIC_AVERAGES) + ('micro', 'binary', 'samples')


def plain(v):
    """the golden's JSON form of an output"""
    if isinstance(v, dict):
        return {str(k): plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, np.ndarray)):
        return [plain(x) for x in list(v)]
    if isinstance(v, np.integer):
        return int(v)
    if isinstance(v, (np.floating, float)):
        return float(v)
    return v


def assert_same(got, want, where=''):
    if isinstance(want, dict):
        assert isinstance(got, dict) and sorted(got) == sorted(want), (where, got, want)
        for k in want:
            assert_same(got[k], want[k], '%s[%s]' % (where, k))
    elif isinstance(want, list):
        assert isinstance(got, list) and len(got) == len(want), (where, got, want)
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, '%s[%d]' % (where, i))
    elif isinstance(want, float) and np.isnan(want):
        assert isinstance(got, float) and np.isnan(got), (where, got, want)
    else:
        assert got == want, (where, got, want)


def golden_cases():
    data = np.load(os.path.join(GOLDEN, 'classification_reference.npz'))
    return data, json.loads(str(data['cases']))


def run_case(module, data, case):
    """(plain output, None) or (None, exception type name) of one golden case through ``module``"""
    args = [list(data[k]) if case['func'] == 'compute_stat_per_image' else data[k] for k in case['inputs']]
    if case['func'] == 'compute_classif_stat_segm_annot':
        args = [(args[0], args[1], case['name'])]
    try:
        out = getattr(module, case['func'])(*args, **case['kwargs'])
    except Exception as err:
        return None, type(err).__name__
    if case['func'] == 'compute_stat_per_image':
        out = {str(idx): row.to_dict() for idx, row in out.iterrows()}
    return plain(out), None


def check_golden(module):
    data, cases = golden_cases()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        logging.disable(logging.CRITICAL)
        try:
            for case in cases:
                out, err = run_case(module, data, case)
                if 'raises' in case:
                    assert err == case['raises'], (case['name'], out, err)
                else:
                    assert err is None, (case['name'], err)
                    assert_same(out, case['value'], case['name'])
        finally:
            logging.disable(logging.NOTSET)


def test_oracle_equals_reference_goldens():
    check_golden(oc)


def test_golden_file_is_small():
    assert os.path.getsize(os.path.join(GOLDEN, 'classification_reference.npz')) < 64 * 1024


def test_public_names_and_constants():
    import imsegm.classification as alias
    assert alias is clf
    for name in ('compute_classif_metrics', 'compute_classif_stat_segm_annot', 'compute_stat_per_image', 'compute_tp_tn_fp_fn',
                 'compute_metric_fpfn_tpfn', 'compute_metric_tpfp_tpfn', 'relabel_sequential'):
        assert callable(getattr(clf, name))
    assert clf.METRIC_AVERAGES == ('macro', 'weighted')
    assert clf.METRIC_SCORING == ('f1_macro', 'accuracy', 'precision_macro', 'recall_macro')
    assert sorted(clf.DICT_SCORING) == ['accuracy', 'f1', 'precision', 'recall']
    assert clf.TEMPLATE_NAME_CLF.format('x') == 'classifier_x.pkl'
    assert (clf.DEFAULT_CLASSIF_NAME, clf.DEFAULT_CLUSTERING) == ('RandForest', 'kMeans')


def test_relabel_sequential_host():
    assert clf.relabel_sequential([0, 0, 0, 5, 5, 5, 0, 5]) == [0, 0, 0, 1, 1, 1, 0, 1]
    for labels, uq in (([-1, 0, 0, -1], [-1, 0]), ([3, 7, 3], None), ([2, 2], [2])):
        assert clf.relabel_sequential(labels, uq) == oc.relabel_sequential(labels, uq)


def _expanded(rng, shape, dense, ties):
    ov = rng.randint(1, 4 if ties else 50, shape) * (rng.rand(*shape) < dense)
    if shape[0] > 2:
        ov[rng.randint(shape[0])] = 0       # an empty row
    return ov


@pytest.mark.parametrize('keep_bg', [False, True])
def test_sparse_lut_equals_dense(keep_bg):
    rng = np.random.RandomState(3)
    for trial in range(300):
        shape = (rng.randint(1, 9), rng.randint(1, 9))
        ov = _expanded(rng, shape, rng.choice([0.1, 0.4, 1.0]), trial % 2 == 0)
        r, c = np.nonzero(ov)
        want = max_overlap_unique_lut(ov, shape[1], keep_bg)
        got = clf._unique_lut(r, c, ov[r, c], shape[1], keep_bg, np.arange(shape[1]))
        assert got.tolist() == want, (ov, got, want)


def _numpy_table(t, p, drop=()):
    keep = ~(np.isin(t, drop) | np.isin(p, drop))
    t, p = t[keep].astype(np.int64), p[keep].astype(np.int64)
    vt, it = np.unique(t, return_inverse=True)
    vp, ip = np.unique(p, return_inverse=True)
    counts = np.zeros((len(vt), len(vp)), np.int64)
    np.add.at(counts, (it.ravel(), ip.ravel()), 1)
    return vt, vp, counts


def _outcome(func, *args, **kwargs):
    try:
        out = func(*args, **kwargs)
    except Exception as err:
        return None, type(err).__name__
    if hasattr(out, 'iterrows'):
        out = {str(idx): row.to_dict() for idx, row in out.iterrows()}
    return plain(out), None


def assert_same_outcome(func, oracle_func, *args, **kwargs):
    got, got_err = _outcome(func, *args, **kwargs)
    want, want_err = _outcome(oracle_func, *args, **kwargs)
    assert got_err == want_err, (got_err, want_err)
    if want_err is None:
        assert_same(got, want)


def _random_maps(rng, n):
    lo, hi = rng.randint(-3, 1), rng.randint(1, 7)
    a = rng.randint(lo, hi, n)
    b = rng.randint(lo, rng.randint(lo + 1, hi + 1), n)
    return a, b


def test_host_metrics_from_numpy_table_equal_oracle(monkeypatch):
    monkeypatch.setattr(clf, '_contingency', _numpy_table)
    rng = np.random.RandomState(11)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        logging.disable(logging.CRITICAL)
        try:
            for trial in range(150):
                a, b = _random_maps(rng, rng.randint(1, 400))
                if trial % 4 == 0:
                    a, b = np.abs(a), np.abs(b)
                assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, a, b, AVERAGES)
                for relabel in (False, True):
                    for drop in (None, [-1], [0, 5], [1, 2, 3]):
                        assert_same_outcome(clf.compute_classif_stat_segm_annot, oc.compute_classif_stat_segm_annot, (a, b, 'x'),
                                            drop_labels=drop, relabel=relabel)
                for func in ('compute_tp_tn_fp_fn', 'compute_metric_fpfn_tpfn', 'compute_metric_tpfp_tpfn'):
                    assert_same_outcome(getattr(clf, func), getattr(oc, func), a % 2 * 3, b % 2 * 3)
            # the reference's quirks: -1 and 0 collapse into one class; float maps with two labels raise TypeError
            assert clf.compute_classif_metrics([-1, 0, 0, -1, 0], [0, 0, -1, -1, 0])['confusion'] == [[5]]
            assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.ones(5), np.zeros(5))
            assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.arange(5.), np.arange(5.)[::-1])
            assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.arange(5) * .5, np.arange(5.))
            assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, np.zeros(3), np.zeros(4))
            for a, b in ((np.arange(12).reshape(3, 4) % 5, np.arange(12).reshape(3, 4) % 3), (np.eye(3), np.eye(3)),
                         (np.eye(3, dtype=int) - 1, np.eye(3, dtype=int))):
                assert_same_outcome(clf.compute_classif_metrics, oc.compute_classif_metrics, a, b)    # 2-D maps
            a, b = np.zeros((3, 3), int), np.zeros((3, 4), int)
            with pytest.raises(ImageDimensionError):
                clf.compute_classif_stat_segm_annot((a, b, 'x'))
            with pytest.raises(RuntimeError):
                clf.compute_stat_per_image([a], [])
        finally:
            logging.disable(logging.NOTSET)


def test_weighted_cells_equal_pixel_arrays_bit_for_bit():
    """precision_recall_fscore_support on the cells weighted by their counts returns what it returns on the pixels"""
    from sklearn import metrics
    rng = np.random.RandomState(5)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for _ in range(100):
            a, b = _random_maps(rng, rng.randint(2, 2000))
            vt, vp, counts = _numpy_table(a, b)
            r, c = np.nonzero(counts)
            for avg in (None, ) + AVERAGES:
                try:
                    want = metrics.precision_recall_fscore_support(a, b, average=avg)
                except ValueError as err:
                    with pytest.raises(type(err)):
                        metrics.precision_recall_fscore_support(vt[r], vp[c], average=avg, sample_weight=counts[r, c])
                    continue
                got = metrics.precision_recall_fscore_support(vt[r], vp[c], average=avg, sample_weight=counts[r, c])
                for g, w in zip(got, want):
                    if w is None:
                        assert g is None
                    elif avg is None and w.dtype.kind == 'i':
                        assert np.array_equal(g, w)     # support: float sums of integer weights
                    else:
                        assert np.array_equal(np.asarray(g), np.asarray(w), equal_nan=True) and np.asarray(g).dtype == np.asarray(w).dtype


def test_cabi_entry_points_are_declared():
    import ctypes as C
    from pyimsegm_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip('the library is not built')
    handle = C.CDLL(_lib.LIB_PATH)
    f = handle.isb_contingency_workspace_bytes
    f.restype, f.argtypes = C.c_size_t, [C.c_int, C.c_int]
    assert f(0, 0) > 0 and f(2, 0) == 0        # float32 maps are not label maps
    assert f(8, 8) > f(0, 0)                   # 64-bit maps reserve the 2^26-value presence table
