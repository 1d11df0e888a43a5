"""GPU tests of isb_forest_fit (csrc/forest_fit.cu): every node field bit-identical to the numpy oracle (oracle/forest.py) over sizes,
feature counts, class counts and parameters at their edges; determinism; one-feature forests equal to scikit-learn's; the class limit;
and the supervised path end to end (superpixel features and labels, balanced set, RandForest training, segmentation of held-out
images)."""
import ctypes as C

import numpy as np
import pytest
from sklearn.ensemble import RandomForestClassifier

from conftest import synth_regions
from oracle import forest as of
from pyimsegm_b200 import _lib, forest_fit, pipelines
from pyimsegm_b200 import classification as clf

pytestmark = pytest.mark.gpu

FIELDS = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
          'class_counts')


def _data(n, D, K, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D).astype(np.float32)
    y = ((X[:, 0] * K + rng.rand(n) * 1.5).astype(int) % K) if n else np.zeros(0, int)
    return X, y


def _bootstrap(n, T, seed):
    rng = np.random.RandomState(seed)
    return np.stack([np.bincount(rng.randint(0, n, n), minlength=n) for _ in range(T)])


def _compare(X, y, K, counts, seeds, m, mss=2, msl=1, max_depth=-1, mid=0.0):
    dev = forest_fit._fit_arrays(X, y, K, counts, seeds, m, mss, msl, max_depth, mid)
    ref = of.fit_arrays(X, y, K, counts, seeds, m, mss, msl, max_depth, mid)
    levels = max(r['n_levels'] for r in ref)
    for t, (d, r) in enumerate(zip(dev, ref)):
        assert d['node_count'] == r['node_count'], (t, d['node_count'], r['node_count'])
        for f in FIELDS:
            a, b = np.asarray(d[f]), np.asarray(r[f])
            assert a.dtype.kind == b.dtype.kind or f == 'threshold'
            assert np.array_equal(a.view(np.uint8) if a.dtype == np.float64 else a,
                                  np.ascontiguousarray(b, dtype=a.dtype).view(np.uint8) if a.dtype == np.float64 else b), (t, f)
        assert d['n_levels'] == levels
    return dev


@pytest.mark.parametrize('n', [1, 2, 3, 31, 32, 33, 1000])
def test_sizes(n):
    X, y = _data(n, 9, 2, seed=n)
    _compare(X, y, 2, _bootstrap(n, 3, n), np.array([11, 12, 13]), 3, 3, 2)


def test_forty_thousand_rows():
    X, y = _data(40000, 9, 2, seed=1)
    _compare(X, y, 2, _bootstrap(40000, 2, 5), np.array([1, 2]), 3, 3, 2)


@pytest.mark.parametrize('D,m,T', [(1, 1, 4), (189, 13, 2), (300, 300, 1)])
def test_feature_counts(D, m, T):
    n = 600 if D < 300 else 300
    X, y = _data(n, D, 3, seed=D)
    _compare(X, y, 3, _bootstrap(n, T, D), np.arange(T) + 100, m, 3, 2)


@pytest.mark.parametrize('K', [1, 2, 64])
def test_class_counts(K):
    X, y = _data(2000, 9, K, seed=K)
    if K == 64:
        y = (X[:, 0] * 64).astype(int) % 64
    _compare(X, y, K, _bootstrap(2000, 2, K), np.array([5, 6]), 3)


def test_constant_columns_and_duplicate_rows():
    X, y = _data(800, 12, 3, seed=3)
    X[:, 5:9] = 0.25
    X[400:] = X[:400]
    y[400:] = y[:400]
    _compare(X, y, 3, _bootstrap(800, 3, 1), np.array([7, 8, 9]), 4)
    Xc = np.full((50, 4), 2.0, np.float32)                     # every column constant: one leaf per tree
    dev = _compare(Xc, np.arange(50) % 2, 2, np.ones((2, 50), int), np.array([1, 2]), 2)
    assert all(d['node_count'] == 1 for d in dev)


def test_differences_below_the_feature_threshold():
    rng = np.random.RandomState(4)
    base = np.float32(0.5)
    steps = np.array([np.nextafter(base, np.float32(1))] * 3, np.float32)
    X = (base + rng.randint(0, 40, (600, 3)).astype(np.float32) * np.float32(4e-8)).astype(np.float32)
    X[:, 2] = rng.randint(0, 5, 600) * np.float32(3e-7) + steps[0]
    y = rng.randint(0, 2, 600)
    _compare(X, y, 2, _bootstrap(600, 3, 4), np.array([1, 2, 3]), 2)


def test_signed_zeros_and_extreme_values():
    rng = np.random.RandomState(5)
    vals = np.array([-0.0, 0.0, 3.4e38, -3.4e38, np.finfo(np.float32).max, -np.finfo(np.float32).max, 1e-30, -1e-30], np.float32)
    X = vals[rng.randint(0, len(vals), (500, 4))]
    y = (np.signbit(X[:, 0]) ^ (X[:, 1] > 1)).astype(int)
    y[rng.rand(500) < 0.2] ^= 1
    _compare(X, y, 2, _bootstrap(500, 3, 5), np.array([4, 5, 6]), 2)


@pytest.mark.parametrize('max_depth,msl', [(-1, 1), (-1, 2), (-1, 9), (3, 1), (5, 2)])
def test_depth_and_leaf_size(max_depth, msl):
    X, y = _data(1500, 9, 3, seed=9)
    _compare(X, y, 3, _bootstrap(1500, 3, 9), np.array([21, 22, 23]), 3, max(2, 2 * msl), msl, max_depth)


def test_min_impurity_decrease():
    X, y = _data(1500, 9, 3, seed=10)
    _compare(X, y, 3, _bootstrap(1500, 2, 10), np.array([1, 2]), 3, mid=0.002)


def test_a_tree_of_more_than_64_levels():
    n = 150
    X = np.arange(n, dtype=np.float32)[:, None]
    y = np.arange(n) % 2                                       # alternating classes: every split peels one row off an end
    dev = _compare(X, y, 2, np.ones((1, n), int), np.array([3]), 1)
    assert dev[0]['n_levels'] >= 64


def _parity(k):
    """k binary-code columns and a column g in {0, 1, 2}, y = parity of the bits xor [0, 1, 0][g]: a full-depth tree whose levels
    hold far more leaves than splittable nodes in front of the last splittable ones"""
    n = 3 * 2 ** k
    i = np.arange(n)
    bits = (i[:, None] >> np.arange(k)) & 1
    g = i // 2 ** k
    X = np.concatenate([bits, g[:, None]], axis=1).astype(np.float32)
    y = (bits.sum(1) % 2) ^ np.array([0, 1, 0])[g]
    return X, y


@pytest.mark.parametrize('k', [3, 5, 7])
def test_levels_with_leaves_before_splittable_nodes(k):
    X, y = _parity(k)
    n, D = X.shape
    dev = _compare(X, y, 2, np.ones((1, n), int), np.array([0]), D, 2, 1)
    assert dev[0]['n_levels'] >= k + 2
    # the same through the estimator: DecisionTreeClassifier() as the reference's 'DecTree' creates it, and a forest without bootstrap
    from sklearn.tree import DecisionTreeClassifier
    est = forest_fit.fit_tree_model(DecisionTreeClassifier(random_state=0), X, y)
    assert np.array_equal(est.predict(X), y)
    ref = of.fit_arrays(X, y, 2, np.ones((3, n), int), np.array([1, 2, 3]), 2, 2, 1, -1, 0.0)
    got = forest_fit._fit_arrays(X, y, 2, np.ones((3, n), int), np.array([1, 2, 3]), 2, 2, 1, -1, 0.0)
    for a, b in zip(got, ref):
        for f in FIELDS:
            assert np.array_equal(np.asarray(a[f]), np.asarray(b[f]).astype(np.asarray(a[f]).dtype)), f


@pytest.mark.parametrize('D,m', [(1000, 31), (2048, 45), (2048, 2047)])
def test_candidate_selection_at_wide_feature_rows(D, m):
    X, y = _data(160, D, 3, seed=D + m)
    X[:, 7::9] = 0.5                                           # constant columns among the hashed ones
    _compare(X, y, 3, _bootstrap(160, 2, m), np.array([m, m + 1]), m, 2, 1)


def test_two_runs_are_bit_identical():
    X, y = _data(5000, 20, 3, seed=12)
    counts, seeds = _bootstrap(5000, 5, 12), np.arange(5)
    a = forest_fit._fit_arrays(X, y, 3, counts, seeds, 4, 3, 2, -1, 0.0)
    b = forest_fit._fit_arrays(X, y, 3, counts, seeds, 4, 3, 2, -1, 0.0)
    for ta, tb in zip(a, b):
        for f in FIELDS:
            assert np.array_equal(ta[f], tb[f]), f


@pytest.mark.parametrize('seed', [0, 3])
def test_one_feature_forest_is_sklearns(seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(2000, 1)
    X[:300] = np.round(X[:300], 2)
    y = (X[:, 0] + 0.4 * rng.rand(2000) > 0.6).astype(int) + (X[:, 0] > 0.9)
    kw = dict(n_estimators=20, min_samples_leaf=2, min_samples_split=3, random_state=seed)
    ref = RandomForestClassifier(**kw).fit(X, y)
    ours = forest_fit.fit_tree_model(RandomForestClassifier(**kw), X, y)
    for a, b in zip(ref.estimators_, ours.estimators_):
        na, nb = a.tree_.__getstate__()['nodes'], b.tree_.__getstate__()['nodes']
        assert len(na) == len(nb)
        inner = na['left_child'] >= 0
        for f in na.dtype.names:
            x1, x2 = (na[f][inner], nb[f][inner]) if f == 'missing_go_to_left' else (na[f], nb[f])
            assert np.array_equal(x1, x2), f
        assert np.array_equal(a.tree_.value, b.tree_.value)
    assert np.array_equal(ref.predict_proba(X), ours.predict_proba(X))


def test_more_than_64_classes_is_unsupported():
    import torch
    lib = _lib.lib()
    assert lib.isb_forest_fit_workspace_bytes(100, 4, 1, 65, 2) == 0
    z = torch.zeros(1 << 12, dtype=torch.float64, device='cuda')
    p = _lib.ptr(z)
    levels = C.c_int(0)
    st = lib.isb_forest_fit(p, 100, 4, p, 65, p, 1, p, 2, 2, 1, -1, C.c_double(0.0), 199, p, p, p, p, p, p, p, p, p, p, C.byref(levels),
                            p, C.c_size_t(z.numel() * 8), _lib.stream_ptr())
    assert st == _lib.ISB_ERR_UNSUPPORTED
    assert b'65 classes' in lib.isb_last_error()


class _HostModel(object):
    """the pipeline behind an object compile_model does not know: its predict_proba runs on the host"""

    def __init__(self, model):
        self.model, self.classes_ = model, model.classes_

    def predict_proba(self, x):
        return self.model.predict_proba(x)


def test_supervised_path_end_to_end():
    feats = {'color': ['mean', 'std', 'median']}
    images = [synth_regions(256, 256, n_classes=3, seed=s) for s in range(6)]
    d_fts, d_lbs = {}, {}
    for i, (img, annot) in enumerate(images[:4]):
        _, fts, lbs = pipelines.wrapper_compute_color2d_slic_features_labels((img, annot), 12, 0.2, feats, 0.9)
        d_fts['img%d' % i], d_lbs['img%d' % i] = fts, lbs
    fts, lbs, _ = clf.convert_set_features_labels_2_dataset(d_fts, d_lbs, drop_labels=[-1], balance_type='random')
    np.random.seed(0)
    model, _ = clf.create_classif_search_train_export('RandForest', fts, lbs, nb_search_iter=0, pca_coef=None)
    assert type(model.steps[-1][1]) is RandomForestClassifier
    np.random.seed(0)
    ref = clf.create_clf_pipeline('RandForest', None).fit(fts, lbs)
    acc_dev, acc_ref = [], []
    for img, annot in images[4:]:
        segm, _ = pipelines.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=12, gc_regul=0.)
        segm_h, _ = pipelines.segment_color2d_slic_features_model_graphcut(img, _HostModel(model), feats, sp_size=12, gc_regul=0.)
        assert np.array_equal(segm, segm_h)
        segm_r, _ = pipelines.segment_color2d_slic_features_model_graphcut(img, ref, feats, sp_size=12, gc_regul=0.)
        acc_dev.append(np.mean(segm == annot))
        acc_ref.append(np.mean(segm_r == annot))
    assert abs(np.mean(acc_dev) - np.mean(acc_ref)) <= 0.02, (acc_dev, acc_ref)
    assert np.mean(acc_dev) > 0.8
