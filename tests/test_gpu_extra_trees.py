"""GPU tests of ``isb_extra_trees_fit`` (csrc/extra_trees_fit.cu): every node field of every tree bit-identical to scikit-learn
1.9's own ``ExtraTreesClassifier`` trees, through the block path and the warp path, over the parameters and inputs that steer the
draws; chunked calls equal to one call; ``feature_scoring_selection`` equal to the reference's outputs; a device-fitted forest
compiled by ``class_models.compile_model``; and the reference's training sequence (``load_train_classifier``) through
``imsegm.classification``."""
import json
import os
import warnings

import numpy as np
import pytest
from sklearn.base import clone
from sklearn.ensemble import ExtraTreesClassifier

from extra_trees_reference import first_difference, tree_arrays
from pyimsegm_b200 import classification, forest_fit

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'feature_scoring_reference.npz')
#: small_rows of the calls: the default split between the paths, every node but single rows on the block path, and the warp path
#: from 256 rows down
PATHS = [0, 1, 256]


def _device_trees(est, X, y, small_rows=0, budget=None):
    prep = forest_fit._prepare(clone(est), X, y, admit=forest_fit._supported_extra)
    assert prep is not None
    return forest_fit._fit_arrays_extra(prep.X, prep.y, prep.K, prep.counts, forest_fit._rand_r_states(prep.seeds), prep.max_features,
                                        prep.mss, prep.msl, prep.max_depth, prep.mid, budget=budget, small_rows=small_rows)


def _assert_sklearns(X, y, small_rows=0, **params):
    est = ExtraTreesClassifier(**params)
    ref = clone(est).fit(X, y)
    trees = _device_trees(est, X, y, small_rows)
    K = len(ref.classes_)
    assert len(trees) == len(ref.estimators_)
    for t, (got, tree_est) in enumerate(zip(trees, ref.estimators_)):
        diff = first_difference(got, tree_arrays(tree_est, K))
        assert diff is None, 'tree %d: %s' % (t, diff)
    return trees, ref


def _table(n, D, K, seed=0, noise=0.3):
    rng = np.random.RandomState(seed)
    X = rng.normal(size=(n, D)).astype(np.float32)
    score = X[:, 0] + 0.5 * X[:, 1 % D] + rng.normal(scale=noise, size=n)
    y = np.clip(((score - score.min()) / (np.ptp(score) + 1e-9) * K).astype(int), 0, K - 1)
    return X, y


@pytest.mark.parametrize('small_rows', PATHS)
@pytest.mark.parametrize('max_features', [1, 'sqrt', 'log2', None, 0.3])
def test_max_features(max_features, small_rows):
    X, y = _table(400, 12, 3)
    _assert_sklearns(X, y, small_rows, n_estimators=6, random_state=1, max_features=max_features)


@pytest.mark.parametrize('small_rows', PATHS)
@pytest.mark.parametrize('params', [dict(min_samples_split=7, min_samples_leaf=4), dict(min_samples_leaf=25),
                                    dict(min_samples_split=0.1, min_samples_leaf=0.02), dict(max_depth=3),
                                    dict(min_impurity_decrease=0.004), dict(bootstrap=True), dict(bootstrap=True, min_samples_leaf=3)])
def test_tree_parameters(params, small_rows):
    X, y = _table(600, 7, 4, seed=2)
    _assert_sklearns(X, y, small_rows, n_estimators=5, random_state=4, **params)


@pytest.mark.parametrize('small_rows', PATHS)
@pytest.mark.parametrize('K', [2, 64])
def test_class_counts(K, small_rows):
    X, y = _table(1500, 6, K, seed=K)
    y[:K] = np.arange(K)                               # every class present
    _assert_sklearns(X, y, small_rows, n_estimators=4, random_state=0)


def test_one_row_and_an_all_constant_root():
    _assert_sklearns(np.array([[1.0, 2.0]], dtype=np.float32), np.array([3]), n_estimators=3, random_state=0)
    X = np.ones((50, 4), dtype=np.float32)
    y = np.arange(50) % 2
    trees, _ = _assert_sklearns(X, y, n_estimators=3, random_state=0)
    assert all(t['node_count'] == 1 for t in trees)


@pytest.mark.parametrize('small_rows', PATHS)
def test_constant_features_inherited_by_a_subtree(small_rows):
    rng = np.random.RandomState(5)
    n = 800
    X = rng.normal(size=(n, 6)).astype(np.float32)
    y = (X[:, 0] > 0).astype(int) * 2 + (rng.rand(n) > 0.5)
    right = X[:, 0] > 0
    X[right, 1] = 3.0                                  # constant only where feature 0 is positive
    X[right, 2] = -1.0
    X[X[:, 3] > 0.5, 4] = 0.25
    _assert_sklearns(X, y, small_rows, n_estimators=8, random_state=2, max_features=2)


@pytest.mark.parametrize('small_rows', PATHS)
def test_ranges_within_the_constant_threshold_and_ties(small_rows):
    rng = np.random.RandomState(6)
    n = 600
    one, up1, up2 = np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2)), np.float32(1.0) + 2 * np.finfo(np.float32).eps
    X = np.empty((n, 6), dtype=np.float32)
    X[:, 0] = np.where(rng.rand(n) > 0.5, one, up1)    # one ulp apart: constant after the float32 + 1e-7f
    X[:, 1] = np.where(rng.rand(n) > 0.5, one, up2)    # two ulps apart: not constant
    X[:, 2] = np.round(rng.normal(size=n), 1)          # ties
    X[:, 3] = rng.randint(0, 3, n)
    X[:, 4:] = rng.normal(size=(n, 2))
    X[300:] = X[:300]                                  # duplicate rows
    y = (X[:, 2] + X[:, 4] > 0).astype(int) + (X[:, 1] > 1).astype(int)
    _assert_sklearns(X, y, small_rows, n_estimators=6, random_state=3, max_features=None)
    _assert_sklearns(X, y, small_rows, n_estimators=6, random_state=3)


def test_extreme_values():
    rng = np.random.RandomState(7)
    X = rng.normal(size=(500, 4)).astype(np.float32)
    X[:, 0] = np.where(X[:, 0] > 0, 1e38, -1e38)
    X[::5, 1] = 3e38
    X[::7, 2] = -3e38
    y = (X[:, 3] > 0).astype(int) + (X[:, 0] > 0)
    _assert_sklearns(X, y, n_estimators=6, random_state=1, max_features=None)
    _assert_sklearns(X, y, n_estimators=6, random_state=1)


def test_a_tree_of_more_than_1e5_nodes():
    X, y = _table(200000, 8, 4, seed=9, noise=3.0)
    trees, _ = _assert_sklearns(X, y, n_estimators=1, random_state=0)
    assert trees[0]['node_count'] > 100000
    rows = trees[0]['n_node_samples']
    assert (rows > 64).sum() > 100 and (rows <= 64).sum() > 50000      # both paths


def test_more_trees_than_sms():
    import torch
    X, y = _table(300, 5, 3, seed=10)
    T = torch.cuda.get_device_properties(0).multi_processor_count + 37
    _assert_sklearns(X, y, n_estimators=T, random_state=8, bootstrap=True)


def test_chunked_calls_equal_one_call():
    X, y = _table(500, 6, 3, seed=11)
    est = ExtraTreesClassifier(n_estimators=9, random_state=5)
    one = _device_trees(est, X, y)
    from pyimsegm_b200.engine import get_engine
    ws1 = get_engine().lib.isb_extra_trees_fit_workspace_bytes(500, 6, 1, 3, 2)
    per_tree = ws1 + 4 * 500 + 4 + 999 * (16 + 24 + 1 + 12)
    assert len(forest_fit._extra_chunks(9, 500, 3, ws1, 2 * per_tree)) == 5
    chunked = _device_trees(est, X, y, budget=2 * per_tree)
    assert len(chunked) == len(one)
    for a, b in zip(chunked, one):
        assert first_difference(a, b) is None


def test_fit_extra_trees_is_sklearns_fit():
    X, y = _table(700, 9, 3, seed=12)
    y = np.array(['bg', 'cell', 'nucleus'])[y]
    est = forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=20, random_state=0, bootstrap=True), X, y)
    ref = ExtraTreesClassifier(n_estimators=20, random_state=0, bootstrap=True).fit(X, y)
    assert est.feature_importances_.tobytes() == ref.feature_importances_.tobytes()
    assert np.array_equal(est.predict_proba(X), ref.predict_proba(X))
    assert np.array_equal(est.predict(X), ref.predict(X))


def test_compile_model_of_a_device_forest():
    from pyimsegm_b200.class_models import compile_model
    X, y = _table(900, 6, 3, seed=13)
    est = forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=15, random_state=2, max_depth=12), X, y)
    ref = ExtraTreesClassifier(n_estimators=15, random_state=2, max_depth=12).fit(X, y)
    Xt = _table(400, 6, 3, seed=14)[0]
    model = compile_model(est)
    assert model is not None
    got = model.predict_proba(Xt)
    assert np.abs(got - ref.predict_proba(Xt)).max() < 1e-9
    assert np.array_equal(np.argmax(got, axis=1), ref.predict(Xt))


def test_feature_scoring_equals_the_reference(tmp_path):
    data = np.load(GOLDEN)
    meta = json.loads(str(data['meta']))
    for case in meta:
        name = case['name']
        fts, lbs = data[name + '/features'], data[name + '/labels']
        args = (fts.tolist(), lbs.tolist()) if case['as_lists'] else (fts, lbs)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            indices, df = classification.feature_scoring_selection(*args, names=case['names'], path_out=str(tmp_path))
        assert np.array_equal(indices, data[name + '/indices']), name
        want = data[name + '/values']
        got = df.to_numpy(dtype=np.float64)
        assert got[:, 0].tobytes() == want[:, 0].tobytes(), name          # ExtTree: the reference's bits
        assert np.array_equal(got, want, equal_nan=True), name
        assert list(df.columns) == case['columns'] and [str(i) for i in df.index] == case['index']


def test_reference_doctest_numbers():
    from sklearn.datasets import make_classification
    fts, lbs = make_classification(n_samples=250, n_features=5, n_informative=3, n_redundant=0, n_repeated=0, n_classes=2,
                                   random_state=0, shuffle=False)
    indices, df = classification.feature_scoring_selection(fts, lbs)
    assert indices.tolist() == [1, 0, 2, 3, 4]
    assert [round(v, 4) for v in df['ExtTree']] == [0.2485, 0.3308, 0.2216, 0.1064, 0.0926]
    fts[:, 2] = 1
    indices, _ = classification.feature_scoring_selection(fts.tolist(), lbs.tolist())
    assert indices.tolist() == [1, 0, 3, 4, 2]


def test_load_train_classifier_sequence(tmp_path):
    """the four classification calls of the reference's load_train_classifier
    (experiments_segmentation/run_segm_slic_classif_graphcut.py:584-621), in its order and with its arguments"""
    import imsegm.classification as seg_clf
    rng = np.random.RandomState(21)
    sizes = [int(s) for s in rng.randint(40, 80, 8)]
    n = sum(sizes)
    labels = rng.randint(0, 3, n)
    features = rng.normal(size=(n, 9)) + labels[:, None] * np.linspace(0.2, 1.0, 9)
    feature_names = ['color-mean_%d' % i for i in range(9)]
    params = {'path_exp': str(tmp_path), 'classif': 'RandForest', 'pca_coef': None, 'nb_classif_search': 2, 'nb_workers': 1}
    nb_holdout = 2
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        seg_clf.feature_scoring_selection(features, labels, feature_names, path_out=params['path_exp'])
        cv = seg_clf.CrossValidateGroups(sizes, nb_hold_out=nb_holdout)
        classif, path_classif = seg_clf.create_classif_search_train_export(
            params['classif'], features, labels, cross_val=cv, params=params, feature_names=feature_names,
            pca_coef=params['pca_coef'], eval_metric=params.get('classif_metric', 'f1'),
            nb_search_iter=params.get('nb_classif_search', 1), nb_workers=params['nb_workers'], path_out=params['path_exp'])
        params['path_classif'] = path_classif
        cv = seg_clf.CrossValidateGroups(sizes, nb_hold_out=nb_holdout)
        scores = seg_clf.eval_classif_cross_val_scores(params['classif'], classif, features, labels, cross_val=cv,
                                                       path_out=params['path_exp'])
        roc = seg_clf.eval_classif_cross_val_roc(params['classif'], classif, features, labels, cross_val=cv,
                                                 path_out=params['path_exp'])
    assert os.path.isfile(os.path.join(str(tmp_path), seg_clf.NAME_CSV_FEATURES_SELECT))
    assert os.path.isfile(path_classif)
    assert scores is not None and roc is not None
