"""CPU tests of the tree and forest fit (pyimsegm_b200/forest_fit.py) and of its oracle (oracle/forest.py): the oracle passes its own
optimality checker, the checker accepts scikit-learn's trees and rejects a perturbed one, one-feature forests equal scikit-learn's
node for node, the bootstrap and every root are scikit-learn's, and the fitted objects behave as scikit-learn's.  The oracle stands in
for the device call.  Then the reference's doctests of the classifier half of ``classification``."""
import glob
import os
import pickle

import numpy as np
import pytest
from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
from sklearn.tree import DecisionTreeClassifier
from sklearn.utils.validation import check_is_fitted

from oracle import forest as of
from pyimsegm_b200 import class_models, forest_fit
from pyimsegm_b200 import classification as clf


@pytest.fixture
def oracle_fit(monkeypatch):
    monkeypatch.setattr(forest_fit, '_fit_arrays', of.fit_arrays)


def _data(n, D, K, seed=0, dup=False, const_cols=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    y = (X[:, 0] * K + rng.rand(n) * 0.7).astype(int) % K
    if dup:
        X[n // 2:] = X[:n - n // 2]
        y[n // 2:] = y[:n - n // 2]
    if const_cols:
        X[:, -const_cols:] = 0.5
    return X, y


def _sk_arrays(est):
    """the node arrays of a fitted scikit-learn tree in the oracle's layout"""
    st = est.tree_.__getstate__()
    nodes = st['nodes']
    return dict(left=nodes['left_child'], right=nodes['right_child'], feature=nodes['feature'], threshold=nodes['threshold'],
                impurity=nodes['impurity'], n_node_samples=nodes['n_node_samples'],
                weighted_n_node_samples=nodes['weighted_n_node_samples'])


@pytest.mark.parametrize('case', ['random', 'duplicates', 'constant', 'one_class', 'k64'])
def test_oracle_passes_its_checker(case):
    n, D, K = 400, 6, 3
    kw = {}
    if case == 'duplicates':
        kw['dup'] = True
    if case == 'constant':
        kw['const_cols'] = 3
    if case == 'k64':
        n, K = 640, 64
    X, y = _data(n, D, K, seed=3, **kw)
    if case == 'one_class':
        y[:] = 0
        K = 1
    counts = np.random.RandomState(1).randint(0, 3, n)
    for m, msl, mss, md in ((2, 1, 2, None), (D, 2, 5, None), (3, 9, 3, 4)):
        tree = of.build_tree(X, y, counts, K, 12345, m, mss, msl, md)
        assert of.check_tree(tree, X, y, counts, K, 12345, m, mss, msl, md)
        if case == 'one_class':
            assert tree['node_count'] == 1


def test_checker_accepts_sklearn_trees():
    for seed in range(3):
        X, y = _data(300, 5, 3, seed=seed, dup=seed == 1)
        est = DecisionTreeClassifier(min_samples_leaf=2, min_samples_split=3, random_state=seed).fit(X, y)
        assert of.check_tree(_sk_arrays(est), X, y, np.ones(len(X), int), 3, None, None, 4, 2)


def test_checker_rejects_a_perturbed_threshold():
    X, y = _data(300, 4, 2, seed=5)
    tree = of.build_tree(X, y, np.ones(300, int), 2, 7, 2, 2, 1)
    inner = np.nonzero(tree['left'] >= 0)[0]
    bad = dict(tree, threshold=tree['threshold'].copy())
    i = inner[len(inner) // 2]
    v = np.sort(np.unique(X[:, tree['feature'][i]].astype(np.float32)))
    bad['threshold'][i] = v[np.searchsorted(v, tree['threshold'][i]) - 2] if np.searchsorted(v, tree['threshold'][i]) >= 2 else v[-1]
    with pytest.raises(AssertionError):
        of.check_tree(bad, X, y, np.ones(300, int), 2, 7, 2, 2, 1)


def _same_nodes(a, b):
    na, nb = a.tree_.__getstate__()['nodes'], b.tree_.__getstate__()['nodes']
    assert len(na) == len(nb)
    inner = na['left_child'] >= 0
    for f in na.dtype.names:
        x1, x2 = na[f], nb[f]
        if f == 'missing_go_to_left':       # scikit-learn leaves it uninitialised at leaves
            x1, x2 = x1[inner], x2[inner]
        assert np.array_equal(x1, x2), f
    assert np.array_equal(a.tree_.value, b.tree_.value)
    assert a.tree_.max_depth == b.tree_.max_depth


@pytest.mark.parametrize('seed', [0, 1, 7, 42])
def test_one_feature_forest_is_sklearns(oracle_fit, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(400, 1)
    X[:80] = np.round(X[:80], 1)                # ties
    y = (X[:, 0] + 0.3 * rng.rand(400) > 0.6).astype(int) + (X[:, 0] > 0.85)
    kw = dict(n_estimators=20, min_samples_leaf=2, min_samples_split=3, random_state=seed)
    ref = RandomForestClassifier(**kw).fit(X, y)
    ours = forest_fit.fit_tree_model(RandomForestClassifier(**kw), X, y)
    for a, b in zip(ref.estimators_, ours.estimators_):
        _same_nodes(a, b)
    assert np.array_equal(ref.predict_proba(X), ours.predict_proba(X))


def test_decision_tree_with_every_feature_is_sklearns(oracle_fit):
    X, y = _data(300, 1, 3, seed=2)
    ref = DecisionTreeClassifier(random_state=0).fit(X, y)
    ours = forest_fit.fit_tree_model(DecisionTreeClassifier(random_state=0), X, y)
    _same_nodes(ref, ours)


def test_bootstrap_and_roots_are_sklearns(oracle_fit):
    X, y = _data(500, 7, 3, seed=4)
    kw = dict(n_estimators=6, min_samples_leaf=2, min_samples_split=3, random_state=3)
    ref = RandomForestClassifier(**kw).fit(X, y)
    ours = forest_fit.fit_tree_model(RandomForestClassifier(**kw), X, y)
    for a, b in zip(ref.estimators_samples_, ours.estimators_samples_):
        assert np.array_equal(a, b)
    for a, b in zip(ref.estimators_, ours.estimators_):
        assert a.random_state == b.random_state
        na, nb = a.tree_.__getstate__()['nodes'][0], b.tree_.__getstate__()['nodes'][0]
        for f in ('n_node_samples', 'weighted_n_node_samples', 'impurity'):
            assert na[f] == nb[f], f
        assert np.array_equal(a.tree_.value[0], b.tree_.value[0])


def test_fitted_objects_behave_as_sklearns(oracle_fit):
    X, y = _data(300, 5, 3, seed=6)
    y = np.array(['a', 'b', 'c'])[y]
    for est in (RandomForestClassifier(n_estimators=4, random_state=0), DecisionTreeClassifier(max_depth=4, random_state=1)):
        ref = type(est)(**est.get_params()).fit(X, y)
        fitted = forest_fit.fit_tree_model(est, X, y)
        assert type(fitted) is type(est)
        check_is_fitted(fitted)
        assert sorted(vars(ref)) == sorted(vars(fitted))
        trees = fitted.estimators_ if hasattr(fitted, 'estimators_') else [fitted]
        ref_trees = ref.estimators_ if hasattr(ref, 'estimators_') else [ref]
        for a, b in zip(ref_trees, trees):
            assert sorted(vars(a)) == sorted(vars(b))
            assert repr(a.classes_) == repr(b.classes_) and repr(a.n_classes_) == repr(b.n_classes_)
            assert a.max_features_ == b.max_features_
        again = pickle.loads(pickle.dumps(fitted))
        assert np.array_equal(again.predict_proba(X), fitted.predict_proba(X))
        assert np.array_equal(fitted.classes_, ref.classes_)
        assert class_models.compile_model(fitted) is not None


def test_predict_proba_is_the_leaf_class_fractions(monkeypatch):
    X, y = _data(400, 5, 3, seed=8)
    built = []

    def recording(*args):
        built.extend(of.fit_arrays(*args))
        return built[-len(args[3]):]
    monkeypatch.setattr(forest_fit, '_fit_arrays', recording)
    X32 = X.astype(np.float32)
    for est in (DecisionTreeClassifier(min_samples_leaf=3, random_state=2), RandomForestClassifier(n_estimators=3, random_state=5)):
        del built[:]
        fitted = forest_fit.fit_tree_model(est, X, y)
        trees = fitted.estimators_ if hasattr(fitted, 'estimators_') else [fitted]
        assert len(trees) == len(built)
        for tree, arrays in zip(trees, built):
            leaf = tree.apply(X32)
            # the leaf a row reaches by the stored thresholds, in the builder's preorder ids, and its class counts / weight
            node = np.zeros(len(X32), dtype=np.int64)
            for _ in range(arrays['n_levels']):
                inner = arrays['left'][node] >= 0
                go_left = X32[np.arange(len(X32)), np.maximum(arrays['feature'][node], 0)].astype(np.float64) <= arrays['threshold'][node]
                node = np.where(inner, np.where(go_left, arrays['left'][node], arrays['right'][node]), node)
            assert np.array_equal(leaf, node)
            expect = arrays['class_counts'][node] / arrays['weighted_n_node_samples'][node][:, None]
            assert np.array_equal(tree.predict_proba(X32), expect)
        if len(trees) > 1:
            assert np.allclose(fitted.predict_proba(X32), np.mean([t.predict_proba(X32) for t in trees], axis=0), rtol=0, atol=1e-15)


@pytest.mark.parametrize('params', [dict(criterion='entropy'), dict(class_weight='balanced'), dict(max_leaf_nodes=8),
                                    dict(ccp_alpha=0.1), dict(min_weight_fraction_leaf=0.1), dict(max_samples=0.5), dict(oob_score=True),
                                    dict(warm_start=True), dict(monotonic_cst=[1, 0, 0])])
def test_unsupported_parameters_give_none(params):
    X, y = _data(100, 3, 2)
    assert forest_fit.fit_tree_model(RandomForestClassifier(**params), X, y) is None


def test_unsupported_inputs_give_none():
    X, y = _data(100, 3, 2)
    assert forest_fit.fit_tree_model(DecisionTreeClassifier(splitter='random'), X, y) is None
    assert forest_fit.fit_tree_model(ExtraTreesClassifier(), X, y) is None
    Xn = X.copy()
    Xn[0, 0] = np.nan
    assert forest_fit.fit_tree_model(DecisionTreeClassifier(), Xn, y) is None
    assert forest_fit.fit_tree_model(DecisionTreeClassifier(), X * 1e39, y) is None      # inf as float32
    assert forest_fit.fit_tree_model(DecisionTreeClassifier(), np.repeat(X, 1, 0)[:65 * 2], np.arange(130) % 65) is None
    assert forest_fit.fit_tree_model(DecisionTreeClassifier(), X, np.stack([y, y], 1)) is None


# ---- the reference's doctests ----

def test_create_classifiers_and_grids():
    classifs = clf.create_classifiers()
    assert sorted(classifs) == ['AdaBoost', 'DecTree', 'GradBoost', 'KNN', 'LogistRegr', 'RandForest', 'SVM']
    assert sum(isinstance(clf.create_clf_param_search_grid(k), dict) for k in classifs) == 7
    assert sum(isinstance(clf.create_clf_param_search_distrib(k), dict) for k in classifs) == 7
    assert all(len(clf.create_clf_param_search_grid(k)) > 0 for k in classifs)
    assert all(len(clf.create_clf_param_search_distrib(k)) > 0 for k in classifs)
    assert clf.create_clf_param_search_grid('none') == {}
    assert clf.create_clf_param_search_distrib('none') == {}
    assert repr(clf.create_clf_pipeline()).startswith('Pipeline(')
    assert repr(clf.create_clf_param_search_grid('RandForest')).startswith("{'classif__")
    rf = classifs['RandForest'].get_params()
    assert (rf['n_estimators'], rf['min_samples_leaf'], rf['min_samples_split']) == (20, 2, 3)


def test_search_params_cut_down_max_nb_iter():
    params = clf.create_clf_param_search_grid(clf.DEFAULT_CLASSIF_NAME)
    assert clf.search_params_cut_down_max_nb_iter(params, 100) == 100
    assert clf.search_params_cut_down_max_nb_iter(params, 1e6) == 1450
    assert clf.search_params_cut_down_max_nb_iter(clf.create_clf_param_search_distrib(), 7) == 7


def test_save_and_load_classifier(tmp_path):
    p_clf = clf.save_classifier(str(tmp_path), clf.create_classifiers()['RandForest'], 'TESTINNG', {})
    assert os.path.basename(p_clf) == 'classifier_TESTINNG.pkl'
    d_clf = clf.load_classifier(p_clf)
    assert sorted(d_clf) == ['clf_pipeline', 'features', 'label_names', 'name', 'params']
    assert repr(d_clf['clf_pipeline']).startswith('RandomForestClassifier(')
    assert d_clf['name'] == 'TESTINNG'
    assert clf.load_classifier('none.abc') is None
    with pytest.raises(FileNotFoundError):
        clf.save_classifier(str(tmp_path / 'missing'), None, 'x', {})


def _doctest_data():
    np.random.seed(0)
    lbs = np.random.randint(0, 3, 150)
    fts = np.random.random((150, 5)) + np.tile(lbs, (5, 1)).T
    return fts, lbs


def test_train_export_logistic_regression():
    fts, lbs = _doctest_data()
    model, path = clf.create_classif_search_train_export('LogistRegr', fts, lbs, nb_search_iter=0)
    assert repr(model).startswith('Pipeline(') and path is None
    assert model.predict(fts).shape == (150, )


def test_train_export_adaboost_grid_search(capsys):
    fts, lbs = _doctest_data()
    model, path = clf.create_classif_search_train_export('AdaBoost', fts, lbs, nb_search_iter=2, path_out='', search_type='grid',
                                                         nb_workers=1)
    assert 'Fitting ' in capsys.readouterr().out
    assert repr(model).startswith('Pipeline(') and path == ''


def test_train_export_random_forest_random_search(oracle_fit, tmp_path, capsys):
    fts, lbs = _doctest_data()
    model, path = clf.create_classif_search_train_export('RandForest', fts, lbs, nb_search_iter=2, path_out=str(tmp_path),
                                                         search_type='random', nb_workers=1)
    assert 'Fitting ' in capsys.readouterr().out
    assert repr(model).startswith('Pipeline(')
    assert os.path.basename(path) == 'classifier_RandForest.pkl'
    files = sorted(os.path.basename(p) for p in glob.glob(os.path.join(str(tmp_path), 'classif_*.txt')))
    assert files == ['classif_RandForest_search_params_best.txt', 'classif_RandForest_search_params_scores.txt']
    assert type(model.steps[-1][1]) is RandomForestClassifier
    loaded = clf.load_classifier(path)['clf_pipeline']
    # n_jobs=-1: scikit-learn adds the trees' probabilities from threads, in any order
    assert np.allclose(loaded.predict_proba(fts), model.predict_proba(fts), rtol=0, atol=1e-12)
    assert (model.predict(fts) == lbs).mean() > 0.9


def test_train_export_fits_trees_through_the_device_call(monkeypatch):
    fts, lbs = _doctest_data()
    calls = []

    def fake(*args):
        calls.append(args[3].shape)
        return of.fit_arrays(*args)
    monkeypatch.setattr(forest_fit, '_fit_arrays', fake)
    np.random.seed(1)
    model, _ = clf.create_classif_search_train_export('RandForest', fts, lbs, nb_search_iter=0)
    assert calls == [(20, 150)]
    Xt = model[:-1].transform(fts)
    assert model.steps[-1][1].n_features_in_ == Xt.shape[1]
    # the scaler and PCA are scikit-learn's own fit
    ref = clf.create_clf_pipeline('RandForest', 0.98)
    ref.steps[-1] = ('classif', DecisionTreeClassifier())
    ref.fit(np.nan_to_num(fts), lbs)
    assert np.array_equal(ref[:-1].transform(fts), Xt)
    model2, _ = clf.create_classif_search_train_export('KNN', fts, lbs, nb_search_iter=0)
    assert calls == [(20, 150)]
