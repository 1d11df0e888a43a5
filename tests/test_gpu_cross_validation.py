"""GPU tests of the grouped forest fit (isb_forest_fit_groups, forest_fit._fit_arrays_groups) and of the cross-validation it serves:
every node field of every tree bit-identical to the grouped oracle (tests/grouped_forest_oracle.py) over groups that differ in
features, max_features, leaf sizes and training rows; a tree built in a group equal to the tree built alone; a forced split into
chunks equal to one call; cross-validation scores and ROC equal to a per-fold ``fit_tree_model`` loop and, with one feature, to
scikit-learn's route; other classifiers on scikit-learn."""
import warnings

import numpy as np
import pandas as pd
import pytest
from sklearn import pipeline, preprocessing
from sklearn.base import clone
from sklearn.ensemble import RandomForestClassifier
from sklearn.model_selection import cross_val_score

from grouped_forest_oracle import fit_arrays_groups
from pyimsegm_b200 import classification as clf
from pyimsegm_b200 import forest_fit

pytestmark = pytest.mark.gpu

FIELDS = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
          'class_counts')


def _same_tree(a, b, where):
    assert a['node_count'] == b['node_count'], where
    for f in FIELDS:
        x, y = np.asarray(a[f]), np.ascontiguousarray(b[f], dtype=np.asarray(a[f]).dtype)
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (where, f)


def _groups(n, dims, K, trees, seed=0):
    """per group its own features (ties: values on a grid of 16; a constant column), per tree a bootstrap of its group's rows"""
    rng = np.random.RandomState(seed)
    y = rng.randint(0, K, n)
    Xs = []
    for D in dims:
        X = (np.floor(rng.rand(n, D) * 16) / 16 + (y[:, None] % 4) * 0.3 * rng.rand(1, D)).astype(np.float32)
        if D > 2:
            X[:, 1] = 0.5
        Xs.append(X)
    counts, seeds, tree_group = [], [], []
    for g, T in enumerate(trees):
        rows = rng.rand(n) < (0.5 + 0.1 * g)                  # each group's own training rows
        for _ in range(T):
            c = np.bincount(rng.randint(0, n, n), minlength=n) * rows
            c[np.nonzero(rows)[0][0]] += 1
            counts.append(c)
            seeds.append(rng.randint(1 << 31))
            tree_group.append(g)
    return Xs, y, np.array(counts), np.array(seeds), np.array(tree_group)


CASES = {
    'mixed': dict(n=600, dims=[5, 12, 1, 40], K=3, trees=[3, 1, 2, 2], m=[2, 12, 1, 6], mss=[2, 5, 3, 2], msl=[1, 2, 1, 3]),
    'k64': dict(n=3000, dims=[9, 20], K=64, trees=[2, 3], m=[3, 4], mss=[3, 2], msl=[2, 1]),
    'depth': dict(n=800, dims=[7, 3, 30], K=5, trees=[2, 2, 1], m=[7, 1, 5], mss=[2, 10, 4], msl=[1, 3, 2], max_depth=4, mid=1e-3),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_grouped_fit_equals_the_oracle(case):
    c = CASES[case]
    Xs, y, counts, seeds, tg = _groups(c['n'], c['dims'], c['K'], c['trees'], seed=len(case))
    args = (Xs, y, c['K'], counts, seeds, tg, np.array(c['m']), np.array(c['mss']), np.array(c['msl']), c.get('max_depth', -1),
            c.get('mid', 0.0))
    dev = forest_fit._fit_arrays_groups(*args)
    ref = fit_arrays_groups(*args)
    assert len(dev) == len(ref) == len(seeds)
    for t, (d, r) in enumerate(zip(dev, ref)):
        _same_tree(d, r, (case, t))
        assert d['n_levels'] == r['n_levels']
    # each tree equals the same tree built alone by isb_forest_fit
    for t in range(len(seeds)):
        g = tg[t]
        alone = forest_fit._fit_arrays(Xs[g], y, c['K'], counts[t:t + 1], seeds[t:t + 1], c['m'][g], c['mss'][g], c['msl'][g],
                                       c.get('max_depth', -1), c.get('mid', 0.0))
        _same_tree(dev[t], alone[0], (case, 'alone', t))


def test_forced_chunks_equal_one_call(monkeypatch):
    c = CASES['mixed']
    Xs, y, counts, seeds, tg = _groups(c['n'], c['dims'], c['K'], c['trees'], seed=3)
    args = (Xs, y, c['K'], counts, seeds, tg, np.array(c['m']), np.array(c['mss']), np.array(c['msl']), -1, 0.0)
    one = forest_fit._fit_arrays_groups(*args)
    monkeypatch.setattr(forest_fit, 'GROUP_MAX_TREES', 3)
    calls = []
    real = forest_fit._lib.check

    def counting(rc):
        calls.append(rc)
        return real(rc)
    monkeypatch.setattr(forest_fit._lib, 'check', counting)
    chunked = forest_fit._fit_arrays_groups(*args)
    assert len(calls) == 3                                  # groups of 3, 1 + 2 and 2 trees
    for t, (a, b) in enumerate(zip(one, chunked)):
        _same_tree(a, b, t)


# ---- cross-validation ----

def _per_fold_fits(classif, features, labels, fold_lists, catch=True):
    """the per-fold route: every fold's pipeline fitted by classification._fit_pipeline (one fit_tree_model call per fold)"""
    out = []
    for folds in fold_lists:
        models = []
        for train, _ in folds:
            model = clone(classif)
            if type(model) is pipeline.Pipeline:
                model = clf._fit_pipeline(model, features[train], labels[train])
            else:
                model = forest_fit.fit_tree_model(model, features[train], labels[train])
            models.append(model)
        out.append(models)
    return out


def _superpixel_like(n_groups=8, per=120, D=12, seed=0):
    rng = np.random.RandomState(seed)
    labels = rng.randint(0, 3, n_groups * per)
    feats = rng.randn(n_groups * per, D) + labels[:, None] * rng.rand(1, D) * 1.5
    return feats, labels, [per] * n_groups


@pytest.mark.parametrize('pca', [None, 0.95])
def test_grouped_equals_per_fold(monkeypatch, pca):
    feats, labels, sizes = _superpixel_like()
    # one thread for predict_proba: with n_jobs=-1 scikit-learn adds the trees' probabilities in thread order, which moves the ROC
    classif = clf.create_clf_pipeline('RandForest', pca).set_params(classif__n_jobs=1)
    cv = clf.CrossValidateGroups(sizes, 2)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        np.random.seed(11)
        df = clf.eval_classif_cross_val_scores('RandForest', classif, feats, labels, cross_val=cv)
        roc, auc = clf.eval_classif_cross_val_roc('RandForest', classif, feats, labels, cv)
        monkeypatch.setattr(clf, '_fit_folds', _per_fold_fits)
        np.random.seed(11)
        df_ref = clf.eval_classif_cross_val_scores('RandForest', classif, feats, labels, cross_val=cv)
        roc_ref, auc_ref = clf.eval_classif_cross_val_roc('RandForest', classif, feats, labels, cv)
    assert df.shape == (4, 4)
    pd.testing.assert_frame_equal(df, df_ref, check_exact=True)
    pd.testing.assert_frame_equal(roc, roc_ref, check_exact=True)
    assert auc == auc_ref


def test_one_feature_equals_sklearns_route(monkeypatch):
    feats, labels, sizes = _superpixel_like(D=1, per=60)
    classif = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                 ('classif', RandomForestClassifier(n_estimators=20, min_samples_leaf=2, min_samples_split=3))])
    cv = clf.CrossValidateGroups(sizes, 2)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        np.random.seed(4)
        df = clf.eval_classif_cross_val_scores('RandForest', classif, feats, labels, cross_val=cv)
        roc, auc = clf.eval_classif_cross_val_roc('RandForest', classif, feats, labels, cv)
        monkeypatch.setattr(clf, '_device_folds', lambda c: False)
        np.random.seed(4)
        df_ref = clf.eval_classif_cross_val_scores('RandForest', classif, feats, labels, cross_val=cv)
        roc_ref, auc_ref = clf.eval_classif_cross_val_roc('RandForest', classif, feats, labels, cv)
    pd.testing.assert_frame_equal(df, df_ref, check_exact=True)
    pd.testing.assert_frame_equal(roc, roc_ref, check_exact=True)
    assert auc == auc_ref


@pytest.mark.parametrize('name', ['KNN', 'SVM'])
def test_other_classifiers_stay_on_sklearn(monkeypatch, name):
    feats, labels, sizes = _superpixel_like(n_groups=4, per=40, D=4)

    def no_device(*args):
        raise AssertionError('the device fit must not be called')
    monkeypatch.setattr(forest_fit, '_fit_arrays_groups', no_device)
    classif = clf.create_clf_pipeline(name, None)
    cv = clf.CrossValidateGroups(sizes, 2)
    np.random.seed(0)
    df = clf.eval_classif_cross_val_scores(name, classif, feats, labels, cross_val=cv)
    np.random.seed(0)
    expect = {s: cross_val_score(classif, feats, labels, cv=cv, scoring=s) for s in clf.METRIC_SCORING}
    pd.testing.assert_frame_equal(df, pd.DataFrame(expect), check_exact=True)
