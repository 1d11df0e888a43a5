"""CPU tests of the cross-validation half of ``classification``: the fold generators against the reference's examples, the scores and
mean ROC of the grouped tree fit against scikit-learn's own route (with the numpy restatement of the grouped device call standing in
for the device), the files they write, and the argument errors of ``isb_forest_fit_groups``."""
import ctypes as C
import os
import warnings

import numpy as np
import pandas as pd
import pytest
from sklearn import pipeline, preprocessing
from sklearn.ensemble import RandomForestClassifier
from sklearn.model_selection import StratifiedKFold
from sklearn.tree import DecisionTreeClassifier

from grouped_forest_oracle import fit_arrays_groups
from pyimsegm_b200 import classification as clf
from pyimsegm_b200 import forest_fit


@pytest.fixture
def grouped_oracle(monkeypatch):
    calls = []

    def fake(*args):
        calls.append(len(args[3]))
        return fit_arrays_groups(*args)
    monkeypatch.setattr(forest_fit, '_fit_arrays_groups', fake)
    return calls


# ---- fold generators: the reference's examples ----

def test_hold_out():
    ho = clf.HoldOut(10, 7, rand_seed=None)
    assert len(ho) == 1
    assert list(ho) == [([0, 1, 2, 3, 4, 5, 6], [7, 8, 9])]
    assert list(clf.HoldOut(10, 7, rand_seed=0)) == [([2, 8, 4, 9, 1, 6, 7], [3, 0, 5])]
    with pytest.raises(ValueError):
        clf.HoldOut(5, 5)


def test_cross_validate():
    cv = clf.CrossValidate(6, 3, rand_seed=False)
    assert cv.indexes == [0, 1, 2, 3, 4, 5] and len(cv) == 2
    assert list(cv) == [([3, 4, 5], [0, 1, 2]), ([0, 1, 2], [3, 4, 5])]
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidate(340, 0.41)] == [(201, 139)] * 3
    cv = clf.CrossValidate(7, 3, rand_seed=0)
    assert list(cv) == [([3, 0, 5, 4], [6, 2, 1]), ([6, 2, 1, 4], [3, 0, 5]), ([1, 3, 0, 5], [4, 6, 2])]
    assert len(cv) == 3 and cv.indexes == [6, 2, 1, 3, 0, 5, 4]
    # reverse mode: more held out than kept
    cv = clf.CrossValidate(7, 5, rand_seed=0)
    assert list(cv) == [([6, 2], [1, 3, 0, 5, 4]), ([1, 3], [6, 2, 0, 5, 4]), ([0, 5], [6, 2, 1, 3, 4]), ([4, 6], [2, 1, 3, 0, 5])]
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidate(340, 0.55)] == [(153, 187)] * 3
    # ignore_overflow: a short last fold dropped, or kept short instead of reusing the first indices
    assert len(clf.CrossValidate(340, 0.33, ignore_overflow=0.0)) == 4
    assert len(clf.CrossValidate(340, 0.33, ignore_overflow=0.05)) == 3
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidate(4651, 0.25, ignore_overflow=0.)] == [(3488, 1163)] * 4
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidate(4651, 0.25, ignore_overflow=1e-2)] == [(3488, 1163)] * 3 + [(3489, 1162)]
    for bad in [(5, 5), (5, 0), (100, 0.01, None, 0.02)]:
        with pytest.raises(ValueError):
            clf.CrossValidate(*bad)


def test_cross_validate_groups():
    cv = clf.CrossValidateGroups([2, 3, 2, 3], 2, rand_seed=False)
    assert cv.set_indexes == [[0, 1], [2, 3, 4], [5, 6], [7, 8, 9]] and len(cv) == 2
    assert list(cv) == [([5, 6, 7, 8, 9], [0, 1, 2, 3, 4]), ([0, 1, 2, 3, 4], [5, 6, 7, 8, 9])]
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidateGroups([7] * 340, 0.41)] == [(1407, 973)] * 3
    cv = clf.CrossValidateGroups([2, 2, 1, 2, 1], 2, rand_seed=0)
    assert cv.set_indexes == [[0, 1], [2, 3], [4], [5, 6], [7]]
    assert list(cv) == [([2, 3, 5, 6, 7], [4, 0, 1]), ([4, 0, 1, 7], [2, 3, 5, 6]), ([0, 1, 2, 3, 5, 6], [7, 4])]
    assert len(cv) == 3 and cv.indexes == [2, 0, 1, 3, 4]
    cv = clf.CrossValidateGroups([2, 2, 1, 2, 1, 1], 4, rand_seed=0)
    assert list(cv) == [([8, 4], [2, 3, 5, 6, 0, 1, 7]), ([2, 3, 5, 6], [8, 4, 0, 1, 7]), ([0, 1, 7], [8, 4, 2, 3, 5, 6])]
    assert [(len(tr), len(ts)) for tr, ts in clf.CrossValidateGroups([7] * 340, 0.55)] == [(1071, 1309)] * 3


def test_seeded_generators_reseed_numpy():
    clf.CrossValidate(50, 10, rand_seed=3)
    a = np.random.rand()
    np.random.seed(3)
    np.random.shuffle(list(range(50)))
    assert np.random.rand() == a


# ---- scores and ROC against scikit-learn's route ----

def _data(n_groups=6, per=12, seed=0):
    """one feature column (the trees are scikit-learn's node for node), three classes, groups of rows; group 0 holds every row of
    class 2, so the fold that holds group 0 out trains without class 2"""
    rng = np.random.RandomState(seed)
    sizes = [per] * n_groups
    labels = rng.randint(0, 2, n_groups * per)
    labels[:per // 2] = 2
    feats = (labels + rng.rand(len(labels)) * 1.6).reshape(-1, 1)
    return feats, labels, sizes


def _sklearn_route(monkeypatch, fn, *args, **kw):
    with monkeypatch.context() as m:
        m.setattr(clf, '_device_folds', lambda classif: False)
        return fn(*args, **kw)


CLASSIFIERS = {
    'forest': lambda: RandomForestClassifier(n_estimators=3, min_samples_leaf=2, min_samples_split=3),
    'tree': lambda: DecisionTreeClassifier(min_samples_leaf=2),
    'scaled_forest': lambda: pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                                ('classif', RandomForestClassifier(n_estimators=3, min_samples_leaf=2))]),
    'scaled_tree': lambda: pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('classif', DecisionTreeClassifier())]),
}


@pytest.mark.parametrize('name', sorted(CLASSIFIERS))
def test_scores_equal_sklearns_route(monkeypatch, grouped_oracle, name):
    feats, labels, sizes = _data()
    for cv in (3, clf.CrossValidateGroups(sizes, 2), StratifiedKFold(3, shuffle=True)):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            np.random.seed(5)
            ours = clf.eval_classif_cross_val_scores(name, CLASSIFIERS[name](), feats, labels, cross_val=cv)
            state = np.random.rand()
            np.random.seed(5)
            ref = _sklearn_route(monkeypatch, clf.eval_classif_cross_val_scores, name, CLASSIFIERS[name](), feats, labels, cross_val=cv)
            assert np.random.rand() == state, 'the global RNG must be consumed as scikit-learn consumes it'
        assert list(ours.columns) == list(clf.METRIC_SCORING)
        pd.testing.assert_frame_equal(ours, ref, check_exact=True)
    # every (scoring, fold) tree of one call in one grouped fit
    assert len(grouped_oracle) == 3


def test_scores_of_two_labels_are_relabelled(monkeypatch, grouped_oracle):
    feats, labels, sizes = _data()
    labels = np.where(labels == 2, 7, 3)
    np.random.seed(1)
    ours = clf.eval_classif_cross_val_scores('x', CLASSIFIERS['forest'](), feats, labels, cross_val=clf.CrossValidateGroups(sizes, 3))
    np.random.seed(1)
    ref = _sklearn_route(monkeypatch, clf.eval_classif_cross_val_scores, 'x', CLASSIFIERS['forest'](), feats, labels,
                         cross_val=clf.CrossValidateGroups(sizes, 3))
    pd.testing.assert_frame_equal(ours, ref, check_exact=True)


def test_a_failing_scoring_leaves_its_column_out(grouped_oracle):
    feats, labels, _ = _data()
    df = clf.eval_classif_cross_val_scores('x', CLASSIFIERS['tree'](), feats, labels, cross_val=3, scorings=('accuracy', 'no-such'))
    assert list(df.columns) == ['accuracy'] and len(df) == 3


@pytest.mark.parametrize('name', sorted(CLASSIFIERS))
def test_roc_equals_sklearns_route(monkeypatch, grouped_oracle, name):
    feats, labels, _ = _data()
    labels[labels == 2] = 0                            # every fold of the ROC must train on every class
    labels[::7] = 2
    cv = StratifiedKFold(4, shuffle=True, random_state=1)
    np.random.seed(2)
    ours, auc = clf.eval_classif_cross_val_roc(name, CLASSIFIERS[name](), feats, labels, cv, nb_steps=21)
    np.random.seed(2)
    ref, auc_ref = _sklearn_route(monkeypatch, clf.eval_classif_cross_val_roc, name, CLASSIFIERS[name](), feats, labels, cv, nb_steps=21)
    pd.testing.assert_frame_equal(ours, ref, check_exact=True)
    assert auc == auc_ref
    assert ours['TP'].iloc[0] == 0 and ours['TP'].iloc[-1] == 1
    assert len(grouped_oracle) == 1


def test_roc_rejects_negative_labels():
    feats, labels, _ = _data()
    with pytest.raises(ValueError):
        clf.eval_classif_cross_val_roc('x', CLASSIFIERS['tree'](), feats, labels - 1, 3)


def test_files(tmp_path, grouped_oracle):
    feats, labels, sizes = _data()
    cv = clf.CrossValidateGroups(sizes, 2)
    clf.eval_classif_cross_val_scores('RandForest', CLASSIFIERS['forest'](), feats, labels, cross_val=cv, path_out=str(tmp_path))
    labels[labels == 2] = 1
    clf.eval_classif_cross_val_roc('RandForest', CLASSIFIERS['forest'](), feats, labels, cv, path_out=str(tmp_path), nb_steps=5)
    assert sorted(os.listdir(str(tmp_path))) == ['classif_RandForest_cross-val_AUC-mean.txt', 'classif_RandForest_cross-val_ROC-mean.csv',
                                                 'classif_RandForest_cross-val_scores-all-folds.csv',
                                                 'classif_RandForest_cross-val_scores-statistic.csv']
    stat = pd.read_csv(str(tmp_path / 'classif_RandForest_cross-val_scores-statistic.csv'), index_col=0)
    assert list(stat.index) == ['count', 'mean', 'std', 'min', '25%', '50%', '75%', 'max']
    with pytest.raises(FileNotFoundError):
        clf.eval_classif_cross_val_scores('x', CLASSIFIERS['tree'](), feats, labels, cross_val=3, path_out=str(tmp_path / 'none'))


# ---- the grouped host fit ----

def test_fit_tree_models_equal_separate_fits(monkeypatch, grouped_oracle):
    from oracle import forest as of
    monkeypatch.setattr(forest_fit, '_fit_arrays', of.fit_arrays)
    rng = np.random.RandomState(4)
    labels = rng.randint(0, 3, 80)
    X1 = rng.rand(80, 4) + labels[:, None]
    X2 = rng.rand(80, 2) + labels[:, None]
    rows = [np.arange(0, 60), np.arange(20, 80), None]
    ests = [RandomForestClassifier(n_estimators=2, max_features=2), DecisionTreeClassifier(min_samples_leaf=0.05),
            RandomForestClassifier(n_estimators=2, criterion='entropy')]          # the last one is scikit-learn's
    np.random.seed(9)
    grouped = forest_fit.fit_tree_models(ests, [X1, X2, X1], labels, rows)
    np.random.seed(9)
    alone = [forest_fit.fit_tree_model(RandomForestClassifier(n_estimators=2, max_features=2), X1[:60], labels[:60]),
             forest_fit.fit_tree_model(DecisionTreeClassifier(min_samples_leaf=0.05), X2[20:], labels[20:]),
             RandomForestClassifier(n_estimators=2, criterion='entropy').fit(X1, labels)]
    assert len(grouped_oracle) == 1
    for a, b in zip(grouped, alone):
        assert np.array_equal(a.predict_proba(X1 if a.n_features_in_ == 4 else X2), b.predict_proba(X1 if b.n_features_in_ == 4 else X2))


def test_group_argument_errors_need_no_device():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()

    def call(D, mf, mss, msl, tree_group, Dmax=4, G=None):
        G = len(D) if G is None else G
        arr = [np.ascontiguousarray(v, dtype=np.int32) for v in (D, mf, mss, msl, tree_group)]
        dummy = C.c_void_p(1)
        return lib.isb_forest_fit_groups(dummy, 10, Dmax, G, *[a.ctypes.data for a in arr[:4]], dummy, 2, dummy, len(tree_group),
                                         arr[4].ctypes.data, dummy, -1, C.c_double(0.0), 19, *[dummy] * 10, None, dummy,
                                         C.c_size_t(1 << 40), None)
    assert call([4, 3], [2, 1], [2, 2], [1, 1], [0, 2]) == _lib.ISB_ERR_ARG           # group index out of range
    assert b'group' in lib.isb_last_error()
    assert call([4, 3], [2, 1], [2, 2], [1, 1], [0, -1]) == _lib.ISB_ERR_ARG
    assert call([4, 3], [2, 4], [2, 2], [1, 1], [0, 1]) == _lib.ISB_ERR_ARG           # m_g > D_g
    assert call([4, 3], [0, 1], [2, 2], [1, 1], [0, 1]) == _lib.ISB_ERR_ARG           # m_g < 1
    assert call([5, 3], [2, 1], [2, 2], [1, 1], [0, 1]) == _lib.ISB_ERR_ARG           # D_g > Dmax
    assert call([4, 3], [2, 1], [1, 2], [1, 1], [0, 1]) == _lib.ISB_ERR_ARG           # min_samples_split < 2
    assert call([4, 3], [2, 1], [2, 2], [1, 0], [0, 1]) == _lib.ISB_ERR_ARG           # min_samples_leaf < 1
    assert call([4], [2], [2], [1], [0], G=0) == _lib.ISB_ERR_ARG
    assert lib.isb_forest_fit_groups_workspace_bytes(100, 8, 2, 4, 65, 2) == 0        # more than 64 classes
    assert lib.isb_forest_fit_groups_workspace_bytes(100, 8, 2, 4, 3, 2) >= lib.isb_forest_fit_workspace_bytes(100, 8, 4, 3, 2) > 0
