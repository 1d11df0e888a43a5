"""CPU tests of the feature scoring: ``forest_fit.fit_extra_trees`` with the device call replaced by scikit-learn's own extra trees
(tests/extra_trees_reference.py) -- the per-tree seeds and splitter states, the assembled forest against ``ExtraTreesClassifier.fit``
-- and ``classification.feature_scoring_selection`` against the reference's outputs (tests/golden/feature_scoring_reference.npz),
the C argument errors of ``isb_extra_trees_fit`` and ``create_pipeline_neuron_net``."""
import ctypes as C
import io
import json
import os
import pickle
import warnings

import numpy as np
import pandas as pd
import pytest
from sklearn.base import clone
from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
from sklearn.linear_model import LogisticRegression
from sklearn.neural_network import BernoulliRBM
from sklearn.pipeline import Pipeline

from extra_trees_reference import forest_arrays
from pyimsegm_b200 import classification, forest_fit

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'feature_scoring_reference.npz')


def _data(n=300, D=6, K=3, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.normal(size=(n, D))
    y = (X[:, 0] + 0.5 * X[:, 1] + rng.normal(scale=0.5, size=n) > 0).astype(int) + (X[:, 2] > 1).astype(int) * (K - 2)
    return X, y


class SklearnDevice(object):
    """stands in for _fit_arrays_extra: scikit-learn fits the same forest, and the call's arguments are recorded"""

    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(forest_fit, '_fit_arrays_extra', self)

    def __call__(self, X, y, K, counts, states, *params, **kw):
        self.calls.append(dict(X=X, y=y, K=K, counts=counts, states=states, params=params))
        return forest_arrays(self.reference)


def _fit_both(monkeypatch, X, y, **params):
    device = SklearnDevice(monkeypatch)
    est = ExtraTreesClassifier(**params)
    device.reference = clone(est).fit(X, y)
    return forest_fit.fit_extra_trees(est, X, y), device


def test_seeds_and_splitter_states_are_sklearns(monkeypatch):
    X, y = _data()
    fitted, device = _fit_both(monkeypatch, X, y, n_estimators=7, random_state=3, bootstrap=True)
    call, ref = device.calls[0], device.reference
    seeds = [e.random_state for e in ref.estimators_]
    assert [e.random_state for e in fitted.estimators_] == seeds
    assert call['states'].dtype == np.uint32
    assert call['states'].tolist() == [np.random.RandomState(s).randint(0, 2 ** 31 - 1) for s in seeds]
    for t, s in enumerate(seeds):                      # _generate_sample_indices from each tree's seed
        want = np.bincount(np.random.RandomState(s).randint(0, len(X), len(X)), minlength=len(X))
        assert np.array_equal(call['counts'][t], want)
    assert call['X'].dtype == np.float32 and call['K'] == 3
    mf, mss, msl, md, mid = call['params']
    assert (mf, mss, msl, md, mid) == (2, 2, 1, -1, 0.0)


@pytest.mark.parametrize('params', [dict(n_estimators=10, random_state=0), dict(n_estimators=5, random_state=1, bootstrap=True),
                                    dict(n_estimators=4, random_state=2, max_features=None, min_samples_leaf=3),
                                    dict(n_estimators=3, random_state=5, max_depth=4, min_samples_split=0.05)])
def test_assembled_forest_is_sklearns(monkeypatch, params):
    X, y = _data(K=3)
    fitted, device = _fit_both(monkeypatch, X, y, **params)
    ref = device.reference
    assert type(fitted) is ExtraTreesClassifier
    assert np.array_equal(fitted.feature_importances_, ref.feature_importances_)
    assert fitted.feature_importances_.tobytes() == ref.feature_importances_.tobytes()
    assert np.array_equal(fitted.predict_proba(X), ref.predict_proba(X))
    assert np.array_equal(fitted.classes_, ref.classes_)
    assert sorted(k for k in vars(ref) if k.endswith('_') and not k.startswith('_')) == \
        sorted(k for k in vars(fitted) if k.endswith('_') and not k.startswith('_'))
    again = pickle.loads(pickle.dumps(fitted))
    assert np.array_equal(again.predict_proba(X), ref.predict_proba(X))


def test_random_state_none_draws_from_the_global_rng(monkeypatch):
    X, y = _data()
    device = SklearnDevice(monkeypatch)
    np.random.seed(11)
    device.reference = ExtraTreesClassifier(n_estimators=4).fit(X, y)
    np.random.seed(11)
    fitted = forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=4), X, y)
    assert [e.random_state for e in fitted.estimators_] == [e.random_state for e in device.reference.estimators_]


@pytest.mark.parametrize('params', [dict(criterion='entropy'), dict(criterion='log_loss'), dict(class_weight='balanced'),
                                    dict(max_leaf_nodes=8), dict(ccp_alpha=0.01), dict(min_weight_fraction_leaf=0.1),
                                    dict(bootstrap=True, max_samples=0.5), dict(bootstrap=True, oob_score=True),
                                    dict(warm_start=True), dict(monotonic_cst=[0, 0, 0, 0, 0, 0])])
def test_unsupported_parameters_give_none(monkeypatch, params):
    monkeypatch.setattr(forest_fit, '_fit_arrays_extra', None)      # never reached
    X, y = _data()
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2, **params), X, y) is None


def test_unsupported_estimators_and_inputs_give_none(monkeypatch):
    monkeypatch.setattr(forest_fit, '_fit_arrays_extra', None)
    X, y = _data()
    assert forest_fit.fit_extra_trees(RandomForestClassifier(n_estimators=2), X, y) is None
    bad = X.copy()
    bad[3, 1] = np.inf
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2), bad, y) is None
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2), X * 1e300, y) is None   # not finite as float32
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2), X[:65], np.arange(65)) is None
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2), X, np.stack([y, y], 1)) is None
    assert forest_fit.fit_extra_trees(ExtraTreesClassifier(n_estimators=2, max_features=7), X, y) is None
    # the exact-split routes keep refusing extra trees
    assert forest_fit.fit_tree_model(ExtraTreesClassifier(n_estimators=2), X, y) is None


def test_chunks_are_whole_trees_within_the_budget():
    assert forest_fit._extra_chunks(10, 100, 2, 1000, 1e12) == [(0, 10)]
    per_tree = 1000 + 4 * 100 + 4 + 199 * (16 + 24 + 1 + 8)
    assert forest_fit._extra_chunks(10, 100, 2, 1000, 3 * per_tree) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert forest_fit._extra_chunks(3, 100, 2, 1000, 1) == [(0, 1), (1, 2), (2, 3)]


# ---- feature_scoring_selection against the reference's outputs ----

def _golden():
    data = np.load(GOLDEN)
    return data, json.loads(str(data['meta']))


CASES = [c['name'] for c in _golden()[1]]


@pytest.mark.parametrize('name', CASES)
def test_feature_scoring_equals_the_reference(monkeypatch, tmp_path, name):
    data, meta = _golden()
    case = next(c for c in meta if c['name'] == name)
    fts, lbs = data[name + '/features'], data[name + '/labels']
    device = SklearnDevice(monkeypatch)
    device.reference = ExtraTreesClassifier(n_estimators=125, random_state=0).fit(fts, lbs)
    args = (fts.tolist(), lbs.tolist()) if case['as_lists'] else (fts, lbs)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        indices, df = classification.feature_scoring_selection(*args, names=case['names'], path_out=str(tmp_path))
    assert len(device.calls) == 1
    assert np.array_equal(indices, data[name + '/indices'])
    assert list(df.columns) == case['columns']
    assert [str(i) for i in df.index] == case['index'] and df.index.name == case['index_name']
    want = data[name + '/values']
    got = df.to_numpy(dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
    # the reference's CSV has 12 digits (its package sets numpy's legacy printing); the columns, labels and values are the same
    csv = pd.read_csv(tmp_path / classification.NAME_CSV_FEATURES_SELECT, index_col=0, dtype={'feature': str})
    ref = pd.read_csv(io.StringIO(case['csv']), index_col=0, dtype={'feature': str})
    assert list(csv.columns) == list(ref.columns) and list(csv.index) == list(ref.index) and csv.index.name == ref.index.name
    assert np.allclose(csv.to_numpy(), ref.to_numpy(), rtol=1e-10, atol=0, equal_nan=True)


def test_feature_scoring_names_and_no_file(monkeypatch, tmp_path):
    X, y = _data(D=4)
    device = SklearnDevice(monkeypatch)
    device.reference = ExtraTreesClassifier(n_estimators=125, random_state=0).fit(X, y)
    _, df = classification.feature_scoring_selection(X, y, names=['a', 'b', 'c', 'd', 'e'], path_out=str(tmp_path / 'missing'))
    assert list(df.index) == ['a', 'b', 'c', 'd']                  # the first D names
    assert not os.path.exists(tmp_path / 'missing')
    _, df = classification.feature_scoring_selection(X, y, names=('a', 'b'))
    assert list(df.index) == ['1', '2', '3', '4']


def test_feature_scoring_fits_non_finite_features_with_sklearn(monkeypatch):
    monkeypatch.setattr(forest_fit, '_fit_arrays_extra', None)      # never reached
    fits = []
    sk_fit = ExtraTreesClassifier.fit

    def recording(self, X, y, **kw):
        fits.append(sk_fit(self, X, y, **kw))
        return fits[-1]
    monkeypatch.setattr(ExtraTreesClassifier, 'fit', recording)
    X, y = _data(D=4)
    X[::7, 1] = np.nan                                 # scikit-learn's extra trees take missing values, its f_regression raises
    with pytest.raises(ValueError):
        classification.feature_scoring_selection(X, y)
    assert len(fits) == 1
    ref = sk_fit(ExtraTreesClassifier(n_estimators=125, random_state=0), X, y)
    assert np.array_equal(fits[0].feature_importances_, ref.feature_importances_)
    X[:, 1] = 0.5
    X[0, 1] = 1e39                                     # finite as float64, infinite as float32: scikit-learn raises, as in the reference
    with pytest.raises(ValueError):
        classification.feature_scoring_selection(X, y)


def test_create_pipeline_neuron_net():
    clf = classification.create_pipeline_neuron_net()
    assert type(clf) is Pipeline and [n for n, _ in clf.steps] == ['rbm', 'logistic']
    rbm, logistic = clf.steps[0][1], clf.steps[1][1]
    assert type(rbm) is BernoulliRBM and type(logistic) is LogisticRegression
    assert (rbm.learning_rate, rbm.n_components, rbm.n_iter, rbm.verbose) == (0.05, 35, 299, False)
    assert not hasattr(rbm, 'components_') and not hasattr(logistic, 'coef_')
    assert logistic.get_params() == LogisticRegression().get_params()


def test_imsegm_classification_has_every_public_name_of_the_reference():
    import imsegm.classification as ic
    for name in ('feature_scoring_selection', 'create_pipeline_neuron_net', 'create_classif_search_train_export',
                 'eval_classif_cross_val_scores', 'eval_classif_cross_val_roc', 'CrossValidateGroups'):
        assert callable(getattr(ic, name))


def test_extra_trees_argument_errors():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    dummy = C.c_void_p(16)

    def call(n=10, D=4, K=2, T=3, m=2, mss=2, msl=1, md=-1, mid=0.0, small=0, cap=19, ptr=dummy, ws=1 << 40):
        return lib.isb_extra_trees_fit(ptr, n, D, dummy, K, dummy, T, dummy, m, mss, msl, md, C.c_double(mid), small, cap,
                                       *[dummy] * 10, dummy, C.c_size_t(ws), None)
    assert call(ptr=None) == _lib.ISB_ERR_ARG
    assert call(m=0) == _lib.ISB_ERR_ARG
    assert call(m=5) == _lib.ISB_ERR_ARG
    assert call(mss=1) == _lib.ISB_ERR_ARG
    assert call(msl=0) == _lib.ISB_ERR_ARG
    assert call(md=-2) == _lib.ISB_ERR_ARG
    assert call(mid=float('nan')) == _lib.ISB_ERR_ARG
    assert call(small=-1) == _lib.ISB_ERR_ARG
    assert call(cap=0) == _lib.ISB_ERR_ARG
    assert call(n=0) == _lib.ISB_ERR_ARG
    assert call(ws=16) == _lib.ISB_ERR_ARG
    assert lib.isb_last_error()
    assert call(K=65) == _lib.ISB_ERR_UNSUPPORTED
    assert call(D=2049, m=2) == _lib.ISB_ERR_UNSUPPORTED
    assert lib.isb_extra_trees_fit_workspace_bytes(10, 4, 3, 65, 2) == 0
    assert lib.isb_extra_trees_fit_workspace_bytes(10, 4, 3, 2, 5) == 0
    assert lib.isb_extra_trees_fit_workspace_bytes(100, 4, 3, 2, 2) >= 3 * 100 * 28
