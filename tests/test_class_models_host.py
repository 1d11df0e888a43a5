"""CPU tests of the caller-fitted class-model compilation (pyimsegm_b200/class_models.py): the compiled tables, evaluated with numpy
the way the device kernels evaluate them, reproduce scikit-learn; which models are recognised; the snapshot notices a refit; the new
C-ABI entries reject bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
from sklearn import decomposition, ensemble, mixture, pipeline, preprocessing, svm, tree

from pyimsegm_b200 import class_models as cmod

LOG_2PI = 1.8378770664093453


def tables_transform(cm, X):
    """isb_class_transform in numpy"""
    t = cm.tables
    x = np.nan_to_num(np.asarray(X, dtype=np.float64), nan=0.0, posinf=np.inf, neginf=-np.inf)
    if 'sc_mean' in t:
        x = x - t['sc_mean']
    if 'sc_scale' in t:
        x = x / t['sc_scale']
    if 'pca_comp' in t:
        x = x @ t['pca_comp'].T - t['pca_mean']
        if 'pca_scale' in t:
            x = x / t['pca_scale']
    return x


def tables_forest(cm, X):
    """isb_forest_predict_proba in numpy: float32 inputs, `<=` goes left, leaf values added in tree order onto zeros, one division"""
    t = cm.tables
    x = tables_transform(cm, X).astype(np.float32).astype(np.float64)
    out = np.zeros((len(x), cm.n_classes))
    rows = np.arange(len(x))
    for root in t['roots']:
        node = np.full(len(x), root)
        while True:
            inner = t['left'][node] >= 0
            if not inner.any():
                break
            go_left = x[rows, t['feature'][node]] <= t['threshold'][node]
            node = np.where(inner, np.where(go_left, t['left'][node], t['right'][node]), node)
        out += t['value'][node]
    return out / len(t['roots']) if cm.average else out


def tables_weighted_log_prob(cm, X):
    """log w_k + log N(x | k) from the mixture tables: c_k - (D log 2 pi + |x U_k - b_k|^2) / 2"""
    t = cm.tables
    x = tables_transform(cm, X)
    q = np.stack([np.sum((x @ t['prec_chol'][k] - t['bvec'][k]) ** 2, axis=1) for k in range(cm.n_classes)], axis=1)
    return t['log_const'][None] - 0.5 * (x.shape[1] * LOG_2PI + q)


def _data(n, d, k, seed):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0, 1, (k, d))
    y = rng.randint(0, k, n)
    return centres[y] + rng.normal(0, 0.15, (n, d)), y


def _on_thresholds(model, X):
    """rows placed exactly on split thresholds of the first tree (the `<=` tie, after the float32 cast)"""
    est = model.steps[-1][1] if isinstance(model, pipeline.Pipeline) else model
    t0 = (est.estimators_[0] if hasattr(est, 'estimators_') else est).tree_
    inner = np.flatnonzero(t0.children_left >= 0)[:16]
    rows = np.repeat(X[:1], len(inner), axis=0).copy()
    scaler = model.steps[0][1] if isinstance(model, pipeline.Pipeline) else None
    for r, node in enumerate(inner):
        f, thr = t0.feature[node], t0.threshold[node]
        for v in (thr, float(np.float32(thr))):
            rows[r, f] = v * scaler.scale_[f] + scaler.mean_[f] if scaler is not None else v
    return rows


@pytest.mark.parametrize('kind', ['tree', 'forest', 'extra'])
@pytest.mark.parametrize('K,D', [(2, 3), (3, 9), (12, 189), (3, 189)])
@pytest.mark.parametrize('scaled', [False, True])
def test_tree_tables_equal_sklearn_bit_for_bit(kind, K, D, scaled):
    X, y = _data(600, D, K, seed=K * 1000 + D)
    labels = np.array([3, 7, 11] + list(range(20, 20 + K)))[:K]        # non-contiguous classes_
    est = {'tree': tree.DecisionTreeClassifier(random_state=0),
           'forest': ensemble.RandomForestClassifier(n_estimators=20, min_samples_leaf=2, min_samples_split=3, random_state=0),
           'extra': ensemble.ExtraTreesClassifier(n_estimators=20, min_samples_leaf=2, min_samples_split=3, random_state=0)}[kind]
    model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('classif', est)]) if scaled else est
    model.fit(X, labels[y])
    cm = cmod.compile_model(model)
    assert cm is not None and cm.kind == 'forest' and cm.n_classes == K and cm.average == (kind != 'tree')
    assert np.array_equal(cm.classes_, model.classes_) and np.array_equal(cm.classes_, labels)
    Xt, _ = _data(300, D, K, seed=7)
    Xt = np.vstack([Xt, _on_thresholds(model, Xt)])
    assert np.array_equal(tables_forest(cm, Xt), model.predict_proba(Xt))


@pytest.mark.parametrize('cov', ['full', 'tied', 'diag', 'spherical'])
@pytest.mark.parametrize('kind', ['gmm', 'bgm_dp', 'bgm_dd'])
def test_mixture_constants_reproduce_weighted_log_prob(cov, kind):
    X, _ = _data(500, 5, 3, seed=3)
    if kind == 'gmm':
        mm = mixture.GaussianMixture(3, covariance_type=cov, random_state=0)
    else:
        prior = 'dirichlet_process' if kind == 'bgm_dp' else 'dirichlet_distribution'
        mm = mixture.BayesianGaussianMixture(n_components=3, covariance_type=cov, weight_concentration_prior_type=prior, random_state=0)
    model = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()), ('model', mm)]).fit(X)
    cm = cmod.compile_model(model)
    assert cm is not None and cm.kind == 'mixture' and cm.classes_ is None
    Xt = model.steps[0][1].transform(X)
    want = mm._estimate_weighted_log_prob(Xt)
    np.testing.assert_allclose(tables_weighted_log_prob(cm, X), want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize('whiten', [False, True])
@pytest.mark.parametrize('n_comp', [0.95, 4])
def test_pca_transform_tables(whiten, n_comp):
    X, _ = _data(400, 9, 3, seed=4)
    model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(n_comp, whiten=whiten)),
                               ('model', mixture.GaussianMixture(3, random_state=0))]).fit(X)
    cm = cmod.compile_model(model)
    assert cm is not None and cm.n_features_in == 9 and cm.n_dims == model.steps[1][1].n_components_
    want = model[:-1].transform(X)
    got = tables_transform(cm, X)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_scaler_variants_and_nan():
    X, y = _data(300, 4, 3, seed=5)
    for with_mean, with_std in ((True, True), (False, True), (True, False), (False, False)):
        model = pipeline.Pipeline([('s', preprocessing.StandardScaler(with_mean=with_mean, with_std=with_std)),
                                   ('c', tree.DecisionTreeClassifier(random_state=0))]).fit(X, y)
        cm = cmod.compile_model(model)
        assert ('sc_mean' in cm.tables) == with_mean and ('sc_scale' in cm.tables) == with_std
        Xn = X.copy()
        Xn[::7, 1] = np.nan
        assert np.array_equal(tables_forest(cm, Xn), model.predict_proba(np.nan_to_num(Xn)))


def test_supported_and_unsupported_models():
    X, y = _data(200, 3, 3, seed=6)
    sc = preprocessing.StandardScaler
    supported = [mixture.GaussianMixture(3, random_state=0).fit(X),
                 pipeline.Pipeline([('std_scaler', sc()), ('model', mixture.GaussianMixture(3, random_state=0))]).fit(X),
                 pipeline.Pipeline([('scaler', sc()), ('reduce_dim', decomposition.PCA(2)), ('classif', tree.DecisionTreeClassifier())]).fit(X, y),
                 ensemble.RandomForestClassifier(n_estimators=3).fit(X, y)]
    unsupported = [ensemble.GradientBoostingClassifier(n_estimators=3).fit(X, y), ensemble.AdaBoostClassifier(n_estimators=3).fit(X, y),
                   svm.SVC(probability=True).fit(X, y), pipeline.Pipeline([('pca', decomposition.PCA(2)), ('s', sc()),
                                                                            ('m', mixture.GaussianMixture(2))]).fit(X),
                   mixture.GaussianMixture(3),                                           # not fitted
                   mixture.GaussianMixture(9, random_state=0).fit(np.vstack([X] * 4)),  # more components than the device handles
                   ensemble.RandomForestClassifier(n_estimators=2).fit(X, np.stack([y, y], 1)),   # multi-output
                   object(), 'model']

    class WithClasses(object):
        def __init__(self, inner):
            self.inner, self.classes_ = inner, np.array([7, 3, 11])

        def predict_proba(self, x):
            return self.inner.predict_proba(x)

    unsupported.append(WithClasses(supported[1]))
    for m in supported:
        cm = cmod.compile_model(m)
        assert cm is not None, m
        try:
            want = getattr(m, 'classes_', None)
        except AttributeError:
            want = None
        assert (cm.classes_ is None and want is None) or np.array_equal(cm.classes_, want)
    for m in unsupported:
        assert cmod.compile_model(m) is None, m


def test_snapshot_is_reused_and_a_refit_is_noticed():
    X, y = _data(300, 3, 3, seed=8)
    model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                               ('classif', ensemble.RandomForestClassifier(n_estimators=4, random_state=0))]).fit(X, y)
    a = cmod.compile_model(model)
    assert cmod.compile_model(model) is a
    model.fit(X[::-1], (y[::-1] + 1) % 3)
    b = cmod.compile_model(model)
    assert b is not a and b.digest != a.digest
    assert np.array_equal(tables_forest(b, X), model.predict_proba(X))
    gmm = mixture.GaussianMixture(3, random_state=0).fit(X)
    d0 = cmod.compile_model(gmm).digest
    gmm.fit(X * 2)
    assert cmod.compile_model(gmm).digest != d0
    gmm.set_params(covariance_type='diag')       # a parameter change without a refit is noticed too: the factors are not diagonal ones
    assert cmod.compile_model(gmm) is None


def test_shared_model_benchmark_class_map_is_the_images():
    """scripts/bench_shared_model.py trains its forest on synth_classes(seed): it must be the class map behind bench.synth_image(seed)"""
    import bench
    from scripts.bench_shared_model import synth_classes
    img = bench.synth_image(6000, 256, 320)
    cl = synth_classes(6000, 256, 320)
    means = np.linspace(0.2, 0.8, bench.NB_CLASSES)
    assert cl.shape == img.shape[:2] and set(np.unique(cl)) <= set(range(bench.NB_CLASSES))
    assert np.median(np.abs(img[..., 0] - means[cl])) < 0.05


def test_new_cabi_entries_reject_bad_arguments_without_a_gpu():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    err = lambda: lib.isb_last_error().decode()  # noqa: E731
    assert lib.isb_abi_version() == 8
    assert lib.isb_class_transform(None, 4, 3, None, 3, None, None, None, None, None, 3, p, None, 0, None) == _lib.ISB_ERR_ARG
    assert 'null' in err()
    assert lib.isb_class_transform(p, 4, 2, None, 3, None, None, None, None, None, 3, p, None, 0, None) == _lib.ISB_ERR_ARG
    assert 'bad sizes' in err()
    assert lib.isb_class_transform(p, 4, 3, None, 3, None, None, None, None, None, 2, p, None, 0, None) == _lib.ISB_ERR_ARG
    assert lib.isb_class_transform(p, 4, 3, None, 3, None, None, p, p, None, 2, p, p, 8, None) == _lib.ISB_ERR_ARG
    assert 'workspace' in err()
    assert lib.isb_class_transform_workspace_bytes(100, 9, 1) >= 100 * 9 * 8 and lib.isb_class_transform_workspace_bytes(100, 9, 0) == 0
    assert lib.isb_mixture_predict_proba(None, 4, None, 3, 2, p, p, p, p, None, 0, None) == _lib.ISB_ERR_ARG
    assert lib.isb_mixture_predict_proba(p, 0, None, 3, 2, p, p, p, p, None, 0, None) == _lib.ISB_ERR_ARG
    assert lib.isb_mixture_predict_proba(p, 4, None, 233, 2, p, p, p, p, p, 1 << 40, None) == _lib.ISB_ERR_UNSUPPORTED
    assert 'D <=' in err()
    assert lib.isb_mixture_predict_proba(p, 4, None, 3, 9, p, p, p, p, p, 1 << 40, None) == _lib.ISB_ERR_UNSUPPORTED
    assert lib.isb_mixture_predict_proba(p, 100, None, 40, 2, p, p, p, p, p, 8, None) == _lib.ISB_ERR_ARG
    assert 'workspace' in err()
    assert lib.isb_mixture_predict_workspace_bytes(100, 16, 4) == 0 and lib.isb_mixture_predict_workspace_bytes(100, 17, 4) >= 100 * 17 * 4 * 8
    fa = [p, 4, None, 3, 20, p, p, p, p, p, 100, p, 3, 1, p, p, 1 << 20, None]
    for i, bad in ((0, None), (5, None), (14, None), (15, None), (1, 0), (4, 0), (10, 0)):
        args = list(fa)
        args[i] = bad
        assert lib.isb_forest_predict_proba(*args) == _lib.ISB_ERR_ARG, i
    args = list(fa)
    args[12] = 65
    assert lib.isb_forest_predict_proba(*args) == _lib.ISB_ERR_UNSUPPORTED and 'K <=' in err()
    args = list(fa)
    args[16] = 8
    assert lib.isb_forest_predict_proba(*args) == _lib.ISB_ERR_ARG and 'workspace' in err()
    assert lib.isb_forest_predict_workspace_bytes(1000, 20) >= 1000 * 20 * 4
