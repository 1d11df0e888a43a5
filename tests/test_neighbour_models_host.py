"""CPU tests of the k-nearest-neighbour and logistic-regression compilation (pyimsegm_b200/class_models.py): which models are taken,
what their tables hold, that a refit or a parameter change is noticed, that the numpy oracle (oracle/neighbours.py) reproduces
scikit-learn, and that the two new C-ABI entries reject bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
from sklearn import decomposition, ensemble, linear_model, neighbors, pipeline, preprocessing, svm

from oracle import neighbours as onb
from pyimsegm_b200 import class_models as cmod


def _data(n, d, k, seed):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0, 1, (k, d))
    y = rng.randint(0, k, n)
    return centres[y] + rng.normal(0, 0.15, (n, d)), y


def _transform(cm, X):
    """isb_class_transform in numpy (scaler only, as the accepting tests below need)"""
    x = np.asarray(X, dtype=np.float64)
    if 'sc_mean' in cm.tables:
        x = x - cm.tables['sc_mean']
    if 'sc_scale' in cm.tables:
        x = x / cm.tables['sc_scale']
    return x


def clear_of_ties(x, fit_x, k):
    """queries whose k-th and (k+1)-th squared distances are more than 1e-9 (|x|^2 + max |t|^2) apart: scikit-learn's distances
    (kd-tree or the |x|^2 - 2 x.t + |t|^2 expansion) pick the same k neighbours there"""
    if k >= len(fit_x):
        return np.ones(len(x), bool)
    d2 = np.sort(onb.squared_distances(x, fit_x), axis=1)
    scale = np.sum(x * x, axis=1) + np.max(np.sum(fit_x * fit_x, axis=1))
    return d2[:, k] - d2[:, k - 1] > 1e-9 * scale


def test_accepted_variants():
    X, y = _data(400, 9, 3, seed=1)
    labels = np.array([2, 5, 7])[y]
    sc, pca = preprocessing.StandardScaler, decomposition.PCA
    cases = [(neighbors.KNeighborsClassifier(), 'knn', 9),
             (neighbors.KNeighborsClassifier(7, weights='distance', metric='euclidean'), 'knn', 9),
             (pipeline.Pipeline([('scaler', sc()), ('classif', neighbors.KNeighborsClassifier(64))]), 'knn', 9),
             (pipeline.Pipeline([('scaler', sc()), ('reduce_dim', pca(0.95)), ('classif', neighbors.KNeighborsClassifier())]), 'knn', None),
             (linear_model.LogisticRegression(), 'linear', 9),
             (pipeline.Pipeline([('scaler', sc()), ('reduce_dim', pca(0.95)), ('classif', linear_model.LogisticRegression(solver='sag'))]),
              'linear', None)]
    for model, kind, dims in cases:
        model.fit(X, labels)
        cm = cmod.compile_model(model)
        assert cm is not None and cm.kind == kind, model
        assert cm.n_features_in == 9 and cm.n_classes == 3 and np.array_equal(cm.classes_, [2, 5, 7])
        assert cm.n_dims == (dims if dims is not None else model.steps[1][1].n_components_)
        final = model.steps[-1][1] if isinstance(model, pipeline.Pipeline) else model
        if kind == 'knn':
            assert cm.tables['fit_x'].dtype == np.float64 and np.array_equal(cm.tables['fit_x'], final._fit_X)
            assert cm.tables['y'].dtype == np.int32 and np.array_equal(cm.tables['y'], final._y)
            assert cm.params == {'n_neighbors': final.n_neighbors, 'weights': cmod.KNN_WEIGHTS[final.weights]}
        else:
            assert cm.tables['coef'].shape == (3, cm.n_dims) and cm.tables['intercept'].shape == (3, )
    binary = linear_model.LogisticRegression().fit(X, y % 2)
    cm = cmod.compile_model(binary)
    assert cm.kind == 'linear' and cm.n_classes == 2 and cm.tables['coef'].shape == (1, 9)
    minkowski = neighbors.KNeighborsClassifier(3, metric='minkowski', p=2).fit(X, y)
    assert cmod.compile_model(minkowski).kind == 'knn'


def test_refused_models():
    X, y = _data(300, 4, 3, seed=2)
    knn = neighbors.KNeighborsClassifier
    refused = [knn(weights=lambda d: np.ones_like(d)).fit(X, y), knn(p=1).fit(X, y), knn(metric='cosine').fit(X, y),
               knn(metric_params={'p': 2}).fit(X, y), knn(65).fit(X, y), knn(5).fit(X[:4], y[:4]),
               knn().fit(X, np.stack([y, y], 1)), knn(), linear_model.LogisticRegression(),
               neighbors.RadiusNeighborsClassifier(radius=1.0).fit(X, y),
               ensemble.GradientBoostingClassifier(n_estimators=3).fit(X, y), ensemble.AdaBoostClassifier(n_estimators=3).fit(X, y),
               svm.SVC(probability=True).fit(X, y)]
    for m in refused:
        assert cmod.compile_model(m) is None, m
    assert cmod.compile_model(knn(64).fit(X, y)) is not None


def test_refit_and_set_params_change_the_digest():
    X, y = _data(300, 5, 3, seed=3)
    knn = neighbors.KNeighborsClassifier().fit(X, y)
    a = cmod.compile_model(knn)
    assert cmod.compile_model(knn) is a
    knn.fit(X[::-1] * 2, y[::-1])
    b = cmod.compile_model(knn)
    assert b.digest != a.digest
    knn.set_params(n_neighbors=7)                      # no refit: kneighbors reads n_neighbors at call time
    c = cmod.compile_model(knn)
    assert c.digest != b.digest and c.params['n_neighbors'] == 7
    knn.set_params(weights='distance')
    d = cmod.compile_model(knn)
    assert d.digest != c.digest and d.params['weights'] == 1
    knn.set_params(p=1)                                # not Euclidean any more (and not refitted): the host path
    assert cmod.compile_model(knn) is None
    knn.set_params(p=2)
    assert cmod.compile_model(knn).digest == d.digest
    lr = linear_model.LogisticRegression().fit(X, y)
    e = cmod.compile_model(lr)
    lr.fit(X, (y + 1) % 3)
    assert cmod.compile_model(lr).digest != e.digest


@pytest.mark.parametrize('algorithm', ['auto', 'brute'])
@pytest.mark.parametrize('D,k', [(1, 5), (3, 1), (9, 5), (9, 64), (40, 5)])
def test_oracle_equals_sklearn(algorithm, D, k):
    X, y = _data(2000, D, 4, seed=D * 100 + k)
    Xq, _ = _data(500, D, 4, seed=7)
    Xq[:20] = X[:20]                                   # zero distances
    for weights in ('uniform', 'distance'):
        model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                   ('classif', neighbors.KNeighborsClassifier(k, weights=weights, algorithm=algorithm))]).fit(X, y * 3)
        cm = cmod.compile_model(model)
        xt = _transform(cm, Xq)
        got = onb.knn_predict_proba(xt, cm.tables['fit_x'], cm.tables['y'], k, cm.n_classes, weights)
        want = model.predict_proba(Xq)
        clear = clear_of_ties(xt, cm.tables['fit_x'], k)
        assert clear.mean() > 0.9
        if weights == 'uniform':
            assert np.array_equal(got[clear], want[clear])
            continue
        # 1 / distance carries the relative error of scikit-learn's distances, which its brute-force expansion makes large for
        # near neighbours: compare where those distances are within 1e-14 of the exact ones (every row of the kd-tree)
        dist, _ = model[-1].kneighbors(model[:-1].transform(Xq))
        exact = np.sqrt(onb.kneighbours(xt, cm.tables['fit_x'], k)[0])
        sharp = clear & np.all(np.abs(dist - exact) <= 1e-14 * exact, axis=1)
        if model[-1]._fit_method == 'kd_tree':
            assert sharp[20:].mean() > 0.99 and sharp[:20].all()       # the first 20 rows have zero distances
        assert sharp.any()
        assert np.abs(got[sharp] - want[sharp]).max() <= 1e-12


def test_oracle_ties_and_zero_distances():
    fit_x = np.array([[0.0], [1.0], [1.0], [2.0], [-1.0]])
    y = np.array([0, 1, 2, 0, 1])
    # query 0.0: zero distance at index 0; then (1, idx 1), (1, idx 2), (1, idx 4) tie -- the lower indices win
    d2, idx = onb.kneighbours(np.array([[0.0], [1.0]]), fit_x, 3)
    assert idx.tolist() == [[0, 1, 2], [1, 2, 0]]
    p = onb.knn_predict_proba(np.array([[0.0], [1.0], [0.5]]), fit_x, y, 3, 3, 'distance')
    assert p[0].tolist() == [1.0, 0.0, 0.0]            # the indicator of the zero distances
    assert p[1].tolist() == [0.0, 0.5, 0.5]
    assert np.all(p[2] > 0)


@pytest.mark.parametrize('K', [2, 3, 12])
def test_linear_oracle_equals_sklearn(K):
    X, y = _data(600, 9, K, seed=K)
    model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(0.95)),
                               ('classif', linear_model.LogisticRegression(solver='sag', max_iter=500))]).fit(X, y)
    cm = cmod.compile_model(model)
    xt = model[:-1].transform(X)
    got = onb.linear_predict_proba(xt, cm.tables['coef'], cm.tables['intercept'])
    assert np.abs(got - model.predict_proba(X)).max() <= 1e-12


def test_new_cabi_entries_reject_bad_arguments_without_a_gpu():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    err = lambda: lib.isb_last_error().decode()  # noqa: E731
    big = 1 << 40
    # x, N, n_dev, D, fit_x, N_t, y, k, K, weights, proba, ws, ws_bytes, stream
    fa = [p, 100, None, 9, p, 1000, p, 5, 3, 0, p, p, big, None]
    for i, bad, msg in ((0, None, 'null'), (4, None, 'null'), (6, None, 'null'), (10, None, 'null'), (11, None, 'null'),
                        (1, 0, 'bad sizes'), (3, 0, 'bad sizes'), (5, 0, 'bad sizes'), (8, 0, 'bad sizes'), (7, 0, 'k must'),
                        (7, 65, 'k must'), (8, 65, 'K <='), (9, 2, 'weights'), (12, 8, 'workspace')):
        args = list(fa)
        args[i] = bad
        assert lib.isb_knn_predict_proba(*args) == _lib.ISB_ERR_ARG, i
        assert msg in err(), (i, err())
    args = list(fa)
    args[5], args[7] = 4, 5
    assert lib.isb_knn_predict_proba(*args) == _lib.ISB_ERR_ARG and 'training rows' in err()
    assert lib.isb_knn_predict_workspace_bytes(5000, 40000, 5) >= 5000 * 5 * 12
    assert lib.isb_knn_predict_workspace_bytes(80000, 100000, 64) >= 80000 * 64 * 12
    # x, N, n_dev, D, coef, intercept, n_coef, proba, ws, ws_bytes, stream
    la = [p, 100, None, 9, p, p, 3, p, None, 0, None]
    for i, bad in ((0, None), (4, None), (5, None), (7, None), (1, 0), (3, 0), (6, 0), (6, 65)):
        args = list(la)
        args[i] = bad
        assert lib.isb_linear_predict_proba(*args) == _lib.ISB_ERR_ARG, i
    assert lib.isb_linear_predict_workspace_bytes(100, 3) == 0
    assert lib.isb_abi_version() == 8
