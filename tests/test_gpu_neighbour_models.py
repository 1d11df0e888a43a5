"""GPU tests of device predict_proba for k-nearest-neighbour and logistic-regression models (isb_knn_predict_proba /
isb_linear_predict_proba): the kernels against the numpy oracle (oracle/neighbours.py) and scikit-learn at their size edges, and the
shared-model pipelines against the host round trip (graph_cuts.USE_DEVICE_PREDICT = False)."""
import numpy as np
import pytest
from sklearn import decomposition, linear_model, neighbors, pipeline, preprocessing

from conftest import synth_regions
from oracle import neighbours as onb

pytestmark = pytest.mark.gpu

FEATS = {'color': ('mean', 'std')}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _clustered(n, d, k, seed):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(-1, 1, (k, d))
    y = rng.randint(0, k, n)
    return centres[y] + rng.normal(0, 0.3, (n, d)), y


def _device_knn(eng, x, fit_x, y, k, n_classes, weights, n_dev=None):
    from pyimsegm_b200.class_models import KNN_WEIGHTS, CompiledModel
    cm = CompiledModel('knn', x.shape[1], x.shape[1], n_classes, None, {'fit_x': fit_x, 'y': y.astype(np.int32)},
                       params={'n_neighbors': k, 'weights': KNN_WEIGHTS[weights]})
    d_n = None if n_dev is None else eng.to_device(np.array([n_dev], dtype=np.int32), 'knn_test_n')
    proba = eng.class_model_predict(eng.to_device(np.ascontiguousarray(x), 'knn_test_x'), cm, d_n=d_n)
    return eng.to_host(proba).copy()


# N_t at 1, k, one training tile (64) +- 1 and 100 000; D from 1 to the feature tables' 232; k 1, 5, 64; N 1, 5 000, 80 000
@pytest.mark.parametrize('N,N_t,D,k', [(5000, 1, 1, 1), (1, 5, 3, 5), (80000, 63, 9, 5), (5000, 65, 189, 64), (1, 64, 232, 64),
                                       (5000, 64, 9, 64), (2000, 100000, 3, 64), (1000, 100000, 9, 5), (1000, 4000, 232, 1),
                                       (80000, 2000, 1, 5)])
def test_knn_kernel_against_oracle(eng, N, N_t, D, k):
    x, _ = _clustered(N, D, 4, seed=N + D)
    fit_x, y = _clustered(N_t, D, 4, seed=N_t + k)
    x[:min(N, N_t, 7)] = fit_x[:min(N, N_t, 7)]             # zero distances
    for weights in ('uniform', 'distance'):
        got = _device_knn(eng, x, fit_x, y, k, 4, weights)
        want = onb.knn_predict_proba(x, fit_x, y, k, 4, weights)
        if weights == 'uniform':
            assert np.array_equal(got, want)
        else:
            assert np.abs(got - want).max() <= 1e-12


def test_knn_reads_only_the_device_row_count(eng):
    x, _ = _clustered(5000, 9, 3, seed=1)
    fit_x, y = _clustered(3000, 9, 3, seed=2)
    full = _device_knn(eng, x, fit_x, y, 5, 3, 'uniform')
    n_dev = 3001
    x2 = x.copy()
    x2[n_dev:] = np.nan                                     # rows past n_dev are not read
    got = _device_knn(eng, x2, fit_x, y, 5, 3, 'uniform', n_dev=n_dev)
    assert np.array_equal(got[:n_dev], full[:n_dev])
    assert np.array_equal(got[:n_dev], onb.knn_predict_proba(x[:n_dev], fit_x, y, 5, 3))


def test_knn_duplicated_rows_lower_index_wins(eng):
    rng = np.random.RandomState(3)
    base = rng.normal(0, 1, (50, 4))
    fit_x = np.vstack([base, base, base])                   # every row three times, with three labels
    y = np.repeat([0, 1, 2], 50)
    x = np.vstack([base, base + rng.normal(0, 1e-3, base.shape)])
    for k in (1, 2, 5):
        want = onb.knn_predict_proba(x, fit_x, y, k, 3)
        assert np.array_equal(_device_knn(eng, x, fit_x, y, k, 3, 'uniform'), want)
        for weights in ('uniform', 'distance'):
            assert np.abs(_device_knn(eng, x, fit_x, y, k, 3, weights) - onb.knn_predict_proba(x, fit_x, y, k, 3, weights)).max() <= 1e-12
    one = _device_knn(eng, x, fit_x, y, 1, 3, 'uniform')
    assert np.array_equal(one[:50], np.tile([1.0, 0.0, 0.0], (50, 1)))    # the first copy (label 0) wins
    zero = _device_knn(eng, base, fit_x, y, 5, 3, 'distance')       # three zero distances, one per label: the indicator weights
    assert np.array_equal(zero, onb.knn_predict_proba(base, fit_x, y, 5, 3, 'distance'))
    assert np.array_equal(zero, np.full((50, 3), 1.0 / 3))


@pytest.mark.parametrize('K', [2, 3, 12])
@pytest.mark.parametrize('D', [9, 189])
def test_linear_against_sklearn(K, D):
    from pyimsegm_b200.class_models import compile_model
    X, y = _clustered(3000, D, K, seed=K * D)
    Xt, _ = _clustered(5000, D, K, seed=5)
    for model in (linear_model.LogisticRegression(max_iter=300),
                  pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('classif', linear_model.LogisticRegression(solver='sag'))])):
        model.fit(X, y)
        cm = compile_model(model)
        assert cm.kind == 'linear'
        assert np.abs(cm.predict_proba(Xt) - model.predict_proba(Xt)).max() <= 1e-12


def create_clf_pipeline(name):
    """the reference's classification.create_clf_pipeline(name) with its default PCA(0.95)"""
    classif = {'KNN': neighbors.KNeighborsClassifier(), 'LogistRegr': linear_model.LogisticRegression(solver='sag')}[name]
    return pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(0.95)), ('classif', classif)])


def _fitted(name, seeds=(101, ), shape=(320, 384)):
    from pyimsegm_b200 import pipelines as pl
    feats, labels = [], []
    for s in seeds:
        img, annot = synth_regions(shape[0], shape[1], seed=s)
        _, f, lab = pl.wrapper_compute_color2d_slic_features_labels((img, np.array([2, 5, 7])[annot]), 16, 0.2, FEATS, 0.9)
        feats.append(f[lab >= 0])
        labels.append(lab[lab >= 0])
    return create_clf_pipeline(name).fit(np.vstack(feats), np.hstack(labels))


class _host_predict(object):
    """graph_cuts.USE_DEVICE_PREDICT = False inside the block"""

    def __enter__(self):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = False

    def __exit__(self, *exc):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = True


def _no_near_ties(model, img):
    from pyimsegm_b200 import pipelines as pl
    _, f = pl.compute_color2d_superpixels_features(img, FEATS, sp_size=16)
    knn = model.steps[-1][1]
    x = model[:-1].transform(np.nan_to_num(f))
    k = knn.n_neighbors
    d2 = np.sort(onb.squared_distances(x, knn._fit_X), axis=1)
    scale = np.sum(x * x, axis=1) + np.max(np.sum(knn._fit_X ** 2, axis=1))
    return bool(np.all(d2[:, k] - d2[:, k - 1] > 1e-9 * scale))


@pytest.fixture(scope='module')
def models():
    return {name: _fitted(name) for name in ('KNN', 'LogistRegr')}


def _test_images():
    return [synth_regions(320, 384, seed=s)[0] for s in (111, 112, 113)]


@pytest.mark.parametrize('name', ['KNN', 'LogistRegr'])
def test_reference_pipeline_matches_host(models, name):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.class_models import compile_model
    model = models[name]
    assert compile_model(model).kind == {'KNN': 'knn', 'LogistRegr': 'linear'}[name]
    for img in _test_images():
        if name == 'KNN':
            assert _no_near_ties(model, img)
        dev = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
        with _host_predict():
            host = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
        assert np.array_equal(dev[0], host[0]) and set(np.unique(dev[0])) <= {2, 5, 7}
        if name == 'KNN':
            assert np.array_equal(dev[1], host[1])
        else:
            assert np.abs(dev[1] - host[1]).max() < 1e-9


@pytest.mark.parametrize('name', ['KNN', 'LogistRegr'])
def test_batch_equals_single_calls(models, name):
    from pyimsegm_b200 import pipelines as pl
    imgs = _test_images()
    single = [pl.segment_color2d_slic_features_model_graphcut(im, models[name], FEATS, sp_size=16) for im in imgs]
    batch = pl.segment_images_batch(imgs, dict_features=FEATS, sp_size=16, model_pipeline=models[name])
    for (s, ss), (b, bs) in zip(single, batch):
        assert np.array_equal(s, b) and np.array_equal(ss, bs)


def test_graph_replay_equals_eager(models):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    imgs = _test_images()
    for model in models.values():
        pl.USE_CUDA_GRAPHS = False
        try:
            eager = pl.segment_images_batch(imgs, dict_features=FEATS, sp_size=16, model_pipeline=model)
            eager_res = [get_engine().to_host(t).copy() for t in pl.segment_resident(get_engine().to_device(imgs[0]), model, FEATS,
                                                                                       sp_size=16)]
        finally:
            pl.USE_CUDA_GRAPHS = True
        n_graphs = sum(isinstance(v, tuple) for v in pl._GRAPHS.values())
        for _ in range(3):
            graph = pl.segment_images_batch(imgs * 2, dict_features=FEATS, sp_size=16, model_pipeline=model)
        d_img = get_engine().to_device(imgs[0], 'image')
        for _ in range(3):
            res = [get_engine().to_host(t).copy() for t in pl.segment_resident(d_img, model, FEATS, sp_size=16)]
        assert sum(isinstance(v, tuple) for v in pl._GRAPHS.values()) > n_graphs, 'no CUDA graph was captured'
        for i, (segm, soft) in enumerate(graph):
            assert np.array_equal(segm, eager[i % len(imgs)][0]) and np.array_equal(soft, eager[i % len(imgs)][1])
        assert np.array_equal(res[0], eager_res[0]) and np.array_equal(res[1], eager_res[1])


@pytest.mark.parametrize('name', ['KNN', 'LogistRegr'])
def test_banded_equals_single_image(models, name):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.tiled import segment_color2d_slic_features_model_graphcut_tiled
    img = synth_regions(600, 448, seed=121)[0]
    segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, models[name], FEATS, sp_size=20, sp_regul=0.2)
    for n_bands in (1, 3):
        got, got_soft, _ = segment_color2d_slic_features_model_graphcut_tiled(img, models[name], FEATS, sp_size=20, sp_regul=0.2,
                                                                              bands_per_rank=n_bands)
        assert np.array_equal(got, segm), n_bands
        if name == 'KNN':
            assert np.array_equal(got_soft, soft), n_bands
        else:
            assert np.abs(got_soft - soft).max() < 1e-9, n_bands
