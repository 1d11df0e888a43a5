"""GPU tests of device predict_proba for caller-fitted models (class_models.py, isb_class_transform / isb_mixture_predict_proba /
isb_forest_predict_proba): against scikit-learn directly, and the shared-model pipelines against the host round trip
(graph_cuts.USE_DEVICE_PREDICT = False)."""
import numpy as np
import pytest
from sklearn import decomposition, ensemble, mixture, pipeline, preprocessing, svm, tree

from conftest import synth_regions

pytestmark = pytest.mark.gpu

RF = dict(n_estimators=20, min_samples_leaf=2, min_samples_split=3)     # the reference's RandForest (classification.py:101)


def _data(n, d, k, seed):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0, 1, (k, d))
    y = rng.randint(0, k, n)
    return centres[y] + rng.normal(0, 0.15, (n, d)), y


class _host_predict(object):
    """graph_cuts.USE_DEVICE_PREDICT = False inside the block"""

    def __enter__(self):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = False

    def __exit__(self, *exc):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = True


@pytest.mark.parametrize('kind', ['tree', 'forest', 'extra'])
@pytest.mark.parametrize('K,D', [(2, 3), (12, 9), (3, 189)])
@pytest.mark.parametrize('scaled', [False, True])
def test_device_forest_is_bit_exact(kind, K, D, scaled):
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(800, D, K, seed=K + D)
    est = {'tree': tree.DecisionTreeClassifier(random_state=0), 'forest': ensemble.RandomForestClassifier(random_state=0, **RF),
           'extra': ensemble.ExtraTreesClassifier(random_state=0, **RF)}[kind]
    model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('classif', est)]) if scaled else est
    model.fit(X, np.array([3, 7, 11] + list(range(20, 32)))[:K][y])
    Xt, _ = _data(5000, D, K, seed=99)
    Xt[::13, 0] = np.nan
    got = compile_model(model).predict_proba(Xt)
    assert np.array_equal(got, model.predict_proba(np.nan_to_num(Xt)))


def _mixture(kind, cov, K):
    if kind == 'gmm':
        return mixture.GaussianMixture(K, covariance_type=cov, random_state=0, reg_covar=1e-3, max_iter=20)
    prior = 'dirichlet_process' if kind == 'bgm_dp' else 'dirichlet_distribution'
    return mixture.BayesianGaussianMixture(n_components=K, covariance_type=cov, weight_concentration_prior_type=prior, random_state=0,
                                           reg_covar=1e-3, max_iter=20)


@pytest.mark.parametrize('kind', ['gmm', 'bgm_dp', 'bgm_dd'])
@pytest.mark.parametrize('cov', ['full', 'tied', 'diag', 'spherical'])
@pytest.mark.parametrize('D,K', [(3, 2), (16, 4), (17, 8), (40, 4), (189, 4)])
def test_device_mixture_within_1e9(kind, cov, D, K):
    import warnings
    from pyimsegm_b200.class_models import compile_model
    X, _ = _data(1500, D, K, seed=D * 10 + K)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()), ('model', _mixture(kind, cov, K))]).fit(X)
    got = compile_model(model).predict_proba(X)
    assert np.abs(got - model.predict_proba(X)).max() < 1e-9
    bare = model.steps[-1][1]                              # without the scaler: the mixture on the raw features
    Xs = model.steps[0][1].transform(X)
    assert np.abs(compile_model(bare).predict_proba(Xs) - bare.predict_proba(Xs)).max() < 1e-9


@pytest.mark.parametrize('whiten', [False, True])
@pytest.mark.parametrize('n_comp', [0.9, 5])
@pytest.mark.parametrize('D', [9, 40])
def test_device_pca_pipelines(whiten, n_comp, D):
    from pyimsegm_b200.class_models import compile_model
    from pyimsegm_b200.engine import get_engine
    X, y = _data(1200, D, 3, seed=D)
    gmm = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(n_comp, whiten=whiten)),
                             ('model', mixture.GaussianMixture(3, random_state=0))]).fit(X)
    cm = compile_model(gmm)
    assert np.abs(cm.predict_proba(X) - gmm.predict_proba(X)).max() < 1e-9
    # the transform itself, within 1e-12 of sklearn's relative to the transformed values' scale
    eng = get_engine()
    d_x = eng.to_device(X, 'cm_test_in')
    eng.class_model_predict(d_x, cm)
    xt = eng.to_host(eng.buf('cm_x', (len(X), cm.n_dims), eng.torch.float64)).copy()
    want = gmm[:-1].transform(X)
    assert np.abs(xt - want).max() <= 1e-12 * np.abs(want).max()
    # a forest after PCA: bit-identical wherever the transformed value is not within 1e-9 of a split threshold
    forest = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(n_comp, whiten=whiten)),
                                ('classif', ensemble.RandomForestClassifier(random_state=0, **RF))]).fit(X, y)
    got, ref = compile_model(forest).predict_proba(X), forest.predict_proba(X)
    xt32 = forest[:-1].transform(X).astype(np.float32).astype(np.float64)
    thr = np.concatenate([e.tree_.threshold[e.tree_.children_left >= 0] for e in forest.steps[-1][1].estimators_])
    near = np.zeros(len(X), bool)
    for j in range(xt32.shape[1]):
        ts = np.sort(thr)
        pos = np.clip(np.searchsorted(ts, xt32[:, j]), 1, len(ts) - 1)
        near |= np.minimum(np.abs(ts[pos] - xt32[:, j]), np.abs(ts[pos - 1] - xt32[:, j])) <= 1e-9 * np.maximum(np.abs(xt32[:, j]), 1)
    assert np.array_equal(got[~near], ref[~near])


def _forest_for(img, annot, feats, sp_size):
    from pyimsegm_b200 import pipelines as pl
    _, fts, labels = pl.wrapper_compute_color2d_slic_features_labels((img, annot), sp_size, 0.2, feats, 0.9)
    sel = labels >= 0
    return pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                              ('classif', ensemble.RandomForestClassifier(random_state=0, n_jobs=1, **RF))]).fit(fts[sel], labels[sel] * 4 + 1)


@pytest.mark.parametrize('shape,sp_size', [((384, 512), 16), ((2048, 2048), 29)])
def test_forest_pipeline_bit_identical_to_host(shape, sp_size):
    import bench
    from scripts.bench_shared_model import synth_classes
    from pyimsegm_b200 import pipelines as pl
    img, annot = synth_regions(shape[0], shape[1], seed=12) if shape[0] < 2048 else (bench.synth_image(2), synth_classes(2))
    feats = {'color': ['mean', 'std']}
    model = _forest_for(img, annot, feats, sp_size)
    dev = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=sp_size, sp_regul=0.2)
    with _host_predict():
        host = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=sp_size, sp_regul=0.2)
    assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
    assert set(np.unique(dev[0])) <= {1, 5, 9}                 # classes_ relabel


def test_group_gmm_pipeline_matches_host():
    from pyimsegm_b200 import pipelines as pl
    imgs = [synth_regions(384, 512, seed=s)[0] for s in (51, 52, 53)]
    feats = {'color': ('mean', 'std')}
    model, _ = pl.estim_model_classes_group(imgs, 3, feats, sp_size=16, sp_regul=0.2)
    for img in imgs:
        dev = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16, sp_regul=0.2)
        with _host_predict():
            host = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16, sp_regul=0.2)
        assert np.array_equal(dev[0], host[0])
        assert np.abs(dev[1] - host[1]).max() < 1e-9


def test_config3_shaped_shared_gmm():
    """colour + Leung-Malik statistics (D = 189), a shared 4-class GMM: the large-D device evaluation against the host round trip"""
    import bench
    from pyimsegm_b200 import pipelines as pl
    img = bench.synth_texture_image(78, 192, 256, n_classes=4, cell=32)
    feats = {'color': ('mean', 'std', 'energy'), 'tLM': ('mean', 'std', 'energy')}
    model, list_fts = pl.estim_model_classes_group([img], 4, feats, sp_size=16, sp_regul=0.2)
    assert list_fts[0].shape[1] == 189
    dev = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16, sp_regul=0.2)
    with _host_predict():
        host = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16, sp_regul=0.2)
    assert np.array_equal(dev[0], host[0])
    assert np.abs(dev[1] - host[1]).max() < 1e-9


def test_sklearn_predict_proba_is_not_called_for_supported_models(monkeypatch):
    from pyimsegm_b200 import pipelines as pl
    img, annot = synth_regions(256, 320, seed=61)
    feats = {'color': ['mean']}
    forest = _forest_for(img, annot, feats, 16)
    gmm, _ = pl.estim_model_classes_group([img], 3, feats, sp_size=16, sp_regul=0.2)
    want = {id(m): pl.segment_color2d_slic_features_model_graphcut(img, m, feats, sp_size=16) for m in (forest, gmm)}

    def boom(*a, **k):
        raise AssertionError('sklearn predict_proba was called')

    for m in (forest, gmm):
        monkeypatch.setattr(type(m.steps[-1][1]), 'predict_proba', boom)
        segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, m, feats, sp_size=16)
        assert np.array_equal(segm, want[id(m)][0]) and np.array_equal(soft, want[id(m)][1])
        batch = pl.segment_images_batch([img], dict_features=feats, sp_size=16, model_pipeline=m)
        assert np.array_equal(batch[0][0], segm)
        monkeypatch.undo()


def test_unsupported_models_still_take_the_host_path():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.class_models import compile_model
    img, annot = synth_regions(256, 320, seed=62)
    feats = {'color': ['mean']}
    _, fts, labels = pl.wrapper_compute_color2d_slic_features_labels((img, annot), 16, 0.2, feats, 0.9)
    sel = labels >= 0
    calls = []

    class Counting(object):
        def __init__(self, inner):
            self.inner = inner

        def predict_proba(self, x):
            calls.append(len(x))
            return self.inner.predict_proba(x)

    for m in (ensemble.GradientBoostingClassifier(n_estimators=10, random_state=0).fit(fts[sel], labels[sel]),
              svm.SVC(probability=True, random_state=0).fit(fts[sel], labels[sel])):
        assert compile_model(m) is None
        wrapped = Counting(m)
        segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, wrapped, feats, sp_size=16)
        assert calls, 'the host predict_proba was not called'
        del calls[:]
        slic, f = pl.compute_color2d_superpixels_features(img, feats, sp_size=16)
        np.testing.assert_allclose(soft, m.predict_proba(f)[slic], rtol=1e-6, atol=1e-9)


def test_batch_equals_single_calls_with_relabel():
    from pyimsegm_b200 import pipelines as pl
    imgs = [synth_regions(300, 360, seed=s) for s in (71, 72, 73, 74)]
    feats = {'color': ['mean', 'std']}
    model = _forest_for(imgs[0][0], imgs[0][1], feats, 16)
    single = [pl.segment_color2d_slic_features_model_graphcut(im, model, feats, sp_size=16) for im, _ in imgs]
    batch = pl.segment_images_batch([im for im, _ in imgs], dict_features=feats, sp_size=16, model_pipeline=model)
    for (s, ss), (b, bs) in zip(single, batch):
        assert np.array_equal(s, b) and np.array_equal(ss, bs)
        assert set(np.unique(b)) <= set(model.classes_)


def test_graph_replay_equals_eager_for_compiled_models():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    imgs = [synth_regions(200, 264, seed=s) for s in (81, 82, 83)]
    feats = {'color': ['mean']}
    forest = _forest_for(imgs[0][0], imgs[0][1], feats, 16)
    pl.USE_CUDA_GRAPHS = False
    try:
        eager = pl.segment_images_batch([im for im, _ in imgs], dict_features=feats, sp_size=16, model_pipeline=forest)
        eager_res = [get_engine().to_host(t).copy() for t in pl.segment_resident(get_engine().to_device(imgs[0][0]), forest, feats,
                                                                                   sp_size=16)]
    finally:
        pl.USE_CUDA_GRAPHS = True
    n_graphs = sum(isinstance(v, tuple) for v in pl._GRAPHS.values())
    for _ in range(3):
        graph = pl.segment_images_batch([im for im, _ in imgs] * 2, dict_features=feats, sp_size=16, model_pipeline=forest)
    d_img = get_engine().to_device(imgs[0][0], 'image')
    for _ in range(3):
        res = [get_engine().to_host(t).copy() for t in pl.segment_resident(d_img, forest.predict_proba, feats, sp_size=16)]
    assert sum(isinstance(v, tuple) for v in pl._GRAPHS.values()) > n_graphs, 'no CUDA graph was captured'
    for i, (segm, soft) in enumerate(graph):
        assert np.array_equal(segm, eager[i % len(imgs)][0]) and np.array_equal(soft, eager[i % len(imgs)][1])
    assert np.array_equal(res[0], eager_res[0]) and np.array_equal(res[1], eager_res[1])


def test_refit_in_place_between_calls():
    from pyimsegm_b200 import pipelines as pl
    img, annot = synth_regions(256, 320, seed=91)
    feats = {'color': ['mean']}
    model = _forest_for(img, annot, feats, 16)
    for _ in range(3):                                          # eager, capture, replay with the first parameters
        first = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16)
    _, fts, labels = pl.wrapper_compute_color2d_slic_features_labels((img, annot), 16, 0.2, feats, 0.9)
    sel = labels >= 0
    model.fit(fts[sel], (labels[sel] + 1) % 3)                  # in place: other labels, other trees
    second = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16)
    with _host_predict():
        host = pl.segment_color2d_slic_features_model_graphcut(img, model, feats, sp_size=16)
    assert np.array_equal(second[0], host[0]) and np.array_equal(second[1], host[1])
    assert not np.array_equal(second[0], first[0])
