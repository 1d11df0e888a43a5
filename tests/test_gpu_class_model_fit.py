"""GPU tests of the device fit of every estim_model variant and of pca_coef (graph_cuts.class_model_spec, isb_mixture_fit_predict,
isb_pca_fit): BayesianGaussianMixture and PCA against scikit-learn, the pipelines against the device fit of the same features, and
proof that no scikit-learn fit runs."""
import numpy as np
import pytest
from sklearn import decomposition, mixture, preprocessing

from conftest import synth_regions
from oracle.mixture import shared_start_fit

pytestmark = pytest.mark.gpu

VARIANTS = ['GMM', 'GMM_kmeans', 'GMM_Otsu', 'kmeans', 'kmeans_quantiles', 'BGM', 'Otsu']
FEATS = {'color': ['mean', 'std']}


def _blobs(D, K, seed, n=5000):
    """K well separated blobs in D dimensions and a half-informed hard start (as the shared-start GMM parity tests)"""
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0, 1, (K, D))
    y = rng.randint(0, K, n)
    X = centres[y] + rng.normal(0, 0.04 if D <= 16 else 0.15, (n, D))
    y0 = rng.randint(0, K, n)
    y0[:20 * K] = np.repeat(np.arange(K), 20)
    y0[::2] = y[::2]
    return X, y, y0


def _ref_bgm(Z, K, y0, max_iter):
    return shared_start_fit(Z, y0, K, 'BGM', max_iter)


def _check_bgm(bgm, ref):
    assert bgm.n_iter_ == ref.n_iter_ and bgm.converged_ == ref.converged_
    for a, b in zip(bgm.weight_concentration_, ref.weight_concentration_):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-8)
    for name in ('mean_precision_', 'degrees_of_freedom_', 'means_', 'covariances_', 'weights_'):
        np.testing.assert_allclose(getattr(bgm, name), getattr(ref, name), rtol=1e-6, atol=1e-8, err_msg=name)
    np.testing.assert_allclose(bgm.mean_prior_, ref.mean_prior_, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(bgm.covariance_prior_, ref.covariance_prior_, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(bgm.lower_bound_, ref.lower_bound_, rtol=1e-8)


@pytest.mark.parametrize('max_iter', [99, 1])
@pytest.mark.parametrize('D,K', [(3, 3), (16, 8), (40, 3), (189, 4)])
def test_device_bgm_matches_sklearn_from_shared_start(D, K, max_iter):
    from pyimsegm_b200 import graph_cuts as gc
    X, _, y0 = _blobs(D, K, seed=D + K)
    model = gc.estim_class_model_device(X, K, max_iter=max_iter, init_labels=y0, estim_model='BGM')
    assert [n for n, _ in model.steps] == ['std_scaler', 'model']
    bgm = model.named_steps['model']
    assert type(bgm) is mixture.BayesianGaussianMixture
    Z = preprocessing.StandardScaler().fit_transform(X)
    ref = _ref_bgm(Z, K, y0, max_iter)
    _check_bgm(bgm, ref)
    np.testing.assert_allclose(model.predict_proba(X), ref.predict_proba(Z), rtol=1e-5, atol=1e-9)


def _spectrum_data(D, seed, n=6000):
    """features whose scaled covariance has a clearly separated spectrum"""
    rng = np.random.RandomState(seed)
    scales = 0.8 ** np.arange(D) + 0.05
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    X = (rng.normal(size=(n, D)) * scales) @ Q.T
    return X * rng.uniform(0.5, 3, D) + rng.uniform(-2, 2, D)


def _device_pca(X, coef, use_scaler=True):
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    d_x, d_params, dims = eng.pca_fit_transform(eng.to_device(np.ascontiguousarray(X, dtype=np.float64)), use_scaler, coef)
    return eng.to_host(d_x).copy(), gc._pca_from_device(eng.to_host(d_params), X.shape[1], coef), dims


@pytest.mark.parametrize('coef', [0.5, 0.95, 0.98, 2])
@pytest.mark.parametrize('D', [3, 9, 40, 189])
def test_device_pca_matches_sklearn(D, coef):
    X = _spectrum_data(D, seed=D)
    Z = preprocessing.StandardScaler().fit_transform(X)
    ref = decomposition.PCA(coef).fit(Z)
    assert ref._fit_svd_solver == 'covariance_eigh'
    xt, pca, dims = _device_pca(X, coef)
    assert pca.n_components_ == ref.n_components_ == dims
    ev_ref = decomposition.PCA().fit(Z).explained_variance_
    np.testing.assert_allclose(pca.explained_variance_, ref.explained_variance_, rtol=1e-10, atol=1e-13 * ev_ref[0])
    np.testing.assert_allclose(pca.explained_variance_ratio_, ref.explained_variance_ratio_, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(pca.singular_values_, ref.singular_values_, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(pca.mean_, ref.mean_, atol=1e-12)       # both are rounding noise around 0
    np.testing.assert_allclose(pca.noise_variance_, ref.noise_variance_, rtol=1e-9, atol=1e-13)
    np.testing.assert_allclose(pca.components_, ref.components_, atol=1e-9)       # signs included (svd_flip)
    np.testing.assert_allclose(xt, ref.transform(Z), atol=1e-9)
    np.testing.assert_allclose(pca.transform(Z), ref.transform(Z), atol=1e-9)


def test_device_pca_degenerate_columns():
    """a constant column (eigenvalue 0) and two duplicated columns (a second 0): eigenvalues, and the subspace of the kept components"""
    X = _spectrum_data(9, seed=5)
    X = np.concatenate([X, np.full((len(X), 1), 3.5), X[:, :1]], axis=1)
    Z = preprocessing.StandardScaler().fit_transform(X)
    full = decomposition.PCA().fit(Z)
    for coef in (0.95, 11):
        ref = decomposition.PCA(coef).fit(Z)
        _, pca, dims = _device_pca(X, coef)
        assert pca.n_components_ == ref.n_components_ == dims
        np.testing.assert_allclose(pca.explained_variance_, ref.explained_variance_, rtol=1e-10, atol=1e-12 * full.explained_variance_[0])
        keep = ref.explained_variance_ > 1e-8
        C, R = pca.components_[keep], ref.components_[keep]
        np.testing.assert_allclose(C.T @ C, R.T @ R, atol=1e-9)
        np.testing.assert_allclose(np.abs(np.sum(C * R, axis=1)), 1, atol=1e-9)


@pytest.mark.parametrize('kind', ['GMM', 'BGM'])
@pytest.mark.parametrize('D,K', [(9, 3), (40, 3)])
def test_scaler_pca_mixture_matches_sklearn_pipeline(kind, D, K):
    from pyimsegm_b200 import graph_cuts as gc
    X, _, y0 = _blobs(D, K, seed=7 * D)
    model = gc.estim_class_model_device(X, K, init_labels=y0, estim_model=kind, pca_coef=0.95)
    assert [n for n, _ in model.steps] == ['std_scaler', 'reduce_dim', 'model']
    Z = preprocessing.StandardScaler().fit_transform(X)
    pca = decomposition.PCA(0.95).fit(Z)
    P = pca.transform(Z)
    assert model.named_steps['reduce_dim'].n_components_ == pca.n_components_
    mm = model.named_steps['model']
    if kind == 'BGM':
        ref = _ref_bgm(P, K, y0, 99)
        _check_bgm(mm, ref)
    else:
        ref = shared_start_fit(P, y0, K, 'GMM', 99)
        assert mm.n_iter_ == ref.n_iter_ and mm.converged_ == ref.converged_
        np.testing.assert_allclose(mm.means_, ref.means_, rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(mm.lower_bound_, ref.lower_bound_, rtol=1e-8)
    np.testing.assert_allclose(model.predict_proba(X), ref.predict_proba(P), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize('variant,K', [('kmeans', 3), ('kmeans_quantiles', 3), ('Otsu', 2), ('GMM_kmeans', 3), ('GMM_Otsu', 3),
                                       ('BGM', 3)])
def test_variant_iterations_and_purity(variant, K):
    from pyimsegm_b200 import graph_cuts as gc
    X, y, _ = _blobs(3, K, seed=11)
    model = gc.estim_class_model(X, K, variant)
    mm = model.named_steps['model']
    kind, n_init, max_iter = gc.class_model_spec(variant, K)
    assert type(mm) is (mixture.BayesianGaussianMixture if kind == 'BGM' else mixture.GaussianMixture)
    assert (mm.n_init, mm.max_iter) == (n_init, max_iter)
    if max_iter == 1:
        assert mm.n_iter_ == 1 and not mm.converged_
    lab = model.predict_proba(X).argmax(1)
    purity = sum(np.bincount(lab[y == k], minlength=K).max() for k in range(K)) / len(X)
    assert purity > 0.98


@pytest.fixture
def no_sklearn_fit(monkeypatch):
    def boom(*args, **kwargs):
        raise AssertionError('a scikit-learn fit ran on the host')
    for cls in (mixture.GaussianMixture, mixture.BayesianGaussianMixture, decomposition.PCA):
        for name in ('fit', 'fit_predict', 'fit_transform'):
            if hasattr(cls, name):
                monkeypatch.setattr(cls, name, boom)


@pytest.mark.parametrize('pca_coef', [None, 0.95, 2])
def test_every_variant_stays_on_the_device(no_sklearn_fit, pca_coef):
    from pyimsegm_b200 import pipelines as pl
    imgs = [synth_regions(128, 160, seed=s)[0] for s in (31, 32)]
    for v in VARIANTS:
        K = 2 if v == 'Otsu' else 3
        segm, soft = pl.pipe_color2d_slic_features_model_graphcut(imgs[0], K, FEATS, sp_size=10, pca_coef=pca_coef, estim_model=v)
        assert segm.shape == imgs[0].shape[:2] and soft.shape == imgs[0].shape[:2] + (K, )
        out = pl.segment_images_batch(imgs, K, FEATS, sp_size=10, estim_model=v, pca_coef=pca_coef)
        assert len(out) == 2 and out[1][1].shape[-1] == K
        model, fts = pl.estim_model_classes_group(imgs, K, FEATS, sp_size=10, pca_coef=pca_coef, model_type=v)
        assert model.predict_proba(fts[0]).shape == (len(fts[0]), K)


@pytest.mark.parametrize('variant,pca_coef', [('GMM', None), ('kmeans', None), ('BGM', None), ('Otsu', None), ('GMM', 0.95),
                                              ('BGM', 0.95), ('GMM_kmeans', 3)])
def test_pipeline_equals_fit_on_the_same_features(variant, pca_coef):
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200 import pipelines as pl
    K = 2 if variant == 'Otsu' else 3
    imgs = [synth_regions(192, 256, seed=s)[0] for s in (41, 42, 43)]
    single = [pl.pipe_color2d_slic_features_model_graphcut(im, K, FEATS, sp_size=12, pca_coef=pca_coef, estim_model=variant)
              for im in imgs]
    _, fts = pl.compute_color2d_superpixels_features(imgs[0], FEATS, sp_size=12)
    model = gc.estim_class_model(fts, K, variant, pca_coef)
    ref = pl.segment_color2d_slic_features_model_graphcut(imgs[0], model, FEATS, sp_size=12)
    assert np.array_equal(single[0][0], ref[0])
    np.testing.assert_allclose(single[0][1], ref[1], rtol=1e-6, atol=1e-9)
    batch = pl.segment_images_batch(imgs, K, FEATS, sp_size=12, estim_model=variant, pca_coef=pca_coef)
    for (a, sa), (b, sb) in zip(batch, single):
        assert np.array_equal(a, b)
        np.testing.assert_allclose(sa, sb, rtol=1e-9, atol=1e-12)


def test_bgm_graph_replay_equals_eager():
    from pyimsegm_b200 import pipelines as pl
    img = synth_regions(200, 240, seed=51)[0]        # a configuration no other test has run: its graph is captured here
    pl.USE_CUDA_GRAPHS = False
    try:
        eager = pl.pipe_color2d_slic_features_model_graphcut(img, 3, FEATS, sp_size=13, estim_model='BGM')
    finally:
        pl.USE_CUDA_GRAPHS = True
    n_graphs = sum(isinstance(v, tuple) for v in pl._GRAPHS.values())
    for _ in range(3):
        res = pl.pipe_color2d_slic_features_model_graphcut(img, 3, FEATS, sp_size=13, estim_model='BGM')
        assert np.array_equal(res[0], eager[0]) and np.array_equal(res[1], eager[1])
    assert sum(isinstance(v, tuple) for v in pl._GRAPHS.values()) > n_graphs, 'no CUDA graph was captured'


def test_host_switch_runs_every_variant_through_sklearn():
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200 import pipelines as pl
    img = synth_regions(128, 160, seed=61)[0]
    gc.USE_DEVICE_GMM = False
    try:
        for v in VARIANTS:
            for pca_coef in (None, 0.95):
                K = 2 if v == 'Otsu' else 3
                segm, soft = pl.pipe_color2d_slic_features_model_graphcut(img, K, FEATS, sp_size=10, pca_coef=pca_coef, estim_model=v)
                assert segm.shape == img.shape[:2] and soft.shape[-1] == K
    finally:
        gc.USE_DEVICE_GMM = True
