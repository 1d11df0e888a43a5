"""The estim_model variant table of the device fit (graph_cuts.class_model_spec) against the Pipeline the scikit-learn branch of
estim_class_model builds, and argument validation of the device fit entries (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
from sklearn import mixture

#: (estim_model, nb_classes): every row of the variant table, and names the reference does not know
VARIANTS = [('GMM', 3), ('GMM_kmeans', 3), ('GMM_Otsu', 3), ('kmeans', 3), ('kmeans_quantiles', 3), ('BGM', 3), ('BGM_kmeans', 3),
            ('Otsu', 2), ('Otsu', 3), ('unknown', 3), ('GMM_other', 2)]


@pytest.fixture
def host_fit():
    from pyimsegm_b200 import graph_cuts
    graph_cuts.USE_DEVICE_GMM = False
    yield graph_cuts
    graph_cuts.USE_DEVICE_GMM = True


@pytest.mark.parametrize('max_iter', [99, 4, 1])
@pytest.mark.parametrize('estim_model,K', VARIANTS)
def test_device_spec_equals_host_pipeline(host_fit, estim_model, K, max_iter):
    import warnings
    rng = np.random.RandomState(0)
    X = np.concatenate([c + rng.normal(0, 0.05, (40, 3)) for c in np.linspace(0, 1, K)])
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = host_fit.estim_class_model(X, K, estim_model, max_iter=max_iter)
    mm = model.steps[-1][1]
    kind, n_init, n_iter = host_fit.class_model_spec(estim_model, K, max_iter)
    assert type(mm) is {'GMM': mixture.GaussianMixture, 'BGM': mixture.BayesianGaussianMixture}[kind]
    assert (mm.n_init, mm.max_iter) == (n_init, n_iter)
    if type(mm) is mixture.BayesianGaussianMixture:
        assert mm.covariance_type == 'full' and mm.weight_concentration_prior_type == 'dirichlet_process'


def test_device_applicability():
    from pyimsegm_b200 import graph_cuts as gc
    for v, _ in VARIANTS:
        assert gc.device_gmm_applicable(6, 3, v, None)
    for p in (0.5, 0.95, np.float64(0.98), 1, 6, np.int64(3)):
        assert gc.device_gmm_applicable(6, 3, 'BGM', p), p
    for p in ('mle', 0.0, 1.0, 1.5, 0, 7, True, -2):
        assert not gc.device_gmm_applicable(6, 3, 'GMM', p), p
    assert not gc.device_gmm_applicable(233, 3) and not gc.device_gmm_applicable(6, 9)
    gc.USE_DEVICE_GMM = False
    try:
        assert not gc.device_gmm_applicable(6, 3)
    finally:
        gc.USE_DEVICE_GMM = True


def test_resident_model_tuple():
    from pyimsegm_b200 import pipelines as pl
    assert pl._fit_model(3, True) == ('fit', 3, True, 99)
    assert pl._fit_spec(('fit', 3, True, 99)) == (3, True, 99, 'GMM', 9, None)
    bgm, km, pca = pl._fit_model(3, True, 'BGM'), pl._fit_model(3, True, 'kmeans'), pl._fit_model(3, True, 'GMM', 0.95)
    assert len({bgm, km, pca, pl._fit_model(3, True)}) == 4
    assert pl._fit_spec(bgm) == (3, True, 99, 'BGM', 9, None)
    assert pl._fit_spec(km) == (3, True, 1, 'GMM', 9, None)
    assert pl._fit_spec(pca) == (3, True, 99, 'GMM', 9, 0.95)


def test_fit_entries_reject_bad_arguments_without_a_gpu():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    err = lambda: lib.isb_last_error().decode()  # noqa: E731
    assert lib.isb_abi_version() == 8
    big = 1 << 40
    # isb_mixture_fit_predict(kind, feat, N, D, ld, n_dev, K, n_init, max_iter, tol, reg, use_scaler, seed, init, proba, params, ws, ws_bytes, st)
    fa = [1, p, 100, 3, 3, None, 2, 1, 10, 1e-3, 1e-6, 1, 0, None, p, p, p, big, None]
    for i, bad in ((1, None), (14, None), (16, None), (2, 0), (3, 0), (4, 2), (6, 0), (7, 0), (8, 0)):
        args = list(fa)
        args[i] = bad
        assert lib.isb_mixture_fit_predict(*args) == _lib.ISB_ERR_ARG, i
    args = list(fa)
    args[0] = 2
    assert lib.isb_mixture_fit_predict(*args) == _lib.ISB_ERR_ARG and 'kind' in err()
    for i, bad in ((3, 233), (6, 9)):
        args = list(fa)
        args[i] = bad
        if i == 3:
            args[4] = 233
        assert lib.isb_mixture_fit_predict(*args) == _lib.ISB_ERR_UNSUPPORTED and 'D <=' in err()
    args = list(fa)
    args[17] = 64
    assert lib.isb_mixture_fit_predict(*args) == _lib.ISB_ERR_ARG and 'workspace' in err()
    # kind 1 adds its priors to the GMM workspace and parameter layout
    assert lib.isb_mixture_fit_workspace_bytes(1, 5000, 6, 3, 9) > lib.isb_mixture_fit_workspace_bytes(0, 5000, 6, 3, 9)
    assert lib.isb_mixture_fit_params_len(1, 6, 3) == lib.isb_mixture_fit_params_len(0, 6, 3) + 6 + 36
    # isb_pca_fit(feat, N, D, ld, n_dev, use_scaler, coef, n_components, params, n_comp_out, ws, ws_bytes, st)
    pa = [p, 100, 3, 3, None, 1, 0.95, 0, p, None, p, big, None]
    for i, bad in ((0, None), (8, None), (10, None), (1, 1), (2, 0), (3, 2), (6, 1.0), (6, 0.0), (7, 4), (11, 64)):
        args = list(pa)
        args[i] = bad
        assert lib.isb_pca_fit(*args) == _lib.ISB_ERR_ARG, i
    args = list(pa)
    args[6], args[7] = 7.0, 2          # a component count overrides coef
    args[11] = 64
    assert lib.isb_pca_fit(*args) == _lib.ISB_ERR_ARG and 'workspace' in err()
    args = list(pa)
    args[2] = args[3] = 233
    assert lib.isb_pca_fit(*args) == _lib.ISB_ERR_UNSUPPORTED and 'D <=' in err()
    assert lib.isb_pca_params_len(189) == 189 * 189 + 7 * 189 + 4
    assert lib.isb_pca_workspace_bytes(5000, 189) >= 8 * (5000 * 189 + 11 * 189 * 189)


@pytest.mark.parametrize('N,D,k', [(30, 40, 31), (30, 40, 40), (400, 40, 41), (100, 40, 41), (2, 189, 3)])
def test_component_count_above_min_n_d_is_sklearns_error(N, D, k):
    """an integer pca_coef above min(N, D) raises the ValueError of the reference's PCA(pca_coef), message included, in the device
    fit's entry before any device work (so also on a machine without a GPU)"""
    from sklearn import decomposition
    from pyimsegm_b200 import graph_cuts as gc
    X = np.random.RandomState(N + D).normal(size=(N, D))
    with pytest.raises(ValueError) as ref:
        decomposition.PCA(k).fit(X)
    with pytest.raises(ValueError) as dev:
        gc.fit_class_model_device(X, 2, True, 'GMM', 1, 10, k)
    assert str(dev.value) == str(ref.value)
    gc._check_pca_count(min(N, D), N, D)
    gc._check_pca_count(0.95, N, D)
