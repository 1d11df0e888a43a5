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


def _device_pca(X, coef, use_scaler=True, n_dev=None):
    """(transform of the rows, fitted PCA, component count) of the device fit on X; with ``n_dev`` only the first n_dev rows are
    samples (a device-side count), and only their transform is returned"""
    import torch
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    d_n = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device='cuda')
    d_x, d_params, dims = eng.pca_fit_transform(eng.to_device(np.ascontiguousarray(X, dtype=np.float64)), use_scaler, coef, d_n=d_n)
    xt = eng.to_host(d_x).copy()
    return xt[:len(X) if n_dev is None else n_dev], gc._pca_from_device(eng.to_host(d_params), X.shape[1], coef), dims


# ---- PCA error bounds -------------------------------------------------------------------------------------------------------------
# Both sides compute the spectrum of the same covariance C of the (scaled) features Z [N, D]; the reference is scikit-learn's exact
# 'full' solver (LAPACK SVD of the centred Z), the device forms C from a one-pass Gram matrix and runs Householder + implicit QL.
# B bounds |lambda_device - lambda_reference| for every eigenvalue (Weyl: an eigenvalue moves by at most the 2-norm of the
# perturbation of the matrix), as the sum of
#   * C_EIG * D * u * lambda_max: both eigensolvers are backward stable (the computed eigenvalues are exact for C + F with
#     |F|_2 <= p(D) u |C|_2, p a modest multiple of D), and scikit-learn's centring of Z rounds each element once (a singular value
#     moves by at most u |Z_c|_F, an eigenvalue by at most 2 sqrt(D) u lambda_max);
#   * |E|_2, E = gamma_{N+2} (|Z|^T |Z| + N |mu| |mu|^T) / (N - 1): the rounding of the one-pass covariance (X^T X - N mu mu^T) /
#     (N - 1), N products summed per entry, then the centring term and the division (entrywise error bound, |E|_2 bounds the
#     matrix it sums to);
#   * with the scaler, 3 gamma_{N+4} lambda_max: the device's column scales differ from StandardScaler's by a relative
#     delta <= gamma_{N+4} (a sum of N squares and a square root on each side), so its covariance is S C S with |S - I| <= delta,
#     |S C S - C|_2 <= (2 delta + delta^2) lambda_max.  A shift of a column's mean is removed by the centring.
U = 2.0 ** -53
#: the constant c of the eigensolver term c * D * u * lambda_max
C_EIG = 32


def _gamma(n):
    return n * U / (1 - n * U)


def _pca_bound(Z, lam_max, use_scaler):
    N, D = Z.shape
    A, mu = np.abs(Z), np.abs(Z.mean(axis=0))
    E = _gamma(N + 2) * (A.T @ A + N * np.outer(mu, mu)) / (N - 1)
    return C_EIG * D * U * lam_max + np.linalg.norm(E, 2) + (3 * _gamma(N + 4) * lam_max if use_scaler else 0.0)


def _check_pca(pca, xt, dims, X, coef, use_scaler=True):
    """the device PCA ``pca`` (its transform ``xt`` of X, its component count ``dims``) against PCA(coef, svd_solver='full') on the
    StandardScaler output of X (on X itself without the scaler), within the bounds derived above"""
    N, D = X.shape
    Z = preprocessing.StandardScaler().fit_transform(X) if use_scaler else np.asarray(X, dtype=np.float64)
    ref = decomposition.PCA(coef, svd_solver='full').fit(Z)
    nc = ref.n_components_
    assert pca.n_components_ == nc == dims and pca.n_samples_ == N
    lam = np.concatenate([decomposition.PCA(svd_solver='full').fit(Z).explained_variance_, np.zeros(max(0, D - N))])
    lam_max, B = lam[0], _pca_bound(Z, lam[0], use_scaler)
    # eigenvalues, and the noise variance as their mean over nc .. min(N, D) - 1
    np.testing.assert_array_less(np.abs(pca.explained_variance_ - ref.explained_variance_), B)
    assert abs(pca.noise_variance_ - ref.noise_variance_) <= B, (pca.noise_variance_, ref.noise_variance_, B)
    # ratios lambda / T: |T_device - T| <= D B (D eigenvalues on the device, min(N, D) in the reference, the rest within B of 0),
    # so |r_device - r| <= (B + r D B) / (T - D B)
    T = lam.sum()
    np.testing.assert_array_less(np.abs(pca.explained_variance_ratio_ - ref.explained_variance_ratio_),
                                 (B + ref.explained_variance_ratio_ * D * B) / (T - D * B))
    # singular values sqrt((N - 1) lambda): |sqrt(a) - sqrt(b)| <= min(sqrt(|a - b|), |a - b| / sqrt(b))
    d = (N - 1) * B
    np.testing.assert_array_less(np.abs(pca.singular_values_ - ref.singular_values_),
                                 np.minimum(np.sqrt(d), d / np.maximum(ref.singular_values_, 1e-300)) * (1 + 4 * U))
    # the mean of the scaled features (0 up to rounding with the scaler): N terms summed on either side, the scales' relative
    # difference, and the difference of the two scalers' means, |x| gamma_N on either side, over the scale
    xs = np.abs(X).mean(axis=0) / (preprocessing.StandardScaler().fit(X).scale_ if use_scaler else 1.0)
    np.testing.assert_array_less(np.abs(pca.mean_ - ref.mean_), 3 * _gamma(N + 4) * (np.abs(Z).mean(axis=0) + xs) + 1e-300)
    # components: Davis-Kahan bounds the angle of each side's eigenvector to the exact one by B / (gap - B), so two unit vectors
    # differ by at most 2 sqrt(2) B / (gap - B), plus the eigensolvers' loss of orthogonality C_EIG D u.  Only components whose gap
    # to every other eigenvalue exceeds both 1e3 D u lambda_max and 4 B are compared as vectors; sklearn's svd_flip makes the
    # largest |entry| positive, so the signs must agree wherever the two largest |entries| are further apart than the error
    gaps = np.array([np.min(np.abs(np.delete(lam, k) - lam[k])) if D > 1 else np.inf for k in range(nc)])
    sep = gaps > np.maximum(1e3 * D * U * lam_max, 4 * B)
    Zc = Z - ref.mean_
    for k in np.flatnonzero(sep):
        tol = 2 * np.sqrt(2) * B / (gaps[k] - B) + C_EIG * D * U
        v, r = pca.components_[k], ref.components_[k]
        top = np.sort(np.abs(r))[::-1]
        if D > 1 and top[0] - top[1] <= 2 * tol:
            v = v * np.sign(v @ r)
        assert np.abs(v - r).max() <= tol, (k, np.abs(v - r).max(), tol)
        # the device transform of component k: the vector's error over |z_i - mu|, the scales' relative error, and the
        # rounding of the dot product the device takes as z . v - mu . v
        atol = (np.linalg.norm(Zc, axis=1) * tol + _gamma(N + 4) * (np.abs(Zc) @ np.abs(r))
                + _gamma(D + 2) * (np.abs(Z) @ np.abs(r) + np.abs(ref.mean_) @ np.abs(r)))
        np.testing.assert_array_less(np.abs(xt[:, k] * np.sign(v @ pca.components_[k]) - ref.transform(Z)[:, k]), atol * (1 + 4 * U))
    # the kept subspace: |P_device - P|_2 <= sum of the two sides' sin(Theta) <= 2 B / (gap - B) where the cut at nc is separated
    if nc < D and lam[nc - 1] - lam[nc] > max(1e3 * D * U * lam_max, 4 * B):
        P, R = pca.components_, ref.components_
        assert np.linalg.norm(P.T @ P - R.T @ R, 2) <= 2 * B / (lam[nc - 1] - lam[nc] - B) + 2 * C_EIG * D * U * nc


@pytest.mark.parametrize('coef', [0.5, 0.95, 0.98, 2])
@pytest.mark.parametrize('D', [3, 9, 40, 189, 1, 2, 16, 17, 31, 32, 33, 95, 96, 97, 232])
def test_device_pca_matches_sklearn(D, coef):
    """the widths at the kernels' edges: the warp lanes (31 / 32 / 33), the 96-wide Gram tiles, DBIG = 232; at D = 1 the count 2
    is the whole width.  The fixed tolerances below stay for the widths first tested with them; the new widths are held to the
    derived bounds alone (at D = 2 both entries of each component have magnitude 1 / sqrt(2) in exact arithmetic, so svd_flip's
    sign is decided by rounding there)"""
    coef = min(coef, D) if isinstance(coef, int) else coef
    X = _spectrum_data(D, seed=D)
    Z = preprocessing.StandardScaler().fit_transform(X)
    ref = decomposition.PCA(coef).fit(Z)
    assert ref._fit_svd_solver == 'covariance_eigh'
    xt, pca, dims = _device_pca(X, coef)
    _check_pca(pca, xt, dims, X, coef)
    if D not in (3, 9, 40, 189):
        return
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


@pytest.mark.parametrize('D,N', [(D, N) for D in (40, 189) for N in (10 * D - 1, 2 * D, D + 1, D, D - 1, D // 10, 2)])
@pytest.mark.parametrize('coef', [0.5, 0.95])
def test_device_pca_sample_regimes(coef, D, N):
    """fewer than 10 D samples, where scikit-learn's 'auto' leaves the covariance solver, down to fewer samples than features (a
    superpixel table of fewer than 10 x 189 rows): the noise variance averages explained_variance_[nc:], min(N, D) entries"""
    X = _spectrum_data(D, N + D, n=N)
    xt, pca, dims = _device_pca(X, coef)
    _check_pca(pca, xt, dims, X, coef)


@pytest.mark.parametrize('D,N', [(40, 400), (189, 1500), (189, 60)])
def test_device_pca_component_count_at_every_position(D, N):
    """coef halfway between the reference's cumulative ratios k - 1 and k keeps exactly k + 1 components (searchsorted(side=
    'right') + 1), for every k whose half-gap exceeds the bound on a cumulative ratio: |c_device - c| <= ((k + 1) B + c D B) /
    (T - D B) + gamma_D c (the ratio bound of _check_pca summed over k + 1 ratios, and the device's running sum)"""
    X = _spectrum_data(D, 3 * D + N, n=N)
    Z = preprocessing.StandardScaler().fit_transform(X)
    full = decomposition.PCA(svd_solver='full').fit(Z)
    lam = full.explained_variance_
    B, T = _pca_bound(Z, lam[0], True), lam.sum()
    c = np.cumsum(full.explained_variance_ratio_)
    tested = 0
    for k in range(len(c) - 1):
        lo = c[k - 1] if k else 0.0
        coef = (lo + c[k]) / 2
        err = ((k + 1) * B + c[k] * D * B) / (T - D * B) + _gamma(D) * c[k]
        if (c[k] - lo) / 2 <= 2 * err or not 0 < coef < 1:
            continue
        assert decomposition.PCA(coef, svd_solver='full').fit(Z).n_components_ == k + 1
        _, pca, dims = _device_pca(X, coef)
        assert pca.n_components_ == dims == k + 1, (k, coef, dims)
        tested += 1
    assert tested >= 0.9 * (min(N, D) - 1), tested


def _refusal(X, k):
    """the ValueError scikit-learn raises for PCA(k) on X, as the reference fits it (svd_solver='auto')"""
    with pytest.raises(ValueError) as err:
        decomposition.PCA(k).fit(preprocessing.StandardScaler().fit_transform(X))
    return str(err.value)


@pytest.mark.parametrize('D,N', [(40, 400), (40, 30), (189, 1500), (189, 60)])
def test_device_pca_integer_counts(D, N):
    """counts 1, min(N, D), D and min(N, D) + 1: a count above min(N, D) is scikit-learn's ValueError, raised before any launch
    by every entry point that knows N on the host"""
    import re
    from pyimsegm_b200 import _lib
    from pyimsegm_b200 import graph_cuts as gc
    lib = _lib.lib()
    X = _spectrum_data(D, D + 2 * N, n=N)
    for k in sorted({1, min(N, D), D, min(N, D) + 1}):
        if k <= min(N, D):
            xt, pca, dims = _device_pca(X, k)
            _check_pca(pca, xt, dims, X, k)
            continue
        msg = re.escape(_refusal(X, k))
        for fit in (lambda: gc.estim_class_model(X, 2, 'GMM', k),
                    lambda: gc.estim_class_model_device(X, 2, pca_coef=k),
                    lambda: gc.fit_class_model_device(X, 2, True, 'GMM', 1, 10, k)):
            n0 = lib.isb_launch_count()
            with pytest.raises(ValueError, match=msg):
                fit()
            assert lib.isb_launch_count() == n0


@pytest.mark.parametrize('D', [1, 7, 40])
def test_device_pca_constant_columns(D):
    """every column constant (the scaled features exactly 0): one component, ratios NaN (0 / 0), noise variance 0, as scikit-learn"""
    X = np.tile(0.5 * np.arange(D) - 1.0, (300, 1))
    Z = preprocessing.StandardScaler().fit_transform(X)
    assert not Z.any()
    with np.errstate(invalid='ignore', divide='ignore'):
        ref = decomposition.PCA(0.95, svd_solver='full').fit(Z)
    assert (ref.n_components_, ref.noise_variance_) == (1, 0.0) and np.isnan(ref.explained_variance_ratio_).all()
    xt, pca, dims = _device_pca(X, 0.95)
    assert pca.n_components_ == dims == 1 and pca.noise_variance_ == 0.0
    assert np.isnan(pca.explained_variance_ratio_).all()
    assert not pca.explained_variance_.any() and not pca.singular_values_.any() and not xt.any()


@pytest.mark.parametrize('coef', [0.95, 3])
@pytest.mark.parametrize('D', [9, 40])
def test_device_pca_without_scaler_large_means(D, coef):
    """use_scaler=False with column means near 1e4 and unit spread: the one-pass centring term of the bound dominates"""
    rng = np.random.RandomState(D)
    X = _spectrum_data(D, seed=D + 1, n=2000) / 2 + rng.uniform(0.9e4, 1.1e4, D)
    xt, pca, dims = _device_pca(X, coef, use_scaler=False)
    _check_pca(pca, xt, dims, X, coef, use_scaler=False)


@pytest.mark.parametrize('D,N_in,n_dev', [(40, 4000, 3000), (189, 2000, 300), (40, 500, 2), (189, 500, 2)])
def test_device_pca_rows_past_n_dev_are_not_samples(D, N_in, n_dev):
    """a buffer of N_in rows, NaN past the device count n_dev: the fit of the first n_dev rows, bit for bit (the scaler, the
    Gram's split-K ranges and the eigensolver all follow n_dev), and within the bounds of scikit-learn's"""
    X = _spectrum_data(D, n_dev + D, n=n_dev)
    Xp = np.full((N_in, D), np.nan)
    Xp[:n_dev] = X
    xt, pca, dims = _device_pca(Xp, 0.95, n_dev=n_dev)
    assert np.isfinite(xt).all()
    xt1, pca1, dims1 = _device_pca(X, 0.95)
    assert dims == dims1 and np.array_equal(xt, xt1)
    for name in ('mean_', 'components_', 'explained_variance_', 'explained_variance_ratio_', 'singular_values_', 'noise_variance_',
                 'n_samples_'):
        assert np.array_equal(getattr(pca, name), getattr(pca1, name)), name
    _check_pca(pca, xt, dims, X, 0.95)


@pytest.mark.parametrize('kind', ['GMM', 'BGM'])
@pytest.mark.parametrize('D,K,n,coef', [pytest.param(9, 3, 5000, 0.95, id='9-3'), pytest.param(40, 3, 5000, 0.95, id='40-3'),
                                        pytest.param(189, 3, 1500, 0.5, id='189-3-1500-0.5')])
def test_scaler_pca_mixture_matches_sklearn_pipeline(kind, D, K, n, coef):
    """the shared start through scaler, PCA and mixture; at 1500 x 189 (fewer than 10 D samples) PCA(0.5) keeps the few components
    of the blob centres, far fewer than N / K, so that the EM stays well conditioned"""
    from pyimsegm_b200 import graph_cuts as gc
    X, _, y0 = _blobs(D, K, seed=7 * D, n=n)
    model = gc.estim_class_model_device(X, K, init_labels=y0, estim_model=kind, pca_coef=coef)
    assert [n for n, _ in model.steps] == ['std_scaler', 'reduce_dim', 'model']
    Z = preprocessing.StandardScaler().fit_transform(X)
    pca = decomposition.PCA(coef, svd_solver='full').fit(Z)
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
