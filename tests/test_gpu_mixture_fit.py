"""GPU tests of the device mixture fit (isb_mixture_fit_predict, csrc/gmm.cu) against the float64 references of oracle/mixture.py at
the edges of its kernels: the thread-block cluster size of the single-kernel path (CL = 1, 2, 4, 8 CTAs per restart for N <= 1024,
<= 4096, <= 16384 and above), the feature widths around DMAX = 16, the 32-feature scaler blocks, the 96-wide GEMM tiles and DBIG = 232,
the class counts 1, 2 and KMAX = 8, the sample counts of the large-D E-step (8 per CTA), GEMM rows (96) and split-K Gram ranges,
a device-side sample count below the buffer height, the device's own k-means++ start (bit for bit), the choice among restarts, failed
restarts and degenerate inputs.  Every case but the failed restarts runs for both kinds, GaussianMixture and
BayesianGaussianMixture (BGM: digamma terms, Dirichlet-process weights, the priors, the ELBO as convergence and restart criterion);
the BGM's covariance prior keeps every covariance positive definite, so a BGM restart cannot fail.

Tolerances are those of the other shared-start tests: scaler rtol 1e-12; weights, means and covariances rtol 1e-6, atol 1e-8; lower
bound rtol 1e-8; n_iter_ and converged_ exact; predict_proba rtol 1e-5, atol 1e-9."""
import ctypes as C

import numpy as np
import pytest
from sklearn import preprocessing

from oracle import mixture as om

pytestmark = pytest.mark.gpu


def _with_bgm(cases, bgm_cases=None):
    """parameters (kind, *case): the GaussianMixture cases under the ids they had before the kind was a parameter, then the
    BayesianGaussianMixture cases (by default the same) with ids prefixed 'BGM-'"""
    name = lambda c: '-'.join(map(str, c))  # noqa: E731
    return ([pytest.param('GMM', *c, id=name(c)) for c in cases]
            + [pytest.param('BGM', *c, id='BGM-' + name(c)) for c in (cases if bgm_cases is None else bgm_cases)])


def _blobs(D, K, n, seed, inform=0.6):
    """K blobs in D dimensions (centres in [0.5, 1.5]^D, so that no feature mean is near 0) and a hard start in which a fraction
    ``inform`` of the samples carries its blob's label and the rest a random one; every label occurs in the start"""
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0.5, 1.5, (K, D))
    y = rng.randint(0, K, n)
    y[:min(K, n)] = np.arange(min(K, n))
    X = centres[y] + rng.normal(0, 0.04 if D <= 16 else 0.15, (n, D))
    y0 = np.where(rng.rand(n) < inform, y, rng.randint(0, K, n))
    y0[:min(K, n)] = np.arange(min(K, n))
    return X, y, y0.astype(np.int32)


def _fit(X, K, kind='GMM', n_init=1, max_iter=99, init=None, use_scaler=True, seed=0, reg_covar=1e-6, n_dev=None):
    """(proba [n, K], params) of the device fit on the rows of X; with ``n_dev`` only the first n_dev rows are samples"""
    import torch
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    d_x = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float64)).cuda()
    d_n = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device='cuda')
    if init is not None:
        init = np.ascontiguousarray(np.atleast_2d(init), dtype=np.int32)
        n_init = len(init)
    proba, params = eng.mixture_fit_predict(d_x, K, n_init, max_iter, use_scaler, seed, d_n=d_n, init_labels=init, reg_covar=reg_covar,
                                            kind=kind)
    n = len(X) if n_dev is None else n_dev
    return proba[:n].cpu().numpy().copy(), params.cpu().numpy().copy()


def _best_index(params, D, K):
    """the restart the device exported (the slot after the parameters and the lower_bound | n_iter | converged | ok tail)"""
    return int(params[2 * D + K + K * D + 2 * K * D * D + 4])


def _model(params, X, K, kind='GMM', use_scaler=True, max_iter=99):
    from pyimsegm_b200 import graph_cuts as gc
    return gc.sklearn_pipeline_from_device(params, X.shape[1], K, len(X), use_scaler, 1, max_iter, kind)


def _check(params, proba, X, ref, K, kind='GMM', use_scaler=True):
    """the device fit (params, proba on X) against the scikit-learn fit ``ref`` of the scaled X"""
    model = _model(params, X, K, kind, use_scaler, ref.max_iter)
    mm = model.named_steps['model']
    assert (mm.n_iter_, mm.converged_) == (ref.n_iter_, ref.converged_), \
        'n_iter %d/%d converged %s/%s; least | |change| - tol | of the reference: %.3g' % (
            mm.n_iter_, ref.n_iter_, mm.converged_, ref.converged_, om.tol_margin(ref))
    if use_scaler:
        sc = preprocessing.StandardScaler().fit(X)
        np.testing.assert_allclose(model.named_steps['std_scaler'].mean_, sc.mean_, rtol=1e-12)
        np.testing.assert_allclose(model.named_steps['std_scaler'].scale_, sc.scale_, rtol=1e-12)
        Z = sc.transform(X)
    else:
        D = X.shape[1]
        assert np.array_equal(params[:D], np.zeros(D)) and np.array_equal(params[D:2 * D], np.ones(D))
        Z = X
    names = ('weights_', 'means_', 'covariances_')
    if kind == 'BGM':
        names += ('mean_precision_', 'degrees_of_freedom_')
        for a, b in zip(mm.weight_concentration_, ref.weight_concentration_):
            np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(mm.mean_prior_, ref.mean_prior_, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(mm.covariance_prior_, ref.covariance_prior_, rtol=1e-9, atol=1e-12)
    for name in names:
        np.testing.assert_allclose(getattr(mm, name), getattr(ref, name), rtol=1e-6, atol=1e-8, err_msg=name)
    np.testing.assert_allclose(mm.lower_bound_, ref.lower_bound_, rtol=1e-8)
    np.testing.assert_allclose(proba, ref.predict_proba(Z), rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(model.predict_proba(X), proba, rtol=1e-5, atol=1e-9)


def _compare(X, y0, K, kind='GMM', max_iter=99):
    proba, params = _fit(X, K, kind, max_iter=max_iter, init=y0)
    Z = preprocessing.StandardScaler().fit_transform(X)
    _check(params, proba, X, om.shared_start_fit(Z, y0, K, kind, max_iter), K, kind)


# ---- the cluster size of the single-kernel path -------------------------------------------------------------------------------

@pytest.mark.parametrize('N', [4, 200, 1024, 1025, 4096, 4097, 16384, 16385, 40000])
@pytest.mark.parametrize('D', [3, 16])
@pytest.mark.parametrize('kind', ['GMM', 'BGM'])
def test_cluster_sizes_match_sklearn(kind, D, N):
    X, _, y0 = _blobs(D, 3, N, seed=N + D)
    _compare(X, y0, 3, kind)


# ---- feature widths and class counts --------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,D', [('GMM', d) for d in (1, 2, 15, 16, 17, 32, 33, 95, 96, 97, 192, 193, 232)]
                         + [('BGM', d) for d in (1, 2, 15, 16, 17, 33, 96, 97, 193, 232)])
def test_dimensions_match_sklearn(kind, D):
    X, _, y0 = _blobs(D, 3, 3000 if D <= 33 else 1500, seed=3 * D + 1)
    _compare(X, y0, 3, kind)


@pytest.mark.parametrize('kind,D,K', _with_bgm([(D, K) for D in (9, 189) for K in (1, 2, 8)]))
def test_class_counts_match_sklearn(kind, D, K):
    X, _, y0 = _blobs(D, K, 3000 if D <= 16 else 1500, seed=D + 11 * K)
    _compare(X, y0, K, kind, max_iter=99 if D <= 16 else 15)


def test_unsupported_sizes_are_refused_and_fit_on_the_host(monkeypatch):
    import torch
    from pyimsegm_b200 import _lib
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200.engine import Engine
    lib = _lib.lib()
    N, D, K = 64, 233, 3
    feat = torch.zeros((N, D), dtype=torch.float64, device='cuda')
    proba = torch.zeros((N, K), dtype=torch.float64, device='cuda')
    wsb = lib.isb_mixture_fit_workspace_bytes(0, N, D, K, 1)
    ws = torch.zeros(wsb, dtype=torch.uint8, device='cuda')
    rc = lib.isb_mixture_fit_predict(0, _lib.ptr(feat), N, D, D, None, K, 1, 10, C.c_double(1e-3), C.c_double(1e-6), 1, C.c_ulonglong(0),
                                     None, _lib.ptr(proba), None, _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr())
    assert rc == _lib.ISB_ERR_UNSUPPORTED and 'D <=' in lib.isb_last_error().decode()

    def boom(*args, **kwargs):
        raise AssertionError('the device fit ran')
    monkeypatch.setattr(Engine, 'mixture_fit_predict', boom)
    monkeypatch.setattr(gc, 'estim_class_model_device', boom)
    for D, K in ((233, 2), (3, 9)):
        X, _, _ = _blobs(D, K, 600, seed=D + K)
        n0 = lib.isb_launch_count()
        model = gc.estim_class_model(X, K, max_iter=4)
        assert lib.isb_launch_count() == n0
        mm = model.named_steps['model']
        assert (mm.n_components, mm.n_init, mm.max_iter) == (K, 2, 4) and mm.means_.shape == (K, D)


@pytest.mark.parametrize('N', [4, 7, 8, 9, 95, 96, 97, 127, 128, 129, 1000])
def test_large_d_sample_counts_match_sklearn(N):
    X, _, y0 = _blobs(40, 3, N, seed=N)
    _compare(X, y0, 3)


# ---- a device-side sample count below the buffer height --------------------------------------------------------------------------

@pytest.mark.parametrize('kind,D,N_in,n_dev', _with_bgm([(3, 4000, 3000), (3, 20000, 700), (3, 20000, 21), (40, 4000, 3000),
                                                        (40, 20000, 700)]))
def test_rows_past_n_dev_are_not_samples(kind, D, N_in, n_dev):
    """the buffer holds N_in rows, the device count n_dev; the rows past it are NaN.  The fit must be the one of the first n_dev
    rows; when the cluster size does not change (same CL bucket, or the large-D path, whose launches follow n_dev) bit for bit"""
    X, _, y0 = _blobs(D, 3, n_dev, seed=n_dev + D)
    Xp = np.full((N_in, D), np.nan)
    Xp[:n_dev] = X
    y0p = np.zeros(N_in, np.int32)
    y0p[:n_dev] = y0
    cl = lambda n: 1 if n <= 1024 else 2 if n <= 4096 else 4 if n <= 16384 else 8  # noqa: E731
    same = D > 16 or cl(N_in) == cl(n_dev)
    proba, params = _fit(Xp, 3, kind, init=y0p, n_dev=n_dev)
    assert np.isfinite(proba).all()
    Z = preprocessing.StandardScaler().fit_transform(X)
    _check(params, proba, X, om.shared_start_fit(Z, y0, 3, kind), 3, kind)
    proba1, params1 = _fit(X, 3, kind, init=y0)
    if same:
        assert np.array_equal(params, params1) and np.array_equal(proba, proba1)
    # the device's own start, 9 restarts: equal to the oracle's k-means++ labels of the first n_dev rows handed in as init_labels
    Y, least = om.kmeanspp_starts(Z, 3, 0, 9)
    assert min(least.values()) > 1e-9, least
    Yp = np.zeros((9, N_in), np.int32)
    Yp[:, :n_dev] = Y
    proba2, params2 = _fit(Xp, 3, kind, n_init=9, n_dev=n_dev)
    proba3, params3 = _fit(Xp, 3, kind, init=Yp, n_dev=n_dev)
    assert np.array_equal(params2, params3) and np.array_equal(proba2, proba3)
    if same:
        assert np.array_equal(params2, _fit(X, 3, kind, n_init=9)[1])


# ---- the device's k-means++ / Lloyd start, exactly -------------------------------------------------------------------------------

def _overlapping(D, K, n, seed):
    """blobs that overlap so much that every restart's Lloyd labels depend on its draws"""
    rng = np.random.RandomState(seed)
    c = rng.uniform(0, 1, (K, D))
    y = rng.randint(0, K, n)
    return c[y] + rng.normal(0, 1.0, (n, D))


@pytest.mark.parametrize('seed', [0, 1, 7])
@pytest.mark.parametrize('kind,D,N,K', _with_bgm([(3, 500, 3), (3, 3000, 3), (3, 20000, 3), (40, 500, 3), (40, 3000, 3), (16, 3000, 8)]))
def test_device_kmeanspp_start_is_the_oracle_start(kind, D, N, K, seed):
    """9 restarts from the device's own start against the same fit from the oracle's restatement of that start: the EM from equal
    labels is one deterministic kernel, so the two parameter vectors are equal bit for bit exactly when every restart drew the
    same centres and ended Lloyd with the same labels.  (16, 3000, 8) is the widest Lloyd exchange of the single kernel.  The
    'BGM' variant of estim_class_model runs its 9 restarts from the same start."""
    X = _overlapping(D, K, N, seed=100 + N + D)
    Z = preprocessing.StandardScaler().fit_transform(X)
    Y, least = om.kmeanspp_starts(Z, K, seed, 9)
    # every draw and every assignment is decided far above rounding, and no two restarts end with the same labels (so a start
    # drawn for the wrong restart changes the exported vector, whose last slot is the winner's index)
    assert min(least.values()) > 1e-9, least
    assert len({r.tobytes() for r in Y}) == 9
    proba, params = _fit(X, K, kind, n_init=9, seed=seed)
    proba_o, params_o = _fit(X, K, kind, init=Y, seed=seed)
    assert np.array_equal(params, params_o), 'exported restart %d (oracle start: %d)' % (_best_index(params, D, K), _best_index(params_o, D, K))
    assert np.array_equal(proba, proba_o)


# ---- the choice among restarts, failed restarts ----------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,D,case', _with_bgm([(D, case) for D in (3, 40) for case in ('quality', 'tie')]))
def test_restart_choice_is_sklearns(kind, D, case):
    """four EM iterations from starts of different quality: the device exports the restart with the largest lower bound (the
    ELBO for the BGM), the first one on a tie (sklearn's strict >), with that restart's n_iter_, converged_ and lower bound"""
    X, y, _ = _blobs(D, 3, 2000, seed=D + 5)
    rng = np.random.RandomState(D)
    start = lambda f: np.where(rng.rand(len(y)) < f, y, rng.randint(0, 3, len(y))).astype(np.int32)  # noqa: E731
    Y0 = np.stack([start(0.1), start(0.5), start(0.3)]) if case == 'quality' else np.stack([start(0.1), *[start(0.4)] * 2])
    if case == 'tie':
        Y0[2] = Y0[1]
    Z = preprocessing.StandardScaler().fit_transform(X)
    best, ref, lowers = om.shared_start_best(Z, Y0, 3, kind, max_iter=4)
    runner_up = max(lb for i, lb in enumerate(lowers) if i != best and lb != lowers[best])
    assert lowers[best] - runner_up > 1e-6 * abs(lowers[best]), lowers
    assert best == 1
    proba, params = _fit(X, 3, kind, init=Y0, max_iter=4)
    assert _best_index(params, D, 3) == best
    _check(params, proba, X, ref, 3, kind)


def _failing_start(D, seed):
    """unscaled blobs, the first centred at the origin with 5 samples exactly at it; a good start, and degenerate starts whose
    component 0 holds only the 5 origin samples (an exactly zero covariance: with reg_covar = 0 not positive definite)"""
    rng = np.random.RandomState(seed)
    centres = np.vstack([np.zeros(D), rng.uniform(2, 3, (2, D))])
    y = np.concatenate([np.zeros(5, int), rng.randint(0, 3, 1495)])
    X = centres[y] + rng.normal(0, 0.2, (len(y), D))
    X[:5] = 0.0
    bad = np.where(y == 0, 1, y)
    bad[:5] = 0
    bad2 = np.where(bad == 1, 2, np.where(bad == 2, 1, bad))
    return X, y.astype(np.int32), bad.astype(np.int32), bad2.astype(np.int32)


@pytest.mark.parametrize('D', [3, 40])
def test_failed_restart_is_dropped(D):
    """a restart whose covariance is not positive definite is a numerical failure (ok = 0), not a fault: the device drops it and
    exports the best of the others, where scikit-learn raises on it"""
    X, y, bad, _ = _failing_start(D, seed=D)
    with pytest.raises(ValueError):
        om.shared_start_fit(X, bad, 3, reg_covar=0.0)
    ref = om.shared_start_fit(X, y, 3, reg_covar=0.0)
    proba, params = _fit(X, 3, init=np.stack([bad, y]), use_scaler=False, reg_covar=0.0)
    assert _best_index(params, D, 3) == 1
    _check(params, proba, X, ref, 3, use_scaler=False)


@pytest.mark.parametrize('D', [3, 40])
def test_every_restart_failed(D):
    from pyimsegm_b200 import graph_cuts as gc
    X, _, bad, bad2 = _failing_start(D, seed=D + 1)
    proba, params = _fit(X, 3, init=np.stack([bad, bad2]), use_scaler=False, reg_covar=0.0)
    assert np.isnan(proba).all()
    with pytest.raises(ValueError, match='ill-defined empirical covariance'):
        gc.sklearn_pipeline_from_device(params, D, 3, len(X), False, 2, 99)


# ---- degenerate inputs ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,D,case', _with_bgm([(D, case) for D in (5, 40)
                                                   for case in ('empty_component', 'constant_columns', 'no_scaler', 'one_iteration')]))
def test_degenerate_inputs_match_sklearn(kind, D, case):
    X, y, y0 = _blobs(D, 3, 2500, seed=D + len(case))
    Z = preprocessing.StandardScaler().fit_transform(X)
    if case == 'empty_component':
        y0 = np.where(y0 == 2, 1, y0).astype(np.int32)             # component 2 has no member: nk = 10 eps, covariance reg_covar I
        _compare(X, y0, 3, kind)                                   # (for the BGM: the covariance prior)
    elif case == 'constant_columns':
        X[:, 1], X[:, 3] = 0.1, 2.5                                # scale 1, the centred column rounding noise (0.1) or exactly 0
        proba, params = _fit(X, 3, kind, init=y0)
        assert params[D + 1] == 1.0 and params[D + 3] == 1.0
        Z = preprocessing.StandardScaler().fit_transform(X)
        _check(params, proba, X, om.shared_start_fit(Z, y0, 3, kind), 3, kind)
    elif case == 'no_scaler':
        proba, params = _fit(X, 3, kind, init=y0, use_scaler=False)
        _check(params, proba, X, om.shared_start_fit(X, y0, 3, kind), 3, kind, use_scaler=False)
    else:
        # the 'kmeans' variant's shape: 9 restarts, one iteration each, never converged
        rng = np.random.RandomState(D)
        Y0 = np.stack([np.where(rng.rand(len(y)) < f, y, rng.randint(0, 3, len(y))) for f in np.linspace(0.1, 0.5, 9)]).astype(np.int32)
        best, ref, lowers = om.shared_start_best(Z, Y0, 3, kind, max_iter=1)
        assert sorted(lowers)[-1] - sorted(lowers)[-2] > 1e-6 * abs(lowers[best]), lowers
        proba, params = _fit(X, 3, kind, init=Y0, max_iter=1)
        assert _best_index(params, D, 3) == best
        _check(params, proba, X, ref, 3, kind)
        assert ref.n_iter_ == 1 and not ref.converged_


@pytest.mark.parametrize('kind', ['GMM', 'BGM'])
@pytest.mark.parametrize('D', [3, 40])
def test_reruns_are_bit_identical(D, kind):
    X, _, y0 = _blobs(D, 3, 5000, seed=D)
    for init in (None, y0):
        a = _fit(X, 3, kind, n_init=9, init=init)
        b = _fit(X, 3, kind, n_init=9, init=init)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
