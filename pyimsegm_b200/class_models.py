"""
Device ``predict_proba`` of a caller-fitted class model.

The reference's shared-model entry point (``segment_color2d_slic_features_model_graphcut``, reference pipelines.py:160-241) takes
a model fitted elsewhere: the group mixture of ``estim_model_classes_group`` (:113-157) or a trained classifier
(``classification.py:101``, a random forest by default).  :func:`compile_model` turns such a model into flat tables that
``isb_class_transform`` / ``isb_mixture_predict_proba`` / ``isb_forest_predict_proba`` / ``isb_knn_predict_proba`` /
``isb_linear_predict_proba`` (include/imsegm_b200.h) evaluate on the device, so the pipeline keeps its features on the GPU and
never waits for the host.

Supported: a bare estimator or a ``Pipeline`` of an optional ``StandardScaler``, an optional ``PCA`` and one of
``GaussianMixture`` / ``BayesianGaussianMixture`` (any covariance type, <= 232 features after the transforms, <= 8 components) or
``DecisionTreeClassifier`` / ``RandomForestClassifier`` / ``ExtraTreesClassifier`` (single output, <= 64 classes) or
``KNeighborsClassifier`` (single output, ``weights`` 'uniform' or 'distance', Euclidean metric -- 'euclidean', or 'minkowski' with
p = 2 and no ``metric_params`` -- 1 <= n_neighbors <= 64 and <= the training rows, <= 64 classes; ``isb_knn_predict_proba``) or
``LogisticRegression`` (``coef_`` [1 or K, D], <= 64 classes; ``isb_linear_predict_proba``).  Anything else gives ``None`` and the
caller keeps the host round trip.

Trees and forests are bit-identical to scikit-learn (``n_jobs=None``) when no PCA is involved; mixtures and PCA differ only by the
order of floating-point sums.  k-nearest neighbours take their squared distances as a left-to-right float64 loop and order ties by
training index: with uniform weights the result is bit-identical to scikit-learn wherever scikit-learn's own distances (its kd-tree
or its ||x||^2 - 2 x.t + ||t||^2 expansion) pick the same neighbours, i.e. away from near ties of the k-th and (k+1)-th distances;
distance weights and logistic regression differ by the rounding of their sums.
"""
import hashlib
import weakref

import numpy as np

#: limits of isb_mixture_predict_proba (csrc/gmm.cu DBIG, KMAX) and of isb_forest_predict_proba (the alpha-expansion's K)
MIXTURE_MAX_FEATURES, MIXTURE_MAX_CLASSES = 232, 8
FOREST_MAX_CLASSES = 64

#: fitted attributes a refit replaces: a snapshot holds them, so an unchanged model is not compiled again
_FITTED_ATTRS = ('mean_', 'scale_', 'components_', 'explained_variance_', 'weights_', 'means_', 'precisions_cholesky_',
                 'weight_concentration_', 'degrees_of_freedom_', 'mean_precision_', 'tree_', 'estimators_', '_fit_X', '_y', 'coef_',
                 'intercept_')
#: parameters that change what predict_proba computes without a refit
_PREDICT_PARAMS = ('with_mean', 'with_std', 'whiten', 'covariance_type', 'weight_concentration_prior_type', 'n_neighbors', 'weights', 'p',
                   'metric', 'metric_params')
#: isb_knn_predict_proba's weights codes
KNN_WEIGHTS = {'uniform': 0, 'distance': 1}
KNN_MAX_NEIGHBOURS = 64

_CACHE = weakref.WeakKeyDictionary()


class CompiledModel(object):
    """device tables of one fitted model.

    :ivar str kind: 'mixture', 'forest', 'knn' or 'linear'
    :ivar int n_features_in: feature columns the model takes
    :ivar int n_dims: dimensions after the transforms (what the final estimator sees)
    :ivar int n_classes: columns of ``predict_proba``
    :ivar classes_: ``getattr(model, 'classes_', None)`` of the source model
    :ivar dict tables: name -> contiguous ndarray (see the C-ABI for the layouts)
    :ivar dict params: scalar arguments of the evaluation ('knn': n_neighbors and the weights code)
    :ivar bytes digest: content digest of the tables and parameters (device constants and CUDA graphs are keyed on it)
    """

    def __init__(self, kind, n_features_in, n_dims, n_classes, classes, tables, average=False, params=None):
        self.kind, self.n_features_in, self.n_dims, self.n_classes = kind, int(n_features_in), int(n_dims), int(n_classes)
        self.classes_ = classes
        self.average = bool(average)
        self.params = {k: int(v) for k, v in (params or {}).items()}
        self.tables = {k: np.ascontiguousarray(v) for k, v in tables.items()}
        key = (kind, self.n_features_in, self.n_dims, self.n_classes, self.average) + ((sorted(self.params.items()), ) if self.params else ())
        h = hashlib.blake2b(repr(key).encode(), digest_size=16)
        for name in sorted(self.tables):
            arr = self.tables[name]
            h.update(repr((name, arr.shape, arr.dtype.str)).encode())
            h.update(arr.tobytes())
        self.digest = h.digest()

    def predict_proba(self, features):
        """``predict_proba`` on the device: features [N, n_features_in] (host) -> probabilities [N, n_classes] (host)"""
        from .engine import get_engine
        x = np.ascontiguousarray(features, dtype=np.float64)
        if x.ndim != 2 or x.shape[1] != self.n_features_in:
            raise ValueError('X has %r features, but the model is expecting %d features as input'
                             % (x.shape[1:] if x.ndim == 2 else x.shape, self.n_features_in))
        if len(x) == 0:
            return np.zeros((0, self.n_classes))
        eng = get_engine()
        proba = eng.class_model_predict(eng.to_device(x, 'cm_feat_in'), self)
        return eng.to_host(proba).copy()


def _steps(model):
    from sklearn.pipeline import Pipeline
    if type(model) is Pipeline:
        return [s for _, s in model.steps if s is not None and not (isinstance(s, str) and s == 'passthrough')]
    return [model]


def _fitted_state(model):
    objs, params = [], []
    for step in _steps(model):
        objs.append(step)
        for a in _FITTED_ATTRS:
            objs.append(getattr(step, a, None))
        for est in getattr(step, 'estimators_', None) or ():
            objs += [est, getattr(est, 'tree_', None)]
        params.append(tuple(getattr(step, a, None) for a in _PREDICT_PARAMS))
    return objs, params


def compile_model(model):
    """device form of a fitted scikit-learn model, or None when it is not supported (or not fitted).  Compiled once per model and
    reused while its fitted attributes are the same objects: a refit (which replaces them) is noticed and compiled again."""
    try:
        state = _fitted_state(model)
    except Exception:  # noqa: BLE001 -- an object we cannot inspect is simply not supported
        return None
    try:
        hit = _CACHE.get(model)
    except TypeError:       # not weakly referenceable / not hashable: compile every time
        hit = None
    if hit is not None and hit[0][1] == state[1] and len(hit[0][0]) == len(state[0]) \
            and all(a is b for a, b in zip(hit[0][0], state[0])):
        return hit[1]
    try:
        compiled = _compile(model)
    except (AttributeError, TypeError, ValueError):     # not fitted / unexpected attribute layout: the host path reports it
        compiled = None
    if compiled is not None:
        try:
            _CACHE[model] = (state, compiled)
        except TypeError:
            pass
    return compiled


def _compile(model):
    from sklearn.decomposition import PCA
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.mixture import BayesianGaussianMixture, GaussianMixture
    from sklearn.neighbors import KNeighborsClassifier
    from sklearn.preprocessing import StandardScaler
    from sklearn.tree import DecisionTreeClassifier
    steps = _steps(model)
    if not steps:
        return None
    *transforms, final = steps
    scaler = pca = None
    for t in transforms:
        if type(t) is StandardScaler and scaler is None and pca is None:
            scaler = t
        elif type(t) is PCA and pca is None:
            pca = t
        else:
            return None
    if type(final) in (GaussianMixture, BayesianGaussianMixture):
        kind = 'mixture'
    elif type(final) in (DecisionTreeClassifier, RandomForestClassifier, ExtraTreesClassifier):
        kind = 'forest'
    elif type(final) is KNeighborsClassifier:
        kind = 'knn'
    elif type(final) is LogisticRegression:
        kind = 'linear'
    else:
        return None
    first = transforms[0] if transforms else final
    n_in = int(first.n_features_in_)
    tables, dims = _transform_tables(scaler, pca, n_in)
    if dims is None or int(final.n_features_in_) != dims:
        return None
    average, params = False, None
    if kind == 'mixture':
        final_tables, n_classes = _mixture_tables(final, dims)
    elif kind == 'forest':
        final_tables, n_classes, average = _forest_tables(final, dims)
    elif kind == 'knn':
        final_tables, n_classes, params = _knn_tables(final, dims)
    else:
        final_tables, n_classes = _linear_tables(final, dims)
    if final_tables is None:
        return None
    tables.update(final_tables)
    try:
        classes = getattr(model, 'classes_', None)
    except Exception:  # noqa: BLE001 -- Pipeline.classes_ raises when the final step has none
        classes = None
    return CompiledModel(kind, n_in, dims, n_classes, classes, tables, average, params)


def _transform_tables(scaler, pca, n_in):
    """StandardScaler / PCA -> (tables, dimensions after the transforms); (None, None) when the steps do not chain"""
    tables, dims = {}, n_in
    if scaler is not None:
        if int(scaler.n_features_in_) != dims:
            return None, None
        if scaler.with_mean:
            tables['sc_mean'] = np.asarray(scaler.mean_, dtype=np.float64)
        if scaler.with_std:
            tables['sc_scale'] = np.asarray(scaler.scale_, dtype=np.float64)
    if pca is not None:
        comp = np.asarray(pca.components_, dtype=np.float64)
        if comp.ndim != 2 or comp.shape[1] != dims:
            return None, None
        tables['pca_comp'] = comp
        # sklearn PCA._transform: X C^T - reshape(mean_, (1, -1)) C^T -- the same product, so the same bits
        tables['pca_mean'] = (np.reshape(np.asarray(pca.mean_, dtype=np.float64), (1, -1)) @ comp.T).ravel()
        if pca.whiten:
            scale = np.sqrt(np.asarray(pca.explained_variance_, dtype=np.float64))
            scale[scale < np.finfo(scale.dtype).eps] = np.finfo(scale.dtype).eps
            tables['pca_scale'] = scale
        dims = comp.shape[0]
    return tables, dims


def _mixture_tables(mm, D):
    """per-component constants of _estimate_weighted_log_prob: the precision Cholesky factor U_k [K, D, D] in the full form,
    b_k = means_k U_k, and c_k = log|U_k| + log weight_k (+ the variational terms of BayesianGaussianMixture)"""
    from sklearn.mixture import BayesianGaussianMixture
    means = np.asarray(mm.means_, dtype=np.float64)
    K = means.shape[0]
    if means.shape != (K, D) or D > MIXTURE_MAX_FEATURES or K > MIXTURE_MAX_CLASSES:
        return None, None
    pc = np.asarray(mm.precisions_cholesky_, dtype=np.float64)
    ct = mm.covariance_type
    if pc.shape != {'full': (K, D, D), 'tied': (D, D), 'diag': (K, D), 'spherical': (K, )}.get(ct):
        return None, None
    if ct == 'full':
        U = pc
        log_det = np.sum(np.log(pc.reshape(K, -1)[:, ::D + 1]), 1)
    elif ct == 'tied':
        U = np.broadcast_to(pc, (K, D, D))
        log_det = np.full(K, np.sum(np.log(np.diag(pc))))
    elif ct == 'diag':
        U = np.stack([np.diag(p) for p in pc])
        log_det = np.sum(np.log(pc), axis=1)
    elif ct == 'spherical':
        U = pc[:, None, None] * np.eye(D)[None]
        log_det = D * np.log(pc)
    else:
        return None, None
    U = np.ascontiguousarray(U, dtype=np.float64)
    bvec = np.stack([means[k] @ U[k] for k in range(K)])
    if type(mm) is BayesianGaussianMixture:
        from scipy.special import digamma
        # BayesianGaussianMixture._estimate_log_weights and _estimate_log_prob
        if mm.weight_concentration_prior_type == 'dirichlet_process':
            a, b = (np.asarray(v, dtype=np.float64) for v in mm.weight_concentration_)
            digamma_sum = digamma(a + b)
            log_w = digamma(a) - digamma_sum + np.hstack((0, np.cumsum(digamma(b) - digamma_sum)[:-1]))
        else:
            wc = np.asarray(mm.weight_concentration_, dtype=np.float64)
            log_w = digamma(wc) - digamma(np.sum(wc))
        dof = np.asarray(mm.degrees_of_freedom_, dtype=np.float64)
        log_lambda = D * np.log(2.0) + np.sum(digamma(0.5 * (dof - np.arange(0, D)[:, np.newaxis])), 0)
        const = log_det - 0.5 * D * np.log(dof) + 0.5 * (log_lambda - D / np.asarray(mm.mean_precision_, dtype=np.float64)) + log_w
    else:
        const = log_det + np.log(np.asarray(mm.weights_, dtype=np.float64))
    return {'prec_chol': U, 'bvec': np.ascontiguousarray(bvec), 'log_const': np.ascontiguousarray(const, dtype=np.float64)}, K


def _forest_tables(est, D):
    """structure-of-arrays node tables of every tree, children as global node indices, one root per tree; value = the leaf class
    fractions sklearn's tree predict_proba returns"""
    from sklearn.tree import DecisionTreeClassifier
    if int(getattr(est, 'n_outputs_', 1)) != 1:
        return None, None, None
    K = int(est.n_classes_)
    if K > FOREST_MAX_CLASSES:
        return None, None, None
    trees = [est] if type(est) is DecisionTreeClassifier else list(est.estimators_)
    if not trees:
        return None, None, None
    feature, threshold, left, right, value, roots = [], [], [], [], [], []
    off = 0
    for t in trees:
        tr = t.tree_
        val = np.asarray(tr.value)
        if tr.n_outputs != 1 or val.shape[2] < K:
            return None, None, None
        f = np.asarray(tr.feature, dtype=np.int64)
        lc, rc = np.asarray(tr.children_left, dtype=np.int64), np.asarray(tr.children_right, dtype=np.int64)
        inner = lc >= 0
        if np.any(f[inner] >= D) or np.any(f[inner] < 0):
            return None, None, None
        roots.append(off)
        feature.append(np.where(inner, f, 0))
        threshold.append(np.asarray(tr.threshold, dtype=np.float64))
        left.append(np.where(inner, lc + off, -1))
        right.append(np.where(inner, rc + off, -1))
        value.append(val[:, 0, :K])
        off += len(lc)
    i32 = np.int32
    tables = {'roots': np.asarray(roots, dtype=i32), 'feature': np.concatenate(feature).astype(i32),
              'threshold': np.concatenate(threshold), 'left': np.concatenate(left).astype(i32),
              'right': np.concatenate(right).astype(i32), 'value': np.ascontiguousarray(np.concatenate(value), dtype=np.float64)}
    return tables, K, type(est) is not DecisionTreeClassifier


def _knn_tables(est, D):
    """the training rows (_fit_X as float64) and their class indices (_y) of a Euclidean KNeighborsClassifier, with n_neighbors and
    the weights code; (None, None, None) for anything isb_knn_predict_proba does not compute the same way"""
    weights = est.weights
    if not isinstance(weights, str) or weights not in KNN_WEIGHTS:
        return None, None, None
    p, metric = est.p, est.metric
    if est.metric_params or not (metric == 'euclidean' or (metric == 'minkowski' and p == 2)):
        return None, None, None
    # the metric the model was fitted with (kneighbors uses it): a parameter change without a refit must agree with it
    if getattr(est, 'effective_metric_', None) != 'euclidean' or getattr(est, 'effective_metric_params_', None):
        return None, None, None
    if getattr(est, 'outputs_2d_', True) or not isinstance(est._fit_X, np.ndarray):
        return None, None, None
    fit_x = np.asarray(est._fit_X, dtype=np.float64)
    y = np.asarray(est._y)
    K = len(est.classes_)
    k = est.n_neighbors
    if fit_x.ndim != 2 or fit_x.shape[1] != D or y.shape != (len(fit_x), ) or not isinstance(k, (int, np.integer)):
        return None, None, None
    if not (1 <= k <= min(KNN_MAX_NEIGHBOURS, len(fit_x))) or K > FOREST_MAX_CLASSES or len(fit_x) >= 2 ** 31:
        return None, None, None
    if len(y) and (y.min() < 0 or y.max() >= K):
        return None, None, None
    return {'fit_x': fit_x, 'y': y.astype(np.int32)}, K, {'n_neighbors': int(k), 'weights': KNN_WEIGHTS[weights]}


def _linear_tables(est, D):
    """coef_ [1 or K, D] and intercept_ of a LogisticRegression; (None, None) for any other layout"""
    coef = np.asarray(est.coef_, dtype=np.float64)
    K = len(est.classes_)
    if coef.ndim != 2 or coef.shape[1] != D or coef.shape[0] != (1 if K == 2 else K) or K < 2 or K > FOREST_MAX_CLASSES:
        return None, None
    intercept = np.broadcast_to(np.asarray(est.intercept_, dtype=np.float64), (coef.shape[0], ))
    return {'coef': coef, 'intercept': np.array(intercept)}, K
