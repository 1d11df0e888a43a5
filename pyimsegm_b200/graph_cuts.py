"""
GraphCut on the superpixel graph, on the GPU.

Mirror of the reference module ``imsegm/graph_cuts.py`` (same public names, arguments, error types).  The graph,
the energies and the alpha-expansion itself run in CUDA behind ``include/imsegm_b200.h``
(``isb_adjacency_edges`` / ``isb_gc_energies`` / ``isb_alpha_expansion``); the class model (``estim_class_model``, reference
graph_cuts.py:73-163) is fitted on the device for every ``estim_model`` variant and ``pca_coef`` (``class_model_spec``) and returned
as the reference's scikit-learn Pipeline; K > 8 and ``pca_coef='mle'`` fit with scikit-learn on the host.
"""
import logging

import numpy as np

from .engine import EDGE_GIVEN, EDGE_MODES, VECTOR_EDGE_METRICS, get_engine
from .superpixels import (
    device_adjacency,
    make_graph_segm_connect_grid2d_conn4,
    make_graph_segm_connect_grid3d_conn6,
    superpixel_centers,
)

#: number of iterations in Graph-Cut optimisation (reference graph_cuts.py:32)
DEFAULT_GC_ITERATIONS = 25
#: minimal probability of a class in the unary term (reference graph_cuts.py:36)
MIN_UNARY_PROB = 0.01
#: cap of the pairwise (smoothness) term (reference graph_cuts.py:38)
MAX_PAIRWISE_COST = 1e5
#: edge weights are clamped to [1 / val, val] (reference graph_cuts.py:40)
MIN_MAX_EDGE_WEIGHT = 1e3
#: the class model of every estim_model variant, with or without PCA, is fitted on the GPU (isb_mixture_fit_predict /
#: isb_pca_fit) when it fits the device kernels (<= 232 features, <= 8 classes, pca_coef None, in (0, 1)
#: or a component count); set False to force scikit-learn on the host
USE_DEVICE_GMM = True
#: a caller-fitted model (segment_color2d_slic_features_model_graphcut, segment_images_batch(model_pipeline=...), segment_resident)
#: that class_models.compile_model supports runs its predict_proba on the device; set False to force the host round trip
USE_DEVICE_PREDICT = True
#: seed of the device k-means++ initialisation (the reference leaves its model unseeded)
RANDOM_SEED = 0
#: D <= 16 runs as one kernel (a CTA per restart), 16 < D <= 256 (colour + Leung-Malik = 189) as batched FP64 GEMMs
DEVICE_GMM_MAX_FEATURES, DEVICE_GMM_MAX_CLASSES = 232, 8   # = DBIG of csrc/gmm.cu
#: up to this many features the fit is one kernel without any host synchronisation (csrc/gmm.cu DMAX)
DEVICE_GMM_SINGLE_KERNEL_MAX_FEATURES = 16


# ---------------------------------------------------------------------------------------------------------------------
# class model (host, scikit-learn -- unchanged behaviour of the reference)
# ---------------------------------------------------------------------------------------------------------------------

def estim_gmm_params(features, prob):
    """ GMM parameters from a soft labelling, hard-assigned by argmax (reference graph_cuts.py:43-70) """
    nb_samples, nb_classes = prob.shape
    labels = np.argmax(prob, axis=1)
    params = {'weights': [], 'means': [], 'covars': []}
    for lb in range(nb_classes):
        sel = labels == lb
        params['weights'].append(np.sum(sel) / float(nb_samples))
        params['means'].append(np.mean(features[sel], axis=0))
        params['covars'].append(np.cov(features[sel]))
    for n in ('means', 'covars'):
        params[n] = np.array([m.tolist() for m in params[n]])
    return params


def compute_multivarian_otsu(features):
    """ per-dimension Otsu split combined by majority vote (reference graph_cuts.py:166-193) """
    features = np.asarray(features)
    votes = np.zeros(features.shape)
    for i in range(features.shape[-1]):
        assign = features[:, i] > _threshold_otsu(features[:, i])
        if i > 0:
            m = np.mean(votes[:, :i], axis=1)
            if np.mean(np.abs(~assign - m)) < np.mean(np.abs(assign - m)):
                assign = ~assign
        votes[:, i] = assign
    return np.mean(votes, axis=1) > 0.5


def _threshold_otsu(values, nbins=256):
    """Otsu threshold on a 1-D sample (the reference takes it from skimage.filters, graph_cuts.py:183)"""
    hist, edges = np.histogram(np.asarray(values, dtype=float).ravel(), bins=nbins)
    centers = (edges[:-1] + edges[1:]) / 2.
    hist = hist.astype(float)
    w1 = np.cumsum(hist)
    w2 = np.cumsum(hist[::-1])[::-1]
    m1 = np.cumsum(hist * centers) / np.maximum(w1, 1e-300)
    m2 = (np.cumsum((hist * centers)[::-1]) / np.maximum(w2[::-1], 1e-300))[::-1]
    var12 = w1[:-1] * w2[1:] * (m1[:-1] - m2[1:]) ** 2
    return centers[:-1][np.argmax(var12)]


def estim_class_model_gmm(features, nb_classes, init='kmeans'):
    """ GMM over the features, optionally initialised by k-means (reference graph_cuts.py:221-249) """
    from sklearn import cluster, mixture
    gmm = mixture.GaussianMixture(n_components=nb_classes, covariance_type='full', max_iter=99)
    if init == 'kmeans':
        y = cluster.KMeans(n_clusters=nb_classes, init='k-means++').fit_predict(features)
        gmm.fit(features, y)
    else:
        gmm.fit(features)
    return gmm


def estim_class_model_kmeans(features, nb_classes, init_type='k-means++', max_iter=99):
    """ Gaussians fitted on a k-means clustering (reference graph_cuts.py:252-285) """
    from sklearn import cluster, mixture
    if init_type == 'quantiles':
        init_perc = np.array(np.percentile(features, np.linspace(5, 95, nb_classes).tolist(), axis=0))
        kmeans = cluster.KMeans(nb_classes, init=init_perc, max_iter=2)
    else:
        kmeans = cluster.KMeans(nb_classes, init=init_type, max_iter=max_iter, n_init=max(1, int(np.sqrt(max_iter))))
    y = kmeans.fit_predict(features)
    gmm = mixture.GaussianMixture(n_components=nb_classes, covariance_type='full', max_iter=1)
    gmm.fit(features, y)
    return gmm, y


def class_model_spec(estim_model, nb_classes, max_iter=99):
    """ (kind, n_init, max_iter) of the mixture that :func:`estim_class_model` fits for ``estim_model`` (reference
    graph_cuts.py:107-163).  The reference's ``Pipeline.fit(X, y)`` hands the k-means / Otsu labels it computes to
    ``GaussianMixture.fit``, which ignores them, so every variant but 'BGM' is a plain GaussianMixture with its own restart and
    iteration counts.  This is the one place that interprets ``estim_model`` for the device fit.

    :return tuple(str,int,int): kind 'GMM' (GaussianMixture) or 'BGM' (BayesianGaussianMixture), n_init, max_iter
    """
    nb_inits = max(1, int(np.sqrt(max_iter)))
    name, init_type = estim_model, ''
    if '_' in estim_model:
        name, init_type = estim_model.split('_')[0], estim_model.split('_')[-1]
    if name == 'GMM' and init_type in ('kmeans', 'Otsu'):
        return 'GMM', 1, max_iter
    if name == 'kmeans':
        return 'GMM', nb_inits, 1
    if name == 'BGM':
        return 'BGM', nb_inits, max_iter
    if name == 'Otsu' and nb_classes == 2:
        return 'GMM', 1, 1
    return 'GMM', nb_inits, max_iter


def _device_pca_coef(pca_coef, nb_features):
    """whether the device PCA takes this ``pca_coef``: None, a float in (0, 1) or a component count in [1, nb_features]"""
    if pca_coef is None:
        return True
    if isinstance(pca_coef, (bool, np.bool_)):
        return False
    if isinstance(pca_coef, (int, np.integer)):
        return 1 <= pca_coef <= nb_features
    return isinstance(pca_coef, (float, np.floating)) and 0. < pca_coef < 1.


def device_gmm_applicable(nb_features, nb_classes, estim_model='GMM', pca_coef=None):
    """ whether :func:`estim_class_model` fits on the device: any ``estim_model`` string, ``pca_coef`` as in
    :func:`_device_pca_coef`, <= 232 features and <= 8 classes ('mle' PCA and K > 8 stay on the host) """
    return (USE_DEVICE_GMM and isinstance(estim_model, str) and _device_pca_coef(pca_coef, nb_features)
            and nb_features <= DEVICE_GMM_MAX_FEATURES and nb_classes <= DEVICE_GMM_MAX_CLASSES)


def _pca_from_device(params, nb_features, pca_coef):
    """the fitted sklearn PCA of isb_pca_fit's parameters (host copy)"""
    from sklearn import decomposition
    p, D = np.asarray(params, dtype=np.float64), int(nb_features)
    o = 3 * D
    comp = p[o:o + D * D].reshape(D, D)
    o += D * D
    ev, ratio, sv = p[o:o + D], p[o + D:o + 2 * D], p[o + 2 * D:o + 3 * D]
    nc, noise, n_samples, ok = p[o + 4 * D:o + 4 * D + 4]
    if not ok:
        raise np.linalg.LinAlgError('the device eigensolver of the PCA did not converge')
    nc = int(nc)
    pca = decomposition.PCA(pca_coef)
    pca.mean_ = p[2 * D:3 * D].copy()
    pca.components_ = comp[:nc].copy()
    pca.explained_variance_, pca.explained_variance_ratio_, pca.singular_values_ = ev[:nc].copy(), ratio[:nc].copy(), sv[:nc].copy()
    pca.n_components_, pca.noise_variance_, pca.n_samples_, pca.n_features_in_ = nc, float(noise), int(n_samples), D
    pca._fit_svd_solver = 'covariance_eigh'
    return pca


def sklearn_pipeline_from_device(params, nb_features, nb_classes, nb_samples, use_scaler=True, n_init=1, max_iter=99, kind='GMM',
                                 pca_params=None, pca_coef=None, nb_features_in=None):
    """ wrap the parameters fitted by ``isb_mixture_fit_predict`` (and ``isb_pca_fit``) into the
    scikit-learn objects the reference returns (Pipeline[StandardScaler?, PCA?, GaussianMixture | BayesianGaussianMixture]) so that
    ``predict_proba`` & co. keep working on the host.  With ``pca_params`` the scaler is the PCA fit's and ``nb_features`` counts
    the PCA components the mixture saw; ``nb_features_in`` is then the width of the raw features. """
    from sklearn import mixture, pipeline, preprocessing
    p = np.asarray(params, dtype=np.float64)
    D, K = int(nb_features), int(nb_classes)
    mean, scale = p[:D].copy(), p[D:2 * D].copy()
    o = 2 * D
    weights = p[o:o + K].copy()
    o += K
    means = p[o:o + K * D].reshape(K, D).copy()
    o += K * D
    covs = p[o:o + K * D * D].reshape(K, D, D).copy()
    o += K * D * D
    prec_chol = p[o:o + K * D * D].reshape(K, D, D).copy()
    o += K * D * D
    lower, n_iter, converged, ok = p[o:o + 4]
    if not ok:
        raise ValueError('Fitting the mixture model failed because some components have ill-defined empirical covariance '
                         '(for instance caused by singleton or collapsed samples). Try to decrease the number of components')
    steps = []
    if pca_params is not None:
        D_in = int(nb_features_in)
        if use_scaler:
            pp = np.asarray(pca_params, dtype=np.float64)
            mean, scale = pp[:D_in].copy(), pp[D_in:2 * D_in].copy()
        pca = _pca_from_device(pca_params, D_in, pca_coef)
    else:
        D_in = D
    if use_scaler:
        sc = preprocessing.StandardScaler()
        sc.mean_, sc.scale_, sc.var_ = mean, scale, scale ** 2
        sc.n_features_in_, sc.n_samples_seen_ = D_in, int(nb_samples)
        steps.append(('std_scaler', sc))
    if pca_params is not None:
        steps.append(('reduce_dim', pca))
    if kind == 'BGM':
        nk = weights
        mm = mixture.BayesianGaussianMixture(n_components=K, covariance_type='full', n_init=n_init, max_iter=max_iter)
        o += 5   # lower_bound | n_iter | converged | ok | best_init, then the priors
        mm.weight_concentration_prior_, mm.mean_precision_prior_, mm.degrees_of_freedom_prior_ = 1. / K, 1., float(D)
        mm.mean_prior_, mm.covariance_prior_ = p[o:o + D].copy(), p[o + D:o + D + D * D].reshape(D, D).copy()
        # _estimate_weights / _estimate_means / _estimate_wishart_full from nk, then sklearn's own weights_ and precisions_
        wc = (1. + nk, 1. / K + np.hstack((np.cumsum(nk[::-1])[-2::-1], 0)))
        mm._set_parameters((wc, 1. + nk, means, D + nk, covs, prec_chol))
    else:
        mm = mixture.GaussianMixture(n_components=K, covariance_type='full', n_init=n_init, max_iter=max_iter)
        mm.weights_, mm.means_, mm.covariances_, mm.precisions_cholesky_ = weights, means, covs, prec_chol
        mm.precisions_ = np.array([u @ u.T for u in prec_chol])
    mm.converged_, mm.n_iter_, mm.lower_bound_, mm.n_features_in_ = bool(converged), int(n_iter), float(lower), D
    steps.append(('model', mm))
    return pipeline.Pipeline(steps)


def device_fit_predict(eng, d_feat, nb_classes, use_scaler, kind, n_init, max_iter, pca_coef=None, seed=None, d_n=None, init_labels=None):
    """ the class model fitted on device features [N, D] and evaluated on them, nothing leaves the device (a float ``pca_coef``
    reads its component count back): returns (proba [N, K] device, mixture params, PCA params or None, dimensions the mixture saw) """
    seed = RANDOM_SEED if seed is None else seed
    d_pca, dims = None, int(d_feat.shape[1])
    if pca_coef is not None:
        d_feat, d_pca, dims = eng.pca_fit_transform(d_feat, use_scaler, pca_coef, d_n=d_n)
        use_scaler = False   # the PCA fit owns the scaler
    proba, params = eng.mixture_fit_predict(d_feat, nb_classes, n_init, max_iter, use_scaler, seed, d_n=d_n, init_labels=init_labels,
                                            kind=kind)
    return proba, params, d_pca, dims


def _check_pca_count(pca_coef, nb_samples, nb_features):
    """ the ValueError of the reference's ``PCA(pca_coef)`` (scikit-learn's ``PCA._fit_full``) for a component count above
    min(n_samples, n_features), raised before any device work; the message names the solver scikit-learn's 'auto' picks """
    N, D = int(nb_samples), int(nb_features)
    if isinstance(pca_coef, (int, np.integer)) and not isinstance(pca_coef, (bool, np.bool_)) and pca_coef > min(N, D):
        solver = 'covariance_eigh' if D <= 1000 and N >= 10 * D else 'full'
        raise ValueError('n_components=%d must be between 0 and min(n_samples, n_features)=%d with svd_solver=%r'
                         % (pca_coef, min(N, D), solver))


def fit_class_model_device(features, nb_classes, use_scaler, kind, n_init, max_iter, pca_coef=None, init_labels=None, seed=None):
    """ the class model of a :func:`class_model_spec` triple fitted on the GPU: the same kind of object as :func:`estim_class_model` """
    features = np.ascontiguousarray(features, dtype=np.float64)
    _check_pca_count(pca_coef, features.shape[0], features.shape[1])
    eng = get_engine()
    d_feat = eng.to_device(features, 'feat_in')
    if init_labels is not None:
        init_labels = np.atleast_2d(init_labels)
    _, params, d_pca, dims = device_fit_predict(eng, d_feat, nb_classes, use_scaler, kind, n_init, max_iter, pca_coef, seed,
                                                init_labels=init_labels)
    return sklearn_pipeline_from_device(eng.to_host(params), dims, nb_classes, len(features), use_scaler, n_init, max_iter, kind,
                                        None if d_pca is None else eng.to_host(d_pca), pca_coef, features.shape[1])


def estim_class_model_device(features, nb_classes, use_scaler=True, max_iter=99, init_labels=None, seed=None, estim_model='GMM',
                             pca_coef=None):
    """ :func:`estim_class_model` fitted on the GPU (every ``estim_model`` variant, optional PCA); ``init_labels`` [n_init, N]
    replaces the device k-means++ start (one restart per row) """
    kind, n_init, max_iter = class_model_spec(estim_model, nb_classes, max_iter)
    if init_labels is not None:
        n_init = len(np.atleast_2d(init_labels))
    return fit_class_model_device(features, nb_classes, use_scaler, kind, n_init, max_iter, pca_coef, init_labels, seed)


def estim_class_model(features, nb_classes, estim_model='GMM', pca_coef=None, use_scaler=True, max_iter=99):
    """ scikit-learn pipeline (scaler, PCA, mixture model) fitted on the features (reference graph_cuts.py:73-163)

    :param ndarray features: [nb_samples, nb_features]
    :param int nb_classes: number of classes
    :param str estim_model: 'GMM', 'GMM_kmeans', 'GMM_Otsu', 'kmeans', 'kmeans_quantiles', 'BGM', 'Otsu'
    :return: fitted sklearn Pipeline with ``predict_proba``
    """
    features = np.asarray(features)
    if device_gmm_applicable(features.shape[1], nb_classes, estim_model, pca_coef):
        import torch
        if torch.cuda.is_available():
            return estim_class_model_device(features, nb_classes, use_scaler, max_iter, estim_model=estim_model, pca_coef=pca_coef)
    from sklearn import cluster, decomposition, mixture, pipeline, preprocessing
    steps = []
    if use_scaler:
        steps.append(('std_scaler', preprocessing.StandardScaler()))
    if pca_coef is not None:
        steps.append(('reduce_dim', decomposition.PCA(pca_coef)))
    nb_inits = max(1, int(np.sqrt(max_iter)))
    mm = mixture.GaussianMixture(n_components=nb_classes, covariance_type='full', n_init=nb_inits, max_iter=max_iter)
    init_type = ''
    if '_' in estim_model:
        estim_model, init_type = estim_model.split('_')[0], estim_model.split('_')[-1]
    y = None
    if estim_model == 'GMM':
        if init_type == 'kmeans':
            mm.set_params(n_init=1)
            y = cluster.KMeans(n_clusters=nb_classes, init='k-means++').fit_predict(features)
        elif init_type == 'Otsu':
            mm.set_params(n_init=1)
            y = compute_multivarian_otsu(features)
    elif estim_model == 'kmeans':
        mm.set_params(max_iter=1)
        init_type = 'quantiles' if init_type == 'quantiles' else 'k-means++'
        _, y = estim_class_model_kmeans(features, nb_classes, init_type=init_type, max_iter=max_iter)
    elif estim_model == 'BGM':
        mm = mixture.BayesianGaussianMixture(n_components=nb_classes, covariance_type='full', n_init=nb_inits,
                                             max_iter=max_iter)
    elif estim_model == 'Otsu' and nb_classes == 2:
        mm.set_params(max_iter=1, n_init=1)
        y = compute_multivarian_otsu(features)
    steps.append(('model', mm))
    model = pipeline.Pipeline(steps)
    if y is not None:
        model.fit(features, y)
    else:
        model.fit(features)
    return model


# ---------------------------------------------------------------------------------------------------------------------
# graph + energies
# ---------------------------------------------------------------------------------------------------------------------

def get_vertexes_edges(segments):
    """ vertices and edges of the region adjacency graph, 2-D or 3-D (reference graph_cuts.py:288-300) """
    segments = np.asarray(segments)
    if segments.ndim == 3:
        return make_graph_segm_connect_grid3d_conn6(segments)
    if segments.ndim == 2:
        return make_graph_segm_connect_grid2d_conn4(segments)
    return None, None


def compute_spatial_dist(centres, edges, relative=False):
    """ Euclidean distance between the centres of connected segments (reference graph_cuts.py:303-336) """
    if np.max(edges) >= len(centres):
        raise ValueError('max vertex %i exceed size of centres %i' % (np.max(edges), len(centres)))
    ndim = np.max([len(c) for c in centres if c is not None])
    centres = [[np.nan] * ndim if (c is None or len(c) == 0) else c for c in centres]
    centres = np.nan_to_num(np.asarray(centres, dtype=float))
    edges = np.asarray(edges)
    diff = centres[edges[:, 0]] - centres[edges[:, 1]]
    dist = np.sqrt(np.einsum('ij,ij->i', diff, diff))
    if relative:
        dist = dist / np.mean(dist)
    return dist


def compute_edge_model(edges, proba, metric='l_T'):
    """ edge weight exp(-d / (2 std(d)^2)) from the class probabilities of the two vertices, d by ``metric``
    'l1' / 'l2' / 'lT' (reference graph_cuts.py:383-439) """
    edges, proba = np.asarray(edges), np.asarray(proba)
    if np.max(edges) >= len(proba):
        raise ValueError('max vertex %i exceed size of proba %r' % (np.max(edges), proba.shape))
    v1, v2 = proba[edges[:, 0]], proba[edges[:, 1]]
    if metric == 'l1':
        dist = np.abs(v1 - v2).sum(axis=1)
    elif metric == 'l2':
        d = v1 - v2
        dist = np.sqrt(np.einsum('ij,ij->i', d, d))
    elif metric == 'lT':
        dist = np.max((v1 - v2) ** 2, axis=1)
    else:
        logging.error('not implemented for: %s', metric)
        return np.ones(len(edges))
    return np.exp(-dist / (2 * np.std(dist) ** 2))


def create_pairwise_matrix_uniform(gc_reg, nb_classes):
    """ Potts matrix gc_reg * (1 - I) (reference graph_cuts.py:442-456) """
    return (np.ones(nb_classes) - np.eye(nb_classes)) * gc_reg


def create_pairwise_matrix_specif(pos_weights, nb_classes=None):
    """ Potts matrix with given symmetric entries (reference graph_cuts.py:459-482) """
    if not nb_classes:
        nb_classes = np.max([list(c) for c, _ in pos_weights]) + 1
    pairwise = np.ones(nb_classes) - np.eye(nb_classes)
    for (i, j), w in pos_weights:
        pairwise[i, j] = pairwise[j, i] = w
    return pairwise


def create_pairwise_matrix(gc_regul, nb_classes):
    """ uniform / listed / full-matrix pairwise term (reference graph_cuts.py:485-520) """
    if isinstance(gc_regul, np.ndarray):
        if not gc_regul.shape[0] == gc_regul.shape[1] == nb_classes:
            raise ValueError('GC regul matrix %r should match match number of classes (%i)' % (gc_regul.shape, nb_classes))
        return gc_regul - np.min(gc_regul)
    if isinstance(gc_regul, list):
        return create_pairwise_matrix_specif(gc_regul, nb_classes)
    return create_pairwise_matrix_uniform(gc_regul, nb_classes)


def compute_unary_cost(proba, min_prob=MIN_UNARY_PROB):
    """ |-log(clip(proba, min_prob, 1 - min_prob))| (reference graph_cuts.py:523-540) """
    proba = np.clip(np.asarray(proba, dtype=float), min_prob, 1 - min_prob)
    return np.abs(np.array(-np.log(proba), dtype=np.float64))


def compute_pairwise_cost(gc_regul, proba_shape, max_pairwise_cost=MAX_PAIRWISE_COST):
    """ pairwise matrix capped at ``max_pairwise_cost`` (reference graph_cuts.py:543-555) """
    cost = np.array(create_pairwise_matrix(gc_regul, proba_shape[1]), dtype=np.float64)
    cost[cost > max_pairwise_cost] = max_pairwise_cost
    return cost


def insert_gc_debug_images(debug_visual, segments, graph_labels, unary_cost, edges, edge_weights):
    """ raw intermediates for debugging (reference graph_cuts.py:558-571; the rendered figures of
    ``imsegm.utilities.drawing`` are out of scope, the arrays they are drawn from are kept) """
    if debug_visual is None:
        return
    debug_visual['segments'] = segments
    debug_visual['edges'] = edges
    debug_visual['edge_weights'] = edge_weights
    debug_visual['imgs_unary_cost'] = [np.asarray(unary_cost)[:, i][segments] for i in range(np.asarray(unary_cost).shape[1])]
    debug_visual['img_graph_edges'] = None
    debug_visual['img_graph_segm'] = np.asarray(graph_labels)[segments]


def _edge_mode(edge_type):
    if edge_type.startswith('model'):
        metric = edge_type.split('_')[-1] if '_' in edge_type else 'lT'
        key = 'model_' + metric
        if edge_type == 'model':
            return EDGE_MODES['model']
        if key not in EDGE_MODES:
            logging.error('not implemented for: %s', metric)
            return EDGE_MODES['']
        return EDGE_MODES[key]
    return EDGE_MODES.get(edge_type, EDGE_MODES[''])


def _device_energies(eng, segments, proba, edge_type, edge_cost, pairwise):
    """label map [H, W] + class probabilities [>= nb, K] -> (device edges, E, what :meth:`~.engine.Engine.gc_energies` returns)"""
    nb = int(segments.max()) + 1
    if len(proba) < nb:
        raise ValueError('max vertex %i exceed size of proba %r' % (nb - 1, proba.shape))
    mode = _edge_mode(edge_type)
    d_seg = eng.to_device(segments.astype(np.int32, copy=False), 'seg_in')
    d_edges, E = device_adjacency(eng, d_seg, nb)
    d_proba = eng.to_device(proba, 'proba')
    centres = None
    if mode[1]:
        _, centres, _ = eng.segment_stats(None, d_seg, nb, (), want_centres=True)
    return d_edges, E, eng.gc_energies(d_proba, d_edges, E, None, centres, mode, float(edge_cost), pairwise)


def check_edge_type(edge_type):
    """ValueError unless the device pipelines know ``edge_type``: '', 'spatial', 'model', 'model_lT' / '_l1' / '_l2', 'color' or
    'features' (compute_edge_weights would weight any other name by ones)"""
    if not (isinstance(edge_type, str) and (edge_type in EDGE_MODES or edge_type in VECTOR_EDGE_METRICS)):
        raise ValueError('unknown gc_edge_type %r: expected one of %s' % (edge_type, sorted(set(EDGE_MODES) | set(VECTOR_EDGE_METRICS))))


def reference_edge_type(edge_type):
    """the edge type whose device weights are those compute_edge_weights gives ``edge_type``: itself when :func:`check_edge_type`
    takes it, else '' -- the reference weights an unknown name, or a 'model_<metric>' of an unknown metric, by ones without the
    spatial term"""
    if isinstance(edge_type, str) and (edge_type in EDGE_MODES or edge_type in VECTOR_EDGE_METRICS):
        return edge_type
    _edge_mode(edge_type)     # logs an unknown model metric as the reference does
    return ''


def device_edge_vectors(eng, edge_type, d_img, d_seg, nb, d_feat, d_n):
    """the per-label vectors [nb, D] (device) that compute_edge_weights compares for ``edge_type``, None for the types that need
    none; nothing is read back.  'color': the mean RGB of the image as np.array(image, dtype=float), divided by 255 when its maximum
    is above 1 (labels [H, W] of an [H, W, 3] device image); 'features': the feature table [>= nb, D] standardised by StandardScaler
    over the ``d_n`` (device) real rows.  The device feature tables hold no NaN (every statistic kernel writes np.nan_to_num's
    values), so they are already the table with NaN set to 0 that compute_color2d_superpixels_features returns."""
    if edge_type == 'color':
        if d_img.dim() != 3 or int(d_img.shape[2]) != 3:
            raise ValueError("gc_edge_type 'color' needs an RGB image [H, W, 3], got shape %r" % (tuple(d_img.shape), ))
        vec = eng.buf('edge_vec', (nb, 3), eng.torch.float64)
        eng.group_stats(eng.unit_scaled_image(d_img), d_seg, nb, ('mean', ), vec, 0)
        return vec
    if edge_type == 'features':
        return eng.standard_scaler(d_feat, d_n, names=('edge_feat', 'edge_feat_params'))[0]
    return None


def device_graphcut(eng, d_seg, d_centres, nb, d_proba, gc_regul, gc_edge_type, d_n_nodes, edge_cap, edge_vectors=None):
    """graph-cut tail of the device pipelines over the label map ``d_seg`` and its centroids ``d_centres``: adjacency,
    energies, alpha-expansion (all asynchronous).  A label volume [D, H, W] takes its 6-connected graph and its (z, y, x) centroids
    from :meth:`~.engine.Engine.graph3d` instead (pass ``d_centres`` None).  ``nb`` may be an upper bound of the label count
    when ``d_n_nodes`` (device scalar) carries the real one.  'color' and 'features' weigh the edges of a label map by the vectors
    ``edge_vectors`` [nb, D] (device, :func:`device_edge_vectors`).  Returns (class per label [nb] device, n_edges device int32[1]);
    the result only holds when the table of ``edge_cap`` rows took every edge, see :func:`~.engine.edges_fit`"""
    check_edge_type(gc_edge_type)
    metric = VECTOR_EDGE_METRICS.get(gc_edge_type)
    if metric is not None and (d_seg.dim() != 2 or edge_vectors is None):
        raise ValueError('gc_edge_type %r compares per-superpixel vectors over a 2-D label map: pass them as edge_vectors' % gc_edge_type)
    K = int(d_proba.shape[1])
    pairwise = compute_pairwise_cost(gc_regul, (nb, K))
    if d_seg.dim() == 3:
        d_edges, d_n_edges, _, d_centres = eng.graph3d(d_seg, nb, edge_cap)
    else:
        d_edges, d_n_edges, _ = eng.adjacency(d_seg, nb, edge_cap)
    mode, edge_w = _edge_mode(gc_edge_type), None
    if metric is not None:
        edge_w = eng.vector_edge_weights(edge_vectors, d_edges, edge_cap, d_n_edges, d_centres, metric)
        mode = EDGE_GIVEN
    _, _, unary_i, edge_wi, smooth_i = eng.gc_energies(d_proba, d_edges, edge_cap, d_n_edges, d_centres, mode, 1.0, pairwise,
                                                       d_n_nodes=d_n_nodes, edge_w=edge_w)
    d_labels, _, _ = eng.alpha_expansion(nb, K, edge_cap, d_n_edges, d_edges, edge_wi, unary_i, smooth_i, -1, d_n_nodes=d_n_nodes)
    return d_labels, d_n_edges


def compute_edge_weights(segments, image=None, features=None, proba=None, edge_type=''):
    """ edges of the superpixel graph and their weights (reference graph_cuts.py:574-657)

    :param ndarray segments: superpixels
    :param str edge_type: '', 'spatial', 'model[_l1|_l2|_lT]', 'color', 'features'
    :return tuple(ndarray,ndarray): edges [E, 2] int32, weights [E] float64 clamped to [1e-3, 1e3]
    """
    segments = np.asarray(segments)
    eng = get_engine()
    if edge_type.startswith('model') and (proba is None or len(proba) == 0):
        raise ValueError('"proba" is required')
    if edge_type in ('color', 'features'):
        # these two compare host-side vectors (mean colour / standardised features): same kernel, different vectors
        _, edges = get_vertexes_edges(segments)
        edges = np.array(edges, dtype=np.int32)
        if edge_type == 'color':
            if image is None:
                raise RuntimeError('"image" is required')
            from .descriptors import compute_selected_features_img2d
            image_float = np.array(image, dtype=float)
            if np.max(image) > 1:
                image_float /= 255.
            vec, _ = compute_selected_features_img2d(image_float, segments, {'color': ['mean']})
            dist = np.abs(vec[edges[:, 0]] - vec[edges[:, 1]]).sum(axis=1)
        else:
            if features is None:
                raise RuntimeError('"features" is required')
            from sklearn import preprocessing
            vec = preprocessing.StandardScaler().fit_transform(features)
            d = vec[edges[:, 0]] - vec[edges[:, 1]]
            dist = np.sqrt(np.einsum('ij,ij->i', d, d))
        weights = np.exp(-(dist.astype(float) / (2 * np.std(dist) ** 2)))
        weights /= compute_spatial_dist(superpixel_centers(segments), edges, relative=True)
        weights[weights < 1. / MIN_MAX_EDGE_WEIGHT] = 1. / MIN_MAX_EDGE_WEIGHT
        weights[weights > MIN_MAX_EDGE_WEIGHT] = MIN_MAX_EDGE_WEIGHT
        return edges, weights
    if segments.ndim == 3:
        return _edge_weights_volume(eng, segments, proba, edge_type)
    K = 1 if proba is None else int(np.asarray(proba).shape[1])
    p = np.ones((int(segments.max()) + 1, K)) if proba is None else np.ascontiguousarray(proba, dtype=np.float64)
    d_edges, E, (_, edge_w, _, _, _) = _device_energies(eng, segments, p, edge_type, 1.0, np.zeros((K, K)))
    edges = eng.to_host(d_edges[:E]).copy() if E else np.zeros((0, 2), dtype=np.int32)
    weights = eng.to_host(edge_w[:E]).copy() if E else np.zeros(0)
    return edges, weights


def _edge_weights_volume(eng, segments, proba, edge_type):
    """edges and weights of a label VOLUME: the 6-connected pairs and the centres come from the device (isb_adjacency_edges_3d,
    isb_centroids_3d), the per-edge arithmetic -- a few thousand edges -- follows the reference on the host (graph_cuts.py:617-657)"""
    _edge_mode(edge_type)     # validates the name
    nb = int(segments.max()) + 1
    d_seg = eng.to_device(segments.astype(np.int32, copy=False), 'seg_in3d')
    E, (d_edges, _, _, d_centres) = eng.edge_table(lambda cap: eng.graph3d(d_seg, nb, cap), nb, ndim=3)
    edges = eng.to_host(d_edges[:E]).copy() if E else np.zeros((0, 2), dtype=np.int32)
    if not E:
        return edges, np.zeros(0)
    if edge_type.startswith('model'):
        metric = edge_type.split('_')[-1] if '_' in edge_type else 'lT'
        weights = np.array(compute_edge_model(edges, proba, metric), dtype=float)
    else:
        weights = np.ones(len(edges))
    if edge_type in ('model', 'spatial'):
        weights = weights / compute_spatial_dist(eng.to_host(d_centres).copy(), edges, relative=True)
    weights[weights < 1. / MIN_MAX_EDGE_WEIGHT] = 1. / MIN_MAX_EDGE_WEIGHT
    weights[weights > MIN_MAX_EDGE_WEIGHT] = MIN_MAX_EDGE_WEIGHT
    return edges, weights


def segment_graph_cut_general(segments, proba, image=None, features=None, gc_regul=1., edge_type='model', edge_cost=1.,
                              debug_visual=None):
    """ GraphCut labelling of the superpixels (reference graph_cuts.py:660-747)

    :param ndarray segments: superpixel map
    :param ndarray proba: class probabilities per superpixel [N, K]
    :param gc_regul: regularisation (float, list of ((i, j), w) or full matrix)
    :param str edge_type: see :func:`compute_edge_weights`
    :return ndarray: label per superpixel, int32
    """
    segments = np.asarray(segments)
    proba = np.ascontiguousarray(proba, dtype=np.float64)
    pairwise_cost = compute_pairwise_cost(gc_regul, proba.shape)
    scalar_regul = not isinstance(gc_regul, (list, np.ndarray))
    if scalar_regul and gc_regul <= 0:
        unary_cost = compute_unary_cost(proba)
        graph_labels = np.argmin(unary_cost, axis=-1).astype(np.int32)
        if debug_visual is not None:
            edges, edge_weights = compute_edge_weights(segments, image, features, proba, edge_type)
            insert_gc_debug_images(debug_visual, segments, graph_labels, unary_cost, edges, edge_weights * edge_cost)
        return graph_labels
    eng = get_engine()
    if edge_type in ('color', 'features') or segments.ndim == 3:
        edges, edge_weights = compute_edge_weights(segments, image, features, proba, edge_type)
        edge_weights = edge_weights * edge_cost
        unary_cost = compute_unary_cost(proba)
        graph_labels = cut_general_graph(edges, edge_weights, unary_cost, pairwise_cost, n_iter=-1)
    else:
        d_edges, E, (unary, edge_w, unary_i, edge_wi, smooth_i) = _device_energies(eng, segments, proba, edge_type, edge_cost,
                                                                                    pairwise_cost)
        labels, _, _ = eng.alpha_expansion(len(proba), proba.shape[1], E, None, d_edges, edge_wi, unary_i, smooth_i, -1)
        graph_labels = eng.to_host(labels).copy()
        if debug_visual is not None:
            edges, edge_weights = eng.to_host(d_edges[:E]).copy(), eng.to_host(edge_w[:E]).copy()
            unary_cost = eng.to_host(unary).copy()
    if debug_visual is not None:
        insert_gc_debug_images(debug_visual, segments, graph_labels, unary_cost, edges, edge_weights)
    return graph_labels


def _canonical_int_edges(edges, w_i):
    """pairs as (a, b) with a < b, self loops dropped, parallel edges merged by adding their (already integer) weights -- the energy
    GCO builds when ``setNeighbors`` is called for both orders or twice for the same pair"""
    edges = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    lo, hi = edges.min(axis=1), edges.max(axis=1)
    keep = lo != hi
    lo, hi, w_i = lo[keep], hi[keep], np.asarray(w_i, dtype=np.int64)[keep]
    if not len(lo):
        return np.zeros((0, 2), np.int32), np.zeros(0, np.intc)
    key = lo * (int(hi.max()) + 1) + hi
    uniq, inverse = np.unique(key, return_inverse=True)
    if len(uniq) == len(key) and (edges[keep][:, 0] < edges[keep][:, 1]).all():
        return np.ascontiguousarray(edges[keep], dtype=np.int32), np.ascontiguousarray(w_i, dtype=np.intc)
    merged_w = np.bincount(inverse, weights=w_i.astype(np.float64), minlength=len(uniq))
    first = np.zeros(len(uniq), dtype=np.int64)
    first[inverse[::-1]] = np.arange(len(key))[::-1]                      # first occurrence of every pair
    order = np.argsort(first, kind='stable')
    out = np.stack([lo[first], hi[first]], axis=1)[order]
    return np.ascontiguousarray(out, dtype=np.int32), np.ascontiguousarray(np.minimum(merged_w[order], 2 ** 31 - 1), dtype=np.intc)


def integerise_energies(edge_weights, unary_cost, pairwise_cost, down_weight_factor=None):
    """ pyGCO's float -> int conversion of ``cut_general_graph``, as ``k_gc_energies`` (csrc/graph.cu) does it on the device:
    truncation towards zero of ``unary / f * 1e5``, ``w / f * 1e3`` and ``pairwise * 100`` with
    ``f = max(|unary|.max(), |w|.max() * pairwise.max()) + 1e-10``.  An edge weight that is NaN (a degenerate edge model: every
    edge at the same distance, or coincident centroids under a weight that underflowed, DESIGN.md section 2) is left out of ``f``
    and becomes capacity 0, where pyGCO's C cast of NaN is undefined; no edge (E = 0) counts as a largest weight of 0.

    :return tuple(ndarray,ndarray,ndarray): int32 (edge weights [E], unary [N, K], pairwise [K, K])
    """
    w, un, pw = np.asarray(edge_weights), np.asarray(unary_cost), np.asarray(pairwise_cost)   # in their own types, as pyGCO does
    nan_w = np.isnan(w)
    if down_weight_factor is None:
        w_max = np.abs(w[~nan_w]).max() if not nan_w.all() else 0.
        down_weight_factor = max(np.abs(un).max(), w_max * pw.max()) + 1e-10
    un_i = (un / down_weight_factor * 100000).astype(np.intc)
    w_i = ((np.where(nan_w, 0, w) if nan_w.any() else w) / down_weight_factor * 1000).astype(np.intc)
    return w_i, un_i, (pw * 100).astype(np.intc)


def cut_general_graph(edges, edge_weights, unary_cost, pairwise_cost, n_iter=-1, algorithm='expansion', init_labels=None,
                      down_weight_factor=None):
    """ drop-in for ``gco.cut_general_graph`` (pyGCO) as the reference calls it (graph_cuts.py:735-744,
    region_growing.py:148,1698): float energies are integerised like pyGCO does, alpha-expansion runs on the GPU.  Edges may come in
    either orientation and more than once (region_growing.py:1433-1444 lists an edge from both of its ends): parallel edges add up.

    :return ndarray: labels int32 [N]
    """
    if algorithm != 'expansion':
        raise NotImplementedError('only algorithm="expansion" is used by the reference hot path')
    eng = get_engine()
    w = np.asarray(edge_weights)
    un = np.asarray(unary_cost)
    pw = np.asarray(pairwise_cost)
    is_float = any(a.dtype.kind == 'f' for a in (w, un, pw))
    if is_float:
        w_i, un_i, pw_i = integerise_energies(w, un, pw, down_weight_factor)
    else:
        un_i, w_i, pw_i = un.astype(np.intc), w.astype(np.intc), pw.astype(np.intc)
    edges, w_i = _canonical_int_edges(edges, w_i)
    N, K = un_i.shape
    if len(edges) and int(edges.max()) >= N:
        raise ValueError('an edge refers to vertex %d, the unary table has %d rows' % (int(edges.max()), N))
    E = len(edges)
    d_edges = eng.to_device(edges if E else np.zeros((1, 2), np.int32), 'edges_in')
    d_w = eng.to_device(np.ascontiguousarray(w_i) if E else np.zeros(1, np.intc), 'edge_wi_in')
    d_un = eng.to_device(np.ascontiguousarray(un_i), 'unary_i_in')
    d_pw = eng.to_device(np.ascontiguousarray(pw_i), 'smooth_i_in')
    init = None
    if init_labels is not None:
        init = eng.to_device(np.ascontiguousarray(init_labels, dtype=np.int32), 'init_labels')
    labels, _, stats = eng.alpha_expansion(N, K, E, None, d_edges, d_w, d_un, d_pw, int(n_iter), init)
    (labels, stats), done = eng.download((labels, stats))
    done.synchronize()
    _raise_on_refused_move(stats.numpy())
    return labels.numpy().copy()


def _raise_on_refused_move(stats):
    """the device refuses an expansion move whose capacities do not fit its 32-bit flow arrays (``stats`` of isb_alpha_expansion);
    GCO would solve that move, so the labels would differ from pyGCO's: raise instead of returning them"""
    if stats[6]:
        raise RuntimeError('alpha-expansion: a terminal capacity of a move reached 2^29 (unary costs plus the edge terms they absorb '
                           'must stay below 2^29)')
    if stats[7]:
        raise RuntimeError('alpha-expansion: a pair capacity of a move reached 2^30 (w_ij * (V[a, alpha] + V[alpha, b] - V[a, b] - '
                           'V[alpha, alpha]) must stay below 2^30)')


def cut_grid_graph(unary_cost, pairwise_cost, cost_v, cost_h, n_iter=-1, algorithm='expansion'):
    """ drop-in for ``gco.cut_grid_graph`` (pyGCO) as the reference calls it (region_growing.py:248): alpha-expansion over the
    4-connected pixel grid, ``cost_v[y, x]`` weighting the edge (y, x)-(y+1, x) and ``cost_h[y, x]`` the edge (y, x)-(y, x+1)

    :param ndarray unary_cost: [H, W, K]
    :return ndarray: labels int32 [H * W]
    """
    unary_cost = np.asarray(unary_cost)
    height, width, nb_labels = unary_cost.shape
    idx = np.arange(height * width).reshape(height, width)
    edges = np.concatenate([np.stack([idx[:-1].ravel(), idx[1:].ravel()], 1), np.stack([idx[:, :-1].ravel(), idx[:, 1:].ravel()], 1)])
    weights = np.concatenate([np.asarray(cost_v, dtype=float).ravel(), np.asarray(cost_h, dtype=float).ravel()])
    return cut_general_graph(edges, weights, unary_cost.reshape(-1, nb_labels), pairwise_cost, n_iter=n_iter, algorithm=algorithm,
                             down_weight_factor=1.0)


def count_label_transitions_connected_segments(dict_slics, dict_labels, nb_labels=None):
    """ label co-occurrence counts over connected segments (reference graph_cuts.py:750-793) """
    if not nb_labels:
        nb_labels = int(max(np.max(lbs) for lbs in dict_labels.values())) + 1
    transitions = np.zeros((nb_labels, nb_labels))
    for name in dict_slics:
        if (np.max(dict_slics[name]) + 1) != len(dict_labels[name]):
            raise ValueError('dims are not matching - max slic (%i) and label (%i)' %
                             (np.max(dict_slics[name]), len(dict_labels[name])))
        _, edges = get_vertexes_edges(dict_slics[name])
        pairs = np.asarray(dict_labels[name])[np.asarray(edges)]
        np.add.at(transitions, (pairs[:, 0], pairs[:, 1]), 1)
        np.add.at(transitions, (pairs[:, 1], pairs[:, 0]), 1)
    transitions[np.diag_indices(nb_labels)] /= 2
    return transitions


def compute_pairwise_cost_from_transitions(trans, min_prob=1e-9):
    """ pairwise cost log(1 / ratio) from the transition counts (reference graph_cuts.py:796-832) """
    trans = np.asarray(trans, dtype=float)
    ratio = trans / np.tile(np.sum(trans, axis=0), (len(trans), 1))
    ratio = np.maximum(ratio, ratio.T) if ratio.ndim == 2 else ratio
    ratio[ratio < min_prob] = min_prob
    return np.log(1. / ratio)
