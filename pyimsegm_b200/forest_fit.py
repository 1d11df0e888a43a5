"""
Fit scikit-learn's ``DecisionTreeClassifier`` and ``RandomForestClassifier`` on the device (``isb_forest_fit``, csrc/forest_fit.cu).

:func:`fit_tree_model` takes an unfitted estimator and returns it fitted, as the same scikit-learn type with the attributes a real
``fit`` leaves, so ``predict_proba``, pickling and ``class_models.compile_model`` work unchanged.  It returns ``None`` for a parameter
the device does not compute (the caller then fits on the host, as with ``compile_model``).

What matches scikit-learn 1.9: the float32 cast of X, the class encoding, the resolution of ``max_features`` / ``min_samples_split`` /
``min_samples_leaf``, the per-tree seeds and bootstrap rows drawn from the forest's ``random_state`` exactly as scikit-learn draws
them (so the bootstrap counts, ``estimators_samples_`` and every root are scikit-learn's), and the split rules at every node (Gini
proxy improvement, allowed positions, midpoint thresholds, leaf tests, preorder node ids).  What differs: the features a node draws.
scikit-learn draws them from one sequential RNG whose state runs through the nodes in depth-first order; the device hashes (tree seed,
breadth-first node index, feature) instead and takes the ``max_features`` non-constant features of least hash.  The distribution is the
same, the draws are not; with ``max_features`` equal to the number of features (or one feature) the trees are scikit-learn's node for
node, except that equal improvements go to the lowest feature index where scikit-learn keeps the first feature it drew.

:func:`fit_tree_models` fits many estimators, each on its own training rows and its own transformed features (the folds of a
cross-validation), in one device call (``isb_forest_fit_groups``): every tree of every forest is built level by level together, and
each tree is node for node the tree :func:`fit_tree_model` builds for that estimator alone.  The seeds and bootstrap rows are drawn
estimator by estimator in list order, so numpy's global RNG is consumed as scikit-learn's sequential fits consume it.

:func:`fit_extra_trees` fits an ``ExtraTreesClassifier`` (``isb_extra_trees_fit``, csrc/extra_trees_fit.cu) with scikit-learn's own
draws: each tree's splitter state is ``RandomState(tree seed).randint(0, 2^31 - 1)`` as ``Splitter.init`` draws it, and one CTA per
tree replays the depth-first build and every draw of ``node_split_random``, so the trees are scikit-learn's node for node and
``feature_importances_`` / ``predict_proba`` are its bits.  :func:`fit_tree_model` and the grouped fits do not take extra trees.
"""
import collections
import ctypes as C
import numbers
from math import ceil

import numpy as np

from . import _lib

#: isb_forest_fit's limits
MAX_CLASSES, MAX_FEATURES = 64, 2048
_MAX_INT = np.iinfo(np.int32).max
#: the most trees one isb_forest_fit_groups call builds; a larger batch goes in consecutive calls of whole forests
GROUP_MAX_TREES = 1 << 16
#: the share of the free device memory one isb_forest_fit_groups call may take
GROUP_MEMORY_SHARE = 0.8


def _supported(est):
    """the parameters of ``est`` that isb_forest_fit computes, or None"""
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.tree import DecisionTreeClassifier
    kind = type(est)
    if kind not in (DecisionTreeClassifier, RandomForestClassifier):
        return None
    p = est.get_params(deep=False)
    if p.get('criterion') != 'gini' or p.get('class_weight') is not None or p.get('max_leaf_nodes') is not None:
        return None
    if p.get('ccp_alpha', 0.0) > 0 or p.get('min_weight_fraction_leaf', 0.0) > 0 or p.get('monotonic_cst') is not None:
        return None
    if kind is DecisionTreeClassifier and p.get('splitter') != 'best':
        return None
    if kind is RandomForestClassifier and (p.get('max_samples') is not None or p.get('oob_score') or p.get('warm_start')):
        return None
    return p


def _resolve(p, n_samples, n_features):
    """(max_features, min_samples_split, min_samples_leaf, max_depth) as DecisionTreeClassifier._fit resolves them"""
    msl = p['min_samples_leaf']
    msl = msl if isinstance(msl, numbers.Integral) else int(ceil(msl * n_samples))
    mss = p['min_samples_split']
    mss = mss if isinstance(mss, numbers.Integral) else max(2, int(ceil(mss * n_samples)))
    mss = max(mss, 2 * msl)
    mf = p['max_features']
    if isinstance(mf, str):
        mf = max(1, int(np.sqrt(n_features))) if mf == 'sqrt' else max(1, int(np.log2(n_features)))
    elif mf is None:
        mf = n_features
    elif not isinstance(mf, numbers.Integral):
        mf = max(1, int(mf * n_features)) if mf > 0.0 else 0
    md = p['max_depth']
    return int(mf), int(mss), int(msl), (-1 if md is None else int(md))


def _fit_arrays(X, y, K, counts, seeds, max_features, min_samples_split, min_samples_leaf, max_depth, min_impurity_decrease):
    """every tree on the device: X [n, D] float32, y [n] class indices, counts [T, n], seeds [T] -> list of per-tree dicts of preorder
    node arrays (left, right, feature, threshold, impurity, n_node_samples, weighted_n_node_samples, missing_go_to_left,
    class_counts [nodes, K]) with 'node_count' and 'n_levels'"""
    import torch
    from .engine import get_engine
    eng = get_engine()
    lib, st = eng.lib, _lib.stream_ptr()
    n, D = X.shape
    T = len(counts)
    ws_bytes = lib.isb_forest_fit_workspace_bytes(n, D, T, K, max_features)
    if ws_bytes == 0:
        raise NotImplementedError('imsegm_b200: a forest of %d trees over %d rows x %d features with max_features %d is above the '
                                  'limits of isb_forest_fit' % (T, n, D, max_features))
    cap = 2 * int((counts > 0).sum(axis=1).max()) - 1
    d_x = eng.to_device(np.ascontiguousarray(X, dtype=np.float32), 'ff_x')
    d_y = eng.to_device(np.ascontiguousarray(y, dtype=np.int32), 'ff_y')
    d_c = eng.to_device(np.ascontiguousarray(counts, dtype=np.int32), 'ff_counts')
    d_s = eng.to_device(np.ascontiguousarray(seeds, dtype=np.uint64).view(np.int64), 'ff_seeds')
    i32, f64 = torch.int32, torch.float64
    out = {'left': eng.buf('ff_left', (T, cap), i32), 'right': eng.buf('ff_right', (T, cap), i32),
           'feature': eng.buf('ff_feature', (T, cap), i32), 'threshold': eng.buf('ff_threshold', (T, cap), f64),
           'impurity': eng.buf('ff_impurity', (T, cap), f64), 'n_node_samples': eng.buf('ff_n_node_samples', (T, cap), i32),
           'weighted_n_node_samples': eng.buf('ff_weighted', (T, cap), f64),
           'missing_go_to_left': eng.buf('ff_mgl', (T, cap), torch.uint8), 'class_counts': eng.buf('ff_class_counts', (T, cap, K), i32),
           'node_count': eng.buf('ff_node_count', T, i32)}
    ws = eng.buf('ff_ws', ws_bytes, torch.uint8)
    levels = C.c_int(0)
    names = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
             'class_counts', 'node_count')
    _lib.check(lib.isb_forest_fit(_lib.ptr(d_x), n, D, _lib.ptr(d_y), K, _lib.ptr(d_c), T, _lib.ptr(d_s), max_features, min_samples_split,
                                  min_samples_leaf, max_depth, C.c_double(min_impurity_decrease), cap,
                                  *[_lib.ptr(out[k]) for k in names], C.byref(levels), _lib.ptr(ws), C.c_size_t(ws_bytes), st))
    shapes = {'class_counts': (T, cap, K), 'node_count': (T, )}
    host = {k: eng.to_host(out[k].view(-1)[:int(np.prod(shapes.get(k, (T, cap))))]).reshape(shapes.get(k, (T, cap))).copy()
            for k in names}
    trees = []
    for t in range(T):
        nn = int(host['node_count'][t])
        tree = {k: host[k][t, :nn] for k in names if k != 'node_count'}
        tree['node_count'] = nn
        tree['n_levels'] = int(levels.value)
        trees.append(tree)
    return trees


def _tree_depth(left, right):
    """the largest node depth of a tree, one vectorised step per level"""
    left, right = np.asarray(left), np.asarray(right)
    level, depth = np.zeros(1, dtype=np.int64), 0
    while True:
        inner = level[left[level] >= 0]
        if len(inner) == 0:
            return depth
        level = np.concatenate([left[inner], right[inner]])
        depth += 1


def _sklearn_tree(arrays, n_features, K):
    """a sklearn.tree._tree.Tree filled with the node arrays; values are the class fractions scikit-learn 1.9 stores"""
    from sklearn.tree._tree import NODE_DTYPE, Tree
    nn = arrays['node_count']
    nodes = np.zeros(nn, dtype=NODE_DTYPE)
    for k in ('left_child', 'right_child'):
        nodes[k] = arrays['left' if k == 'left_child' else 'right']
    for k in ('feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left'):
        nodes[k] = arrays[k]
    counts = np.asarray(arrays['class_counts'], dtype=np.float64).reshape(nn, 1, K)
    values = counts / np.asarray(arrays['weighted_n_node_samples'], dtype=np.float64).reshape(nn, 1, 1)
    tree = Tree(n_features, np.array([K], dtype=np.intp), 1)
    tree.__setstate__({'max_depth': _tree_depth(arrays['left'], arrays['right']), 'node_count': nn, 'nodes': nodes,
                       'values': np.ascontiguousarray(values)})
    return tree


def _set_tree(tree_est, arrays, n_features, classes, max_features, seed=None):
    tree_est.n_features_in_ = n_features
    tree_est.n_outputs_ = 1
    tree_est.classes_ = classes
    tree_est.n_classes_ = np.intp(len(classes))
    tree_est.max_features_ = max_features
    tree_est.tree_ = _sklearn_tree(arrays, n_features, len(classes))
    if seed is not None:
        tree_est.random_state = seed


class _Prepared(object):
    """an estimator's fit resolved and drawn: the arguments of its device call, and what assembling the fitted estimator needs"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _within_limits(T, n, D, m):
    """whether isb_forest_fit takes a forest of T trees over n rows x D features with max_features m"""
    E = T * n
    return D <= MAX_FEATURES and 2 * E < 2 ** 31 and E * m < 2 ** 31 and E < 2 ** 30


def _prepare(estimator, X, y, n_rows=None, admit=_supported):
    """the parameters of ``estimator`` resolved against (X, y) and its seeds and bootstrap counts drawn from ``random_state`` as
    scikit-learn draws them, or None -- before any draw -- when the device does not compute the fit.  ``n_rows``: the rows of the
    device call the forest will be part of (its limits are checked at that size); ``admit``: the estimator's parameters, or None"""
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    from sklearn.utils import check_random_state
    p = admit(estimator)
    if p is None:
        return None
    X = np.asarray(X)
    y = np.asarray(y)
    if X.ndim != 2 or len(X) == 0 or X.shape[1] == 0 or X.shape[1] > MAX_FEATURES or len(y) != len(X):
        return None
    if y.ndim == 2 and y.shape[1] == 1:
        y = y.ravel()
    if y.ndim != 1:
        return None
    with np.errstate(over='ignore'):
        X32 = np.ascontiguousarray(X, dtype=np.float32)
    if not np.all(np.isfinite(X32)):
        return None
    classes, y_enc = np.unique(y, return_inverse=True)
    K = len(classes)
    if K > MAX_CLASSES:
        return None
    n, D = X32.shape
    max_features, mss, msl, max_depth = _resolve(p, n, D)
    if not 1 <= max_features <= D:
        return None
    forest = type(estimator) in (RandomForestClassifier, ExtraTreesClassifier)
    T = int(p['n_estimators']) if forest else 1
    if n_rows is not None and not _within_limits(T, n_rows, D, max_features):
        return None
    mid = float(p['min_impurity_decrease'])
    y_enc = y_enc.astype(np.int32).ravel()
    if forest:
        random_state = check_random_state(p['random_state'])
        # BaseEnsemble._make_estimator -> _set_random_states: one randint(MAX_INT) per tree, in order
        seeds = np.array([random_state.randint(_MAX_INT) for _ in range(T)], dtype=np.int64)
        if p['bootstrap']:
            # _generate_sample_indices: randint(0, n, n) from each tree's own seed
            counts = np.stack([np.bincount(np.random.RandomState(int(s)).randint(0, n, n), minlength=n) for s in seeds])
        else:
            counts = np.ones((T, n), dtype=np.int64)
    else:
        rs = p['random_state']
        seed = rs if isinstance(rs, numbers.Integral) else check_random_state(rs).randint(_MAX_INT)
        seeds, counts = np.array([int(seed)], dtype=np.int64), np.ones((1, n), dtype=np.int64)
    return _Prepared(estimator=estimator, p=p, forest=forest, X=X32, y=y_enc, classes=classes, K=K, n=n, D=D, T=T, seeds=seeds,
                     counts=counts, max_features=max_features, mss=mss, msl=msl, max_depth=max_depth, mid=mid)


def _assemble(prep, trees):
    """the estimator of ``prep`` fitted with ``trees`` (class counts over ``prep.classes``)"""
    from sklearn.base import clone
    estimator, p, D, K = prep.estimator, prep.p, prep.D, prep.K
    if prep.forest:
        estimator.estimator_ = clone(estimator.estimator)
        estimator.estimators_ = []
        for t in range(prep.T):
            est = clone(estimator.estimator_).set_params(**{k: p[k] for k in estimator.estimator_params})
            _set_tree(est, trees[t], D, np.arange(K, dtype=np.float64), prep.max_features, int(prep.seeds[t]))
            estimator.estimators_.append(est)
        estimator.n_features_in_ = D
        estimator._n_samples, estimator.n_outputs_ = prep.n, 1
        estimator._sample_weight = None
        estimator._n_samples_bootstrap = prep.n if p['bootstrap'] else None
        estimator.classes_ = prep.classes
        estimator.n_classes_ = K
    else:
        _set_tree(estimator, trees[0], D, prep.classes, prep.max_features)
    return estimator


def fit_tree_model(estimator, X, y):
    """``estimator.fit(X, y)`` on the device for an unfitted DecisionTreeClassifier / RandomForestClassifier: returns the estimator,
    fitted, or None when one of its parameters is outside what the device computes (criterion other than 'gini', splitter other than
    'best', class_weight, max_leaf_nodes, ccp_alpha > 0, min_weight_fraction_leaf > 0, max_samples, oob_score, warm_start,
    monotonic_cst), when X is not finite as float32, y has several outputs or more than 64 classes, or the size is above the kernel's
    limits.  ``random_state=None`` draws from numpy's global RNG, as scikit-learn does."""
    prep = _prepare(estimator, X, y)
    if prep is None:
        return None
    try:
        trees = _fit_arrays(prep.X, prep.y, prep.K, prep.counts, prep.seeds, prep.max_features, prep.mss, prep.msl, prep.max_depth,
                            prep.mid)
    except NotImplementedError:
        return None
    return _assemble(prep, trees)


def _group_chunks(lib, n, K, dims, tree_counts, max_features, budget):
    """consecutive ranges [g0, g1) of the groups, each one isb_forest_fit_groups call within the kernel's limits, GROUP_MAX_TREES and
    ``budget`` bytes of device memory"""
    def need(g0, g1):
        T, Dmax, m = sum(tree_counts[g0:g1]), max(dims[g0:g1]), max(max_features[g0:g1])
        if T > GROUP_MAX_TREES:
            return None
        ws = lib.isb_forest_fit_groups_workspace_bytes(n, Dmax, g1 - g0, T, K, m)
        if ws == 0:
            return None
        cap = 2 * n - 1
        return ws + 4 * (g1 - g0) * n * Dmax + 12 * T * n + T * cap * (4 * 4 + 8 * 3 + 1 + 4 * K)
    chunks, g0 = [], 0
    while g0 < len(dims):
        g1 = g0 + 1
        while g1 < len(dims):
            b = need(g0, g1 + 1)
            if b is None or b > budget:
                break
            g1 += 1
        chunks.append((g0, g1))
        g0 = g1
    return chunks


def _fit_arrays_groups(Xs, y, K, counts, seeds, tree_group, max_features, min_samples_split, min_samples_leaf, max_depth,
                       min_impurity_decrease):
    """the trees of G groups on the device: Xs [G] float32 arrays [n, D_g] (group g's rows), y [n] class indices shared by the groups,
    counts [T, n], seeds [T], tree_group [T] non-decreasing (the trees of a group consecutive), max_features / min_samples_split /
    min_samples_leaf [G] -> list of per-tree dicts as :func:`_fit_arrays` returns them, in tree order.  A batch above the kernel's
    limits, GROUP_MAX_TREES or the free device memory is built in consecutive calls of whole groups"""
    import torch
    from .engine import get_engine
    eng = get_engine()
    lib, st = eng.lib, _lib.stream_ptr()
    G, n = len(Xs), len(y)
    dims = [int(x.shape[1]) for x in Xs]
    tree_group = np.asarray(tree_group, dtype=np.int64)
    tree_counts = np.bincount(tree_group, minlength=G).tolist()
    if np.any(np.diff(tree_group) < 0):
        raise ValueError('the trees of a group must be consecutive')
    free, _ = torch.cuda.mem_get_info(eng.device)
    budget = GROUP_MEMORY_SHARE * (free + torch.cuda.memory_reserved(eng.device) - torch.cuda.memory_allocated(eng.device))
    d_y = eng.to_device(np.ascontiguousarray(y, dtype=np.int32), 'ff_y')
    names = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
             'class_counts', 'node_count')
    i32, f64 = torch.int32, torch.float64
    trees = []
    for g0, g1 in _group_chunks(lib, n, K, dims, tree_counts, list(max_features), budget):
        t0, t1 = sum(tree_counts[:g0]), sum(tree_counts[:g1])
        T, Gc, Dmax = t1 - t0, g1 - g0, max(dims[g0:g1])
        mf = np.ascontiguousarray(max_features[g0:g1], dtype=np.int32)
        ws_bytes = lib.isb_forest_fit_groups_workspace_bytes(n, Dmax, Gc, T, K, int(mf.max()))
        if ws_bytes == 0:
            raise NotImplementedError('imsegm_b200: a forest of %d trees over %d rows x %d features with max_features %d is above the '
                                      'limits of isb_forest_fit_groups' % (T, n, Dmax, int(mf.max())))
        x = np.zeros((Gc, n, Dmax), dtype=np.float32)
        for g in range(g0, g1):
            x[g - g0, :, :dims[g]] = Xs[g]
        cnt = np.ascontiguousarray(counts[t0:t1], dtype=np.int32)
        cap = 2 * int((cnt > 0).sum(axis=1).max()) - 1
        d_x = eng.to_device(x, 'ffg_x')
        del x
        d_c = eng.to_device(cnt, 'ff_counts')
        d_s = eng.to_device(np.ascontiguousarray(seeds[t0:t1], dtype=np.uint64).view(np.int64), 'ff_seeds')
        dev = eng.device
        out = {'left': torch.empty((T, cap), dtype=i32, device=dev), 'right': torch.empty((T, cap), dtype=i32, device=dev),
               'feature': torch.empty((T, cap), dtype=i32, device=dev), 'threshold': torch.empty((T, cap), dtype=f64, device=dev),
               'impurity': torch.empty((T, cap), dtype=f64, device=dev), 'n_node_samples': torch.empty((T, cap), dtype=i32, device=dev),
               'weighted_n_node_samples': torch.empty((T, cap), dtype=f64, device=dev),
               'missing_go_to_left': torch.empty((T, cap), dtype=torch.uint8, device=dev),
               'class_counts': torch.empty((T, cap, K), dtype=i32, device=dev), 'node_count': torch.empty(T, dtype=i32, device=dev)}
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        levels = C.c_int(0)
        per_group = [np.ascontiguousarray(v[g0:g1], dtype=np.int32) for v in (dims, max_features, min_samples_split, min_samples_leaf)]
        tg = np.ascontiguousarray(tree_group[t0:t1] - g0, dtype=np.int32)
        _lib.check(lib.isb_forest_fit_groups(_lib.ptr(d_x), n, Dmax, Gc, *[a.ctypes.data for a in per_group], _lib.ptr(d_y), K,
                                             _lib.ptr(d_c), T, tg.ctypes.data, _lib.ptr(d_s), max_depth, C.c_double(min_impurity_decrease),
                                             cap, *[_lib.ptr(out[k]) for k in names], C.byref(levels), _lib.ptr(ws), C.c_size_t(ws_bytes),
                                             st))
        del ws
        host = {k: eng.to_host(out[k]) for k in names}
        for t in range(T):
            nn = int(host['node_count'][t])
            tree = {k: host[k][t, :nn].copy() for k in names if k != 'node_count'}
            tree['node_count'] = nn
            tree['n_levels'] = int(levels.value)
            trees.append(tree)
    return trees


class TreeBatch(object):
    """estimators fitted on training sets that are subsets of one set of ``labels`` [n], built in one device call.

    :meth:`add` prepares an estimator at once -- its parameters resolved against its own training rows, its seeds and bootstrap rows
    drawn from its ``random_state`` -- so numpy's global RNG is consumed in the order of the calls, as scikit-learn's sequential fits
    consume it; an estimator the device does not compute, or a single forest above the kernel's limits, is fitted by scikit-learn there
    and then.  :meth:`fit` builds every prepared tree and forest in one :func:`_fit_arrays_groups` call per (max_depth,
    min_impurity_decrease) and returns every estimator fitted, in the order of :meth:`add`.  A training set that lacks some of the
    labels is built with all of them (a class of count 0 changes no Gini value) and its estimator keeps the classes of its own rows, as
    scikit-learn's.  Training rows given twice are fitted by a call of their own."""

    def __init__(self, labels):
        labels = np.asarray(labels)
        if labels.ndim == 2 and labels.shape[1] == 1:
            labels = labels.ravel()
        self.labels, self.n = labels, len(labels)
        self.classes, self.y = np.unique(labels, return_inverse=True) if labels.ndim == 1 else (None, None)
        self.shared = labels.ndim == 1 and len(self.classes) <= MAX_CLASSES
        self.fitted, self.preps = [], {}

    def add(self, estimator, X, rows):
        """``estimator.fit(X, labels[rows])``: X [len(rows), D] the features of the training rows, ``rows`` their indices"""
        rows = np.asarray(rows, dtype=np.int64).ravel()
        X = np.asarray(X)
        y = self.labels[rows]
        grouped = self.shared and len(np.unique(rows)) == len(rows)
        prep = _prepare(estimator, X, y, self.n if grouped else len(rows))
        if prep is None:
            self.fitted.append(estimator.fit(X, y))
            return
        prep.rows, prep.grouped = rows, grouped
        self.preps[len(self.fitted)] = prep
        self.fitted.append(None)

    def fit(self):
        batches = collections.OrderedDict()
        for i, prep in self.preps.items():
            if not prep.grouped:
                self.fitted[i] = _assemble(prep, _fit_arrays(prep.X, prep.y, prep.K, prep.counts, prep.seeds, prep.max_features, prep.mss,
                                                             prep.msl, prep.max_depth, prep.mid))
            else:
                batches.setdefault((prep.max_depth, prep.mid), []).append(i)
        n = self.n
        for (max_depth, mid), idx in batches.items():
            ps = [self.preps[i] for i in idx]
            counts = np.zeros((sum(p.T for p in ps), n), dtype=np.int32)
            Xs, t = [], 0
            for p in ps:
                counts[t:t + p.T, p.rows] = p.counts
                t += p.T
                x = np.zeros((n, p.D), dtype=np.float32)
                x[p.rows] = p.X
                Xs.append(x)
            trees = _fit_arrays_groups(Xs, self.y.astype(np.int32), len(self.classes), counts, np.concatenate([p.seeds for p in ps]),
                                       np.repeat(np.arange(len(ps)), [p.T for p in ps]), np.array([p.max_features for p in ps]),
                                       np.array([p.mss for p in ps]), np.array([p.msl for p in ps]), max_depth, mid)
            t = 0
            for i, p in zip(idx, ps):
                cols = np.searchsorted(self.classes, p.classes)     # the classes of its own rows, as its own fit encodes them
                own = []
                for tree in trees[t:t + p.T]:
                    tree = dict(tree)
                    tree['class_counts'] = np.ascontiguousarray(np.asarray(tree['class_counts'])[:, cols])
                    own.append(tree)
                self.fitted[i] = _assemble(p, own)
                t += p.T
        self.preps = {}
        return self.fitted


def fit_tree_models(estimators, features, labels, train_rows=None):
    """``[est.fit(X[rows], labels[rows]) for est, X, rows in zip(estimators, features, train_rows)]`` with every tree and forest built
    in one device call (see :class:`TreeBatch`): ``features`` one array [n, D_i] per estimator (the rows of a fold after its own
    scaler and PCA), ``labels`` [n] shared, ``train_rows`` per estimator the indices of its training rows (None: all rows).  Returns
    the fitted estimators."""
    if train_rows is None:
        train_rows = [None] * len(estimators)
    if not len(features) == len(train_rows) == len(estimators):
        raise ValueError('one feature array and one training set per estimator')
    batch = TreeBatch(labels)
    for est, X, rows in zip(estimators, features, train_rows):
        X = np.asarray(X)
        if len(X) != batch.n:
            raise ValueError('%d feature rows for %d labels' % (len(X), batch.n))
        rows = np.arange(batch.n) if rows is None else np.asarray(rows, dtype=np.int64).ravel()
        batch.add(est, X[rows], rows)
    return batch.fit()


# ---- extra trees (isb_extra_trees_fit, csrc/extra_trees_fit.cu) ----

#: the share of the free device memory one isb_extra_trees_fit call may take; a larger forest goes in consecutive calls of whole trees
EXTRA_MEMORY_SHARE = 0.8
_RAND_R_MAX = 2 ** 31 - 1


def _supported_extra(est):
    """the parameters of an ExtraTreesClassifier that isb_extra_trees_fit computes, or None"""
    from sklearn.ensemble import ExtraTreesClassifier
    if type(est) is not ExtraTreesClassifier:
        return None
    p = est.get_params(deep=False)
    if p.get('criterion') != 'gini' or p.get('class_weight') is not None or p.get('max_leaf_nodes') is not None:
        return None
    if p.get('ccp_alpha', 0.0) > 0 or p.get('min_weight_fraction_leaf', 0.0) > 0 or p.get('monotonic_cst') is not None:
        return None
    if p.get('max_samples') is not None or p.get('oob_score') or p.get('warm_start'):
        return None
    return p


def _rand_r_states(seeds):
    """each tree's splitter state: Splitter.init draws ``randint(0, RAND_R_MAX)`` from the tree's RandomState(seed), the first draw
    from it (DecisionTreeClassifier._fit hands the RandomState to the splitter untouched)"""
    return np.array([np.random.RandomState(int(s)).randint(0, _RAND_R_MAX) for s in seeds], dtype=np.uint32)


def _extra_chunks(T, n, K, ws_per_tree, budget):
    """consecutive ranges [t0, t1) of the trees, each one isb_extra_trees_fit call within ``budget`` bytes of device memory"""
    cap = 2 * n - 1
    per_tree = ws_per_tree + 4 * n + 4 + cap * (4 * 4 + 8 * 3 + 1 + 4 * K)
    step = max(1, min(T, int(budget // per_tree)))
    return [(t0, min(T, t0 + step)) for t0 in range(0, T, step)]


def _fit_arrays_extra(X, y, K, counts, states, max_features, min_samples_split, min_samples_leaf, max_depth, min_impurity_decrease,
                      budget=None, small_rows=0):
    """every extra tree on the device: X [n, D] float32, y [n] class indices, counts [T, n], states [T] u32 -> list of per-tree dicts
    of preorder node arrays as :func:`_fit_arrays` returns them.  A forest above ``budget`` bytes (default: EXTRA_MEMORY_SHARE of the
    free device memory) is built in consecutive calls of whole trees"""
    import torch
    from .engine import get_engine
    eng = get_engine()
    lib, st = eng.lib, _lib.stream_ptr()
    n, D = X.shape
    T = len(counts)
    ws1 = lib.isb_extra_trees_fit_workspace_bytes(n, D, 1, K, max_features)
    if ws1 == 0:
        raise NotImplementedError('imsegm_b200: extra trees over %d rows x %d features, %d classes, are above the limits of '
                                  'isb_extra_trees_fit' % (n, D, K))
    if budget is None:
        free, _ = torch.cuda.mem_get_info(eng.device)
        budget = EXTRA_MEMORY_SHARE * (free + torch.cuda.memory_reserved(eng.device) - torch.cuda.memory_allocated(eng.device))
    d_x = eng.to_device(np.ascontiguousarray(X, dtype=np.float32), 'et_x')
    d_y = eng.to_device(np.ascontiguousarray(y, dtype=np.int32), 'et_y')
    names = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
             'class_counts')
    i32, f64, dev = torch.int32, torch.float64, eng.device
    kinds = {'threshold': f64, 'impurity': f64, 'weighted_n_node_samples': f64, 'missing_go_to_left': torch.uint8}
    trees = []
    for t0, t1 in _extra_chunks(T, n, K, ws1, budget):
        Tc = t1 - t0
        cnt = np.ascontiguousarray(counts[t0:t1], dtype=np.int32)
        cap = 2 * int((cnt > 0).sum(axis=1).max()) - 1
        ws_bytes = lib.isb_extra_trees_fit_workspace_bytes(n, D, Tc, K, max_features)
        if ws_bytes == 0:
            raise NotImplementedError('imsegm_b200: %d extra trees over %d rows are above the limits of isb_extra_trees_fit' % (Tc, n))
        d_c = eng.to_device(cnt, 'et_counts')
        d_s = eng.to_device(np.ascontiguousarray(states[t0:t1], dtype=np.uint32).view(np.int32), 'et_states')
        out = {k: torch.empty((Tc, cap, K) if k == 'class_counts' else (Tc, cap), dtype=kinds.get(k, i32), device=dev) for k in names}
        node_count = torch.empty(Tc, dtype=i32, device=dev)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.isb_extra_trees_fit(_lib.ptr(d_x), n, D, _lib.ptr(d_y), K, _lib.ptr(d_c), Tc, _lib.ptr(d_s), max_features,
                                           min_samples_split, min_samples_leaf, max_depth, C.c_double(min_impurity_decrease),
                                           small_rows, cap, *[_lib.ptr(out[k]) for k in names], _lib.ptr(node_count), _lib.ptr(ws),
                                           C.c_size_t(ws_bytes), st))
        del ws
        nodes = eng.to_host(node_count).astype(np.int64)
        width = int(nodes.max())
        host = {k: eng.to_host(out[k][:, :width].contiguous()) for k in names}
        del out
        for t in range(Tc):
            nn = int(nodes[t])
            tree = {k: host[k][t, :nn].copy() for k in names}
            tree['node_count'] = nn
            trees.append(tree)
    return trees


def fit_extra_trees(estimator, X, y):
    """``estimator.fit(X, y)`` on the device for an unfitted ExtraTreesClassifier: returns the estimator, fitted -- the trees are
    scikit-learn's node for node, so ``feature_importances_`` and ``predict_proba`` are its bits -- or None when one of its parameters is
    outside what the device computes (criterion other than 'gini', class_weight, max_leaf_nodes, ccp_alpha > 0, min_weight_fraction_leaf
    > 0, max_samples, oob_score, warm_start, monotonic_cst), when X is not finite as float32, y has several outputs or more than 64
    classes, or the size is above the kernel's limits.  The seeds, bootstrap rows and splitter states are drawn from ``random_state`` as
    scikit-learn draws them (``random_state=None`` draws from numpy's global RNG)."""
    prep = _prepare(estimator, X, y, admit=_supported_extra)
    if prep is None:
        return None
    if prep.T * prep.n >= 2 ** 31:
        return None
    try:
        trees = _fit_arrays_extra(prep.X, prep.y, prep.K, prep.counts, _rand_r_states(prep.seeds), prep.max_features, prep.mss, prep.msl,
                                  prep.max_depth, prep.mid)
    except NotImplementedError:
        return None
    return _assemble(prep, trees)
