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
"""
import ctypes as C
import numbers
from math import ceil

import numpy as np

from . import _lib

#: isb_forest_fit's limits
MAX_CLASSES, MAX_FEATURES = 64, 2048
_MAX_INT = np.iinfo(np.int32).max


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


def fit_tree_model(estimator, X, y):
    """``estimator.fit(X, y)`` on the device for an unfitted DecisionTreeClassifier / RandomForestClassifier: returns the estimator,
    fitted, or None when one of its parameters is outside what the device computes (criterion other than 'gini', splitter other than
    'best', class_weight, max_leaf_nodes, ccp_alpha > 0, min_weight_fraction_leaf > 0, max_samples, oob_score, warm_start,
    monotonic_cst), when X is not finite as float32, y has several outputs or more than 64 classes, or the size is above the kernel's
    limits.  ``random_state=None`` draws from numpy's global RNG, as scikit-learn does."""
    from sklearn.base import clone
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.utils import check_random_state
    p = _supported(estimator)
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
    mid = float(p['min_impurity_decrease'])
    y_enc = y_enc.astype(np.int32).ravel()
    if type(estimator) is RandomForestClassifier:
        random_state = check_random_state(p['random_state'])
        T = int(p['n_estimators'])
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
        seeds, counts, T = np.array([int(seed)], dtype=np.int64), np.ones((1, n), dtype=np.int64), 1
    try:
        trees = _fit_arrays(X32, y_enc, K, counts, seeds, max_features, mss, msl, max_depth, mid)
    except NotImplementedError:
        return None
    if type(estimator) is RandomForestClassifier:
        estimator.estimator_ = clone(estimator.estimator)
        estimator.estimators_ = []
        for t in range(T):
            est = clone(estimator.estimator_).set_params(**{k: p[k] for k in estimator.estimator_params})
            _set_tree(est, trees[t], D, np.arange(K, dtype=np.float64), max_features, int(seeds[t]))
            estimator.estimators_.append(est)
        estimator.n_features_in_ = D
        estimator._n_samples, estimator.n_outputs_ = n, 1
        estimator._sample_weight = None
        estimator._n_samples_bootstrap = n if p['bootstrap'] else None
        estimator.classes_ = classes
        estimator.n_classes_ = K
    else:
        _set_tree(estimator, trees[0], D, classes, max_features)
    return estimator
