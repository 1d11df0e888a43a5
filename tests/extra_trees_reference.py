"""
scikit-learn's own extra trees as the node arrays ``forest_fit._fit_arrays_extra`` returns (test helper): the reference the device
must equal node for node, and the stand-in for the device call in the CPU tests.
"""
import numpy as np

FIELDS = ('left', 'right', 'feature', 'threshold', 'impurity', 'n_node_samples', 'weighted_n_node_samples', 'missing_go_to_left',
          'class_counts')


def tree_arrays(tree_est, K):
    """one fitted ExtraTreeClassifier / DecisionTreeClassifier -> dict of preorder node arrays with class counts over K classes"""
    t = tree_est.tree_
    w = t.weighted_n_node_samples
    counts = np.rint(t.value[:, 0, :] * w[:, None]).astype(np.int32)
    full = np.zeros((t.node_count, K), dtype=np.int32)
    full[:, :counts.shape[1]] = counts
    return {'left': t.children_left.astype(np.int32), 'right': t.children_right.astype(np.int32), 'feature': t.feature.astype(np.int32),
            'threshold': t.threshold.copy(), 'impurity': t.impurity.copy(), 'n_node_samples': t.n_node_samples.astype(np.int32),
            'weighted_n_node_samples': w.copy(), 'missing_go_to_left': t.missing_go_to_left.astype(np.uint8), 'class_counts': full,
            'node_count': int(t.node_count)}


def forest_arrays(forest):
    """every tree of a fitted ExtraTreesClassifier as node arrays"""
    K = len(forest.classes_)
    return [tree_arrays(est, K) for est in forest.estimators_]


def first_difference(got, want):
    """None when two trees' node arrays are bit-identical, else a message naming the first differing field and node"""
    if got['node_count'] != want['node_count']:
        return 'node_count %d != %d' % (got['node_count'], want['node_count'])
    for k in FIELDS:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        if a.dtype.kind == 'f':
            same = a.view(np.uint64) == b.view(np.uint64)
        else:
            same = a == b
        if same.ndim > 1:
            same = same.all(axis=1)
        if not same.all():
            i = int(np.argmin(same))
            return '%s differs first at node %d: %r != %r' % (k, i, a[i], b[i])
    return None
