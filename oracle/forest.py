"""
numpy restatement of ``isb_forest_fit`` (csrc/forest_fit.cu): exact-split Gini trees with scikit-learn 1.9's split rules and the
device's feature sampling, in float64 and integers, node for node the same bits as the device.  And an optimality checker that does not
share the builder's code: it re-derives each node's rows, candidates and best split by brute force over the distinct values.

Rules (scikit-learn's ``_splitter.pyx`` node_split_best, ``_partitioner.pyx`` next_p, ``_criterion.pyx`` Gini, ``_tree.pyx``
DepthFirstTreeBuilder):
- proxy improvement ``-w_r * gini_r - w_l * gini_l`` with ``gini = 1.0 - sum(count^2) / (w * w)`` from the weighted class counts;
- a position p of the sorted values is allowed when ``x[p] > x[p-1] + 1e-7`` in float32 and both sides keep min_samples_leaf rows;
- threshold ``x[p-1] / 2.0 + x[p] / 2.0`` in float64; rows go left when ``x <= threshold``;
- a node is a leaf on the depth limit, below min_samples_split or 2 * min_samples_leaf rows, at impurity <= eps, without an
  allowed position, or when ``improvement + eps < min_impurity_decrease``;
- candidates: the m non-constant features (max > min + 1e-7 in float32) of least (hash, feature), hash = splitmix64(splitmix64(
  splitmix64(seed) ^ b) ^ feature), b the node's breadth-first index in its tree; equal proxies go to the lowest feature, then the
  lowest position.
"""
import numpy as np

FEATURE_THRESHOLD = np.float32(1e-7)
EPSILON = np.finfo(np.float64).eps
_M64 = (1 << 64) - 1


def splitmix64(z):
    """splitmix64 of Python ints or a uint64 array"""
    if isinstance(z, np.ndarray):
        with np.errstate(over='ignore'):
            z = z.astype(np.uint64) + np.uint64(0x9e3779b97f4a7c15)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
            return z ^ (z >> np.uint64(31))
    z = (int(z) + 0x9e3779b97f4a7c15) & _M64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & _M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & _M64
    return z ^ (z >> 31)


def feature_hashes(seed, bfs_index, n_features):
    """uint64 [D]: the sampling key of every feature at the node of breadth-first index ``bfs_index`` of the tree ``seed``"""
    key = splitmix64(splitmix64(seed) ^ int(bfs_index))
    return splitmix64(np.uint64(key) ^ np.arange(n_features, dtype=np.uint64))


def candidates(x_node, seed, bfs_index, max_features):
    """ascending candidate features of a node from its rows x_node [n, D] float32 (all non-constant ones when max_features is None)"""
    lo, hi = x_node.min(axis=0), x_node.max(axis=0)
    nonconst = np.nonzero(~(hi <= lo + FEATURE_THRESHOLD))[0]
    if max_features is None or len(nonconst) <= max_features:
        return nonconst
    h = feature_hashes(seed, bfs_index, x_node.shape[1])[nonconst]
    order = np.lexsort((nonconst, h))
    return np.sort(nonconst[order[:max_features]])


def gini(sq, w):
    """Gini.node_impurity / children_impurity from the (exact) sum of squared weighted counts and the weight, float64"""
    w = np.asarray(w, dtype=np.float64)
    return 1.0 - np.asarray(sq, dtype=np.float64) / (w * w)


def proxy(sq_l, w_l, sq_r, w_r):
    """proxy_impurity_improvement"""
    w_l, w_r = np.asarray(w_l, dtype=np.float64), np.asarray(w_r, dtype=np.float64)
    return -w_r * gini(sq_r, w_r) - w_l * gini(sq_l, w_l)


def improvement(w_node, w_total, imp, sq_l, w_l, sq_r, w_r):
    """impurity_improvement"""
    w_node, w_l, w_r = (np.asarray(v, dtype=np.float64) for v in (w_node, w_l, w_r))
    return (w_node / np.float64(w_total)) * (imp - (w_r / w_node * gini(sq_r, w_r)) - (w_l / w_node * gini(sq_l, w_l)))


def _best_split_of_feature(v, cls, wts, cc, K, msl):
    """(proxy, position, threshold, w_l, sq_l, sq_r) of the first best allowed position of one feature, or None"""
    n = len(v)
    order = np.argsort(v, kind='stable')
    vs, cs, ws = v[order], cls[order], wts[order]
    onehot = np.zeros((n, K), dtype=np.int64)
    onehot[np.arange(n), cs] = ws
    left = np.cumsum(onehot, axis=0)[:-1]                   # after the first p rows, p = 1 .. n-1
    p = np.arange(1, n)
    allowed = (vs[1:] > vs[:-1] + FEATURE_THRESHOLD) & (p >= msl) & (n - p >= msl)
    if not np.any(allowed):
        return None
    left = left[allowed]
    right = cc[None, :] - left
    sq_l, sq_r = (left * left).sum(1), (right * right).sum(1)
    w_l = left.sum(1)
    w_r = cc.sum() - w_l
    pr = proxy(sq_l, w_l, sq_r, w_r)
    a = int(np.argmax(pr))                                  # the first maximum: the strict > of the scan
    pos = int(p[allowed][a])
    thr = np.float64(vs[pos - 1]) / 2.0 + np.float64(vs[pos]) / 2.0
    return pr[a], pos, thr, int(w_l[a]), int(sq_l[a]), int(sq_r[a])


def build_tree(X, y, counts, K, seed, max_features, min_samples_split, min_samples_leaf, max_depth=None, min_impurity_decrease=0.0):
    """one tree (max_depth None or -1: no limit): dict of preorder node arrays (as isb_forest_fit writes them) plus 'node_count' and 'n_levels'"""
    X = np.asarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.int64)
    counts = np.asarray(counts, dtype=np.int64)
    max_depth = None if max_depth is None or max_depth < 0 else max_depth
    w_total = int(counts.sum())
    nodes = [dict(rows=np.nonzero(counts)[0], depth=0, bfs=0)]
    head = 0
    while head < len(nodes):                                # breadth-first, children of earlier parents first
        nd = nodes[head]
        head += 1
        rows = nd['rows']
        cc = np.bincount(y[rows], weights=counts[rows], minlength=K).astype(np.int64)
        w = int(cc.sum())
        imp = gini(int((cc * cc).sum()), w)
        nd.update(cc=cc, w=w, imp=imp, split=False)
        n = len(rows)
        if (max_depth is not None and nd['depth'] >= max_depth) or n < min_samples_split or n < 2 * min_samples_leaf \
                or imp <= EPSILON:
            continue
        best = None
        for f in candidates(X[rows], seed, nd['bfs'], max_features):
            res = _best_split_of_feature(X[rows, f], y[rows], counts[rows], cc, K, min_samples_leaf)
            if res is not None and (best is None or res[0] > best[0][0]):
                best = (res, int(f))
        if best is None:
            continue
        (pr, pos, thr, w_l, sq_l, sq_r), f = best
        if improvement(w, w_total, imp, sq_l, w_l, sq_r, w - w_l) + EPSILON < min_impurity_decrease:
            continue
        go_left = X[rows, f].astype(np.float64) <= thr
        nd.update(split=True, feature=f, threshold=thr, mgl=int(pos > n - pos))
        nd['children'] = (len(nodes), len(nodes) + 1)
        base = nodes[-1]['bfs'] + 1
        nodes.append(dict(rows=rows[go_left], depth=nd['depth'] + 1, bfs=base))
        nodes.append(dict(rows=rows[~go_left], depth=nd['depth'] + 1, bfs=base + 1))
    return _preorder(nodes, K)


def _preorder(nodes, K):
    order, stack = [], [0]
    while stack:
        i = stack.pop()
        order.append(i)
        if nodes[i]['split']:
            stack += [nodes[i]['children'][1], nodes[i]['children'][0]]
    pre = np.empty(len(nodes), dtype=np.int64)
    pre[order] = np.arange(len(nodes))
    nn = len(nodes)
    out = dict(left=np.full(nn, -1, np.int32), right=np.full(nn, -1, np.int32), feature=np.full(nn, -2, np.int32),
               threshold=np.full(nn, -2.0), impurity=np.zeros(nn), n_node_samples=np.zeros(nn, np.int32),
               weighted_n_node_samples=np.zeros(nn), missing_go_to_left=np.zeros(nn, np.uint8), class_counts=np.zeros((nn, K), np.int32))
    for i, nd in enumerate(nodes):
        o = pre[i]
        if nd['split']:
            out['left'][o], out['right'][o] = pre[nd['children'][0]], pre[nd['children'][1]]
            out['feature'][o], out['threshold'][o], out['missing_go_to_left'][o] = nd['feature'], nd['threshold'], nd['mgl']
        out['impurity'][o] = nd['imp']
        out['n_node_samples'][o] = len(nd['rows'])
        out['weighted_n_node_samples'][o] = nd['w']
        out['class_counts'][o] = nd['cc']
    out['node_count'] = nn
    out['n_levels'] = max(nd['depth'] for nd in nodes) + 1
    return out


def fit_arrays(X, y, K, counts, seeds, max_features, min_samples_split, min_samples_leaf, max_depth, min_impurity_decrease):
    """every tree of a forest: counts [T, n], seeds [T] -> list of build_tree dicts (the device call's signature in forest_fit.py)"""
    return [build_tree(X, y, counts[t], K, int(seeds[t]), max_features, min_samples_split, min_samples_leaf, max_depth,
                       min_impurity_decrease) for t in range(len(counts))]


# ---------------------------------------------------------------------------------------------------------------------
# optimality checker
# ---------------------------------------------------------------------------------------------------------------------

def _stats(rows, y, counts, K):
    cc = np.zeros(K, dtype=np.int64)
    np.add.at(cc, y[rows], counts[rows])
    return cc


def check_tree(tree, X, y, counts, K, seed=None, max_features=None, min_samples_split=2, min_samples_leaf=1, max_depth=None,
               min_impurity_decrease=0.0):
    """assert that a tree (preorder arrays: left, right, feature, threshold, impurity, n_node_samples, weighted_n_node_samples,
    class counts as 'class_counts' or fractions as 'value') is optimal for its rows: every internal node's proxy improvement is the
    best over all (candidate feature, allowed position) pairs and every leaf meets a leaf condition.  ``max_features=None`` takes
    every non-constant feature as a candidate (scikit-learn's own trees); otherwise the candidates follow the hash rule with ``seed``."""
    X = np.asarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.int64)
    counts = np.asarray(counts, dtype=np.int64)
    left, right = np.asarray(tree['left']), np.asarray(tree['right'])
    max_depth = None if max_depth is None or max_depth < 0 else max_depth
    w_total = int(counts.sum())
    # rows, depth and breadth-first index of every node from the structure
    rows_of, depth_of, bfs_of = {0: np.nonzero(counts)[0]}, {0: 0}, {0: 0}
    queue, b = [0], 1
    while queue:
        nxt = []
        for i in queue:
            if left[i] < 0:
                continue
            r = rows_of[i]
            go = X[r, tree['feature'][i]].astype(np.float64) <= tree['threshold'][i]
            for c, sel in ((left[i], go), (right[i], ~go)):
                rows_of[c], depth_of[c], bfs_of[c] = r[sel], depth_of[i] + 1, b
                b += 1
                nxt.append(c)
        queue = nxt
    assert len(rows_of) == len(left), 'unreachable nodes'
    for i, rows in rows_of.items():
        n = len(rows)
        cc = _stats(rows, y, counts, K)
        w = int(cc.sum())
        assert tree['n_node_samples'][i] == n, (i, 'rows')
        assert tree['weighted_n_node_samples'][i] == w, (i, 'weight')
        imp = gini(int((cc * cc).sum()), w)
        assert tree['impurity'][i] == imp, (i, 'impurity', tree['impurity'][i], imp)
        if 'class_counts' in tree:
            assert np.array_equal(np.asarray(tree['class_counts'][i]), cc), (i, 'class counts')
        # brute force: every candidate feature, every pair of adjacent distinct values far enough apart
        best, best_impr = -np.inf, None
        pre_leaf = (max_depth is not None and depth_of[i] >= max_depth) or n < min_samples_split or n < 2 * min_samples_leaf \
            or imp <= EPSILON
        if not pre_leaf:
            for f in candidates(X[rows], seed, bfs_of[i], max_features):
                v = X[rows, f]
                u = np.unique(v)
                for a, c in zip(u[:-1], u[1:]):
                    if not c > a + FEATURE_THRESHOLD:
                        continue
                    sel = v <= a
                    n_l = int(sel.sum())
                    if n_l < min_samples_leaf or n - n_l < min_samples_leaf:
                        continue
                    cl = _stats(rows[sel], y, counts, K)
                    cr = cc - cl
                    w_l = int(cl.sum())
                    pr = proxy(int((cl * cl).sum()), w_l, int((cr * cr).sum()), w - w_l)
                    if pr > best:
                        best = pr
                        best_impr = improvement(w, w_total, imp, int((cl * cl).sum()), w_l, int((cr * cr).sum()), w - w_l)
        if left[i] >= 0:
            assert not pre_leaf and best_impr is not None, (i, 'split of a node that must be a leaf')
            f, thr = tree['feature'][i], tree['threshold'][i]
            v = X[rows, f]
            sel = v.astype(np.float64) <= thr
            a, c = v[sel].max(), v[~sel].min()
            assert thr == np.float64(a) / 2.0 + np.float64(c) / 2.0, (i, 'threshold is not the midpoint')
            cl = _stats(rows[sel], y, counts, K)
            cr = cc - cl
            pr = proxy(int((cl * cl).sum()), int(cl.sum()), int((cr * cr).sum()), int(cr.sum()))
            assert pr == best, (i, 'not the best split', pr, best)
            assert not best_impr + EPSILON < min_impurity_decrease, (i, 'improvement below min_impurity_decrease')
        else:
            assert pre_leaf or best_impr is None or best_impr + EPSILON < min_impurity_decrease, (i, 'a leaf that has a split')
    return True
