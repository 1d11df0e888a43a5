"""GPU tests of device predict_proba for caller-fitted models at their class-count, split and threshold edges: the forest
(k_forest_leaves / k_forest_sum), k-nearest-neighbour (k_knn_partial / k_knn_vote), logistic-regression (k_linear_proba) and mixture
(k_mix_proba and the large-D GEMM route) evaluations against scikit-learn and the numpy oracle (oracle/neighbours.py), driven through
class_models.compile_model and through hand-built CompiledModel tables, and one 40-class forest through the shared-model pipeline
against the host round trip (graph_cuts.USE_DEVICE_PREDICT = False)."""
import warnings

import numpy as np
import pytest
from sklearn import ensemble, linear_model, mixture, neighbors, pipeline, preprocessing, tree

from conftest import synth_regions
from oracle import neighbours as onb

pytestmark = pytest.mark.gpu

RF = dict(n_estimators=20, min_samples_leaf=2, min_samples_split=3)     # the reference's RandForest (classification.py:101)
FEATS = {'color': ('mean', 'std')}
SENTINEL = -3.25


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _data(n, d, k, seed, noise=0.15):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(0, 1, (k, d))
    y = np.arange(n) % k                                    # every class present
    rng.shuffle(y)
    return centres[y] + rng.normal(0, noise, (n, d)), y


def _spread(K):
    """class labels that are not arange(K): 3, 10, 17, ..."""
    return 3 + 7 * np.arange(K)


class _host_predict(object):
    """graph_cuts.USE_DEVICE_PREDICT = False inside the block"""

    def __enter__(self):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = False

    def __exit__(self, *exc):
        from pyimsegm_b200 import graph_cuts
        graph_cuts.USE_DEVICE_PREDICT = True


def _forest(kind, scaled):
    est = {'tree': tree.DecisionTreeClassifier(random_state=0), 'forest': ensemble.RandomForestClassifier(random_state=0, **RF),
           'extra': ensemble.ExtraTreesClassifier(random_state=0, **RF)}[kind]
    return pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('classif', est)]) if scaled else est


def _trees(model):
    est = model.steps[-1][1] if isinstance(model, pipeline.Pipeline) else model
    return [est] if isinstance(est, tree.DecisionTreeClassifier) else list(est.estimators_)


def _device_rows_only(eng, cm, x, n_dev):
    """class_model_predict on the buffer x with n_dev live rows, after the transform and probability buffers are filled with a
    sentinel: returns (probabilities [N, K], transformed features [N, n_dims]), both buffers whole"""
    torch = eng.torch
    d_x = eng.to_device(np.ascontiguousarray(x), 'edge_test_x')
    d_n = eng.to_device(np.array([n_dev], dtype=np.int32), 'edge_test_n')
    eng.class_model_predict(d_x, cm, d_n=d_n)             # sizes every buffer, so the ones filled below are the ones it writes
    eng.buf('cm_x', (len(x), cm.n_dims), torch.float64).fill_(SENTINEL)
    eng.buf('proba', (len(x), cm.n_classes), torch.float64).fill_(SENTINEL)
    proba = eng.to_host(eng.class_model_predict(d_x, cm, d_n=d_n)).copy()
    return proba, eng.to_host(eng.buf('cm_x', (len(x), cm.n_dims), torch.float64)).copy()


# ---------------------------------------------------------------------------------------------------------------------------------
# forests and trees


@pytest.mark.parametrize('kind', ['tree', 'forest', 'extra'])
@pytest.mark.parametrize('K', [1, 2, 33, 64])
@pytest.mark.parametrize('scaled', [False, True])
def test_forest_class_counts_bit_exact(kind, K, scaled):
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(40 * K + 200, 7, K, seed=K)
    model = _forest(kind, scaled).fit(X, _spread(K)[y])
    assert np.array_equal(model.classes_, _spread(K))
    cm = compile_model(model)
    assert cm.kind == 'forest' and cm.n_classes == K
    rng = np.random.RandomState(99)
    Xt = X[rng.randint(0, len(X), 4000)] + rng.normal(0, 0.1, (4000, X.shape[1]))
    Xt[::13, 0] = np.nan
    got = cm.predict_proba(Xt)
    want = model.predict_proba(np.nan_to_num(Xt))
    assert got.shape == (len(Xt), K)
    assert np.array_equal(got, want)
    if K == 1:                                              # root-only trees: every row gets 1.0
        assert all(t.tree_.node_count == 1 for t in _trees(model))
        assert np.all(got == 1.0)
    if K > 32:                                              # every column above 32 carries probability somewhere
        assert np.count_nonzero(want[:, 32:].max(axis=0)) == K - 32


def test_forest_65_classes_is_refused(eng):
    import ctypes as C
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(65 * 8, 5, 65, seed=65)
    for model in (tree.DecisionTreeClassifier(random_state=0), _forest('forest', True)):
        model.fit(X, _spread(65)[y])
        assert compile_model(model) is None
    # the kernel itself: ISB_ERR_UNSUPPORTED, nothing launched, nothing written
    torch, lib = eng.torch, eng.lib
    N, T, n_nodes, K = 16, 1, 1, 65
    dev = eng.device
    x = torch.zeros((N, 5), dtype=torch.float64, device=dev)
    i32 = torch.zeros(n_nodes, dtype=torch.int32, device=dev)
    left = torch.full((n_nodes, ), -1, dtype=torch.int32, device=dev)
    thr = torch.zeros(n_nodes, dtype=torch.float64, device=dev)
    value = torch.full((n_nodes, K), 1.0 / K, dtype=torch.float64, device=dev)
    proba = torch.full((N, K), SENTINEL, dtype=torch.float64, device=dev)
    wsb = lib.isb_forest_predict_workspace_bytes(N, T)
    ws = torch.zeros(max(wsb, 1), dtype=torch.uint8, device=dev)
    n0 = lib.isb_launch_count()
    st = lib.isb_forest_predict_proba(_lib.ptr(x), N, None, 5, T, _lib.ptr(i32), _lib.ptr(i32), _lib.ptr(thr), _lib.ptr(left),
                                      _lib.ptr(left), n_nodes, _lib.ptr(value), K, 1, _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb),
                                      _lib.stream_ptr())
    assert st == _lib.ISB_ERR_UNSUPPORTED
    assert lib.isb_launch_count() == n0
    torch.cuda.synchronize()
    assert bool((proba == SENTINEL).all())
    # K = 64 with the same tables is evaluated: [N, 64] rows of the root's first 64 values
    st = lib.isb_forest_predict_proba(_lib.ptr(x), N, None, 5, T, _lib.ptr(i32), _lib.ptr(i32), _lib.ptr(thr), _lib.ptr(left),
                                      _lib.ptr(left), n_nodes, _lib.ptr(value), 64, 1, _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb),
                                      _lib.stream_ptr())
    assert st == _lib.ISB_OK and lib.isb_launch_count() == n0 + 2
    flat = proba.view(-1)
    assert bool((flat[:N * 64] == 1.0 / 65).all()) and bool((flat[N * 64:] == SENTINEL).all())


def _colour_training(seeds, n_classes, shape=(320, 384)):
    """colour features of synthetic images and a label per superpixel: quantile bins of the mean red value, so every one of
    n_classes classes is present"""
    from pyimsegm_b200 import pipelines as pl
    feats = np.vstack([pl.compute_color2d_superpixels_features(synth_regions(shape[0], shape[1], seed=s)[0], FEATS, sp_size=16)[1]
                       for s in seeds])
    feats = np.nan_to_num(feats)
    edges = np.quantile(feats[:, 0], np.linspace(0, 1, n_classes + 1)[1:-1])
    y = np.searchsorted(edges, feats[:, 0])
    assert len(np.unique(y)) == n_classes
    return feats, y


def test_forest_65_classes_pipeline_takes_the_host_path():
    from pyimsegm_b200 import pipelines as pl
    feats, y = _colour_training((131, 132), 65)
    model = ensemble.RandomForestClassifier(random_state=0, n_jobs=1, **RF).fit(feats, _spread(65)[y])
    img = synth_regions(320, 384, seed=133)[0]
    dev = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2, gc_regul=0.)
    with _host_predict():
        host = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2, gc_regul=0.)
    assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
    slic, f = pl.compute_color2d_superpixels_features(img, FEATS, sp_size=16)
    assert np.array_equal(dev[1], model.predict_proba(np.nan_to_num(f))[slic])
    assert set(np.unique(dev[0])) <= set(model.classes_)


def _tie_values(t):
    """float64 values on and around the float64 threshold t: t and its float64 neighbours; the float32 values on both sides of t
    (two each); the float32 rounding boundaries (midpoints of adjacent float32 values) around t and their float64 neighbours"""
    inf = np.float32(np.inf)
    f = np.float32(t)
    lo = f if float(f) <= t else np.nextafter(f, -inf)     # largest float32 <= t
    hi = np.nextafter(lo, inf)                              # smallest float32 > t
    f32 = [np.nextafter(lo, -inf), lo, hi, np.nextafter(hi, inf)]
    vals = [t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)] + [float(v) for v in f32]
    for a, b in zip(f32[:-1], f32[1:]):
        m = (float(a) + float(b)) / 2                       # exact in float64
        vals += [m, np.nextafter(m, -np.inf), np.nextafter(m, np.inf)]
    return np.array(vals, dtype=np.float64)


def _tie_rows(model, X, max_nodes=60, seed=0):
    """test rows that put the split feature of internal nodes on and around the node's threshold.  Each row starts from a training
    row that reaches the node; with a StandardScaler in front, the raw value is chosen (among the float64 neighbours of the exact
    preimage) so that the SCALED value, computed as sklearn and the device compute it, lands on the tie value.  Only rows that
    sklearn's own decision_path takes through their node are kept.
    Returns (rows [R, D] raw, the value the node compares [R], its threshold [R])."""
    scaler = model.steps[0][1] if isinstance(model, pipeline.Pipeline) else None
    Z = scaler.transform(X) if scaler is not None else X
    rng = np.random.RandomState(seed)
    rows, tid, nid = [], [], []
    for e, est in enumerate(_trees(model)):
        tr = est.tree_
        inner = np.flatnonzero(tr.children_left >= 0)
        inner = inner[rng.permutation(len(inner))[:max_nodes]]
        path = est.decision_path(Z).tocsc()
        for node in inner:
            base = X[path[:, node].indices[0]]
            f, vals = tr.feature[node], _tie_values(tr.threshold[node])
            if scaler is not None:                          # raw preimages: x = z s + m and two float64 neighbours each side
                x0 = vals * scaler.scale_[f] + scaler.mean_[f]
                near = [x0]
                for step in (-np.inf, np.inf):
                    near += [np.nextafter(x0, step), np.nextafter(np.nextafter(x0, step), step)]
                vals = np.concatenate(near)
            r = np.repeat(base[None], len(vals), axis=0)
            r[:, f] = vals
            rows.append(r)
            tid += [e] * len(vals)
            nid += [node] * len(vals)
    rows, tid, nid = np.vstack(rows), np.array(tid), np.array(nid)
    Zr = scaler.transform(rows) if scaler is not None else rows
    trees = _trees(model)
    feat = np.array([trees[e].tree_.feature[n] for e, n in zip(tid, nid)])
    thr = np.array([trees[e].tree_.threshold[n] for e, n in zip(tid, nid)])
    reached = np.zeros(len(rows), bool)
    for e, est in enumerate(trees):                         # sklearn's own path (float32 inputs): the row reaches its node
        sel = np.flatnonzero(tid == e)
        reached[sel] = np.asarray(est.decision_path(Zr[sel])[np.arange(len(sel)), nid[sel]]).ravel() > 0
    return rows[reached], Zr[reached, feat[reached]], thr[reached]


def _predict_without_cast(model, rows):
    """predict_proba with the float64 feature compared to the threshold directly (no float32 cast)"""
    scaler = model.steps[0][1] if isinstance(model, pipeline.Pipeline) else None
    Z = scaler.transform(rows) if scaler is not None else rows
    out = 0.0
    trees = _trees(model)
    for est in trees:
        tr = est.tree_
        node = np.zeros(len(Z), dtype=np.int64)
        while True:
            inner = tr.children_left[node] >= 0
            if not inner.any():
                break
            n = node[inner]
            go_left = Z[np.flatnonzero(inner), tr.feature[n]] <= tr.threshold[n]
            node[inner] = np.where(go_left, tr.children_left[n], tr.children_right[n])
        out = out + tr.value[node, 0, :]
    return out / len(trees) if len(trees) > 1 else out


@pytest.mark.parametrize('kind', ['tree', 'forest', 'extra'])
@pytest.mark.parametrize('scaled', [False, True])
def test_forest_threshold_ties_bit_exact(kind, scaled):
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(900, 4, 5, seed=7)
    if not scaled:
        X = np.round(X * 64) / 64                           # coarse values: split midpoints are float32 numbers
    model = _forest(kind, scaled).fit(X, _spread(5)[y])
    rows, z, thr = _tie_rows(model, X)
    z32 = z.astype(np.float32).astype(np.float64)
    on = z == thr
    flips = (z32 <= thr) != (z <= thr)                      # the float32 cast decides the branch
    above_left = (z > thr) & (z32 <= thr)                   # just above the threshold, rounded onto or below it: left
    below_right = (z <= thr) & (z32 > thr)
    f32_on = (z == z32) & (z32 == thr)
    f32_side = (z == z32) & (z32 != thr) & (np.abs(z - thr) <= 2 * np.spacing(np.abs(thr).astype(np.float32)))
    # the edges are reached, not only requested: counts of rows that arrive at their node with such a value
    assert np.count_nonzero(flips) >= 100, np.count_nonzero(flips)
    assert np.count_nonzero(above_left) >= 50, np.count_nonzero(above_left)
    assert np.count_nonzero(on) >= 20, np.count_nonzero(on)
    assert np.count_nonzero(f32_side) >= 100, np.count_nonzero(f32_side)
    if not scaled and kind != 'extra':                      # midpoint thresholds of coarse values are float32 numbers
        assert np.count_nonzero(f32_on) >= 50 and np.count_nonzero(below_right) == 0
    want = model.predict_proba(rows)
    # the float32 cast changes predict_proba on these rows, so a kernel without it cannot pass
    assert np.count_nonzero(np.any(_predict_without_cast(model, rows) != want, axis=1)) >= 20
    got = compile_model(model).predict_proba(rows)
    assert np.array_equal(got, want)


@pytest.mark.parametrize('kind', ['tree', 'forest'])
def test_forest_rows_past_n_dev_are_not_read(eng, kind):
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(1500, 6, 33, seed=33)
    model = _forest(kind, True).fit(X, _spread(33)[y])
    cm = compile_model(model)
    Xt, _ = _data(3000, 6, 33, seed=34)
    n_dev = 1777
    x = Xt.copy()
    x[n_dev:] = np.nan
    got, xt = _device_rows_only(eng, cm, x, n_dev)
    assert np.array_equal(got[:n_dev], model.predict_proba(Xt[:n_dev]))
    assert np.all(got[n_dev:] == SENTINEL) and np.all(xt[n_dev:] == SENTINEL)


# ---------------------------------------------------------------------------------------------------------------------------------
# k-nearest neighbours

KNN_QT, KNN_TT, KNN_TARGET_CTAS, KNN_MAX_SPLITS = 64, 64, 2 * 132, 32      # csrc/class_models.cu


def _knn_plan(N, N_t):
    """(splits, rows per split) of knn_plan"""
    q_tiles, t_tiles = -(-N // KNN_QT), -(-N_t // KNN_TT)
    s = min(max(-(-KNN_TARGET_CTAS // q_tiles), 1), KNN_MAX_SPLITS, t_tiles)
    per = -(-t_tiles // s)
    return -(-t_tiles // per), per * KNN_TT


def _knn_ws_bytes(splits, N, k):
    def align(b):
        return -(-b // 256) * 256
    return align(8 * splits * N * k) + align(4 * splits * N * k)


def _device_knn(eng, x, fit_x, y, k, n_classes, weights):
    from pyimsegm_b200.class_models import KNN_WEIGHTS, CompiledModel
    cm = CompiledModel('knn', x.shape[1], x.shape[1], n_classes, None, {'fit_x': fit_x, 'y': y.astype(np.int32)},
                       params={'n_neighbors': k, 'weights': KNN_WEIGHTS[weights]})
    proba = eng.class_model_predict(eng.to_device(np.ascontiguousarray(x), 'knn_edge_x'), cm)
    return eng.to_host(proba).copy()


def _check_knn(eng, x, fit_x, y, k, K):
    """both weightings against the oracle: uniform bit for bit, distance within 1e-12; returns the uniform oracle result"""
    want = onb.knn_predict_proba(x, fit_x, y, k, K)
    assert np.array_equal(_device_knn(eng, x, fit_x, y, k, K, 'uniform'), want)
    got = _device_knn(eng, x, fit_x, y, k, K, 'distance')
    assert np.abs(got - onb.knn_predict_proba(x, fit_x, y, k, K, 'distance')).max() <= 1e-12
    return want


@pytest.mark.parametrize('K', [31, 32, 33, 63, 64])
@pytest.mark.parametrize('k', [1, 33, 64])
def test_knn_class_columns(eng, K, k):
    from pyimsegm_b200.class_models import compile_model
    rng = np.random.RandomState(K * 100 + k)
    D = 3
    centres = rng.uniform(-20, 20, (K, D))
    counts = np.full(K, 40)
    single = [c for c in (0, 31, 32, K - 1) if c < K]      # classes with one training row, on both sides of 32
    counts[single] = 1
    y = rng.permutation(np.repeat(np.arange(K), counts))
    fit_x = centres[y] + rng.normal(0, 1.0, (len(y), D))
    x = centres[rng.randint(0, K, 3000)] + rng.normal(0, 1.5, (3000, D))
    x[:len(single)] = fit_x[[np.flatnonzero(y == c)[0] for c in single]]    # on the single rows: zero distances
    want = _check_knn(eng, x, fit_x, y, k, K)
    assert np.all(want[np.arange(len(single)), single] > 0)
    assert np.all(np.any(want == 0.0, axis=1))             # every row has classes none of its neighbours belongs to
    if K > 32:
        assert np.count_nonzero(want[:, 32:].max(axis=0)) == K - 32
    # the same tables from scikit-learn's layout (non-contiguous labels): identical to the oracle, and to sklearn away from near ties
    model = neighbors.KNeighborsClassifier(n_neighbors=k).fit(fit_x, _spread(K)[y])
    got = compile_model(model).predict_proba(x)
    assert np.array_equal(got, want)
    d2 = np.sort(onb.squared_distances(x, fit_x), axis=1)
    clear = d2[:, k] - d2[:, k - 1] > 1e-9 * (1 + d2[:, k])
    assert np.count_nonzero(clear) > len(x) // 2
    assert np.array_equal(got[clear], model.predict_proba(x[clear]))


@pytest.mark.parametrize('N', [1, 64])
def test_knn_32_splits(eng, N):
    N_t, D, K = 100000, 5, 64
    splits, per = _knn_plan(N, N_t)
    assert splits == KNN_MAX_SPLITS
    for k in (1, 33, 64):
        assert eng.lib.isb_knn_predict_workspace_bytes(N, N_t, k) == _knn_ws_bytes(KNN_MAX_SPLITS, N, k)
    assert _knn_ws_bytes(KNN_MAX_SPLITS, N, 64) != _knn_ws_bytes(KNN_MAX_SPLITS - 1, N, 64)   # the size tells 32 splits from 31
    rng = np.random.RandomState(N)
    fit_x = rng.uniform(-1, 1, (N_t, D))
    y = rng.randint(0, K, N_t)
    x = rng.uniform(-1, 1, (N, D))
    # near copies of every query in every split, the closest ones in the last split: each split holds some of the k nearest
    for s in range(splits):
        at = s * per + rng.choice(min(per, N_t - s * per), 2 * N, replace=False)
        fit_x[at] = np.repeat(x, 2, axis=0) + rng.normal(0, 1e-5 if s == splits - 1 else 1e-3, (2 * N, D))
    for k in (1, 33, 64):
        _check_knn(eng, x, fit_x, y, k, K)
        _, idx = onb.kneighbours(x, fit_x, k)
        assert np.all(idx[:, 0] // per == splits - 1)      # the nearest of all sits in the last split
        if k == 64:                                         # every split holds two of each query's 64 nearest
            assert all(np.array_equal(np.bincount(r // per, minlength=splits), np.full(splits, 2)) for r in idx)


@pytest.mark.parametrize('N', [1, 64])
def test_knn_last_split_shorter_than_k(eng, N):
    N_t, k, D, K = 2049, 64, 4, 40
    splits, per = _knn_plan(N, N_t)
    assert N_t - (splits - 1) * per == 1                   # the last split holds one row
    assert eng.lib.isb_knn_predict_workspace_bytes(N, N_t, k) == _knn_ws_bytes(splits, N, k)
    rng = np.random.RandomState(N + 1)
    fit_x = rng.normal(0, 1, (N_t, D))
    y = rng.randint(0, K - 1, N_t)
    y[-1] = K - 1                                           # the last row's class is its own
    x = rng.normal(0, 1, (N, D))
    fit_x[-1] = x[0]
    for kk in (1, 33, 64):
        want = _check_knn(eng, x, fit_x, y, kk, K)
        assert want[0, K - 1] > 0


def test_knn_duplicates_straddle_splits(eng):
    N, N_t, D, K = 64, 100000, 3, 64
    splits, per = _knn_plan(N, N_t)
    assert splits == KNN_MAX_SPLITS
    rng = np.random.RandomState(5)
    fit_x = rng.uniform(-1, 1, (N_t, D))
    y = rng.randint(0, K, N_t)
    x = rng.uniform(-1, 1, (N, D))
    # copies of each query on both sides of split boundaries, each copy with a class of its own
    for q in range(N):
        b = (q % (splits - 1) + 1) * per
        at = np.array([b - 1 - q, b + q, b + per // 2 + q]) % N_t
        fit_x[at] = x[q]
        y[at] = (np.arange(3) + 3 * q) % K
    for k in (1, 2, 3, 33, 64):
        _check_knn(eng, x, fit_x, y, k, K)
    _, idx = onb.kneighbours(x, fit_x, 3)
    assert np.all(fit_x[idx] == x[:, None])                 # the three copies are the three nearest
    assert np.all(idx[:, 0] // per != idx[:, 1] // per)     # and the lowest two sit in different splits
    one = _device_knn(eng, x, fit_x, y, 1, K, 'uniform')
    lowest = np.array([y[np.flatnonzero(np.all(fit_x == x[q], axis=1)).min()] for q in range(N)])
    assert np.array_equal(one, np.eye(K)[lowest])


def test_knn_rows_past_n_dev_are_not_read(eng):
    from pyimsegm_b200.class_models import compile_model
    X, y = _data(3000, 5, 40, seed=40, noise=0.05)
    model = neighbors.KNeighborsClassifier(n_neighbors=33).fit(X, _spread(40)[y])
    cm = compile_model(model)
    Xt, _ = _data(3000, 5, 40, seed=41, noise=0.05)
    n_dev = 1777
    x = Xt.copy()
    x[n_dev:] = np.nan
    got, xt = _device_rows_only(eng, cm, x, n_dev)
    assert np.array_equal(got[:n_dev], onb.knn_predict_proba(Xt[:n_dev], X, y, 33, 40))
    assert np.all(got[n_dev:] == SENTINEL) and np.all(xt[n_dev:] == SENTINEL)


# ---------------------------------------------------------------------------------------------------------------------------------
# logistic regression


def _logistic(K, D):
    X, y = _data(max(40 * K, 600), D, K, seed=K * 1000 + D, noise=0.3)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return linear_model.LogisticRegression(max_iter=200).fit(X, _spread(K)[y]), X


@pytest.mark.parametrize('K', [2, 33, 64])
@pytest.mark.parametrize('D', [1, 232])
def test_linear_extreme_decisions(K, D):
    import copy
    from pyimsegm_b200.class_models import compile_model
    model, X = _logistic(K, D)
    base, _ = _data(400, D, K, seed=5)
    base = base - X.mean(axis=0)
    lin = base @ model.coef_.T                              # the decision without the intercept
    rows = []
    for target in (40.0, 700.0, 800.0):                     # each row scaled so its largest |decision| is about the target
        a = target / np.abs(lin).max(axis=1)
        rows += [base * a[:, None], -base * a[:, None]]
    rows = np.vstack(rows)
    shifted = copy.deepcopy(model)                          # the same probabilities, every decision 900 lower
    shifted.intercept_ = model.intercept_ - 900.0
    for m in ((model, shifted) if K > 2 else (model, )):
        dec = m.decision_function(rows)
        assert np.abs(dec).max() > 790
        if K > 2 and m is model:
            assert np.any(dec.max(axis=1) > 710)            # exp() of the largest decision overflows without the shift
        if m is shifted:
            assert np.all(dec[:2 * len(base)].max(axis=1) < -746)   # the +-40 rows: exp() of every decision underflows unshifted
        if K == 2:
            assert np.any(dec > 37) and np.any(dec < -746)  # expit saturates at 1, and exp(-d) overflows to give 0
        cm = compile_model(m)
        assert cm.kind == 'linear' and cm.n_classes == K
        got = cm.predict_proba(rows)
        assert not np.isnan(got).any()
        assert np.abs(got - m.predict_proba(rows)).max() <= 1e-12
        with np.errstate(over='ignore'):                    # the oracle's exp(-d) overflows to inf, as the kernel's does
            want = onb.linear_predict_proba(rows, m.coef_, m.intercept_)
        assert np.abs(got - want).max() <= 1e-12
        assert np.abs(got.sum(axis=1) - 1).max() <= 1e-12


def test_linear_rows_past_n_dev_are_not_read(eng):
    from pyimsegm_b200.class_models import compile_model
    model, X = _logistic(64, 9)
    cm = compile_model(model)
    n_dev = 1777
    x = np.vstack([X, X])[:3000].copy()
    x[n_dev:] = np.nan
    got, xt = _device_rows_only(eng, cm, x, n_dev)
    assert np.abs(got[:n_dev] - model.predict_proba(x[:n_dev])).max() <= 1e-12
    assert np.all(got[n_dev:] == SENTINEL) and np.all(xt[n_dev:] == SENTINEL)


# ---------------------------------------------------------------------------------------------------------------------------------
# mixtures


def _mixture(kind, cov, K, max_iter=20):
    if kind == 'gmm':
        return mixture.GaussianMixture(K, covariance_type=cov, random_state=0, reg_covar=1e-3, max_iter=max_iter)
    prior = 'dirichlet_process' if kind == 'bgm_dp' else 'dirichlet_distribution'
    return mixture.BayesianGaussianMixture(n_components=K, covariance_type=cov, weight_concentration_prior_type=prior, random_state=0,
                                           reg_covar=1e-3, max_iter=max_iter)


def _fit_mixture(kind, cov, D, K, n=1500, seed=0):
    X, _ = _data(n, D, K, seed=seed + D * 10 + K)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()),
                                   ('model', _mixture(kind, cov, K, max_iter=20 if D < 200 else 8))]).fit(X)
    return model, X


@pytest.mark.parametrize('kind', ['gmm', 'bgm_dp', 'bgm_dd'])
@pytest.mark.parametrize('cov', ['full', 'tied', 'diag', 'spherical'])
@pytest.mark.parametrize('D,K', [(1, 1), (1, 8), (16, 8), (17, 8), (232, 2), (232, 8)])
def test_mixture_edges_within_1e9(kind, cov, D, K):
    from pyimsegm_b200.class_models import compile_model
    model, X = _fit_mixture(kind, cov, D, K, n=2000 if D > 200 else 1500)
    cm = compile_model(model)
    assert cm.kind == 'mixture' and (cm.n_dims, cm.n_classes) == (D, K)
    rng = np.random.RandomState(D + K)
    # rows 1e3 standard deviations (of the data, along a random direction) from the data and so from every component.  Their
    # log-densities are of order -1e6: float64 holds them to ~1e-10, the same order as the spread between sklearn's and any
    # other evaluation order, so 1e3 (not more) is where 1e-9 still separates a right log-sum-exp from a wrong one
    u = rng.normal(0, 1, (200, D))
    far = X.mean(axis=0) + 1e3 * X.std(axis=0) * u / np.linalg.norm(u, axis=1, keepdims=True)
    rows = np.vstack([X, far])
    got = cm.predict_proba(rows)
    want = model.predict_proba(rows)
    assert np.abs(got - want).max() < 1e-9
    g = got[len(X):]
    assert np.all(np.isfinite(g)) and np.abs(g.sum(axis=1) - 1).max() < 1e-9
    # the far rows do reach the edge: every component's weighted density underflows, only the log-sum-exp shift keeps them finite
    wlp = model.steps[-1][1]._estimate_weighted_log_prob(model.steps[0][1].transform(far))
    assert np.all(wlp.max(axis=1) < -746)


def test_mixture_limits_are_refused(eng):
    import ctypes as C
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.class_models import compile_model
    torch, lib = eng.torch, eng.lib
    for D, K in ((233, 2), (16, 9)):
        for kind in ('gmm', 'bgm_dp'):
            model, X = _fit_mixture(kind, 'diag', D, K)
            assert compile_model(model) is None and compile_model(model.steps[-1][1]) is None
        N = 8
        x = torch.zeros((N, D), dtype=torch.float64, device=eng.device)
        pc = torch.zeros((K, D, D), dtype=torch.float64, device=eng.device)
        bvec = torch.zeros((K, D), dtype=torch.float64, device=eng.device)
        cst = torch.zeros(K, dtype=torch.float64, device=eng.device)
        proba = torch.full((N, K), SENTINEL, dtype=torch.float64, device=eng.device)
        wsb = lib.isb_mixture_predict_workspace_bytes(N, D, K)
        ws = torch.zeros(max(wsb, 1), dtype=torch.uint8, device=eng.device)
        n0 = lib.isb_launch_count()
        st = lib.isb_mixture_predict_proba(_lib.ptr(x), N, None, D, K, _lib.ptr(pc), _lib.ptr(bvec), _lib.ptr(cst), _lib.ptr(proba),
                                           _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr())
        assert st == _lib.ISB_ERR_UNSUPPORTED and lib.isb_launch_count() == n0
        torch.cuda.synchronize()
        assert bool((proba == SENTINEL).all())


def test_mixture_nine_components_pipeline_takes_the_host_path():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.class_models import compile_model
    feats, _ = _colour_training((141, ), 2)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()), ('model', _mixture('gmm', 'full', 9))]).fit(feats)
    assert compile_model(model) is None
    img = synth_regions(320, 384, seed=142)[0]
    dev = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
    with _host_predict():
        host = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
    assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
    slic, f = pl.compute_color2d_superpixels_features(img, FEATS, sp_size=16)
    assert np.array_equal(dev[1], model.predict_proba(np.nan_to_num(f))[slic])


@pytest.mark.parametrize('D', [16, 232])
def test_mixture_rows_past_n_dev_are_not_read(eng, D):
    from pyimsegm_b200.class_models import compile_model
    model, X = _fit_mixture('gmm', 'full', D, 8, n=3000)
    cm = compile_model(model)
    n_dev = 1777
    x = X.copy()
    x[n_dev:] = np.nan
    got, xt = _device_rows_only(eng, cm, x, n_dev)
    assert np.abs(got[:n_dev] - model.predict_proba(X[:n_dev])).max() < 1e-9
    assert np.all(got[n_dev:] == SENTINEL) and np.all(xt[n_dev:] == SENTINEL)


# ---------------------------------------------------------------------------------------------------------------------------------
# end to end


def test_forty_class_forest_pipeline_matches_host():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.class_models import compile_model
    feats, y = _colour_training((151, 152, 153), 40)
    model = ensemble.RandomForestClassifier(random_state=0, n_jobs=1, **RF).fit(feats, 7 * y + 3)
    assert compile_model(model).n_classes == 40
    imgs = [synth_regions(320, 384, seed=s)[0] for s in (151, 154)]
    for img in imgs:
        dev = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
        with _host_predict():
            host = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16, sp_regul=0.2)
        assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
        assert set(np.unique(dev[0])) <= set(model.classes_)
        assert np.any(np.isin(dev[0], model.classes_[32:]))    # labels from the columns above 32 win somewhere
        assert np.count_nonzero(dev[1][..., 32:].max(axis=(0, 1))) >= 4
    batch = pl.segment_images_batch(imgs, dict_features=FEATS, sp_size=16, model_pipeline=model)
    for img, (segm, soft) in zip(imgs, batch):
        single = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=16)
        assert np.array_equal(segm, single[0]) and np.array_equal(soft, single[1])
