"""GPU tests of the k-means down-sampling of balance_dataset_by_(..., 'kmeans') (csrc/kmeans_sample.cu): one sweep against the float64
oracle (oracle/dataset.py) at the tile edges, whole runs against scikit-learn with the same seed, duplicate rows that empty clusters,
determinism, and the reference's own outputs (tests/golden/dataset_reference.npz).

Selected rows.  The row kept for a centre is the one of least exact squared distance; scikit-learn takes the least of
|x|^2 - 2 x.c + |c|^2 from its BLAS.  Two rows at the same true distance -- the two members of a two-member cluster are equidistant
from their mean -- are told apart by rounding only, differently on the two sides.  So the selected rows must be identical except
where both picks lie within the expansion's rounding bound of the least distance (oracle/dataset.py selection_ties).

Label bound.  The device labels a row by v_j = fl(|c_j|^2 - 2 x.c_j), dot products of depth D accumulated in float64 (tensor-core
FMA steps), and the oracle by d_j = sum_d (x_d - c_jd)^2 with the differences taken first.  With u = 2^-53 and gamma_m = m u / (1 - m u),
|v_j - (d_j - |x|^2)| <= gamma_(D+1) (|c_j|^2 + 2 sum_d |x_d c_jd|) <= gamma_(D+1) (|c_j|^2 + 2 |x| |c_j|) (Cauchy-Schwarz), and the
oracle's |fl(d_j) - d_j| <= gamma_(D+2) d_j.  Both labels are the same row's true nearest centre, hence equal, when the oracle's margin
d_(2) - d_(1) exceeds twice the first bound with the largest centre plus the second for d_(1) and d_(2):
    bound_i = 2 gamma_(D+2) (max_j |c_j|^2 + 2 |x_i| max_j |c_j|) + gamma_(D+2) (d_(1) + d_(2)),
which the test doubles.
"""
import ctypes as C
import warnings

import numpy as np
import pytest

from oracle import dataset as od
from pyimsegm_b200 import _lib
from pyimsegm_b200 import classification as clf
from pyimsegm_b200.engine import get_engine
from test_dataset_balance_host import ARRAYS, CASES, assert_same, run_case, uses_kmeans

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def label_bound(X, centres, best, margin):
    D = X.shape[1]
    gamma = (D + 2) * U / (1 - (D + 2) * U)
    cn = np.sqrt((centres ** 2).sum(axis=1)).max()
    xn = np.sqrt((X ** 2).sum(axis=1))
    return 2 * (2 * gamma * (cn * cn + 2 * xn * cn) + gamma * (2 * best + margin))


def device_run(X, centres, max_iter, tol, status=(0, 0, 0, 0)):
    """one isb_kmeans_lloyd call from the given status: (labels, centres, inertia, status); status (2, 0, 0, 0) only labels the rows"""
    eng = get_engine()
    torch, lib, st = eng.torch, eng.lib, _lib.stream_ptr()
    n, D = X.shape
    k = len(centres)
    d_x = eng.to_device(np.ascontiguousarray(X, np.float64))
    d_c = eng.to_device(np.ascontiguousarray(centres, np.float64))
    labels = eng.to_device(np.full(n, -1, np.int32))
    d_st = eng.to_device(np.array(status, np.int32))
    sums = torch.empty((k, D), dtype=torch.float64, device=eng.device)
    counts = torch.empty(k, dtype=torch.int32, device=eng.device)
    inertia = torch.empty(1, dtype=torch.float64, device=eng.device)
    ws_bytes = lib.isb_kmeans_workspace_bytes(n, k, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=eng.device)
    sweeps = max_iter if status[0] == 0 else 0
    _lib.check(lib.isb_kmeans_lloyd(_lib.ptr(d_x), n, D, k, max_iter, sweeps, C.c_double(tol), _lib.ptr(d_c), _lib.ptr(labels), _lib.ptr(d_st),
                                    _lib.ptr(sums), _lib.ptr(counts), _lib.ptr(inertia), _lib.ptr(ws), C.c_size_t(ws_bytes), st))
    return eng.to_host(labels).copy(), eng.to_host(d_c).copy(), float(eng.to_host(inertia)[0]), eng.to_host(d_st).copy()


SWEEP_SIZES = [(1, 1, 1), (127, 1, 9), (129, 64, 189), (128, 63, 232), (300, 65, 31), (257, 256, 33), (1000, 999, 9), (200, 199, 189),
               (131, 7, 232), (4099, 130, 189), (96, 65, 4)]


@pytest.mark.parametrize('n,k,D', SWEEP_SIZES)
def test_one_sweep_against_float64_oracle(n, k, D):
    rng = np.random.RandomState(n + 7 * k + D)
    X = rng.randn(n, D) * rng.uniform(0.5, 4.0, D) + rng.randn(D)
    C0 = X[rng.choice(n, k, replace=False)]
    # labels against the given centres (the status of a run that stopped on its shift: only the E-step and the inertia run)
    lab, c_out, inertia, status = device_run(X, C0, 1, 0.0, status=(2, 0, 0, 0))
    assert np.array_equal(c_out, C0) and status[0] == 2
    want, best, margin = od.assign(X, C0)
    clear = np.isinf(margin) | (margin > label_bound(X, C0, best, margin))
    assert clear.mean() > 0.99
    assert np.array_equal(lab[clear], want[clear])
    exact = ((X - C0[lab]) ** 2).sum()
    assert abs(inertia - exact) <= 1e-12 * exact + 1e-300
    # one sweep: centres = the member means of those labels, then the E-step against them
    lab1, c1, inertia1, status1 = device_run(X, C0, 1, -1.0)
    assert tuple(status1[:2]) == (4, 1)
    means, counts = od.member_means(X, lab, k)
    full = counts > 0
    assert np.all(np.abs(c1[full] - means[full]) <= 1e-12 * np.maximum(np.abs(means[full]), np.abs(X).max()))
    want1, best1, margin1 = od.assign(X, c1)
    clear1 = np.isinf(margin1) | (margin1 > label_bound(X, c1, best1, margin1))
    assert np.array_equal(lab1[clear1], want1[clear1])


def blobs(n, k_blobs, D, seed, spread=0.3):
    rng = np.random.RandomState(seed)
    centres = rng.randn(k_blobs, D) * 3
    return centres[rng.randint(0, k_blobs, n)] + rng.randn(n, D) * spread


def check_against_sklearn(X, k, seed):
    runs, selected = od.sklearn_runs(X, k, seed)
    np.random.seed(seed)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        got, dev_runs, best = clf._kmeans_sample(X, k)
    for (labels, inertia, _), run in zip(runs, dev_runs):
        assert np.array_equal(run.labels, labels)
        assert abs(run.inertia - inertia) <= 1e-10 * abs(inertia)
    n_diff, ties = od.selection_ties(X, best.centres + X.mean(axis=0), got, selected)
    assert ties, '%d selected rows differ beyond rounding' % n_diff
    return caught


@pytest.mark.parametrize('n,k,D,seed', [(600, 40, 9, 0), (2000, 150, 189, 1), (3000, 500, 232, 2), (5000, 1000, 33, 3)])
def test_whole_function_against_sklearn(n, k, D, seed):
    check_against_sklearn(blobs(n, max(2 * k, 8), D, seed), k, seed)


def test_whole_function_against_sklearn_30000_x_189():
    X = blobs(30000, 6000, 189, 5)
    # the premise of label equality: every row's nearest start clears the label bound by far
    np.random.seed(5)
    starts = X[clf._kmeans_seeds(len(X), 3000)] - X.mean(axis=0)
    _, best, margin = od.assign(X[:2000] - X.mean(axis=0), starts)
    assert np.all(margin > 1e3 * label_bound(X[:2000] - X.mean(axis=0), starts, best, margin))
    check_against_sklearn(X, 3000, 5)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_duplicate_rows_relocate_empty_clusters_as_sklearn(seed, monkeypatch):
    rng = np.random.RandomState(seed)
    X = np.repeat(rng.randn(40, 6), 5, axis=0)[rng.permutation(200)]
    calls = []
    relocate = clf._relocate_empty_clusters
    monkeypatch.setattr(clf, '_relocate_empty_clusters', lambda *a: calls.append(1) or relocate(*a))
    check_against_sklearn(X, 30, seed)
    assert calls, 'no sweep left a cluster empty'


def test_more_clusters_than_distinct_rows_warns_as_sklearn():
    X = np.repeat(np.random.RandomState(4).randn(12, 3), 4, axis=0)
    caught = check_against_sklearn(X, 20, 1)
    assert any('Number of distinct clusters (12) found smaller than n_clusters (20)' in str(w.message) for w in caught)


def test_identical_rows_tie_to_the_lowest_index():
    X = np.zeros((10, 3))
    X[5:] = 1.0
    nearest, _, _ = clf._kmeans_sample(X, 2)
    assert sorted(nearest.tolist()) == [0, 5]
    lab, _, _, _ = device_run(X, np.ones((2, 3)), 1, 0.0, status=(2, 0, 0, 0))
    assert lab.tolist() == [0] * 10


def record_kmeans(monkeypatch=None):
    """calls of clf._kmeans_sample from here on, as (features, selected rows, uncentred best centres)"""
    calls = []
    inner = clf._kmeans_sample

    def wrapped(features, nb_samples):
        out = inner(features, nb_samples)
        calls.append((np.asarray(features, np.float64), out[0], out[2].centres + np.asarray(features, np.float64).mean(axis=0)))
        return out
    (monkeypatch.setattr if monkeypatch else setattr)(clf, '_kmeans_sample', wrapped)
    return calls


def test_class_already_at_nb_samples_is_copied(monkeypatch):
    X = blobs(90, 10, 5, 6)
    y = np.r_[np.zeros(50, int), np.ones(20, int), np.full(20, 2)]
    np.random.seed(3)
    calls = record_kmeans(monkeypatch)
    fts, lbs = clf.balance_dataset_by_(X, y, balance_type='kmeans')
    _, selected = od.sklearn_runs(X[:50], 20, 3)
    assert len(calls) == 1 and np.array_equal(fts[20:], X[50:])
    assert od.selection_ties(X[:50], calls[0][2], calls[0][1], selected)[1]
    assert np.array_equal(fts[:20], X[:50][calls[0][1]])
    assert lbs == [0] * 20 + [1] * 20 + [2] * 20


def test_two_runs_are_bit_identical():
    X = blobs(6000, 400, 189, 8)
    outs = []
    for _ in range(2):
        np.random.seed(11)
        outs.append(clf._kmeans_sample(X, 300))
    (sel_a, runs_a, best_a), (sel_b, runs_b, best_b) = outs
    assert np.array_equal(sel_a, sel_b)
    for ra, rb in zip(runs_a, runs_b):
        assert np.array_equal(ra.labels, rb.labels) and ra.inertia == rb.inertia and np.array_equal(ra.centres, rb.centres)


def test_wide_features_raise_not_implemented():
    with pytest.raises(NotImplementedError):
        clf._kmeans_sample(np.random.RandomState(0).randn(20, 257), 3)


def is_tie(g, w, calls):
    """row g of the device output and row w of the reference's were kept for the same centre and are a rounding tie"""
    for X, sel, centres in calls:
        for j in np.where(np.all(X[sel] == g, axis=1))[0]:
            r = np.where(np.all(X == w, axis=1))[0]
            if len(r) and od.selection_ties(X, centres[j:j + 1], sel[j:j + 1], r[:1])[1]:
                return True
    return False


def assert_same_up_to_ties(got, node, arrays, calls, where):
    """assert_same, except that a feature row may differ from the reference's where the two are a rounding tie"""
    if node['type'] == 'ndarray' and arrays[node['key']].ndim == 2 and arrays[node['key']].dtype.kind == 'f':
        want = arrays[node['key']]
        assert got.dtype == want.dtype and got.shape == want.shape, where
        for p in np.where(~np.all(got == want, axis=1))[0]:
            assert is_tie(got[p], want[p], calls), (where, p)
    elif node['type'] == 'dict':
        assert [(k, type(k).__name__) for k in got] == [(k, t) for k, t, _ in node['items']], where
        for (_, _, val), g in zip(node['items'], got.values()):
            assert_same_up_to_ties(g, val, arrays, calls, where)
    elif 'items' in node:
        assert type(got).__name__ == node['type'] and len(got) == len(node['items']), where
        for g, val in zip(got, node['items']):
            assert_same_up_to_ties(g, val, arrays, calls, where)
    else:
        assert_same(got, node, arrays, where)


@pytest.mark.parametrize('name', [c['name'] for c in CASES if uses_kmeans(c)])
def test_kmeans_cases_equal_reference(name, monkeypatch):
    case = next(c for c in CASES if c['name'] == name)
    calls = record_kmeans(monkeypatch)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = run_case(case, ARRAYS)
    assert calls
    assert_same_up_to_ties(got, case['out'], ARRAYS, calls, name)
