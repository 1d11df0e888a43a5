"""CPU tests of the training-set half of imsegm.classification: the host functions against the reference's own outputs
(tests/golden/dataset_reference.npz, made by make_dataset_goldens.py) with their types, the k-means starts against scikit-learn's
_init_centroids, the host steps of the k-means (empty-cluster relocation, best-run rule) against scikit-learn's, and the C entry
points' argument checks (no launch).  The k-means cases of the goldens run on the GPU (test_gpu_dataset_balance.py)."""
import ctypes as C
import json
import logging
import os
import random

import numpy as np
import pytest

from pyimsegm_b200 import classification as clf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

#: the training-set names of the reference's imsegm/classification.py
DATASET_NAMES = [
    'compose_dict_label_features', 'convert_dict_label_features_2_vectors', 'shuffle_features_labels', 'down_sample_dict_features_random',
    'down_sample_dict_features_kmean', 'unique_rows', 'down_sample_dict_features_unique', 'balance_dataset_by_',
    'convert_set_features_labels_2_dataset',
]


def load_gold():
    z = np.load(os.path.join(GOLDEN, 'dataset_reference.npz'))
    return json.loads(str(z['cases'])), {k: z[k] for k in z.files if k != 'cases'}


def unpack(node, arrays):
    """the value make_dataset_goldens.pack stored"""
    kind = node['type']
    if kind == 'ndarray':
        return arrays[node['key']]
    if kind == 'dict':
        out = {}
        for key, key_type, val in node['items']:
            out[np.dtype(key_type).type(key) if key_type.startswith(('int', 'uint')) and key_type != 'int' else key] = unpack(val, arrays)
        return out
    if 'key' in node:
        vals = arrays[node['key']].tolist()
        return tuple(vals) if kind == 'tuple' else vals
    if 'items' in node:
        items = [unpack(x, arrays) for x in node['items']]
        return tuple(items) if kind == 'tuple' else items
    return node['value']


def assert_same(got, node, arrays, where):
    """got equals the stored value with the same types: arrays with dtype and shape (NaN equal to NaN), lists and tuples with the type
    of every item, dicts with their keys, key types and order"""
    kind = node['type']
    if kind == 'ndarray':
        want = arrays[node['key']]
        assert isinstance(got, np.ndarray), where
        assert got.dtype == want.dtype and got.shape == want.shape, (where, got.dtype, want.dtype, got.shape, want.shape)
        assert np.array_equal(got, want, equal_nan=want.dtype.kind == 'f'), where
    elif kind == 'dict':
        assert isinstance(got, dict), where
        assert [(k, type(k).__name__) for k in got] == [(k, t) for k, t, _ in node['items']], where
        for (_, _, val), g in zip(node['items'], got.values()):
            assert_same(g, val, arrays, where)
    elif 'key' in node:
        assert type(got).__name__ == kind, where
        assert sorted({type(x).__name__ for x in got}) == node['elem'], where
        assert list(got) == arrays[node['key']].tolist(), where
    elif 'items' in node:
        assert type(got).__name__ == kind and len(got) == len(node['items']), where
        for g, val in zip(got, node['items']):
            assert_same(g, val, arrays, where)
    else:
        assert type(got).__name__ == kind and got == node['value'], where


def run_case(case, arrays):
    args = [unpack(a, arrays) for a in case['args']]
    if case['np_seed'] is not None:
        np.random.seed(case['np_seed'])
    if case['py_seed'] is not None:
        random.seed(case['py_seed'])
    return getattr(clf, case['func'])(*args, **case['kwargs'])


def uses_kmeans(case):
    return case['func'] == 'down_sample_dict_features_kmean' or str(case['kwargs'].get('balance_type', '')).lower() == 'kmeans'


CASES, ARRAYS = load_gold()


def test_every_dataset_name_is_importable():
    import importlib
    mod = importlib.import_module('imsegm.classification')
    for name in DATASET_NAMES:
        assert callable(getattr(mod, name)), name
    assert mod.ROUND_UNIQUE_FTS_DIGITS == 3
    assert {c['func'] for c in CASES} <= set(DATASET_NAMES)


@pytest.mark.parametrize('name', [c['name'] for c in CASES if not uses_kmeans(c)])
def test_host_functions_equal_reference(name):
    case = next(c for c in CASES if c['name'] == name)
    if 'raises' in case:
        with pytest.raises(Exception) as err:
            run_case(case, ARRAYS)
        assert type(err.value).__name__ == case['raises'][0] and str(err.value) == case['raises'][1]
        return
    assert_same(run_case(case, ARRAYS), case['out'], ARRAYS, name)


def test_unknown_balance_type_warns_and_keeps_every_row(caplog):
    fts, lbs = np.arange(12.).reshape(6, 2), np.array([0, 1, 1, 0, 1, 1])
    with caplog.at_level(logging.WARNING):
        out, labels = clf.balance_dataset_by_(fts, lbs, balance_type='median')
    assert 'not defined balancing method "median"' in caplog.text
    assert out.tolist() == fts[[0, 3, 1, 2, 4, 5]].tolist() and labels == [0, 0, 1, 1, 1, 1]


@pytest.mark.parametrize('seed', [0, 3, 17])
def test_kmeans_starts_equal_sklearn_init_centroids(seed):
    from sklearn.cluster import KMeans
    X = np.random.RandomState(seed).randn(57, 4)
    k = 9
    rs = np.random.RandomState(seed)
    km = KMeans(n_clusters=k, init='random')
    want = [km._init_centroids(X, np.einsum('ij,ij->i', X, X), 'random', rs, np.ones(len(X))) for _ in range(3)]
    np.random.seed(seed)
    got = [X[clf._kmeans_seeds(len(X), k)] for _ in range(3)]
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize('seed', range(6))
def test_relocation_and_average_equal_sklearn(seed):
    from sklearn.cluster._k_means_common import _relocate_empty_clusters_dense
    rng = np.random.RandomState(seed)
    n, k, D = 40, 9, 3
    X = np.round(rng.randn(n, D), 1)
    if seed % 2:
        X[10:] = X[0]                                   # many duplicates
    labels = rng.randint(0, k - 3, n).astype(np.int32)  # clusters k-3.. are empty
    centres_old = rng.randn(k, D)
    sums = np.zeros((k, D))
    np.add.at(sums, labels, X)
    weights = np.bincount(labels, minlength=k).astype(np.float64)
    want_s, want_w = sums.copy(), weights.copy()
    _relocate_empty_clusters_dense(X, np.ones(n), centres_old, want_s, want_w, labels)
    got_s, got_w = sums.copy(), weights.copy()
    clf._relocate_empty_clusters(X, centres_old, got_s, got_w, labels)
    assert np.array_equal(got_s, want_s) and np.array_equal(got_w, want_w)
    # _average_centers (cdef) restated: an empty cluster copies the heaviest one's row as the in-place loop has it at that point
    want = want_s.copy()
    heaviest = int(np.argmax(want_w))
    for j in range(k):
        if want_w[j] > 0:
            want[j] *= 1.0 / want_w[j]
        else:
            want[j] = want[heaviest]
    assert np.array_equal(clf._average_centres(want_s, want_w), want)


def test_same_clustering_equals_sklearn():
    from sklearn.cluster._k_means_common import _is_same_clustering
    rng = np.random.RandomState(1)
    for _ in range(50):
        a = rng.randint(0, 4, 12).astype(np.int32)
        perm = rng.permutation(4).astype(np.int32)
        for b in (perm[a], rng.randint(0, 4, 12).astype(np.int32), np.where(a == 0, 1, a).astype(np.int32)):
            assert clf._same_clustering(a, b, 4) == _is_same_clustering(a, b, 4)


def test_kmeans_entry_points_reject_bad_arguments():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    assert lib.isb_abi_version() == 8
    for name in ('isb_kmeans_workspace_bytes', 'isb_kmeans_lloyd', 'isb_kmeans_nearest'):
        assert name in _lib.SIGNATURES
    assert lib.isb_kmeans_workspace_bytes(100, 10, 257) == 0
    assert lib.isb_kmeans_workspace_bytes(10, 11, 3) == 0
    lloyd = lambda n, D, k, max_iter, sweeps=1, ptr=p: lib.isb_kmeans_lloyd(ptr, n, D, k, max_iter, sweeps, C.c_double(0.), p, p, p, p, p,
                                                                             p, p, C.c_size_t(1 << 40), None)
    assert lloyd(100, 257, 10, 5) == _lib.ISB_ERR_UNSUPPORTED and b'256' in lib.isb_last_error()
    assert lloyd(10, 3, 11, 5) == _lib.ISB_ERR_ARG
    assert lloyd(10, 3, 0, 5) == _lib.ISB_ERR_ARG
    assert lloyd(10, 3, 4, 0) == _lib.ISB_ERR_ARG
    assert lloyd(10, 3, 4, 5, ptr=None) == _lib.ISB_ERR_ARG
    assert lloyd(10, 3, 4, 5, sweeps=6) == _lib.ISB_ERR_ARG and lloyd(10, 3, 4, 5, sweeps=-1) == _lib.ISB_ERR_ARG
    assert lib.isb_kmeans_nearest(p, 100, 300, p, 10, p, p, C.c_size_t(1 << 40), None) == _lib.ISB_ERR_UNSUPPORTED
    assert lib.isb_kmeans_nearest(p, 5, 3, p, 6, p, p, C.c_size_t(1 << 40), None) == _lib.ISB_ERR_ARG


def test_kmeans_input_errors_raise_before_the_device():
    with pytest.raises(ValueError, match='NaN'):
        clf._kmeans_sample(np.full((5, 2), np.nan), 2)
    with pytest.raises(ValueError, match='n_clusters'):
        clf._kmeans_sample(np.zeros((5, 2)), 6)
