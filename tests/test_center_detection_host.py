"""CPU tests of the centre detection (pyimsegm_b200/center_detection.py): the feature table's names, column order and ``params``
handling against the reference's composition on the oracle, with the device calls replaced by host twins; the host twin of the
ring counts against oracle.label_histograms_positions; the integer disc half-widths; ``label_close_points`` on both centre formats;
and the argument checks of the new C-ABI entries, which return before any CUDA call."""
import os
import sys

import numpy as np
import pytest

import oracle
from pyimsegm_b200 import center_detection as cd
from pyimsegm_b200 import descriptors as ds

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import center_host_reference as chr_  # noqa: E402
from make_center_goldens import load  # noqa: E402


@pytest.fixture(scope='module')
def ovary():
    oracle.build()
    with np.load(os.path.join(HERE, 'golden', 'center_detection_reference.npz')) as z:
        return load(z, 'insitu7545')


@pytest.fixture
def host_devices(monkeypatch):
    monkeypatch.setattr(ds, '_device_label_hists', chr_.device_hists_on_host)
    monkeypatch.setattr(ds, 'cython_ray_features_seg2d', chr_.ray_tracer)


def test_disc_half_widths_are_exact_up_to_2000():
    for d in range(0, 2001):
        dys = np.arange(-d, d + 1, dtype=np.int64)
        w = chr_.disc_half_widths(d, dys)
        assert np.all(dys ** 2 + w ** 2 <= d * d) and np.all(dys ** 2 + (w + 1) ** 2 > d * d), d
    for d in (0, 1, 2, 5, 17):                  # skimage.morphology.disk(d) row by row
        disk = oracle.disk(d)
        np.testing.assert_array_equal(disk.sum(axis=1), 2 * chr_.disc_half_widths(d, np.arange(-d, d + 1)) + 1)


@pytest.mark.parametrize('nb_labels', [1, 3, 7])
def test_host_ring_counts_equal_the_oracle(nb_labels):
    rng = np.random.RandomState(nb_labels)
    H, W = 23, 31
    segm = rng.randint(-1, nb_labels + 2, (H, W))
    positions = [[0, 0], [0, W - 1], [H - 1, 0], [H - 1, W - 1], [H // 2, W // 3], [5, 0], [0, 7]]
    diameters = [0, 1, 3, 8, 40]
    hist, sizes = chr_.label_disc_counts(segm, positions, diameters, nb_labels)
    for i, pos in enumerate(positions):
        for j, d in enumerate(diameters):
            want, size = oracle.label_hist_selem(segm, pos, oracle.disk(d), nb_labels)
            np.testing.assert_array_equal(hist[i, j], want)
            assert sizes[i, j] == size
    segm = np.clip(segm, 0, None)
    pos, diams = positions[:5], [1, 3, 8, 40]
    np.testing.assert_array_equal(chr_.label_histograms_positions(segm, pos, diams), oracle.label_histograms_positions(segm, pos, diams))


PARAMS = [
    dict(cd.CENTER_PARAMS),
    dict(cd.CENTER_PARAMS, fts_ray_types=[('up', [0]), ('down', [1])]),
    dict(cd.CENTER_PARAMS, fts_ray_types=[('up', [0]), ('down', [1])], fts_ray_closer=False, fts_ray_smooth=1),
    dict(cd.CENTER_PARAMS, fts_hist_diams=None),
    dict(cd.CENTER_PARAMS, fts_ray_step=None),
    dict(cd.CENTER_PARAMS, fts_hist_diams=[5, 25], fts_ray_step=30, fts_ray_types=[('up', [0, 1])]),
]


@pytest.mark.parametrize('params', PARAMS, ids=['default', 'closer', 'two_types', 'no_hist', 'no_rays', 'short'])
def test_points_features_names_and_columns(ovary, host_devices, params):
    _, segm, _, _ = ovary
    rng = np.random.RandomState(3)
    points = [(float(r), float(c)) for r, c in zip(rng.uniform(0, segm.shape[0] - 1, 40), rng.uniform(0, segm.shape[1] - 1, 40))]
    got, names = cd.compute_points_features(segm, points, params)
    want, want_names = chr_.points_features(segm, points, params)
    assert names == want_names
    assert got.shape == (len(points), len(names))
    np.testing.assert_array_equal(got, want)
    nb = int(segm.max()) + 1
    n_hist = len(params['fts_hist_diams']) * nb if params.get('fts_hist_diams') else 0
    assert all(n.startswith('hist-d_') for n in names[:n_hist]) and all(n.startswith('ray-lb_') for n in names[n_hist:])


def test_points_features_of_no_parameters_are_empty(ovary):
    _, segm, _, _ = ovary
    got, names = cd.compute_points_features(segm, [(3, 4), (10, 10)], {})
    assert got.shape == (2, 0) and names == []


def test_estim_points_rejects_mismatched_shapes():
    with pytest.raises(Exception, match='not matching shapes'):
        cd.estim_points_compute_features('x', np.zeros((10, 12, 3)), np.zeros((10, 11)), cd.CENTER_PARAMS)


def test_label_close_points_on_both_centre_formats(ovary):
    _, _, levels, centres = ovary
    rng = np.random.RandomState(0)
    points = [(int(r), int(c)) for r, c in zip(rng.randint(0, levels.shape[0], 200), rng.randint(0, levels.shape[1], 200))]
    points += [tuple(map(int, c)) for c in centres]
    got = cd.label_close_points([tuple(c) for c in centres], points, {'center_dist_thr': 50})
    d = np.sqrt(((np.array(points)[:, None, :] - centres[None]) ** 2).sum(-1)).min(axis=1)
    np.testing.assert_array_equal(got, d <= 50)
    assert got[-len(centres):].all()
    got = cd.label_close_points(levels, points, {})
    np.testing.assert_array_equal(got, [levels[r, c] for r, c in points])
    assert cd.label_close_points(None, points, {}) == [-1] * len(points)


def test_cluster_center_candidates_of_no_points():
    centres, labels = cd.cluster_center_candidates([])
    assert isinstance(centres, np.ndarray) and centres.size == 0 and labels == []
    centres, labels = cd.cluster_center_candidates(np.zeros((0, 2)))
    assert centres.shape == (0, 2) and labels == []


@pytest.mark.parametrize('kw', [dict(max_dist=0), dict(max_dist=-1.), dict(min_samples=0), dict(min_samples=1.5)])
def test_cluster_center_candidates_rejects_bad_parameters(kw):
    with pytest.raises(ValueError):
        cd.cluster_center_candidates([[0., 0.], [1., 1.]], **kw)


def test_cluster_center_candidates_rejects_non_finite_points():
    with pytest.raises(ValueError):
        cd.cluster_center_candidates([[0., 0.], [np.nan, 1.]])


def test_new_entries_reject_bad_arguments_without_a_device():
    import ctypes as C
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    assert lib.isb_label_runs_workspace_bytes(0, 5) == 0 and lib.isb_label_runs_workspace_bytes(4, 5) >= 2 * 4 * 20
    bad = [
        lambda: lib.isb_ring_label_hist(None, 8, 8, p, 1, p, 1, 3, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, None, 1, p, 1, 3, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 1, p, 1, 3, p, p, None, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 0, 8, p, 1, p, 1, 3, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 0, p, 1, 3, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 1, p, 0, 3, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 1, p, 1, 0, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 1, p, 1, 4097, p, p, p, 1 << 20, None),
        lambda: lib.isb_ring_label_hist(p, 8, 8, p, 1, p, 1, 3, p, p, p, 16, None),
        lambda: lib.isb_dbscan(p, 4, 1.0, 1, p, None, None, p, 1 << 20, None),
        lambda: lib.isb_dbscan(None, 4, 1.0, 1, p, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, 4, 1.0, 1, None, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, -1, 1.0, 1, p, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, 4, 0.0, 1, p, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, 4, float('nan'), 1, p, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, 4, float('inf'), 1, p, None, C.byref(C.c_int()), p, 1 << 20, None),
        lambda: lib.isb_dbscan(p, 4, 1.0, 0, p, None, C.byref(C.c_int()), p, 1 << 20, None),
    ]
    for i, call in enumerate(bad):
        assert call() == _lib.ISB_ERR_ARG, i
        assert lib.isb_last_error()
    k = C.c_int(7)
    assert lib.isb_dbscan(None, 0, 1.0, 1, None, None, C.byref(k), None, 0, None) == _lib.ISB_OK and k.value == 0


def test_abi_version_is_unchanged():
    from pyimsegm_b200 import _lib
    assert _lib.lib().isb_abi_version() == 8


def test_imsegm_alias():
    import imsegm.center_detection
    assert imsegm.center_detection is cd
