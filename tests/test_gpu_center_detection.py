"""GPU tests of the centre detection: the run-length ring histograms (``isb_ring_label_hist``) bit-equal to the oracle and to
``isb_disc_label_hist`` at their position, diameter, shape, label and count edges; DBSCAN labels and cluster centres identical to
scikit-learn's; and the whole detection on the ovary fixtures identical to the host composition (oracle features, scikit-learn
predict, scikit-learn DBSCAN)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import center_host_reference as chr_  # noqa: E402
from make_center_goldens import load  # noqa: E402

pytestmark = pytest.mark.gpu


def _both_routes(segm, positions, diameters, nb_labels):
    """(run-length counts, pixel-walk counts) of _device_label_hists"""
    from pyimsegm_b200 import descriptors as ds
    new = ds._device_label_hists(segm, positions, nb_labels, diameters=diameters)
    ds.RUN_LENGTH_DISCS = False
    try:
        old = ds._device_label_hists(segm, positions, nb_labels, diameters=diameters)
    finally:
        ds.RUN_LENGTH_DISCS = True
    return new, old


def _check_counts(oracle, segm, positions, diameters, nb_labels, exhaustive=True):
    (hist, sizes), (hist_o, sizes_o) = _both_routes(segm, positions, diameters, nb_labels)
    assert np.array_equal(hist, hist_o) and np.array_equal(sizes, sizes_o)
    want_h, want_s = chr_.label_disc_counts(np.where(np.isnan(np.asarray(segm, float)), -1, segm).astype(np.int64),
                                            [list(map(int, p)) for p in positions], diameters, nb_labels)
    assert np.array_equal(hist, want_h) and np.array_equal(sizes, want_s)
    if exhaustive:
        for i, pos in enumerate(positions):
            for j, d in enumerate(diameters):
                want, size = oracle.label_hist_selem(np.where(np.isnan(np.asarray(segm, float)), -1, segm), pos, oracle.disk(d), nb_labels)
                np.testing.assert_array_equal(hist[i, j], want, err_msg='position %r diameter %d' % (pos, d))
                assert sizes[i, j] == size


def _edges(H, W):
    return [[0, 0], [0, W - 1], [H - 1, 0], [H - 1, W - 1], [H // 2, W // 2], [0, W // 2], [H - 1, W // 3], [H // 2, 0], [H // 3, W - 1]]


@pytest.mark.parametrize('shape', [(37, 53), (1, 40), (40, 1), (1, 1), (5, 300)], ids=str)
def test_ring_counts_at_corners_borders_and_diameters(oracle, shape):
    H, W = shape
    rng = np.random.RandomState(H * 7 + W)
    segm = rng.randint(-2, 6, (H, W))                 # negative labels and labels >= nb_labels = 4
    _check_counts(oracle, segm, _edges(H, W), [0, 1, 2, 7, max(H, W) + 5, 3 * (H + W)], 4)


@pytest.mark.parametrize('kind', ['one_run_per_row', 'change_every_pixel', 'stripes', 'nan'])
def test_ring_counts_run_patterns(oracle, kind):
    H, W = 45, 61
    yy, xx = np.mgrid[:H, :W]
    segm = {'one_run_per_row': yy % 3, 'change_every_pixel': (xx + yy) % 3, 'stripes': (xx // 5) % 4,
            'nan': np.where((xx + 2 * yy) % 7 == 0, np.nan, (xx // 3) % 3)}[kind]
    _check_counts(oracle, segm, _edges(H, W), [0, 1, 4, 10, 30, 100], 3)


@pytest.mark.parametrize('nb_labels', [1, 2, 33, 189, 191, 255, 511, 700, 1023, 4096])
def test_ring_counts_label_counts(oracle, nb_labels):
    rng = np.random.RandomState(nb_labels)
    H, W = 71, 83
    segm = rng.randint(0, nb_labels, (H, W))
    segm[:, ::2] = np.repeat(rng.randint(0, nb_labels, (H, 1)), (W + 1) // 2, axis=1)
    _check_counts(oracle, segm, _edges(H, W), [0, 3, 20, 150], nb_labels, exhaustive=nb_labels <= 33)


def test_ring_counts_every_label_count():
    """nb_labels 1 .. 4096: the counters of up to 32 diameters share one CTA's shared memory with its static arrays, so the
    number of diameters per pass changes with the label count; every count must launch and count right"""
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(0)
    H, W = 9, 11
    positions, diameters = [[0, 0], [4, 5], [8, 10]], [0, 2, 4, 20]
    for nb_labels in range(1, 4097):
        segm = rng.randint(0, nb_labels + 1, (H, W))
        hist, sizes = ds._device_label_hists(segm, positions, nb_labels, diameters=diameters)
        want_h, want_s = chr_.label_disc_counts(segm, positions, diameters, nb_labels)
        assert np.array_equal(hist, want_h) and np.array_equal(sizes, want_s), nb_labels


@pytest.mark.parametrize('n_pos', [1, 20000])
def test_ring_counts_many_positions(oracle, n_pos):
    rng = np.random.RandomState(n_pos)
    H, W = 160, 210
    from scipy import ndimage
    segm = (ndimage.gaussian_filter(rng.rand(H, W), 3) * 40).astype(int) % 5
    positions = np.stack([rng.randint(0, H, n_pos), rng.randint(0, W, n_pos)], axis=1).tolist()
    _check_counts(oracle, segm, positions, [10, 50, 100], 5, exhaustive=False)


def test_ring_histograms_equal_the_oracle(oracle):
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(5)
    segm = rng.randint(0, 4, (90, 120))
    positions = _edges(90, 120) + rng.randint(0, 90, (30, 2)).tolist()
    diameters = [1, 5, 12, 40, 200]
    got, _ = ds.compute_label_histograms_positions(segm, positions, diameters)
    assert np.array_equal(got, oracle.label_histograms_positions(segm, positions, diameters))


# ---------------------------------------------------------------------------------------------------------------------------------
# DBSCAN
# ---------------------------------------------------------------------------------------------------------------------------------

def _check_dbscan(points, eps, min_samples):
    from pyimsegm_b200 import center_detection as cd
    got_c, got_l = cd.cluster_center_candidates(points, eps, min_samples)
    want_c, want_l = chr_.cluster_center_candidates(points, eps, min_samples)
    assert np.array_equal(np.asarray(got_l), np.asarray(want_l))
    assert np.asarray(got_c).shape == np.asarray(want_c).shape and np.array_equal(got_c, want_c)
    return got_l


@pytest.mark.parametrize('min_samples', [1, 2, 5])
@pytest.mark.parametrize('kind', ['float', 'integer'])
def test_dbscan_random_sets(kind, min_samples):
    rng = np.random.RandomState(min_samples)
    for n, eps in ((12, 0.2), (300, 0.05), (3000, 0.02)):
        pts = rng.rand(n, 2) if kind == 'float' else rng.randint(0, int(np.sqrt(n) * 3), (n, 2))
        _check_dbscan(pts, eps if kind == 'float' else 2., min_samples)


def test_dbscan_clustered_candidates():
    rng = np.random.RandomState(1)
    centres = rng.rand(40, 2) * 1000
    pts = np.concatenate([c + rng.normal(0, 15, (rng.randint(1, 30), 2)) for c in centres])
    for eps, ms in ((50, 1), (20, 3), (8, 2)):
        _check_dbscan(pts, eps, ms)


def test_dbscan_border_points_between_two_clusters():
    # two dense clusters; the border points at x = 5 are within eps of a core point of each; x = 10.5 joins the right one only
    left = np.array([[0., 0.], [0., 1.], [1., 0.], [1., 1.], [4., 0.5]])
    right = np.array([[10., 0.], [10., 1.], [9., 0.], [9., 1.], [6., 0.5]])
    border = np.array([[5., 0.5], [5., 0.6], [10.5, 20.]])
    for pts in (np.concatenate([left, right, border]), np.concatenate([border, right, left]), np.concatenate([right, border, left])):
        labels = _check_dbscan(pts, 1.5, 3)
        assert (np.asarray(labels) >= 0).sum() >= 10


def test_dbscan_all_noise_and_exact_eps_pairs():
    labels = _check_dbscan(np.arange(40, dtype=float).reshape(20, 2) * 10, 1., 2)
    assert np.all(np.asarray(labels) == -1)
    # pairs exactly eps apart on integer coordinates: neighbours (distance <= eps)
    pts = np.array([[0, 0], [3, 4], [100, 100], [100, 105], [200, 0], [205, 1], [300, 300], [303, 296], [306, 292]], dtype=float)
    for ms in (1, 2, 3):
        _check_dbscan(pts, 5., ms)
    grid = np.stack(np.meshgrid(np.arange(0, 60, 3), np.arange(0, 45, 3)), -1).reshape(-1, 2)
    for ms in (1, 3, 5, 6):
        _check_dbscan(grid, 3., ms)


def _near_eps_pairs(eps, count, seed):
    """points [2 count, 2] in pairs 1000 apart, and per pair whether dx*dx + dy*dy <= eps*eps: pairs about eps apart on which
    that squared test and sqrt(dx*dx + dy*dy) <= eps disagree, found by trying random directions"""
    rng = np.random.RandomState(seed)
    pts, squared = [], []
    while len(squared) < count:
        t = rng.rand() * 2 * np.pi
        a = rng.rand(2) * 10 + 1000. * len(squared)
        b = a + eps * np.array([np.cos(t), np.sin(t)])
        dx, dy = b[0] - a[0], b[1] - a[1]
        sq = dx * dx + dy * dy
        if (sq <= eps * eps) != (np.sqrt(sq) <= eps):
            pts += [a, b]
            squared.append(sq <= eps * eps)
    return np.array(pts), squared


def test_dbscan_pairs_a_rounding_from_eps_follow_the_kd_tree():
    """pairs on which the squared and the square-root distance tests disagree, 20 of them far apart (40 points, so scikit-learn
    searches a KD-tree): the device labels are scikit-learn's, and those follow the squared test"""
    eps = 0.7
    pts, squared = _near_eps_pairs(eps, 20, 3)
    labels = np.asarray(_check_dbscan(pts, eps, 2))
    for i, sq in enumerate(squared):
        assert (labels[2 * i] >= 0) == sq and (labels[2 * i + 1] >= 0) == sq


def test_dbscan_tiny_eps_over_wide_coordinates():
    """eps 1e-3 over coordinates up to 1e12 (about 1e15 cells of side eps): the grid coarsens and the labels stay scikit-learn's"""
    rng = np.random.RandomState(4)
    base = rng.rand(150, 2) * 1e12
    t = rng.rand(150) * 2 * np.pi
    step = np.where(np.arange(150) % 3 == 0, 2e-3, 5e-4)[:, None] * np.stack([np.cos(t), np.sin(t)], axis=1)
    pts = np.concatenate([base, base + step])
    labels = _check_dbscan(pts, 1e-3, 2)
    assert (np.asarray(labels) >= 0).any() and (np.asarray(labels) == -1).any()
    _check_dbscan(np.array([[-1e300, 0.], [1e300, 1.], [1e300, 1.5]] + [[i * 1e290, 0.] for i in range(12)]), 1., 2)


@pytest.mark.parametrize('n', [1, 2, 100000])
def test_dbscan_sizes(n):
    rng = np.random.RandomState(n)
    pts = rng.rand(n, 2) * np.sqrt(n) * 10
    _check_dbscan(pts, 5., 2)


# ---------------------------------------------------------------------------------------------------------------------------------
# the whole detection on the ovary fixtures
# ---------------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def ovary_images(oracle):
    with np.load(os.path.join(HERE, 'golden', 'center_detection_reference.npz')) as z:
        return [load(z, str(n)) for n in z['names']]


def _params(**kw):
    from pyimsegm_b200 import center_detection as cd
    p = dict(cd.CENTER_PARAMS)
    p.update(cd.CLUSTER_PARAMS)
    p.update(kw)
    return p


@pytest.mark.parametrize('params', [_params(), _params(fts_ray_types=[('up', [0]), ('down', [1])])], ids=['default', 'closer'])
def test_points_features_on_ovary_equal_the_host(ovary_images, params):
    from pyimsegm_b200 import center_detection as cd
    img, segm, _, _ = ovary_images[0]
    _, slic, points, got, names = cd.estim_points_compute_features('x', img / 255., segm, params)
    want, want_names = chr_.points_features(segm, points, params)
    assert names == want_names and np.array_equal(got, want)


def test_detect_center_candidates_on_ovary_equal_the_host(ovary_images):
    from sklearn.ensemble import RandomForestClassifier
    from pyimsegm_b200 import center_detection as cd
    params = _params()
    img, segm, levels, _ = ovary_images[0]
    _, _, points, feats, _ = cd.estim_points_compute_features('train', img / 255., segm, params)
    lut = np.array([0, 0, -1, 1])                  # run_center_candidate_training.LUT_ANNOT_CENTER_RELABEL
    labels = np.asarray(lut[np.asarray(cd.label_close_points(levels, points, params))])
    keep = labels >= 0
    classif = RandomForestClassifier(n_estimators=20, random_state=0).fit(feats[keep], labels[keep])
    for img, segm, _, _ in ovary_images:
        got = cd.detect_center_candidates_points(img / 255., segm, classif, params)
        want = chr_.detect_center_candidates_points(img / 255., segm, classif, params)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        assert np.array_equal(got[3], want[3]) and np.array_equal(np.asarray(got[4]), np.asarray(want[4]))
        assert got[2].any()
