"""GPU tests of imsegm.labeling: the doctests of the reference module through the device, and bit equality with the host oracle
(oracle/labeling.py, scipy's distance_transform_edt) for boundary maps, contour maps, the distance transform, boundary points and
distances, overlap matrices and relabelled maps -- on odd and degenerate shapes, negative labels, Voronoi maps, a SLIC output and one
8192 x 8192 pair."""
import numpy as np
import pytest
from scipy import ndimage
from scipy.spatial import cKDTree

from conftest import synth_regions
from oracle import labeling as ol
from test_labeling_host import _bg_doctests, _rect, _relabel_doctests

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lb():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import labeling
    return labeling


def _contour_np(seg, label=1, include_boundary=False):
    """contour_binary_map without its Python loops (checked against the oracle's loops on the small maps below)"""
    on = seg == label
    out = np.zeros(seg.shape, dtype=bool)
    if seg.shape[0] > 2 and seg.shape[1] > 2:
        c = on[1:-1, 1:-1]
        nb = (seg[:-2, 1:-1] != label) | (seg[2:, 1:-1] != label) | (seg[1:-1, :-2] != label) | (seg[1:-1, 2:] != label)
        out[1:-1, 1:-1] = c & nb
    if include_boundary:
        for sl in ((slice(None), 0), (slice(None), -1), (0, slice(None)), (-1, slice(None))):
            out[sl] |= on[sl]
    return out.astype(np.int64)


def _overlap_np(a, b):
    keep = (a >= 0) & (b >= 0)
    shape = (int(a.max()) + 1, int(b.max()) + 1)
    return np.bincount(a[keep].astype(np.int64) * shape[1] + b[keep], minlength=shape[0] * shape[1]).reshape(shape)


def _voronoi(h, w, n, seed):
    rng = np.random.RandomState(seed)
    pts = rng.rand(n, 2) * [h, w]
    _, idx = cKDTree(pts).query(np.indices((h, w)).reshape(2, -1).T)
    return idx.reshape(h, w).astype(np.int64)


def _small_maps():
    rng = np.random.RandomState(5)
    maps = [np.zeros((1, 9), int), np.zeros((9, 1), int), np.zeros((2, 2), int), np.full((5, 7), 3)]
    for shape in [(1, 9), (9, 1), (2, 2), (3, 3), (5, 7), (17, 33), (31, 1), (64, 65)]:
        maps.append(rng.randint(0, 3, shape))
        maps.append(rng.randint(-2, 2, shape))                 # negative labels are ordinary values
        m = np.zeros(shape, int)
        m[shape[0] // 3:, shape[1] // 2:] = 1
        maps.append(m)
    return maps


def _check_maps(lb, seg, ref, small):
    eng = lb.get_engine()
    bnd = ol.find_boundaries_thick(seg)
    assert np.array_equal(eng.to_host(lb._boundary_mask(eng, seg, 't_bnd')).astype(bool), bnd)
    for label in (1, int(seg.flat[0])):
        for inc in (False, True):
            want = ol.contour_binary_map(seg, label, inc) if small else _contour_np(seg, label, inc)
            if small:
                assert np.array_equal(want, _contour_np(seg, label, inc))
            got = lb.contour_binary_map(seg, label, inc)
            assert got.dtype == np.int64 and np.array_equal(got, want)
            want_pts = ol.contour_coords(seg, label, inc) if small else None
            if small:
                assert lb.contour_coords(seg, label, inc) == want_pts
        dmap = lb.compute_distance_map(seg, label)
        want = ndimage.distance_transform_edt(1 - (ol.contour_binary_map(seg, label) if small else _contour_np(seg, label)))
        assert dmap.dtype == np.float64 and np.array_equal(dmap, want)
    pts, dist = lb.compute_boundary_distances(ref, seg)
    want_pts, want_dist = ol.compute_boundary_distances(ref, seg)
    assert pts.dtype == np.int64 and dist.dtype == np.float64
    assert pts.shape == (len(want_dist), 2) and np.array_equal(pts, want_pts.reshape(-1, 2)) and np.array_equal(dist, want_dist)


def test_reference_doctests_through_device(lb):
    img = _rect()
    assert lb.contour_binary_map(img).tolist() == ol.contour_binary_map(img).tolist()
    assert lb.contour_binary_map(img, include_boundary=True).tolist() == ol.contour_binary_map(img, include_boundary=True).tolist()
    assert lb.contour_coords(img) == [[1, 2], [1, 3], [1, 4], [2, 2], [3, 2], [4, 2], [4, 3], [4, 4]]
    assert lb.contour_coords(img, include_boundary=True)[8:] == [[1, 5], [2, 5], [3, 5], [4, 5]]
    assert np.round(lb.compute_distance_map(img), 2).tolist() == np.round(ol.compute_distance_map(img), 2).tolist()
    assert np.array_equal(lb.compute_distance_map(img), ol.compute_distance_map(img))
    seg1 = np.zeros((7, 15), dtype=int)
    seg1[1:4, 5:10] = 3
    seg1[5:7, 6:13] = 2
    seg2 = np.zeros((7, 15), dtype=int)
    seg2[2:5, 7:12] = 1
    seg2[4:7, 7:14] = 3
    assert lb.compute_labels_overlap_matrix(seg1, seg1).tolist() == [[76, 0, 0, 0], [0, 0, 0, 0], [0, 0, 14, 0], [0, 0, 0, 15]]
    assert lb.compute_labels_overlap_matrix(seg1, seg2).tolist() == [[63, 4, 0, 9], [0, 0, 0, 0], [2, 0, 0, 12], [9, 6, 0, 0]]
    for args, want in _relabel_doctests():
        got = getattr(lb, args[0])(*args[1:])
        assert got.dtype == np.int64 and got.tolist() == want, args[0]
    for segm, want in _bg_doctests():
        assert lb.assume_bg_on_boundary(segm, boundary_size=1).tolist() == want
    segm_ref = np.zeros((6, 10), dtype=int)
    segm_ref[3:4, 4:5] = 1
    segm = np.zeros((6, 10), dtype=int)
    segm[:, 2:9] = 1
    pts, dist = lb.compute_boundary_distances(segm_ref, segm)
    assert pts.tolist() == [[2, 4], [3, 3], [3, 4], [3, 5], [4, 4]] and dist.tolist() == [2.0, 1.0, 2.0, 3.0, 2.0]
    slic = np.array([[0] * 3 + [1] * 3 + [2] * 3] * 4 + [[4] * 3 + [5] * 3 + [6] * 3] * 4)
    segm = np.zeros(slic.shape, dtype=int)
    segm[4:, 5:] = 2
    assert lb.histogram_regions_labels_counts(slic, segm)[5].tolist() == [8., 0., 4.]


def test_small_odd_degenerate_and_negative_maps(lb):
    maps = _small_maps()
    for i, seg in enumerate(maps):
        _check_maps(lb, seg, maps[(i + 3) % len(maps)] if maps[(i + 3) % len(maps)].shape == seg.shape else seg[::-1, ::-1].copy(), True)


def test_single_label_gives_the_degenerate_transform(lb):
    seg = np.full((37, 53), 4)
    want = ol.edt_without_sites(seg.shape)
    assert np.array_equal(lb.compute_distance_map(seg, 4), want)
    ref = np.zeros_like(seg)
    ref[10:20, 5:9] = 1
    pts, dist = lb.compute_boundary_distances(ref, seg)
    assert np.array_equal(dist, want[tuple(pts.T)])
    pts, dist = lb.compute_boundary_distances(seg, ref)
    assert pts.shape == (0, 2) and pts.dtype == np.int64 and dist.shape == (0, ) and dist.dtype == np.float64


def test_tall_maps_and_labels_outside_int32(lb):
    rng = np.random.RandomState(9)
    tall = rng.randint(0, 2, (70000, 3))
    assert np.array_equal(lb.contour_binary_map(tall, 1, True), _contour_np(tall, 1, True))
    assert np.array_equal(lb.contour_binary_map(tall.T.copy(), 1), _contour_np(tall.T, 1))
    big = np.array([[5, 1, 1], [2 ** 40, 1, 1], [1, 1, 5], [5, 5, 5]], dtype=np.int64)
    for label in (1, 5, 2 ** 40):
        assert np.array_equal(lb.contour_binary_map(big, label, True), ol.contour_binary_map(big, label, True))
        assert lb.contour_coords(big, label, True) == ol.contour_coords(big, label, True)
        assert np.array_equal(lb.compute_distance_map(big, label), ol.compute_distance_map(big, label))


def test_edt_on_random_sites(lb):
    eng = lb.get_engine()
    rng = np.random.RandomState(1)
    for shape, p in [((1, 1), 0.5), ((1, 300), 0.01), ((300, 1), 0.01), ((97, 211), 0.001), ((257, 129), 0.3), ((1031, 2053), 1e-5),
                     ((64, 4096), 2e-4)]:
        sites = rng.rand(*shape) < p
        d_sites = eng.to_device(sites.astype(np.uint8), 't_sites')
        got = eng.to_host(lb._edt(eng, d_sites, shape)).copy()
        want = ndimage.distance_transform_edt(~sites) if sites.any() else ol.edt_without_sites(shape)
        assert np.array_equal(got, want), shape


def test_voronoi_maps(lb):
    seg, ref = _voronoi(1031, 2053, 300, 0), _voronoi(1031, 2053, 200, 1)
    _check_maps(lb, seg, ref, False)
    assert np.array_equal(lb.compute_labels_overlap_matrix(ref, seg), _overlap_np(ref, seg))
    for keep_bg in (False, True):
        lut = ol.max_overlap_unique_lut(_overlap_np(ref, seg), seg.max() + 1, keep_bg)
        assert np.array_equal(lb.relabel_max_overlap_unique(ref, seg, keep_bg), np.array(lut)[seg])


def test_slic_against_annotation(lb):
    from pyimsegm_b200 import superpixels
    img, annot = synth_regions(2048, 2048)
    slic = superpixels.segment_slic_img2d(img, 30, 0.2)
    _check_maps(lb, slic, annot, False)
    assert np.array_equal(lb.compute_labels_overlap_matrix(slic, annot), _overlap_np(slic, annot))
    for keep_bg in (False, True):
        got = lb.relabel_max_overlap_unique(annot, slic, keep_bg)
        lut = ol.max_overlap_unique_lut(_overlap_np(annot, slic), slic.max() + 1, keep_bg)
        assert np.array_equal(got, np.array(lut)[slic])


def test_overlap_and_relabel_against_oracle(lb):
    rng = np.random.RandomState(4)
    for _ in range(40):
        shape = (rng.randint(1, 20), rng.randint(1, 20))
        ref = rng.choice(rng.choice(9, rng.randint(1, 6), replace=False), shape)
        rel = rng.choice(rng.choice(9, rng.randint(1, 6), replace=False), shape)
        if rng.rand() < 0.5:
            rel[rng.rand(*shape) < 0.2] = -1
        if rng.rand() < 0.5:
            ref[rng.rand(*shape) < 0.2] = -2
        if ref.max() < 0 or rel.max() < 0:
            continue
        assert np.array_equal(lb.compute_labels_overlap_matrix(ref, rel), ol.compute_labels_overlap_matrix(ref, rel))
        for keep_bg in (False, True):
            assert np.array_equal(lb.relabel_max_overlap_unique(ref, rel, keep_bg), ol.relabel_max_overlap_unique(ref, rel, keep_bg))
            try:
                want = ol.relabel_max_overlap_merge(ref, rel, keep_bg)
            except (IndexError, ValueError) as err:       # a label past the table, numpy's argmax of an empty slice
                with pytest.raises(type(err)):
                    lb.relabel_max_overlap_merge(ref, rel, keep_bg)
                continue
            assert np.array_equal(lb.relabel_max_overlap_merge(ref, rel, keep_bg), want)
    vol = rng.randint(-1, 4, (3, 5, 6))
    assert np.array_equal(lb.compute_labels_overlap_matrix(vol, vol[::-1]), ol.compute_labels_overlap_matrix(vol, vol[::-1]))
    neg = np.full((4, 4), -1)
    assert lb.compute_labels_overlap_matrix(neg, np.ones((4, 4), int)).shape == (0, 2)
    assert lb.compute_labels_overlap_matrix(np.ones((4, 4), int), neg).shape == (2, 0)


def test_large_map_int32_indexing(lb):
    seg = np.kron(_voronoi(128, 128, 60, 2), np.ones((64, 64), dtype=np.int64))
    ref = np.kron(_voronoi(256, 256, 90, 3), np.ones((32, 32), dtype=np.int64))
    pts, dist = lb.compute_boundary_distances(ref, seg)
    want_pts, want_dist = ol.compute_boundary_distances(ref, seg)
    assert len(dist) > 0 and np.array_equal(pts, want_pts) and np.array_equal(dist, want_dist)
    got = lb.relabel_max_overlap_unique(ref, seg, True)
    lut = ol.max_overlap_unique_lut(_overlap_np(ref, seg), seg.max() + 1, True)
    assert np.array_equal(got, np.array(lut)[seg])


def test_argument_errors_raise_before_any_launch(lb):
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.utilities import ImageDimensionError
    before = _lib.lib().isb_launch_count()
    a, b = np.zeros((4, 5), int), np.zeros((5, 4), int)
    for fn in (lb.compute_labels_overlap_matrix, lb.relabel_max_overlap_unique, lb.relabel_max_overlap_merge, lb.compute_boundary_distances,
               lb.segm_labels_assignment):
        with pytest.raises(ImageDimensionError):
            fn(a, b)
    with pytest.raises(ValueError):
        lb.compute_labels_overlap_matrix(np.full((2, 2), -3), np.zeros((2, 2), int))       # np.zeros with a negative dimension
    with pytest.raises(ValueError):
        lb.histogram_regions_labels_counts(np.zeros((2, 2), int), np.full((2, 2), -1))
    neg_inside = np.zeros((5, 5), int)
    neg_inside[2, 2] = -1
    with pytest.raises(ValueError):
        lb.assume_bg_on_boundary(neg_inside)
    with pytest.raises(ValueError):
        lb.compute_distance_map(np.zeros((32769, 1), np.uint8))
    with pytest.raises(ValueError):
        lb.compute_boundary_distances(np.zeros((1, 32769), np.uint8), np.zeros((1, 32769), np.uint8))
    assert _lib.lib().isb_launch_count() == before
