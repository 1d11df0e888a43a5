"""CPU tests of imsegm.labeling: the oracle (oracle/labeling.py) against the doctests of the reference module, the fast host
restatements against the oracle's literal loops, the degenerate distance transform against scipy, and the argument checks of the
new C entry points (no launch)."""
import ctypes as C

import numpy as np
import pytest
from scipy import ndimage

from oracle import labeling as ol
from pyimsegm_b200 import labeling as lb

#: every public name of the reference's imsegm/labeling.py
REFERENCE_NAMES = [
    'neighbour_connect4', 'contour_binary_map', 'contour_coords', 'binary_image_from_coords', 'compute_distance_map',
    'segm_labels_assignment', 'histogram_regions_labels_counts', 'histogram_regions_labels_norm', 'assign_label_by_threshold',
    'assign_label_by_max', 'convert_segms_2_list', 'mask_segm_labels', 'sequence_labels_merge', 'relabel_by_dict',
    'merge_probab_labeling_2d', 'compute_labels_overlap_matrix', 'relabel_max_overlap_unique', 'relabel_max_overlap_merge',
    'compute_boundary_distances', 'assume_bg_on_boundary',
]


def test_every_reference_name_is_importable():
    import importlib
    mod = importlib.import_module('imsegm.labeling')
    for name in REFERENCE_NAMES:
        assert callable(getattr(mod, name)), name


def _atlases():
    a1 = np.zeros((7, 15), dtype=int)
    a1[1:4, 5:10] = 1
    a1[5:7, 3:13] = 2
    a2 = np.zeros((7, 15), dtype=int)
    a2[0:3, 7:12] = 1
    a2[3:7, 1:7] = 2
    a2[4:7, 7:14] = 3
    a2[:2, :3] = 5
    return a1, a2


def _rect():
    img = np.zeros((6, 6), dtype=int)
    img[1:5, 2:] = 1
    return img


def test_oracle_reproduces_reference_doctests():
    assert ol.neighbour_connect4(np.eye(5), 1, (2, 2)) is True
    assert ol.neighbour_connect4(np.ones((5, 5)), 1, (3, 3)) is False
    img = _rect()
    c0 = [[0] * 6, [0, 0, 1, 1, 1, 0], [0, 0, 1, 0, 0, 0], [0, 0, 1, 0, 0, 0], [0, 0, 1, 1, 1, 0], [0] * 6]
    c1 = [[0] * 6, [0, 0, 1, 1, 1, 1], [0, 0, 1, 0, 0, 1], [0, 0, 1, 0, 0, 1], [0, 0, 1, 1, 1, 1], [0] * 6]
    assert ol.contour_binary_map(img).tolist() == c0
    assert ol.contour_binary_map(img, include_boundary=True).tolist() == c1
    pts = [[1, 2], [1, 3], [1, 4], [2, 2], [3, 2], [4, 2], [4, 3], [4, 4]]
    assert ol.contour_coords(img) == pts
    assert ol.contour_coords(img, include_boundary=True) == pts + [[1, 5], [2, 5], [3, 5], [4, 5]]
    assert ol.binary_image_from_coords(ol.contour_coords(img), img.shape).tolist() == c0
    dist = np.round(ol.compute_distance_map(img), 2)
    assert dist.tolist() == [[2.24, 1.41, 1., 1., 1., 1.41], [2., 1., 0., 0., 0., 1.], [2., 1., 0., 1., 1., 1.41],
                             [2., 1., 0., 1., 1., 1.41], [2., 1., 0., 0., 0., 1.], [2.24, 1.41, 1., 1., 1., 1.41]]

    slic = np.array([[0] * 3 + [1] * 3 + [2] * 3 + [3] * 3] * 4 + [[4] * 3 + [5] * 3 + [6] * 3 + [7] * 3] * 4)
    segm = np.zeros(slic.shape, dtype=int)
    segm[4:, 6:] = 1
    hist = ol.segm_labels_assignment(slic, segm)
    assert {int(k): [int(x) for x in v] for k, v in hist.items()} == {k: [int(k >= 6)] * 12 for k in range(8)}

    slic = np.array([[0] * 4 + [1] * 3 + [2] * 3 + [3] * 3] * 4 + [[4] * 3 + [5] * 3 + [6] * 3 + [7] * 4] * 4)
    segm = np.zeros(slic.shape, dtype=int)
    segm[4:, 6:] = 1
    hist = ol.segm_labels_assignment(slic, segm)
    assert ol.assign_label_by_threshold(hist).tolist() == [0, 0, 0, 0, 0, 0, 1, 1]
    assert ol.assign_label_by_max(hist).tolist() == [0, 0, 0, 0, 0, 0, 1, 1]

    seg = np.ones((2, 3), dtype=int)
    assert ol.convert_segms_2_list([seg, seg * 0, seg * 2]) == [1] * 6 + [0] * 6 + [2] * 6

    img = np.zeros((4, 6))
    img[:-1, 1:] = 1
    img[1:2, 2:4] = 2
    m = ol.mask_segm_labels(img, [1])
    assert m.tolist() == [[False] + [True] * 5, [False, True, False, False, True, True], [False] + [True] * 5, [False] * 6]
    assert ol.mask_segm_labels(img, [2], np.full(img.shape, True, dtype=bool)).all()

    colors = {0: [], 1: [], 2: []}
    assert ol.sequence_labels_merge(np.zeros((8, 1, 1)), colors, [0]).tolist() == [[-1]]
    assert ol.sequence_labels_merge(np.ones((8, 1, 1)), colors, [0]).tolist() == [[1]]
    assert ol.sequence_labels_merge(np.array([[1], [1], [2], [1], [1], [1], [2], [1]]), colors, [0]).tolist() == [-1]
    assert ol.sequence_labels_merge(np.array([[1], [0], [1], [1], [1], [1], [0], [0]]), colors, [0]).tolist() == [1]

    labels = np.array([2, 1, 0, 3, 3, 0, 2, 3, 0, 0])
    assert ol.relabel_by_dict(labels, {0: [1, 2], 1: [0, 3]}).tolist() == [0, 0, 1, 1, 1, 1, 0, 1, 1, 1]

    p = np.ones((5, 5))
    proba = np.rollaxis(np.array([p * 0.3, p * 0.4, p * 0.2]), 0, 3)
    new = ol.merge_probab_labeling_2d(proba, {0: [1, 2], 1: [0]})
    assert new.shape == (5, 5, 2) and np.allclose(new[0, 0], [0.6, 0.3])

    seg1 = np.zeros((7, 15), dtype=int)
    seg1[1:4, 5:10] = 3
    seg1[5:7, 6:13] = 2
    seg2 = np.zeros((7, 15), dtype=int)
    seg2[2:5, 7:12] = 1
    seg2[4:7, 7:14] = 3
    assert ol.compute_labels_overlap_matrix(seg1, seg1).tolist() == [[76, 0, 0, 0], [0, 0, 0, 0], [0, 0, 14, 0], [0, 0, 0, 15]]
    assert ol.compute_labels_overlap_matrix(seg1, seg2).tolist() == [[63, 4, 0, 9], [0, 0, 0, 0], [2, 0, 0, 12], [9, 6, 0, 0]]

    for args, want in _relabel_doctests():
        assert ol.__dict__[args[0]](*args[1:]).tolist() == want

    segm_ref = np.zeros((6, 10), dtype=int)
    segm_ref[3:4, 4:5] = 1
    segm = np.zeros((6, 10), dtype=int)
    segm[:, 2:9] = 1
    pts, dist = ol.compute_boundary_distances(segm_ref, segm)
    assert pts.tolist() == [[2, 4], [3, 3], [3, 4], [3, 5], [4, 4]]
    assert dist.tolist() == [2.0, 1.0, 2.0, 3.0, 2.0]

    for segm, want in _bg_doctests():
        assert ol.assume_bg_on_boundary(segm, boundary_size=1).tolist() == want


def _relabel_doctests():
    """(oracle function name and arguments, expected map) of labeling.py:545-577 and :637-660"""
    a1, a2 = _atlases()
    u1 = [[5, 5, 5, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0], [5, 5, 5, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0],
          [0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0], [0, 3, 3, 3, 3, 3, 3, 0, 0, 0, 0, 0, 0, 0, 0]] + \
         [[0, 3, 3, 3, 3, 3, 3, 2, 2, 2, 2, 2, 2, 2, 0]] * 3
    u2 = [[0] * 15] + [[0] * 5 + [1] * 5 + [0] * 5] * 3 + [[0] * 15] + [[0] * 3 + [3] * 10 + [0] * 2] * 2
    u3 = [list(r) for r in u1]
    u3[0][0] = -1
    a2n = a2.copy()
    a2n[0, 0] = -1
    m1 = [[1, 1, 1, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0]] * 2 + [[0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0],
                                                                   [0, 2, 2, 2, 2, 2, 2, 0, 0, 0, 0, 0, 0, 0, 0]] + \
         [[0] + [2] * 13 + [0]] * 3
    m2 = [[0] * 15] + [[0] * 5 + [1] * 5 + [0] * 5] * 3 + [[0] * 15] + [[0] * 3 + [2] * 10 + [0] * 2] * 2
    m3 = [[0] * 15] * 4 + [[0] * 7 + [2] * 7 + [0]] * 3
    return [(('relabel_max_overlap_unique', a1, a2, True), u1), (('relabel_max_overlap_unique', a2, a1, True), u2),
            (('relabel_max_overlap_unique', a1, a2, False), u1), (('relabel_max_overlap_unique', a1, a2n, True), u3),
            (('relabel_max_overlap_merge', a1, a2, True), m1), (('relabel_max_overlap_merge', a2, a1, True), m2),
            (('relabel_max_overlap_merge', a1, a2, False), m3)]


def _bg_doctests():
    """labeling.py:727-743"""
    segm = np.zeros((6, 12), dtype=int)
    segm[1:4, 4:] = 2
    want = [[0] * 12] + [[0] * 4 + [2] * 8] * 3 + [[0] * 12] * 2
    other = segm.copy()
    other[other == 0] = 1
    return [(segm, want), (other, want)]


def _random_pair(rng):
    """a small random (seg_ref, seg_relabel) with label gaps, either side larger, and sometimes negative labels"""
    h, w = rng.randint(1, 9), rng.randint(1, 9)
    n_ref, n_rel = rng.randint(1, 9), rng.randint(1, 9)
    ref = rng.choice(rng.choice(12, n_ref, replace=False), (h, w))
    rel = rng.choice(rng.choice(12, n_rel, replace=False), (h, w))
    if rng.rand() < 0.3:
        rel[rng.rand(h, w) < 0.2] = -rng.randint(1, 3)
    if rng.rand() < 0.3:
        ref[rng.rand(h, w) < 0.2] = -1
    return ref, rel


def test_fast_unique_lut_equals_the_literal_loops():
    rng = np.random.RandomState(7)
    kinds = set()
    for _ in range(400):
        ref, rel = _random_pair(rng)
        if ref.max() < 0 or rel.max() < 0:
            continue
        kinds.add((ref.max() > rel.max(), ref.max() < rel.max(), bool((rel < 0).any())))
        overlap = ol.compute_labels_overlap_matrix(ref, rel)
        for keep_bg in (False, True):
            want = ol.max_overlap_unique_lut(overlap, rel.max() + 1, keep_bg)
            assert lb.max_overlap_unique_lut(overlap, rel.max() + 1, keep_bg) == [int(v) for v in want]
    assert len(kinds) >= 5


def test_host_functions_against_oracle():
    rng = np.random.RandomState(3)
    for _ in range(50):
        segm = rng.randint(0, 6, (rng.randint(1, 12), rng.randint(1, 12)))
        gt = rng.randint(0, 4, segm.shape)
        want, got = ol.segm_labels_assignment(segm, gt), lb.segm_labels_assignment(segm, gt)
        assert list(want) == list(got)
        assert all([int(x) for x in want[k]] == [int(x) for x in got[k]] for k in want)
        for th in (0.3, 0.5, 0.75):
            assert lb.assign_label_by_threshold(got, th).tolist() == ol.assign_label_by_threshold(want, th).tolist()
        assert lb.assign_label_by_max(got).tolist() == ol.assign_label_by_max(want).tolist()
        assert lb.convert_segms_2_list([segm, gt]) == ol.convert_segms_2_list([segm, gt])
        assert lb.mask_segm_labels(segm, [1, 3]).tolist() == ol.mask_segm_labels(segm, [1, 3]).tolist()
        init = rng.rand(*segm.shape) < 0.2
        assert lb.mask_segm_labels(segm, [2], init).tolist() == ol.mask_segm_labels(segm, [2], init).tolist()
        d = {0: [1, 2], 3: [0, 5, 2], 1: [4]}
        assert lb.relabel_by_dict(segm, d).tolist() == ol.relabel_by_dict(segm, d).tolist()
        stack = rng.choice([0, 1, 2, -1], (6,) + segm.shape, p=[0.4, 0.5, 0.05, 0.05])
        colors = {0: [], 1: [], 2: []}
        assert lb.sequence_labels_merge(stack, colors, [0]).tolist() == ol.sequence_labels_merge(stack, colors, [0]).tolist()
        pts = rng.randint(-2, 14, (20, 2)).tolist()
        assert lb.binary_image_from_coords(pts, segm.shape).tolist() == ol.binary_image_from_coords(pts, segm.shape).tolist()
        pad = np.pad(segm, 1)
        r, c = rng.randint(1, pad.shape[0] - 1), rng.randint(1, pad.shape[1] - 1)
        assert lb.neighbour_connect4(pad, 1, (r, c)) == ol.neighbour_connect4(pad, 1, (r, c))
    proba = rng.rand(4, 5, 3)
    d = {0: [1, 2], 2: [0]}
    assert np.array_equal(lb.merge_probab_labeling_2d(proba, d), ol.merge_probab_labeling_2d(proba, d))
    with pytest.raises(ValueError):
        lb.relabel_by_dict(np.zeros(3), {})
    with pytest.raises(ValueError):
        lb.sequence_labels_merge(np.full((2, 1, 1), 7), {0: [], 1: []}, [0])
    with pytest.raises(ValueError):
        lb.merge_probab_labeling_2d(np.zeros((2, 2)), {0: [0]})


def test_neighbour_connect4_stops_at_the_first_differing_neighbour():
    # on the last row / column: the neighbour above or on the left differs before the one past the border is read
    for seg, pos in [([[1, 0], [0, 1]], (1, 1)), ([[0, 0], [1, 1]], (1, 0)), ([[1, 1], [0, 1]], (1, 1))]:
        seg = np.array(seg)
        assert ol.neighbour_connect4(seg, 1, pos) is True
        assert lb.neighbour_connect4(seg, 1, pos) is True
    with pytest.raises(IndexError):
        ol.neighbour_connect4(np.ones((2, 2)), 1, (1, 1))
    with pytest.raises(IndexError):
        lb.neighbour_connect4(np.ones((2, 2)), 1, (1, 1))


def test_degenerate_edt_matches_scipy():
    for shape in [(1, 1), (1, 7), (7, 1), (2, 2), (5, 9), (33, 17)]:
        assert np.array_equal(ndimage.distance_transform_edt(np.ones(shape)), ol.edt_without_sites(shape))


def test_labeling_entry_points_reject_bad_arguments():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    assert lib.isb_abi_version() == 8
    assert lib.isb_label_boundary_map(None, 4, 4, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_label_contour_map(p, 0, 4, 1, 0, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_edt_workspace_bytes(0, 4) == 0
    ws = lib.isb_edt_workspace_bytes(40000, 4)
    assert lib.isb_edt_2d(p, 40000, 4, p, p, ws, None) == _lib.ISB_ERR_ARG and b'32768' in lib.isb_last_error()
    assert lib.isb_edt_2d(p, 8, 8, p, p, lib.isb_edt_workspace_bytes(8, 8) - 1, None) == _lib.ISB_ERR_ARG
    assert lib.isb_mask_compact_count(p, 8, 8, p, 0, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_mask_compact_write(p, 8, 8, p, p, lib.isb_mask_compact_workspace_bytes(8, 8), p, None, None) == _lib.ISB_ERR_ARG
    assert lib.isb_relabel_gather(p, 0, p, 4, p, None) == _lib.ISB_ERR_ARG
