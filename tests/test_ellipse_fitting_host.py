"""CPU tests of the ellipse fitting: the host oracle (oracle/ellipse.py) against the doctest values of the reference's
imsegm/ellipse_fitting.py and imsegm/utilities/drawing.py, the host-side sampling and validation of the module, and the argument
checks of its C-ABI entries (no compute call)."""
import numpy as np
import pytest

from oracle import ellipse as oe

# imsegm/ellipse_fitting.py:296-310 and :313-327
ADD_OVERLAP_1 = ['00000000000000000000', '00000000000000000000', '00000000011111111000', '00000001111111111000',
                 '00000011111111111100', '00000111111111111100', '00001111111111111100', '00001111111111111000',
                 '00011111111111111000', '00011111111111110000', '00011111111111100000', '00001111111111000000',
                 '00001111111100000000', '00000000000000000000', '00000000000000000000']
ADD_OVERLAP_2 = ['00000000000000000000', '00000000000000000000', '00022200011111111000', '00022221111111111000',
                 '00022222111111111100', '00002222111111111100', '00001222111111111100', '00001111111111111000',
                 '00011111111111111000', '00011111111111110000', '00011111111111100000', '00001111111111000000',
                 '00001111111100000000', '00000000000000000000', '00000000000000000000']
# imsegm/utilities/drawing.py:167-184
DRAW_PERIMETER = ['00000000000000000000', '00000000000000111100', '00000000000111000010', '00000000011000000010',
                  '00000000100000000100', '00000011000000001000', '00000100000000010000', '00001000000000100000',
                  '00010000000011000000', '00100000000100000000', '01000000011000000000', '01000011100000000000',
                  '00111100000000000000', '00000000000000000000']
# imsegm/utilities/drawing.py:132-146
DRAW_ELLIPSE = ['00000000000000000000', '00000000000000000000', '00000000000000011100', '00000000000011111100',
                '00000000001111111100', '00000000111111111100', '00000001111111111000', '00000111111111110000',
                '00001111111111000000', '00011111111110000000', '00011111111000000000', '00011111100000000000',
                '00011100000000000000', '00000000000000000000']
# imsegm/ellipse_fitting.py:412-433 (seg_bg; seg_fc is its complement)
SPLIT_BG = ['11111111111111111111', '11111111110000011111', '11111111000000001111', '11111110000000001111',
            '11111100000000001111', '11111000000000001111', '11111000000000011111', '11111000000000111111',
            '11111000000001111111', '11111100000111111111']


def _arr(rows):
    return np.array([[int(c) for c in r] for r in rows])


def _add_overlap_oracle(segm, params, label, thr=1.):
    c1, c2, h, w, phi = params
    rr, cc = oe.draw_ellipse(int(c1), int(c2), int(h), int(w), segm.shape, phi)
    mask = np.zeros(segm.shape)
    mask[rr, cc] = 1
    for lb in range(1, int(np.max(segm) + 1)):
        sizes = [s for s in [np.sum(segm == lb), np.sum(mask == 1)] if s > 0]
        if not sizes or np.sum(np.logical_and(segm == lb, mask == 1)) / float(min(sizes)) > thr:
            return segm
    segm[mask == 1] = label
    return segm


def perimeter_points():
    """the pixels of the EllipseModelSegm doctest (imsegm/ellipse_fitting.py:51-54): drawing.ellipse_perimeter negates the angle"""
    rr, cc = oe.draw_ellipse_perimeter(20, 30, 12, 16, -np.deg2rad(30))
    return np.array([rr, cc]).T


def test_oracle_estimate_and_residuals_doctest():
    img = np.zeros((14, 20), dtype=int)
    rr, cc = oe.draw_ellipse_perimeter(7, 10, 3, 9, -np.deg2rad(30), img.shape)
    img[rr, cc] = 1
    assert np.array_equal(img, _arr(DRAW_PERIMETER))
    for canonical in (False, True):
        model = oe.EllipseModel()
        assert model.estimate(perimeter_points(), canonical=canonical)
        assert np.round(model.params, 2).tolist() == [19.5, 29.5, 12.45, 16.52, 0.53]
    params = 20, 30, 12, 16, np.deg2rad(30)
    model = oe.EllipseModel()
    xy = model.predict_xy(np.linspace(0, 2 * np.pi, 25), params)
    assert model.estimate(xy)
    assert np.round(model.params, 2).tolist() == [20., 30., 12., 16., 0.52]
    assert np.all(np.round(np.abs(model.residuals(xy)), 5) == 0)
    model.params[2] += 2
    model.params[3] += 2
    assert np.all(np.round(np.abs(model.residuals(xy))) == 2)


def test_oracle_canonical_sign_is_the_same_ellipse():
    rng = np.random.RandomState(3)
    swapped = 0
    for _ in range(40):
        pts = rng.uniform(0, 100, (12, 2))
        m_lapack, m_canon = oe.EllipseModel(), oe.EllipseModel()
        if not m_lapack.estimate(pts, canonical=False):
            continue
        assert m_canon.estimate(pts)
        p, q = np.array(m_lapack.params), np.array(m_canon.params)
        assert q[2] <= q[3]
        np.testing.assert_allclose(q[:2], p[:2], rtol=1e-12)
        if not np.allclose(p[2:4], q[2:4]):
            swapped += 1
            np.testing.assert_allclose(q[2:4], p[3:1:-1], rtol=1e-9)
            assert abs(abs(q[4] - p[4]) - np.pi / 2) < 1e-9
    assert swapped > 0


def test_oracle_criterion_doctest():
    seg = np.zeros((10, 15), dtype=int)
    r, c = np.meshgrid(range(seg.shape[1]), range(seg.shape[0]))
    el = oe.EllipseModel()
    el.params = [4, 7, 3, 6, np.deg2rad(10)]
    weights = np.ones(seg.ravel().shape)
    pts = np.array([r.ravel(), c.ravel()]).T
    seg[4:5, 6:8] = 1
    assert str(el.criterion(pts, weights, seg.ravel(), [[0.1, 0.9]])).startswith('87.888')
    seg[2:7, 4:11] = 1
    assert str(el.criterion(pts, weights, seg.ravel(), [[0.1, 0.9]])).startswith('17.577')
    seg[1:9, 1:14] = 1
    assert str(el.criterion(pts, weights, seg.ravel(), [[0.1, 0.9]])).startswith('-70.311')


def test_oracle_drawing_add_overlap_and_split_doctests():
    img = np.zeros((14, 20), dtype=int)
    rr, cc = oe.draw_ellipse(7, 10, 3, 9, img.shape, np.deg2rad(30))
    img[rr, cc] = 1
    assert np.array_equal(img, _arr(DRAW_ELLIPSE))
    seg = _add_overlap_oracle(np.zeros((15, 20), dtype=int), (7, 10, 5, 8, np.deg2rad(30)), 1)
    assert np.array_equal(seg, _arr(ADD_OVERLAP_1))
    seg = _add_overlap_oracle(seg, (4, 5, 2, 3, np.deg2rad(-30)), 2)
    assert np.array_equal(seg, _arr(ADD_OVERLAP_2))
    assert oe.disk(1.5).shape == (4, 4) and oe.disk(1.5).sum() == 4
    from scipy import ndimage
    seg = _add_overlap_oracle(np.zeros((10, 20), dtype=int), (5, 10, 4, 6, np.deg2rad(30)), 1)
    seg_bg = oe.opening(1 - ndimage.binary_fill_holes(seg > 0), oe.disk(1.5))
    assert np.array_equal(seg_bg, _arr(SPLIT_BG))
    assert np.array_equal(seg == 1, 1 - _arr(SPLIT_BG))


def test_ransac_and_criterion_validation():
    from pyimsegm_b200 import ellipse_fitting as ef
    pts = np.random.RandomState(0).uniform(0, 50, (40, 2))
    with pytest.raises(ValueError):
        ef._check_ransac_args(pts, 1.5, 10)
    with pytest.raises(ValueError):
        ef._check_ransac_args(pts, 41, 10)
    with pytest.raises(ValueError):
        ef._check_ransac_args(pts, 5, -1)
    assert ef._check_ransac_args(pts, 0.35, 10) == 14
    with pytest.raises(ValueError):
        ef._label_terms(np.ones(5), np.zeros(5, int), [[0.1, 0.9], [0.9, 0.1], [0.5, 0.5]])
    with pytest.raises(ValueError):
        ef._label_terms(np.ones(5), np.full(5, 3), [0.1, 0.9])
    np.testing.assert_allclose(ef._label_terms([2., 3.], [0, 1], [0.1, 0.9]),
                               [2 * (-np.log(0.1) + np.log(0.9)), 3 * (-np.log(0.9) + np.log(0.1))])
    with pytest.raises(ValueError):
        ef._label_terms(np.ones(3), [0, -1, 1], [0.1, 0.9])
    # fewer weights than classes fails only when a weightless label lies inside an ellipse, as weights[labels_in] does there
    term = ef._label_terms([2., 3.], [0, 1], [[0.1, 0.9, 0.5]])
    assert np.isnan(term[2]) and np.isfinite(term[:2]).all()
    ef._check_criteria([1, 0], [1.5, np.nan], term, 2)
    with pytest.raises(IndexError):
        ef._check_criteria([1, 0], [np.nan, 0.], term, 2)


def test_disk_offsets_of_an_even_footprint():
    from pyimsegm_b200 import descriptors as ds
    offs, even = ds._disk_offsets(1.5, False)
    assert even and sorted(map(tuple, offs.tolist())) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    offs, _ = ds._disk_offsets(1.5, True)
    assert sorted(map(tuple, offs.tolist())) == [(-1, -1), (-1, 0), (0, -1), (0, 0)]


def test_ellipse_entries_reject_bad_arguments():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    assert lib.isb_ellipse_ransac(0, None, None, None, None, 1, None, None, 1., None, None, None, 0, None, None, None, None, None, None,
                                  None) == _lib.ISB_ERR_ARG
    assert lib.isb_ellipse_ransac(4, None, None, None, None, 1, None, None, 1., None, None, None, 0, None, None, None, None, None, None,
                                  None) == _lib.ISB_ERR_ARG
    assert 'null' in lib.isb_last_error().decode()
    assert lib.isb_ellipse_overlap(None, 8, 8, 2, None, None, None, None, None) == _lib.ISB_ERR_ARG
    assert lib.isb_binary_morph_footprint(None, 8, 8, None, 4, 0, None, None) == _lib.ISB_ERR_ARG
    import ctypes as C
    buf = (C.c_double * 16)()
    p = C.cast(buf, C.c_void_p)
    assert lib.isb_binary_morph_footprint(p, 8, 8, p, 4, 2, C.cast((C.c_double * 16)(), C.c_void_p), None) == _lib.ISB_ERR_ARG
    assert 'op' in lib.isb_last_error().decode()
    assert lib.isb_abi_version() == 8


def test_ransac_draws_the_reference_sample_sequence(monkeypatch):
    """ransac_segm and ransac_segm_centres draw np.random.choice(len(points), min_samples, replace=False) once per trial, centre
    by centre, and nothing else from the global RNG"""
    from pyimsegm_b200 import ellipse_fitting as ef
    rng = np.random.RandomState(0)
    centres = [rng.uniform(0, 50, (n, 2)) for n in (40, 31, 17)]
    pts_all, labels = rng.uniform(0, 50, (20, 2)), rng.randint(0, 2, 20)
    weights = np.ones(20)
    recorded = []

    def fake_run(point_sets, trial_centre, samples=None, **kw):
        recorded.append([np.array(s) for s in samples])
        T = len(trial_centre)
        return np.zeros(T, np.int32), np.zeros((T, 5)), np.zeros(T, np.int32), np.zeros(T), np.zeros(1)

    monkeypatch.setattr(ef, '_run_trials', fake_run)
    np.random.seed(3)
    expected = [np.random.choice(len(p), int(0.35 * len(p)), replace=False) for p in centres for _ in range(7)]
    state = np.random.get_state()[1].copy()
    np.random.seed(3)
    res = ef.ransac_segm_centres(centres, ef.EllipseModelSegm, pts_all, weights, labels, [0.1, 0.9], 0.35, 1, 7)
    assert res == [(None, None)] * 3
    assert len(recorded[0]) == len(expected) and all(np.array_equal(a, b) for a, b in zip(recorded[0], expected))
    assert np.array_equal(np.random.get_state()[1], state)
    recorded.clear()
    np.random.seed(3)
    for p in centres:
        assert ef.ransac_segm(p, ef.EllipseModelSegm, pts_all, weights, labels, [0.1, 0.9], 0.35, 1, 7) == (None, None)
    assert all(np.array_equal(a, b) for a, b in zip([s for r in recorded for s in r], expected))
    assert np.array_equal(np.random.get_state()[1], state)


def test_selection_rule_matches_the_reference_loop():
    """strict < on the criterion (earliest trial wins a tie), the inlier mask replaced only inside that branch and only by a
    larger count, failed trials skipped (imsegm/ellipse_fitting.py:228-254)"""
    from pyimsegm_b200 import ellipse_fitting as ef
    rng = np.random.RandomState(1)
    n_pts = 30
    for _ in range(200):
        T = 12
        ok = (rng.rand(T) > 0.2).astype(np.int32)
        crit = rng.choice([-3., -2., -2., -1., 0.], T)          # ties on purpose
        n_inl = rng.randint(0, n_pts, T).astype(np.int32)
        masks = []
        for t in range(T):
            m = np.zeros(n_pts, bool)
            m[rng.choice(n_pts, n_inl[t], replace=False)] = True
            masks.append(m)
        trials = [(bool(ok[t]), [float(t)] * 5, masks[t], crit[t]) for t in range(T)]
        # the reference's loop without its refit (the refit is a fit, checked on the device)
        best, best_fit, best_inl, best_num = -1, np.inf, None, 0
        for t, (o, _, m, c) in enumerate(trials):
            if o and c < best_fit:
                best, best_fit = t, c
                if np.sum(m) > best_num:
                    best_inl, best_num = m, np.sum(m)
        idx, inl_trial = ef._select(ok, n_inl, crit)
        assert (idx if idx is not None else -1) == best
        assert (best_inl is None and inl_trial is None) or np.array_equal(masks[inl_trial], best_inl)
