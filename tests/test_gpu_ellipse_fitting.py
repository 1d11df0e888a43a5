"""GPU tests of imsegm.ellipse_fitting: every RANSAC trial against the host oracle (oracle/ellipse.py) from the same seed, the
single-model calls against the trial values bit for bit, and the doctests of the reference module through the device."""
import os
import sys

import numpy as np
import pytest

from oracle import ellipse as oe

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = [0.01, 0.95, 0.95, 0.85]


@pytest.fixture(scope='module')
def ef():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import ellipse_fitting
    return ellipse_fitting


def _eggs(seed=0):
    sys.path.insert(0, ROOT)
    import bench
    from scipy import ndimage
    img, annot, centres = bench.synth_eggs_image(seed, 320, 512)
    smooth = ndimage.gaussian_filter(img.mean(axis=-1), 2)
    seg = np.digitize(smooth, [0.36, 0.42, 0.5])      # 0 background, 3 egg core, 1-2 the rim
    seg = np.choose(seg, [0, 2, 3, 1])
    return seg, annot, centres


def _sensitivity(samples):
    """the fit's own sensitivity to the order of its sums: how far the oracle moves on the reversed samples"""
    m1, m2 = oe.EllipseModel(), oe.EllipseModel()
    if not (m1.estimate(samples) and m2.estimate(samples[::-1])):
        return 0.
    return float(np.max(np.abs(np.subtract(m1.params, m2.params))))


def _fit_tolerance(samples):
    """parameters agree to 1e-9 plus ten times that sensitivity (the uncentred direct fit is ill-conditioned)"""
    return 1e-9 + 10 * _sensitivity(samples)


def test_trials_against_oracle_and_single_model_calls(ef):
    seg, annot, centres = _eggs()
    slic, points_all, labels = ef.get_slic_points_labels(seg, slic_size=15, slic_regul=0.1)
    weights = np.bincount(slic.ravel())
    points = ef.prepare_boundary_points_ray_edge(seg, centres[:1], 5, sel_bg=3, sel_fg=2)[0]
    n_smp, thr, T = int(0.35 * len(points)), 25., 60
    np.random.seed(11)
    samples = [np.random.choice(len(points), n_smp, replace=False) for _ in range(T)]
    term = ef._label_terms(weights, labels, TABLE)
    run = lambda: ef._run_trials([points], [0] * T, samples=samples, crit_input=(points_all, labels, term), thr=thr,  # noqa: E731
                                 want_resid=True)
    ok, par, n_inl, crit, resid = run()
    again = run()
    assert all(np.array_equal(a, b) for a, b in zip((ok, par, n_inl, crit, resid), again)), 'two runs differ'
    near = solver = 0
    ratio = max_dp = 0.
    for t in range(T):
        smp = points[samples[t]]
        m = oe.EllipseModel()
        assert bool(m.estimate(smp)) == (ok[t] == 1)
        if ok[t] != 1:
            continue
        dp = float(np.max(np.abs(par[t] - m.params)))
        max_dp = max(max_dp, dp)
        ratio = max(ratio, dp / (1e-9 + _sensitivity(smp)))
        np.testing.assert_allclose(par[t], m.params, rtol=0, atol=_fit_tolerance(smp))
        # residuals and criterion of the same parameters
        m.params = list(par[t])
        r_o = m.residuals(points)
        r_d = resid[t * len(points):(t + 1) * len(points)]
        agree = np.abs(r_o - r_d) <= 1e-6
        solver += int(np.sum(~agree))
        border = np.abs(r_o - thr) <= 1e-6
        near += int(np.sum(border))
        keep = agree & ~border
        assert np.sum((r_d < thr)[keep]) == np.sum((r_o < thr)[keep])
        np.testing.assert_allclose(crit[t], m.criterion(points_all, weights, labels, TABLE), rtol=1e-12)
        # the single-model calls give the trial's bits
        model = ef.EllipseModelSegm()
        assert model.estimate(smp) and np.array_equal(model.params, par[t])
        assert np.array_equal(model.residuals(points), r_d)
        assert model.criterion(points_all, weights, labels, TABLE) == crit[t]
    print('\nresiduals within 1e-6 of the threshold: %d; points where Newton and leastsq reached different stationary points: %d'
          % (near, solver))
    print('parameters: max |device - oracle| %.3g; largest ratio to the oracle\'s own order sensitivity (+1e-9) %.3g' % (max_dp, ratio))
    assert solver <= max(2, T * len(points) // 1000)


def test_selection_against_oracle(ef):
    seg, _, centres = _eggs(1)
    slic, points_all, labels = ef.get_slic_points_labels(seg, slic_size=15, slic_regul=0.1)
    weights = np.bincount(slic.ravel())
    points = ef.prepare_boundary_points_ray_join(seg, centres[:1], 5, sel_bg=3, sel_fg=2)[0]
    np.random.seed(5)
    trials = oe.ransac_trials(points, points_all, weights, labels, TABLE, 0.35, 25, 40)
    best_o, inl_o, idx_o = oe.ransac_select(points, trials)
    np.random.seed(5)
    model, inl = ef.ransac_segm(points, ef.EllipseModelSegm, points_all, weights, labels, TABLE, 0.35, 25, 40)
    np.random.seed(5)
    samples = [np.random.choice(len(points), int(0.35 * len(points)), replace=False) for _ in range(40)]
    ok, _, n_inl, crit, _ = ef._run_trials([points], [0] * 40, samples=samples, crit_input=(points_all, labels,
                                           ef._label_terms(weights, labels, TABLE)), thr=25)
    idx_d, _ = ef._select(ok, n_inl, crit)
    assert idx_d == idx_o
    assert np.array_equal(inl, inl_o)
    np.testing.assert_allclose(model.params, best_o, rtol=0, atol=_fit_tolerance(points[inl_o]))


def _host_goldens():
    import importlib.util
    spec = importlib.util.spec_from_file_location('ellipse_host', os.path.join(ROOT, 'tests', 'test_ellipse_fitting_host.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_module_doctests_through_the_device(ef):
    g = _host_goldens()
    seg = ef.add_overlap_ellipse(np.zeros((15, 20), dtype=int), (7, 10, 5, 8, np.deg2rad(30)), 1)
    assert np.array_equal(seg, g._arr(g.ADD_OVERLAP_1))
    assert np.array_equal(ef.add_overlap_ellipse(seg, (4, 5, 2, 3, np.deg2rad(-30)), 2), g._arr(g.ADD_OVERLAP_2))
    seg = ef.add_overlap_ellipse(np.zeros((10, 20), dtype=int), (5, 10, 4, 6, np.deg2rad(30)), 1)
    seg_bg, seg_fc = ef.split_segm_background_foreground(seg, 1.5, 0)
    assert np.array_equal(seg_bg.astype(int), g._arr(g.SPLIT_BG))
    assert np.array_equal(seg_fc.astype(int), 1 - g._arr(g.SPLIT_BG))
    # imsegm/ellipse_fitting.py:373-379, :467-474, :518-525, :565-575
    assert np.round(ef.prepare_boundary_points_ray_join(seg, [(4, 9)], 5., 3, sel_bg=1, sel_fg=0)).tolist() == \
        [[[4.0, 16.0], [7.0, 10.0], [9.0, 5.0], [4.0, 16.0], [7.0, 10.0]]]
    edge = [[[4.0, 16.0], [7.0, 15.0], [9.0, 5.0], [4.0, 5.0], [1.0, 7.0], [0.0, 14.0]]]
    assert np.round(ef.prepare_boundary_points_ray_edge(seg, [(4, 9)], 2.5, 3, sel_bg=1, sel_fg=0)).tolist() == edge
    assert np.round(ef.prepare_boundary_points_ray_mean(seg, [(4, 9)], 2.5, 3, sel_bg=1, sel_fg=0)).tolist() == edge
    assert np.round(ef.prepare_boundary_points_ray_dist(seg, [(4, 9)], 2, sel_bg=0, sel_fg=0), 2).tolist() == \
        [[[4.0, 16.0], [6.8, 15.0], [9.0, 5.5], [4.35, 5.0], [1.0, 6.9], [1.0, 9.26], [0.0, 11.31], [0.5, 14.0], [1.45, 16.0]]]
    # EllipseModelSegm doctest (:51-73) and criterion doctest (:91-105)
    el = ef.EllipseModelSegm()
    assert el.estimate(g.perimeter_points()) and np.round(el.params, 2).tolist() == [19.5, 29.5, 12.45, 16.52, 0.53]
    params = 20, 30, 12, 16, np.deg2rad(30)
    xy = ef.EllipseModelSegm().predict_xy(np.linspace(0, 2 * np.pi, 25), params)
    el = ef.EllipseModelSegm()
    assert el.estimate(xy) and np.round(el.params, 2).tolist() == [20., 30., 12., 16., 0.52]
    assert np.all(np.round(np.abs(el.residuals(xy)), 5) == 0)
    el.params[2] += 2
    el.params[3] += 2
    assert np.all(np.round(np.abs(el.residuals(xy))) == 2)
    with pytest.raises(np.linalg.LinAlgError):
        ef.EllipseModelSegm().estimate(np.zeros((6, 2)))
    seg = np.zeros((10, 15), dtype=int)
    r, c = np.meshgrid(range(seg.shape[1]), range(seg.shape[0]))
    el.params = [4, 7, 3, 6, np.deg2rad(10)]
    pts, w = np.array([r.ravel(), c.ravel()]).T, np.ones(seg.size)
    for rows, cols, val in (((4, 5), (6, 8), '87.888'), ((2, 7), (4, 11), '17.577'), ((1, 9), (1, 14), '-70.311')):
        seg[rows[0]:rows[1], cols[0]:cols[1]] = 1
        assert str(el.criterion(pts, w, seg.ravel(), [[0.1, 0.9]])).startswith(val)


def test_ransac_doctest_and_seeds(ef):
    def doctest_run(seed, fn):
        seg = ef.add_overlap_ellipse(np.zeros((120, 150), dtype=int), (60, 75, 40, 65, np.deg2rad(30)), 1)
        slic, points_all, labels = ef.get_slic_points_labels(seg, slic_size=10, slic_regul=0.3)
        points = ef.prepare_boundary_points_ray_dist(seg, [(40, 90)], 2, sel_bg=1, sel_fg=0)[0]
        weights = np.bincount(slic.ravel())
        table = [[0.01, 0.75, 0.95, 0.9], [0.99, 0.25, 0.05, 0.1]]
        np.random.seed(seed)
        return fn(points, points_all, weights, labels, table)

    def device(points, points_all, weights, labels, table):
        model, _ = ef.ransac_segm(points, ef.EllipseModelSegm, points_all, weights, labels, table, 0.6, 3, max_trials=15)
        return model.params

    def oracle(points, points_all, weights, labels, table):
        return oe.ransac_select(points, oe.ransac_trials(points, points_all, weights, labels, table, 0.6, 3, 15))[0]

    def hit(params):
        return params is not None and np.round(params[:4]).astype(int).tolist() == [60, 75, 41, 65] and np.round(params[4], 1) == 0.5

    dev = [hit(doctest_run(s, device)) for s in range(20)]
    orc = [hit(doctest_run(s, oracle)) for s in range(20)]
    print('\nransac doctest reproduced by %d of 20 seeds on the device, %d in the oracle' % (sum(dev), sum(orc)))
    assert dev == orc
    assert dev[0]


def test_eggs_fitted_and_centres_equal_loop(ef):
    seg, annot, centres = _eggs(2)
    slic, points_all, labels = ef.get_slic_points_labels(seg, slic_size=15, slic_regul=0.1)
    weights = np.bincount(slic.ravel())
    pts = ef.prepare_boundary_points_ray_edge(seg, centres, 5, sel_bg=3, sel_fg=2)
    np.random.seed(0)
    loop = [ef.ransac_segm(p, ef.EllipseModelSegm, points_all, weights, labels, TABLE, 0.35, 25, 100) for p in pts]
    np.random.seed(0)
    batch = ef.ransac_segm_centres(pts, ef.EllipseModelSegm, points_all, weights, labels, TABLE, 0.35, 25, 100)
    for (m1, i1), (m2, i2), (cy, cx) in zip(loop, batch, centres):
        assert np.array_equal(m1.params, m2.params) and np.array_equal(i1, i2)
        assert np.hypot(m1.params[0] - cy, m1.params[1] - cx) < 6


def test_success_flags_on_near_degenerate_samples(ef):
    """near-circular and pixelated samples give numpy's success flag; on short noisy arcs the flag is decided by rounding, and
    numpy itself changes it when only the order of its sums changes -- the device may disagree no more often than that"""
    rng = np.random.RandomState(2)
    sets = {'near_circle': [], 'pixelated_circle': [], 'short_arc': []}
    for _ in range(300):
        xc, yc = rng.uniform(50, 500, 2)
        r = rng.uniform(5, 80)
        t = rng.uniform(0, 2 * np.pi, 20)
        sets['near_circle'].append(np.c_[xc + r * np.cos(t), yc + r * (1 + 1e-7) * np.sin(t)] + rng.normal(0, 1e-9, (20, 2)))
        t = rng.uniform(0, 2 * np.pi, 25)
        sets['pixelated_circle'].append(np.round(np.c_[xc + r * np.cos(t), yc + r * np.sin(t)]))
        t = rng.uniform(0, 0.3, 12)
        sets['short_arc'].append(np.c_[xc + r * np.cos(t), yc + 1.3 * r * np.sin(t)] + rng.normal(0, 0.5, (12, 2)))
    report = {}
    for name, pts in sets.items():
        ok = ef._run_trials(pts, np.arange(len(pts)), samples=[np.arange(len(p)) for p in pts])[0]
        ref = np.array([oe.EllipseModel().estimate(p) for p in pts])
        self_flip = sum(oe.EllipseModel().estimate(p) != oe.EllipseModel().estimate(p[::-1]) for p in pts)
        report[name] = (int(np.sum((ok == 1) != ref)), int(self_flip))
    print('\nflag mismatches device vs numpy (numpy vs numpy on reversed samples): %r' % report)
    assert report['near_circle'][0] == 0 and report['pixelated_circle'][0] == 0
    assert report['short_arc'][0] <= 1.3 * report['short_arc'][1] + 5


def test_overlap_with_many_and_negative_labels(ef):
    seg = np.arange(60 * 80).reshape(60, 80) + 1                 # 4 800 labels: global counters
    seg[:30] = -1
    mask_seg = ef.add_overlap_ellipse(np.zeros((60, 80), dtype=int), (40, 40, 5, 8, 0.3), 1)
    out = ef.add_overlap_ellipse(seg.copy(), (40, 40, 5, 8, 0.3), 9999, thr_overlap=1.)
    assert np.array_equal(out == 9999, mask_seg == 1)              # every label overlaps by at most 1 / its size <= 1
    out = ef.add_overlap_ellipse(seg.copy(), (40, 40, 5, 8, 0.3), 9999, thr_overlap=0.5)
    assert np.array_equal(out, seg)                                # a one-pixel label inside overlaps by 1 > 0.5
    neg = np.full((20, 20), -3)
    assert np.array_equal(ef.add_overlap_ellipse(neg.copy(), (10, 10, 3, 4, 0.), 2) == 2,
                          ef.add_overlap_ellipse(np.zeros((20, 20), dtype=int), (10, 10, 3, 4, 0.), 2) == 2)
