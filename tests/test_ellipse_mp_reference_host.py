"""CPU tests of the extended-precision ellipse references (tests/ellipse_mp_reference.py): closed forms, exact recovery of sampled
ellipses, and agreement with the float64 oracle (oracle/ellipse.py) where its fit is well conditioned, so that the GPU tests can rely
on them."""
import numpy as np
import pytest

from oracle import ellipse as oe
import ellipse_mp_reference as mr


def test_circle_distances_closed_form():
    rng = np.random.RandomState(0)
    for xc, yc, r, th in ((0., 0., 1., 0.), (10.5, -3.25, 7., 0.3), (500., 8000., 40., 2.)):
        params = (xc, yc, r, r, th)
        pts = np.r_[rng.uniform(-3 * r, 3 * r, (12, 2)) + [xc, yc], [[xc + r, yc], [xc, yc + 0.5 * r]]]
        for p in pts:
            d = mr.mp_stationary_distances(params, p)
            assert abs(d[0] - abs(np.hypot(p[0] - xc, p[1] - yc) - r)) <= 1e-12 * (1 + r)
            assert abs(d[-1] - (np.hypot(p[0] - xc, p[1] - yc) + r)) <= 1e-12 * (1 + r)
        # the centre: every angle is stationary at distance r
        assert mr.mp_stationary_distances(params, (xc, yc)) == pytest.approx([r], rel=1e-15)


def test_degenerate_ellipse_distances():
    """a = 0 or b = 0 is a segment, a = b = 0 a point"""
    assert mr.mp_stationary_distances((0., 0., 0., 0., 0.3), (3., 4.)) == pytest.approx([5.], rel=1e-15)
    d = mr.mp_stationary_distances((0., 0., 0., 5., 0.), (3., 4.))      # the segment x = 0, |y| <= 5
    assert d[0] == pytest.approx(3., rel=1e-15)
    d = mr.mp_stationary_distances((0., 0., 5., 0., 0.), (7., 1.))      # the segment y = 0, |x| <= 5
    assert d[0] == pytest.approx(np.hypot(2., 1.), rel=1e-15)


def test_axis_ellipse_distances_on_axes():
    """points on the axes of an axis-aligned ellipse: the stationary distances are the axis crossings, and inside the evolute
    also the two oblique normals"""
    a, b = 10., 30.
    params = (0., 0., a, b, 0.)
    assert mr.mp_stationary_distances(params, (15., 0.))[0] == pytest.approx(5., rel=1e-15)
    assert mr.mp_stationary_distances(params, (0., 45.))[0] == pytest.approx(15., rel=1e-15)
    d = mr.mp_stationary_distances(params, (0., 0.))
    assert d[0] == pytest.approx(a, rel=1e-15) and d[-1] == pytest.approx(b, rel=1e-15)


def test_fit_recovers_sampled_ellipses():
    """ellipses sampled by predict_xy give their parameters back (shorter semi-axis first, theta modulo pi)"""
    m = oe.EllipseModel()
    for params in ((0., 0., 10., 20., 0.), (3., -7., 5., 50., 0.), (250., 120., 30., 31., 1.1), (8000., 8000., 60., 90., 0.4),
                   (-40., 15., 1., 1000., 2.5)):
        t = np.linspace(0, 2 * np.pi, 37)[:-1]
        pts = m.predict_xy(t, params)
        r = mr.mp_fit(pts)
        assert r['status'] == 1 and r['n_admissible'] == 1
        p = np.array(r['params'])
        scale = max(abs(params[0]), abs(params[1]), params[3])
        np.testing.assert_allclose(p[:4], params[:4], rtol=0, atol=1e-10 * scale)
        dth = (p[4] - params[4] + np.pi / 2) % np.pi - np.pi / 2
        assert abs(dth) * (params[3] - params[2]) <= 1e-10 * scale


def test_fit_agrees_with_float64_oracle_when_well_conditioned():
    rng = np.random.RandomState(1)
    for _ in range(20):
        a, b = sorted(rng.uniform(5, 40, 2))
        params = (rng.uniform(-2, 2), rng.uniform(-2, 2), a, b * 1.5, rng.uniform(0, np.pi))
        t = rng.uniform(0, 2 * np.pi, 30)
        pts = oe.EllipseModel().predict_xy(t, params) + rng.normal(0, 0.3, (30, 2))
        r = mr.mp_fit(pts)
        m = oe.EllipseModel()
        assert m.estimate(pts) and r['status'] == 1
        d = np.subtract(m.params, r['params'])
        d[4] = (d[4] + np.pi / 2) % np.pi - np.pi / 2
        assert np.max(np.abs(d)) <= 1e-10
        # and the distances: from outside, leastsq reaches the smallest stationary distance, to its own xtol (1.49e-8 in t)
        q = np.array(r['params'][:2]) + rng.uniform(-3 * b, 3 * b, (5, 2))
        out = np.array([mr.mp_distance(r['params'], p) for p in q])
        m.params = r['params']
        res = m.residuals(q)
        far = out > 0.5 * b
        assert np.all(np.abs(res[far] - out[far]) <= 1e-6 * (1 + b))


def test_fit_flags_of_degenerate_sets():
    """collinear points and fewer than three distinct points make S3 singular.  numpy raises LinAlgError where its elimination
    meets an exactly zero pivot; on a vertical line or two distinct points the float64 pivot is a rounding error instead and numpy
    returns False.  Points on a hyperbola still give exactly one admissible eigenvector: the direct fit is ellipse-specific."""
    x = np.arange(10.)
    for pts, numpy_raises in ((np.c_[x, np.zeros(10)], True), (np.c_[x, x], True), (np.c_[x, -x], True),
                              (np.tile([[2., 5.]], (6, 1)), True), (np.c_[np.full(10, 3.), x], False),
                              (np.r_[np.tile([[2., 5.]], (3, 1)), np.tile([[7., -1.]], (3, 1))], False)):
        assert mr.mp_fit(pts)['status'] == -1
        if numpy_raises:
            with pytest.raises(np.linalg.LinAlgError):
                oe.EllipseModel().estimate(pts)
        else:
            assert not oe.EllipseModel().estimate(pts)
    s = np.linspace(-1.5, 1.5, 9)
    for pts in (np.c_[np.cosh(s), np.sinh(s)], np.r_[np.c_[np.cosh(s), np.sinh(s)], np.c_[-np.cosh(s), np.sinh(s)]] * [3, 2] + [100, 50]):
        r = mr.mp_fit(pts)
        assert r['status'] == 1 and r['n_admissible'] == 1 and min(abs(c) for c in r['cond']) > 1e-3
        assert oe.EllipseModel().estimate(pts)


def test_exact_scatter_is_exact():
    pts = np.array([[0.1, 1e8], [-3.5, 2.0 ** -30], [1e-300, 7.]])
    S1, S2, S3, den = mr.exact_scatter(pts)
    from fractions import Fraction as F
    x = [F(v) for v in pts[:, 0]]
    y = [F(v) for v in pts[:, 1]]
    assert F(S1[0][1], den ** 4) == sum(xi ** 3 * yi for xi, yi in zip(x, y))
    assert F(S2[2][0], den ** 3) == sum(yi ** 2 * xi for xi, yi in zip(x, y))
    assert F(S3[2][2], den ** 2) == 3
