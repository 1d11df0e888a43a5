"""GPU tests of csrc/ellipse_fit.cu at the edges where its kernels branch, against extended-precision references
(tests/ellipse_mp_reference.py) for the arithmetic and the float64 oracle (oracle/ellipse.py) for the semantics.

* ``k_ellipse_trials``: the direct fit at sample counts around the 32-lane scatter stride, on exact, rotated, thin and far-off
  ellipses; the residual loop and the criterion loop at point counts around ``ETHREADS`` = 128; a batch of trials against the
  same trials launched alone.
* ``k_ellipse_overlap``: the raster at every border, rotation and radius edge, on images past the 132 x 8-block grid cap, with
  label counts on both sides of ``ELL_SMEM_LABELS`` = 4096.
* ``k_binary_morph``: openings whose disc is many times the mask, so the reflection wraps more than once.
"""
import ctypes as C
import math

import numpy as np
import pytest
from scipy import ndimage

from oracle import ellipse as oe
import ellipse_mp_reference as mr

pytestmark = pytest.mark.gpu

ETHREADS = 128
ELL_SMEM_LABELS = 4096
GRID_CAP_THREADS = 132 * 8 * 256


@pytest.fixture(scope='module')
def ef():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import ellipse_fitting
    return ellipse_fitting


# ----------------------------------------------------------------------------------------------------------------- A. the fit

SAMPLE_COUNTS = [5, 6, 31, 32, 33, 64, 1000, 20000]     # around the 32-lane stride of the scatter sums, and far past it


def _lattice_circle(r):
    """the integer points of the circle of radius r about the origin"""
    pts = []
    for x in range(-r, r + 1):
        y = math.isqrt(r * r - x * x)
        if x * x + y * y == r * r:
            pts += [(x, y), (x, -y)] if y else [(x, 0)]
    return np.array(pts, dtype=np.float64)


PIXEL_CIRCLE = _lattice_circle(1105)        # 1105^2 = 5^2 13^2 17^2: 108 points


def _shape_specs():
    """(name, (xc, yc, a, b, theta), noise); the centre offsets 0, 500 and 8000 px cost the uncentred sums their digits"""
    q = np.pi / 4
    specs = [('circle_int', (0., 0., 20., 20., 0.), 0.), ('circle_int_500', (500., 500., 20., 20., 0.), 0.),
             ('circle_pixel', None, 0.), ('axis', (0., 0., 10., 25., 0.), 0.), ('axis_500', (500., -500., 10., 25., 0.), 0.),
             ('axis_noisy', (3., 4., 10., 25., 0.), 0.5), ('far_8000', (8000., 8000., 40., 60., 0.7), 0.),
             ('far_8000_noisy', (8000., 8000., 40., 60., 0.7), 0.5), ('far_2000', (2000., -2000., 40., 60., 0.7), 0.),
             ('far_4000', (4000., 4000., 40., 60., 2.2), 0.), ('ratio_1e3', (0., 0., 0.05, 50., 1.2), 0.),
             ('ratio_1e3_500', (500., 0., 1., 1000., 0.3), 0.)]
    for th in (0.3, q - 1e-12, q, q + 1e-12, 1.5, np.pi / 2, 2.5, 3 * q, np.pi - 1e-9):
        specs.append(('theta_%.13g' % th, (0., 0., 12., 30., th), 0.))
        specs.append(('theta_%.13g_noisy' % th, (0., 0., 12., 30., th), 0.4))
    return specs


def fit_cases():
    """every (name, points) of the fit section; deterministic"""
    rng = np.random.RandomState(7)
    m = oe.EllipseModel()
    cases = []
    for n in SAMPLE_COUNTS:
        for name, params, noise in _shape_specs():
            if params is None:          # integer points exactly on the circle of radius 1105 about (300, 200), cycled
                pts = PIXEL_CIRCLE[rng.permutation(len(PIXEL_CIRCLE))][np.arange(n) % len(PIXEL_CIRCLE)] + [300., 200.]
            else:
                pts = m.predict_xy(rng.uniform(0, 2 * np.pi, n), params)
                if noise:
                    pts = pts + rng.normal(0, noise, pts.shape)
            cases.append(('%s/n=%d' % (name, n), np.ascontiguousarray(pts)))
    return cases


def _perr(p, ref):
    """distance between two parameter vectors: the centre and semi-axes in px, theta modulo pi weighted by b - a of the reference
    (the boundary moves by at most that much per radian; a circle has no orientation)"""
    d = np.abs(np.subtract(p, ref))
    d[4] = abs((p[4] - ref[4] + np.pi / 2) % np.pi - np.pi / 2) * abs(ref[3] - ref[2])
    return float(np.max(d))


def _oracle_fit(points):
    m = oe.EllipseModel()
    try:
        return m.params if m.estimate(points) else None
    except np.linalg.LinAlgError:
        return None


def test_fit_against_extended_precision(ef):
    """The flag and the parameters of every case against mp_fit, centres 0 to 8 000 px out and axis ratios up to 1e3.

    * Flag: equal to the mp flag wherever all three mp values of 4ac - b^2 are clear of zero by 1e-9 (unit eigenvectors) and numpy's
      float64 route, in both sample orders, gets the mp flag too.  Where numpy itself misses it (five samples of a circle 500 px out,
      some ellipses 8 000 px out or of axis ratio 1e3), the cases are printed, not asserted.
    * Parameters: no further from mp than ten times the numpy oracle's own error or its sensitivity to the order of the samples, plus
      1e-12 of the scale (the centre and semi-axes in px, theta modulo pi weighted by b - a).

    Before the device took its sums about the samples' mean and its eigenvectors by inverse iteration on M, it returned False for
    ellipses 8 000 px out and of axis ratio 1e3 that numpy and mp fit, and its parameters at ratio 1e3 were up to 5e3 times
    numpy's error from mp.
    """
    cases = fit_cases()
    sets = [p for _, p in cases]
    ok, par, _, _, _ = ef._run_trials(sets, np.arange(len(sets)), samples=[np.arange(len(p)) for p in sets])
    fails, worst, flags, skipped, float64_lost = [], [], 0, [], []
    for (name, pts), o, p in zip(cases, ok, par):
        ref = mr.mp_fit(pts)
        npy, rev = _oracle_fit(pts), _oracle_fit(pts[::-1].copy())
        clear = ref['status'] == -1 or min(abs(c) for c in ref['cond']) > 1e-9
        if clear and (npy is not None) == (rev is not None) == (ref['status'] == 1):
            flags += 1
            if (o == 1) != (ref['status'] == 1):
                fails.append(('flag', name, int(o), ref['status']))
        elif (o == 1) != (ref['status'] == 1):
            float64_lost.append(name)
        if o != 1 or ref['status'] != 1:
            continue
        if npy is None or rev is None:
            skipped.append(name)
            continue
        scale = max(abs(ref['params'][0]), abs(ref['params'][1]), ref['params'][3])
        e_dev, e_np, sens = _perr(p, ref['params']), _perr(npy, ref['params']), _perr(npy, rev)
        worst.append((e_dev / max(e_np, sens, 1e-16 * scale), name, e_dev, e_np, sens))
        if e_dev > 10 * max(e_np, sens) + 1e-12 * scale:
            fails.append(('params', name, e_dev, e_np, sens))
    worst.sort(reverse=True)
    print('\nfit: %d cases, %d flags checked, %d fits compared' % (len(cases), flags, len(worst)))
    print('flag differs from mp where numpy\'s float64 route also misses it: %r; numpy failed, device fitted: %r' % (float64_lost, skipped))
    for w in worst[:3]:
        print('|device - mp| / max(|numpy - mp|, numpy order sensitivity) %.3g (%s: device %.3g, numpy %.3g, sensitivity %.3g)' % w)
    assert not fails, fails
    assert flags >= 0.9 * len(cases)


def test_fit_single_model_calls_match_batch(ef):
    """EllipseModelSegm.estimate is a batch of one: the same bits as the batched trial"""
    cases = fit_cases()[::7]
    sets = [p for _, p in cases]
    ok, par, _, _, _ = ef._run_trials(sets, np.arange(len(sets)), samples=[np.arange(len(p)) for p in sets])
    for (name, pts), o, p in zip(cases, ok, par):
        m = ef.EllipseModelSegm()
        assert m.estimate(pts) == (o == 1), name
        if o == 1:
            assert np.array_equal(m.params, p), name


def test_fit_degenerate_sets(ef):
    """collinear points and fewer than three distinct points: S3 is singular (mp).  Where numpy's elimination meets an exactly zero
    pivot it raises LinAlgError, and so must the device; where its pivot is a rounding error instead (a vertical line, two
    distinct points) numpy returns False, and the device may return False or raise but not fit.  Points on a hyperbola give exactly one admissible eigenvector (the direct fit is
    ellipse-specific), so both fit an ellipse there, and its parameters follow mp as any fit's do."""
    x = np.arange(10.)
    raising = [np.c_[x, np.zeros(10)], np.c_[x, x], np.c_[x, -x], np.tile([[2., 5.]], (6, 1)), np.tile([[0., 0.]], (40, 1)),
               np.c_[np.arange(33.), np.zeros(33)] + [8000., 0.]]
    for pts in raising:
        assert mr.mp_fit(pts)['status'] == -1
        with pytest.raises(np.linalg.LinAlgError):
            oe.EllipseModel().estimate(pts)
        with pytest.raises(np.linalg.LinAlgError):
            ef.EllipseModelSegm().estimate(pts)
    for pts in (np.c_[np.full(10, 3.), x], np.r_[np.tile([[2., 5.]], (3, 1)), np.tile([[7., -1.]], (3, 1))]):
        assert mr.mp_fit(pts)['status'] == -1 and not oe.EllipseModel().estimate(pts)
        try:
            assert not ef.EllipseModelSegm().estimate(pts)
        except np.linalg.LinAlgError:
            pass
    s = np.linspace(-1.5, 1.5, 33)
    for pts in (np.c_[np.cosh(s), np.sinh(s)], np.r_[np.c_[np.cosh(s), np.sinh(s)], np.c_[-np.cosh(s), np.sinh(s)]] * [3, 2] + [100, 50],
                np.c_[s + 2, 1 / (s + 2)]):
        ref = mr.mp_fit(pts)
        assert ref['status'] == 1 and min(abs(c) for c in ref['cond']) > 1e-9
        m = ef.EllipseModelSegm()
        assert m.estimate(pts)
        npy, rev = _oracle_fit(pts), _oracle_fit(pts[::-1].copy())
        assert _perr(m.params, ref['params']) <= 10 * max(_perr(npy, ref['params']), _perr(npy, rev)) + 1e-12 * 200


# ----------------------------------------------------------------------------------------------- B. residuals and inlier counts

POINT_COUNTS = [0, 1, 127, 128, 129, 100000]            # around the ETHREADS-strided residual loop
RESID_PARAMS = [(3., 4., 10., 30., 0.6), (500., 500., 20., 21., 2.0), (0., 0., 15., 15., 0.), (100., -50., 5., 40., 0.),
                (8000., 20., 25., 60., 3.0), (10., 10., 0., 20., 0.4), (10., 10., 20., 0., 0.4), (7., 7., 0., 0., 0.)]
MP_PER_SET = 24


def _resid_points(params, n, rng):
    """n points cycling through: outside (1.2 to 3 times the ellipse), inside (0 to 0.9 times), exactly the centre, on the
    ellipse (predict_xy)"""
    xc, yc, a, b, th = params
    t = rng.uniform(0, 2 * np.pi, n)
    k = np.arange(n) % 4
    f = np.where(k == 0, rng.uniform(1.2, 3, n), np.where(k == 1, rng.uniform(0, 0.9, n), np.where(k == 2, 0., 1.)))
    pts = oe.EllipseModel().predict_xy(t, (0., 0., a, b, th)) * f[:, None] + [xc, yc]
    # a degenerate ellipse is a segment or a point: push the "outside" points off it sideways as well
    pts[k == 0] += rng.uniform(-5, 5, (int(np.sum(k == 0)), 2)) * (min(a, b) == 0)
    pts[k == 2] = [xc, yc]
    return np.ascontiguousarray(pts), k


def test_residuals_against_stationary_distances(ef):
    """Every residual against the mp stationary distances of its point.  A point with exactly two stationary points (outside the
    evolute) has one minimum, and the device must find it to 1e-9 (1 + scale); any other point (inside, at the centre, and for
    elongated ellipses some outside points near the minor vertices) must get some stationary distance, never below the minimum.
    n_inl must count the returned residuals below thr, and equal the mp count wherever no residual is within 1e-9 of thr."""
    rng = np.random.RandomState(3)
    sets, kinds, params = [], [], []
    for p in RESID_PARAMS:
        for n in POINT_COUNTS:
            pts, k = _resid_points(p, n, rng)
            sets.append(pts)
            kinds.append(k)
            params.append(p)
    thr = 4.
    ok, _, n_inl, _, resid = ef._run_trials(sets, np.arange(len(sets)), params=params, thr=thr, want_resid=True)
    assert np.all(ok == 1)
    off = np.concatenate([[0], np.cumsum([len(s) for s in sets])])
    strict = loose = 0
    worst = 0.
    for i, (pts, p) in enumerate(zip(sets, params)):
        r = resid[off[i]:off[i + 1]]
        assert np.all(np.isfinite(r)) and np.all(r >= 0)
        assert n_inl[i] == np.sum(r < thr), (i, n_inl[i], np.sum(r < thr))
        scale = max(abs(p[0]), abs(p[1]), p[2], p[3])
        tol = 1e-9 * (1 + scale)
        pick = np.unique(np.r_[np.arange(min(len(pts), 8)), rng.choice(len(pts), min(len(pts), MP_PER_SET - 8), replace=False)]) \
            if len(pts) else []
        mp_count = dev_count = 0
        for j in pick:
            d = np.array(mr.mp_stationary_distances(p, pts[j]))
            if len(d) == 2:
                strict += 1
                assert abs(r[j] - d[0]) <= tol, (p, pts[j], r[j], d)
                worst = max(worst, abs(r[j] - d[0]) / (1 + scale))
            else:
                loose += 1
                assert np.min(np.abs(d - r[j])) <= tol and r[j] >= d[0] - tol, (p, pts[j], r[j], d)
            near = d[np.argmin(np.abs(d - r[j]))]
            if abs(near - thr) > 1e-9:
                mp_count += near < thr
                dev_count += r[j] < thr
        assert mp_count == dev_count
    print('\nresiduals: %d points with one minimum, %d with several; worst |device - mp| / (1 + scale) %.3g' % (strict, loose, worst))
    assert strict >= 200 and loose >= 100
    # a threshold equal to a returned residual: that residual is not an inlier
    i = len(POINT_COUNTS) - 1
    r = resid[off[i]:off[i + 1]]
    for thr in (float(r[5]), float(np.sort(r)[len(r) // 2])):
        _, _, n2, _, _ = ef._run_trials([sets[i]], [0], params=[params[i]], thr=thr)
        assert n2[0] == np.sum(r < thr) < np.sum(r <= thr)


def test_single_model_residuals_match_batch(ef):
    rng = np.random.RandomState(4)
    for p in RESID_PARAMS[:5]:
        pts, _ = _resid_points(p, 129, rng)
        m = ef.EllipseModelSegm()
        m.params = list(p)
        r = ef._run_trials([pts], [0], params=[p], want_resid=True)[4][:129]
        assert np.array_equal(m.residuals(pts), r)
    assert len(ef.EllipseModelSegm().residuals(np.zeros((0, 2)))) == 0


# ------------------------------------------------------------------------------------------------------------- C. the criterion

CRIT_COUNTS = [0, 1, 127, 128, 129, 10 ** 6]           # around the ETHREADS-strided criterion loop and its tree reduction
CRIT_PARAMS = [(20., 30., 8., 16., 0.), (20., 30., 8., 16., 0.7), (-5., 40., 32., 4., 2.9), (20., 30., 0., 16., 0.), (20., 30., 8., 0., 0.3),
               (20., 30., 0., 0., 0.), (20., 30., 1e3, 1e3, 4.0)]


def _crit_points(n, rng):
    """n points: the axis vertices of the first ellipse of CRIT_PARAMS (exactly on its boundary, u^2 + w^2 == 1 in float64), its
    centre (0 / 0 for a zero radius), then random points about it"""
    exact = np.array([[28., 30.], [12., 30.], [20., 46.], [20., 14.], [20., 30.], [24., 30.], [20., 38.], [28.5, 30.]])
    pts = np.r_[exact, rng.uniform(-5, 45, (max(n - len(exact), 0), 2)) + [0., 10.]][:n]
    return np.ascontiguousarray(pts)


def _inside(params, pts):
    """the criterion's inside test as the reference writes it (ellipse_fitting.py:121-137), in float64"""
    xc, yc, a, b, phi = params
    s, c = np.sin(phi), np.cos(phi)
    r, cc = pts[:, 0] - xc, pts[:, 1] - yc
    with np.errstate(divide='ignore', invalid='ignore'):
        u, w = (r * c + cc * s) / a, (r * s - cc * c) / b
        return u * u + w * w <= 1


def _crit(ef, pts, labels, term, params=CRIT_PARAMS):
    return ef._run_trials([np.zeros((0, 2))], [0] * len(params), params=params, crit_input=(pts, labels, term))[3]


def test_criterion_membership_bits(ef):
    """each point in its own label with term 2^j (52 at a time): the criterion's bits spell out which points fell inside, and must
    equal numpy's <= 1 mask exactly -- including the points on the boundary and the NaN of a zero radius (outside)"""
    rng = np.random.RandomState(5)
    for n in CRIT_COUNTS[:5]:
        pts = _crit_points(n, rng)
        labels = np.arange(n, dtype=np.int32)
        masks = np.array([_inside(p, pts) for p in CRIT_PARAMS]).reshape(len(CRIT_PARAMS), n)
        if n >= 8:
            assert masks[0, :4].all() and masks[0, 4:7].all() and not masks[0, 7]      # the boundary is inside
            assert not masks[3:6].any()                                                   # zero radii: nothing inside
        got = np.zeros_like(masks)
        for lo in range(0, max(n, 1), 52):
            term = np.zeros(max(n, 1))
            hi = min(lo + 52, n)
            term[lo:hi] = 2.0 ** np.arange(hi - lo)
            crit = _crit(ef, pts, labels, term)
            for t, v in enumerate(crit):
                bits = int(v)
                assert float(bits) == v
                got[t, lo:hi] = [(bits >> j) & 1 for j in range(hi - lo)]
        assert np.array_equal(got, masks), n


def test_criterion_sums_and_counts(ef):
    """with random positive terms, the sum to rtol 1e-12 of math.fsum over numpy's mask; with unit terms, the count exactly"""
    rng = np.random.RandomState(6)
    for n in CRIT_COUNTS:
        pts = _crit_points(n, rng)
        labels = rng.randint(0, 1000, n).astype(np.int32)
        term = rng.uniform(0.5, 1.5, 1000)
        crit = _crit(ef, pts, labels, term)
        ones = _crit(ef, pts, np.zeros(n, np.int32), np.ones(1))
        for t, p in enumerate(CRIT_PARAMS):
            m = _inside(p, pts)
            assert ones[t] == np.sum(m), (n, p)
            ref = math.fsum(term[labels[m]])
            assert abs(crit[t] - ref) <= 1e-12 * abs(ref), (n, p, crit[t], ref)


# ---------------------------------------------------------------------------------------------------------------- D. batching

def test_batch_equals_trials_launched_alone(ef):
    """thousands of trials over centres of 0 to 5 000 points, in non-monotone centre order: every output of every trial has the
    bits of the same trial launched alone (ellipse_fit.cu:2-4), on the sample path and on the params_in path"""
    rng = np.random.RandomState(8)
    sizes = [0, 5, 6, 31, 32, 33, 127, 128, 129, 1000, 5000] + list(rng.randint(5, 400, 9))
    m = oe.EllipseModel()
    sets = []
    for n in sizes:
        p = (rng.uniform(0, 600), rng.uniform(0, 600), rng.uniform(5, 30), rng.uniform(30, 60), rng.uniform(0, np.pi))
        sets.append(np.ascontiguousarray(m.predict_xy(rng.uniform(0, 2 * np.pi, n), p) + rng.normal(0, 2, (n, 2))))
    sp = rng.uniform(0, 600, (3000, 2))
    labels = rng.randint(0, 50, 3000).astype(np.int32)
    crit_in = (sp, labels, rng.normal(0, 1, 50))
    T = 2000
    centre = rng.randint(0, len(sizes), T)
    samples = [rng.choice(len(sets[c]), rng.randint(5, min(len(sets[c]), 200) + 1), replace=False) if len(sets[c]) >= 5
               else np.arange(len(sets[c])) for c in centre]
    thr = 3.
    batch = ef._run_trials(sets, centre, samples=samples, crit_input=crit_in, thr=thr, want_resid=True)
    roff = np.concatenate([[0], np.cumsum(np.array(sizes)[centre])])
    assert set(batch[0]) >= {-1, 1}
    params = rng.uniform(0, 600, (T, 5)) * [1, 1, 0.1, 0.1, 0.005]
    pbatch = ef._run_trials(sets, centre, params=params, crit_input=crit_in, thr=thr, want_resid=True)
    for b, kw in ((batch, lambda t: dict(samples=[samples[t]])), (pbatch, lambda t: dict(params=[params[t]]))):
        for t in range(T):
            c = centre[t]
            alone = ef._run_trials([sets[c]], [0], crit_input=crit_in, thr=thr, want_resid=True, **kw(t))
            for k in range(4):
                assert np.array_equal(alone[k][0], b[k][t]), (t, c, k)
            assert np.array_equal(alone[4][:sizes[c]], b[4][roff[t]:roff[t + 1]]), (t, c)


# ---------------------------------------------------------------------------------------------------- E. raster and overlap

def _device_overlap(ef, segm, params):
    """one isb_ellipse_overlap launch as add_overlap_ellipse makes it: (mask, area per label, overlap per label, ellipse area)"""
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.engine import get_engine
    c1, c2, h, w, phi = params
    bbox, geom = ef._draw_ellipse_geometry(int(c1), int(c2), int(h), int(w), phi, segm.shape)
    n = max(int(np.max(segm)) + 1, 1)
    eng = get_engine()
    d_seg = eng.to_device(np.ascontiguousarray(segm, dtype=np.int32))
    mask = eng.torch.empty(segm.shape, dtype=eng.torch.uint8, device=eng.device)
    counts = eng.torch.empty(2 * n + 1, dtype=eng.torch.int64, device=eng.device)
    _lib.check(eng.lib.isb_ellipse_overlap(_lib.ptr(d_seg), segm.shape[0], segm.shape[1], n, bbox.ctypes.data_as(C.POINTER(C.c_int32)),
                                           geom.ctypes.data_as(C.POINTER(C.c_double)), _lib.ptr(mask), _lib.ptr(counts), _lib.stream_ptr()))
    cnt = eng.to_host(counts)
    return eng.to_host(mask).astype(bool), cnt[:n], cnt[n:2 * n], int(cnt[2 * n])


def _oracle_mask(shape, params):
    c1, c2, h, w, phi = params
    mask = np.zeros(shape, dtype=bool)
    with np.errstate(divide='ignore', invalid='ignore'):
        rr, cc = oe.draw_ellipse(int(c1), int(c2), int(h), int(w), shape, phi)
    mask[rr, cc] = True
    return mask


def _host_add(segm, mask, label, thr):
    """the reference's add_overlap_ellipse (ellipse_fitting.py:282-345) over np.bincount counts"""
    n = max(int(np.max(segm)) + 1, 1)
    valid = segm >= 0
    area = np.bincount(segm[valid], minlength=n)
    overlap = np.bincount(segm[valid & mask], minlength=n)
    for lb in range(1, n):
        sizes = [s for s in (int(area[lb]), int(mask.sum())) if s > 0]
        if not sizes or overlap[lb] / float(min(sizes)) > thr:
            return segm
    out = segm.copy()
    out[mask] = label
    return out


def _label_maps(shape, rng):
    """label maps with 1 label (all 0, or all negative), 4 096 (shared-memory counters) and 4 097 (global counters), with
    negative labels mixed in"""
    size = int(np.prod(shape))
    out = [np.zeros(shape, np.int64), np.full(shape, -2, np.int64)]
    for n in (ELL_SMEM_LABELS, ELL_SMEM_LABELS + 1):
        seg = rng.randint(-2, n, size)
        seg[rng.randint(size)] = n - 1
        out.append(seg.reshape(shape))
    return out


def _ellipses(H, W):
    rots = [0., np.pi / 4, np.pi / 2, 3 * np.pi / 4, np.pi, -0.7, 4.0]
    radii = [(0, 0), (1, 2), (2, 1), (0, 3), (max(H, W) // 3 + 1, max(H, W) // 2 + 2)]
    centres = [(H // 2, W // 2), (0, W // 2), (H - 1, W // 2), (H // 2, 0), (H // 2, W - 1), (-3, W // 2), (H + 2, W // 2),
               (H // 2, -4), (H // 2, W + 1), (-H - 50, -W - 50)]
    out = []
    for i, (r, c) in enumerate(centres):
        for j, rot in enumerate(rots):
            h, w = radii[(i + j) % len(radii)]
            out.append((r, c, h, w, rot))
    out += [(H // 2, W // 2, h, w, rot) for h, w in radii for rot in rots]
    out += [(H // 2, W // 2, 3 * H + 2, 3 * W + 2, 0.3), (H // 2 + 0.7, W // 2 - 0.2, 2.9, 1.6, 0.5)]
    return out


@pytest.mark.parametrize('shape', [(1, 1), (1, 37), (37, 1), (45, 61), (600, 601)],
                         ids=['1x1', '1xN', 'Nx1', 'odd', 'past_grid_cap'])
def test_raster_and_overlap_counts(ef, shape):
    """mask bit for bit against oracle.draw_ellipse, the per-label area and overlap and the ellipse area exactly against
    np.bincount, and every add-or-skip decision of add_overlap_ellipse against the host composition; 600 x 601 pixels run the
    grid-stride loop past the 132 x 8 blocks of 256 threads"""
    rng = np.random.RandomState(sum(shape))
    maps = _label_maps(shape, rng)
    big = shape[0] * shape[1] > GRID_CAP_THREADS
    for k, params in enumerate(_ellipses(*shape)[::3] if big else _ellipses(*shape)):
        segm = maps[k % len(maps)]
        mask, area, overlap, m_area = _device_overlap(ef, segm, params)
        ref = _oracle_mask(shape, params)
        assert np.array_equal(mask, ref), (shape, params)
        n = len(area)
        valid = segm >= 0
        assert np.array_equal(area, np.bincount(segm[valid], minlength=n)), (shape, params)
        assert np.array_equal(overlap, np.bincount(segm[valid & ref], minlength=n)), (shape, params)
        assert m_area == int(ref.sum())
        if n > 1 and (big or shape[0] * shape[1] > 100 and k % 3):
            continue        # the decision loop over 4 096 labels is host work: sample it on the larger images
        for thr in (1., 0.5, 0.):
            out = ef.add_overlap_ellipse(segm.copy(), params, 7777, thr)
            assert np.array_equal(out, _host_add(segm, ref, 7777, thr)), (shape, params, thr)


def test_raster_4096_square(ef):
    """16.7 M pixels, 62 times the capped grid, with 4 096 and 4 097 labels"""
    shape = (4096, 4096)
    rng = np.random.RandomState(9)
    assert shape[0] * shape[1] > GRID_CAP_THREADS
    for n, params in ((ELL_SMEM_LABELS, (2047, 2047, 3000, 5000, 0.)), (ELL_SMEM_LABELS + 1, (4000, 100, 1500, 900, 2.2)),
                      (ELL_SMEM_LABELS, (-200, 4300, 800, 1500, np.pi / 4))):
        segm = rng.randint(-1, n, shape, dtype=np.int32)
        segm[0, 0] = n - 1
        mask, area, overlap, m_area = _device_overlap(ef, segm, params)
        ref = _oracle_mask(shape, params)
        assert np.array_equal(mask, ref)
        valid = segm >= 0
        assert np.array_equal(area, np.bincount(segm[valid], minlength=n))
        assert np.array_equal(overlap, np.bincount(segm[valid & ref], minlength=n))
        assert m_area == int(ref.sum())


# ---------------------------------------------------------------------------------------------------------------- F. opening

MORPH_SHAPES = [(1, 1), (1, 40), (40, 1), (2, 3), (7, 7)]


def _reflect_morph(mask, radius, op):
    """grey erosion (np.minimum) or dilation (np.maximum) of a 0/1 mask with disk(radius), the border mirrored about the edge
    (scipy's mode 'reflect' is numpy's pad mode 'symmetric', which reflects as often as the pad needs)"""
    fp = oe.disk(radius).astype(bool)
    r = fp.shape[0] // 2
    pad = np.pad(mask, r, mode='symmetric')
    out = mask.copy()
    for dy, dx in zip(*np.nonzero(fp)):
        out = op(out, pad[dy:dy + mask.shape[0], dx:dx + mask.shape[1]])
    return out


def _reflect_opening(mask, radius):
    return _reflect_morph(_reflect_morph(mask, radius, np.minimum), radius, np.maximum)


@pytest.mark.parametrize('radius', [1, 1.5, 5, 15])
def test_opening_footprints_larger_than_the_mask(ef, radius):
    """binary_opening_disk bit for bit against grey erosion then dilation with the border reflected (numpy's symmetric padding) for a
    whole-pixel radius, and against oracle.opening (edge padding for the even disc) for radius 1.5; the disc is up to 31 x 31 on
    masks of 1 to 49 pixels.  scipy.ndimage.grey_erosion (mode reflect) is compared too and must agree except where a footprint
    exceeds the mask so far that scipy stops reflecting: scipy 1.18 erodes an all-ones 2 x 3 mask with disk(15) to zeros."""
    from pyimsegm_b200.descriptors import binary_opening_disk
    rng = np.random.RandomState(int(radius * 10))
    scipy_differs = 0
    for shape in MORPH_SHAPES:
        for mask in (rng.rand(*shape) < 0.6, np.ones(shape, bool), np.zeros(shape, bool), rng.rand(*shape) < 0.9):
            m8 = mask.astype(np.uint8)
            got = binary_opening_disk(m8, radius)
            if float(radius).is_integer():
                ref = _reflect_opening(m8, radius).astype(bool)
                fp = oe.disk(radius).astype(bool)
                sp = ndimage.grey_dilation(ndimage.grey_erosion(m8, footprint=fp, mode='reflect'), footprint=fp, mode='reflect')
                if 2 * radius + 1 <= 2 * min(shape) + 1:
                    assert np.array_equal(ref, sp.astype(bool)), (shape, radius, m8)
                else:
                    scipy_differs += not np.array_equal(ref, sp.astype(bool))
            else:
                ref = oe.opening(m8, oe.disk(radius)).astype(bool)
            assert np.array_equal(got, ref), (shape, radius, m8)
    print('\nradius %g: scipy differs from the reflected reference on %d masks smaller than the disc' % (radius, scipy_differs))


def test_split_background_foreground_small_masks(ef):
    """split_segm_background_foreground with its default discs (15 and 5) on masks smaller than the discs"""
    from scipy.ndimage import binary_fill_holes
    rng = np.random.RandomState(10)
    for shape in MORPH_SHAPES + [(12, 9)]:
        seg = rng.randint(0, 3, shape)
        bg, fg = ef.split_segm_background_foreground(seg)
        ref_bg = _reflect_opening((1 - binary_fill_holes(seg > 0)).astype(np.uint8), 15)
        ref_fg = _reflect_opening((seg == 1).astype(np.uint8), 5).astype(bool)
        assert np.array_equal(bg, ref_bg) and np.array_equal(fg, ref_fg), shape
