"""
Extended-precision references of the ellipse fit and of the point-to-ellipse distance (test infrastructure, host only).

``mp_fit`` is the direct (Halir-Flusser) fit of ``oracle/ellipse.py`` without its rounding: the 21 scatter sums are exact
(every float64 is a dyadic rational, so the sums of products are integers over one power of two), and the solve and the eigenvectors
run in mpmath at ``DPS`` digits.  ``mp_stationary_distances`` lists the distance from a point to every stationary point of the
squared distance over the ellipse angle, from the roots of a quartic; the smallest one is the true distance.

These are precision references only: the numpy oracle stays the semantic reference (flags, sign rule, raster).
"""
import mpmath

DPS = 60


def _dyadic(values):
    """integers X and one power of two ``den`` with values == X / den exactly"""
    ratios = [float(v).as_integer_ratio() for v in values]
    den = max([d for _, d in ratios] + [1])
    return [n * (den // d) for n, d in ratios], den


def exact_scatter(points):
    """the integer scatter sums and their common denominators: S1 = D1^T D1 over den^4, S2 = D1^T D2 over den^3, S3 = D2^T D2 over
    den^2, with D1 = [x^2, xy, y^2] and D2 = [x, y, 1] (rows of integers over den and den^2)"""
    xs = [float(p[0]) for p in points]
    ys = [float(p[1]) for p in points]
    X, den = _dyadic(xs + ys)
    X, Y = X[:len(xs)], X[len(xs):]
    d1 = [[x * x for x in X], [x * y for x, y in zip(X, Y)], [y * y for y in Y]]
    d2 = [X, Y, [den] * len(X)]
    dot = lambda u, v: sum(a * b for a, b in zip(u, v))  # noqa: E731
    S1 = [[dot(d1[i], d1[j]) for j in range(3)] for i in range(3)]
    S2 = [[dot(d1[i], d2[j]) for j in range(3)] for i in range(3)]
    S3 = [[dot(d2[i], d2[j]) for j in range(3)] for i in range(3)]
    return S1, S2, S3, den


def _det3(A):
    return (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
            + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]))


def _conic_params(v, P):
    """ellipse parameters of the conic (a, b, c) = v and (d, f, g) = P v, as oracle/ellipse.py computes them; an invalid square
    root or division gives 0, as numpy's nan_to_num does there"""
    a, b, c = v
    d, f, g = (sum(P[i, j] * v[j] for j in range(3)) for i in range(3))
    b, d, f = b / 2, d / 2, f / 2
    den = b * b - a * c
    if den == 0:
        return [mpmath.mpf(0)] * 5
    x0 = (c * d - b * f) / den
    y0 = (a * f - b * d) / den
    num = a * f * f + c * d * d + g * b * b - 2 * b * d * f - a * c * g
    term = mpmath.sqrt((a - c) ** 2 + 4 * b * b)
    axes = []
    for sgn in (1, -1):
        q = den * (sgn * term - (a + c))
        r = 2 * num / q if q != 0 else mpmath.mpf(-1)
        axes.append(mpmath.sqrt(r) if r >= 0 else mpmath.mpf(0))
    # skimage's rule (a > c, and sign(b) pi / 4 where a == c) on purpose: at 60 digits a == c does not occur for sampled data,
    # and the device's a >= c differs from it only there
    if a != c:
        phi = mpmath.atan(2 * b / (a - c)) / 2
    else:
        phi = mpmath.sign(b) * mpmath.pi / 4
    if a > c:
        phi += mpmath.pi / 2
    return [x0, y0, axes[0], axes[1], phi]


def mp_fit(points):
    """the direct fit of ``points`` ([n, 2] float64) in extended precision

    :return dict: ``status`` 1 fitted, 0 not exactly one admissible eigenvector, -1 singular S3 (numpy raises LinAlgError);
        ``n_admissible``; ``cond``: 4ac - b^2 of each unit eigenvector of M (floats; [] when S3 is singular); ``params``: (xc, yc, a,
        b, theta) as floats with the shorter semi-axis first, or None; ``eigenvalues`` of M (floats)
    """
    S1i, S2i, S3i, den = exact_scatter(points)
    out = {'status': -1, 'n_admissible': 0, 'cond': [], 'params': None, 'eigenvalues': []}
    if _det3(S3i) == 0:
        return out
    with mpmath.workdps(DPS):
        m = lambda A, k: mpmath.matrix([[mpmath.mpf(A[i][j]) / mpmath.mpf(den) ** k for j in range(3)] for i in range(3)])  # noqa
        S1, S2, S3 = m(S1i, 4), m(S2i, 3), m(S3i, 2)
        iS3 = mpmath.inverse(S3)
        R = S1 - S2 * iS3 * S2.T
        M = mpmath.matrix(3, 3)
        for j in range(3):
            M[0, j], M[1, j], M[2, j] = R[2, j] / 2, -R[1, j], R[0, j] / 2
        P = -iS3 * S2.T
        E, ER = mpmath.eig(M)
        vecs, cond = [], []
        for k in range(3):
            v = [mpmath.re(ER[i, k]) for i in range(3)]
            nrm = mpmath.sqrt(sum(x * x for x in v))
            v = [x / nrm for x in v]
            vecs.append(v)
            cond.append(4 * v[0] * v[2] - v[1] * v[1])
        adm = [k for k in range(3) if cond[k] > 0]
        out.update(n_admissible=len(adm), cond=[float(c) for c in cond], eigenvalues=[float(mpmath.re(e)) for e in E])
        if len(adm) != 1:
            out['status'] = 0
            return out
        v = vecs[adm[0]]
        par = _conic_params(v, P)
        if par[2] > par[3]:
            par = _conic_params([-x for x in v], P)
        out.update(status=1, params=[float(x) for x in par])
    return out


def mp_stationary_distances(params, point):
    """distances from ``point`` to every stationary point of the squared distance over the ellipse angle t, ascending

    In the ellipse's frame the point is (u, v) and the ellipse (a cos t, b sin t); the derivative (b^2 - a^2) sin t cos t +
    a u sin t - b v cos t vanishes at the roots tau = tan(t / 2) of
    b v tau^4 + 2 (a^2 - b^2 + a u) tau^3 + 2 (b^2 - a^2 + a u) tau - b v, and at t = pi when the leading coefficient is 0.  When
    every coefficient is 0 (the centre of a circle, or a = b = 0) every t is stationary and the one distance is returned.
    """
    with mpmath.workdps(DPS):
        xc, yc, a, b, th = (mpmath.mpf(float(p)) for p in params)
        x, y = mpmath.mpf(float(point[0])), mpmath.mpf(float(point[1]))
        ct, st = mpmath.cos(th), mpmath.sin(th)
        u = ct * (x - xc) + st * (y - yc)
        v = -st * (x - xc) + ct * (y - yc)
        dist = lambda t: mpmath.sqrt((a * mpmath.cos(t) - u) ** 2 + (b * mpmath.sin(t) - v) ** 2)  # noqa: E731
        coef = [b * v, 2 * (a * a - b * b + a * u), mpmath.mpf(0), 2 * (b * b - a * a + a * u), -b * v]
        ts = []
        if coef[0] == 0:
            ts.append(mpmath.pi)
        while coef and coef[0] == 0:
            coef.pop(0)
        if not coef:
            return [float(dist(mpmath.mpf(0)))]
        if len(coef) > 1:
            roots = mpmath.polyroots(coef, maxsteps=400, extraprec=4 * DPS * 4)
            for r in roots:
                r = mpmath.mpc(r)
                if abs(r.imag) <= mpmath.mpf(10) ** (-DPS // 3) * (1 + abs(r)):
                    ts.append(2 * mpmath.atan(r.real))
        return sorted(float(dist(t)) for t in ts)


def mp_distance(params, point):
    """the distance from ``point`` to the ellipse: the smallest stationary distance"""
    return mp_stationary_distances(params, point)[0]
