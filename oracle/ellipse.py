"""
Host oracle of the ellipse fitting (numpy / scipy only; test infrastructure, never imported by the product).

Restates, from their documented behaviour, what the reference's ``imsegm/ellipse_fitting.py`` builds on: scikit-image 0.14-0.18
``measure.EllipseModel`` (``estimate``: Halir-Flusser direct fit with ``numpy.linalg.eig``; ``residuals``: one scipy ``leastsq``
per point), ``draw.ellipse``, ``draw.ellipse_perimeter``, ``morphology.disk`` and ``morphology.opening`` (0.16-0.18: edge padding
for even footprints), and the reference's sequential RANSAC loop.

``estimate(canonical=True)`` fixes the sign of the eigenvector the way the device does (shorter semi-axis first).  skimage keeps
whatever sign LAPACK returns; the other sign describes the same ellipse with the semi-axes swapped and theta moved by pi / 2.
"""
import math

import numpy as np
from scipy import ndimage, optimize


def _conic_params(a1, P):
    a, b, c = a1
    d, f, g = P @ a1
    b, d, f = b / 2., d / 2., f / 2.
    x0 = (c * d - b * f) / (b ** 2. - a * c)
    y0 = (a * f - b * d) / (b ** 2. - a * c)
    numerator = a * f ** 2 + c * d ** 2 + g * b ** 2 - 2 * b * d * f - a * c * g
    term = np.sqrt((a - c) ** 2 + 4 * b ** 2)
    denominator1 = (b ** 2 - a * c) * (term - (a + c))
    denominator2 = (b ** 2 - a * c) * (-term - (a + c))
    with np.errstate(invalid='ignore', divide='ignore'):
        width = np.sqrt(2 * numerator / denominator1)
        height = np.sqrt(2 * numerator / denominator2)
        phi = 0.5 * np.arctan((2. * b) / (a - c))
    if a > c:
        phi += 0.5 * np.pi
    return [float(v) for v in np.nan_to_num([x0, y0, width, height, phi])]


class EllipseModel(object):
    """skimage.measure.EllipseModel (0.14-0.18) with the reference's ``criterion``"""

    def __init__(self):
        self.params = None

    def estimate(self, data, canonical=True):
        data = np.asarray(data, dtype=float)
        x, y = data[:, 0], data[:, 1]
        D1 = np.vstack([x ** 2, x * y, y ** 2]).T
        D2 = np.vstack([x, y, np.ones(len(x))]).T
        S1, S2, S3 = D1.T @ D1, D1.T @ D2, D2.T @ D2
        C1 = np.array([[0., 0., 2.], [0., -1., 0.], [2., 0., 0.]])
        inv_s3 = np.linalg.inv(S3)                    # LinAlgError on a singular S3
        M = np.linalg.inv(C1) @ (S1 - S2 @ inv_s3 @ S2.T)
        _, eig_vecs = np.linalg.eig(M)
        cond = 4 * np.multiply(eig_vecs[0, :], eig_vecs[2, :]) - np.power(eig_vecs[1, :], 2)
        a1 = eig_vecs[:, (cond > 0)]
        if 0 in a1.shape or len(a1.ravel()) != 3:
            return False
        a1 = np.real(a1.ravel())
        P = -inv_s3 @ S2.T
        params = _conic_params(a1, P)
        if canonical and params[2] > params[3]:
            params = _conic_params(-a1, P)
        self.params = params
        return True

    def predict_xy(self, t, params=None):
        xc, yc, a, b, theta = self.params if params is None else params
        ct, st = np.cos(t), np.sin(t)
        ctheta, stheta = math.cos(theta), math.sin(theta)
        x = xc + a * ctheta * ct - b * stheta * st
        y = yc + a * stheta * ct + b * ctheta * st
        return np.concatenate((x[..., None], y[..., None]), axis=t.ndim)

    def residuals(self, data):
        data = np.asarray(data, dtype=float)
        xc, yc, a, b, theta = self.params
        ctheta, stheta = math.cos(theta), math.sin(theta)

        def fun(t, xi, yi):
            ct, st = math.cos(t), math.sin(t)
            xt = xc + a * ctheta * ct - b * stheta * st
            yt = yc + a * stheta * ct + b * ctheta * st
            return (xi - xt) ** 2 + (yi - yt) ** 2

        x, y = data[:, 0], data[:, 1]
        t0 = np.arctan2(y - yc, x - xc) - theta
        res = np.empty(len(data))
        for i in range(len(data)):
            t, _ = optimize.leastsq(lambda tt, xi, yi: fun(tt[0], xi, yi), t0[i], args=(x[i], y[i]))
            res[i] = np.sqrt(fun(t[0], x[i], y[i]))
        return res

    def criterion(self, points, weights, labels, table_prob=(0.1, 0.9)):
        if not len(points) == len(weights) == len(labels):
            raise ValueError('different sizes')
        table_prob = np.array(table_prob)
        if 1 in (table_prob.ndim, table_prob.shape[0]):
            if table_prob.shape[0] == 1:
                table_prob = table_prob[0]
            table_prob = np.array([table_prob, 1. - table_prob])
        if table_prob.shape[0] != 2:
            raise ValueError('table shape %r' % (table_prob.shape, ))
        if np.max(labels) >= table_prob.shape[1]:
            raise ValueError('labels exceed the table')
        points = np.asarray(points, dtype=float)
        r_org, c_org, r_rad, c_rad, phi = self.params
        sin_phi, cos_phi = np.sin(phi), np.cos(phi)
        r, c = points[:, 0] - r_org, points[:, 1] - c_org
        inside = (((r * cos_phi + c * sin_phi) / r_rad) ** 2 + ((r * sin_phi - c * cos_phi) / c_rad) ** 2) <= 1
        table_q = -np.log(table_prob)
        labels_in = np.asarray(labels)[inside].astype(int)
        return np.sum(np.asarray(weights)[labels_in] * (table_q[0, labels_in] - table_q[1, labels_in]))


def ransac_trials(points, points_all, weights, labels, table_prob, min_samples, residual_threshold=1, max_trials=100):
    """every trial of the reference's loop (samples from the global numpy RNG): [(success, params, inliers, criterion)]"""
    points = np.array(points)
    if isinstance(min_samples, float):
        min_samples = int(min_samples * len(points))
    out = []
    for _ in range(max_trials):
        idx = np.random.choice(len(points), min_samples, replace=False)
        model = EllipseModel()
        if not model.estimate(points[idx]):
            out.append((False, None, None, None))
            continue
        inl = np.abs(model.residuals(points)) < residual_threshold
        out.append((True, model.params, inl, model.criterion(points_all, weights, labels, table_prob)))
    return out


def ransac_select(points, trials):
    """the reference's sequential selection over ransac_trials and its final refit: (params, inliers, best trial index)"""
    best, best_fit, best_inl, best_num, best_idx = None, np.inf, None, 0, -1
    for i, (ok, params, inl, fit) in enumerate(trials):
        if not ok:
            continue
        if fit < best_fit:
            best, best_fit, best_idx = params, fit, i
            if np.sum(inl) > best_num:
                best_inl, best_num = inl, np.sum(inl)
    if best_inl is not None:
        model = EllipseModel()
        model.params = list(best)
        model.estimate(np.asarray(points)[best_inl])
        best = model.params
    return best, best_inl, best_idx


def draw_ellipse(r, c, r_radius, c_radius, shape=None, rotation=0.):
    """skimage.draw.ellipse (0.14-0.18)"""
    center = np.array([r, c])
    radii = np.array([r_radius, c_radius])
    rotation %= np.pi
    r_radius_rot = abs(r_radius * np.cos(rotation)) + c_radius * np.sin(rotation)
    c_radius_rot = r_radius * np.sin(rotation) + abs(c_radius * np.cos(rotation))
    radii_rot = np.array([r_radius_rot, c_radius_rot])
    upper_left = np.ceil(center - radii_rot).astype(int)
    lower_right = np.floor(center + radii_rot).astype(int)
    if shape is not None:
        upper_left = np.maximum(upper_left, np.array([0, 0]))
        lower_right = np.minimum(lower_right, np.array(shape[:2]) - 1)
    shifted_center = center - upper_left
    bounding_shape = lower_right - upper_left + 1
    r_lim, c_lim = np.ogrid[0:float(bounding_shape[0]), 0:float(bounding_shape[1])]
    sin_alpha, cos_alpha = np.sin(rotation), np.cos(rotation)
    rr_, cc_ = r_lim - shifted_center[0], c_lim - shifted_center[1]
    dist = ((rr_ * cos_alpha + cc_ * sin_alpha) / radii[0]) ** 2 + ((rr_ * sin_alpha - cc_ * cos_alpha) / radii[1]) ** 2
    rr, cc = np.nonzero(dist < 1)
    return rr + upper_left[0], cc + upper_left[1]


def _line(r0, c0, r1, c1):
    """skimage.draw.line (Bresenham)"""
    steep = 0; r, c = r0, c0
    dr, dc = abs(r1 - r0), abs(c1 - c0)
    sc = 1 if (c1 - c) > 0 else -1
    sr = 1 if (r1 - r) > 0 else -1
    if dr > dc:
        steep = 1; c, r = r, c; dc, dr = dr, dc; sc, sr = sr, sc
    d = 2 * dr - dc
    rr, cc = [], []
    for _ in range(dc):
        if steep: rr.append(c); cc.append(r)
        else: rr.append(r); cc.append(c)
        while d >= 0:
            r += sr; d -= 2 * dc
        c += sc; d += 2 * dr
    rr.append(r1); cc.append(c1)
    return rr, cc

def _bezier_segment(y0, x0, y1, x1, y2, x2, w, rr, cc):
    """one rational quadratic Bezier segment (Zingl), y = row, x = column; pixels appended to rr, cc"""
    sx, sy = x2 - x1, y2 - y1
    dx, dy, xx, yy = x0 - x2, y0 - y2, x0 - x1, y0 - y1
    xy, cur = xx * sy + yy * sx, xx * sy - yy * sx
    if cur != 0 and w > 0:
        if sx * sx + sy * sy > xx * xx + yy * yy:
            x2 = x0; x0 -= dx; y2 = y0; y0 -= dy; cur = -cur
        xx = 2.0 * (4.0 * w * sx * xx + dx * dx)
        yy = 2.0 * (4.0 * w * sy * yy + dy * dy)
        sx = 1 if x0 < x2 else -1
        sy = 1 if y0 < y2 else -1
        xy = -2.0 * sx * sy * (2.0 * w * xy + dx * dy)
        if cur * sx * sy < 0:
            xx, yy, xy, cur = -xx, -yy, -xy, -cur
        dx = 4.0 * w * (x1 - x0) * sy * cur + xx / 2.0 + xy
        dy = 4.0 * w * (y0 - y1) * sx * cur + yy / 2.0 + xy
        if w < 0.5 and (dy > xy or dx < xy):
            cur = (w + 1.0) / 2.0; w = math.sqrt(w); xy = 1.0 / (w + 1.0)
            sx = math.floor((x0 + 2.0 * w * x1 + x2) * xy / 2.0 + 0.5)
            sy = math.floor((y0 + 2.0 * w * y1 + y2) * xy / 2.0 + 0.5)
            dx = math.floor((w * x1 + x0) * xy + 0.5); dy = math.floor((y1 * w + y0) * xy + 0.5)
            _bezier_segment(y0, x0, dy, dx, sy, sx, cur, rr, cc)
            dx = math.floor((w * x1 + x2) * xy + 0.5); dy = math.floor((y1 * w + y2) * xy + 0.5)
            _bezier_segment(sy, sx, dy, dx, y2, x2, cur, rr, cc)
            return
        err = dx + dy - xy
        while True:
            rr.append(y0); cc.append(x0)
            if x0 == x2 and y0 == y2:
                return
            t1 = 2 * err > dy
            t2 = 2 * (err + yy) < -dy
            if 2 * err < dx or t2:
                y0 += sy; dy += xy; dx += xx; err += dx
            if 2 * err > dx or t1:
                x0 += sx; dx += xy; dy += yy; err += dy
            if not (dy <= xy and dx >= xy):
                break
    r_, c_ = _line(int(y0), int(x0), int(y2), int(x2))
    rr.extend(r_); cc.extend(c_)

def draw_ellipse_perimeter(r_o, c_o, r_radius, c_radius, orientation=0., shape=None):
    """skimage.draw.ellipse_perimeter (0.14-0.18): Zingl's rational Bezier quadrants about the rotated bounding rectangle;
    duplicate pixels are kept, as there"""
    rr, cc = [], []
    rd, cd = r_radius * r_radius, c_radius * c_radius
    if orientation == 0:
        c, r = -c_radius, 0; e2 = rd; err = c * (2 * e2 + c) + e2
        while c <= 0:
            rr += [r_o + r, r_o + r, r_o - r, r_o - r]; cc += [c_o - c, c_o + c, c_o + c, c_o - c]
            e2 = 2 * err
            if e2 >= (2 * r + 1) * cd:
                r += 1; err += (2 * r + 1) * cd
            if e2 <= (2 * c + 1) * rd:
                c += 1; err += (2 * c + 1) * rd
        while r < r_radius:
            r += 1; rr += [r_o + r, r_o - r]; cc += [c_o, c_o]
    else:
        s = math.sin(orientation)
        za = (cd - rd) * s
        ca = math.sqrt(cd - za * s); ra = math.sqrt(rd + za * s)
        a = ca + 0.5; b = ra + 0.5
        za = za * a * b / (ca * ra)
        ir0, ic0, ir1, ic1 = int(r_o - b), int(c_o - a), int(r_o + b), int(c_o + a)
        ca, ra = ic1 - ic0, ir1 - ir0
        za = 4 * za * math.cos(orientation)
        w = ca * ra
        if w != 0:
            w = (w - za) / (w + w)
        icd, ird = int(math.floor(ca * w + 0.5)), int(math.floor(ra * w + 0.5))
        _bezier_segment(ir0 + ird, ic0, ir0, ic0, ir0, ic0 + icd, 1 - w, rr, cc)
        _bezier_segment(ir0 + ird, ic0, ir1, ic0, ir1, ic1 - icd, w, rr, cc)
        _bezier_segment(ir1 - ird, ic1, ir1, ic1, ir1, ic1 - icd, 1 - w, rr, cc)
        _bezier_segment(ir1 - ird, ic1, ir0, ic1, ir0, ic0 + icd, w, rr, cc)
    rr, cc = np.array(rr, dtype=np.intp), np.array(cc, dtype=np.intp)
    if shape is not None:
        keep = (rr >= 0) & (rr < shape[0]) & (cc >= 0) & (cc < shape[1])
        rr, cc = rr[keep], cc[keep]
    return rr, cc


def disk(radius):
    """skimage.morphology.disk"""
    L = np.arange(-radius, radius + 1)
    X, Y = np.meshgrid(L, L)
    return np.array((X ** 2 + Y ** 2) <= radius ** 2, dtype=np.uint8)


def _shift(selem, shift):
    m, n = selem.shape
    if m % 2 == 0:
        row = np.zeros((1, n), selem.dtype)
        selem = np.vstack((selem, row) if shift else (row, selem))
        m += 1
    if n % 2 == 0:
        col = np.zeros((m, 1), selem.dtype)
        selem = np.hstack((selem, col) if shift else (col, selem))
    return selem


def opening(image, selem):
    """skimage.morphology.opening (0.16-0.18): an even footprint side pads the image by side - 1 with its edge values"""
    image = np.asarray(image)
    pad = [(s - 1, s - 1) if s % 2 == 0 else (0, 0) for s in selem.shape]
    padded = np.pad(image, pad, mode='edge')
    eroded = ndimage.grey_erosion(padded, footprint=_shift(selem, False))
    out = ndimage.grey_dilation(eroded, footprint=_shift(selem, True)[::-1, ::-1])
    return out[pad[0][0]:out.shape[0] - pad[0][1], pad[1][0]:out.shape[1] - pad[1][1]]
