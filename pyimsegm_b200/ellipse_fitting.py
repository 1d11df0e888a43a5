"""
Ellipse fitting of egg segmentation on the GPU.

Mirror of the reference module ``imsegm/ellipse_fitting.py`` (same public names, arguments, return types and exceptions).  The
RANSAC trials of :func:`ransac_segm` -- the direct fit of the samples, the distance of every boundary point to the ellipse and the
segmentation criterion over the superpixel centres -- run as one launch of ``isb_ellipse_ransac``, one CTA per trial; the samples
are drawn on the host from the global numpy RNG in the reference's order, so a seed gives the reference's samples.  The single-model
calls (``estimate``, ``residuals``, ``criterion``, the final refit) run through the same kernel as a batch of one, so they return the
same bits as the trial that used the same model.

Where the reference inherits from scikit-image (``EllipseModel``, ``draw.ellipse``, ``morphology.disk`` / ``opening``) this module
restates the behaviour of scikit-image 0.14-0.18 as recalled; two differences are deliberate:

* the eigenvector of the direct fit has no defined sign (skimage keeps whichever LAPACK's QR sweeps return); here it is fixed so
  that ``params[2] <= params[3]``.  The other sign describes the same ellipse with the semi-axes swapped and theta moved by pi / 2.
* ``residuals`` runs safeguarded Newton steps on the ellipse angle from skimage's start angle instead of scipy ``leastsq``; both
  converge to a stationary point of the distance, and agree to the solver tolerance, not bit for bit.
"""
import numpy as np
from scipy import ndimage, spatial

from . import _lib
from .descriptors import binary_opening_disk, cython_ray_features_seg2d, reconstruct_ray_features_2d, reduce_close_points
from .engine import get_engine
from .superpixels import make_graph_segm_connect_grid2d_conn4, segment_slic_img2d, superpixel_centers

#: define minimal size of estimated ellipse
MIN_ELLIPSE_DAIM = 25.
#: define maximal Figure size in larger dimension
MAX_FIGURE_SIZE = 14
#: smoothing background with morphological operation
STRUC_ELEM_BG = 15
#: smoothing foreground with morphological operation
STRUC_ELEM_FG = 5


def _label_terms(weights, labels, table_prob):
    """the reference's criterion checks (ellipse_fitting.py:107-119) and the per-label term weights[l] * (q0[l] - q1[l]); a class
    beyond the weights gets NaN, which :func:`_check_criteria` turns into the IndexError the reference raises when such a label
    falls inside an ellipse"""
    if not len(weights) == len(labels):
        raise ValueError('different sizes for weights %i and labels %i' % (len(weights), len(labels)))
    table_prob = np.array(table_prob)
    if 1 in (table_prob.ndim, table_prob.shape[0]):
        if table_prob.shape[0] == 1:
            table_prob = table_prob[0]
        table_prob = np.array([table_prob, 1. - table_prob])
    if table_prob.shape[0] != 2:
        raise ValueError('table shape %r' % (table_prob.shape, ))
    labels = np.asarray(labels)
    if np.max(labels) >= table_prob.shape[1]:
        raise ValueError('labels (%i) exceed the table %r' % (np.max(labels), table_prob.shape))
    if np.min(labels) < 0:
        raise ValueError('negative label %i' % np.min(labels))
    table_q = -np.log(table_prob)
    weights = np.asarray(weights, dtype=np.float64)
    n_w = min(len(weights), table_q.shape[1])
    # weights are indexed by LABEL, not by point (ellipse_fitting.py:137)
    term = np.full(table_q.shape[1], np.nan)
    term[:n_w] = weights[:n_w] * (table_q[0, :n_w] - table_q[1, :n_w])
    return term


def _check_criteria(ok, crit, term, n_weights):
    """raise the reference's IndexError when a label without a weight fell inside a fitted ellipse"""
    if n_weights < len(term) and not np.isnan(term[:n_weights]).any() and np.isnan(np.asarray(crit)[np.asarray(ok) == 1]).any():
        raise IndexError('a label inside the ellipse has no weight (%i weights)' % n_weights)


def _run_trials(point_sets, trial_centre, samples=None, params=None, crit_input=None, thr=0., want_resid=False):
    """one launch of isb_ellipse_ransac; returns host arrays (ok, params, n_inliers, criterion, residuals or None)"""
    eng = get_engine()
    torch = eng.torch
    T = len(trial_centre)
    sizes = np.array([len(p) for p in point_sets], dtype=np.int64)
    pt_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    pts = np.concatenate([np.asarray(p, dtype=np.float64).reshape(-1, 2) for p in point_sets] + [np.zeros((1, 2))])
    trial_centre = np.asarray(trial_centre, dtype=np.int32)
    d = lambda a: eng.to_device(np.ascontiguousarray(a))  # noqa: E731
    d_pts, d_off, d_tc = d(pts), d(pt_off), d(trial_centre)
    d_so = d_si = d_par = None
    if params is not None:
        d_par = d(np.asarray(params, dtype=np.float64).reshape(T, 5))
    else:
        samp_off = np.concatenate([[0], np.cumsum([len(s) for s in samples])]).astype(np.int32)
        samp_idx = np.concatenate([np.asarray(s, dtype=np.int32) for s in samples] + [np.zeros(1, np.int32)])
        d_so, d_si = d(samp_off), d(samp_idx)
    N, d_sp, d_lab, d_term = 0, None, None, None
    if crit_input is not None:
        sp_pts, sp_lab, term = crit_input
        N = len(sp_lab)
        d_sp, d_lab, d_term = d(np.asarray(sp_pts, dtype=np.float64).reshape(-1, 2)), d(np.asarray(sp_lab, dtype=np.int32)), d(term)
    ok = torch.empty(T, dtype=torch.int32, device=eng.device)
    par = torch.empty((T, 5), dtype=torch.float64, device=eng.device)
    n_inl = torch.empty(T, dtype=torch.int32, device=eng.device)
    crit = torch.empty(T, dtype=torch.float64, device=eng.device)
    resid = d_roff = None
    if want_resid:
        roff = np.concatenate([[0], np.cumsum(sizes[trial_centre])]).astype(np.int64)
        resid = torch.empty(max(int(roff[-1]), 1), dtype=torch.float64, device=eng.device)
        d_roff = d(roff[:-1])
    _lib.check(eng.lib.isb_ellipse_ransac(T, _lib.ptr(d_tc), _lib.ptr(d_so), _lib.ptr(d_si), _lib.ptr(d_par), len(point_sets), _lib.ptr(d_pts),
                                          _lib.ptr(d_off), float(thr), _lib.ptr(d_sp), _lib.ptr(d_lab), _lib.ptr(d_term), N, _lib.ptr(ok),
                                          _lib.ptr(par), _lib.ptr(n_inl), _lib.ptr(crit), _lib.ptr(resid), _lib.ptr(d_roff), _lib.stream_ptr()))
    out = [eng.to_host(x).copy() for x in (ok, par, n_inl, crit)]
    out.append(eng.to_host(resid).copy() if want_resid else None)
    return out


class EllipseModelSegm(object):
    """Total least squares estimator for 2D ellipses, with the segmentation criterion of the reference.

    The interface of skimage's ``EllipseModel``: ``params = (xc, yc, a, b, theta)``, ``estimate(data) -> bool``,
    ``predict_xy(t, params=None)``, ``residuals(data)``; the functional model is::

        xt = xc + a*cos(theta)*cos(t) - b*sin(theta)*sin(t)
        yt = yc + a*sin(theta)*cos(t) + b*cos(theta)*sin(t)

    ``estimate``, ``residuals`` and ``criterion`` run on the GPU (``isb_ellipse_ransac``, a batch of one).
    """

    def __init__(self):
        self.params = None

    @staticmethod
    def _check_data(data):
        data = np.asarray(data, dtype=np.float64)
        if data.ndim != 2 or data.shape[1] != 2:
            raise ValueError('Input data must have shape (N, 2).')
        return data

    def estimate(self, data):
        """direct least-squares fit (Halir-Flusser); False when not exactly one eigenvector satisfies 4ac - b^2 > 0

        :raises numpy.linalg.LinAlgError: the scatter matrix of the linear terms is singular (as numpy's ``inv`` inside skimage)
        """
        data = self._check_data(data)
        ok, par, _, _, _ = _run_trials([data], [0], samples=[np.arange(len(data))])
        if ok[0] < 0:
            raise np.linalg.LinAlgError('Singular matrix')
        if ok[0] == 0:
            return False
        self.params = [float(v) for v in par[0]]
        return True

    def predict_xy(self, t, params=None):
        """points on the ellipse at angles ``t``: [..., 2]"""
        xc, yc, a, b, theta = self.params if params is None else params
        t = np.asarray(t)
        ct, st = np.cos(t), np.sin(t)
        ctheta, stheta = np.cos(theta), np.sin(theta)
        x = xc + a * ctheta * ct - b * stheta * st
        y = yc + a * stheta * ct + b * ctheta * st
        return np.concatenate((x[..., None], y[..., None]), axis=t.ndim)

    def residuals(self, data):
        """distance of every point to the ellipse (the stationary point reached from skimage's start angle)"""
        data = self._check_data(data)
        if not len(data):
            return np.zeros(0)
        return _run_trials([data], [0], params=[self.params], want_resid=True)[4][:len(data)]

    def criterion(self, points, weights, labels, table_prob=(0.1, 0.9)):
        """ sum over the points inside the ellipse of ``weights[label] * (-log p_fg[label] + log p_bg[label])``

        Note that ``weights`` is indexed by the LABEL of a point, not by the point (as the reference does, ellipse_fitting.py:137).

        :param points: points coordinates
        :param weights: weight for each point represent the region size
        :param labels: vector of labels for each point
        :param table_prob: vector of foreground probabilities per class (background is its supplement to 1), or a matrix
            whose first row is the foreground and second the background probability
        :return float:
        """
        if not len(points) == len(weights) == len(labels):
            raise ValueError('different sizes for points %i and weights %i and labels %i' % (len(points), len(weights), len(labels)))
        term = _label_terms(weights, labels, table_prob)
        crit_in = (np.asarray(points, dtype=np.float64), np.asarray(labels), term)
        crit = _run_trials([np.zeros((0, 2))], [0], params=[self.params], crit_input=crit_in)[3]
        _check_criteria([1], crit, term, len(weights))
        return float(crit[0])


def _device_model(model_class):
    return all(getattr(model_class, m) is getattr(EllipseModelSegm, m) for m in ('estimate', 'residuals', 'criterion'))


def _check_ransac_args(points, min_samples, max_trials):
    if isinstance(min_samples, float):
        if not 0 < min_samples <= 1:
            raise ValueError("`min_samples` as ration must be in range (0, 1]")
        min_samples = int(min_samples * len(points))
    if not 0 < min_samples <= len(points):
        raise ValueError("`min_samples` must be in range (0, <nb-samples>]")
    if max_trials < 0:
        raise ValueError("`max_trials` must be greater than zero")
    return min_samples


def _select(ok, n_inl, crit):
    """the reference's sequential rule (ellipse_fitting.py:228-254) over the trials of one centre: the trial indices of the best
    model and of the mask kept as inliers (None when no trial succeeded)"""
    best, best_fit, inl_trial, best_num = None, np.inf, None, 0
    for t in range(len(ok)):
        if ok[t] < 0:
            raise np.linalg.LinAlgError('Singular matrix')
        if ok[t] == 0:
            continue
        if crit[t] < best_fit:
            best, best_fit = t, crit[t]
            if n_inl[t] > best_num:
                inl_trial, best_num = t, n_inl[t]
    return best, inl_trial


def ransac_segm_centres(points_centers, model_class, points_all, weights, labels, table_prob, min_samples, residual_threshold=1,
                        max_trials=100):
    """ :func:`ransac_segm` for every centre: the list ``[ransac_segm(points, ...) for points in points_centers]`` returns, from the
    same draws of the global numpy RNG (centre by centre, trial by trial).  Every trial of every centre is evaluated in one launch,
    and the final refits of all centres in a second one.

    :return list(tuple(EllipseModelSegm,ndarray)): (model or None, inlier mask or None) per centre
    """
    if not _device_model(model_class):
        return [ransac_segm(p, model_class, points_all, weights, labels, table_prob, min_samples, residual_threshold, max_trials)
                for p in points_centers]
    if not len(points_all) == len(weights) == len(labels):
        raise ValueError('different sizes for points %i and weights %i and labels %i' % (len(points_all), len(weights), len(labels)))
    point_sets = [np.array(p, dtype=np.float64).reshape(len(p), -1) for p in points_centers]
    trial_centre, samples = [], []
    for c, pts in enumerate(point_sets):
        n_smp = _check_ransac_args(pts, min_samples, max_trials)
        for _ in range(max_trials):
            samples.append(np.random.choice(len(pts), n_smp, replace=False))
            trial_centre.append(c)
    results = [(None, None)] * len(point_sets)
    if not trial_centre:
        return results
    term = _label_terms(weights, labels, table_prob)
    crit_in = (np.asarray(points_all, dtype=np.float64), np.asarray(labels), term)
    ok, par, n_inl, crit, resid = _run_trials(point_sets, trial_centre, samples=samples, crit_input=crit_in, thr=residual_threshold,
                                               want_resid=True)
    _check_criteria(ok, crit, term, len(weights))
    sizes = np.array([len(p) for p in point_sets])
    roff = np.concatenate([[0], np.cumsum(sizes[np.asarray(trial_centre)])])
    refit_sets, refit_centre, refit_of = [], [], []
    t0 = 0
    for c, pts in enumerate(point_sets):
        sl = slice(t0, t0 + max_trials)
        best, inl_trial = _select(ok[sl], n_inl[sl], crit[sl])
        if best is not None:
            model = model_class()
            model.params = [float(v) for v in par[t0 + best]]
            inliers = None
            if inl_trial is not None:
                r0 = roff[t0 + inl_trial]
                inliers = np.abs(resid[r0:r0 + len(pts)]) < residual_threshold
                refit_sets.append(pts[inliers])
                refit_centre.append(len(refit_centre))
                refit_of.append(c)
            results[c] = (model, inliers)
        t0 += max_trials
    if refit_sets:
        ok_f, par_f, _, _, _ = _run_trials(refit_sets, refit_centre, samples=[np.arange(len(s)) for s in refit_sets])
        for k, c in enumerate(refit_of):
            if ok_f[k] < 0:
                raise np.linalg.LinAlgError('Singular matrix')
            if ok_f[k] == 1:
                results[c][0].params = [float(v) for v in par_f[k]]
    return results


def ransac_segm(points, model_class, points_all, weights, labels, table_prob, min_samples, residual_threshold=1, max_trials=100):
    """ Fit a model to points with the RANSAC (random sample consensus); the model is judged by its ``criterion`` over
    ``points_all`` and the largest consensus set among the improving models is refitted.

    Every trial of an :class:`EllipseModelSegm` runs in one launch; another ``model_class`` runs its own methods trial by trial.

    :param ndarray points: (N, 2) boundary points
    :param class model_class: model with ``estimate``, ``residuals`` and ``criterion``
    :param points_all: superpixel centres
    :param weights: weights, indexed by label
    :param labels: label of each superpixel centre
    :param table_prob: see :meth:`EllipseModelSegm.criterion`
    :param int|float min_samples: number of samples per trial, or its ratio to the number of points
    :param float residual_threshold: maximum distance of an inlier
    :param int max_trials: number of trials
    :return tuple: best model (or None), boolean inlier mask (or None)
    """
    if _device_model(model_class):
        return ransac_segm_centres([points], model_class, points_all, weights, labels, table_prob, min_samples, residual_threshold,
                                   max_trials)[0]
    best_model, best_inlier_num, best_model_fit, best_inliers = None, 0, np.inf, None
    min_samples = _check_ransac_args(points, min_samples, max_trials)
    points = np.array(points)
    for _ in range(max_trials):
        samples = points[np.random.choice(len(points), min_samples, replace=False)]
        model = model_class()
        success = model.estimate(samples)
        if success is not None and not success:
            continue
        model_inliers = np.abs(model.residuals(points)) < residual_threshold
        model_fit = model.criterion(points_all, weights, labels, table_prob)
        sample_inlier_num = np.sum(model_inliers)
        if model_fit < best_model_fit:
            best_model, best_model_fit = model, model_fit
            if sample_inlier_num > best_inlier_num:
                best_inliers, best_inlier_num = model_inliers, sample_inlier_num
    if best_inliers is not None:
        best_model.estimate(points[best_inliers])
    return best_model, best_inliers


def get_slic_points_labels(segm, img=None, slic_size=20, slic_regul=0.1):
    """ SLIC superpixels of the image (or of the segmentation), their centres and the segmentation label at every centre

    :return tuple(ndarray,ndarray,ndarray): superpixels, centres [N, 2] int, labels [N]
    """
    if not img:
        img = segm / float(segm.max())
    slic = segment_slic_img2d(img, sp_size=slic_size, relative_compact=slic_regul)
    slic_centers = np.array(superpixel_centers(slic)).astype(int)
    labels = segm[slic_centers[:, 0], slic_centers[:, 1]]
    return slic, slic_centers, labels


def _draw_ellipse_geometry(r, c, r_radius, c_radius, rotation, shape):
    """clipped bounding box and centre offset of skimage.draw.ellipse (0.14-0.18, as recalled)"""
    center = np.array([r, c])
    rotation %= np.pi
    r_radius_rot = abs(r_radius * np.cos(rotation)) + c_radius * np.sin(rotation)
    c_radius_rot = r_radius * np.sin(rotation) + abs(c_radius * np.cos(rotation))
    radii_rot = np.array([r_radius_rot, c_radius_rot])
    upper_left = np.maximum(np.ceil(center - radii_rot).astype(int), 0)
    lower_right = np.minimum(np.floor(center + radii_rot).astype(int), np.array(shape[:2]) - 1)
    shifted = center - upper_left
    bbox = np.array([upper_left[0], upper_left[1], lower_right[0], lower_right[1]], dtype=np.int32)
    geom = np.array([shifted[0], shifted[1], r_radius, c_radius, np.sin(rotation), np.cos(rotation)], dtype=np.float64)
    return bbox, geom


def add_overlap_ellipse(segm, ellipse_params, label, thr_overlap=1.):
    """ add an ellipse with the given label into the segmentation unless it overlaps an existing object by more than
    ``thr_overlap`` (overlap over the smaller of the two areas); the ellipse is rasterised like skimage.draw.ellipse

    :param ndarray segm: segmentation (modified in place)
    :param tuple ellipse_params: (row, col, row radius, col radius, orientation)
    :param int label: selected label
    :param float thr_overlap: relative overlap with existing objects
    :return ndarray:
    """
    import ctypes as C
    if not ellipse_params:
        return segm
    c1, c2, h, w, phi = ellipse_params
    bbox, geom = _draw_ellipse_geometry(int(c1), int(c2), int(h), int(w), phi, segm.shape)
    n_labels = max(int(np.max(segm)) + 1, 1) if segm.size else 1
    eng = get_engine()
    torch = eng.torch
    d_seg = eng.to_device(np.asarray(segm, dtype=np.int32))
    mask = torch.empty(segm.shape, dtype=torch.uint8, device=eng.device)
    counts = torch.empty(2 * n_labels + 1, dtype=torch.int64, device=eng.device)
    _lib.check(eng.lib.isb_ellipse_overlap(_lib.ptr(d_seg), segm.shape[0], segm.shape[1], n_labels, bbox.ctypes.data_as(C.POINTER(C.c_int32)),
                                           geom.ctypes.data_as(C.POINTER(C.c_double)), _lib.ptr(mask), _lib.ptr(counts), _lib.stream_ptr()))
    cnt = eng.to_host(counts)
    area, overlap, mask_area = cnt[:n_labels], cnt[n_labels:2 * n_labels], int(cnt[-1])
    for lb in range(1, n_labels):
        sizes = [s for s in [int(area[lb]), mask_area] if s > 0]
        if not sizes:
            return segm
        if float(overlap[lb]) / float(min(sizes)) > thr_overlap:
            return segm
    segm[eng.to_host(mask).astype(bool)] = label
    return segm


def split_segm_background_foreground(seg, sel_bg=STRUC_ELEM_BG, sel_fg=STRUC_ELEM_FG):
    """ smoothing segmentation with morphological operation

    :param ndarray seg: input segmentation
    :param int|float sel_bg: smoothing background with morphological operation
    :param int sel_fg: smoothing foreground with morphological operation
    :return tuple(ndarray,ndarray):
    """
    seg_bg = (seg > 0)
    seg_bg = 1 - ndimage.binary_fill_holes(seg_bg)
    if sel_bg > 0:
        seg_bg = binary_opening_disk(seg_bg, sel_bg).astype(seg_bg.dtype)
    seg_fg = (seg == 1)
    if sel_fg > 0:
        seg_fg = binary_opening_disk(seg_fg, sel_fg)
    return seg_bg, seg_fg


def _rays(seg_binary, centers, edge):
    """Ray features of every centre in one launch, [n_centres, 72] float32"""
    return np.atleast_2d(cython_ray_features_seg2d(np.asarray(seg_binary).astype(bool), np.array(centers, dtype=int).reshape(-1, 2), 5., edge))


def prepare_boundary_points_ray_join(seg, centers, close_points=5, min_diam=MIN_ELLIPSE_DAIM, sel_bg=STRUC_ELEM_BG,
                                     sel_fg=STRUC_ELEM_FG):
    """ boundary points about every centre: background and foreground rays, each clipped below at ``min_diam``

    :return list(ndarray):
    """
    seg_bg, seg_fg = split_segm_background_foreground(seg, sel_bg, sel_fg)
    rays_bg, rays_fg = _rays(seg_bg, centers, 'up'), _rays(seg_fg, centers, 'down')
    points_centers = []
    for center, ray_bg, ray_fc in zip(centers, rays_bg, rays_fg):
        ray_bg[ray_bg < min_diam] = min_diam
        points_bg = reduce_close_points(reconstruct_ray_features_2d(center, ray_bg), close_points)
        ray_fc[ray_fc < min_diam] = min_diam
        points_fc = reduce_close_points(reconstruct_ray_features_2d(center, ray_fc), close_points)
        points_centers.append(np.vstack((points_bg, points_fc)))
    return points_centers


def _both_rays(seg, centers, min_diam, sel_bg, sel_fg):
    seg_bg, seg_fc = split_segm_background_foreground(seg, sel_bg, sel_fg)
    rays_bg, rays_fc = _rays(seg_bg, centers, 'up'), _rays(seg_fc, centers, 'down')
    for ray_bg, ray_fc in zip(rays_bg, rays_fc):
        rays = np.array([ray_bg, ray_fc], dtype=float)
        rays[rays < 0] = np.inf
        rays[rays < min_diam] = min_diam
        yield rays


def prepare_boundary_points_ray_edge(seg, centers, close_points=5, min_diam=MIN_ELLIPSE_DAIM, sel_bg=STRUC_ELEM_BG,
                                     sel_fg=STRUC_ELEM_FG):
    """ boundary points about every centre: the closer of the background and foreground edges along each ray

    :return list(ndarray):
    """
    points_centers = []
    for center, rays in zip(centers, _both_rays(seg, centers, min_diam, sel_bg, sel_fg)):
        points_close = reconstruct_ray_features_2d(center, np.min(rays, axis=0))
        points_centers.append(reduce_close_points(points_close, close_points))
    return points_centers


def prepare_boundary_points_ray_mean(seg, centers, close_points=5, min_diam=MIN_ELLIPSE_DAIM, sel_bg=STRUC_ELEM_BG,
                                     sel_fg=STRUC_ELEM_FG):
    """ boundary points about every centre: the mean of the background and foreground edges along each ray (the closer one
    where only one is found)

    :return list(ndarray):
    """
    points_centers = []
    for center, rays in zip(centers, _both_rays(seg, centers, min_diam, sel_bg, sel_fg)):
        ray_min = np.min(rays, axis=0)
        ray_mean = np.mean(rays, axis=0)
        ray_mean[np.isinf(ray_mean)] = ray_min[np.isinf(ray_mean)]
        points_centers.append(reduce_close_points(reconstruct_ray_features_2d(center, ray_mean), close_points))
    return points_centers


def prepare_boundary_points_ray_dist(seg, centers, close_points=1, sel_bg=STRUC_ELEM_BG, sel_fg=STRUC_ELEM_FG):
    """ background-edge points of all centres, each assigned to its closest centre

    :return list(ndarray):
    """
    seg_bg, _ = split_segm_background_foreground(seg, sel_bg, sel_fg)
    points = []
    for center, ray in zip(centers, _rays(seg_bg, centers, 'up')):
        points_bg = reduce_close_points(reconstruct_ray_features_2d(center, ray, 0), close_points)
        points += points_bg.tolist()
    points = np.array(points)
    points[(points < 0) & (points > -1e-3)] = 0.
    close_center = np.argmin(spatial.distance.cdist(points, centers, metric='euclidean'), axis=1)
    return [points[close_center == i] for i in range(close_center.max() + 1)]


def filter_boundary_points(segm, slic):
    """ superpixel centres on the foreground boundary: background superpixels with a non-background neighbour and label-1
    superpixels with a background neighbour (4-connected superpixel graph)

    :return ndarray: centres [M, 2] int
    """
    slic_centers = np.array(superpixel_centers(slic)).astype(int)
    labels = segm[slic_centers[:, 0], slic_centers[:, 1]]
    vertices, edges = make_graph_segm_connect_grid2d_conn4(slic)
    nb_vertices = np.max(vertices) + 1
    nb_labels = labels.max() + 1
    neighbour_labels = np.zeros((nb_vertices, nb_labels))
    edges = np.asarray(edges, dtype=int).reshape(-1, 2)
    np.add.at(neighbour_labels, (edges[:, 0], labels[edges[:, 1]]), 1)
    np.add.at(neighbour_labels, (edges[:, 1], labels[edges[:, 0]]), 1)
    sums = np.tile(np.sum(neighbour_labels, axis=1), (nb_labels, 1)).T
    neighbour_labels = neighbour_labels / sums
    filter_bg = np.logical_and(labels == 0, neighbour_labels[:, 0] < 1)
    filter_fc = np.logical_and(labels == 1, neighbour_labels[:, 0] > 0)
    return slic_centers[np.logical_or(filter_bg, filter_fc)]


def prepare_boundary_points_close(seg, centers, sp_size=25, relative_compact=0.3):
    """ boundary superpixel centres (:func:`filter_boundary_points`) assigned to their closest centre

    :return list(ndarray):
    """
    slic = segment_slic_img2d(seg / float(seg.max()), sp_size=sp_size, relative_compact=relative_compact)
    points_all = filter_boundary_points(seg, slic)
    close_center = np.argmin(spatial.distance.cdist(points_all, centers, metric='euclidean'), axis=1)
    return [points_all[close_center == i] for i in range(int(close_center.max() + 1))]
