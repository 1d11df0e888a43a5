"""
Object-centre detection on the GPU: the third pipeline of the reference (experiments_ovary_centres).

Superpixels on the image, point features at every superpixel centre (label histograms in concentric rings and Ray features of
a segmentation), a classifier marking centre candidates, and DBSCAN clustering of the candidates into one centre per cluster.
The names, arguments, ``params`` keys and return values are those of ``run_center_candidate_training.py``
(``estim_points_compute_features`` :378-397, ``compute_points_features`` :400-448, ``label_close_points`` :456-476) and
``run_center_clustering.py`` (``cluster_center_candidates`` :61-83).  The centres feed region growing (``region_growing``) and
ellipse fitting (``ellipse_fitting``).

Device work: the SLIC and the superpixel centres (``superpixels``), the ring histograms (``isb_ring_label_hist``, from run-length
rows of the label map), one Ray trace per ray type (``isb_ray_features_2d``), the classifier when ``class_models.compile_model``
takes it, and DBSCAN with the cluster means (``isb_dbscan``).  The Ray shift stays numpy's FFT on the host: the table is
[N, ~50] and its bits are numpy's.  The DBSCAN labels are scikit-learn's KD-tree labels (scikit-learn's own choice from 12 points
up); for fewer points scikit-learn measures brute-force distances, which may judge a pair a rounding away from eps otherwise
(see :func:`cluster_center_candidates`).
"""
import logging

import numpy as np

from . import descriptors as seg_fts
from . import superpixels as seg_spx
from .engine import get_engine
from .utilities import ImageDimensionError

#: the reference's defaults of the centre-candidate experiment (run_center_candidate_training.py:86-109), without its paths
CENTER_PARAMS = {
    'slic_size': 25,
    'slic_regul': 0.3,
    'fts_hist_diams': [10, 50, 100, 200, 300],
    'fts_ray_step': 15,
    'fts_ray_types': [('up', [0])],
    'fts_ray_closer': True,
    'fts_ray_smooth': 0,
    'pca_coef': None,
    'balance': 'unique',
    'classif': 'RandForest',
    'nb_classif_search': 50,
    'dict_relabel': None,
    'center_dist_thr': 50,
}
#: run_center_clustering.py:46-49
CLUSTER_PARAMS = {
    'DBSCAN_max_dist': 50,
    'DBSCAN_min_samples': 1,
}


def _ray_blocks(segm, points, params):
    """the Ray-feature blocks of ``params['fts_ray_types']``: [(table [N, n_angles], names)], one device trace per type.  With
    ``fts_ray_closer`` and more than one type, a single block: per angle the nearest boundary over the types, shifted afterwards
    (the names are those of the last type)."""
    types = list(params['fts_ray_types'])
    nearest = bool(params.get('fts_ray_closer', False)) and len(types) > 1
    traced = [seg_fts.compute_ray_features_positions(segm, points, angle_step=params['fts_ray_step'], edge=edge, border_labels=border,
                                                     smooth_ray=params['fts_ray_smooth'], shifting=not nearest)
              for edge, border in types]
    if not nearest:
        return [(rays, names) for rays, _, names in traced]
    closest = np.min(np.array([rays for rays, _, _ in traced]), axis=0)
    return [(np.array([seg_fts.shift_ray_features(row)[0] for row in closest]), traced[-1][2])]


def compute_points_features(segm, points, params):
    """ point features of a segmentation (reference run_center_candidate_training.py:400-448): for ``params['fts_hist_diams']``
    the label histograms in the rings between consecutive discs about each point (every disc of every point in one launch over the
    run-length rows of the label map), then for ``params['fts_ray_step']`` the Ray features of each ``fts_ray_types`` entry
    ``(edge, border_labels)``, smoothed by ``fts_ray_smooth`` and rotated to their dominant direction.  A missing or None
    ``fts_hist_diams`` / ``fts_ray_step`` leaves that group out.

    :param ndarray segm: label map [H, W]
    :param points: [N, 2] (row, col) positions; fractional ones are truncated
    :param dict params: the keys above
    :return tuple(ndarray,list(str)): features [N, nb_features] (histogram columns first), their names
    """
    blocks, names = [np.empty((len(points), 0))], []
    if params.get('fts_hist_diams') is not None:
        hist, hist_names = seg_fts.compute_label_histograms_positions(segm, points, diameters=params['fts_hist_diams'])
        blocks.append(hist)
        names += hist_names
    if params.get('fts_ray_step') is not None:
        for rays, ray_names in _ray_blocks(segm, points, params):
            blocks.append(rays)
            names += ray_names
    return np.hstack(blocks), names


def estim_points_compute_features(name, img, segm, params):
    """ superpixel centres of an image as candidate points, and their features (reference run_center_candidate_training.py:378-397):
    the device SLIC of ``params['slic_size']`` / ``params['slic_regul']``, its centres, then :func:`compute_points_features`

    :param str name: passed through
    :param ndarray img: image [H, W, 3] or [H, W]
    :param ndarray segm: label map [H, W] of the same size
    :param dict params: SLIC and feature parameters
    :return tuple: name, superpixels [H, W], centres (list of (row, col)), features [N, nb_features], feature names
    """
    if img.shape[:2] != segm.shape[:2]:
        raise ImageDimensionError('not matching shapes: %r : %r' % (img.shape, segm.shape))
    slic = seg_spx.segment_slic_img2d(img, params['slic_size'], params['slic_regul'])
    centres = seg_spx.superpixel_centers(slic)
    features, names = compute_points_features(segm, centres, params)
    return name, slic, centres, features, names


def compute_min_dist_2_centers(centers, points):
    """ Euclidean distance from every point to its nearest centre, and that centre's index
    (reference run_center_candidate_training.py:325-335)

    :return tuple(ndarray,ndarray): distances [N], indices [N]
    """
    from scipy.spatial.distance import cdist
    table = cdist(np.array(points), np.array(centers))
    return table.min(axis=1), table.argmin(axis=1)


def label_close_points(centers, points, params):
    """ training labels of candidate points (reference run_center_candidate_training.py:456-476).  Given a list of annotated
    (row, col) centres, a point is True when its nearest centre lies within ``params['center_dist_thr']``; given an annotation
    image, a point takes the image's value at its (truncated) pixel; anything else labels every point -1, with a warning.

    :return: labels [N] (bool array, annotation values, or a list of -1)
    """
    if isinstance(centers, list):
        labels = compute_min_dist_2_centers(centers, points)[0] <= params['center_dist_thr']
    elif isinstance(centers, np.ndarray):
        rows, cols = np.array(points, dtype=int).reshape(-1, 2).T
        labels = centers[rows, cols]
    else:
        logging.warning('not relevant centers info of type "%s"', type(centers))
        labels = [-1] * len(points)
    if len(labels) != len(points):
        raise RuntimeError('not equal lengths of points (%i) and labels (%i)' % (len(points), len(labels)))
    return labels


def _dbscan(points, eps, min_samples):
    """labels [n] (int64, scikit-learn's ``labels_``) and centres [k, 2] of ``isb_dbscan`` over float64 points [n, 2]"""
    import ctypes as C
    from . import _lib
    pts = np.ascontiguousarray(points, dtype=np.float64)
    n = len(pts)
    eng = get_engine()
    torch = eng.torch
    d_pts = eng.to_device(pts, 'db_points')
    labels = eng.buf('db_labels', (n, ), torch.int32)
    centres = eng.buf('db_centres', (n, 2), torch.float64)
    ws_bytes = eng.lib.isb_dbscan_workspace_bytes(n)
    ws = eng.buf('db_ws', (ws_bytes, ), torch.uint8)
    k = C.c_int(0)
    _lib.check(eng.lib.isb_dbscan(_lib.ptr(d_pts), n, float(eps), int(min_samples), _lib.ptr(labels), _lib.ptr(centres), C.byref(k),
                                  _lib.ptr(ws), ws_bytes, _lib.stream_ptr()))
    return eng.to_host(labels).astype(np.intp), eng.to_host(centres[:k.value]).copy()


def cluster_center_candidates(points, max_dist=100, min_samples=1):
    """ one centre per dense group of candidate points (reference run_center_clustering.py:61-83): the labels of
    ``sklearn.cluster.DBSCAN(eps=max_dist, min_samples=min_samples)`` and the mean of each cluster's points, both computed on the
    device (``isb_dbscan``).  The labels are scikit-learn's from 12 points up, where it searches a KD-tree and tests
    dx^2 + dy^2 <= eps^2 as the device does; below that it takes brute-force distances through a matrix product, and a pair whose
    distance lies within a rounding of ``max_dist`` may be judged otherwise there.  Any finite points and positive ``max_dist``
    are clustered.

    :param points: [n, 2] candidate positions
    :param float max_dist: the neighbourhood radius (eps)
    :param int min_samples: neighbours (the point itself included) that make a point a core point
    :return tuple(ndarray,ndarray): centres [k, 2] (an empty array when there is no cluster), labels [n] (-1 for noise);
        ``(points, [])`` for no points
    """
    points = np.array(points)
    if not list(points):
        return points, []
    if points.ndim != 2 or points.shape[1] != 2:
        raise ValueError('points have to be (row, col) pairs, got shape %r' % (points.shape, ))
    if not np.isfinite(points.astype(np.float64)).all():
        raise ValueError('Input X contains NaN or infinity.')
    if not max_dist > 0:
        raise ValueError('The \'eps\' parameter of DBSCAN must be a float in the range (0.0, inf). Got %r instead.' % (max_dist, ))
    if int(min_samples) != min_samples or min_samples < 1:
        raise ValueError('The \'min_samples\' parameter of DBSCAN must be an int in the range [1, inf). Got %r instead.' % (min_samples, ))
    labels, centres = _dbscan(points, max_dist, min_samples)
    return (centres if len(centres) else np.array([])), labels


def _predict(classif, features):
    """``classif.predict(features)``: on the device when ``class_models.compile_model`` takes the model as a forest (predict_proba
    there equals scikit-learn's bit for bit, and predict is the class of its first maximum, as the forest's predict), else on the
    host"""
    from .class_models import compile_model
    cm = compile_model(classif)
    if cm is None or cm.kind != 'forest' or cm.classes_ is None or cm.n_features_in != features.shape[1]:
        return np.asarray(classif.predict(features))
    return np.asarray(cm.classes_).take(np.argmax(cm.predict_proba(features), axis=1), axis=0)


def detect_center_candidates_points(img, segm, classif, params):
    """ the prediction of centre candidates and their clustering for one image (run_center_prediction.py:72-85 through
    ``detect_center_candidates`` and ``cluster_points_draw_export``, without their file and figure exports)

    :param ndarray img: image [H, W, 3] or [H, W]
    :param ndarray segm: segmentation [H, W] (label map)
    :param classif: fitted classifier of the point features (a label 1 marks a candidate)
    :param dict params: ``slic_size``, ``slic_regul``, the ``fts_*`` keys, ``DBSCAN_max_dist`` and ``DBSCAN_min_samples``
    :return tuple: points [N, 2] (superpixel centres), features [N, F], candidate mask [N] (bool), centres [k, 2],
        cluster labels of the candidates [n_candidates]
    """
    _, _, points, features, _ = estim_points_compute_features('', img, segm, params)
    labels = _predict(classif, features)
    mask = np.asarray(labels) == 1
    candidates = np.asarray(points)[mask]
    centres, clust_labels = cluster_center_candidates(candidates, max_dist=params.get('DBSCAN_max_dist', CLUSTER_PARAMS['DBSCAN_max_dist']),
                                                      min_samples=params.get('DBSCAN_min_samples', CLUSTER_PARAMS['DBSCAN_min_samples']))
    return np.asarray(points), features, mask, centres, clust_labels
