"""Host composition of the centre detection, shared by tests/test_center_detection_host.py, tests/test_gpu_center_detection.py and
scripts/bench_center_detection.py: the reference's ``compute_points_features`` with the oracle's label counts and Ray tracer,
scikit-learn's predict and scikit-learn's DBSCAN.

``label_histograms_positions`` is oracle.label_histograms_positions (the crop-and-disc counts of compute_label_hist_segm) in a
form fast enough for whole images: per label, prefix sums along every row, and per disc row the count between its clipped ends.
The host tests check it against the oracle itself."""
import numpy as np

import oracle


def disc_half_widths(d, dys):
    """w = floor(sqrt(d^2 - dy^2)) for |dy| <= d, in integers: the largest w with dy^2 + w^2 <= d^2"""
    r2 = int(d) * int(d) - np.asarray(dys, dtype=np.int64) ** 2
    w = np.floor(np.sqrt(r2.astype(np.float64))).astype(np.int64)
    w -= (w * w > r2)
    w += ((w + 1) * (w + 1) <= r2)
    return w


def label_disc_counts(segm, positions, diameters, nb_labels):
    """(hist [n_pos, n_diam, nb_labels], sizes [n_pos, n_diam]) of the disc dy^2 + dx^2 <= d^2 about each position, clipped to the
    image; labels outside [0, nb_labels) count in the size only"""
    segm = np.asarray(segm)
    H, W = segm.shape
    pref = np.zeros((nb_labels, H, W + 1), dtype=np.int32)
    chunk = max(1, (1 << 24) // (H * W))
    for lb in range(0, nb_labels, chunk):
        labels = np.arange(lb, min(lb + chunk, nb_labels))[:, None, None]
        pref[lb:lb + chunk, :, 1:] = np.cumsum(segm[None] == labels, axis=2, dtype=np.int32)
    hist = np.zeros((len(positions), len(diameters), nb_labels))
    sizes = np.zeros((len(positions), len(diameters)))
    for i, (py, px) in enumerate(positions):
        for j, d in enumerate(diameters):
            if d < 0:
                continue
            dys = np.arange(max(-d, -py), min(d, H - 1 - py) + 1)
            if not len(dys):
                continue
            w = disc_half_widths(d, dys)
            x0, x1 = np.maximum(px - w, 0), np.minimum(px + w, W - 1)
            keep = x0 <= x1
            ys, x0, x1 = py + dys[keep], x0[keep], x1[keep]
            sizes[i, j] = float(np.sum(x1 - x0 + 1))
            hist[i, j] = (pref[:, ys, x1 + 1] - pref[:, ys, x0]).sum(axis=1, dtype=np.int64)
    return hist, sizes


def label_histograms_positions(segm, positions, diameters, nb_labels=None):
    """oracle.label_histograms_positions for a label map: the ring counts over the ring sizes, per position"""
    segm = np.asarray(segm)
    nb_labels = int(segm.max()) + 1 if nb_labels is None else int(nb_labels)
    pos = [[int(p) for p in q] for q in positions]
    hist, sizes = label_disc_counts(segm, pos, list(diameters), nb_labels)
    ring_size = np.diff(np.concatenate([np.zeros((len(pos), 1)), sizes], axis=1), axis=1)
    ring_hist = np.diff(np.concatenate([np.zeros((len(pos), 1, nb_labels)), hist], axis=1), axis=1)
    return (ring_hist / ring_size[:, :, None]).reshape(len(pos), -1)


def ray_tracer(seg_binary, position, angle_step=5., edge='up'):
    """a drop-in for descriptors.cython_ray_features_seg2d tracing every position with the oracle"""
    e = {'down': -1, 'up': 1}[edge]
    pos = np.atleast_2d(np.array(position, dtype=np.int32))
    rays = np.array([oracle.ray_features2d(seg_binary, p, angle_step, e) for p in pos], dtype=np.float32)
    return rays[0] if np.ndim(position) == 1 else rays


def device_hists_on_host(segm, positions, nb_labels, diameters=None, struc_elem=None):
    """a drop-in for descriptors._device_label_hists (label maps and discs) on the host"""
    lab = np.array(segm, dtype=float)
    lab[np.isnan(lab)] = -1
    return label_disc_counts(lab.astype(np.int64), [[int(p) for p in q] for q in np.atleast_2d(positions)], list(diameters), int(nb_labels))


def points_features(segm, points, params):
    """run_center_candidate_training.py:400-448 on the host: the oracle's ring histograms and Ray tracer, numpy's shift"""
    from pyimsegm_b200 import descriptors as ds
    features, names = np.empty((len(points), 0)), []
    if params.get('fts_hist_diams') is not None:
        diams = params['fts_hist_diams']
        nb = int(np.asarray(segm).max()) + 1
        features = np.hstack((features, label_histograms_positions(segm, points, diams, nb)))
        names += ['hist-d_%i-lb_%i' % (d, lb) for d in diams for lb in range(nb)]
    if params.get('fts_ray_step') is not None:
        step, rays_all, names_ray = params['fts_ray_step'], [], []
        closer = bool(params.get('fts_ray_closer')) and len(params['fts_ray_types']) > 1
        pos = [tuple(map(int, p)) for p in points]
        for edge, border in params['fts_ray_types']:
            mask = np.isin(np.asarray(segm), list(border))
            rays = np.atleast_2d(ray_tracer(mask, np.asarray(pos), step, edge))
            rows = []
            for ray in rays:
                ray = ds._smooth_rays(ray, params['fts_ray_smooth'])
                rows.append(ray if closer else ds.shift_ray_features(ray)[0])
            names_ray = ['ray-lb_%s-agl_%i' % (''.join(map(str, border)), int(a)) for a in np.linspace(0, 360 - step, rays.shape[1])]
            if closer:
                rays_all.append(np.array(rows))
            else:
                features = np.hstack((features, np.array(rows)))
                names += names_ray
        if closer:
            features = np.hstack((features, np.array([ds.shift_ray_features(r)[0] for r in np.min(np.array(rays_all), axis=0)])))
            names += names_ray
    return features, names


def cluster_center_candidates(points, max_dist=100, min_samples=1):
    """run_center_clustering.py:61-83: scikit-learn's DBSCAN and np.mean per cluster"""
    from sklearn import cluster
    points = np.array(points)
    if not list(points):
        return points, []
    labels = cluster.DBSCAN(eps=max_dist, min_samples=min_samples).fit(points).labels_.copy()
    centers = [np.mean(points[labels == i], axis=0) for i in range(max(labels) + 1) if np.any(labels == i)]
    return np.array(centers), labels


def detect_center_candidates_points(img, segm, classif, params):
    """the host composition of center_detection.detect_center_candidates_points (the SLIC and its centres from the device, as
    both sides share them): oracle features, scikit-learn predict, scikit-learn DBSCAN"""
    from pyimsegm_b200 import superpixels as spx
    slic = spx.segment_slic_img2d(img, params['slic_size'], params['slic_regul'])
    points = spx.superpixel_centers(slic)
    features, _ = points_features(segm, points, params)
    mask = np.asarray(classif.predict(features)) == 1
    centres, labels = cluster_center_candidates(np.asarray(points)[mask], params['DBSCAN_max_dist'], params['DBSCAN_min_samples'])
    return np.asarray(points), features, mask, centres, labels
