"""
oracle -- CPU restatement of the reference's SLIC -> features -> GraphCut path.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this package; nothing under ``pyimsegm_b200/`` does.

Parity status (see DESIGN.md section "Oracle"):
  * descriptors (colour statistics): PINNED -- doctest goldens of imsegm/descriptors.py:218-283,796-813 and the
    reference's own features_cython.pyx compiled unchanged into oracle/_ref.
  * adjacency graph, centroids, edge weights, unary, pairwise: PINNED -- doctest goldens of
    imsegm/superpixels.py:163-168,211-215 and imsegm/graph_cuts.py:311-319,399-413,587-609,687-697.
  * alpha-expansion: pinned on the tiny graphs of imsegm/graph_cuts.py:698-716 only (gco not installed).
  * SLIC label maps: PARITY UNPINNED (scikit-image not installed; the reference pins only the shape).
    Its Gaussian pre-blur is pinned bit-exact against scipy.ndimage, rgb2lab to 1e-12 against a numpy formula.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    """compile oracle/liboracle.so (and oracle/_ref when $IMSEGM_REFERENCE names a checkout of the reference) with the committed Makefile"""
    so = os.path.join(_HERE, 'liboracle.so')
    srcs = [os.path.join(_HERE, f) for f in ('slic_oracle.c', 'slic3d_oracle.c', 'stats_oracle.c', 'gc_oracle.cpp')]
    stale = (not os.path.isfile(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(['make', '-C', _HERE, 'liboracle.so'], stdout=subprocess.DEVNULL)
    ref_dir = os.path.join(_HERE, '_ref')
    has_ref = os.path.isdir(ref_dir) and any(f.startswith('features_cython') for f in os.listdir(ref_dir))
    ref_tree = os.environ.get('IMSEGM_REFERENCE')
    if ref_tree and os.path.isdir(ref_tree) and (force or not has_ref):
        subprocess.call(['make', '-C', _HERE, 'ref', 'REF=' + os.path.abspath(ref_tree)], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, 'liboracle.so')
        if not os.path.isfile(so):
            build()
        _LIB = C.CDLL(so)
        _LIB.oracle_det_cbrt.restype = C.c_double
        _LIB.oracle_det_cbrt.argtypes = [C.c_double]
        _LIB.oracle_det_pow24.restype = C.c_double
        _LIB.oracle_det_pow24.argtypes = [C.c_double]
        _LIB.oracle_enforce_connectivity.restype = C.c_int64
        _LIB.oracle_enforce_connectivity3d.restype = C.c_int64
    return _LIB


def ref_features_cython():
    """the reference's own Cython module compiled unchanged (oracle/_ref), or None when it was not built"""
    import importlib.util
    ref_dir = os.path.join(_HERE, '_ref')
    if not os.path.isdir(ref_dir):
        return None
    for f in os.listdir(ref_dir):
        if f.startswith('features_cython') and f.endswith('.so'):
            spec = importlib.util.spec_from_file_location('features_cython', os.path.join(ref_dir, f))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            return mod
    return None


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


# --------------------------------------------------------------------------------------------------------------------
# SLIC  (imsegm/superpixels.py:22-69 -> skimage.segmentation.slic)
# --------------------------------------------------------------------------------------------------------------------

def gaussian_weights(sigma, truncate=4.0):
    """half kernel [w0, w1..wr] of scipy.ndimage's 1-D Gaussian (order 0): exp(-0.5/sigma^2 x^2) / sum"""
    radius = int(truncate * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    phi = phi / phi.sum()
    return np.ascontiguousarray(phi[radius:]), radius


def regular_grid(shape, n_points):
    """seed grid of skimage.util.regular_grid: per-axis (start, step) for an array of `shape`"""
    shape = np.asarray(shape)
    ndim = len(shape)
    order = np.argsort(np.argsort(shape))
    dims = np.sort(shape)
    space = float(np.prod(shape))
    if space <= n_points:
        return [(0, 1)] * ndim
    steps = np.full(ndim, (space / n_points) ** (1.0 / ndim), dtype=float)
    if (dims < steps).any():
        for d in range(ndim):
            steps[d] = dims[d]
            space = float(np.prod(dims[d + 1:]))
            steps[d + 1:] = (space / n_points) ** (1.0 / (ndim - d - 1))
            if (dims >= steps).all():
                break
    starts = (steps // 2).astype(int)
    steps = np.round(steps).astype(int)
    out = [(int(starts[i]), int(steps[i])) for i in range(ndim)]
    return [out[i] for i in order]


def slic_seeds(H, W, n_segments):
    (_, _), (sy, ty), (sx, tx) = regular_grid((1, H, W), n_segments)
    ys = np.arange(sy, H, ty)
    xs = np.arange(sx, W, tx)
    gy, gx = np.meshgrid(ys, xs, indexing='ij')
    seeds = np.stack([gy.ravel(), gx.ravel()], axis=1).astype(np.float64)
    return np.ascontiguousarray(seeds), ty, tx


def gaussian_blur(img, sigma):
    img = np.ascontiguousarray(img, dtype=np.float64)
    H, W, Cn = img.shape
    w, r = gaussian_weights(sigma)
    out = np.empty_like(img)
    rc = lib().oracle_gaussian_blur(_p(img, C.c_double), H, W, Cn, _p(w, C.c_double), r, _p(out, C.c_double))
    assert rc == 0
    return out


def rgb2lab_scaled(img, ratio=1.0):
    img = np.ascontiguousarray(img, dtype=np.float64)
    out = np.empty_like(img)
    lib().oracle_rgb2lab_scaled(_p(img, C.c_double), C.c_long(img.shape[0] * img.shape[1]), C.c_double(ratio),
                                _p(out, C.c_double))
    return out


def slic_kmeans(lab, n_segments, max_iter=10, slic_zero=False, return_centroids=False):
    lab = np.ascontiguousarray(lab, dtype=np.float64)
    H, W, _ = lab.shape
    seeds, ty, tx = slic_seeds(H, W, n_segments)
    n = len(seeds)
    step = float(max(1, ty, tx))
    labels = np.empty((H, W), dtype=np.int64)
    cent = np.empty((n, 5), dtype=np.float64)
    lib().oracle_slic_kmeans(_p(lab, C.c_double), H, W, _p(seeds, C.c_double), n, int(ty), int(tx), C.c_double(step),
                             int(max_iter), int(bool(slic_zero)), _p(labels, C.c_int64), _p(cent, C.c_double))
    return (labels, cent) if return_centroids else labels


def enforce_connectivity(labels, min_size, max_size):
    labels = np.ascontiguousarray(labels, dtype=np.int64)
    H, W = labels.shape
    out = np.empty_like(labels)
    n = lib().oracle_enforce_connectivity(_p(labels, C.c_int64), H, W, C.c_long(int(min_size)), C.c_long(int(max_size)),
                                          _p(out, C.c_int64))
    assert n >= 0
    return out


def slic(image, n_segments=100, compactness=10., max_iter=10, sigma=0, enforce_conn=True, min_size_factor=0.5,
         max_size_factor=3, slic_zero=False):
    """skimage.segmentation.slic for a 2-D RGB float image in [0, 1] (0.14-0.18 behaviour, labels from 0)"""
    image = np.ascontiguousarray(image, dtype=np.float64)
    H, W, _ = image.shape
    if sigma > 0:
        image = gaussian_blur(image, sigma)
    lab = rgb2lab_scaled(image, 1.0 / compactness)
    labels = slic_kmeans(lab, n_segments, max_iter, slic_zero)
    if enforce_conn:
        segment_size = 1 * H * W / n_segments
        labels = enforce_connectivity(labels, int(min_size_factor * segment_size), int(max_size_factor * segment_size))
    return labels


def segment_slic_img2d(img, sp_size=50, relative_compact=0.1, slico=False):
    """imsegm/superpixels.py:22-69"""
    img = np.asarray(img)
    nb_pixels = np.prod(img.shape[:2])
    if img.ndim == 2:
        img = np.stack([img] * 3, axis=-1)
    lo, hi = img.min(), img.max()
    if lo != 0. or hi != 1.:
        img = (img - lo) / float(hi - lo)
    n_seg = int(nb_pixels / (sp_size ** 2))
    compact = (sp_size * relative_compact) ** 1.5
    return slic(img, n_segments=n_seg, compactness=compact, sigma=1, enforce_conn=True, slic_zero=slico)


# --------------------------------------------------------------------------------------------------------------------
# descriptors  (imsegm/features_cython.pyx, imsegm/descriptors.py:209-296, 787-863)
# --------------------------------------------------------------------------------------------------------------------

def color2d_stat(img, seg, mode, mean=None):
    img = np.ascontiguousarray(img, dtype=np.float32)
    seg = np.ascontiguousarray(seg, dtype=np.int32)
    H, W = seg.shape
    nb = int(seg.max()) + 1
    out = np.zeros((nb, 3), dtype=np.float64)
    m = None
    if mode == 2:
        m = np.ascontiguousarray(mean, dtype=np.float32)
    lib().oracle_color2d_stat(_p(img, C.c_float), _p(seg, C.c_int32), H, W, nb, mode,
                              _p(m, C.c_float) if m is not None else None, _p(out, C.c_double))
    return out


def color2d_mean(img, seg):
    return color2d_stat(img, seg, 0)


def color2d_energy(img, seg):
    return color2d_stat(img, seg, 1)


def color2d_std(img, seg, means=None):
    if means is None:
        means = color2d_mean(img, seg)
    return np.sqrt(color2d_stat(img, seg, 2, means))


def color2d_median(img, seg):
    """imsegm/descriptors.py:420-455 numpy_img2d_color_median: per label and channel, np.median of the member pixels in the image's
    own dtype (a float32 image averages its two middle values in float32, as np.median of the reference's list of float32 values
    does); NaN for a label without pixels and for a label with a NaN pixel"""
    img, seg = np.asarray(img), np.asarray(seg)
    nb = int(seg.max()) + 1
    out = np.full((nb, 3), np.nan)
    for lb in range(nb):
        mask = seg == lb
        if mask.any():
            out[lb] = np.median(img[mask], axis=0)
    return out


def image2d_color_statistic(image, segm, flags):
    """imsegm/descriptors.py:787-863 for the natively computed statistics (mean / std / energy / meanGrad)"""
    image = np.nan_to_num(np.asarray(image))
    cols = []
    mean = None
    if 'mean' in flags:
        mean = color2d_mean(image, segm)
        cols.append(mean)
    if 'std' in flags:
        cols.append(color2d_std(image, segm, mean))
    if 'energy' in flags:
        cols.append(color2d_energy(image, segm))
    if 'median' in flags:
        cols.append(color2d_median(image, segm))
    if 'meanGrad' in flags:
        grad = np.zeros_like(image, dtype=float)
        for i in range(3):
            grad[:, :, i] = np.sum(np.gradient(image[:, :, i]), axis=0)
        cols.append(color2d_mean(grad, segm))
    fts = np.nan_to_num(np.hstack(cols))
    fts[fts == 0] = 0
    return fts


def superpixel_centers(segm):
    segm = np.ascontiguousarray(segm, dtype=np.int32)
    H, W = segm.shape
    nb = int(segm.max()) + 1
    out = np.empty((nb, 2), dtype=np.float64)
    lib().oracle_centroids2d(_p(segm, C.c_int32), H, W, nb, _p(out, C.c_double), None)
    return out


# --------------------------------------------------------------------------------------------------------------------
# graph + energies  (imsegm/superpixels.py:115-177, imsegm/graph_cuts.py:303-336,383-439,523-657)
# --------------------------------------------------------------------------------------------------------------------

def adjacency_edges(grid):
    """4-connected region adjacency: (vertices, edges[E,2]) with a < b, sorted by (b, a)  (superpixels.py:115-177)"""
    grid = np.asarray(grid)
    vertices, inv = np.unique(grid, return_inverse=True)
    g = inv.reshape(grid.shape)
    n = len(vertices)
    pairs = np.concatenate([np.stack([g[:, :-1].ravel(), g[:, 1:].ravel()], 1),
                            np.stack([g[:-1, :].ravel(), g[1:, :].ravel()], 1)])
    pairs = pairs[pairs[:, 0] != pairs[:, 1]]
    pairs.sort(axis=1)
    code = np.unique(pairs[:, 0] + n * pairs[:, 1])
    edges = np.stack([vertices[code % n], vertices[code // n]], 1)
    return vertices, edges


def spatial_dist(centres, edges, relative=False):
    centres = np.nan_to_num(np.asarray(centres, dtype=float))
    d = centres[edges[:, 0]] - centres[edges[:, 1]]
    dist = np.sqrt(np.einsum('ij,ij->i', d, d))
    if relative:
        dist = dist / np.mean(dist)
    return dist


def edge_model(edges, proba, metric='lT'):
    v1, v2 = proba[edges[:, 0]], proba[edges[:, 1]]
    if metric == 'l1':
        dist = np.abs(v1 - v2).sum(axis=1)
    elif metric == 'l2':
        d = v1 - v2
        dist = np.sqrt(np.einsum('ij,ij->i', d, d))
    elif metric == 'lT':
        dist = np.max((v1 - v2) ** 2, axis=1)
    else:
        return np.ones(len(edges))
    return np.exp(-dist / (2 * np.std(dist) ** 2))


def edge_weights(segments, proba=None, edge_type='model', features=None, color_means=None):
    _, edges = adjacency_edges(segments)
    edges = np.array(edges, dtype=np.int32)
    if edge_type.startswith('model'):
        metric = edge_type.split('_')[-1] if '_' in edge_type else 'lT'
        w = edge_model(edges, proba, metric)
    elif edge_type == 'color':
        dist = np.abs(color_means[edges[:, 0]] - color_means[edges[:, 1]]).sum(axis=1)
        w = np.exp(-(dist.astype(float) / (2 * np.std(dist) ** 2)))
    elif edge_type == 'features':
        f = (features - features.mean(axis=0)) / np.where(features.std(axis=0) == 0, 1, features.std(axis=0))
        d = f[edges[:, 0]] - f[edges[:, 1]]
        dist = np.sqrt(np.einsum('ij,ij->i', d, d))
        w = np.exp(-(dist / (2 * np.std(dist) ** 2)))
    else:
        w = np.ones(len(edges))
    w = np.array(w, dtype=float)
    if edge_type in ('model', 'features', 'color', 'spatial'):
        w /= spatial_dist(superpixel_centers(segments), edges, relative=True)
    w[w < 1e-3] = 1e-3
    w[w > 1e3] = 1e3
    return edges, w


def unary_cost(proba, min_prob=0.01):
    p = np.clip(proba, min_prob, 1 - min_prob)
    return np.abs(-np.log(p))


def pairwise_cost(gc_regul, nb_classes, max_cost=1e5):
    pw = (np.ones(nb_classes) - np.eye(nb_classes)) * gc_regul
    pw = np.array(pw, dtype=np.float64)
    pw[pw > max_cost] = max_cost
    return pw


def integerise(edge_w, unary, pairwise):
    """pyGCO cut_general_graph float path: returns int32 (w, unary, pairwise).  A NaN edge weight (degenerate edge model, DESIGN.md
    section 2) is left out of the down-weight factor and becomes 0, where pyGCO's C cast is undefined; no edge at all is accepted"""
    edge_w = np.asarray(edge_w, dtype=float)
    ok = ~np.isnan(edge_w)
    dwf = max(np.abs(unary).max(), (np.abs(edge_w[ok]).max() if ok.any() else 0.) * pairwise.max()) + 1e-10
    u = (unary / dwf * 100000).astype(np.intc)
    w = (np.where(ok, edge_w, 0.) / dwf * 1000).astype(np.intc)
    v = (pairwise * 100).astype(np.intc)
    return w, u, v


def alpha_expansion_int(edges, w, unary, pairwise, n_iter=-1, return_energy=False, init=None):
    """``init``: starting labeling [N] (pyGCO's init_labels); all zeros when None"""
    edges = np.ascontiguousarray(edges, dtype=np.int32).reshape(-1, 2)
    w = np.ascontiguousarray(w, dtype=np.int32)
    unary = np.ascontiguousarray(unary, dtype=np.int32)
    pairwise = np.ascontiguousarray(pairwise, dtype=np.int32)
    N, K = unary.shape
    labels = np.zeros(N, dtype=np.int32) if init is None else np.array(init, dtype=np.int32).reshape(N)
    energy = C.c_int64(0)
    moves = C.c_int(0)
    lib().oracle_alpha_expansion(N, K, len(edges), _p(edges, C.c_int32), _p(w, C.c_int32), _p(unary, C.c_int32),
                                 _p(pairwise, C.c_int32), int(n_iter), _p(labels, C.c_int32), C.byref(energy),
                                 C.byref(moves))
    return (labels, energy.value, moves.value) if return_energy else labels


def cut_general_graph(edges, edge_w, unary, pairwise, n_iter=-1, return_energy=False):
    """gco.cut_general_graph(..., algorithm='expansion')"""
    w, u, v = integerise(np.asarray(edge_w, dtype=float), np.asarray(unary, dtype=float), np.asarray(pairwise, dtype=float))
    return alpha_expansion_int(edges, w, u, v, n_iter, return_energy)


def segment_graph_cut_general(segments, proba, gc_regul=1., edge_type='model', features=None, color_means=None):
    """imsegm/graph_cuts.py:660-747 (labels per superpixel, int32)"""
    edges, w = edge_weights(segments, proba, edge_type, features, color_means)
    un = unary_cost(proba)
    pw = pairwise_cost(gc_regul, proba.shape[1])
    if gc_regul <= 0:
        return np.argmin(un, axis=-1).astype(np.int32)
    return cut_general_graph(edges, w, un, pw, n_iter=-1)


# --------------------------------------------------------------------------------------------------------------------
# pipeline  (imsegm/pipelines.py:160-241 with a given model; :244-270)
# --------------------------------------------------------------------------------------------------------------------

def compute_color2d_superpixels_features(image, flags=('mean',), sp_size=30, sp_regul=0.2):
    slic_map = segment_slic_img2d(image, sp_size=sp_size, relative_compact=sp_regul)
    fts = image2d_color_statistic(image, slic_map, flags)
    fts[np.isnan(fts)] = 0
    return slic_map, fts


def segment_with_model(image, predict_proba, flags=('mean',), sp_size=30, sp_regul=0.2, gc_regul=1., edge_type='model'):
    slic_map, fts = compute_color2d_superpixels_features(image, flags, sp_size, sp_regul)
    proba = predict_proba(fts)
    labels = segment_graph_cut_general(slic_map, proba, gc_regul, edge_type, features=fts)
    return labels[slic_map], proba[slic_map], slic_map, fts


# --------------------------------------------------------------------------------------------------------------------
# the remaining functions of imsegm/features_cython.pyx: gray 3-D statistics, label histogram, ray features
# --------------------------------------------------------------------------------------------------------------------

def gray3d_stat(img, seg, mode, mean=None):
    img = np.ascontiguousarray(img, dtype=np.float32)
    seg = np.ascontiguousarray(seg, dtype=np.int32)
    nb = int(seg.max()) + 1
    out = np.zeros(nb, dtype=np.float64)
    m = np.ascontiguousarray(mean, dtype=np.float32) if mode == 2 else None
    lib().oracle_gray3d_stat(_p(img, C.c_float), _p(seg, C.c_int32), C.c_long(img.size), nb, mode,
                             _p(m, C.c_float) if m is not None else None, _p(out, C.c_double))
    return out


def label_hist2d(segm_select, struc_elem, nb_labels):
    a = np.ascontiguousarray(segm_select, dtype=np.int16)
    b = np.ascontiguousarray(struc_elem, dtype=np.int16)
    hist = np.zeros(int(nb_labels), dtype=np.uint32)
    lib().oracle_label_hist2d(_p(a, C.c_int16), _p(b, C.c_int16), a.shape[0], a.shape[1], int(nb_labels), _p(hist, C.c_uint32))
    return hist


def ray_angles(angle_step):
    """(sin, cos) as float32 exactly like features_cython.pyx:247-268 forms them"""
    angles = np.arange(0, 360, angle_step, dtype=np.float32)
    rads = [float(np.float32(np.deg2rad(a))) for a in angles]          # `rad` is a C float in the reference
    return (np.array([np.sin(r) for r in rads], dtype=np.float32), np.array([np.cos(r) for r in rads], dtype=np.float32))


def ray_features2d(seg_binary, position, angle_step=5., edge=1):
    seg = np.ascontiguousarray(seg_binary, dtype=np.int8)
    s, c = ray_angles(float(angle_step))
    out = np.empty(len(s), dtype=np.float32)
    lib().oracle_ray_features2d(_p(seg, C.c_int8), seg.shape[0], seg.shape[1], int(position[0]), int(position[1]),
                                _p(s, C.c_float), _p(c, C.c_float), len(s), int(edge), _p(out, C.c_float))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# label histograms about positions (imsegm/descriptors.py:1288-1528) -- numpy restatement, pinned by the reference's doctests
# ---------------------------------------------------------------------------------------------------------------------

def disk(radius):
    """skimage.morphology.disk: 1 where dy^2 + dx^2 <= radius^2 on a (2 r + 1)^2 grid"""
    r = int(radius)
    yy, xx = np.mgrid[-r:r + 1, -r:r + 1]
    return (yy ** 2 + xx ** 2 <= r ** 2).astype(np.uint8)


def label_hist_selem(segm, position, struc_elem, nb_labels=None):
    """compute_label_hist_segm (:1396) / compute_label_hist_proba (:1501): the element is centred on the position with
    adjust_bounding_box_crop's rule (:1355): element pixel (iy, ix) lies on image pixel (row - mh // 2 + iy, col - mw // 2 + ix);
    what falls outside the image is dropped.  Returns (hist, size)."""
    segm, struc_elem = np.asarray(segm), np.asarray(struc_elem)
    py, px = int(position[0]), int(position[1])
    mh, mw = struc_elem.shape
    H, W = segm.shape[:2]
    nb = (int(nb_labels) if nb_labels is not None else int(segm.max()) + 1) if segm.ndim == 2 else segm.shape[-1]
    hist = np.zeros(nb)
    size = 0
    for iy in range(mh):
        for ix in range(mw):
            y, x = py - mh // 2 + iy, px - mw // 2 + ix
            if struc_elem[iy, ix] != 1 or y < 0 or y >= H or x < 0 or x >= W:
                continue
            size += 1
            if segm.ndim == 2:
                if 0 <= segm[y, x] < nb:
                    hist[int(segm[y, x])] += 1
            else:
                hist += segm[y, x]
    return hist, size


def label_histograms_positions(segm, positions, diameters, nb_labels=None):
    """compute_label_histograms_positions (:1288-1352): per position, per ring (disc d_i minus disc d_{i-1}) the label
    histogram divided by the ring's pixel count"""
    segm = np.asarray(segm)
    if nb_labels is None:
        nb_labels = int(segm.max()) + 1 if segm.ndim == 2 else segm.shape[-1]
    rows = []
    for pos in positions:
        last_h, last_s, row = np.zeros(nb_labels), 0, []
        for d in diameters:
            h, sz = label_hist_selem(segm, pos, disk(d), nb_labels)
            row += ((h - last_h) / float(sz - last_s)).tolist()
            last_h, last_s = h, sz
        rows.append(row)
    return np.array(rows)


# ---------------------------------------------------------------------------------------------------------------------
# 3-D gray SLIC (imsegm/superpixels.py:72-112 -> skimage slic(multichannel=False, spacing, sigma=1)) -- slic3d_oracle.c
# ---------------------------------------------------------------------------------------------------------------------

def slic_seeds3d(shape, n_segments):
    (sz, tz), (sy, ty), (sx, tx) = regular_grid(shape, n_segments)
    gz, gy, gx = np.meshgrid(np.arange(sz, shape[0], tz), np.arange(sy, shape[1], ty), np.arange(sx, shape[2], tx), indexing='ij')
    seeds = np.stack([gz.ravel(), gy.ravel(), gx.ravel()], axis=1).astype(np.float64)
    return np.ascontiguousarray(seeds), (int(tz), int(ty), int(tx))


def gaussian_blur3d(vol, sigmas):
    vol = np.ascontiguousarray(vol, dtype=np.float64)
    D, H, W = vol.shape
    halves = []
    for s in sigmas:
        halves.append(gaussian_weights(float(s)) if s > 0 else (np.ones(1), 0))
    out = np.empty_like(vol)
    rc = lib().oracle_gaussian_blur3d(_p(vol, C.c_double), D, H, W, _p(halves[0][0], C.c_double), int(halves[0][1]),
                                      _p(halves[1][0], C.c_double), int(halves[1][1]), _p(halves[2][0], C.c_double), int(halves[2][1]),
                                      _p(out, C.c_double))
    assert rc == 0
    return out


def slic3d(vol, n_segments, compactness, spacing=(1, 1, 1), sigma=1.0, max_iter=10, enforce_conn=True, min_size_factor=0.5,
           max_size_factor=3, return_kmeans=False):
    """skimage.segmentation.slic(vol, n_segments, compactness, multichannel=False, spacing=spacing, sigma=sigma), 0.14-0.18"""
    scale = {'uint8': 255.0, 'uint16': 65535.0}.get(str(np.asarray(vol).dtype))      # img_as_float
    vol = np.ascontiguousarray(vol, dtype=np.float64)
    if scale:
        vol = vol / scale
    D, H, W = vol.shape
    spacing = np.ascontiguousarray(spacing, dtype=np.float64)
    if sigma > 0:
        vol = gaussian_blur3d(vol, np.array([sigma, sigma, sigma], dtype=np.float64) / spacing)
    seeds, (tz, ty, tx) = slic_seeds3d((D, H, W), n_segments)
    step = float(max(tz, ty, tx))
    scaled = np.ascontiguousarray(vol * (1.0 / compactness))
    labels = np.empty((D, H, W), dtype=np.int64)
    lib().oracle_slic_kmeans3d(_p(scaled, C.c_double), D, H, W, _p(seeds, C.c_double), len(seeds), tz, ty, tx, C.c_double(step),
                               _p(spacing, C.c_double), int(max_iter), _p(labels, C.c_int64), None)
    if return_kmeans or not enforce_conn:
        return labels
    segment_size = D * H * W / n_segments
    out = np.empty_like(labels)
    n = lib().oracle_enforce_connectivity3d(_p(labels, C.c_int64), D, H, W, C.c_long(int(min_size_factor * segment_size)),
                                            C.c_long(int(max_size_factor * segment_size)), _p(out, C.c_int64))
    assert n >= 0
    return out


def segment_slic_img3d_gray(im, sp_size=50, relative_compact=0.1, space=(1, 1, 1)):
    """imsegm/superpixels.py:72-112.  The closing skimage.measure.label (:111, full connectivity, background 0) renumbers the
    labels in the order of their first voxel and leaves label 0 alone; the connectivity pass already numbers the labels in
    that order, so it changes nothing (checked in tests/test_oracle_goldens.py with scipy.ndimage.label)."""
    im = np.asarray(im)
    nb_pixels = np.prod(im.shape)
    size = np.prod(sp_size / np.asarray(space, dtype=np.float32) * min(space))
    n_seg = int(nb_pixels / size)
    compact = int((size * relative_compact) ** 1.5)
    return slic3d(np.array(im), n_seg, compact, space, sigma=1)
