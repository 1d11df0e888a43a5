"""
Every public function of the reference's ``imsegm/labeling.py``.

The per-pixel work runs on the device (``csrc/labeling.cu`` and the joint histogram of ``csrc/native_misc.cu``): overlap matrices,
the relabelling gathers, boundary and contour maps, and the exact Euclidean distance transform, which is bit-identical to
``scipy.ndimage.distance_transform_edt``.  What stays on the host is vectorised numpy over label tables, image borders or the
caller's lists; no function loops over pixels in Python.

Arrays the reference built with ``np.int`` are ``int64`` here.  The one deliberate difference: ``assume_bg_on_boundary`` rejects
negative labels with ``ValueError`` (the reference raises for one on the image border and silently wraps one inside the image).
"""
import ctypes as C
import logging

import numpy as np

from . import _lib
from .engine import get_engine
from .utilities import ImageDimensionError

_I32 = np.iinfo(np.int32)


def _as_i32_labels(seg):
    """int32 map with the same equality pattern as ``seg`` (what boundary and contour maps depend on)"""
    seg = np.asarray(seg)
    if seg.dtype.kind in 'iub' and (seg.size == 0 or (seg.min() >= _I32.min and seg.max() <= _I32.max)):
        return seg.astype(np.int32, copy=False)
    return np.unique(seg, return_inverse=True)[1].reshape(seg.shape).astype(np.int32)


def _require_2d(*arrays):
    for a in arrays:
        if a.ndim != 2 or a.size == 0:
            raise ValueError('a non-empty 2-D label map is required, got shape %r' % (a.shape, ))


def _contour_mask(eng, seg, label, include_boundary, name):
    """device u8 contour map of ``seg == label`` (contour_binary_map)"""
    seg = np.asarray(seg)
    _require_2d(seg)
    fits = seg.dtype.kind in 'iub' and (seg.size == 0 or (seg.min() >= _I32.min and seg.max() <= _I32.max))
    if fits and _I32.min <= label <= _I32.max and float(label) == int(label):
        d_seg, lb = eng.to_device(seg.astype(np.int32, copy=False), 'lbl_seg'), int(label)
    else:
        d_seg, lb = eng.to_device((seg == label).astype(np.int32), 'lbl_seg'), 1
    out = eng.buf(name, seg.shape, eng.torch.uint8)
    _lib.check(eng.lib.isb_label_contour_map(_lib.ptr(d_seg), seg.shape[0], seg.shape[1], lb, int(bool(include_boundary)), _lib.ptr(out),
                                             _lib.stream_ptr()))
    return out


def _boundary_mask(eng, seg, name):
    """device u8 thick boundary map (find_boundaries(mode='thick'))"""
    out = eng.buf(name, seg.shape, eng.torch.uint8)
    d_seg = eng.to_device(_as_i32_labels(seg), 'lbl_seg')
    _lib.check(eng.lib.isb_label_boundary_map(_lib.ptr(d_seg), seg.shape[0], seg.shape[1], _lib.ptr(out), _lib.stream_ptr()))
    return out


def _edt(eng, d_sites, shape):
    """device f64 distance of every pixel to the nearest nonzero pixel of ``d_sites``"""
    H, W = shape
    if H > 32768 or W > 32768:
        raise ValueError('the distance transform takes images up to 32768 x 32768, got %r' % (shape, ))
    ws_bytes = eng.lib.isb_edt_workspace_bytes(H, W)
    ws = eng.buf('edt_ws', ws_bytes, eng.torch.uint8)
    dist = eng.buf('edt_dist', (H, W), eng.torch.float64)
    _lib.check(eng.lib.isb_edt_2d(_lib.ptr(d_sites), H, W, _lib.ptr(dist), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.stream_ptr()))
    return dist


def _compact(eng, d_mask, shape, d_values=None):
    """(points [P, 2] int64, values [P] f64 or None) of the set pixels of a device mask, in raster order"""
    H, W = shape
    torch = eng.torch
    ws_bytes = eng.lib.isb_mask_compact_workspace_bytes(H, W)
    ws = eng.buf('compact_ws', ws_bytes, torch.uint8)
    total = eng.buf('compact_total', 1, torch.int64)
    _lib.check(eng.lib.isb_mask_compact_count(_lib.ptr(d_mask), H, W, _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(total), _lib.stream_ptr()))
    P = int(eng.to_host(total)[0])
    if P == 0:
        return np.zeros((0, 2), dtype=np.int64), (None if d_values is None else np.zeros(0))
    points = eng.buf('compact_points', (P, 2), torch.int64)
    vals = eng.buf('compact_values', P, torch.float64) if d_values is not None else None
    _lib.check(eng.lib.isb_mask_compact_write(_lib.ptr(d_mask), H, W, _lib.ptr(d_values), _lib.ptr(ws), C.c_size_t(ws_bytes),
                                              _lib.ptr(points), _lib.ptr(vals), _lib.stream_ptr()))
    hosts, done = eng.download([points] + ([vals] if vals is not None else []))
    done.synchronize()
    return hosts[0].numpy().copy(), (hosts[1].numpy().copy() if vals is not None else None)


def _relabel(eng, seg, lut):
    """``lut[seg]`` where ``seg >= 0``, ``seg`` elsewhere, as an int64 array (one device gather)"""
    seg = np.asarray(seg)
    lut = np.asarray(lut, dtype=np.int64)
    if seg.size == 0:
        return np.zeros(seg.shape, dtype=np.int64)
    if lut.min() < _I32.min or lut.max() > _I32.max:
        raise ValueError('relabelled values must fit in int32')
    d_seg = eng.to_device(seg.astype(np.int32, copy=False).reshape(-1), 'lbl_seg')
    d_lut = eng.to_device(lut.astype(np.int32), 'lbl_lut')
    out = eng.buf('lbl_out', seg.size, eng.torch.int32)
    _lib.check(eng.lib.isb_relabel_gather(_lib.ptr(d_seg), C.c_longlong(seg.size), _lib.ptr(d_lut), len(lut), _lib.ptr(out), _lib.stream_ptr()))
    return eng.to_host(out).astype(np.int64).reshape(seg.shape)


def _check_int_labels(*arrays):
    for a in arrays:
        if a.dtype.kind not in 'iub':
            raise TypeError('label maps must be integer arrays, got %s' % a.dtype)
        if a.size and (a.min() < _I32.min or a.max() > _I32.max):
            raise ValueError('labels must fit in int32')


# ---------------------------------------------------------------------------------------------------------------------
# contours and distances (device)
# ---------------------------------------------------------------------------------------------------------------------

def neighbour_connect4(seg, label, pos):
    """ whether one of the 4-neighbours of ``pos`` carries another label (reference labeling.py:17-31)

    >>> neighbour_connect4(np.eye(5), 1, (2, 2))
    True
    >>> neighbour_connect4(np.ones((5, 5)), 1, (3, 3))
    False
    """
    # in the reference's order, stopping at the first differing neighbour (a later one may lie outside the map)
    return any(seg[pos[0] + a, pos[1] + b] != label for a, b in ((-1, 0), (0, -1), (1, 0), (0, 1)))


def contour_binary_map(seg, label=1, include_boundary=False):
    """ 0 / 1 int64 map of the contour of ``label`` (reference labeling.py:34-79): pixels of the label off the outer frame with a
    4-neighbour of another label, and with ``include_boundary`` the label's pixels on the frame

    >>> img = np.zeros((6, 6), dtype=int)
    >>> img[1:5, 2:] = 1
    >>> contour_binary_map(img)
    array([[0, 0, 0, 0, 0, 0],
           [0, 0, 1, 1, 1, 0],
           [0, 0, 1, 0, 0, 0],
           [0, 0, 1, 0, 0, 0],
           [0, 0, 1, 1, 1, 0],
           [0, 0, 0, 0, 0, 0]])
    """
    eng = get_engine()
    return eng.to_host(_contour_mask(eng, seg, label, include_boundary, 'lbl_contour')).astype(np.int64)


def contour_coords(seg, label=1, include_boundary=False):
    """ the contour of ``label`` as a list of [row, col] (reference labeling.py:82-117): the interior points in raster order, then
    with ``include_boundary`` the frame points in the reference's order -- per row [i, 0], [i, W - 1], then per column [0, j],
    [H - 1, j] -- corners included twice

    >>> img = np.zeros((6, 6), dtype=int)
    >>> img[1:5, 2:] = 1
    >>> contour_coords(img)
    [[1, 2], [1, 3], [1, 4], [2, 2], [3, 2], [4, 2], [4, 3], [4, 4]]
    """
    seg = np.asarray(seg)
    eng = get_engine()
    d_mask = _contour_mask(eng, seg, label, False, 'lbl_contour')
    pts, _ = _compact(eng, d_mask, seg.shape)
    res = pts.tolist()
    if include_boundary:
        h, w = seg.shape
        rows, cols = np.arange(h), np.arange(w)
        side = np.stack([seg[:, 0] == label, seg[:, -1] == label], axis=1)
        side_pts = np.stack([np.stack([rows, np.zeros_like(rows)], 1), np.stack([rows, np.full_like(rows, w - 1)], 1)], axis=1)
        topbot = np.stack([seg[0, :] == label, seg[-1, :] == label], axis=1)
        topbot_pts = np.stack([np.stack([np.zeros_like(cols), cols], 1), np.stack([np.full_like(cols, h - 1), cols], 1)], axis=1)
        res += side_pts[side].tolist() + topbot_pts[topbot].tolist()
    return res


def binary_image_from_coords(coords, size):
    """ int64 map with 1 at every coordinate inside ``size`` (reference labeling.py:120-143)

    >>> binary_image_from_coords([[1, 2], [0, 0], [7, 1]], (3, 4))
    array([[1, 0, 0, 0],
           [0, 0, 0, 0],
           [0, 0, 1, 0]])
    """
    contour_map = np.zeros(size, dtype=np.int64)
    w, h = size
    pts = np.asarray(coords, dtype=np.int64).reshape(-1, 2)
    ok = (pts[:, 0] >= 0) & (pts[:, 0] < w) & (pts[:, 1] >= 0) & (pts[:, 1] < h)
    contour_map[pts[ok, 0], pts[ok, 1]] = 1
    return contour_map


def compute_distance_map(seg, label=1):
    """ distance of every pixel to the contour of ``label`` (reference labeling.py:146-169); the contour map goes straight into the
    device EDT.  Bit-identical to scipy.ndimage.distance_transform_edt, including an empty contour (every pixel measured from
    (-1, 0) as scipy does).

    >>> img = np.zeros((6, 6), dtype=int)
    >>> img[1:5, 2:] = 1
    >>> dist = compute_distance_map(img)
    >>> np.round(dist, 2)[0].tolist()
    [2.24, 1.41, 1.0, 1.0, 1.0, 1.41]
    """
    seg = np.asarray(seg)
    eng = get_engine()
    if seg.ndim == 2 and (seg.shape[0] > 32768 or seg.shape[1] > 32768):
        raise ValueError('the distance transform takes images up to 32768 x 32768, got %r' % (seg.shape, ))
    d_mask = _contour_mask(eng, seg, label, False, 'lbl_contour')
    return eng.to_host(_edt(eng, d_mask, seg.shape)).copy()


def compute_boundary_distances(segm_ref, segm):
    """ distance of every boundary pixel of ``segm_ref`` to the nearest boundary pixel of ``segm`` (reference labeling.py:684-716):
    (points [P, 2] int64 (row, col) in raster order, dist [P] f64).  Boundaries are find_boundaries(mode='thick'); the distance is
    the device EDT, bit-identical to scipy's.

    >>> segm_ref = np.zeros((6, 10), dtype=int)
    >>> segm_ref[3:4, 4:5] = 1
    >>> segm = np.zeros((6, 10), dtype=int)
    >>> segm[:, 2:9] = 1
    >>> pts, dist = compute_boundary_distances(segm_ref, segm)
    >>> pts.tolist()
    [[2, 4], [3, 3], [3, 4], [3, 5], [4, 4]]
    >>> dist.tolist()
    [2.0, 1.0, 2.0, 3.0, 2.0]
    """
    segm_ref, segm = np.asarray(segm_ref), np.asarray(segm)
    if segm_ref.shape != segm.shape:
        raise ImageDimensionError('Ref. segm %r and segm %r should match' % (segm_ref.shape, segm.shape))
    _require_2d(segm)
    if segm.shape[0] > 32768 or segm.shape[1] > 32768:
        raise ValueError('the distance transform takes images up to 32768 x 32768, got %r' % (segm.shape, ))
    eng = get_engine()
    d_sites = _boundary_mask(eng, segm, 'lbl_bnd')
    dist = _edt(eng, d_sites, segm.shape)
    d_ref = _boundary_mask(eng, segm_ref, 'lbl_bnd_ref')
    points, values = _compact(eng, d_ref, segm.shape, dist)
    return points, values


# ---------------------------------------------------------------------------------------------------------------------
# overlap and relabelling (device histogram and gather, host label tables)
# ---------------------------------------------------------------------------------------------------------------------

def compute_labels_overlap_matrix(seg1, seg2):
    """ overlap[a, b] = pixels with label a in ``seg1`` and b in ``seg2``, pixels with a negative label in either map skipped
    (reference labeling.py:490-523); int64 [seg1.max() + 1, seg2.max() + 1], any rank

    >>> seg1 = np.zeros((7, 15), dtype=int)
    >>> seg1[1:4, 5:10] = 3
    >>> seg1[5:7, 6:13] = 2
    >>> seg2 = np.zeros((7, 15), dtype=int)
    >>> seg2[2:5, 7:12] = 1
    >>> seg2[4:7, 7:14] = 3
    >>> compute_labels_overlap_matrix(seg1, seg2)
    array([[63,  4,  0,  9],
           [ 0,  0,  0,  0],
           [ 2,  0,  0, 12],
           [ 9,  6,  0,  0]])
    """
    seg1, seg2 = np.asarray(seg1), np.asarray(seg2)
    logging.debug('computing overlap of two seg_pipe of shapes %r <-> %r', seg1.shape, seg2.shape)
    if seg1.shape != seg2.shape:
        raise ImageDimensionError('segm %r and segm %r should match' % (seg1.shape, seg2.shape))
    _check_int_labels(seg1, seg2)
    maxims = [int(np.max(seg1)) + 1, int(np.max(seg2)) + 1]
    overlap = np.zeros(maxims, dtype=np.int64)      # raises numpy's ValueError for a negative dimension
    if overlap.size == 0:
        return overlap
    a, b = (seg1, seg2) if seg1.ndim == 2 else (seg1.reshape(1, -1), seg2.reshape(1, -1))
    eng = get_engine()
    d_a = eng.to_device(a.astype(np.int32, copy=False), 'hist_slic')
    d_b = eng.to_device(b.astype(np.int32, copy=False), 'hist_annot')
    hist = eng.buf('hist_joint', maxims, eng.torch.int32)
    _lib.check(eng.lib.isb_region_label_hist(_lib.ptr(d_a), _lib.ptr(d_b), a.shape[0], a.shape[1], maxims[0], maxims[1], _lib.ptr(hist),
                                             _lib.stream_ptr()))
    return eng.to_host(hist).view(np.uint32).astype(np.int64)


def max_overlap_unique_lut(overlap, n_lut, keep_bg=False):
    """ the look-up table of relabel_max_overlap_unique (reference labeling.py:585-609) in O(L log L) instead of its O(L^3) loops:
    - the greedy part ("take the first maximum in row-major order, zero its row and column") is one pass over the positive
      entries sorted by value descending, ties by the smaller flat index, skipping entries in a used row or column;
    - the first fill sets lut[i] = i in order when i is not yet a value of the table;
    - the second fill has no ``break`` in the reference: each remaining -1 ends as the LARGEST j < len(lut) that no other entry
      holds, or stays -1.
    """
    overlap = np.array(overlap, copy=True)
    lut = [-1] * n_lut
    if keep_bg:
        lut[0] = 0
        overlap[0, :] = 0
        overlap[:, 0] = 0
    if overlap.size:
        flat = overlap.ravel()
        idx = np.flatnonzero(flat > 0)
        idx = idx[np.lexsort((idx, -flat[idx]))]
        used_r, used_c = np.zeros(overlap.shape[0], bool), np.zeros(overlap.shape[1], bool)
        for r, c in zip(*np.unravel_index(idx, overlap.shape)):
            if used_r[r] or used_c[c]:
                continue
            used_r[r] = used_c[c] = True
            lut[c] = int(r)
    values = set(lut)
    for i, lb in enumerate(lut):
        if lb == -1 and i not in values:
            lut[i] = i
            values.add(i)
    j = len(lut) - 1
    for i, lb in enumerate(lut):
        if lb > -1:
            continue
        while j >= 0 and j in values:
            j -= 1
        if j < 0:
            break
        lut[i] = j
        values.add(j)
    return lut


def relabel_max_overlap_unique(seg_ref, seg_relabel, keep_bg=False):
    """ relabel ``seg_relabel`` so that its patterns overlap those of ``seg_ref`` most, one to one (reference labeling.py:526-614);
    negative labels are kept.  The overlap and the final gather run on the device, the table on the host.

    >>> atlas1 = np.zeros((7, 15), dtype=int)
    >>> atlas1[1:4, 5:10] = 1
    >>> atlas1[5:7, 3:13] = 2
    >>> atlas2 = np.zeros((7, 15), dtype=int)
    >>> atlas2[0:3, 7:12] = 1
    >>> atlas2[3:7, 1:7] = 2
    >>> atlas2[4:7, 7:14] = 3
    >>> atlas2[:2, :3] = 5
    >>> relabel_max_overlap_unique(atlas2, atlas1, keep_bg=True)[5].tolist()
    [0, 0, 0, 3, 3, 3, 3, 3, 3, 3, 3, 3, 3, 0, 0]
    """
    seg_ref, seg_relabel = np.asarray(seg_ref), np.asarray(seg_relabel)
    if seg_ref.shape != seg_relabel.shape:
        raise ImageDimensionError('Reference segm. %r and input segm. %r should match' % (seg_ref.shape, seg_relabel.shape))
    overlap = compute_labels_overlap_matrix(seg_ref, seg_relabel)
    n_lut = int(np.max(seg_relabel)) + 1
    lut = max_overlap_unique_lut(overlap, max(n_lut, 0), keep_bg)
    _check_index_range(seg_relabel, len(lut))
    return _relabel(get_engine(), seg_relabel, lut)


def _check_index_range(seg, n):
    """the IndexError numpy raises for ``lut[seg]`` with a table of n entries (a negative label below -n)"""
    lo, hi = int(seg.min()), int(seg.max())
    if hi >= n or lo < -n:
        raise IndexError('index %d is out of bounds for axis 0 with size %d' % (hi if hi >= n else lo, n))


def relabel_max_overlap_merge(seg_ref, seg_relabel, keep_bg=False):
    """ relabel ``seg_relabel`` by the maximal overlap with ``seg_ref``, merging patterns (reference labeling.py:617-681);
    negative labels are kept.  The overlap and the final gather run on the device.

    >>> atlas1 = np.zeros((7, 15), dtype=int)
    >>> atlas1[1:4, 5:10] = 1
    >>> atlas1[5:7, 3:13] = 2
    >>> atlas2 = np.zeros((7, 15), dtype=int)
    >>> atlas2[0:3, 7:12] = 1
    >>> atlas2[3:7, 1:7] = 2
    >>> atlas2[4:7, 7:14] = 3
    >>> atlas2[:2, :3] = 5
    >>> relabel_max_overlap_merge(atlas1, atlas2, keep_bg=True)[0].tolist()
    [1, 1, 1, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0]
    """
    seg_ref, seg_relabel = np.asarray(seg_ref), np.asarray(seg_relabel)
    if seg_ref.shape != seg_relabel.shape:
        raise ImageDimensionError('Ref. segm %r and segm %r should match' % (seg_ref.shape, seg_relabel.shape))
    overlap = compute_labels_overlap_matrix(seg_ref, seg_relabel)
    max_axis = 1 if overlap.shape[0] > overlap.shape[1] else 0
    if keep_bg:
        id_max = np.argmax(overlap[1:, 1:], axis=max_axis) + 1
        lut = np.array([0] + id_max.tolist())
    else:
        lut = np.argmax(overlap, axis=max_axis)
    ptn_sum = np.sum(overlap, axis=0)
    if 0 in ptn_sum:
        lut[ptn_sum == 0] = np.arange(len(lut))[ptn_sum == 0]
    _check_index_range(seg_relabel, len(lut))
    return _relabel(get_engine(), seg_relabel, lut)


def assume_bg_on_boundary(segm, bg_label=0, boundary_size=1):
    """ swap labels so that ``bg_label`` is the label seen most on the image border (reference labeling.py:719-754): the border
    label is argmax(bincount) of the four strips of ``boundary_size`` pixels, corners counted twice.  Negative labels raise
    ``ValueError`` (the one deliberate difference from the reference, which raises for one on the border and wraps one inside).

    >>> segm = np.zeros((6, 12), dtype=int)
    >>> segm[1:4, 4:] = 2
    >>> segm[segm == 0] = 1
    >>> assume_bg_on_boundary(segm, boundary_size=1)[1].tolist()
    [0, 0, 0, 0, 2, 2, 2, 2, 2, 2, 2, 2]
    """
    segm = np.asarray(segm)
    if segm.ndim != 2:
        raise ValueError('a 2-D label map is required, got shape %r' % (segm.shape, ))
    _check_int_labels(segm)
    if segm.size and segm.min() < 0:
        raise ValueError('negative labels are not allowed')
    size = int(boundary_size)
    strips = np.hstack([segm[:size, :], segm[:, :size].T, segm[-size:, :], segm[:, -size:].T])
    boundary_lb = np.argmax(np.bincount(strips.ravel().astype(np.int64)))
    lut = list(range(int(segm.max()) + 1))
    lut[boundary_lb] = bg_label
    lut[bg_label] = boundary_lb
    return _relabel(get_engine(), segm, lut)


# ---------------------------------------------------------------------------------------------------------------------
# superpixel histograms (device)
# ---------------------------------------------------------------------------------------------------------------------

def histogram_regions_labels_counts(slic, segm):
    """ overlap counts between superpixels and an annotation: ``hist[a, b]`` = pixels with superpixel ``a`` and label ``b``
    (reference labeling.py:206-240, a per-pixel Python loop there)

    :param ndarray slic: superpixel map
    :param ndarray segm: annotation, non-negative labels
    :return ndarray: float matrix [slic.max() + 1, segm.max() + 1]
    """
    slic, segm = np.asarray(slic), np.asarray(segm)
    if slic.shape != segm.shape:
        raise ImageDimensionError('dimension does not agree')
    if segm.min() < 0:
        raise ValueError('only positive labels are allowed')
    if slic.ndim != 2:
        slic, segm = slic.reshape(1, -1), segm.reshape(1, -1)
    eng = get_engine()
    nb_a, nb_b = int(slic.max()) + 1, int(segm.max()) + 1
    d_a = eng.to_device(slic.astype(np.int32, copy=False), 'hist_slic')
    d_b = eng.to_device(segm.astype(np.int32, copy=False), 'hist_annot')
    hist = eng.buf('hist_joint', (nb_a, nb_b), eng.torch.int32)
    _lib.check(eng.lib.isb_region_label_hist(_lib.ptr(d_a), _lib.ptr(d_b), slic.shape[0], slic.shape[1], nb_a, nb_b, _lib.ptr(hist),
                                             _lib.stream_ptr()))
    return eng.to_host(hist).astype(float)


def histogram_regions_labels_norm(slic, segm):
    """ relative overlap of every superpixel with the annotation labels, rows sum to 1 (reference labeling.py:243-283) """
    slic, segm = np.asarray(slic), np.asarray(segm)
    if slic.shape != segm.shape:
        raise ImageDimensionError('dimension of SLIC %r and segm %r should match' % (slic.shape, segm.shape))
    if segm.min() < 0:
        raise ValueError('only positive labels are allowed')
    hist = histogram_regions_labels_counts(slic, segm)
    sums = hist.sum(axis=1, keepdims=True)
    sums[sums == 0] = -1.
    hist = np.nan_to_num(hist / sums)
    hist[hist == 0] = 0
    return hist


# ---------------------------------------------------------------------------------------------------------------------
# label tables and lists (host, vectorised numpy)
# ---------------------------------------------------------------------------------------------------------------------

def segm_labels_assignment(segm, segm_gt):
    """ for every label of ``segm`` the list of ``segm_gt`` values under it, in raster order (reference labeling.py:172-204):
    one stable sort by label and a split """
    segm, segm_gt = np.asarray(segm), np.asarray(segm_gt)
    if segm_gt.shape != segm.shape:
        raise ImageDimensionError('segm %r and annot %r should match' % (segm.shape, segm_gt.shape))
    flat, gt = segm.ravel(), segm_gt.ravel()
    labels, inv = np.unique(flat, return_inverse=True)
    order = np.argsort(inv.ravel(), kind='stable')
    parts = np.split(gt[order], np.cumsum(np.bincount(inv.ravel(), minlength=len(labels)))[:-1])
    return {lb: list(part) for lb, part in zip(labels, parts)}


def _label_fractions(dict_label_hist):
    """(keys, fractions [n_keys, max value + 1]) of np.bincount(v) / len(v) for every entry"""
    keys = list(dict_label_hist.keys())
    vals = [np.asarray(dict_label_hist[k]) for k in keys]
    if any(v.size == 0 for v in vals):
        raise ValueError('zero-size array to reduction operation maximum which has no identity')
    width = max(int(v.max()) + 1 if v.size else 1 for v in vals)
    frac = np.zeros((len(keys), width))
    for i, v in enumerate(vals):
        frac[i] = np.bincount(v, minlength=width) / float(len(v))
    return keys, frac


def assign_label_by_threshold(dict_label_hist, thresh=0.75):
    """ label of every region whose purity exceeds ``thresh``, else -1 (reference labeling.py:300-324)

    >>> assign_label_by_threshold({0: [0, 0, 1], 2: [1, 1, 1, 1]}, thresh=0.7)
    array([-1, -1,  1])
    """
    lut = np.zeros(max(dict_label_hist.keys()) + 1, dtype=int) - 1
    keys, frac = _label_fractions(dict_label_hist)
    mx = frac.max(axis=1)
    sel = mx > thresh
    lut[np.asarray(keys, dtype=np.int64)[sel]] = np.argmax(frac, axis=1)[sel]
    return lut


def assign_label_by_max(label_hist):
    """ label seen most in every region (reference labeling.py:327-346)

    >>> assign_label_by_max({0: [0, 0, 1], 2: [1, 1, 1, 1]})
    array([ 0, -1,  1])
    """
    lut = np.zeros(max(label_hist.keys()) + 1, dtype=int) - 1
    keys, frac = _label_fractions(label_hist)
    lut[np.asarray(keys, dtype=np.int64)] = np.argmax(frac, axis=1)
    return lut


def convert_segms_2_list(segms):
    """ all segmentations flattened into one list (reference labeling.py:349-361)

    >>> seg_pipe = np.ones((2, 3), dtype=int)
    >>> convert_segms_2_list([seg_pipe, seg_pipe * 0, seg_pipe * 2])
    [1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 2, 2, 2, 2, 2, 2]
    """
    return np.concatenate(tuple(np.asarray(seg).ravel() for seg in segms), axis=0).tolist()


def mask_segm_labels(img_labeling, labels, mask_init=None):
    """ bool mask of the pixels carrying one of ``labels``, or-ed onto ``mask_init`` (reference labeling.py:364-393)

    >>> img = np.zeros((2, 3))
    >>> img[0, 1:] = 1
    >>> mask_segm_labels(img, [1]).tolist()
    [[False, True, True], [False, False, False]]
    """
    img_labeling = np.asarray(img_labeling)
    mask = np.full(img_labeling.shape, False, dtype=bool) if mask_init is None else np.array(mask_init, copy=True)
    if len(labels):
        mask = np.logical_or(mask, np.isin(img_labeling, list(labels)))
    return mask


def sequence_labels_merge(labels_stack, dict_colors, labels_free, change_label=-1):
    """ per pixel, the one label of ``dict_colors`` that a time series shows apart from the free labels, else ``change_label``
    (reference labeling.py:396-436)

    >>> dict_colors = {0: [], 1: [], 2: []}
    >>> sequence_labels_merge(np.array([[1], [0], [1], [1], [1], [1], [0], [0]]), dict_colors, [0])
    array([1])
    """
    labels_stack = np.array(labels_stack)
    im_labels = np.full(labels_stack.shape[1:], change_label, dtype=np.int64)
    labels_used = [lb for lb in dict_colors if lb not in labels_free]
    lb_all = labels_used + list(labels_free) + [change_label]
    if not np.all(np.isin(np.unique(labels_stack), lb_all)):
        raise ValueError('some extra labels in image stack')
    mask_free = mask_segm_labels(labels_stack, labels_free)
    for lb in labels_used:
        is_lb = labels_stack == lb
        mask = np.logical_and(np.all(is_lb | mask_free, axis=0), np.any(is_lb, axis=0))
        im_labels[mask] = lb
    return im_labels


def relabel_by_dict(labels, dict_labels):
    """ new label of every old one from {new: [old, ...]}; labels not in the dict become 0 and a later entry wins
    (reference labeling.py:439-456)

    >>> labels = np.array([2, 1, 0, 3, 3, 0, 2, 3, 0, 0])
    >>> relabel_by_dict(labels, {0: [1, 2], 1: [0, 3]}).tolist()
    [0, 0, 1, 1, 1, 1, 0, 1, 1, 1]
    """
    if not dict_labels:
        raise ValueError('"dict_labels" is required')
    labels = np.asarray(labels)
    olds = [lb_old for lb_new in dict_labels for lb_old in dict_labels[lb_new]]
    news = [lb_new for lb_new in dict_labels for _ in dict_labels[lb_new]]
    labels_new = np.zeros_like(labels)
    if not olds:
        return labels_new
    uniq, inv = np.unique(np.asarray(olds), return_inverse=True)
    last = np.zeros(len(uniq), dtype=np.int64)
    np.maximum.at(last, inv.ravel(), np.arange(len(olds)))      # a later entry wins
    new_of = np.asarray(news)[last]
    pos = np.clip(np.searchsorted(uniq, labels), 0, len(uniq) - 1)
    hit = uniq[pos] == labels
    labels_new[hit] = new_of[pos[hit]]
    return labels_new


def merge_probab_labeling_2d(proba, dict_labels):
    """ probabilities of merged classes: channel ``new`` = sum of the channels listed for it (reference labeling.py:459-487)

    >>> p = np.ones((5, 5))
    >>> proba = np.rollaxis(np.array([p * 0.3, p * 0.4, p * 0.2]), 0, 3)
    >>> merge_probab_labeling_2d(proba, {0: [1, 2], 1: [0]})[0, 0].tolist()
    [0.6000000000000001, 0.3]
    """
    if proba.ndim != 3:
        raise ValueError
    if not dict_labels:
        raise ValueError('"dict_labels" is required')
    max_label = max(dict_labels.keys()) + 1
    proba_new = np.zeros(proba.shape[:-1] + (max_label, ))
    for lb_new in dict_labels:
        proba_new[:, :, lb_new] = np.sum(proba[:, :, dict_labels[lb_new]], axis=-1)
    return proba_new
