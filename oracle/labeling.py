"""
Host oracle of ``imsegm/labeling.py`` (numpy / scipy only; test infrastructure, never imported by the product).

The reference module imports scikit-image, which the tests cannot rely on, so its functions are restated here with the same
per-pixel loops and the same order of operations -- deliberately slow, so that the fast device and host paths are checked against
the plain meaning of the reference rather than against another clever restatement.  ``np.int`` (removed in numpy 2) is read as
``int``.  ``skimage.segmentation.find_boundaries(mode='thick')`` is grey dilation != grey erosion with the 4-connected cross and
scipy's default 'reflect' border; the distance transform is ``scipy.ndimage.distance_transform_edt``.
"""
import numpy as np
from scipy import ndimage


class ImageDimensionError(ValueError):
    pass


def find_boundaries_thick(label_img):
    cross = ndimage.generate_binary_structure(label_img.ndim, 1)
    return ndimage.grey_dilation(label_img, footprint=cross) != ndimage.grey_erosion(label_img, footprint=cross)


def neighbour_connect4(seg, label, pos):
    for dr, dc in ((-1, 0), (0, -1), (1, 0), (0, 1)):
        if seg[pos[0] + dr, pos[1] + dc] != label:
            return True
    return False


def contour_binary_map(seg, label=1, include_boundary=False):
    rows, cols = seg.shape[:2]
    out = np.zeros((rows, cols), dtype=int)
    for r in range(1, rows - 1):
        for c in range(1, cols - 1):
            if seg[r, c] == label and neighbour_connect4(seg, label, (r, c)):
                out[r, c] = 1
    if include_boundary:
        for r in range(rows):
            if seg[r, 0] == label:
                out[r, 0] = 1
            if seg[r, -1] == label:
                out[r, -1] = 1
        for c in range(cols):
            if seg[0, c] == label:
                out[0, c] = 1
            if seg[-1, c] == label:
                out[-1, c] = 1
    return out


def contour_coords(seg, label=1, include_boundary=False):
    rows, cols = seg.shape[:2]
    pts = []
    for r in range(1, rows - 1):
        for c in range(1, cols - 1):
            if seg[r, c] == label and neighbour_connect4(seg, label, (r, c)):
                pts.append([r, c])
    if include_boundary:
        for r in range(rows):
            if seg[r, 0] == label:
                pts.append([r, 0])
            if seg[r, -1] == label:
                pts.append([r, cols - 1])
        for c in range(cols):
            if seg[0, c] == label:
                pts.append([0, c])
            if seg[-1, c] == label:
                pts.append([rows - 1, c])
    return pts


def binary_image_from_coords(coords, size):
    out = np.zeros(size, dtype=int)
    rows, cols = size
    for pt in coords:
        if 0 <= pt[0] < rows and 0 <= pt[1] < cols:
            out[pt[0], pt[1]] = 1
    return out


def compute_distance_map(seg, label=1):
    contour = binary_image_from_coords(contour_coords(seg, label), seg.shape)
    return ndimage.distance_transform_edt(1 - contour)


def segm_labels_assignment(segm, segm_gt):
    if segm_gt.shape != segm.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (segm.shape, segm_gt.shape))
    out = {lb: [] for lb in np.unique(segm)}
    gt = segm_gt.ravel()
    for i, lb in enumerate(segm.ravel()):
        out[lb].append(gt[i])
    return out


def assign_label_by_threshold(dict_label_hist, thresh=0.75):
    lut = np.zeros(max(dict_label_hist.keys()) + 1, dtype=int) - 1
    for k, v in dict_label_hist.items():
        frac = np.bincount(v) / float(len(v))
        best = frac.max()
        if best > thresh:
            lut[k] = frac.tolist().index(best)
    return lut


def assign_label_by_max(label_hist):
    lut = np.zeros(max(label_hist.keys()) + 1, dtype=int) - 1
    for k, v in label_hist.items():
        lut[k] = np.argmax(np.bincount(v) / float(len(v)))
    return lut


def convert_segms_2_list(segms):
    return np.concatenate([seg.ravel() for seg in segms], axis=0).tolist()


def mask_segm_labels(img_labeling, labels, mask_init=None):
    mask = np.full(img_labeling.shape, False, dtype=bool) if mask_init is None else mask_init.copy()
    for lb in labels:
        mask = np.logical_or(mask, img_labeling == lb)
    return mask


def sequence_labels_merge(labels_stack, dict_colors, labels_free, change_label=-1):
    labels_stack = np.array(labels_stack)
    out = np.full(labels_stack.shape[1:], change_label, dtype=int)
    used = [lb for lb in dict_colors if lb not in labels_free]
    allowed = used + labels_free + [change_label]
    if not all(lb in allowed for lb in np.unique(labels_stack)):
        raise ValueError('some extra labels in image stack')
    free = mask_segm_labels(labels_stack, labels_free)
    for lb in used:
        stays = mask_segm_labels(labels_stack, [lb], free)
        seen = mask_segm_labels(labels_stack, [lb])
        out[np.logical_and(np.all(stays, axis=0), np.any(seen, axis=0))] = lb
    return out


def relabel_by_dict(labels, dict_labels):
    if not dict_labels:
        raise ValueError('"dict_labels" is required')
    out = np.zeros_like(labels)
    for new in dict_labels:
        for old in dict_labels[new]:
            out[labels == old] = new
    return out


def merge_probab_labeling_2d(proba, dict_labels):
    if proba.ndim != 3:
        raise ValueError
    if not dict_labels:
        raise ValueError('"dict_labels" is required')
    out = np.zeros(proba.shape[:-1] + (max(dict_labels.keys()) + 1, ))
    for new in dict_labels:
        out[:, :, new] = np.sum(proba[:, :, dict_labels[new]], axis=-1)
    return out


def compute_labels_overlap_matrix(seg1, seg2):
    if seg1.shape != seg2.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (seg1.shape, seg2.shape))
    overlap = np.zeros([np.max(seg1) + 1, np.max(seg2) + 1], dtype=int)
    for a, b in zip(seg1.ravel(), seg2.ravel()):
        if a >= 0 and b >= 0:
            overlap[a, b] += 1
    return overlap


def max_overlap_unique_lut(overlap, n_lut, keep_bg=False):
    """the table of relabel_max_overlap_unique, with the reference's repeated argmax and its two fill loops"""
    overlap = np.array(overlap, copy=True)
    lut = [-1] * n_lut
    if keep_bg:
        lut[0] = 0
        overlap[0, :] = 0
        overlap[:, 0] = 0
    for _ in range(max(overlap.shape) + 1):
        if np.sum(overlap) == 0:
            break
        r, c = np.argwhere(overlap.max() == overlap)[0]
        lut[c] = r
        overlap[r, :] = 0
        overlap[:, c] = 0
    for i, lb in enumerate(lut):
        if lb == -1 and i not in lut:
            lut[i] = i
    for i, lb in enumerate(lut):
        if lb > -1:
            continue
        for j in range(len(lut)):
            if j not in lut:
                lut[i] = j
    return lut


def relabel_max_overlap_unique(seg_ref, seg_relabel, keep_bg=False):
    if seg_ref.shape != seg_relabel.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (seg_ref.shape, seg_relabel.shape))
    overlap = compute_labels_overlap_matrix(seg_ref, seg_relabel)
    lut = max_overlap_unique_lut(overlap, np.max(seg_relabel) + 1, keep_bg)
    out = np.array(lut)[seg_relabel].astype(int)
    out[seg_relabel < 0] = seg_relabel[seg_relabel < 0]
    return out


def relabel_max_overlap_merge(seg_ref, seg_relabel, keep_bg=False):
    if seg_ref.shape != seg_relabel.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (seg_ref.shape, seg_relabel.shape))
    overlap = compute_labels_overlap_matrix(seg_ref, seg_relabel)
    axis = 1 if overlap.shape[0] > overlap.shape[1] else 0
    if keep_bg:
        lut = np.array([0] + (np.argmax(overlap[1:, 1:], axis=axis) + 1).tolist())
    else:
        lut = np.argmax(overlap, axis=axis)
    col_sum = np.sum(overlap, axis=0)
    if 0 in col_sum:
        lut[col_sum == 0] = np.arange(len(lut))[col_sum == 0]
    out = lut[seg_relabel].astype(int)
    out[seg_relabel < 0] = seg_relabel[seg_relabel < 0]
    return out


def compute_boundary_distances(segm_ref, segm):
    if segm_ref.shape != segm.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (segm_ref.shape, segm.shape))
    cols, rows = np.meshgrid(range(segm_ref.shape[1]), range(segm_ref.shape[0]))
    ref_bnd = find_boundaries_thick(segm_ref)
    points = np.array([rows[ref_bnd].ravel(), cols[ref_bnd].ravel()]).T
    dist_map = ndimage.distance_transform_edt(~find_boundaries_thick(segm))
    return points, dist_map[ref_bnd].ravel()


def image2d_boundary_color(image, size=1):
    """get_image2d_boundary_color (imsegm/utilities/data_io.py) of a 2-D label map"""
    size = int(size)
    strips = np.hstack([image[:size, :], image[:, :size].T, image[-size:, :], image[:, -size:].T])
    return np.argmax(np.bincount(strips.ravel())).astype(image.dtype)


def assume_bg_on_boundary(segm, bg_label=0, boundary_size=1):
    boundary_lb = image2d_boundary_color(segm, size=boundary_size)
    used = np.unique(segm)
    if boundary_lb not in used:
        segm[segm == boundary_lb] = bg_label
        return segm
    lut = list(range(used.max() + 1))
    lut[boundary_lb] = bg_label
    lut[bg_label] = boundary_lb
    return np.array(lut)[segm]


def edt_without_sites(shape):
    """what scipy's distance_transform_edt returns for an input without zeros: every pixel measured from (-1, 0)"""
    yy, xx = np.indices(shape)
    return np.sqrt(((yy + 1) ** 2 + xx ** 2).astype(np.float64))
