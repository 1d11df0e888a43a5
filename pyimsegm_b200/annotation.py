"""
Every public name of the reference's ``imsegm/annotation.py``.

The per-pixel work runs on the device (``csrc/annotation.cu`` and the nearest-site transform of ``csrc/labeling.cu``): the colour
histogram over 2^24 packed-RGB bins and its compaction, the palette lookups (exact match, L1-nearest colour, label -> colour
gather) and the nearest valid pixel of the inpainting, which is the exact Euclidean distance transform giving the index of a
nearest site.  What stays on the host: reading image files (PIL), the ``ratio_threshold`` filter on the compacted colour list and
``load_info_group_by_slices`` (pandas).  There is no CPU fallback.

Palettes hold at most 1024 colours (``NotImplementedError`` above).  uint8 images against integer colours in [0, 255] are compared
in integers; any other image or palette is compared in float64, exact for the values annotation images hold.

Differences from the reference:

- ``unique_image_colors`` and ``image_frequent_colors`` list colours in ascending packed-RGB order (r << 16 | g << 8 | b); PIL's
  hash-table order depends on insertion order and cannot be reproduced from the colour set.  Both take the image as uint8 with 1
  (grey), 3 or 4 channels; other channel counts raise ``ValueError``.
- Label maps are int64, which is what the reference's ``np.int`` meant (NumPy 1.24 removed it, so the reference's own conversions
  no longer run).
- ``image_inpaint_pixels`` takes 2-D arrays (any other rank raises ``ValueError``) and treats every nonzero of ``valid_mask`` as
  valid.  Of equidistant valid pixels it takes the one of smallest column, then of smallest row -- the choice of
  ``scipy.ndimage.distance_transform_edt(..., return_indices=True)`` -- where the reference takes whichever its KD-tree finds.
  The same holds for ``quantize_image_nearest_pixel``.
- A map without any valid pixel raises ``ValueError`` (in the reference scipy raises from inside the interpolator).
- ``convert_img_labels_to_colors`` returns the dtype of all the dictionary's colours as one array; the reference takes only the
  colours of labels between the map's minimum and maximum.
- ``load_info_group_by_slices`` shows no progress bar and joins rows with ``pd.concat`` (``DataFrame.append`` is gone).
"""
import ctypes as C
import logging
import os

import numpy as np

from . import _lib
from .engine import get_engine
from .utilities import ImageDimensionError

#: names of annotated columns
COLUMNS_POSITION = ('ant_x', 'ant_y', 'post_x', 'post_y', 'lat_x', 'lat_y')
SLICE_NAME_GROUPING = 'stack_path'
#: set distance in Z axis whether near slice may still belong to the same egg
ANNOT_SLICE_DIST_TOL = {1: 1, 2: 2, 3: 2, 4: 3, 5: 3, 6: 0}
#: default colors for particular label
DICT_COLOURS = {
    0: (0, 0, 255),  # blue
    1: (255, 0, 0),  # red
    2: (0, 255, 0),  # green
    3: (255, 229, 0),  # yellow
    4: (142, 68, 173),  # purple
    5: (127, 140, 141),  # gray
    6: (0, 212, 255),  # blue
    7: (128, 0, 0),  # brown
}

#: largest palette of the device kernels
PALETTE_MAX = 1024
_EXACT, _NEAREST = 0, 1


# ---------------------------------------------------------------------------------------------------------------------
# colour histogram (device)
# ---------------------------------------------------------------------------------------------------------------------

def _uint8_channels(img):
    """(contiguous uint8 image, channels) of an image for the colour histogram: grey [H, W], or [H, W, 3 | 4]"""
    img = np.asarray(img)
    if img.ndim == 2:
        return np.ascontiguousarray(img, dtype=np.uint8), 1
    if img.ndim == 3 and img.shape[2] in (3, 4):
        return np.ascontiguousarray(img, dtype=np.uint8), img.shape[2]
    raise ValueError('a grey [H, W] or an RGB / RGBA [H, W, 3 | 4] image is required, got shape %r' % (img.shape, ))


def _color_counts(img):
    """(packed colours int64, counts int64) of every colour present in the image, ascending packed order"""
    img, channels = _uint8_channels(img)
    n_px = img.shape[0] * img.shape[1]
    if n_px == 0:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    eng = get_engine()
    torch, lib, st = eng.torch, eng.lib, _lib.stream_ptr()
    d_img = eng.to_device(img, 'ann_img_u8')
    hist = eng.buf('ann_hist', 1 << 24, torch.int64)
    _lib.check(lib.isb_color_hist(_lib.ptr(d_img), C.c_longlong(n_px), channels, 0, _lib.ptr(hist), st))
    ws_bytes = lib.isb_color_hist_workspace_bytes()
    ws = eng.buf('ann_hist_ws', ws_bytes, torch.uint8)
    total = eng.buf('ann_hist_total', 1, torch.int64)
    _lib.check(lib.isb_color_hist_compact_count(_lib.ptr(hist), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(total), st))
    n = int(eng.to_host(total)[0])
    colors = eng.buf('ann_colors', n, torch.int32)
    counts = eng.buf('ann_counts', n, torch.int64)
    _lib.check(lib.isb_color_hist_compact_write(_lib.ptr(hist), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(colors), _lib.ptr(counts), st))
    (h_colors, h_counts), done = eng.download([colors, counts])
    done.synchronize()
    return h_colors.numpy().astype(np.int64), h_counts.numpy().copy()


def _unpack(packed):
    """list of (r, g, b) tuples of packed colours"""
    return list(zip(((packed >> 16) & 255).tolist(), ((packed >> 8) & 255).tolist(), (packed & 255).tolist()))


def unique_image_colors(img):
    """ every colour of the image as a list of (r, g, b), in ascending packed order (reference annotation.py:46-68); the image is
    taken as uint8, grey maps to (v, v, v) and the alpha of RGBA is ignored

    >>> np.random.seed(0)
    >>> img = np.random.randint(0, 2, (50, 50, 3))
    >>> unique_image_colors(img)  # doctest: +NORMALIZE_WHITESPACE
    [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]
    """
    packed, _ = _color_counts(img)
    return _unpack(packed)


def image_frequent_colors(img, ratio_threshold=1e-3):
    """ the colours covering at least ``ratio_threshold`` of the pixels, with their pixel counts (reference annotation.py:163-193);
    keys are (r, g, b) tuples, grey levels for a grey image, in ascending order

    >>> np.random.seed(0)
    >>> img = np.random.randint(0, 2, (50, 50, 3)).astype(np.uint8)
    >>> d = image_frequent_colors(img)
    >>> sorted(d.keys()) # doctest: +NORMALIZE_WHITESPACE
    [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]
    >>> sorted(d.values()) # doctest: +NORMALIZE_WHITESPACE
    [271, 289, 295, 317, 318, 330, 335, 345]
    """
    img = np.asarray(img)
    if img.ndim == 3:
        img = img[:, :, :3]
    nb_pixels = int(np.prod(img.shape[:2]))
    nb_px_min = nb_pixels * ratio_threshold
    packed, counts = _color_counts(img)
    keep = counts >= nb_px_min
    if img.ndim == 2:
        keys = (packed[keep] & 255).tolist()
    else:
        keys = _unpack(packed[keep])
    dict_clrs = dict(zip(keys, counts[keep].tolist()))
    if nb_pixels:
        ration_main_colors = sum(dict_clrs.values()) / float(nb_pixels)
        logging.debug('image main colors=%f and other=%f with colours: \n%r', ration_main_colors, 1. - ration_main_colors, dict_clrs)
    return dict_clrs


def _read_image(path_img):
    from PIL import Image
    with Image.open(path_img) as im:
        if im.mode not in ('L', 'RGB', 'RGBA'):
            im = im.convert('RGB')
        return np.array(im)


def group_images_frequent_colors(paths_img, ratio_threshold=1e-3):
    """ the frequent colours of every image (``image_frequent_colors``, each image with its own threshold) summed over the images
    (reference annotation.py:196-223); the files are read with PIL """
    logging.debug('passing %i images', len(paths_img))
    dict_colors = {}
    for path_im in paths_img:
        for clr, nb in image_frequent_colors(_read_image(path_im), ratio_threshold).items():
            dict_colors[clr] = dict_colors.get(clr, 0) + nb
    logging.info('img folder colours: %r', dict_colors)
    return dict_colors


# ---------------------------------------------------------------------------------------------------------------------
# palettes (device)
# ---------------------------------------------------------------------------------------------------------------------

def _palette_pair(img, colors):
    """(pixels [n, C], palette [P, C]) of one element type: uint8 when the image is uint8 and every colour an integer in [0, 255],
    float64 otherwise"""
    img = np.asarray(img)
    if img.dtype.kind not in 'biuf':
        raise TypeError('images must be real numbers, got %s' % img.dtype)
    if img.ndim < 2:
        raise ValueError('an image [..., channels] is required, got shape %r' % (img.shape, ))
    channels = img.shape[-1]
    try:
        pal = np.asarray(list(colors), dtype=np.float64)
    except (TypeError, ValueError) as err:
        raise ValueError('colours must be numeric sequences of one length: %s' % err)
    if len(pal) == 0:
        raise ValueError('no colours given')
    if pal.ndim != 2 or pal.shape[1] != channels:
        raise ValueError('colours of %r components for an image of %d channels' % (pal.shape[1:], channels))
    if not 1 <= channels <= 4:
        raise ValueError('images with 1 .. 4 channels are supported, got %d' % channels)
    if len(pal) > PALETTE_MAX:
        raise NotImplementedError('a palette of %d colours is above the limit of %d' % (len(pal), PALETTE_MAX))
    if img.dtype == np.uint8 and np.all(np.isfinite(pal)) and np.all(pal == np.round(pal)) and pal.min() >= 0 and pal.max() <= 255:
        return np.ascontiguousarray(img).reshape(-1, channels), pal.astype(np.uint8)
    return np.ascontiguousarray(img, dtype=np.float64).reshape(-1, channels), pal


def _palette_labels(eng, pixels, pal, mode, values=None, want_matched=False):
    """(device int64 labels [n], device matched mask or None, unmatched count or None) of ``isb_palette_map``"""
    torch, lib = eng.torch, eng.lib
    n, channels = pixels.shape
    d_px = eng.to_device(pixels, 'ann_pixels')
    d_pal = eng.to_device(pal, 'ann_palette')
    d_val = None if values is None else eng.to_device(np.ascontiguousarray(values, dtype=np.int64), 'ann_values')
    labels = eng.buf('ann_labels', n, torch.int64)
    matched = eng.buf('ann_matched', n, torch.uint8) if want_matched else None
    unmatched = eng.buf('ann_unmatched', 1, torch.int64) if mode == _EXACT else None
    _lib.check(lib.isb_palette_map(_lib.ptr(d_px), _lib.dtype_code(pixels.dtype), C.c_longlong(n), channels, _lib.ptr(d_pal), len(pal), mode,
                                   _lib.ptr(d_val), _lib.ptr(labels), _lib.ptr(matched), _lib.ptr(unmatched), _lib.stream_ptr()))
    miss = None if unmatched is None else int(eng.to_host(unmatched)[0])
    return labels, matched, miss


def _gather_colors(eng, d_labels, table, keys=None, name='ann_gathered'):
    """(device bytes of table[row of label] for every label, missing count): ``isb_palette_gather``"""
    torch, lib = eng.torch, eng.lib
    table = np.ascontiguousarray(table)
    if len(table) > PALETTE_MAX:
        raise NotImplementedError('a palette of %d colours is above the limit of %d' % (len(table), PALETTE_MAX))
    row_bytes = table.nbytes // len(table)
    if not 1 <= row_bytes <= 32:
        raise ValueError('a colour of %d bytes is outside 1 .. 32' % row_bytes)
    n = int(d_labels.numel())
    d_table = eng.to_device(table.view(np.uint8).reshape(-1), 'ann_table')
    d_keys = None if keys is None else eng.to_device(np.ascontiguousarray(keys, dtype=np.int64), 'ann_keys')
    out = eng.buf(name, n * row_bytes, torch.uint8)
    missing = eng.buf('ann_missing', 1, torch.int64)
    _lib.check(lib.isb_palette_gather(_lib.ptr(d_labels), C.c_longlong(n), _lib.ptr(d_keys), len(table), _lib.ptr(d_table), row_bytes,
                                      _lib.ptr(out), _lib.ptr(missing), _lib.stream_ptr()))
    return out, int(eng.to_host(missing)[0])


def _host_table(d_bytes, dtype, shape):
    eng = get_engine()
    return eng.to_host(d_bytes).view(dtype).reshape(shape).copy()


def convert_img_colors_to_labels(img_rgb, lut_label_color):
    """ label map of an RGB image through {label: colour} (reference annotation.py:71-91); a colour given for several labels takes
    the last of them.  ``ValueError`` when a pixel has none of the colours

    >>> np.random.seed(0)
    >>> seg = np.random.randint(0, 2, (5, 7))
    >>> img = np.array([(0.2, 0.2, 0.2), (0.9, 0.9, 0.9)])[seg]
    >>> d_lb_clr = {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)}
    >>> convert_img_colors_to_labels(img, d_lb_clr)
    array([[0, 1, 1, 0, 1, 1, 1],
           [1, 1, 1, 1, 0, 0, 1],
           [0, 0, 0, 0, 0, 1, 0],
           [1, 1, 0, 0, 1, 1, 1],
           [1, 0, 1, 0, 1, 0, 1]])
    """
    dict_color_label = {lut_label_color[k]: k for k in lut_label_color}
    return convert_img_colors_to_labels_reverted(img_rgb, dict_color_label)


def convert_img_colors_to_labels_reverted(img_rgb, dict_color_label):
    """ label map of an image [..., channels] through {colour: label} (reference annotation.py:94-125): int64 labels (float labels
    truncated, as the reference's float map cast to ``np.int``); ``ValueError`` when a pixel has none of the colours """
    img_rgb = np.asarray(img_rgb)
    shape = img_rgb.shape[:-1]
    if img_rgb.size == 0:
        return np.zeros(shape, dtype=np.int64)
    if not dict_color_label:
        raise ValueError('There is different number of pixels than number of converted labels.')
    colors = list(dict_color_label)
    values = np.asarray([dict_color_label[c] for c in colors], dtype=np.float64).astype(np.int64)
    pixels, pal = _palette_pair(img_rgb, colors)
    eng = get_engine()
    labels, _, miss = _palette_labels(eng, pixels, pal, _EXACT, values)
    if miss:
        raise ValueError('There is different number of pixels than number of converted labels.')
    return eng.to_host(labels).reshape(shape).copy()


def convert_img_labels_to_colors(segm, lut_label_colors):
    """ colour image of a label map through {label: colour} (reference annotation.py:128-160): [*segm.shape, channels] in the dtype of
    all the dictionary's colours; ``ValueError`` when a label has no colour

    >>> np.random.seed(0)
    >>> seg = np.random.randint(0, 2, (5, 7))
    >>> d_lb_clr = {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)}
    >>> img = convert_img_labels_to_colors(seg, d_lb_clr)
    >>> img[:, :, 0]
    array([[0.2, 0.9, 0.9, 0.2, 0.9, 0.9, 0.9],
           [0.9, 0.9, 0.9, 0.9, 0.2, 0.2, 0.9],
           [0.2, 0.2, 0.2, 0.2, 0.2, 0.9, 0.2],
           [0.9, 0.9, 0.2, 0.2, 0.9, 0.9, 0.9],
           [0.9, 0.2, 0.9, 0.2, 0.9, 0.2, 0.9]])
    """
    segm = np.asarray(segm)
    if segm.dtype.kind not in 'biuf':
        raise TypeError('label maps must hold numbers, got %s' % segm.dtype)
    if segm.dtype.kind == 'f':
        if not np.all(np.floor(segm) == segm):
            raise ValueError('labels must be integers')
        segm = segm.astype(np.int64)
    keys = sorted(int(k) for k in lut_label_colors if float(k) == int(k))
    if not keys:
        raise ValueError('some labels %r are missing in dictionary %r' % (np.unique(segm), lut_label_colors.keys()))
    table = np.asarray([lut_label_colors[k] for k in keys])
    if table.dtype.kind not in 'biuf':
        raise ValueError('colours must be numeric sequences of one length')
    out_shape = segm.shape + table.shape[1:]
    if segm.size == 0:
        return np.zeros(out_shape, dtype=table.dtype)
    eng = get_engine()
    d_seg = eng.to_device(np.ascontiguousarray(segm, dtype=np.int64).reshape(-1), 'ann_segm')
    out, missing = _gather_colors(eng, d_seg, table, keys)
    if missing:
        raise ValueError('some labels %r are missing in dictionary %r' % (np.unique(segm), lut_label_colors.keys()))
    return _host_table(out, table.dtype, out_shape)


def image_color_2_labels(img, colors=None):
    """ index of the L1-nearest colour of every pixel of an [H, W, 3] image (reference annotation.py:226-249), the first of equally
    near colours; without ``colors`` the image's frequent colours

    >>> np.random.seed(0)
    >>> rand = np.random.randint(0, 2, (5, 7)).astype(np.uint8)
    >>> img = np.rollaxis(np.array([rand] * 3), 0, 3)
    >>> image_color_2_labels(img)   # the frequent colours in ascending order: (0, 0, 0), (1, 1, 1)
    array([[0, 1, 1, 0, 1, 1, 1],
           [1, 1, 1, 1, 0, 0, 1],
           [0, 0, 0, 0, 0, 1, 0],
           [1, 1, 0, 0, 1, 1, 1],
           [1, 0, 1, 0, 1, 0, 1]])
    """
    img = np.asarray(img)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('an RGB image [H, W, 3] is required, got shape %r' % (img.shape, ))
    if not colors:
        colors = image_frequent_colors(img).keys()
    if img.size == 0:
        return np.zeros(img.shape[:2], dtype=np.int64)
    pixels, pal = _palette_pair(img, colors)
    eng = get_engine()
    labels, _, _ = _palette_labels(eng, pixels, pal, _NEAREST)
    return eng.to_host(labels).reshape(img.shape[:2]).copy()


def quantize_image_nearest_color(img, colors):
    """ every pixel of an [H, W, 3] image replaced by its L1-nearest colour, cast to the image's dtype
    (reference annotation.py:252-276)

    >>> np.random.seed(0)
    >>> img = np.random.randint(0, 2, (5, 7, 3)).astype(np.uint8)
    >>> im = quantize_image_nearest_color(img, [(0, 0, 0), (1, 1, 1)])
    >>> im[:, :, 0]
    array([[1, 1, 1, 1, 0, 0, 0],
           [1, 1, 1, 1, 1, 1, 0],
           [1, 1, 0, 1, 1, 0, 1],
           [0, 0, 1, 0, 1, 0, 1],
           [1, 1, 1, 0, 1, 0, 0]], dtype=uint8)
    """
    img = np.asarray(img)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('an RGB image [H, W, 3] is required, got shape %r' % (img.shape, ))
    pixels, pal = _palette_pair(img, colors)
    table = np.asarray(list(colors)).astype(img.dtype)
    if img.size == 0:
        return np.zeros(img.shape, dtype=img.dtype)
    eng = get_engine()
    labels, _, _ = _palette_labels(eng, pixels, pal, _NEAREST)
    out, _ = _gather_colors(eng, labels, table)
    return _host_table(out, img.dtype, img.shape)


# ---------------------------------------------------------------------------------------------------------------------
# nearest valid pixel (device)
# ---------------------------------------------------------------------------------------------------------------------

def _nearest_site_index(eng, d_valid, shape):
    """device int32 [H * W]: flat index of a nearest valid pixel (isb_edt_2d_indices)"""
    H, W = shape
    if H > 32768 or W > 32768:
        raise ValueError('the distance transform takes images up to 32768 x 32768, got %r' % (shape, ))
    torch, lib = eng.torch, eng.lib
    ws_bytes = lib.isb_edt_index_workspace_bytes(H, W)
    ws = eng.buf('edt_ws', ws_bytes, torch.uint8)
    index = eng.buf('ann_site_index', H * W, torch.int32)
    _lib.check(lib.isb_edt_2d_indices(_lib.ptr(d_valid), H, W, _lib.ptr(index), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.stream_ptr()))
    return index


def _gather_at(eng, d_src, itemsize, d_index, name):
    torch = eng.torch
    n = int(d_index.numel())
    out = eng.buf(name, n * itemsize, torch.uint8)
    _lib.check(eng.lib.isb_gather_at_index(_lib.ptr(d_src), itemsize, _lib.ptr(d_index), C.c_longlong(n), _lib.ptr(out), _lib.stream_ptr()))
    return out


def image_inpaint_pixels(img, valid_mask):
    """ every pixel of a 2-D image replaced by the value of a nearest valid pixel (reference annotation.py:279-286, a KD-tree over
    the valid pixels there): nonzero ``valid_mask`` marks the valid pixels; of equidistant ones the smallest column, then the smallest
    row wins, as in ``scipy.ndimage.distance_transform_edt(..., return_indices=True)``.  Same dtype as ``img``

    >>> img = np.array([[1., 0, 0, 0], [0, 0, 0, 2]])
    >>> image_inpaint_pixels(img, img > 0)
    array([[1., 1., 1., 2.],
           [1., 1., 2., 2.]])
    """
    img, valid_mask = np.asarray(img), np.asarray(valid_mask)
    if img.shape != valid_mask.shape:
        raise ImageDimensionError('image size %r and mask size %r should be equal' % (img.shape, valid_mask.shape))
    if img.ndim != 2:
        raise ValueError('image_inpaint_pixels takes 2-D images (the label maps of this package), got shape %r' % (img.shape, ))
    if img.dtype.itemsize not in (1, 2, 4, 8) or img.dtype.kind not in 'biuf':
        raise TypeError('images of 1, 2, 4 or 8-byte numbers are supported, got %s' % img.dtype)
    valid = valid_mask.view(np.uint8) if valid_mask.dtype == bool else (valid_mask != 0).view(np.uint8)
    if img.size == 0 or not valid.any():
        raise ValueError('no valid pixel to inpaint from')
    eng = get_engine()
    d_valid = eng.to_device(valid, 'ann_valid')
    index = _nearest_site_index(eng, d_valid, img.shape)
    d_img = eng.to_device(np.ascontiguousarray(img).reshape(-1).view(np.uint8), 'ann_inpaint_src')
    out = _gather_at(eng, d_img, img.dtype.itemsize, index, 'ann_inpainted')
    return _host_table(out, img.dtype, img.shape)


def quantize_image_nearest_pixel(img, colors):
    """ every pixel of an [H, W, channels] image that has none of ``colors`` takes the colour of a nearest pixel that has one
    (reference annotation.py:289-321); equal colours in the list: the last one's index counts.  The result holds the colours as
    ``np.asarray(colors)`` does

    >>> np.random.seed(0)
    >>> img = np.random.randint(0, 2, (5, 7, 3)).astype(np.uint8)
    >>> im = quantize_image_nearest_pixel(img, [(0, 0, 0), (1, 1, 1)])
    >>> im[:, :, 0]     # the reference's KD-tree breaks the ties at (1, 4), (2, 5), (3, 0) and (4, 1) the other way
    array([[1, 1, 1, 1, 0, 0, 0],
           [1, 1, 1, 1, 1, 0, 0],
           [1, 1, 1, 1, 1, 1, 0],
           [1, 0, 0, 0, 0, 0, 0],
           [1, 1, 0, 0, 0, 0, 0]])
    """
    img = np.asarray(img)
    if img.ndim != 3:
        raise ValueError('an image [H, W, channels] is required, got shape %r' % (img.shape, ))
    pixels, pal = _palette_pair(img, colors)
    table = np.asarray(list(colors))
    if img.size == 0:
        raise ValueError('no valid pixel to inpaint from')
    eng = get_engine()
    labels, matched, miss = _palette_labels(eng, pixels, pal, _EXACT, want_matched=True)
    if miss == labels.numel():
        raise ValueError('no pixel of the image has one of the colours')
    index = _nearest_site_index(eng, matched, img.shape[:2])
    near = _gather_at(eng, labels, 8, index, 'ann_near_labels').view(eng.torch.int64)
    out, _ = _gather_colors(eng, near, table)
    return _host_table(out, table.dtype, img.shape[:2] + table.shape[1:])


# ---------------------------------------------------------------------------------------------------------------------
# annotation tables (host)
# ---------------------------------------------------------------------------------------------------------------------

def load_info_group_by_slices(path_txt, stages, pos_columns=COLUMNS_POSITION, dict_slice_tol=ANNOT_SLICE_DIST_TOL):
    """ the positions of every image of the selected stages, each with those of the slices of its stack within the stage's tolerance
    (reference annotation.py:324-370): a DataFrame indexed by image name whose cells are arrays """
    import pandas as pd
    logging.info('loading info file and filter stages...')
    df = pd.read_csv(path_txt, sep='\t', index_col=0)
    logging.debug('loaded %i records', len(df))
    df = df[df['stage'].isin(list(stages))]
    logging.debug('filtered %i records', len(df))
    df = df.sort_values(['stage'], ascending=False)
    rows = []
    logging.info('grouping info by stacks...')
    for _, df_group in df.groupby(SLICE_NAME_GROUPING):
        slice_idxs = df_group['slice_index'].values
        slice_tols = np.array([dict_slice_tol[i] for i in df_group['stage'].values])
        for _, row in df_group.iterrows():
            filter_slice = abs(slice_idxs - row['slice_index']) <= slice_tols
            dict_slice = {col: df_group[col].values[filter_slice] for col in pos_columns}
            dict_slice['image'] = os.path.splitext(row['image_path'])[0]
            rows.append(dict_slice)
    if not rows:
        return pd.DataFrame()
    df_marked = pd.concat([pd.DataFrame([r]) for r in rows], ignore_index=True)
    return df_marked.set_index('image')
