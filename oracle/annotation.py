"""
Host oracle of ``imsegm/annotation.py`` (numpy / PIL / scipy only; test infrastructure, never imported by the product).

Each function restates the plain meaning of the reference: colour lists from PIL's ``getcolors`` (so in PIL's order), one full-image
comparison per palette colour, the palette x pixels L1 distance matrix with ``np.argmin``, and the nearest valid pixel from scipy's
``NearestNDInterpolator`` over the valid pixels.  ``np.int`` (removed in numpy 1.24) is read as ``int``.
"""
import numpy as np
from PIL import Image
from scipy import interpolate


class ImageDimensionError(ValueError):
    pass


def unique_image_colors(img):
    image = Image.fromarray(np.asarray(img, dtype=np.uint8)).convert('RGB')
    n_px = int(np.prod(np.asarray(img).shape[:2]))
    return [clr for _, clr in image.getcolors(maxcolors=max(n_px, 1))]


def image_frequent_colors(img, ratio_threshold=1e-3):
    img = np.asarray(img)
    if img.ndim == 3:
        img = img[:, :, :3]
    n_px = int(np.prod(img.shape[:2]))
    colors = Image.fromarray(img).getcolors(maxcolors=n_px)
    if not colors:
        return {}
    return {clr: nb for nb, clr in colors if nb >= n_px * ratio_threshold}


def group_images_frequent_colors(paths_img, ratio_threshold=1e-3):
    total = {}
    for path in paths_img:
        with Image.open(path) as im:
            img = np.asarray(im if im.mode in ('L', 'RGB', 'RGBA') else im.convert('RGB'))
        for clr, nb in image_frequent_colors(img, ratio_threshold).items():
            total[clr] = total.get(clr, 0) + nb
    return total


def convert_img_colors_to_labels_reverted(img_rgb, dict_color_label):
    img_rgb = np.asarray(img_rgb)
    labels = np.zeros(img_rgb.shape[:-1])
    n_converted = 0
    for color, label in dict_color_label.items():
        hit = np.all(img_rgb == color, axis=-1)
        labels[hit] = label
        n_converted += int(hit.sum())
    if n_converted != labels.size:
        raise ValueError('There is different number of pixels than number of converted labels.')
    return labels.astype(int)


def convert_img_colors_to_labels(img_rgb, lut_label_color):
    return convert_img_colors_to_labels_reverted(img_rgb, {clr: lb for lb, clr in lut_label_color.items()})


def convert_img_labels_to_colors(segm, lut_label_colors):
    segm = np.asarray(segm)
    present = np.unique(segm)
    if not all(lb in lut_label_colors for lb in present):
        raise ValueError('some labels %r are missing in dictionary %r' % (present, lut_label_colors.keys()))
    lo, hi = int(segm.min()), int(segm.max())
    lut = [lut_label_colors.get(lb) for lb in range(lo, hi + 1)]
    return np.array(lut)[np.asarray(segm - lo, dtype=int)]


def _l1_nearest(img, colors):
    pixels = np.asarray(img).reshape(-1, 3)
    dist = np.array([np.sum(np.abs(np.subtract(pixels, clr)), axis=1) for clr in colors])
    return np.argmin(dist, axis=0)


def image_color_2_labels(img, colors=None):
    if not colors:
        colors = image_frequent_colors(img).keys()
    return _l1_nearest(img, list(colors)).reshape(np.asarray(img).shape[:2])


def quantize_image_nearest_color(img, colors):
    img = np.asarray(img)
    return np.asarray(np.asarray(colors)[_l1_nearest(img, colors)], dtype=img.dtype).reshape(img.shape)


def image_inpaint_pixels(img, valid_mask):
    img, valid_mask = np.asarray(img), np.asarray(valid_mask, dtype=bool)
    if img.shape != valid_mask.shape:
        raise ImageDimensionError('image size %r and mask size %r should be equal' % (img.shape, valid_mask.shape))
    near = interpolate.NearestNDInterpolator(np.argwhere(valid_mask), img[valid_mask])
    return near(np.indices(img.shape).reshape(img.ndim, -1).T).reshape(img.shape)


def quantize_image_nearest_pixel(img, colors):
    img = np.asarray(img)
    labels = np.full(img.shape[:-1], np.nan)
    for i, clr in enumerate(colors):
        labels[np.sum(np.abs(img - np.tile(clr, labels.shape + (1, ))), axis=-1) == 0] = i
    valid = ~np.isnan(labels)
    return np.asarray(colors)[image_inpaint_pixels(labels, valid).astype(int)]
