"""
Generate tests/golden/median_reference.npz by RUNNING THE REFERENCE'S numpy_img2d_color_median, numpy_img3d_gray_median and
compute_image2d_color_statistic(..., ('median',)) on small inputs (the reference loops over the pixels in Python).

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_median_goldens.py   (needs `make -C oracle ref`, as make_goldens.py)

The cases are the ones where np.median in the image's own dtype matters: a float32 image whose labels all have an even count (the
two middle values are averaged in float32), float64 and float32 images with NaN pixels of either sign and infinite pixels, and a
one-pixel label of 1.5e308 (twice it overflows).  Every case has a label without pixels.  Nothing of the reference is copied: this
script calls it and stores inputs and outputs.
"""
import os
import warnings

import numpy as np

from make_goldens import HERE, import_reference


def cases(rng):
    """name -> (image [H, W, 3], labels [H, W])"""
    out = {}
    # float32 noise, 9 labels of 2 to 16 pixels each (all even), label 4 absent
    h, w = 12, 16
    sizes = [2, 4, 6, 8, 0, 10, 12, 14, 16, 120]
    seg = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(seg)
    img = (rng.random_sample((h, w, 3)) * 3 - 1).astype(np.float32)
    out['f32_even'] = (img, seg.reshape(h, w))
    # NaN of either sign bit and +-inf; labels of odd and even count
    h, w = 10, 14
    seg = rng.randint(0, 7, (h, w))
    seg[seg == 5] = 6                                                  # label 5 absent
    seg[0, :4] = 7                                                     # label 7: four +inf in channel 0 (two middles inf)
    for dt in (np.float64, np.float32):
        img = rng.normal(0, 1, (h, w, 3)).astype(dt)
        img[0, :4, 0] = np.inf
        img[seg == 1, 1] = -np.inf
        flat = img.reshape(-1, 3)
        for lb, sign in ((2, 1.), (3, -1.)):                          # one NaN in label 2 (sign clear) and label 3 (sign set)
            p = np.flatnonzero(seg.ravel() == lb)[0]
            flat[p, lb - 2] = np.copysign(np.nan, sign)
        out['%s_nan' % np.dtype(dt).name] = (img, seg.copy())
    # a one-pixel label of 1.5e308 and a one-pixel label of -1.5e308 among ordinary ones
    h, w = 6, 8
    seg = np.arange(h * w).reshape(h, w) // 5
    seg[seg == 3] = 2                                                  # label 3 absent
    seg[5, 6], seg[5, 7] = seg.max() + 1, seg.max() + 2
    img = rng.random_sample((h, w, 3))
    img[5, 6], img[5, 7] = 1.5e308, -1.5e308
    out['f64_huge'] = (img, seg)
    return out


def main():
    ref = import_reference()
    ds = ref['descriptors']
    rng = np.random.RandomState(20261016)
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)               # np.median of an absent label's empty list is NaN
        for name, (img, seg) in cases(rng).items():
            out[name + '_img'], out[name + '_seg'] = img, seg
            out[name + '_color'] = ds.numpy_img2d_color_median(img, seg)
            out[name + '_gray'] = ds.numpy_img3d_gray_median(img[None, :, :, 0], seg[None])
            out[name + '_table'] = ds.compute_image2d_color_statistic(img, seg, ('median', ))[0]
    return out


if __name__ == '__main__':
    vectors = main()
    path = os.path.join(HERE, 'median_reference.npz')
    np.savez_compressed(path, **vectors)
    print('wrote %s: %d arrays, %.0f KB' % (path, len(vectors), os.path.getsize(path) / 1024))
