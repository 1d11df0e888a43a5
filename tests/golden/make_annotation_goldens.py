"""
Generate tests/golden/annotation_reference.npz by RUNNING THE REFERENCE'S imsegm/annotation.py on the inputs of its doctests.

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_annotation_goldens.py

PIL, pandas and scipy are the real packages; the reference's other imports that are not installable here (scikit-image, nibabel,
tqdm, matplotlib, the OLE readers) are inert stubs, which no function called below touches; ``np.int`` is read as ``int`` and ``np.product`` as ``np.prod``.  Nothing of the
reference is copied: this script calls it and stores inputs and outputs.  ``load_info_group_by_slices`` cannot run on current pandas
(``DataFrame.append`` is gone), so the test pins the table its doctest prints.
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ['IMSEGM_REFERENCE']


def import_reference():
    for name, val in (('int', int), ('product', np.prod)):
        if not hasattr(np, name):       # NumPy-2 removed aliases the reference still uses
            setattr(np, name, val)

    class Stub(types.ModuleType):
        __path__ = []

        def __getattr__(self, k):
            if k.startswith('__'):
                raise AttributeError(k)
            m = Stub(self.__name__ + '.' + k)
            setattr(self, k, m)
            sys.modules[self.__name__ + '.' + k] = m
            return m

        def __call__(self, *a, **k):
            return Stub('call')

        def __getitem__(self, k):
            return 'agg'

    for root in ('skimage', 'nibabel', 'tqdm', 'matplotlib', 'olefile', 'OleFileIO_PL'):
        sys.modules.setdefault(root, Stub(root))
    for sub in ('skimage.color', 'skimage.exposure', 'skimage.io', 'skimage.measure', 'matplotlib.pyplot'):
        root, leaf = sub.split('.', 1)
        getattr(sys.modules[root], leaf)
    sys.path.insert(0, REF)
    return importlib.import_module('imsegm.annotation')


def main():
    an = import_reference()
    out = {}
    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3))
    out['unique_colors'] = np.array(an.unique_image_colors(img))
    img = np.random.randint(0, 256, (150, 150, 3))
    out['unique_img_rand'] = img.astype(np.uint8)
    out['unique_colors_rand'] = np.array(an.unique_image_colors(img), dtype=np.uint8)

    np.random.seed(0)
    seg = np.random.randint(0, 2, (5, 7))
    img = np.array([(0.2, 0.2, 0.2), (0.9, 0.9, 0.9)])[seg]
    out['convert_seg'] = seg
    out['convert_labels'] = an.convert_img_colors_to_labels(img, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)})
    out['convert_labels_reverted'] = an.convert_img_colors_to_labels_reverted(img, {(0.2, 0.2, 0.2): 0, (0.9, 0.9, 0.9): 1})
    out['labels_to_colors'] = an.convert_img_labels_to_colors(seg, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)})

    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3)).astype(np.uint8)
    d = an.image_frequent_colors(img)
    out['frequent_colors'] = np.array(list(d.keys()))
    out['frequent_counts'] = np.array(list(d.values()))

    np.random.seed(0)
    rand = np.random.randint(0, 2, (5, 7)).astype(np.uint8)
    img = np.rollaxis(np.array([rand] * 3), 0, 3)
    out['color_2_labels_img'] = img
    out['color_2_labels_colors'] = np.array(list(an.image_frequent_colors(img).keys()))
    out['color_2_labels'] = an.image_color_2_labels(img)

    np.random.seed(0)
    img = np.random.randint(0, 2, (5, 7, 3)).astype(np.uint8)
    out['quantize_img'] = img
    out['quantize_nearest_color'] = an.quantize_image_nearest_color(img, [(0, 0, 0), (1, 1, 1)])
    out['quantize_nearest_pixel'] = an.quantize_image_nearest_pixel(img, [(0, 0, 0), (1, 1, 1)])

    rng = np.random.RandomState(11)
    vals = rng.rand(23, 31)
    valid = rng.rand(23, 31) < 0.1
    out.update(inpaint_img=vals, inpaint_valid=valid, inpaint=an.image_inpaint_pixels(vals, valid))
    return out


if __name__ == '__main__':
    vectors = main()
    path = os.path.join(HERE, 'annotation_reference.npz')
    np.savez_compressed(path, **vectors)
    print('wrote %s: %d arrays, %.0f KB' % (path, len(vectors), os.path.getsize(path) / 1024))
