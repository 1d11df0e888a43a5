"""
Generate tests/golden/center_detection_reference.npz: two images of the reference's ``data-images/drosophila_ovary_slice`` with
their 4-class segmentation, their 3-level centre annotation and their annotated centres, the inputs of the reference's centre
detection experiment (experiments_ovary_centres).  Data only.

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_center_goldens.py

Per image ``<name>``: ``<name>/image.jpg``, ``<name>/segm.png`` (labels 0..3) and ``<name>/center_levels.png`` (0..3) as the
files' bytes (u8 vectors; :func:`load` decodes them with PIL), and ``<name>/centers_xy`` [k, 2] f64, the (X, Y) columns of the
centres' CSV.
"""
import csv
import io
import os

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ('insitu7545', 'insitu4174')


def load(npz, name):
    """(image [H, W, 3] u8, segm [H, W] u8, center_levels [H, W] u8, centres [k, 2] as (row, col)) of one image of the file"""
    def dec(key, mode):
        return np.array(Image.open(io.BytesIO(npz[name + '/' + key].tobytes())).convert(mode), dtype=np.uint8)
    return dec('image.jpg', 'RGB'), dec('segm.png', 'L'), dec('center_levels.png', 'L'), npz[name + '/centers_xy'][:, ::-1].copy()


def main():
    ref = os.environ.get('IMSEGM_REFERENCE')
    if not ref:
        raise SystemExit('set IMSEGM_REFERENCE to a checkout of the reference')
    base = os.path.join(ref, 'data-images', 'drosophila_ovary_slice')
    arrays = {}
    for name in NAMES:
        for key, path in (('image.jpg', ('image', name + '.jpg')), ('segm.png', ('segm', name + '.png')),
                          ('center_levels.png', ('center_levels', name + '.png'))):
            with open(os.path.join(base, *path), 'rb') as fp:
                arrays[name + '/' + key] = np.frombuffer(fp.read(), dtype=np.uint8)
        with open(os.path.join(base, 'center_levels', name + '.csv')) as fp:
            rows = list(csv.DictReader(fp))
        arrays[name + '/centers_xy'] = np.array([[float(r['X']), float(r['Y'])] for r in rows], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, 'center_detection_reference.npz'), names=np.array(NAMES), **arrays)


if __name__ == '__main__':
    main()
