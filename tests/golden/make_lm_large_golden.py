"""
Generate tests/golden/lm_large.npz: the reference's OWN Leung-Malik texture descriptor (imsegm/descriptors.py:1041-1106, run from
$IMSEGM_REFERENCE with its Cython module compiled unchanged, see make_goldens.py) on an image LARGER than the sigma-150 background
kernel (1201 taps) on both axes -- 1280 x 1280, textured, full bank (20 batteries, 76 kernels), mean / std / energy.

    python tests/golden/make_lm_large_golden.py         (~10-15 min of CPU: 228 float64 33x33 convolutions of 1280^2 + the blur)

The image and the segmentation are regenerated from seeds by the test (bench.synth_texture_image(SEED, SIDE, SIDE) and a ragged block
segmentation), so the fixture holds only the features of every STRIDE-th segment (float64) and check sums of the inputs.
"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

SIDE, SEED, CELL, STRIDE = 1280, 3100, 32, 3


def make_inputs():
    """the textured image of bench.py's config 3 (four classes, sinusoidal textures of period 4..32 px) and a superpixel-like
    segmentation: 32 x 32 blocks with ragged borders, 1 600 labels"""
    import bench
    img = bench.synth_texture_image(SEED, SIDE, SIDE)
    rng = np.random.RandomState(SEED + 1)
    yy, xx = np.mgrid[:SIDE, :SIDE]
    jy = (rng.rand(SIDE, SIDE) < 0.08) * rng.randint(-3, 4, (SIDE, SIDE))
    by = np.clip((yy + jy) // CELL, 0, SIDE // CELL - 1)
    bx = np.clip((xx + jy.T) // CELL, 0, SIDE // CELL - 1)
    seg = (by * (SIDE // CELL) + bx).astype(np.int64)
    return img, seg


def main():
    from make_goldens import import_reference
    ref = import_reference()
    ds = ref['descriptors']
    img, seg = make_inputs()
    t0 = time.time()
    fts, names = ds.compute_texture_desc_lm_img2d_clr(img, seg, ('mean', 'std', 'energy'), 'normal')
    print('reference compute_texture_desc_lm_img2d_clr: %.0f s, features %r' % (time.time() - t0, fts.shape))
    rows = np.arange(0, fts.shape[0], STRIDE)
    out = dict(side=SIDE, seed=SEED, rows=rows, features=fts[rows], names=np.array(names),
               img_sum=float(img.sum()), seg_sum=int(seg.sum()), nb_segments=int(seg.max()) + 1,
               # per battery and channel: the largest energy over ALL segments (the response scale the tolerance is relative to)
               energy_max=np.abs(fts).reshape(fts.shape[0], 20, 3, 3)[:, :, 2, :].max(axis=0))
    path = os.path.join(HERE, 'lm_large.npz')
    np.savez_compressed(path, **out)
    print('wrote %s, %.0f KB' % (path, os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
