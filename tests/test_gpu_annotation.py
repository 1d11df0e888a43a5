"""GPU tests of imsegm.annotation: every function against the host oracle (oracle/annotation.py) and the reference's outputs, on
1x1, 1xN, Nx1, odd sizes across block edges and 4096 x 4096 images.  The colour histogram on a single-colour image, on an image holding
each of the 2^24 colours once and on two images summed in one buffer; palettes with duplicates, L1 ties, absent colours, uint8 and
float64; the nearest valid pixel on single-pixel, one-column, 1 % random, checkerboard and all-valid masks, where the chosen site must
be at scipy's exact distance, equal scipy's own index, and give the oracle's value wherever the nearest valid pixel is unique."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy import ndimage
from scipy.spatial import cKDTree

from oracle import annotation as oa

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SHAPES = [(1, 1), (1, 97), (97, 1), (33, 257), (129, 31), (255, 513)]


@pytest.fixture(scope='module')
def an():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import annotation
    return annotation


def _few_colours(rng, shape, palette):
    return np.asarray(palette, dtype=np.uint8)[rng.randint(0, len(palette), shape)]


def _counts_np(img):
    img = np.asarray(img, dtype=np.uint8)
    rgb = img[..., :3].astype(np.int64) if img.ndim == 3 else np.repeat(img[..., None].astype(np.int64), 3, axis=-1)
    packed = (rgb[..., 0] << 16 | rgb[..., 1] << 8 | rgb[..., 2]).ravel()
    return np.unique(packed, return_counts=True)


def test_reference_outputs_through_device(an):
    gold = dict(np.load(os.path.join(GOLDEN, 'annotation_reference.npz')))
    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3))
    assert an.unique_image_colors(img) == sorted(tuple(c) for c in gold['unique_colors'].tolist())
    assert an.unique_image_colors(gold['unique_img_rand']) == sorted(tuple(c) for c in gold['unique_colors_rand'].tolist())
    seg = gold['convert_seg']
    img = np.array([(0.2, 0.2, 0.2), (0.9, 0.9, 0.9)])[seg]
    got = an.convert_img_colors_to_labels(img, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)})
    assert got.dtype == np.int64 and np.array_equal(got, gold['convert_labels'])
    assert np.array_equal(an.convert_img_colors_to_labels_reverted(img, {(0.2, 0.2, 0.2): 0, (0.9, 0.9, 0.9): 1}), gold['convert_labels_reverted'])
    got = an.convert_img_labels_to_colors(seg, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)})
    assert got.dtype == gold['labels_to_colors'].dtype and np.array_equal(got, gold['labels_to_colors'])
    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3)).astype(np.uint8)
    d = an.image_frequent_colors(img)
    want = dict(zip((tuple(c) for c in gold['frequent_colors'].tolist()), gold['frequent_counts'].tolist()))
    assert d == want and list(d) == sorted(want)
    img = gold['color_2_labels_img']
    colors = [tuple(c) for c in gold['color_2_labels_colors'].tolist()]         # the reference's (PIL's) colour order
    assert np.array_equal(an.image_color_2_labels(img, colors), gold['color_2_labels'])
    assert np.array_equal(an.image_color_2_labels(img), oa.image_color_2_labels(img, sorted(colors)))
    img = gold['quantize_img']
    got = an.quantize_image_nearest_color(img, [(0, 0, 0), (1, 1, 1)])
    assert got.dtype == np.uint8 and np.array_equal(got, gold['quantize_nearest_color'])
    got = an.quantize_image_nearest_pixel(img, [(0, 0, 0), (1, 1, 1)])
    valid = (img[..., None, :] == np.array([(0, 0, 0), (1, 1, 1)], np.uint8)).all(-1).any(-1)
    unique = _unique_nearest(valid)
    assert got.dtype == gold['quantize_nearest_pixel'].dtype and np.array_equal(got[unique], gold['quantize_nearest_pixel'][unique])
    # the reference's KD-tree breaks four ties between differently coloured pixels the other way
    assert np.argwhere((got != gold['quantize_nearest_pixel']).any(-1)).tolist() == [[1, 4], [2, 5], [3, 0], [4, 1]]
    got = an.image_inpaint_pixels(gold['inpaint_img'], gold['inpaint_valid'])
    unique = _unique_nearest(gold['inpaint_valid'])
    assert np.array_equal(got[unique], gold['inpaint'][unique])


def _unique_nearest(valid):
    """pixels whose nearest valid pixel is unique"""
    pts = np.argwhere(valid)
    if len(pts) == 1:
        return np.ones(valid.shape, bool)
    d, _ = cKDTree(pts).query(np.indices(valid.shape).reshape(2, -1).T, k=2)
    return (d[:, 0] < d[:, 1]).reshape(valid.shape)


def test_histogram_sizes_and_channels(an):
    rng = np.random.RandomState(0)
    for shape in SHAPES + [(4096, 4096)]:
        for channels in (None, 3, 4):
            full = shape if channels is None else shape + (channels, )
            img = rng.randint(0, 3, full).astype(np.uint8) * 100 if shape[0] * shape[1] > 10 ** 6 else rng.randint(0, 256, full).astype(np.uint8)
            packed, counts = _counts_np(img)
            got = an.unique_image_colors(img)
            assert got == [tuple(c) for c in np.stack([packed >> 16, packed >> 8 & 255, packed & 255], 1).tolist()], (shape, channels)
            if shape[0] * shape[1] <= 10 ** 5:
                assert sorted(got) == sorted(oa.unique_image_colors(img))
                d = an.image_frequent_colors(img, 0.01)
                assert d == oa.image_frequent_colors(img, 0.01) and list(d) == sorted(d)


def test_histogram_single_colour_and_every_colour(an):
    img = np.full((4096, 4096, 3), (12, 200, 7), np.uint8)
    assert an.image_frequent_colors(img) == {(12, 200, 7): 4096 * 4096}
    every = np.arange(1 << 24, dtype=np.int64)
    rng = np.random.RandomState(1)
    rng.shuffle(every)
    img = np.stack([every >> 16, every >> 8 & 255, every & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    packed, counts = an._color_counts(img)
    assert np.array_equal(packed, np.arange(1 << 24)) and np.all(counts == 1)
    assert an.image_frequent_colors(img, 2.0 / (1 << 24)) == {}


def test_two_images_summed_in_one_histogram(an):
    from pyimsegm_b200 import _lib
    eng = an.get_engine()
    torch, lib, st = eng.torch, eng.lib, _lib.stream_ptr()
    rng = np.random.RandomState(2)
    a = _few_colours(rng, (1031, 777), [(0, 0, 0), (255, 0, 0), (1, 2, 3)])
    b = np.concatenate([_few_colours(rng, (513, 299), [(255, 0, 0), (9, 9, 9)]), np.full((513, 299, 1), 50, np.uint8)], -1)
    hist = torch.empty(1 << 24, dtype=torch.int64, device='cuda')
    for k, img in enumerate((a, b)):
        d = torch.from_numpy(np.ascontiguousarray(img)).cuda()
        _lib.check(lib.isb_color_hist(_lib.ptr(d), C.c_longlong(img.shape[0] * img.shape[1]), img.shape[2], k, _lib.ptr(hist), st))
    ws_bytes = lib.isb_color_hist_workspace_bytes()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    total = torch.empty(1, dtype=torch.int64, device='cuda')
    _lib.check(lib.isb_color_hist_compact_count(_lib.ptr(hist), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(total), st))
    n = int(total.item())
    colors = torch.empty(n, dtype=torch.int32, device='cuda')
    counts = torch.empty(n, dtype=torch.int64, device='cuda')
    _lib.check(lib.isb_color_hist_compact_write(_lib.ptr(hist), _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(colors), _lib.ptr(counts), st))
    pa, ca = _counts_np(a)
    pb, cb = _counts_np(b)
    want = {}
    for p_, c_ in list(zip(pa, ca)) + list(zip(pb, cb)):
        want[int(p_)] = want.get(int(p_), 0) + int(c_)
    assert colors.cpu().tolist() == sorted(want) and counts.cpu().tolist() == [want[k] for k in sorted(want)]


def test_group_images_frequent_colors(an, tmp_path):
    from PIL import Image
    rng = np.random.RandomState(3)
    paths = []
    for k, (shape, pal) in enumerate([((40, 60), [(0, 0, 0), (255, 0, 0)]), ((33, 17), [(255, 0, 0), (0, 9, 0), (1, 1, 1)])]):
        paths.append(str(tmp_path / ('img%d.png' % k)))
        Image.fromarray(_few_colours(rng, shape, pal)).save(paths[-1])
    assert an.group_images_frequent_colors(paths, 0.2) == oa.group_images_frequent_colors(paths, 0.2)


def _palette_cases(rng):
    pal = [(0, 0, 0), (255, 0, 0), (0, 255, 0), (10, 20, 30)]
    for shape in SHAPES + [(4096, 4096)]:
        img = _few_colours(rng, shape, pal)
        yield img, pal
        yield img.astype(np.float64) / 255, [tuple(np.array(c) / 255) for c in pal]
        yield img.astype(np.int16), [(0, 0, 0), (255, 0, 0), (0, 255, 0), (10, 20, 30), (-5, 300, 0)]     # float64 route


def test_exact_palette_labels(an):
    rng = np.random.RandomState(4)
    for img, pal in _palette_cases(rng):
        lut = {k: c for k, c in enumerate(pal)}
        small = img.shape[0] * img.shape[1] <= 10 ** 5
        want = oa.convert_img_colors_to_labels(img, lut) if small else None
        got = an.convert_img_colors_to_labels(img, lut)
        assert got.dtype == np.int64 and got.shape == img.shape[:2]
        if small:
            assert np.array_equal(got, want)
        else:
            assert np.array_equal(np.asarray(pal, dtype=img.dtype)[got], img)
        back = an.convert_img_labels_to_colors(got, lut)
        assert np.array_equal(back, np.asarray(pal)[got])
    img = _few_colours(rng, (37, 41), [(1, 1, 1), (2, 2, 2)])
    dup = {5: (1, 1, 1), 7: (2, 2, 2), 9: (1, 1, 1)}                                   # a colour given twice: the later label
    assert np.array_equal(an.convert_img_colors_to_labels(img, dup), oa.convert_img_colors_to_labels(img, dup))
    assert set(np.unique(an.convert_img_colors_to_labels(img, dup))) <= {7, 9}
    rev = {(1, 1, 1): 2.7, (2, 2, 2): -3}
    assert np.array_equal(an.convert_img_colors_to_labels_reverted(img, rev), oa.convert_img_colors_to_labels_reverted(img, rev))
    with pytest.raises(ValueError, match='different number'):
        an.convert_img_colors_to_labels(img, {0: (1, 1, 1)})                              # unmatched pixels
    with pytest.raises(ValueError, match='missing'):
        an.convert_img_labels_to_colors(np.array([[0, 1], [2, 5]]), {0: (1, 1, 1), 1: (2, 2, 2), 2: (0, 0, 0)})
    seg = rng.randint(-3, 4, (1, 301))
    lut = {int(k): (int(k), 1.5, -2) for k in np.unique(seg)}
    lut[10 ** 12] = (0, 0, 0)
    assert np.array_equal(an.convert_img_labels_to_colors(seg, lut), oa.convert_img_labels_to_colors(seg, lut))


def test_nearest_colour_palettes(an):
    rng = np.random.RandomState(5)
    for shape in SHAPES + [(4096, 4096)]:
        big = shape[0] * shape[1] > 10 ** 6
        img = rng.randint(0, 256, shape + (3, )).astype(np.uint8)
        pals = [[(0, 0, 0), (255, 255, 255), (128, 128, 128), (0, 0, 0)],                 # a duplicate, many L1 ties
                [(10, 0, 0), (0, 10, 0), (0, 0, 10), (5, 5, 0)],                           # ties everywhere near black
                [(300, -20, 0), (128, 128, 128)],                                          # outside uint8: float64 route
                [tuple(c) for c in rng.randint(0, 256, (1024, 3))]]                        # the largest palette
        for pal in pals:
            for im in ((img, ) if big else (img, img.astype(np.float64) + 0.25)):
                got = an.image_color_2_labels(im, pal)
                want = oa.image_color_2_labels(im, pal) if im.size * len(pal) <= 2 * 10 ** 8 else None
                assert got.dtype == np.int64
                if want is not None:
                    assert np.array_equal(got, want), (shape, len(pal), im.dtype)
                    q = an.quantize_image_nearest_color(im, pal)
                    assert q.dtype == im.dtype and np.array_equal(q, oa.quantize_image_nearest_color(im, pal))
    img = np.full((3, 4, 3), np.nan)
    img[0, 0] = 1.
    assert np.array_equal(an.image_color_2_labels(img, [(0, 0, 0), (1, 1, 1)]), oa.image_color_2_labels(img, [(0, 0, 0), (1, 1, 1)]))
    with pytest.raises(NotImplementedError, match='1024'):
        an.quantize_image_nearest_color(img, [(i, 0, 0) for i in range(1025)])


def _masks(rng, shape):
    H, W = shape
    single = np.zeros(shape, bool)
    single[H // 3, W // 2] = True
    column = np.zeros(shape, bool)
    column[:, W // 3] = True
    sparse = rng.rand(*shape) < 0.01
    sparse[H // 2, W // 2] = True
    checker = np.add.outer(np.arange(H), np.arange(W)) % 2 == 0
    return {'single': single, 'column': column, 'random_1pct': sparse, 'checkerboard': checker, 'all_valid': np.ones(shape, bool)}


def _check_inpaint(an, values, valid, small):
    got = an.image_inpaint_pixels(values, valid)
    assert got.dtype == values.dtype
    H, W = valid.shape
    dist, (ri, ci) = ndimage.distance_transform_edt(~valid, return_indices=True)
    eng = an.get_engine()
    index = an._nearest_site_index(eng, eng.to_device(valid.view(np.uint8), 't_valid'), valid.shape)
    index = eng.to_host(index).reshape(H, W).astype(np.int64)
    r, c = index // W, index % W
    assert valid[r, c].all()
    yy, xx = np.indices((H, W))
    assert np.array_equal(np.sqrt(((r - yy) ** 2 + (c - xx) ** 2).astype(np.float64)), dist)   # a site at scipy's exact distance
    assert np.array_equal(r, ri) and np.array_equal(c, ci)                                        # and scipy's own choice
    assert np.array_equal(got, values[r, c])
    if small:
        want = oa.image_inpaint_pixels(values, valid)
        unique = _unique_nearest(valid)
        assert np.array_equal(got[unique], want[unique])


def test_nearest_valid_pixel(an):
    rng = np.random.RandomState(6)
    for shape in SHAPES + [(4096, 4096)]:
        small = shape[0] * shape[1] <= 2 * 10 ** 5
        for name, valid in _masks(rng, shape).items():
            for values in (rng.rand(*shape), rng.randint(-5, 5, shape).astype(np.int8), rng.randint(0, 7, shape).astype(np.int32)):
                _check_inpaint(an, values, valid, small)
                if not small:
                    break


def test_quantize_nearest_pixel(an):
    rng = np.random.RandomState(7)
    pal = [(0, 0, 0), (255, 0, 0), (0, 0, 255), (255, 0, 0)]                         # a duplicate: the later index
    for shape in SHAPES[1:] + [(4096, 4096)]:
        img = _few_colours(rng, shape, pal + [(7, 7, 7), (9, 9, 9)])
        got = an.quantize_image_nearest_pixel(img, pal)
        assert got.dtype == np.asarray(pal).dtype and got.shape == img.shape
        valid = (img[..., None, :] == np.asarray(pal, np.uint8)).all(-1).any(-1)
        assert np.array_equal(got[valid], img[valid])
        labels = np.full(shape, -1)
        for i, clr in enumerate(pal):
            labels[(img == clr).all(-1)] = i
        _, (ri, ci) = ndimage.distance_transform_edt(~valid, return_indices=True)
        assert np.array_equal(got, np.asarray(pal)[labels[ri, ci]])
        if shape[0] * shape[1] <= 2 * 10 ** 5:
            want = oa.quantize_image_nearest_pixel(img, pal)
            unique = _unique_nearest(valid)
            assert np.array_equal(got[unique], want[unique])
    with pytest.raises(ValueError, match='no pixel'):
        an.quantize_image_nearest_pixel(np.full((5, 6, 3), 3, np.uint8), pal)
    flt = rng.rand(9, 11, 3)
    flt[2, 3] = (0.5, 0.25, 1.0)
    assert np.array_equal(an.quantize_image_nearest_pixel(flt, [(0.5, 0.25, 1.0)]), np.broadcast_to([0.5, 0.25, 1.0], flt.shape))

