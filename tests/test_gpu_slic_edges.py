"""
The 2-D SLIC against the oracle, bit for bit, at the edges of its inputs.

* input types: float32 and float16 images are rescaled in their own precision (numpy's arithmetic), integer and boolean images
  as numpy does it, colour and gray, ranges inside [0, 1] and far outside it; the banded route on float32;
* NaN and infinite pixels: numpy's min / max return NaN, so one NaN pixel turns the whole rescaled image into NaN, also when it
  sits in one band of the banded route; at the k-means level, NaN and infinite Lab values inside otherwise finite tiles;
* exact ties: flat colours whose centroids land on half-integers and checkerboards, with and without SLICO;
* compactness extremes: the colour term dominating or vanishing, and Lab values whose squares underflow or overflow;
* coordinates past 2^16 and 2^17 in either axis, in one piece and over bands whose first row is past 2^16;
* step edges: one-pixel superpixels (the sweeps alone: the device connectivity pass refuses pieces that small), windows
  smaller than a tile and windows over tens of tiles, sides of 32 k + 1, and Lab
  planes that the assignment cannot load with a tensor map (odd width, base not 16-byte aligned).
"""
import ctypes as C

import numpy as np
import pytest

from conftest import synth_regions

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _assert_same_labels(got, want):
    assert got.shape == want.shape
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, '%d of %d labels differ, first at %r' % (bad.size, got.size, np.unravel_index(bad[0], got.shape))


def _check_pipeline(oracle, img, sp_size=10, regul=0.2, slico=False):
    from pyimsegm_b200 import superpixels as sp
    got = sp.segment_slic_img2d(img, sp_size, regul, slico)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        want = oracle.segment_slic_img2d(img, sp_size, regul, slico)
    _assert_same_labels(got, want)
    return want


def _check_banded(oracle, eng, img, sp_size=10, regul=0.2, slico=False, n_bands=3):
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import slic_tiled
    n_seg, compact = slic_params(img.shape[:2], sp_size, regul)
    res = slic_tiled(img, n_seg, compact, slic_zero=slico, bands_per_rank=n_bands, eng=eng)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        want = oracle.segment_slic_img2d(img, sp_size, regul, slico)
    _assert_same_labels(eng.to_host(res.d_seg).astype(np.int64), want)
    return res


def _device_kmeans(lab, n_seg, slic_zero, offset=0):
    """isb_slic_kmeans on the planar copy of lab [H, W, 3]; the planes start `offset` doubles into their buffer"""
    import torch
    import oracle
    from pyimsegm_b200 import _lib
    H, W, _ = lab.shape
    seeds, ty, tx = oracle.slic_seeds(H, W, n_seg)
    n = len(seeds)
    lib = _lib.lib()
    planes = torch.from_numpy(np.ascontiguousarray(lab.transpose(2, 0, 1)).ravel())
    buf = torch.zeros(planes.numel() + offset, dtype=torch.float64, device='cuda')
    buf[offset:] = planes.cuda()
    d_seeds = torch.from_numpy(seeds).cuda()
    wsb = lib.isb_slic_kmeans_workspace_bytes(H, W, n, int(ty), int(tx))
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    labels = torch.empty((H, W), dtype=torch.int32, device='cuda')
    cent = torch.empty((n, 5), dtype=torch.float64, device='cuda')
    _lib.check(lib.isb_slic_kmeans(C.c_void_p(buf.data_ptr() + 8 * offset), H, W, _lib.ptr(d_seeds), n, int(ty), int(tx),
                                   C.c_double(float(max(1, ty, tx))), 10, int(slic_zero), _lib.ptr(labels), _lib.ptr(cent),
                                   _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return labels.cpu().numpy(), cent.cpu().numpy()


def _check_kmeans(oracle, lab, n_seg, slico, offset=0):
    got, got_c = _device_kmeans(lab, n_seg, slico, offset)
    want, want_c = oracle.slic_kmeans(lab, n_seg, slic_zero=slico, return_centroids=True)
    _assert_same_labels(got, want.astype(got.dtype))
    # the centroids of the clusters that hold pixels after the last sweep, NaN where the oracle has NaN
    alive = np.unique(want)
    g, w = got_c[alive], want_c[alive]
    assert np.array_equal(np.isnan(g), np.isnan(w))
    ok = ~np.isnan(w)
    assert np.array_equal(g[ok].view(np.int64), w[ok].view(np.int64))
    return want


def _lab(oracle, img, sp_size, regul):
    """the Lab planes and cluster count that segment_slic_img2d gives the k-means sweeps for an image in [0, 1]"""
    n_seg = int(img.shape[0] * img.shape[1] / sp_size ** 2)
    compact = (sp_size * regul) ** 1.5
    return oracle.rgb2lab_scaled(oracle.gaussian_blur(img, 1.0), 1.0 / compact), n_seg


def _regions(h, w, seed, cell=16, noise=0.05):
    return synth_regions(h, w, seed=seed, cell=cell, noise=noise)[0]


# -- input types ----------------------------------------------------------------------------------------------------------------

_RANGES = {
    np.float32: [(0.1, 0.9), (-1e3, 5e4)],
    np.float16: [(0.1, 0.9), (-1e3, 5e4)],
    np.float64: [(0.1, 0.9), (-1e3, 5e4)],
    np.uint8: [(0, 255), (17, 90)],
    np.uint16: [(0, 65535), (1000, 1500)],
    np.int16: [(-1000, 30000), (-7, 9)],
    np.int32: [(-1000, 50000), (-2 ** 29, 2 ** 30)],
}


def _typed(dtype, rng_lo, rng_hi, gray, seed, shape=(90, 110)):
    base = _regions(shape[0], shape[1], seed)
    if gray:
        base = base.mean(axis=2)
    v = rng_lo + base * (float(rng_hi) - rng_lo)
    if np.issubdtype(dtype, np.integer):
        return np.clip(np.round(v), rng_lo, rng_hi).astype(dtype)
    return v.astype(dtype)


@pytest.mark.parametrize('which', [0, 1])
@pytest.mark.parametrize('gray', [False, True])
@pytest.mark.parametrize('dtype', list(_RANGES), ids=lambda d: np.dtype(d).name)
def test_input_types(oracle, dtype, gray, which):
    lo, hi = _RANGES[dtype][which]
    _check_pipeline(oracle, _typed(dtype, lo, hi, gray, seed=7 + which + 2 * gray))


@pytest.mark.parametrize('gray', [False, True])
def test_input_bool(oracle, gray):
    """a boolean image holding both values is already in [0, 1]: numpy leaves it as it is"""
    img = _regions(90, 110, 3) > 0.5
    _check_pipeline(oracle, img[..., 0] if gray else img)


@pytest.mark.parametrize('gray', [False, True])
def test_input_float32_many_decisions(oracle, gray):
    """a noisy float32 image over a wide range: hundreds of thousands of close decisions on values rescaled in float32 (the
    Lab planes themselves are compared bit for bit in test_gpu_slic_prepare_connectivity.py)"""
    rng = np.random.RandomState(5)
    shape = (600, 700) if gray else (600, 700, 3)
    img = (rng.random_sample(shape) * 5e4 - 1e3).astype(np.float32)
    _check_pipeline(oracle, img, sp_size=6, regul=0.15)


@pytest.mark.parametrize('dtype', [np.float32, np.float64, np.uint16])
def test_input_types_banded(oracle, eng, dtype):
    lo, hi = _RANGES[dtype][1]
    _check_banded(oracle, eng, _typed(dtype, lo, hi, False, seed=21, shape=(150, 120)))


# -- NaN and infinite pixels ------------------------------------------------------------------------------------------------------

def _with(img, where, value):
    img = img.copy()
    img[where] = value
    return img


_SPECIALS = {
    'nan_pixel': [((37, 51), np.nan)],
    'nan_column': [((slice(None), 64), np.nan)],
    'pos_inf': [((12, 20), np.inf)],
    'neg_inf': [((70, 3), -np.inf)],
    'both_inf': [((12, 20), np.inf), ((70, 3), -np.inf)],
}


@pytest.mark.parametrize('gray', [False, True])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('case', list(_SPECIALS))
def test_nonfinite_pixels(oracle, case, dtype, gray):
    img = _typed(dtype, 0.1, 0.9, gray, seed=13)
    for where, value in _SPECIALS[case]:
        img = _with(img, where, value)
    _check_pipeline(oracle, img)


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('row', [148, 60, 2])
def test_nan_in_one_band(oracle, eng, dtype, row):
    """a NaN in the owned rows of the last, the middle or the first of three bands reaches every band's rescale"""
    img = _with(_typed(dtype, 0.1, 0.9, False, seed=17, shape=(150, 120)), (row, 33, 1), np.nan)
    _check_banded(oracle, eng, img)


def test_image_minmax_nan_rule():
    """isb_image_minmax: both extrema NaN when any sample is NaN, wherever it sits in the grid-stride reduction"""
    import torch
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    rng = np.random.RandomState(0)
    for n, pos in [(1, 0), (300, 299), (5000, 2047), (3_000_000, 2_999_999), (3_000_000, 1_234_567)]:
        for dtype in (np.float32, np.float64):
            x = rng.random_sample(n).astype(dtype)
            mm = torch.zeros(4, dtype=torch.float64, device='cuda')
            d = torch.from_numpy(x).cuda()
            _lib.check(lib.isb_image_minmax(_lib.ptr(d), _lib.dtype_code(x.dtype), C.c_longlong(n), _lib.ptr(mm), _lib.stream_ptr()))
            assert mm[:2].cpu().tolist() == [float(x.min()), float(x.max())]
            x[pos] = np.nan
            d = torch.from_numpy(x).cuda()
            _lib.check(lib.isb_image_minmax(_lib.ptr(d), _lib.dtype_code(x.dtype), C.c_longlong(n), _lib.ptr(mm), _lib.stream_ptr()))
            assert np.isnan(mm[:2].cpu().numpy()).all(), (n, pos, dtype)


_LAB_SPECIALS = {
    'nan_pixels': [((5, 7, 0), np.nan), ((40, 33, 2), np.nan), ((63, 64, 1), np.nan)],
    'inf_pixels': [((5, 7, 0), np.inf), ((40, 33, 2), -np.inf), ((31, 32, 1), np.inf)],
    'nan_row': [((45, slice(None), slice(None)), np.nan)],
    'nan_column': [((slice(None), 70, 1), np.nan)],
    'inf_row_part': [((20, slice(3, 60), 0), np.inf)],
}


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('case', list(_LAB_SPECIALS))
def test_kmeans_nonfinite_lab(oracle, case, slico):
    """the colour box bound of the assignment and the rule that a pixel no cluster can take keeps its label"""
    lab, n_seg = _lab(oracle, _regions(96, 130, 23), 8, 0.2)
    for where, value in _LAB_SPECIALS[case]:
        lab = _with(lab, where, value)
    _check_kmeans(oracle, lab, n_seg, slico)


# -- exact ties ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('sp_size,shape', [(4, (64, 96)), (6, (72, 84)), (8, (64, 128)), (10, (100, 60))])
def test_flat_half_integer_centroids(oracle, sp_size, shape, slico):
    """two flat halves: the grid cells have even sides, every centroid sits on a half-integer and spatial ties are everywhere"""
    img = np.full(shape + (3,), 0.2)
    img[:, shape[1] // 2:] = [0.7, 0.4, 0.9]
    _check_pipeline(oracle, img, sp_size, 0.2, slico)


def _checkerboard(cell):
    yy, xx = np.mgrid[:60, :74]
    board = ((yy // cell + xx // cell) % 2).astype(bool)
    return np.where(board[..., None], [0.9, 0.1, 0.3], [0.2, 0.6, 0.5])


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('cell', [1, 2])
@pytest.mark.parametrize('sp_size', [3, 4])
def test_checkerboard(oracle, sp_size, cell, slico):
    _check_pipeline(oracle, _checkerboard(cell), sp_size, 0.3, slico)


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('cell', [1, 2])
@pytest.mark.parametrize('sp_size', [2, 3, 4])
def test_kmeans_checkerboard(oracle, sp_size, cell, slico):
    """the sweeps alone, also at sp_size 2, whose superpixels are too small for the device connectivity pass"""
    lab, n_seg = _lab(oracle, _checkerboard(cell), sp_size, 0.3)
    _check_kmeans(oracle, lab, n_seg, slico)


# -- compactness extremes ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('regul', [1e-3, 5.0, 20.0])
def test_compactness_extremes(oracle, regul, slico):
    """relative_compact 1e-3 multiplies Lab by about 10^3; 5 and 20 make the colour about 1e-5 of the spatial term"""
    _check_pipeline(oracle, _regions(90, 110, 29), 10, regul, slico)


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('scale', [1e-150, 1e150])
def test_kmeans_lab_scale_extremes(oracle, scale, slico):
    """squares of the colour differences underflow to zero (1e-150) or overflow to inf (1e150); SLICO divides by them"""
    lab, n_seg = _lab(oracle, _regions(80, 100, 31), 8, 0.2)
    _check_kmeans(oracle, lab * scale, n_seg, slico)


# -- coordinates past 2^16 and 2^17 -----------------------------------------------------------------------------------------------

def _tall_lab(shape, kind, seed):
    """hand-built Lab planes: flat stripes (exact spatial ties) or low-amplitude noise (colour close to the spatial term)"""
    rng = np.random.RandomState(seed)
    H, W = shape
    if kind == 'flat':
        lab = np.zeros((H, W, 3))
        lab[:, W // 2:] = [0.5, -0.25, 0.125]
        lab[(np.arange(H) // 97) % 2 == 1] += [0.25, 0.0, 0.0]
        return lab
    return rng.normal(0.0, 0.3, (H, W, 3))


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('kind', ['flat', 'noisy'])
@pytest.mark.parametrize('sp_size', [2, 3, 10])
@pytest.mark.parametrize('shape', [(70003, 40), (40, 70003), (140001, 24)], ids=['70k_rows', '70k_cols', '140k_rows'])
def test_kmeans_coordinates_past_2_16(oracle, shape, sp_size, kind, slico):
    lab = _tall_lab(shape, kind, seed=sp_size)
    _check_kmeans(oracle, lab, int(shape[0] * shape[1] / sp_size ** 2), slico)


@pytest.mark.parametrize('slico', [False, True])
def test_pipeline_coordinates_past_2_16(oracle, eng, slico):
    """the whole pipeline on 70 003 x 40 in one piece, and 140 001 x 24 over three bands whose last starts past 2^16"""
    _check_pipeline(oracle, _regions(70003, 40, 37, cell=8, noise=0.1), 3, 0.2, slico)
    res = _check_banded(oracle, eng, _regions(140001, 24, 41, cell=8, noise=0.1), 3, 0.2, slico)
    assert not res.fell_back
    assert res.bands[-1].km_lo > 2 ** 16


# -- step edges ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('sp_size,shape', [(3, (97, 161)), (5, (161, 97)), (150, (2000, 1200))],
                         ids=['step3_97x161', 'step5_161x97', 'step150_2000px'])
def test_step_edges(oracle, sp_size, shape, slico):
    """windows inside one 32-px tile, sides of 32 k + 1, and windows of +-300 px that meet about 19 x 19 tiles"""
    _check_pipeline(oracle, _regions(shape[0], shape[1], sp_size + shape[0], cell=8 if sp_size < 10 else 64), sp_size, 0.2, slico)


@pytest.mark.parametrize('slico', [False, True])
@pytest.mark.parametrize('sp_size,shape', [(1, (48, 70)), (1, (33, 65)), (2, (33, 65)), (2, (97, 161))],
                         ids=['step1_48x70', 'step1_33x65', 'step2_33x65', 'step2_97x161'])
def test_kmeans_step_edges(oracle, sp_size, shape, slico):
    """one-pixel superpixels (n_segments = pixel count) and steps of 2, through the sweeps alone"""
    lab, n_seg = _lab(oracle, _regions(shape[0], shape[1], sp_size + shape[0], cell=4), sp_size, 0.2)
    _check_kmeans(oracle, lab, n_seg, slico)


@pytest.mark.parametrize('sp_size', [1, 2])
def test_superpixels_below_the_connectivity_limit_raise(sp_size):
    """superpixels of 1 or 4 px give max_size = 3 * sp_size^2 < 16, which the device connectivity pass refuses: an error, never
    a silently different map"""
    from pyimsegm_b200 import superpixels as sp
    with pytest.raises(ValueError, match='max_size < 16'):
        sp.segment_slic_img2d(_regions(48, 70, 3), sp_size, 0.2)


@pytest.mark.parametrize('offset', [0, 1])
@pytest.mark.parametrize('W', [129, 130, 33])
def test_kmeans_without_tensor_map(oracle, W, offset):
    """an odd width, or planes that start 8 bytes past a 16-byte boundary, are staged by ordinary loads instead of a tensor map"""
    lab, n_seg = _lab(oracle, _regions(97, W, W + offset), 5, 0.2)
    for slico in (False, True):
        _check_kmeans(oracle, lab, n_seg, slico, offset=offset)
