"""The per-segment statistics kernels against float64 references written here, at the sizes where the kernels branch.

- Colour statistics (``isb_segment_stats_2d`` and the banded trio ``_accumulate / _deviation / _finish``, csrc/segment_stats.cu): a
  thread walks one column of a 16-row strip in 256-column blocks and flushes its run sums with atomics whenever the label changes.
  The shapes put W and H on both sides of those blocks and strips; the label maps make runs of one pixel, of a whole strip, of one
  label over millions of pixels and of one label per pixel.
- Gray statistics (``isb_gray_stats``, csrc/native_misc.cu): runs of 16 voxels, any rank.
- Median (``isb_segment_median`` / ``_2d``, csrc/segment_median.cu): labels on both sides of the shared-memory staging cap and
  values where a radix select or np.median's float type decides.
- Disc label histograms (``isb_disc_label_hist``) and 3-D centroids (``isb_centroids_3d``).

Bounds.  The kernels form each term in float32 exactly as the reference's Cython does and add the terms in float64.  The references
here form the same terms and add them with np.bincount.  Both are float64 sums of the same n terms, so each lies within n u A of the
exact sum (u = 2^-53, A = sum |t|); a mean column is within (2n + 2) u A / n of the reference (two sums, two divisions).  A float32
accumulator misses these bounds by orders of magnitude.  Centres, counts and histograms are exact and compared exactly.
"""
import ctypes as C

import numpy as np
import pytest

U = 2.0 ** -53
#: bytes of shared memory a select CTA stages its label's keys in: MED_SMEM_BYTES of pyimsegm_b200/csrc/segment_median.cu
MED_SMEM_BYTES = 96 * 1024
SENTINEL = -12345.625


def med_cap(channels):
    """pixels of the largest label whose keys (8 bytes per channel) the median kernel stages in shared memory"""
    return MED_SMEM_BYTES // (8 * channels)


# ------------------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------------------

def _f32(values):
    """the kernels' load: every dtype to float32 (u8 / u16 exactly, float64 rounded to nearest)"""
    return np.asarray(values).astype(np.float32)


def _check_bound(got, terms, seg, nb, what, square_root=False):
    """got [nb, K] against the per-label mean of terms [n, K] within (2n + 2) u A / n; ``square_root``: got is the root of that mean,
    compared squared with 4 u of the mean added"""
    n = np.bincount(seg, minlength=nb).astype(np.float64)
    present = n > 0
    for k in range(terms.shape[1]):
        s = np.bincount(seg, weights=terms[:, k], minlength=nb)
        a = np.bincount(seg, weights=np.abs(terms[:, k]), minlength=nb)
        want = np.where(present, s / np.maximum(n, 1), 0.0)
        tol = (2 * n + 2) * U * a / np.maximum(n, 1)
        g = got[:, k]
        if square_root:
            tol = tol + 4 * U * np.abs(want)
            g = g * g
        err = np.abs(g - want)
        assert np.all(got[~present, k] == 0), '%s: absent labels must give 0, column %d' % (what, k)
        ratio = np.where(present, err / np.maximum(tol, 1e-300), 0)
        worst = int(np.argmax(ratio))
        assert np.all(err[present] <= tol[present]), '%s, column %d: label %d of %d px: got %r, want %r, error %.3g > bound %.3g' % (
            what, k, worst, int(n[worst]), g[worst], want[worst], err[worst], tol[worst])


def _check_colour(img, seg, nb, mean, std, energy, centres, counts, what):
    """the three statistics (any may be None), the centres and the counts of one colour image"""
    H, W = seg.shape
    s = seg.ravel()
    v = _f32(img).reshape(-1, 3) if img is not None else None
    if mean is not None:
        _check_bound(mean, v.astype(np.float64), s, nb, what + ' mean')
    if energy is not None:
        _check_bound(energy, (v * v).astype(np.float64), s, nb, what + ' energy')
    if std is not None:
        d = v - mean.astype(np.float32)[s]                 # float32, about the float32 of the device's own mean
        _check_bound(std, (d * d).astype(np.float64), s, nb, what + ' std', square_root=True)
    n = np.bincount(s, minlength=nb)
    if counts is not None:
        np.testing.assert_array_equal(counts, n, err_msg=what + ' counts')
    if centres is not None:
        yy, xx = np.divmod(np.arange(H * W), W)
        want = np.full((nb, 2), -1.0)
        ok = n > 0
        want[ok, 0] = np.bincount(s, weights=yy, minlength=nb)[ok] / n[ok]
        want[ok, 1] = np.bincount(s, weights=xx, minlength=nb)[ok] / n[ok]
        np.testing.assert_array_equal(centres, want, err_msg=what + ' centres')


def _median_ref(values, seg, nb):
    """per label np.median of the member values [n, C] in their own dtype; NaN for a label without pixels"""
    values = values.reshape(len(seg), -1)
    out = np.full((nb, values.shape[1]), np.nan)
    order = np.argsort(seg, kind='stable')
    bounds = np.concatenate([[0], np.cumsum(np.bincount(seg, minlength=nb))])
    sv = values[order]
    for lb in range(nb):
        if bounds[lb + 1] > bounds[lb]:
            out[lb] = np.median(sv[bounds[lb]:bounds[lb + 1]], axis=0)
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------

WIDTHS = (1, 255, 256, 257, 513)
HEIGHTS = (1, 15, 16, 17, 33)
DTYPES = ('uint8', 'uint16', 'float32', 'float64')
MAPS = ('one', 'rows', 'cols', 'checker', 'blocks7', 'random')


def _image(shape, dtype, rng):
    if dtype == 'uint8':
        return rng.randint(0, 256, shape).astype(np.uint8)
    if dtype == 'uint16':
        img = rng.randint(0, 65536, shape).astype(np.uint16)
        img.flat[::7] = 65535                               # 65535^2 rounds in float32
        return img
    if dtype == 'float32':
        return rng.normal(0.3, 2.0, shape).astype(np.float32)
    return rng.normal(0.3, 2.0, shape) * (1 + 1e-9 * rng.rand(*shape))        # more than 24 significant bits


def _labels(kind, H, W, rng):
    """label map [H, W] int32 and nb (max + 1)"""
    yy, xx = np.mgrid[:H, :W]
    if kind == 'one':
        seg = np.zeros((H, W), int)
    elif kind == 'rows':                                    # a new label at every row: every pixel ends a run
        seg = yy
    elif kind == 'cols':
        seg = xx
    elif kind == 'checker':
        seg = (yy + xx) % 2
    elif kind == 'blocks7':                                 # 7-row blocks cross the 16-row strips
        seg = (yy // 7) * ((W + 6) // 7) + xx // 7
    else:                                                   # labels 0, the middle one and the one below the maximum absent
        top = 12
        pool = np.array([lb for lb in range(1, top + 1) if lb not in (top // 2, top - 1)])
        seg = pool[rng.randint(0, len(pool), (H, W))]
        seg.flat[-1] = top
    seg = np.ascontiguousarray(seg, dtype=np.int32)
    return seg, int(seg.max()) + 1


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


def _lib():
    from pyimsegm_b200 import _lib as lb
    return lb


# ------------------------------------------------------------------------------------------------------------------------------
# isb_segment_stats_2d
# ------------------------------------------------------------------------------------------------------------------------------

def _stats_2d(img, seg, nb, flags, col0=0, extra=0, centres=True, counts=True):
    """one isb_segment_stats_2d call into a sentinel-filled table of ld = col0 + ncol + extra columns; returns (table, centres,
    counts).  ``img`` None: a centres-only call."""
    torch, lb = _torch(), _lib()
    lib = lb.lib()
    H, W = seg.shape
    ncol = 3 * bin(flags).count('1')
    ld = col0 + ncol + extra
    feat = torch.full((nb, ld), SENTINEL, dtype=torch.float64, device='cuda') if ncol else None
    d_img = _dev(img) if img is not None else None
    d_seg = _dev(seg)
    cen = torch.full((nb, 2), SENTINEL, dtype=torch.float64, device='cuda') if centres else None
    cnt = torch.full((nb, ), -7, dtype=torch.int32, device='cuda') if counts else None
    wsb = lib.isb_segment_stats_workspace_bytes(nb)
    ws = torch.full((wsb, ), 0x5A, dtype=torch.uint8, device='cuda')
    code = lb.dtype_code(img.dtype) if img is not None else 0
    lb.check(lib.isb_segment_stats_2d(lb.ptr(d_img), code, lb.ptr(d_seg), H, W, nb, flags, lb.ptr(feat), ld, col0, lb.ptr(cen),
                                      lb.ptr(cnt), lb.ptr(ws), C.c_size_t(wsb), lb.stream_ptr()))
    return (_host(feat) if feat is not None else None), (_host(cen) if centres else None), (_host(cnt) if counts else None)


def _split(table, col0, flags):
    """(mean, std, energy) column blocks of a table written at col0 with ``flags``"""
    out, col = [], col0
    for bit in (1, 2, 4):
        if flags & bit:
            out.append(table[:, col:col + 3])
            col += 3
        else:
            out.append(None)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('W', WIDTHS)
@pytest.mark.parametrize('H', HEIGHTS)
def test_segment_stats_2d_shapes_and_label_maps(H, W):
    """every label map at every shape, all four dtypes, against the float64 bounds; placement in a wider table at col0 > 0"""
    rng = np.random.RandomState(H * 1000 + W)
    for kind in MAPS:
        seg, nb = _labels(kind, H, W, rng)
        for dtype in DTYPES:
            img = _image((H, W, 3), dtype, rng)
            what = '%dx%d %s %s' % (H, W, kind, dtype)
            col0, extra = 2, 3
            table, centres, counts = _stats_2d(img, seg, nb, 7, col0=col0, extra=extra)
            mean, std, energy = _split(table, col0, 7)
            _check_colour(img, seg, nb, mean, std, energy, centres, counts, what)
            assert np.all(table[:, :col0] == SENTINEL) and np.all(table[:, col0 + 9:] == SENTINEL), what + ': cells outside the block'


@pytest.mark.gpu
@pytest.mark.parametrize('flags', [1, 3, 4, 5])
def test_segment_stats_2d_flag_subsets_keep_their_columns(flags):
    """a subset of the statistics writes its columns in the order mean, std, energy and nothing else (std only with its mean, whose
    float32 the deviation terms are taken about)"""
    rng = np.random.RandomState(flags)
    H, W = 33, 257
    seg, nb = _labels('blocks7', H, W, rng)
    img = _image((H, W, 3), 'float64', rng)
    col0, extra = 1, 2
    table, _, _ = _stats_2d(img, seg, nb, flags, col0=col0, extra=extra, centres=False, counts=False)
    ncol = 3 * bin(flags).count('1')
    assert np.all(table[:, :col0] == SENTINEL) and np.all(table[:, col0 + ncol:] == SENTINEL)
    mean, std, energy = _split(table, col0, flags)
    _check_colour(img, seg, nb, mean, std, energy, None, None, 'flags %d' % flags)


@pytest.mark.gpu
def test_segment_stats_2d_centres_only_call():
    """img = NULL and flags 0: centres and counts only"""
    rng = np.random.RandomState(3)
    seg, nb = _labels('random', 65, 300, rng)
    table, centres, counts = _stats_2d(None, seg, nb, 0)
    assert table is None
    _check_colour(None, seg, nb, None, None, None, centres, counts, 'centres only')


@pytest.mark.gpu
def test_segment_stats_2d_one_label_over_4_million_pixels():
    rng = np.random.RandomState(4)
    H, W = 2048, 2056
    seg = np.zeros((H, W), np.int32)
    for dtype in ('float32', 'float64', 'uint16'):
        img = _image((H, W, 3), dtype, rng)
        table, centres, counts = _stats_2d(img, seg, 1, 7)
        mean, std, energy = _split(table, 0, 7)
        _check_colour(img, seg, 1, mean, std, energy, centres, counts, '%dx%d one label %s' % (H, W, dtype))


@pytest.mark.gpu
def test_segment_stats_2d_one_label_per_pixel():
    """512 x 512 labels of one pixel each: every statistic is its pixel's term"""
    rng = np.random.RandomState(5)
    H = W = 512
    seg = np.arange(H * W, dtype=np.int32).reshape(H, W)
    for dtype in ('uint8', 'float64'):
        img = _image((H, W, 3), dtype, rng)
        table, centres, counts = _stats_2d(img, seg, H * W, 7)
        mean, std, energy = _split(table, 0, 7)
        _check_colour(img, seg, H * W, mean, std, energy, centres, counts, 'per pixel %s' % dtype)
        v = _f32(img).reshape(-1, 3)
        np.testing.assert_array_equal(mean, v.astype(np.float64))
        np.testing.assert_array_equal(energy, (v * v).astype(np.float64))
        np.testing.assert_array_equal(std, 0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# the banded trio: isb_segment_stats_accumulate / _deviation / _finish, one band per call, shared accumulators
# ------------------------------------------------------------------------------------------------------------------------------

def _stats_banded(img, seg, nb, starts, flags=7, col0=1, extra=2):
    torch, lb = _torch(), _lib()
    lib = lb.lib()
    H, W = seg.shape
    d_img, d_seg = _dev(img), _dev(seg)
    code = lb.dtype_code(img.dtype)
    row_img, row_seg = W * 3 * img.itemsize, W * 4
    acc = torch.zeros((nb, 6), dtype=torch.float64, device='cuda')
    iacc = torch.zeros((nb, 3), dtype=torch.int64, device='cuda')
    var = torch.zeros((nb, 3), dtype=torch.float64, device='cuda')
    meanf = torch.zeros((nb, 3), dtype=torch.float32, device='cuda')
    bands = list(zip(starts, list(starts[1:]) + [H]))
    for lo, hi in bands:
        lb.check(lib.isb_segment_stats_accumulate(C.c_void_p(d_img.data_ptr() + lo * row_img), code, C.c_void_p(d_seg.data_ptr() + lo * row_seg),
                                                  hi - lo, W, lo, nb, lb.ptr(acc), lb.ptr(iacc), lb.stream_ptr()))
    for lo, hi in bands:
        lb.check(lib.isb_segment_stats_deviation(C.c_void_p(d_img.data_ptr() + lo * row_img), code, C.c_void_p(d_seg.data_ptr() + lo * row_seg),
                                                 hi - lo, W, nb, lb.ptr(acc), lb.ptr(iacc), lb.ptr(meanf), lb.ptr(var), lb.stream_ptr()))
    ld = col0 + 9 + extra
    feat = torch.full((nb, ld), SENTINEL, dtype=torch.float64, device='cuda')
    cen = torch.full((nb, 2), SENTINEL, dtype=torch.float64, device='cuda')
    cnt = torch.full((nb, ), -7, dtype=torch.int32, device='cuda')
    lb.check(lib.isb_segment_stats_finish(nb, flags, lb.ptr(acc), lb.ptr(var), lb.ptr(iacc), lb.ptr(feat), ld, col0, lb.ptr(cen),
                                          lb.ptr(cnt), lb.stream_ptr()))
    return _host(feat), _host(cen), _host(cnt)


@pytest.mark.gpu
@pytest.mark.parametrize('W', (1, 256, 257, 513))
def test_segment_stats_banded_trio(W):
    """bands starting at rows 0, 1, 17 and H - 1 accumulate into the same buffers: the same bounds, exact centres and counts"""
    rng = np.random.RandomState(W)
    H = 40
    for kind in MAPS:
        seg, nb = _labels(kind, H, W, rng)
        for dtype in DTYPES:
            img = _image((H, W, 3), dtype, rng)
            what = 'banded %dx%d %s %s' % (H, W, kind, dtype)
            table, centres, counts = _stats_banded(img, seg, nb, [0, 1, 17, H - 1])
            mean, std, energy = _split(table, 1, 7)
            _check_colour(img, seg, nb, mean, std, energy, centres, counts, what)
            assert np.all(table[:, :1] == SENTINEL) and np.all(table[:, 10:] == SENTINEL), what + ': cells outside the block'


# ------------------------------------------------------------------------------------------------------------------------------
# isb_gray_stats through cython_img3d_gray_*
# ------------------------------------------------------------------------------------------------------------------------------

def _check_gray(img, seg, what):
    from pyimsegm_b200 import descriptors as ds
    s = seg.ravel()
    nb = int(s.max()) + 1
    v = _f32(img).ravel()
    mean = ds.cython_img3d_gray_mean(img, seg)
    _check_bound(mean[:, None], v.astype(np.float64)[:, None], s, nb, what + ' mean')
    _check_bound(ds.cython_img3d_gray_energy(img, seg)[:, None], (v * v).astype(np.float64)[:, None], s, nb, what + ' energy')
    d = v - mean.astype(np.float32)[s]
    _check_bound(ds.cython_img3d_gray_std(img, seg)[:, None], (d * d).astype(np.float64)[:, None], s, nb, what + ' std', square_root=True)


GRAY_SHAPES = [(1, ), (15, ), (16, ), (17, ), (4097, ), (3, 5), (4, 4), (1, 17), (17, 241), (2, 3, 5), (1, 1, 16), (3, 37, 37)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape', GRAY_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_gray_stats_lengths_ranks_and_runs(shape):
    rng = np.random.RandomState(int(np.prod(shape)))
    n = int(np.prod(shape))
    for runs in (1, 7, 16, 23):                               # runs of 7 and 23 voxels cross the 16-voxel strips
        seg = (np.arange(n) // runs).reshape(shape)
        for dtype in DTYPES:
            _check_gray(_image(shape, dtype, rng), seg, 'gray %r runs %d %s' % (shape, runs, dtype))
    seg = rng.randint(0, 9, shape)
    seg.flat[-1] = 10                                        # absent labels 9 and maybe others
    seg[seg == 4] = 5
    _check_gray(_image(shape, 'float64', rng), seg, 'gray %r random' % (shape, ))


@pytest.mark.gpu
def test_gray_stats_volume_of_16_million_voxels():
    rng = np.random.RandomState(6)
    shape = (256, 256, 257)
    seg = (np.arange(int(np.prod(shape))) // 100003 % 37).reshape(shape)
    seg[:40] = 0                                             # one label of millions of voxels
    _check_gray(rng.normal(0.5, 1.0, shape).astype(np.float32), seg, 'gray 2^24')


# ------------------------------------------------------------------------------------------------------------------------------
# median
# ------------------------------------------------------------------------------------------------------------------------------

def _labels_of_sizes(sizes, rng):
    """flat label array with label i repeated sizes[i] times, shuffled"""
    seg = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    rng.shuffle(seg)
    return seg


def _device_median(values, seg, channels):
    """numpy_img2d_color_median (channels 3) or numpy_img3d_gray_median (channels 1) of flat values [n, channels]"""
    from pyimsegm_b200 import descriptors as ds
    n = len(seg)
    if channels == 3:
        return ds.numpy_img2d_color_median(values.reshape(n, 1, 3), seg.reshape(n, 1))
    return ds.numpy_img3d_gray_median(values.reshape(n), seg)[:, None]


def _check_median(values, seg, channels, what):
    nb = int(seg.max()) + 1
    got = _device_median(values, seg, channels)
    want = _median_ref(values, seg, nb)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        lb, c = np.argwhere(bad)[0]
        raise AssertionError('%s: %d of %d medians differ; label %d (%d px) channel %d: got %r, want %r' % (
            what, bad.sum(), bad.size, lb, int((seg == lb).sum()), c, got[lb, c], want[lb, c]))


@pytest.mark.gpu
@pytest.mark.parametrize('channels', (3, 1))
def test_median_labels_around_the_staging_cap(channels):
    """labels of cap - 1, cap and cap + 1 pixels: the last one selects from the image instead of shared memory"""
    rng = np.random.RandomState(channels)
    cap = med_cap(channels)
    seg = _labels_of_sizes([cap - 1, cap, cap + 1, 0, 5, 6], rng)
    for dtype in DTYPES:
        values = _image((len(seg), channels), dtype, rng)
        _check_median(values, seg, channels, 'cap %d %s' % (cap, dtype))


@pytest.mark.gpu
def test_median_one_label_of_4_million_pixels():
    rng = np.random.RandomState(7)
    seg = np.zeros(1 << 22, np.int32)
    for dtype in ('float64', 'float32', 'uint8'):
        _check_median(_image((len(seg), 3), dtype, rng), seg, 3, 'nb 1 2^22 px %s' % dtype)
    seg = _labels_of_sizes([(1 << 22) + 1, 3, 0, 4], rng)
    _check_median(_image((len(seg), 3), 'float64', rng), seg, 3, '2^22 + 1 px')


@pytest.mark.gpu
def test_median_5000_labels_of_many_pixels():
    rng = np.random.RandomState(8)
    sizes = rng.randint(1, 400, 5000)
    sizes[[0, 17, 2500, 4998]] = 0                            # absent labels -> NaN
    sizes[[5, 6, 7]] = [4095, 4097, 9000]
    seg = _labels_of_sizes(sizes, rng)
    for dtype in DTYPES:
        _check_median(_image((len(seg), 3), dtype, rng), seg, 3, '5000 labels %s' % dtype)
    _check_median(_image((len(seg), 1), 'float64', rng), seg, 1, '5000 labels gray')


def _special_values(rng, n_labels, size, dtype):
    """label after label of the values where a select or np.median's float type decides; flat [n, 3] values and labels"""
    vals, segs = [], []
    big = np.finfo(dtype).max
    tiny = np.finfo(dtype).smallest_subnormal
    for lb in range(n_labels):
        kind = lb % 8
        m = size + (lb % 3)                                   # odd and even counts
        if kind == 0:                                         # a few ulps apart: the last radix byte decides
            v = np.empty(m, dtype)
            v[0] = dtype(rng.normal())
            for i in range(1, m):
                v[i] = np.nextafter(v[i - 1], dtype(np.inf))
            v = np.stack([rng.permutation(v) for _ in range(3)], 1)
        elif kind == 1:                                       # -0.0, +0.0 and subnormals
            pool = np.array([-0.0, 0.0, tiny, -tiny, 3 * tiny, -2 * tiny], dtype)
            v = pool[rng.randint(0, len(pool), (m, 3))]
        elif kind == 2:                                       # infinities among ordinary values
            v = rng.normal(size=(m, 3)).astype(dtype)
            v[rng.rand(m, 3) < 0.3] = np.inf
            v[rng.rand(m, 3) < 0.3] = -np.inf
        elif kind == 3:                                       # even count, middles -inf and +inf -> NaN
            v = np.array([-np.inf] * 3 + [np.inf] * 3, dtype)[:, None].repeat(3, 1)
        elif kind == 4:                                       # one pixel near the top of the range
            v = np.full((1, 3), big * 0.8, dtype)
            v[0, 1] = -v[0, 1]
        elif kind == 5:                                       # even count, middles near the top (their sum overflows)
            v = np.full((4, 3), big * 0.75, dtype)
            v[:, 2] = -v[:, 2]
        elif kind == 6:                                       # NaN with either sign bit among ordinary values
            v = rng.normal(size=(m, 3)).astype(dtype)
            v[rng.randint(m), lb % 3] = np.copysign(np.nan, 1.0 if lb % 2 else -1.0)
        else:                                                 # noise with an even count
            v = rng.normal(size=(2 * m, 3)).astype(dtype)
        vals.append(v.astype(dtype))
        segs.append(np.full(len(v), lb, np.int32))
    values, seg = np.concatenate(vals), np.concatenate(segs)
    perm = rng.permutation(len(seg))
    return values[perm], seg[perm]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ('float64', 'float32'))
@pytest.mark.parametrize('size', (9, 5000))
def test_median_special_values(dtype, size):
    """np.median in the image's float type: ulp chains, signed zeros, subnormals, infinities, NaN, overflow near the top"""
    rng = np.random.RandomState(size)
    values, seg = _special_values(rng, 48, size, getattr(np, dtype))
    _check_median(values, seg, 3, 'special %s size %d' % (dtype, size))
    _check_median(np.ascontiguousarray(values[:, 0]), seg, 1, 'special gray %s size %d' % (dtype, size))


@pytest.mark.gpu
def test_median_u8_ties_and_constant_labels():
    rng = np.random.RandomState(9)
    sizes = rng.randint(1, 30, 300)
    sizes[[3, 9]] = [5000, 20000]
    seg = _labels_of_sizes(sizes, rng)
    values = rng.choice(np.array([0, 1, 2, 254, 255], np.uint8), (len(seg), 3), p=[0.4, 0.1, 0.1, 0.1, 0.3])
    for lb in range(0, 300, 4):                               # labels of one repeated value
        values[seg == lb] = lb % 256
    _check_median(values, seg, 3, 'u8 ties')


@pytest.mark.gpu
def test_median_one_pixel_label_near_dbl_max():
    """an odd count returns the value itself: 0.5 * (v + v) would overflow"""
    values = np.array([[1.5e308, -1.5e308, 1.7976931348623157e308], [1.0, 2.0, 3.0]])
    seg = np.array([0, 1], np.int32)
    got = _device_median(values, seg, 3)
    np.testing.assert_array_equal(got, values)


@pytest.mark.gpu
def test_median_feature_table_route_float32():
    """compute_image2d_color_statistic(..., ('median',)) of a float32 image with labels over the cap, NaN and infinite pixels:
    bit for bit the oracle's restatement (np.nan_to_num, the median in float32, the table's rules)"""
    import oracle
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(10)
    H, W = 96, 160
    yy, xx = np.mgrid[:H, :W]
    seg = (yy // 48) * 2 + xx // 80                           # labels 0 .. 3, label 5 absent
    seg[:, 150:] = 4
    seg[:64, :80] = 0                                         # label 0: 5 118 px, over the cap
    seg[0, :2] = 6                                            # two px of +inf: FLT_MAX + FLT_MAX overflows in float32
    img = rng.normal(0.5, 1.0, (H, W, 3)).astype(np.float32)
    img[0, :2, 0] = np.inf
    img[1, :7, 1] = np.nan
    img[2, :5, 2] = -np.inf
    got, _ = ds.compute_image2d_color_statistic(img, seg, ('median', ))
    want = oracle.image2d_color_statistic(img, seg, ('median', ))
    np.testing.assert_array_equal(got, want)
    assert got[6, 0] == np.finfo(np.float64).max


# ------------------------------------------------------------------------------------------------------------------------------
# reference-run goldens of the median (tests/golden/make_median_goldens.py)
# ------------------------------------------------------------------------------------------------------------------------------

GOLDEN_CASES = ('f32_even', 'float64_nan', 'float32_nan', 'f64_huge')


@pytest.fixture(scope='module')
def median_goldens():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'median_reference.npz'))


@pytest.mark.parametrize('case', GOLDEN_CASES)
def test_oracle_median_equals_reference_goldens(oracle, median_goldens, case):
    img, seg = median_goldens[case + '_img'], median_goldens[case + '_seg']
    np.testing.assert_array_equal(oracle.color2d_median(img, seg), median_goldens[case + '_color'])
    np.testing.assert_array_equal(oracle.image2d_color_statistic(img, seg, ('median', )), median_goldens[case + '_table'])


@pytest.mark.gpu
@pytest.mark.parametrize('case', GOLDEN_CASES)
def test_device_median_equals_reference_goldens(median_goldens, case):
    from pyimsegm_b200 import descriptors as ds
    img, seg = median_goldens[case + '_img'], median_goldens[case + '_seg']
    np.testing.assert_array_equal(ds.numpy_img2d_color_median(img, seg), median_goldens[case + '_color'])
    np.testing.assert_array_equal(ds.numpy_img3d_gray_median(img[None, :, :, 0], seg[None]), median_goldens[case + '_gray'])
    np.testing.assert_array_equal(ds.compute_image2d_color_statistic(img, seg, ('median', ))[0], median_goldens[case + '_table'])


# ------------------------------------------------------------------------------------------------------------------------------
# isb_disc_label_hist
# ------------------------------------------------------------------------------------------------------------------------------

def _corners_and_centre(H, W):
    return [[0, 0], [0, W - 1], [H - 1, 0], [H - 1, W - 1], [H // 2, W // 3]]


@pytest.mark.gpu
@pytest.mark.parametrize('nb_labels', (1, 4095, 4096))
def test_disc_label_hist_label_counts(oracle, nb_labels):
    """counts under discs of diameter 0, 1, 5 and larger than the image diagonal, on all four corners: exact"""
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(nb_labels)
    H, W = 61, 83
    segm = rng.randint(0, nb_labels, (H, W))
    segm.flat[:nb_labels] = np.arange(nb_labels)[:H * W]
    positions, diameters = _corners_and_centre(H, W), [0, 1, 5, 120]
    hist, sizes = ds._device_label_hists(segm, positions, nb_labels, diameters=diameters)
    for i, pos in enumerate(positions):
        for j, d in enumerate(diameters):
            want, size = oracle.label_hist_selem(segm, pos, oracle.disk(d), nb_labels)
            np.testing.assert_array_equal(hist[i, j], want, err_msg='position %r diameter %d' % (pos, d))
            assert sizes[i, j] == size
    got, _ = ds.compute_label_histograms_positions(segm, positions, diameters, nb_labels)
    np.testing.assert_array_equal(got, oracle.label_histograms_positions(segm, positions, diameters, nb_labels))


@pytest.mark.gpu
def test_disc_label_hist_more_than_4096_labels_is_an_argument_error():
    torch, lb = _torch(), _lib()
    segm = torch.zeros((8, 8), dtype=torch.int32, device='cuda')
    pos = torch.zeros((1, 2), dtype=torch.int32, device='cuda')
    diam = torch.ones((1, ), dtype=torch.int32, device='cuda')
    hist = torch.zeros((4097, ), dtype=torch.float64, device='cuda')
    sizes = torch.zeros((1, ), dtype=torch.float64, device='cuda')
    for nb, status in ((4097, lb.ISB_ERR_ARG), (4096, lb.ISB_OK)):
        rc = lb.lib().isb_disc_label_hist(lb.ptr(segm), None, 8, 8, lb.ptr(pos), 1, lb.ptr(diam), 1, None, 0, 0, nb, lb.ptr(hist),
                                          lb.ptr(sizes), lb.stream_ptr())
        assert rc == status, (nb, rc)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(4, 4), (6, 3), (5, 5), (1, 8)], ids=str)
def test_label_hist_structuring_elements(oracle, shape):
    """even-sized elements and element values other than 0 and 1 (only 1 counts), on the corners; proba sums within the bound"""
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(shape[0] * 10 + shape[1])
    H, W, K = 23, 31, 5
    segm = rng.randint(0, K, (H, W))
    proba = rng.dirichlet(np.ones(K), (H, W))
    for _ in range(3):
        selem = rng.choice(np.array([0, 1, 2, -1, 1]), shape)
        for pos in _corners_and_centre(H, W):
            hist, size = ds.compute_label_hist_segm(segm, pos, selem, K)
            want, want_size = oracle.label_hist_selem(segm, pos, selem, K)
            np.testing.assert_array_equal(hist, want)
            assert size == want_size
            got, size = ds.compute_label_hist_proba(proba, pos, selem)
            want, want_size = oracle.label_hist_selem(proba, pos, selem)
            assert size == want_size
            a = oracle.label_hist_selem(np.abs(proba), pos, selem)[0]
            n = max(want_size, 1)
            assert np.all(np.abs(got - want) <= 2 * n * U * a), (pos, selem.tolist(), got - want)


# ------------------------------------------------------------------------------------------------------------------------------
# isb_centroids_3d
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(1, 1, 1), (3, 7, 11), (5, 17, 255), (9, 33, 65)], ids=lambda s: 'x'.join(map(str, s)))
def test_centroids_3d_exact(shape):
    torch, lb = _torch(), _lib()
    rng = np.random.RandomState(int(np.prod(shape)))
    D, H, W = shape
    seg = rng.randint(0, 40, shape).astype(np.int32)
    seg[seg == 3] = 4
    seg.flat[-1] = 41                                        # labels 3 and 40 (at least) absent
    nb = 42
    d_seg = _dev(seg)
    centres = torch.full((nb, 3), SENTINEL, dtype=torch.float64, device='cuda')
    ws = torch.full((4 * nb, ), 77, dtype=torch.int64, device='cuda')
    lb.check(lb.lib().isb_centroids_3d(lb.ptr(d_seg), D, H, W, nb, lb.ptr(centres), lb.ptr(ws), C.c_size_t(32 * nb), lb.stream_ptr()))
    got = _host(centres)
    s = seg.ravel()
    n = np.bincount(s, minlength=nb)
    want = np.full((nb, 3), -1.0)
    idx = np.unravel_index(np.arange(s.size), shape)
    for k in range(3):
        sums = np.bincount(s, weights=idx[k], minlength=nb)
        want[n > 0, k] = sums[n > 0] / n[n > 0]
    np.testing.assert_array_equal(got, want)
