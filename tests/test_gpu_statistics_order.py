"""The per-segment statistics give the same bits on every launch, and those bits are the host model's.

``isb_segment_stats_2d`` / ``_accumulate`` / ``_deviation`` (csrc/segment_stats.cu) and ``isb_gray_stats`` and its banded entries
(csrc/native_misc.cu) add each label's flushed run partials exactly and round once (csrc/exact_sum.cuh), so the result does not
depend on which warp flushes first.  tests/statistics_order_reference.py restates the documented order in numpy; every output here
must equal it bit for bit, on inputs where any other association shows in the last bits (values over the whole float32 range, both
signs), at the strip and warp edges, with NaN, infinite and negative-zero pixels, one label over many warps and one label per pixel.
Three launches of every entry, and launches interleaved on two streams, must give identical bytes.
"""
import ctypes as C

import numpy as np
import pytest

import statistics_order_reference as ref

SENTINEL = -12345.625


def _torch():
    import torch
    return torch


def _lb():
    from pyimsegm_b200 import _lib
    return _lib


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    """an array's bytes as int64 words (float64 compared bit for bit: NaN == NaN, -0 != +0)"""
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _assert_bits(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = np.flatnonzero((g != w).ravel())
    assert bad.size == 0, '%s: %d of %d values differ, first at %d: got %r, want %r' % (
        what, bad.size, g.size, bad[0], np.ravel(got)[bad[0]], np.ravel(want)[bad[0]])


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------

def _wide(shape, rng, dtype):
    """magnitudes over the whole range of the dtype, both signs; float64 from 1e-300 to 1e300 (zero or infinite in float32)"""
    lo, hi = (-300, 300) if dtype == 'float64' else (-44, 38)
    return (10.0 ** rng.uniform(lo, hi, shape) * rng.choice([-1.0, 1.0], shape)).astype(dtype)


def _image(shape, dtype, rng, kind='wide'):
    if dtype == 'uint8':
        return rng.randint(0, 256, shape).astype(np.uint8)
    if dtype == 'uint16':
        return rng.randint(0, 65536, shape).astype(np.uint16)
    if kind == 'wide':
        return _wide(shape, rng, dtype)
    img = rng.normal(0.3, 2.0, shape).astype(dtype)
    if kind == 'special':                                   # NaN, both infinities and -0 on a few pixels
        flat = img.reshape(-1)
        idx = rng.permutation(flat.size)
        k = max(1, flat.size // 50)
        flat[idx[:k]] = np.nan
        flat[idx[k:2 * k]] = np.inf
        flat[idx[2 * k:3 * k]] = -np.inf
        flat[idx[3 * k:4 * k]] = -0.0
    return img


def _labels(kind, H, W, rng):
    """label map [H, W] int32 and the label bound nb"""
    yy, xx = np.mgrid[:H, :W]
    if kind == 'one':
        seg = np.zeros((H, W), int)
    elif kind == 'per_pixel':
        seg = yy * W + xx
    elif kind == 'stripes':                                 # a label repeats on lanes of one warp and across warps and strips
        seg = (yy // 5) * 3 + (xx // 3) % 3
    elif kind == 'stripes32':
        seg = (yy // 40) * 3 + (xx // 32) % 3
    else:                                                   # labels 0 and 5 absent, the bound 2 above the largest
        seg = np.array([1, 2, 3, 4, 6])[rng.randint(0, 5, (H, W))]
        return np.ascontiguousarray(seg, dtype=np.int32), 9
    return np.ascontiguousarray(seg, dtype=np.int32), int(seg.max()) + 1


# ------------------------------------------------------------------------------------------------------------------------------
# device calls
# ------------------------------------------------------------------------------------------------------------------------------

def _stats_2d(d_img, d_seg, nb, stream=None):
    """isb_segment_stats_2d with every statistic, centres and counts -> device (feat [nb, 9], centres, counts)"""
    torch, lb = _torch(), _lb()
    lib = lb.lib()
    H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
    feat = torch.full((nb, 9), SENTINEL, dtype=torch.float64, device='cuda')
    cen = torch.full((nb, 2), SENTINEL, dtype=torch.float64, device='cuda')
    cnt = torch.full((nb, ), -7, dtype=torch.int32, device='cuda')
    wsb = lib.isb_segment_stats_workspace_bytes(nb)
    ws = torch.full((wsb, ), 0x5A, dtype=torch.uint8, device='cuda')
    st = C.c_void_p(stream.cuda_stream) if stream is not None else lb.stream_ptr()
    lb.check(lib.isb_segment_stats_2d(lb.ptr(d_img), lb.dtype_code(d_img.dtype), lb.ptr(d_seg), H, W, nb, 7, lb.ptr(feat), 9, 0,
                                      lb.ptr(cen), lb.ptr(cnt), lb.ptr(ws), C.c_size_t(wsb), st))
    return feat, cen, cnt


def _host_2d(out):
    _torch().cuda.synchronize()
    feat, cen, cnt = (t.cpu().numpy() for t in out)
    return feat[:, :3], feat[:, 3:6], feat[:, 6:9], cen, cnt


def _stats_banded(d_img, d_seg, nb, bands):
    """the banded trio over row bands [(lo, hi), ...] -> (mean, std, energy, centres, counts) on the host"""
    torch, lb = _torch(), _lb()
    lib = lb.lib()
    H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
    code = lb.dtype_code(d_img.dtype)
    row_img, row_seg = W * 3 * d_img.element_size(), W * 4
    acc = torch.zeros((nb, 6), dtype=torch.float64, device='cuda')
    iacc = torch.zeros((nb, 3), dtype=torch.int64, device='cuda')
    var = torch.zeros((nb, 3), dtype=torch.float64, device='cuda')
    meanf = torch.zeros((nb, 3), dtype=torch.float32, device='cuda')
    for lo, hi in bands:
        lb.check(lib.isb_segment_stats_accumulate(C.c_void_p(d_img.data_ptr() + lo * row_img), code, C.c_void_p(d_seg.data_ptr() + lo * row_seg),
                                                  hi - lo, W, lo, nb, lb.ptr(acc), lb.ptr(iacc), lb.stream_ptr()))
    for lo, hi in bands:
        lb.check(lib.isb_segment_stats_deviation(C.c_void_p(d_img.data_ptr() + lo * row_img), code, C.c_void_p(d_seg.data_ptr() + lo * row_seg),
                                                 hi - lo, W, nb, lb.ptr(acc), lb.ptr(iacc), lb.ptr(meanf), lb.ptr(var), lb.stream_ptr()))
    feat = torch.full((nb, 9), SENTINEL, dtype=torch.float64, device='cuda')
    cen = torch.full((nb, 2), SENTINEL, dtype=torch.float64, device='cuda')
    cnt = torch.full((nb, ), -7, dtype=torch.int32, device='cuda')
    lb.check(lib.isb_segment_stats_finish(nb, 7, lb.ptr(acc), lb.ptr(var), lb.ptr(iacc), lb.ptr(feat), 9, 0, lb.ptr(cen), lb.ptr(cnt),
                                          lb.stream_ptr()))
    return _host_2d((feat, cen, cnt))


def _gray(d_vol, d_seg, nb, stream=None):
    """isb_gray_stats with mean, std and energy -> device feat [nb, 3]"""
    torch, lb = _torch(), _lb()
    lib = lb.lib()
    feat = torch.full((nb, 3), SENTINEL, dtype=torch.float64, device='cuda')
    wsb = lib.isb_gray_stats_workspace_bytes(nb)
    ws = torch.full((wsb, ), 0x5A, dtype=torch.uint8, device='cuda')
    st = C.c_void_p(stream.cuda_stream) if stream is not None else lb.stream_ptr()
    lb.check(lib.isb_gray_stats(lb.ptr(d_vol), lb.dtype_code(d_vol.dtype), lb.ptr(d_seg), C.c_longlong(d_vol.numel()), nb, 7, lb.ptr(feat),
                                3, 0, lb.ptr(ws), C.c_size_t(wsb), st))
    return feat


def _gray_banded(d_vol, d_seg, nb, slabs):
    torch, lb = _torch(), _lb()
    lib = lb.lib()
    code, isz = lb.dtype_code(d_vol.dtype), d_vol.element_size()
    acc = torch.zeros((nb, 2), dtype=torch.float64, device='cuda')
    cnt = torch.zeros((nb, ), dtype=torch.int64, device='cuda')
    var = torch.zeros((nb, ), dtype=torch.float64, device='cuda')
    meanf = torch.zeros((nb, ), dtype=torch.float32, device='cuda')
    for lo, hi in slabs:
        lb.check(lib.isb_gray_stats_accumulate(C.c_void_p(d_vol.data_ptr() + lo * isz), code, C.c_void_p(d_seg.data_ptr() + lo * 4),
                                               C.c_longlong(hi - lo), nb, lb.ptr(acc), lb.ptr(cnt), lb.stream_ptr()))
    for lo, hi in slabs:
        lb.check(lib.isb_gray_stats_deviation(C.c_void_p(d_vol.data_ptr() + lo * isz), code, C.c_void_p(d_seg.data_ptr() + lo * 4),
                                              C.c_longlong(hi - lo), nb, lb.ptr(acc), lb.ptr(cnt), lb.ptr(meanf), lb.ptr(var), lb.stream_ptr()))
    feat = torch.full((nb, 3), SENTINEL, dtype=torch.float64, device='cuda')
    lb.check(lib.isb_gray_stats_finish(nb, 7, lb.ptr(acc), lb.ptr(var), lb.ptr(cnt), lb.ptr(feat), 3, 0, lb.stream_ptr()))
    _torch().cuda.synchronize()
    return feat.cpu().numpy()


def _check_2d(img, seg, nb, got, what, bands=None):
    mean, std, energy, centres, counts = ref.colour_stats(img, seg, nb, bands=bands)
    for name, g, w in zip(('mean', 'std', 'energy', 'centres'), got[:4], (mean, std, energy, centres)):
        _assert_bits(g, w, '%s %s' % (what, name))
    np.testing.assert_array_equal(got[4], counts, err_msg=what + ' counts')


def _check_gray(vol, seg, nb, got, what, slabs=None):
    for k, (name, w) in enumerate(zip(('mean', 'std', 'energy'), ref.gray_stats(vol, seg, nb, slabs=slabs))):
        _assert_bits(got[:, k], w, '%s %s' % (what, name))


# ------------------------------------------------------------------------------------------------------------------------------
# colour statistics against the host model, and their reruns
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('W', [31, 32, 33, 257, 300])
@pytest.mark.parametrize('H', [1, 15, 16, 17, 70])
def test_segment_stats_bits_equal_the_host_model(H, W):
    """every label map, dtype and value kind at the strip and warp edges: three launches, each bit for bit the model's"""
    rng = np.random.RandomState(H * 1000 + W)
    for kind in ('one', 'per_pixel', 'stripes', 'stripes32', 'absent'):
        seg, nb = _labels(kind, H, W, rng)
        d_seg = _dev(seg)
        for dtype, values in (('uint8', 'wide'), ('uint16', 'wide'), ('float32', 'wide'), ('float64', 'wide'),
                              ('float32', 'special'), ('float64', 'special')):
            img = _image((H, W, 3), dtype, rng, values)
            d_img = _dev(img)
            what = '%dx%d %s %s %s' % (H, W, kind, dtype, values)
            runs = [_host_2d(_stats_2d(d_img, d_seg, nb)) for _ in range(3)]
            _check_2d(img, seg, nb, runs[0], what)
            for r in runs[1:]:
                for a, b in zip(runs[0], r):
                    assert a.tobytes() == b.tobytes(), what + ': a rerun gave other bytes'


@pytest.mark.gpu
def test_segment_stats_one_label_over_4096_squared():
    """one label over 4096 x 4096: 256 strips of 128 warps flush into it"""
    rng = np.random.RandomState(11)
    H = W = 4096
    seg = np.zeros((H, W), np.int32)
    img = _wide((H, W, 3), rng, 'float32')
    d_img, d_seg = _dev(img), _dev(seg)
    runs = [_host_2d(_stats_2d(d_img, d_seg, 1)) for _ in range(3)]
    _check_2d(img, seg, 1, runs[0], 'one label 4096^2')
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert a.tobytes() == b.tobytes(), 'one label 4096^2: a rerun gave other bytes'


@pytest.mark.gpu
def test_segment_stats_two_streams_interleaved():
    """launches queued alternately on two streams, each with its own buffers, give the bytes of a lone launch"""
    torch = _torch()
    rng = np.random.RandomState(12)
    H, W = 517, 700
    seg, nb = _labels('stripes', H, W, rng)
    img = _wide((H, W, 3), rng, 'float32')
    vol = _wide((40, 64, 70), rng, 'float32')
    vseg = np.ascontiguousarray((np.arange(vol.size) // 37 % 500).reshape(vol.shape), dtype=np.int32)
    d_img, d_seg, d_vol, d_vseg = _dev(img), _dev(seg), _dev(vol), _dev(vseg)
    alone = _host_2d(_stats_2d(d_img, d_seg, nb))
    gray_alone = _gray(d_vol, d_vseg, 500).cpu().numpy()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    outs, gouts = [], []
    for i in range(6):
        s = streams[i % 2]
        with torch.cuda.stream(s):
            outs.append(_stats_2d(d_img, d_seg, nb, stream=s))
            gouts.append(_gray(d_vol, d_vseg, 500, stream=s))
    torch.cuda.synchronize()
    for o, g in zip(outs, gouts):
        for a, b in zip(alone, _host_2d(o)):
            assert a.tobytes() == b.tobytes(), 'colour statistics on two streams gave other bytes'
        assert g.cpu().numpy().tobytes() == gray_alone.tobytes(), 'gray statistics on two streams gave other bytes'


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['uint8', 'float32', 'float64'])
def test_segment_stats_banded_bits_equal_the_host_model(dtype):
    """bands add their rounded totals in band order: bit for bit the model over the same bands, and identical on a rerun"""
    rng = np.random.RandomState(13)
    H, W = 70, 257
    for kind in ('one', 'stripes', 'absent'):
        seg, nb = _labels(kind, H, W, rng)
        img = _image((H, W, 3), dtype, rng, 'special' if dtype != 'uint8' else 'wide')
        d_img, d_seg = _dev(img), _dev(seg)
        bands = [(0, 1), (1, 17), (17, 50), (50, H)]
        got = _stats_banded(d_img, d_seg, nb, bands)
        _check_2d(img, seg, nb, got, 'banded %s %s' % (kind, dtype), bands=bands)
        again = _stats_banded(d_img, d_seg, nb, bands)
        for a, b in zip(got, again):
            assert a.tobytes() == b.tobytes(), 'banded %s %s: a rerun gave other bytes' % (kind, dtype)


# ------------------------------------------------------------------------------------------------------------------------------
# gray statistics
# ------------------------------------------------------------------------------------------------------------------------------

GRAY_SHAPES = [(1, 1, 1), (1, 1, 33), (1, 17, 1), (3, 1, 16), (5, 7, 31), (9, 40, 33)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape', GRAY_SHAPES)
@pytest.mark.parametrize('dtype', ['uint8', 'uint16', 'float32', 'float64'])
def test_gray_stats_bits_equal_the_host_model(shape, dtype):
    rng = np.random.RandomState(sum(shape) * 7 + len(dtype))
    n = int(np.prod(shape))
    for kind in ('one', 'runs', 'per_voxel', 'absent'):
        if kind == 'one':
            seg, nb = np.zeros(n, np.int32), 1
        elif kind == 'runs':                                # runs of 1 to 40 voxels across the 16-voxel strips
            seg = np.repeat(np.arange(n), rng.randint(1, 41, n))[:n] % 5
            nb = int(seg.max()) + 1
        elif kind == 'per_voxel':
            seg, nb = np.arange(n), n
        else:
            seg, nb = np.array([1, 3])[rng.randint(0, 2, n)], 6
        seg = np.ascontiguousarray(seg, dtype=np.int32).reshape(shape)
        for values in (('wide', 'special') if dtype.startswith('float') else ('wide', )):
            vol = _image(shape, dtype, rng, values)
            d_vol, d_seg = _dev(vol), _dev(seg)
            what = 'gray %s %s %s %s' % (shape, dtype, kind, values)
            runs = [_gray(d_vol, d_seg, nb) for _ in range(3)]
            _torch().cuda.synchronize()
            runs = [r.cpu().numpy() for r in runs]
            _check_gray(vol, seg, nb, runs[0], what)
            assert runs[1].tobytes() == runs[0].tobytes() and runs[2].tobytes() == runs[0].tobytes(), what + ': a rerun gave other bytes'
            slabs = [(0, n // 3), (n // 3, n)] if n > 2 else [(0, n)]
            _check_gray(vol, seg, nb, _gray_banded(d_vol, d_seg, nb, slabs), what + ' slabs', slabs=slabs)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['one', 'supervoxels'])
def test_gray_stats_16m_voxels(kind):
    """256^3 voxels: one label (a million strips flush into it) or 8^3 blocks"""
    rng = np.random.RandomState(14)
    shape = (256, 256, 256)
    vol = _wide(shape, rng, 'float32')
    if kind == 'one':
        seg, nb = np.zeros(shape, np.int32), 1
    else:
        z, y, x = np.indices(shape, dtype=np.int32) // 8
        seg, nb = np.ascontiguousarray((z * 32 + y) * 32 + x), 32 ** 3
    d_vol, d_seg = _dev(vol), _dev(seg)
    runs = [_gray(d_vol, d_seg, nb) for _ in range(3)]
    _torch().cuda.synchronize()
    runs = [r.cpu().numpy() for r in runs]
    _check_gray(vol, seg, nb, runs[0], 'gray 256^3 %s' % kind)
    assert runs[1].tobytes() == runs[0].tobytes() and runs[2].tobytes() == runs[0].tobytes()


# ------------------------------------------------------------------------------------------------------------------------------
# failure surface
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_argument_errors_raise_before_any_launch():
    """a short workspace, a missing buffer and a pixel count whose flushes could overflow the exact sums: ValueError, and no kernel
    launched"""
    torch, lb = _torch(), _lb()
    lib = lb.lib()
    nb, H, W = 5, 4, 8
    d_img = torch.zeros((H, W, 3), dtype=torch.float32, device='cuda')
    d_seg = torch.zeros((H, W), dtype=torch.int32, device='cuda')
    acc = torch.zeros((nb, 6), dtype=torch.float64, device='cuda')
    iacc = torch.zeros((nb, 3), dtype=torch.int64, device='cuda')
    var = torch.zeros((nb, 3), dtype=torch.float64, device='cuda')
    meanf = torch.zeros((nb, 3), dtype=torch.float32, device='cuda')
    feat = torch.zeros((nb, 9), dtype=torch.float64, device='cuda')
    wsb = lib.isb_segment_stats_workspace_bytes(nb)
    gwsb = lib.isb_gray_stats_workspace_bytes(nb)
    ws = torch.zeros((max(wsb, gwsb), ), dtype=torch.uint8, device='cuda')
    p, s = lb.ptr, lb.stream_ptr()
    big = 1 << 16                                            # 2^32 pixels
    calls = [
        lambda: lib.isb_segment_stats_2d(p(d_img), 2, p(d_seg), H, W, nb, 7, p(feat), 9, 0, None, None, p(ws), C.c_size_t(wsb - 1), s),
        lambda: lib.isb_segment_stats_2d(p(d_img), 2, p(d_seg), big, big, nb, 7, p(feat), 9, 0, None, None, p(ws), C.c_size_t(wsb), s),
        lambda: lib.isb_segment_stats_accumulate(p(d_img), 2, p(d_seg), big, big, 0, nb, p(acc), p(iacc), s),
        lambda: lib.isb_segment_stats_deviation(p(d_img), 2, p(d_seg), H, W, nb, p(acc), p(iacc), None, p(var), s),
        lambda: lib.isb_segment_stats_deviation(p(d_img), 2, p(d_seg), big, big, nb, p(acc), p(iacc), p(meanf), p(var), s),
        lambda: lib.isb_gray_stats(p(d_img), 2, p(d_seg), C.c_longlong(H * W), nb, 7, p(feat), 9, 0, p(ws), C.c_size_t(gwsb - 1), s),
        lambda: lib.isb_gray_stats(p(d_img), 2, p(d_seg), C.c_longlong((1 << 31) + 1), nb, 7, p(feat), 9, 0, p(ws), C.c_size_t(gwsb), s),
        lambda: lib.isb_gray_stats_accumulate(p(d_img), 2, p(d_seg), C.c_longlong(1 << 32), nb, p(acc), p(iacc), s),
        lambda: lib.isb_gray_stats_deviation(p(d_img), 2, p(d_seg), C.c_longlong(H * W), nb, p(acc), p(iacc), None, p(var), s),
        lambda: lib.isb_gray_stats_deviation(p(d_img), 2, p(d_seg), C.c_longlong(1 << 32), nb, p(acc), p(iacc), p(meanf), p(var), s),
    ]
    torch.cuda.synchronize()
    n0 = lib.isb_launch_count()
    for call in calls:
        with pytest.raises(ValueError):
            lb.check(call())
    assert lib.isb_launch_count() == n0, 'an argument error launched a kernel'
    torch.cuda.synchronize()
