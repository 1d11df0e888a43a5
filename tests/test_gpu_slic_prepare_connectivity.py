"""
The two SLIC stages around the k-means sweeps, each against the oracle bit for bit.

* ``isb_slic_prepare``: the planar Lab image (rescale, gaussian blur, rgb2lab, 1/compactness) for every blur radius, input dtype,
  gray and RGB, images smaller than the radius, widths and heights that do not fill the kernel's tiles, and the band mode that
  takes the min/max from the caller.  Labels can hide a 1-ulp difference in the Lab planes, so the planes are compared directly.
* ``isb_enforce_connectivity``: hand-built label maps that reach every branch of the small-piece BFS (fragments, long
  serpentines, rings, checkerboards, border pieces, long small->small chains, pieces cut out of oversize components, a BFS
  truncated at max_size, min_size above 512 where the BFS queue moves to global memory) and the k-means map of the benchmark image.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


# -- Lab planes ---------------------------------------------------------------------------------------------------------------

def _device_lab(img, sigma, ratio, rescale, minmax=None):
    import torch
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.engine import gaussian_half_kernel
    lib = _lib.lib()
    H, W = img.shape[:2]
    Cn = 1 if img.ndim == 2 else img.shape[2]
    d_img = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    lab = torch.full((3, H, W), 7.0, dtype=torch.float64, device='cuda')
    mm = torch.zeros(4, dtype=torch.float64, device='cuda')
    if minmax is not None:
        mm[0], mm[1] = minmax
    w_half, radius = gaussian_half_kernel(sigma)
    _lib.check(lib.isb_slic_prepare(_lib.ptr(d_img), _lib.dtype_code(img.dtype), H, W, Cn, w_half.ctypes.data_as(C.POINTER(C.c_double)),
                                    radius, C.c_double(ratio), rescale, _lib.ptr(lab), _lib.ptr(mm), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return lab.cpu().numpy().transpose(1, 2, 0)


def _oracle_lab(oracle, img, sigma, ratio, minmax):
    """the reference wrapper's rescale in numpy, in the image's own dtype (float32 stays float32), then f64"""
    x = img
    if x.ndim == 2:
        x = x[..., None]
    if x.shape[2] == 1:
        x = np.repeat(x, 3, axis=2)
    if minmax is not None:
        mn, mx = (x.dtype.type(v) for v in minmax)
        if mn != 0.0 or mx != 1.0:
            x = (x - mn) / float(mx - mn)
    x = x.astype(np.float64)
    if sigma > 0:
        x = oracle.gaussian_blur(x, sigma)
    return oracle.rgb2lab_scaled(x, ratio)


def _assert_same_bits(got, want):
    assert got.shape == want.shape
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w)
    g, w = got[~nan_g], want[~nan_w]
    bad = np.flatnonzero(g.view(np.int64) != w.view(np.int64))
    assert bad.size == 0, '%d values differ, first %r vs %r' % (bad.size, g[bad[:3]], w[bad[:3]])


def _image(shape, dtype, seed):
    rng = np.random.RandomState(seed)
    if dtype == np.uint8:
        return rng.randint(0, 256, shape).astype(np.uint8)
    if dtype == np.uint16:
        return rng.randint(0, 65536, shape).astype(np.uint16)
    return (rng.random_sample(shape) * 3.0 - 1.0).astype(dtype)


def _check_lab(oracle, img, sigma, rescale=1, minmax=None, ratio=0.37):
    if rescale == 1:
        minmax = (float(img.min()), float(img.max()))
    got = _device_lab(img, sigma, ratio, rescale, minmax if rescale == 2 else None)
    want = _oracle_lab(oracle, img, sigma, ratio, minmax if rescale else None)
    _assert_same_bits(got, want)


@pytest.mark.parametrize('sigma', [0, 0.5, 1, 2])
@pytest.mark.parametrize('dtype', [np.uint8, np.uint16, np.float32, np.float64])
@pytest.mark.parametrize('gray', [False, True])
def test_lab_planes_bit_exact_numpy_rescale(oracle, sigma, dtype, gray):
    """the reference's min-max rescale as numpy computes it, in the image's own dtype (float32 in float32), then f64"""
    # 75 x 150: W not a multiple of 32 or of the 128-column tile, H not a multiple of the 64-row strip or the 8-row chunk
    shape = (75, 150) if gray else (75, 150, 3)
    _check_lab(oracle, _image(shape, dtype, seed=int(sigma * 10) + 3 * gray), sigma)


@pytest.mark.parametrize('shape', [(3, 5), (1, 1), (7, 2), (2, 9), (1, 300), (300, 1), (17, 129)])
@pytest.mark.parametrize('sigma', [1, 2])
def test_lab_planes_smaller_than_radius(oracle, shape, sigma):
    """sides below the radius reflect more than once"""
    _check_lab(oracle, _image(shape + (3,), np.float64, seed=shape[0] * 31 + shape[1]), sigma)


@pytest.mark.parametrize('rescale', [0, 2])
@pytest.mark.parametrize('sigma', [0, 1, 2])
def test_lab_planes_rescale_modes(oracle, rescale, sigma):
    """rescale 0 takes the image as it is; rescale 2 (a band of a larger image) takes min/max from the caller"""
    img = _image((70, 133, 3), np.float64, seed=11) * 0.3 + 0.4
    _check_lab(oracle, img, sigma, rescale=rescale, minmax=(0.25, 0.85) if rescale == 2 else None)


def test_lab_planes_constant_image(oracle):
    """0/0 in the rescale: every plane is NaN on both sides"""
    img = np.full((40, 70, 3), 0.5)
    _check_lab(oracle, img, 1)


def test_lab_planes_full_size(oracle):
    from bench import synth_image
    _check_lab(oracle, synth_image(2), 1, ratio=1.0 / (29 * 0.2) ** 1.5)


# -- connectivity -------------------------------------------------------------------------------------------------------------

def _device_conn(labels, min_size, max_size):
    import torch
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    H, W = labels.shape
    d_in = torch.from_numpy(np.ascontiguousarray(labels, dtype=np.int32)).cuda()
    out = torch.empty((H, W), dtype=torch.int32, device='cuda')
    nl = torch.zeros(1, dtype=torch.int32, device='cuda')
    wsb = lib.isb_connectivity_workspace_bytes(H, W)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    _lib.check(lib.isb_enforce_connectivity(_lib.ptr(d_in), H, W, min_size, max_size, _lib.ptr(out), _lib.ptr(nl), _lib.ptr(ws),
                                            C.c_size_t(wsb), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), int(nl.item())


def _check_conn(oracle, labels, min_size, max_size):
    got, n = _device_conn(labels, min_size, max_size)
    want = oracle.enforce_connectivity(labels, min_size, max_size)
    assert np.array_equal(got, want)
    assert n == max(int(want.max()) + 1, 1)


def _blocks(H, W, cell, seed):
    """a background of cell x cell blocks with random labels"""
    rng = np.random.RandomState(seed)
    g = rng.randint(0, 1000, ((H + cell - 1) // cell, (W + cell - 1) // cell))
    return np.kron(g, np.ones((cell, cell), dtype=np.int64))[:H, :W].copy()


def _serpentine(n, width):
    """pixel coordinates of a one-pixel-wide snake of n pixels that turns every `width` columns"""
    pts, y = [], 0
    while len(pts) < n:
        xs = range(width) if (y // 2) % 2 == 0 else range(width - 1, -1, -1)
        if y % 2 == 0:
            pts.extend((y, x) for x in xs)
        else:
            pts.append((y, width - 1 if (y // 2) % 2 == 0 else 0))
        y += 1
    return pts[:n]


@pytest.mark.parametrize('seed', [0, 1])
def test_conn_fragments(oracle, seed):
    """many 1-10 px pieces scattered over large blocks"""
    lab = _blocks(150, 190, 24, seed)
    rng = np.random.RandomState(seed)
    for _ in range(600):
        y, x = rng.randint(0, 150), rng.randint(0, 190)
        h, w = rng.randint(1, 4), rng.randint(1, 4)
        lab[y:y + h, x:x + w] = 2000 + rng.randint(0, 6)
    _check_conn(oracle, lab, 60, 900)


def test_conn_serpentines(oracle):
    """long BFS chains: snakes just under min_size, and one touching all four borders"""
    min_size = 300
    lab = _blocks(200, 260, 40, 3)
    for k, (oy, ox, w) in enumerate([(2, 3, 20), (40, 120, 9), (110, 30, 2), (150, 200, 40)]):
        for y, x in _serpentine(min_size - 1 - k, w):
            if oy + y < 200 and ox + x < 260:
                lab[oy + y, ox + x] = 5000 + k
    lab[0, :] = 6000
    lab[:, 0] = 6000
    lab[-1, :] = 6000
    lab[:, -1] = 6000
    lab[1:5, 1:5] = 6001  # border ring piece of 6000 surrounds it
    _check_conn(oracle, lab, min_size, 3000)


def test_conn_rings_and_checkerboard(oracle):
    lab = _blocks(128, 128, 32, 4)
    yy, xx = np.mgrid[:128, :128]
    for cy, cx, r in [(30, 30, 9), (90, 64, 14), (64, 110, 6)]:
        d = np.hypot(yy - cy, xx - cx)
        lab[(d >= r) & (d < r + 1.5)] = 7000 + r
        lab[d < 2] = 7100 + r
    cb = ((yy // 2 + xx // 2) % 2) + 7200
    lab[100:120, 4:40] = cb[100:120, 4:40]
    _check_conn(oracle, lab, 40, 600)


@pytest.mark.parametrize('min_size,max_size', [(700, 4000), (900, 900), (2500, 6000)])
def test_conn_min_size_over_512(oracle, min_size, max_size):
    lab = _blocks(256, 256, 16, 5)
    rng = np.random.RandomState(6)
    lab[rng.random_sample(lab.shape) < 0.02] = 9999
    _check_conn(oracle, lab, min_size, max_size)


@pytest.mark.parametrize('max_size', [16, 40, 64])
def test_conn_min_size_above_max_size(oracle, max_size):
    """every oversize component is cut into max_size pieces, which are small: their BFS stops at max_size"""
    lab = _blocks(96, 112, 12, 7)
    _check_conn(oracle, lab, 300, max_size)


def test_conn_small_chains(oracle):
    """one-pixel-wide columns, each only touching its left neighbour first: long small -> small merge chains"""
    H, W = 64, 300
    lab = np.zeros((H, W), dtype=np.int64)
    lab[:, :] = np.arange(W)[None, :] + 10
    lab[:8, :] = 1  # one kept piece on top
    _check_conn(oracle, lab, 60, 5000)
    lab[:8, :] = np.arange(W)[None, :] % 2 + 3
    _check_conn(oracle, lab, 60, 5000)


def test_conn_oversize_pieces(oracle):
    """components of max_size and more, split into pieces (negative comp), some of them small"""
    lab = _blocks(180, 200, 45, 8)
    rng = np.random.RandomState(9)
    lab[rng.random_sample(lab.shape) < 0.05] = 12345
    _check_conn(oracle, lab, 150, 400)


def test_conn_very_large_min_size(oracle):
    """min_size far above 512: every piece of the map is small and merges, with and without oversize splits"""
    lab = _blocks(512, 512, 128, 10)
    lab[(np.arange(512)[:, None] + np.arange(512)[None, :]) % 97 == 0] = 77
    _check_conn(oracle, lab, 60000, 200000)
    _check_conn(oracle, lab, 60000, 5000)


def test_conn_benchmark_kmeans_map(oracle, eng):
    """the oracle's k-means map of the benchmark image through the engine's connectivity entry"""
    import torch
    from bench import SP_REGUL, SP_SIZE, synth_image
    from pyimsegm_b200.superpixels import slic_params
    img = synth_image(2)
    n_seg, compact = slic_params(img.shape[:2], SP_SIZE, SP_REGUL)
    lo, hi = img.min(), img.max()
    km = oracle.slic((img - lo) / (hi - lo), n_seg, compact, sigma=1, enforce_conn=False)
    got, n = eng.enforce_connectivity(torch.from_numpy(km.astype(np.int32)).cuda(), n_seg)
    seg = km.shape[0] * km.shape[1] / n_seg
    want = oracle.enforce_connectivity(km, int(0.5 * seg), int(3 * seg))
    assert np.array_equal(got.cpu().numpy(), want) and int(n.item()) == want.max() + 1
