"""
``isb_enforce_connectivity`` against the oracle bit for bit on the maps where labelling in 32 x 64 tiles can go wrong: components
that cross the tile seams many times, components whose first pixel lies in a later tile than most of their pixels, sides that do
not fill the tiles, the oversize path on a whole-map component, small pieces whose window is clipped by the border or does not
fit the shared-memory window, maps with tens of thousands of components, and label ids above 2^16 at the 8192^2 size.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TH, TW = 32, 64


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
    assert np.array_equal(got, want), '%d pixels differ' % int((got != want).sum())
    assert n == max(int(want.max()) + 1, 1)


def _spiral(n):
    """a one-pixel-wide square spiral (label 1) with a one-pixel gap (label 0) between its turns, n x n"""
    lab = np.zeros((n, n), dtype=np.int64)
    y0, x0, y1, x1 = 0, 0, n - 1, n - 1
    while y0 <= y1 and x0 <= x1:
        lab[y0, x0:x1 + 1] = 1
        lab[y0:y1 + 1, x1] = 1
        if y1 > y0:
            lab[y1, x0:x1 + 1] = 1
        if x1 > x0 and y1 - y0 > 2:
            lab[y0 + 2:y1 + 1, x0] = 1
        if y0 + 2 < y1 - 1:
            lab[y0 + 2, x0] = 1
        y0, x0, y1, x1 = y0 + 2, x0 + 2, y1 - 2, x1 - 2
        if y0 <= y1 and x0 <= x1:
            lab[y0, x0 - 1] = 1
    return lab


@pytest.mark.parametrize('min_size,max_size', [(10, 100000), (10, 500), (200000, 400000)])
def test_spiral_crosses_seams(oracle, min_size, max_size):
    """two interleaved spirals: every turn crosses several tile seams, so the seam unions form long chains"""
    _check_conn(oracle, _spiral(301), min_size, max_size)


def test_comb_crosses_seams(oracle):
    """combs whose teeth run across many tile rows and whose spines lie in the last tile row or column"""
    H, W = 300, 410
    lab = np.zeros((H, W), dtype=np.int64)
    lab[:, ::2] = 1          # vertical teeth
    lab[-1, :] = 1           # spine on the bottom row
    lab[:40, :] = np.where(np.arange(40)[:, None] % 2 == 0, 2, 3)  # horizontal teeth
    lab[:40, -1] = 2         # joined on the last column
    _check_conn(oracle, lab, 30, 100000)
    _check_conn(oracle, lab, 30, 700)


@pytest.mark.parametrize('dy,dx', [(0, TW), (TH, 0), (TH, TW)])
def test_first_pixel_in_a_later_tile(oracle, dy, dx):
    """a U whose top-left pixel (its id) lies one tile right of and/or below the bulk of its pixels"""
    H, W = 4 * TH, 4 * TW
    lab = np.zeros((H, W), dtype=np.int64)
    # the U: a thick bar along the bottom rows, two arms going up; the right arm starts higher
    y0, x0 = 5 + dy, 3 + dx
    lab[H - 10:H - 2, 2:W - 2] = 7
    lab[y0:H - 2, x0:x0 + 2] = 7
    lab[H - 40:H - 2, 2:4] = 7
    lab[H - 30:H - 20, 10:20] = 8  # a small piece inside the U
    _check_conn(oracle, lab, 50, 100000)
    _check_conn(oracle, lab, 50, 300)


@pytest.mark.parametrize('shape', [(1, 1), (1, 700), (700, 1), (33, 65), (31, 63), (97, 130), (65, 129)])
def test_sides_not_multiples_of_the_tile(oracle, shape):
    rng = np.random.RandomState(shape[0] * 7 + shape[1])
    lab = rng.randint(0, 3, shape)
    _check_conn(oracle, lab, 4, 64)
    blocks = np.kron(rng.randint(0, 50, (shape[0] // 5 + 1, shape[1] // 5 + 1)), np.ones((5, 5), dtype=np.int64))[:shape[0], :shape[1]]
    _check_conn(oracle, blocks, 20, 60)


def test_one_label_over_4096(oracle):
    """one component over the whole map: oversize, cut by the replay from the box the root pass summed"""
    lab = np.zeros((4096, 4096), dtype=np.int64)
    _check_conn(oracle, lab, 300000, 1 << 20)


def test_small_pieces_outside_the_window(oracle):
    """small pieces whose box with its ring exceeds the window (long lines, a sparse staircase) next to ones that fit"""
    H, W = 256, 1200
    lab = np.zeros((H, W), dtype=np.int64)
    lab[H // 2:, :] = 1
    lab[10, 5:W - 5] = 2                   # a 1 x 1190 line: window 3 x 1192
    for k in range(90):                    # a staircase over a 90 x 180 box
        lab[30 + k, 20 + 2 * k:23 + 2 * k] = 3
    lab[200:203, 100:104] = 4              # fits
    _check_conn(oracle, lab, 2000, 100000)
    _check_conn(oracle, lab, 600, 100000)


def test_small_pieces_on_every_border(oracle):
    """windows clipped by each border and each corner"""
    rng = np.random.RandomState(3)
    H, W = 130, 200
    lab = np.kron(rng.randint(0, 6, (H // 26 + 1, W // 40 + 1)), np.ones((26, 40), dtype=np.int64))[:H, :W]
    for y, x in [(0, 0), (0, W - 3), (H - 3, 0), (H - 3, W - 3), (0, 90), (H - 2, 90), (60, 0), (60, W - 1)]:
        lab[y:y + 3, x:x + 3] = 100 + y + x
    lab[0, :] = 50                         # a whole-border row: a thin piece touching both sides
    _check_conn(oracle, lab, 250, 5000)


def test_three_label_noise_512(oracle):
    """tens of thousands of components, most of them a few pixels"""
    lab = np.random.RandomState(5).randint(0, 3, (512, 512))
    _check_conn(oracle, lab, 8, 200)
    _check_conn(oracle, lab, 40, 30)


def _voronoi(n, cell, seed):
    """a Voronoi map of one jittered seed per cell x cell square (ids row-major over the squares), with 1% pixels relabelled to
    a neighbouring square's id so that every region has small fragments"""
    rng = np.random.RandomState(seed)
    g = n // cell
    sy = (np.arange(g)[:, None] * cell + rng.randint(0, cell, (g, g))).astype(np.float32)
    sx = (np.arange(g)[None, :] * cell + rng.randint(0, cell, (g, g))).astype(np.float32)
    out = np.empty((n, n), dtype=np.int64)
    xs = np.arange(n)
    cx = np.minimum(xs // cell, g - 1)
    for y in range(n):
        cy = min(y // cell, g - 1)
        best = np.full(n, np.inf, dtype=np.float32)
        lab = np.zeros(n, dtype=np.int64)
        for oy in (-1, 0, 1):
            ny = cy + oy
            if ny < 0 or ny >= g:
                continue
            for ox in (-1, 0, 1):
                nx = np.clip(cx + ox, 0, g - 1)
                d = (sy[ny, nx] - y) ** 2 + (sx[ny, nx] - xs) ** 2
                better = d < best
                best[better] = d[better]
                lab[better] = ny * g + nx[better]
        out[y] = lab
    noise = rng.random_sample((n, n)) < 0.01
    out[noise] = np.roll(out, 3, axis=1)[noise]
    return out


def test_voronoi_8192(oracle):
    """the config-5 size, about 80 k labels: ids above 2^16, rank blocks all over the bitmap"""
    lab = _voronoi(8192, 29, 11)
    assert lab.max() >= 1 << 16
    seg = lab.size / (lab.max() + 1)
    _check_conn(oracle, lab, int(0.5 * seg), int(3 * seg))
