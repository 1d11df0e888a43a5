"""The cases the label-map passes' CTA and warp groupings create, beyond tests/test_gpu_segment_statistics.py and
tests/test_gpu_graph_energies.py.

- Colour statistics (``k_stats_pass1`` / ``k_stats_pass2``): runs that end in the same row on neighbouring lanes with one label are
  summed across the warp before one atomic flush.  The maps repeat a label on lanes that are not neighbours, end runs on every row,
  on some rows and at the strip end only, and put W on both sides of a warp and of a 256-column block.
- Adjacency (``k_edge_scan`` / ``k_edge_scan3d``): a CTA collects its pairs in a 512-slot shared-memory set; a tile that meets more
  pairs than that inserts the rest straight into the global table.  Random maps overflow every tile, mixed maps some; shapes that
  are not multiples of the 64 x 16 tile.
- Gather (``k_gather``): four pixels per thread with 16-byte loads and stores when every pointer is 16-byte aligned, one pixel at a
  time otherwise and for the tail.  Pixel counts on both sides of a multiple of four, K = 1, 3 and 8, views at every misalignment,
  and the elements beside the output left untouched.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_graph_energies import ref_edges
from test_gpu_segment_statistics import _check_colour, _image, _split, _stats_2d

pytestmark = pytest.mark.gpu

CANARY_I, CANARY_P = -777, -12345.625


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


# ------------------------------------------------------------------------------------------------------------------------------
# colour statistics
# ------------------------------------------------------------------------------------------------------------------------------

def stripe_map(H, W, col_period, row_period, n_col_labels):
    """label (x // col_period) % n_col_labels in bands of row_period rows, a new set of labels per band: a label repeats on lanes
    that are not neighbours, and every lane of a band's columns ends its run in the band's last row"""
    yy, xx = np.mgrid[:H, :W]
    seg = (yy // row_period) * n_col_labels + (xx // col_period) % n_col_labels
    return seg.astype(np.int32)


@pytest.mark.parametrize('W', [31, 32, 33, 257, 300])
@pytest.mark.parametrize('row_period', [1, 5, 16, 40])
@pytest.mark.parametrize('col_period', [1, 3, 32])
def test_stats_of_labels_repeating_across_a_warp(W, row_period, col_period):
    rng = np.random.RandomState(W * 10000 + row_period * 100 + col_period)
    H = 37
    seg = stripe_map(H, W, col_period, row_period, 3)
    nb = int(seg.max()) + 1
    img = _image((H, W, 3), 'float64', rng)
    table, centres, counts = _stats_2d(img, seg, nb, 7)
    mean, std, energy = _split(table, 0, 7)
    _check_colour(img, seg, nb, mean, std, energy, centres, counts, '%dx%d stripes %d/%d' % (H, W, col_period, row_period))


def test_stats_of_runs_ending_on_scattered_rows():
    """vertical runs of random lengths per column: neighbouring lanes end their runs of one label on different rows"""
    rng = np.random.RandomState(8)
    H, W = 70, 290
    cuts = rng.rand(H, W) < 0.15
    seg = (np.cumsum(cuts, axis=0) % 4 + 4 * (np.arange(W) // 7)[None, :]).astype(np.int32)
    nb = int(seg.max()) + 1
    img = _image((H, W, 3), 'float32', rng)
    table, centres, counts = _stats_2d(img, seg, nb, 7)
    mean, std, energy = _split(table, 0, 7)
    _check_colour(img, seg, nb, mean, std, energy, centres, counts, 'scattered runs')


# ------------------------------------------------------------------------------------------------------------------------------
# adjacency
# ------------------------------------------------------------------------------------------------------------------------------

def check_edges(eng, seg, what):
    seg = np.ascontiguousarray(seg, dtype=np.int32)
    want = ref_edges(seg)
    nb, cap = int(seg.max()) + 1, len(want) + 5
    out = eng.adjacency(eng.to_device(seg), nb, cap) if seg.ndim == 2 else eng.graph3d(eng.to_device(seg), nb, cap)
    n = int(eng.to_host(out[1])[0])
    assert n == len(want), '%s: the device counts %d edges, the map has %d' % (what, n, len(want))
    np.testing.assert_array_equal(eng.to_host(out[0][:n]), want, err_msg=what)


@pytest.mark.parametrize('shape', [(16, 64), (17, 65), (33, 130), (100, 301)])
def test_adjacency_of_tiles_with_more_pairs_than_the_shared_set(eng, shape):
    """random labels: a 64 x 16 tile meets up to 2 048 pairs, four times the set"""
    rng = np.random.RandomState(shape[0] * shape[1])
    check_edges(eng, rng.randint(0, 3000, shape), 'random %r' % (shape, ))


def test_adjacency_of_overflowing_tiles_beside_quiet_ones(eng):
    """random labels in some tiles, large blocks in the others: both routes into the global table in one call"""
    rng = np.random.RandomState(21)
    H, W = 130, 400
    yy, xx = np.mgrid[:H, :W]
    seg = (yy // 29) * 20 + xx // 29
    noisy = ((yy // 16) + (xx // 64)) % 3 == 0
    seg[noisy] = 1000 + rng.randint(0, 5000, int(noisy.sum()))
    check_edges(eng, seg, 'mixed tiles')


@pytest.mark.parametrize('shape', [(1, 1), (1, 70), (70, 1), (19, 67), (47, 129)])
def test_adjacency_of_shapes_off_the_tile_grid(eng, shape):
    rng = np.random.RandomState(shape[0] + 100 * shape[1])
    yy, xx = np.mgrid[:shape[0], :shape[1]]
    seg = (yy // 5) * 30 + xx // 7
    seg = rng.permutation(int(seg.max()) + 1)[seg]
    check_edges(eng, seg, 'blocks %r' % (shape, ))


def test_adjacency_3d_of_random_labels_overflowing_the_shared_set(eng):
    """a 256-voxel CTA meets up to 768 pairs of random labels"""
    rng = np.random.RandomState(5)
    check_edges(eng, rng.randint(0, 4000, (6, 9, 70)), 'random volume')


# ------------------------------------------------------------------------------------------------------------------------------
# gather
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('k', [1, 3, 8])
@pytest.mark.parametrize('npx', [4096, 4097, 4098, 4099])
@pytest.mark.parametrize('offsets', [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (3, 2, 1), (2, 2, 2)])
def test_gather_of_misaligned_views(eng, k, npx, offsets):
    """label map, segm and segm_soft as views `offsets` elements into their buffers (16-byte alignment lost for any nonzero offset
    except an even one of segm_soft)"""
    import torch
    from pyimsegm_b200 import _lib
    o_seg, o_i, o_p = offsets
    rng = np.random.RandomState(npx * 10 + k)
    nb = 97
    seg = rng.randint(0, nb, npx).astype(np.int32)
    lut_i = rng.randint(-2 ** 31, 2 ** 31 - 1, nb).astype(np.int32)
    lut_p = rng.rand(nb, k)
    d_seg = torch.zeros(npx + 8, dtype=torch.int32, device='cuda')
    d_seg[o_seg:o_seg + npx] = torch.from_numpy(seg).cuda()
    d_lut_i, d_lut_p = eng.to_device(lut_i), eng.to_device(lut_p)
    out_i = torch.full((npx + 8, ), CANARY_I, dtype=torch.int32, device='cuda')
    out_p = torch.full(((npx + 8) * k, ), CANARY_P, dtype=torch.float64, device='cuda')
    v_seg, v_i, v_p = d_seg[o_seg:], out_i[o_i:], out_p[o_p:]
    lib = _lib.lib()
    _lib.check(lib.isb_gather(_lib.ptr(v_seg), C.c_longlong(npx), _lib.ptr(d_lut_i), _lib.ptr(d_lut_p), k, _lib.ptr(v_i), _lib.ptr(v_p),
                              _lib.stream_ptr()))
    got_i, got_p = eng.to_host(out_i), eng.to_host(out_p)
    np.testing.assert_array_equal(got_i[o_i:o_i + npx], lut_i[seg])
    assert np.all(got_i[:o_i] == CANARY_I) and np.all(got_i[o_i + npx:] == CANARY_I)
    np.testing.assert_array_equal(got_p[o_p:o_p + npx * k].view(np.int64), lut_p[seg].ravel().view(np.int64))
    assert np.all(got_p[:o_p] == CANARY_P) and np.all(got_p[o_p + npx * k:] == CANARY_P)
