"""The single-CTA integer prefix sums (csrc/block_scan.cuh) at the seams between their 1 024-element rounds, through the kernels that
use them: the median's label offsets (``k_med_scan``), the graph cut's CSR offsets (``k_gc_build_csr``), the mask compaction's tile
offsets (``k_compact_scan``, 4 096 pixels a tile) and the kept-piece ranks of volume connectivity (``c3_rank``).  Every result is
compared exactly with numpy or the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_alpha_expansion import check, integer_problem, random_graph
from test_gpu_segment_statistics import _check_median, _image, _labels_of_sizes

pytestmark = pytest.mark.gpu

ROUND = 1024
CPT_TILE = 4096   # pixels of a compaction tile: CPT_TILE of pyimsegm_b200/csrc/compact.cuh
SEAMS = (ROUND - 1, ROUND, ROUND + 1, 2 * ROUND + 1)


@pytest.mark.parametrize('nb', SEAMS)
def test_median_label_counts_across_scan_rounds(nb):
    rng = np.random.RandomState(nb)
    sizes = rng.randint(0, 6, nb)
    sizes[[0, ROUND // 2]] = 0                                  # absent labels -> NaN
    sizes[-1] = 3                                               # the last label sets nb
    seg = _labels_of_sizes(sizes, rng)
    _check_median(_image((len(seg), 3), 'float64', rng), seg, 3, 'nb %d' % nb)
    _check_median(_image((len(seg), 1), 'uint8', rng), seg, 1, 'nb %d gray' % nb)


@pytest.mark.parametrize('n', SEAMS)
def test_graph_cut_node_counts_across_scan_rounds(oracle, n):
    rng = np.random.RandomState(n)
    edges = random_graph(rng, n)
    w, un, pw = integer_problem(oracle, rng, edges, n, 3)
    check(oracle, edges, w, un, pw)


@pytest.mark.parametrize('n', (ROUND * CPT_TILE - 1, ROUND * CPT_TILE, ROUND * CPT_TILE + 1, 2 * ROUND * CPT_TILE + 1))
def test_mask_compaction_tile_counts_across_scan_rounds(n):
    from pyimsegm_b200 import labeling
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    rng = np.random.RandomState(n % 1000)
    mask = (rng.rand(1, n) < 0.3).astype(np.uint8)
    mask[0, -1] = 1                                             # a set pixel in the last tile
    values = rng.rand(1, n)
    points, got = labeling._compact(eng, eng.to_device(mask, 'scan_mask'), mask.shape, eng.to_device(values, 'scan_values'))
    np.testing.assert_array_equal(points, np.argwhere(mask))
    np.testing.assert_array_equal(got, values[mask.astype(bool)])


@pytest.mark.parametrize('shape', ((1, 1, ROUND - 1), (1, 1, ROUND), (1, 1, ROUND + 1), (2, 32, 32), (1, 3, 683), (3, 41, 50)),
                         ids=lambda s: 'x'.join(map(str, s)))
def test_volume_connectivity_voxel_counts_across_scan_rounds(oracle, shape):
    """runs of one to three voxels of random labels: many pieces, kept (min_size 2) and merged ones on both sides of every seam"""
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    D, H, W = shape
    rng = np.random.RandomState(D * H * W)
    runs = rng.randint(1, 4, D * H * W)
    seg = np.repeat(rng.randint(0, 5, len(runs)), runs)[:D * H * W].reshape(shape).astype(np.int64)
    for min_size, max_size in ((1, 100000), (2, 100000)):
        want = np.empty_like(seg)
        n = oracle.lib().oracle_enforce_connectivity3d(seg.ctypes.data_as(C.POINTER(C.c_int64)), D, H, W, C.c_long(min_size),
                                                       C.c_long(max_size), want.ctypes.data_as(C.POINTER(C.c_int64)))
        d_in = eng.to_device(seg.astype(np.int32), 'scan_conn_in')
        out = eng.buf('scan_conn_out', shape, eng.torch.int32)
        nl = eng.buf('scan_conn_n', (1,), eng.torch.int32)
        wsb = eng.lib.isb_connectivity3d_workspace_bytes(D, H, W, max_size)
        ws = eng.buf('scan_conn_ws', (wsb,), eng.torch.uint8)
        _lib.check(eng.lib.isb_enforce_connectivity3d(_lib.ptr(d_in), D, H, W, min_size, max_size, _lib.ptr(out), _lib.ptr(nl),
                                                      _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
        assert np.array_equal(eng.to_host(out), want), (shape, min_size)
        assert int(eng.to_host(nl)[0]) == max(n, 1)
