"""
The volume SLIC (csrc/slic3d.cu) stage by stage at the shapes, spacings and label layouts where it can go wrong, every result
compared exactly with oracle/slic3d_oracle.c or scipy.ndimage:
  A. the connectivity pass alone (``isb_enforce_connectivity3d``) on constructed label volumes -- oversize components whose
     truncated BFS leaves orphan voxels behind (the "brush"), min_size > max_size, one-voxel pieces, merge chains, degenerate
     shapes, labels near 2**30 -- with a sentinel tail after the workspace it is given, which must come back untouched;
  B. the k-means sweeps alone: one seed per voxel, one seed in all, a collapsed seed axis, strong and weak z spacing, flat
     ties, uint16, float64 outside [0, 1] and clusters that lose every voxel;
  C. the pre-blur alone (``isb_slic3d_prepare``) against scipy's gaussian_filter: axes shorter than the blur radius, a radius
     of 0 and of 16, the four input dtypes;
  D. the whole of ``Engine.slic3d`` with max_size_factor < 1, so that ordinary blob-shaped supervoxels are split;
  E. (host) the brush volumes are the ones that overran the BFS queue when the split reserved max_size entries per piece instead
     of per component, so that A keeps reaching that case.
"""
import ctypes as C

import numpy as np
import pytest
from scipy import ndimage

gpu = pytest.mark.gpu

SENTINEL = 0xA5
TAIL = 64 << 10
# (shape, min_size, max_size) of the brush volumes: their truncated BFS leaves many orphan pieces
BRUSHES = (((3, 40, 40), 1, 40), ((5, 48, 48), 1, 60), ((3, 64, 64), 2, 300))


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _blobs(shape, seed, noise=0.08):
    rng = np.random.RandomState(seed)
    zz, yy, xx = np.mgrid[:shape[0], :shape[1], :shape[2]]
    vol = 0.3 + 0.4 * ((xx > shape[2] // 2) ^ (yy > shape[1] // 3)) + 0.15 * (zz > shape[0] // 2)
    return np.clip(vol + rng.normal(0, noise, shape), 0, 1)


def brush(D, H, W):
    """label 0: the plane z = D // 2 and, in the planes right above and below it, the bristles where (z + y + x) is even;
    label 1 everywhere else"""
    zz, yy, xx = np.mgrid[:D, :H, :W]
    seg = np.ones((D, H, W), dtype=np.int64)
    seg[(zz == D // 2) | ((np.abs(zz - D // 2) == 1) & ((zz + yy + xx) % 2 == 0))] = 0
    return seg


def split_pieces(seg, max_size):
    """the pieces of the connectivity pass before any merge: every 6-connected component of one label, cut by the truncated BFS
    (at most max_size voxels, neighbours x+1, x-1, y+1, y-1, z+1, z-1) started at each of its unassigned voxels in raster order.
    Returns the head (first voxel) of each voxel's piece and the number of pieces cut from components of >= max_size voxels."""
    D, H, W = seg.shape
    V = seg.size
    comp = np.empty(V, dtype=np.int64)
    n_comp = 0
    for value in np.unique(seg):
        lab, n = ndimage.label(seg == value, ndimage.generate_binary_structure(3, 1))
        m = lab.ravel() > 0
        comp[m] = lab.ravel()[m] - 1 + n_comp
        n_comp += n
    comp_size = np.bincount(comp)
    piece = np.full(V, -1, dtype=np.int64)
    steps = ((1, lambda z, y, x: x + 1 < W), (-1, lambda z, y, x: x > 0), (W, lambda z, y, x: y + 1 < H),
             (-W, lambda z, y, x: y > 0), (H * W, lambda z, y, x: z + 1 < D), (-H * W, lambda z, y, x: z > 0))
    n_split = 0
    for head in range(V):
        if piece[head] >= 0:
            continue
        c = comp[head]
        piece[head] = head
        q, visited = [head], 0
        while visited < len(q) and len(q) < max_size:
            u = q[visited]
            z, y, x = u // (H * W), (u // W) % H, u % W
            for off, inside in steps:
                n = u + off
                if inside(z, y, x) and comp[n] == c and piece[n] < 0:
                    piece[n] = head
                    q.append(n)
                    if len(q) >= max_size:
                        break
            visited += 1
        n_split += comp_size[c] >= max_size
    return piece, n_split


def oracle_connectivity(oracle, seg, min_size, max_size):
    seg = np.ascontiguousarray(seg, dtype=np.int64)
    want = np.empty_like(seg)
    n = oracle.lib().oracle_enforce_connectivity3d(seg.ctypes.data_as(C.POINTER(C.c_int64)), *seg.shape, C.c_long(min_size),
                                                   C.c_long(max_size), want.ctypes.data_as(C.POINTER(C.c_int64)))
    assert n >= 0
    return want, int(n)


def check_connectivity(oracle, eng, seg, min_size, max_size):
    """isb_enforce_connectivity3d against the oracle, bit for bit, in a workspace followed by TAIL sentinel bytes"""
    from pyimsegm_b200 import _lib
    torch = eng.torch
    want, n = oracle_connectivity(oracle, seg, min_size, max_size)
    D, H, W = seg.shape
    d_in = torch.from_numpy(np.ascontiguousarray(seg, dtype=np.int32)).to(eng.device)
    out = torch.full((D, H, W), -7, dtype=torch.int32, device=eng.device)
    nl = torch.full((1, ), -7, dtype=torch.int32, device=eng.device)
    wsb = eng.lib.isb_connectivity3d_workspace_bytes(D, H, W, max_size)
    ws = torch.full((wsb + TAIL, ), SENTINEL, dtype=torch.uint8, device=eng.device)
    _lib.check(eng.lib.isb_enforce_connectivity3d(_lib.ptr(d_in), D, H, W, min_size, max_size, _lib.ptr(out), _lib.ptr(nl),
                                                  _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
    tail = ws[wsb:].cpu().numpy()
    assert (tail == SENTINEL).all(), 'workspace overrun: %d bytes after its end written' % (tail != SENTINEL).sum()
    np.testing.assert_array_equal(out.cpu().numpy(), want, err_msg='shape %s min %d max %d' % (seg.shape, min_size, max_size))
    assert int(nl.cpu()[0]) == max(n, 1)
    return want


# ---------------------------------------------------------------------------------------------------------------------
# A. connectivity pass
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('shape,min_size,max_size', BRUSHES, ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_connectivity_brush_orphan_pieces(oracle, eng, shape, min_size, max_size):
    check_connectivity(oracle, eng, brush(*shape), min_size, max_size)


@gpu
@pytest.mark.parametrize('min_size,max_size', ((3, 10), (1, 5), (12, 6), (30, 8), (8, 8), (0, 7), (1, 100000), (0, 100000)))
def test_connectivity_two_labels(oracle, eng, min_size, max_size):
    """random two-label volume; min_size > max_size makes every piece small: nothing is kept, every voxel gets label 0"""
    seg = (np.random.RandomState(min_size * 100 + max_size % 97).rand(6, 20, 24) < 0.45).astype(np.int64)
    out = check_connectivity(oracle, eng, seg, min_size, max_size)
    if min_size > max_size:
        assert not out.any()


@gpu
@pytest.mark.parametrize('min_size', (0, 1, 2))
def test_connectivity_one_voxel_pieces(oracle, eng, min_size):
    """max_size 1: every voxel is a piece of its own"""
    seg = np.random.RandomState(11).randint(0, 3, (4, 9, 13))
    out = check_connectivity(oracle, eng, seg, min_size, 1)
    if min_size <= 1:
        np.testing.assert_array_equal(out.ravel(), np.arange(seg.size))


@gpu
@pytest.mark.parametrize('min_size,max_size', ((1, 100000), (1, 50), (50, 64), (2000, 100000), (0, 1)))
def test_connectivity_one_label(oracle, eng, min_size, max_size):
    check_connectivity(oracle, eng, np.full((7, 9, 11), 3), min_size, max_size)


@gpu
@pytest.mark.parametrize('min_size', (0, 1, 2))
def test_connectivity_every_voxel_distinct(oracle, eng, min_size):
    seg = np.random.RandomState(12).permutation(6 * 10 * 14).reshape(6, 10, 14)
    check_connectivity(oracle, eng, seg, min_size, 10)


@gpu
@pytest.mark.parametrize('max_size', (10, 100000))
def test_connectivity_checkerboard_merge_chains(oracle, eng, max_size):
    """every checkerboard voxel is a one-voxel piece merging into an earlier one: chains as long as the volume is deep, ending
    in one of three solid boxes (split in pieces of 10 when max_size is 10) or in the default label 0"""
    zz, yy, xx = np.mgrid[:9, :10, :12]
    seg = (zz + yy + xx) % 2
    seg[0:2, 0:3, 0:4] = 5
    seg[5:9, 6:10, 8:12] = 6
    seg[2:4, 4:7, 0:3] = 7
    out = check_connectivity(oracle, eng, seg, 2, max_size)
    assert len(np.unique(out)) > 1


@gpu
def test_connectivity_small_piece_takes_last_earlier_neighbour(oracle, eng):
    """a two-voxel piece (label 4) whose BFS meets kept pieces at x-1 (label 3), y-1 (label 2) and z-1 (label 1), in that order:
    it merges into the last of them, the plane z = 0 (new label 1, after the three voxels of label 9 in its corner)"""
    seg = np.full((3, 4, 4), 5)
    seg[0] = 1
    seg[0, 0, :3] = 9
    seg[1:, 0, :] = 2
    seg[1:, 1:, 0] = 3
    seg[1, 1, 1:3] = 4
    out = check_connectivity(oracle, eng, seg, 3, 1000)
    assert out[1, 1, 1] == out[1, 1, 2] == out[0, 1, 1] == 1
    assert len({out[0, 1, 1], out[1, 0, 1], out[1, 1, 0]}) == 3


@gpu
@pytest.mark.parametrize('shape', ((1, 1, 37), (37, 1, 1), (1, 11, 13), (1, 1, 1), (2, 1, 1), (5, 1, 7)), ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('min_size,max_size', ((0, 100000), (2, 100000), (2, 5), (3, 1)))
def test_connectivity_degenerate_shapes(oracle, eng, shape, min_size, max_size):
    """single rows and columns along each axis, one plane, and volumes of one and two voxels (fewer voxels than the pass's
    counters, which its first kernel must still clear)"""
    rng = np.random.RandomState(sum(shape))
    runs = rng.randint(1, 4, int(np.prod(shape)))
    seg = np.repeat(rng.randint(0, 3, len(runs)), runs)[:int(np.prod(shape))].reshape(shape)
    check_connectivity(oracle, eng, seg, min_size, max_size)


@gpu
@pytest.mark.parametrize('min_size,max_size', ((2, 100000), (4, 9)))
def test_connectivity_sparse_large_label_values(oracle, eng, min_size, max_size):
    values = np.array([2 ** 30 - 1, 2 ** 30 + 1, 2 ** 30 + 77, 2 ** 30 - 2 ** 20, 2 ** 30], dtype=np.int64)
    rng = np.random.RandomState(13)
    coarse = rng.randint(0, len(values), (3, 6, 6))
    seg = values[np.kron(coarse, np.ones((2, 3, 3), dtype=np.int64))]
    flip = rng.rand(*seg.shape) < 0.1
    seg[flip] = values[rng.randint(0, len(values), flip.sum())]
    check_connectivity(oracle, eng, seg, min_size, max_size)


# ---------------------------------------------------------------------------------------------------------------------
# B. k-means sweeps
# ---------------------------------------------------------------------------------------------------------------------

def _kmeans_case(case):
    """(volume, n_segments, compactness, spacing)"""
    rng = np.random.RandomState(len(case))
    if case == 'seed_per_voxel':
        return rng.rand(4, 6, 5), 120, 0.5, (1, 1, 1)
    if case == 'more_segments_than_voxels':
        return rng.rand(3, 5, 7), 1000, 2.0, (2, 1, 1)
    if case == 'one_segment':
        return _blobs((6, 20, 24), 21), 1, 0.3, (1, 1, 1)
    if case == 'collapsed_axis':      # D = 2 is shorter than the step: regular_grid spreads the seeds over y and x
        return _blobs((2, 60, 60), 22, noise=0.15), 20, 0.2, (1, 1, 1)
    if case == 'spacing_12':           # z blur radius 0
        return _blobs((5, 40, 50), 23), 30, 0.2, (12, 1, 1)
    if case == 'spacing_quarter':      # z blur radius 16, longer than the axis
        return _blobs((12, 20, 20), 24), 20, 0.3, (0.25, 1, 1)
    if case == 'flat':                 # every colour distance ties, and many spatial ones: the lowest cluster index wins
        return np.full((6, 24, 24), 0.5), 16, 0.1, (1, 1, 1)
    if case == 'uint16':
        return (_blobs((8, 30, 34), 25) * 65535).astype(np.uint16), 24, 0.25, (2, 1, 1)
    if case == 'f64_wide':             # values far outside [0, 1], negatives included
        return _blobs((7, 26, 30), 26, noise=0.2) * 100 - 40, 18, 30.0, (1, 1, 1)
    assert case == 'dead_clusters'     # the seeds of column x = 11 straddle the step: their mean matches no voxel and they die
    xx = np.mgrid[:8, :32, :32][2]
    return (xx >= 12).astype(np.float64), 16, 0.1, (1, 1, 4)


KMEANS_CASES = ('seed_per_voxel', 'more_segments_than_voxels', 'one_segment', 'collapsed_axis', 'spacing_12', 'spacing_quarter',
                'flat', 'uint16', 'f64_wide', 'dead_clusters')


@gpu
@pytest.mark.parametrize('case', KMEANS_CASES)
def test_kmeans_sweeps_bit_exact(oracle, eng, case):
    vol, n_seg, compact, spacing = _kmeans_case(case)
    km, _ = eng.slic3d(eng.to_device(vol, 'edges_vol3d'), n_seg, compact, spacing, enforce_connectivity=False)
    got = eng.to_host(km).copy()
    want = oracle.slic3d(vol, n_seg, compact, spacing, return_kmeans=True)
    n_seeds = len(oracle.slic_seeds3d(vol.shape, n_seg)[0])
    if case in ('seed_per_voxel', 'more_segments_than_voxels'):
        assert n_seeds == vol.size
    if case == 'one_segment':
        assert n_seeds == 1 and not want.any()
    if case == 'dead_clusters':
        assert len(np.unique(want)) < n_seeds
    np.testing.assert_array_equal(got, want, err_msg=case)


# ---------------------------------------------------------------------------------------------------------------------
# C. pre-blur
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('dtype', ('uint8', 'uint16', 'float32', 'float64'))
@pytest.mark.parametrize('shape,spacing', (((1, 20, 30), (1, 1, 1)), ((2, 17, 9), (1, 1, 1)), ((5, 30, 40), (12, 1, 1)),
                                           ((12, 16, 18), (0.25, 1, 1)), ((6, 1, 3), (1, 1, 1)), ((4, 3, 50), (1, 2, 0.5))),
                         ids=('D1', 'D2', 'z_radius0', 'z_radius16', 'H1', 'short_y'))
def test_prepare_matches_scipy_gaussian_filter(eng, dtype, shape, spacing):
    """the blurred, 1 / compactness scaled volume against scipy.ndimage.gaussian_filter in float64 of the img_as_float volume"""
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.engine import gaussian_half_kernel
    torch = eng.torch
    rng = np.random.RandomState(shape[0] * 7 + len(dtype))
    if dtype == 'uint8':
        vol = rng.randint(0, 256, shape).astype(np.uint8)
        as_float = vol / 255.0
    elif dtype == 'uint16':
        vol = rng.randint(0, 65536, shape).astype(np.uint16)
        as_float = vol / 65535.0
    else:
        vol = (rng.rand(*shape) * 3 - 1).astype(dtype)
        as_float = vol.astype(np.float64)
    compactness, sigma = 0.3, 1.0
    sigmas = sigma / np.asarray(spacing, dtype=np.float64)
    want = ndimage.gaussian_filter(as_float, sigmas, mode='reflect', truncate=4.0) * (1.0 / compactness)
    halves = [gaussian_half_kernel(s) for s in sigmas]
    d_w = [torch.from_numpy(w).to(eng.device) for w, _ in halves]
    d_vol = torch.from_numpy(vol).to(eng.device)
    tmp = torch.empty(shape, dtype=torch.float64, device=eng.device)
    out = torch.full(shape, np.nan, dtype=torch.float64, device=eng.device)
    _lib.check(eng.lib.isb_slic3d_prepare(_lib.ptr(d_vol), _lib.dtype_code(vol.dtype), *shape, _lib.ptr(d_w[0]), halves[0][1],
                                          _lib.ptr(d_w[1]), halves[1][1], _lib.ptr(d_w[2]), halves[2][1], C.c_double(1.0 / compactness),
                                          _lib.ptr(tmp), _lib.ptr(out), _lib.stream_ptr()))
    np.testing.assert_array_equal(out.cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------------------------
# D. oversize splits of real supervoxels
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('shape,n_seg,compact,spacing', (((64, 256, 256), 2000, 5.0, (1, 1, 1)), ((12, 160, 192), 150, 2.0, (5, 1, 1))),
                         ids=('64x256x256', 'aniso'))
def test_slic3d_splits_supervoxels(oracle, eng, shape, n_seg, compact, spacing):
    """max_size_factor 0.6 and 0.3 cut ordinary supervoxels; with min_size_factor 0.5, 0.3 makes every piece small"""
    vol = _blobs(shape, 31, noise=0.1)
    km = oracle.slic3d(vol, n_seg, compact, spacing, return_kmeans=True)
    component_sizes = np.bincount(oracle_connectivity(oracle, km, 0, km.size + 1)[0].ravel())
    segment_size = vol.size / n_seg
    d_vol = eng.to_device(vol, 'edges_vol3d')
    for min_factor, max_factor in ((0.5, 0.6), (0.1, 0.3), (0.5, 0.3)):
        min_size, max_size = int(min_factor * segment_size), int(max_factor * segment_size)
        assert (component_sizes >= max_size).sum() >= 10
        want, n = oracle_connectivity(oracle, km, min_size, max_size)
        labels, n_labels = eng.slic3d(d_vol, n_seg, compact, spacing, min_size_factor=min_factor, max_size_factor=max_factor)
        np.testing.assert_array_equal(eng.to_host(labels), want, err_msg='factors %s %s' % (min_factor, max_factor))
        assert int(eng.to_host(n_labels)[0]) == max(n, 1)


# ---------------------------------------------------------------------------------------------------------------------
# E. (host) what the brush volumes reach
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('shape,min_size,max_size', BRUSHES, ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_brush_overruns_a_queue_reserved_per_piece(oracle, shape, min_size, max_size):
    """Replays the queue reservations of the split when it reserved max_size entries for every piece it cut (orphan voxels left
    by a truncated BFS become pieces of their own) followed by the small pieces' replay (psize entries each): the total overran
    the 3 V + max_size + 64 entries the queue then had.  One queue of max_size entries per oversize component fits in V, and so
    do the small pieces."""
    seg = brush(*shape)
    V = seg.size
    piece, n_split = split_pieces(seg, max_size)
    # the replay's pieces are the oracle's: with min_size 0 every piece is kept, labelled by the raster rank of its head
    np.testing.assert_array_equal(np.unique(piece, return_inverse=True)[1], oracle_connectivity(oracle, seg, 0, max_size)[0].ravel())
    psize = np.bincount(piece, minlength=V)
    small = psize[(psize > 0) & (psize < min_size)].sum()
    assert n_split * max_size + small > 3 * V + max_size + 64
    n_big = sum(1 for value in np.unique(seg)
                for size in np.bincount(ndimage.label(seg == value, ndimage.generate_binary_structure(3, 1))[0].ravel())[1:]
                if size >= max_size)
    assert n_big * max_size <= V and small <= V
