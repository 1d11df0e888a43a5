"""
The per-tile candidate lists of the SLIC sweeps (slic_kmeans.cu): every cluster whose centre is set appends its record to the tiles
its window meets, and the assignment reads its tile's list.  The raw k-means label map must be bit-identical to the oracle for
superpixel sizes whose lists take one round, several rounds (longer than a round) and overflowed lists (every cluster scanned),
for SLICO, for the ordinary-load path of odd widths and for the row-band mode with several bands on one GPU.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import synth_regions

pytestmark = pytest.mark.gpu


def _lab_and_segments(oracle, img, sp_size, regul):
    """the Lab image and cluster count that segment_slic_img2d hands to the k-means sweeps"""
    n_seg = int(img.shape[0] * img.shape[1] / sp_size ** 2)
    compact = (sp_size * regul) ** 1.5
    return oracle.rgb2lab_scaled(oracle.gaussian_blur(img, 1.0), 1.0 / compact), n_seg


def _device_kmeans(oracle, lab, n_seg, slic_zero):
    import torch
    from pyimsegm_b200 import _lib
    H, W, _ = lab.shape
    seeds, ty, tx = oracle.slic_seeds(H, W, n_seg)
    n = len(seeds)
    lib = _lib.lib()
    d_lab = torch.from_numpy(np.ascontiguousarray(lab.transpose(2, 0, 1))).cuda()
    d_seeds = torch.from_numpy(seeds).cuda()
    wsb = lib.isb_slic_kmeans_workspace_bytes(H, W, n, int(ty), int(tx))
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    labels = torch.empty((H, W), dtype=torch.int32, device='cuda')
    _lib.check(lib.isb_slic_kmeans(_lib.ptr(d_lab), H, W, _lib.ptr(d_seeds), n, int(ty), int(tx), C.c_double(float(max(1, ty, tx))),
                                   10, int(slic_zero), _lib.ptr(labels), None, _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return labels.cpu().numpy()


def _check(oracle, shape, sp_size, regul, slico=False, seed=0):
    img = synth_regions(shape[0], shape[1], seed=seed)[0]
    lab, n_seg = _lab_and_segments(oracle, img, sp_size, regul)
    got = _device_kmeans(oracle, lab, n_seg, slico)
    want = oracle.slic_kmeans(lab, n_seg, slic_zero=slico)
    assert np.array_equal(got, want)


@pytest.mark.parametrize('regul', [0.1, 0.4])
@pytest.mark.parametrize('sp_size', [29, 10, 5, 3])
def test_tile_lists_bit_exact(oracle, sp_size, regul):
    # sp_size 3: about 200 clusters meet a tile, more than one round of the assignment stages
    _check(oracle, (320, 384), sp_size, regul, seed=sp_size)


@pytest.mark.parametrize('sp_size', [29, 10])
def test_tile_lists_slico(oracle, sp_size):
    _check(oracle, (256, 320), sp_size, 0.2, slico=True, seed=40 + sp_size)


@pytest.mark.parametrize('sp_size', [29, 7])
def test_tile_lists_odd_width(oracle, sp_size):
    # an odd width has no tensor map: the tile's Lab values are staged by ordinary loads
    _check(oracle, (250, 317), sp_size, 0.2, seed=50 + sp_size)


@pytest.mark.parametrize('cap', [1, 12])
def test_overflowed_tiles_scan_every_cluster(oracle, cap):
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    before = lib.isb_slic_full_scan_tiles()
    prev = lib.isb_slic_set_tile_cap(cap)
    try:
        _check(oracle, (256, 288), 10, 0.2, seed=60 + cap)
        _check(oracle, (256, 288), 10, 0.2, slico=True, seed=61 + cap)
    finally:
        lib.isb_slic_set_tile_cap(prev)
    assert lib.isb_slic_full_scan_tiles() > before, 'no tile overflowed'


@pytest.mark.parametrize('n_bands', [2, 3])
@pytest.mark.parametrize('slico', [False, True])
def test_banded_tile_lists(oracle, n_bands, slico):
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import slic_tiled
    eng = get_engine()
    img, sp_size, regul = synth_regions(420, 330, seed=70 + n_bands)[0], 15, 0.2
    want = oracle.segment_slic_img2d(img, sp_size, regul, slico=slico)
    n_seg, compact = slic_params(img.shape[:2], sp_size, regul)
    res = slic_tiled(img, n_seg, compact, bands_per_rank=n_bands, slic_zero=slico, eng=eng)
    assert not res.fell_back
    assert np.array_equal(eng.to_host(res.d_seg), want)
