"""
The SLIC centroid update (k_update in slic_kmeans.cu) over member boxes of every size: one strip of chunks, a few strips, and
boxes of tens of thousands of members that take dozens of strips.  The raw k-means label map and the centroids after the last
sweep must be bit-identical to the oracle's raster-order sequential sums; the banded path (k_update<true>) is checked on large
superpixels with bands thinner than the halo.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import synth_disc, synth_regions

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


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
    cent = torch.empty((n, 5), dtype=torch.float64, device='cuda')
    _lib.check(lib.isb_slic_kmeans(_lib.ptr(d_lab), H, W, _lib.ptr(d_seeds), n, int(ty), int(tx), C.c_double(float(max(1, ty, tx))),
                                   10, int(slic_zero), _lib.ptr(labels), _lib.ptr(cent), _lib.ptr(ws), C.c_size_t(wsb),
                                   _lib.stream_ptr()))
    torch.cuda.synchronize()
    return labels.cpu().numpy(), cent.cpu().numpy()


@pytest.mark.parametrize('case', ['huge_boxes', 'huge_boxes_slico', 'headline_size', 'one_strip', 'flat'])
def test_kmeans_labels_and_centroids_bit_exact(oracle, case):
    slico = False
    if case == 'huge_boxes':           # 18 clusters of ~23 000 members: dozens of strips per cluster
        img, sp_size, regul = synth_regions(600, 700, seed=31)[0], 150, 0.2
    elif case == 'huge_boxes_slico':
        img, sp_size, regul, slico = synth_regions(480, 560, seed=32)[0], 120, 0.2, True
    elif case == 'headline_size':      # the superpixel size of the benchmark: two to four strips per cluster
        img, sp_size, regul = synth_regions(512, 512, seed=33)[0], 29, 0.2
    elif case == 'one_strip':          # every box fits in one strip: the buffers are never refilled
        img, sp_size, regul = synth_regions(200, 230, seed=34, cell=16)[0], 5, 0.3
    else:                              # flat regions tie everywhere: any change in the last bit of a sum shows
        img, sp_size, regul = synth_disc(400, 360, noise=0.0), 60, 0.3
    lab, n_seg = _lab_and_segments(oracle, img, sp_size, regul)
    got, got_c = _device_kmeans(oracle, lab, n_seg, slico)
    want, want_c = oracle.slic_kmeans(lab, n_seg, slic_zero=slico, return_centroids=True)
    assert np.array_equal(got, want)
    # the centroids of the clusters that hold pixels after the last sweep (the last update summed exactly those)
    alive = np.unique(want)
    assert np.array_equal(got_c[alive].view(np.int64), want_c[alive].view(np.int64))


@pytest.mark.parametrize('sp_size,shape', [(150, (600, 700)), (90, (450, 380))])
def test_slic_large_superpixels_bit_exact(oracle, sp_size, shape):
    from pyimsegm_b200 import superpixels as sp
    img, _ = synth_regions(shape[0], shape[1], seed=sp_size)
    assert np.array_equal(sp.segment_slic_img2d(img, sp_size, 0.2), oracle.segment_slic_img2d(img, sp_size, 0.2))


def test_banded_large_superpixels_thin_bands(oracle, eng):
    """k_update<true> on boxes of thousands of members, with bands thinner than the halo"""
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import slic_tiled
    img, sp_size, regul = synth_regions(600, 400, seed=35)[0], 60, 0.2
    want = oracle.segment_slic_img2d(img, sp_size, regul)
    n_seg, compact = slic_params(img.shape[:2], sp_size, regul)
    for n_bands in (3, 7):
        res = slic_tiled(img, n_seg, compact, bands_per_rank=n_bands, eng=eng)
        assert not res.fell_back
        assert np.array_equal(eng.to_host(res.d_seg), want), 'bands=%d' % n_bands
