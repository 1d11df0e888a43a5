"""
torchrun entry of tests/test_gpu_tiled.py::test_two_ranks_nccl (and of a run over N GPUs): one process per GPU, one band (or two)
per process, NCCL between them.  Every rank checks its own rows against the oracle; rank 0 prints TILED-RANKS-OK.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def main():
    import torch
    import torch.distributed as dist
    from conftest import synth_regions
    import oracle as orc
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import GroupComm, pipe_color2d_slic_features_model_graphcut_tiled, slic_tiled
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
    dist.init_process_group('nccl')
    comm = GroupComm()
    orc.build()
    eng = get_engine()
    for shape, sp_size, regul, slico, bpr in (((512, 384), 20, 0.2, False, 1), ((397, 263), 17, 0.25, False, 2), ((360, 300), 15, 0.2, True, 1)):
        img = synth_regions(shape[0], shape[1], seed=31)[0]
        want = orc.segment_slic_img2d(img, sp_size, regul, slico)
        n_seg, compact = slic_params(img.shape[:2], sp_size, regul)
        res = slic_tiled(img, n_seg, compact, slic_zero=slico, comm=comm, bands_per_rank=bpr, eng=eng)
        assert not res.fell_back
        assert np.array_equal(eng.to_host(res.d_seg), want), 'rank %d: label map differs %r' % (comm.rank, shape)
    # whole pipeline: every rank's rows against the oracle pipeline given the same class probabilities is covered on one GPU;
    # here the banded result must equal the single-GPU pipeline run by this rank on the whole image
    from pyimsegm_b200 import pipelines as pl
    img = synth_regions(768, 512, seed=32)[0]
    segm, soft = pl.pipe_color2d_slic_features_model_graphcut(img, 3, {'color': ['mean']}, sp_size=20, sp_regul=0.2)
    got, got_soft, (lo, hi) = pipe_color2d_slic_features_model_graphcut_tiled(img, 3, {'color': ['mean']}, sp_size=20, sp_regul=0.2, comm=comm)
    assert hi - lo == 768 // comm.world or comm.rank == comm.world - 1
    assert np.array_equal(got, segm[lo:hi]), 'rank %d: segmentation differs' % comm.rank
    np.testing.assert_allclose(got_soft, soft[lo:hi], rtol=1e-6, atol=1e-9)
    full, _, _ = pipe_color2d_slic_features_model_graphcut_tiled(img, 3, {'color': ['mean']}, sp_size=20, sp_regul=0.2, comm=comm,
                                                                want_soft=False, gather_segm=True)
    assert np.array_equal(full, segm)
    # Leung-Malik statistics over the bands (each rank: its rows + 616 rows of halo; sums and response norms all-reduced) against the
    # whole-image descriptor this rank computes on its own GPU
    from pyimsegm_b200.texture import device_lm_features
    from pyimsegm_b200.tiled import LM_ROW_MARGIN, texture_stats_tiled
    img = synth_regions(2600, 160, seed=33)[0] + 0.05 * np.random.RandomState(3).standard_normal((2600, 160, 3))
    n_seg, compact = slic_params(img.shape[:2], 24, 0.2)
    res = slic_tiled(img, n_seg, compact, comm=comm, eng=eng, raw_margin=LM_ROW_MARGIN)
    flags = ('mean', 'std', 'energy')
    got = eng.to_host(texture_stats_tiled(res, img.dtype, flags, 'short', comm=comm, eng=eng)).copy()
    want = eng.to_host(device_lm_features(eng, eng.to_device(img, 'image'), res.d_seg, int(res.nb_bound), flags, 'short')[0]).copy()
    np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-9)
    ok = torch.ones(1, device='cuda')
    dist.all_reduce(ok)
    if comm.rank == 0 and int(ok.item()) == comm.world:
        print('TILED-RANKS-OK world=%d' % comm.world)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
