"""
torchrun entry of tests/test_gpu_tiled_volume.py::test_two_ranks_nccl_volume (and of a run over N GPUs): one process per GPU, one
z-slab (or two) per process, NCCL between them.  Every rank checks the label volume against the oracle and its slices of the
pipelines against the single-GPU volume path; rank 0 prints TILED-VOLUME-RANKS-OK.
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
    import oracle as orc
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic3d_params
    from pyimsegm_b200.tiled import (GroupComm, gray_stats_tiled, pipe_gray3d_slic_features_model_graphcut_tiled, slic3d_tiled)
    from test_gpu_tiled_volume import FEATURES, _as, _blobs
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
    dist.init_process_group('nccl')
    comm = GroupComm()
    orc.build()
    eng = get_engine()
    for shape, dtype, spacing, sp_size, regul, bpr in (((30, 60, 52), np.uint8, (12, 1, 1), 10, 0.3, 1),
                                                       ((27, 40, 30), np.float32, (1, 1, 1), 7, 0.25, 2)):
        vol = _as(_blobs(shape, 41), dtype)
        n_seg, compact = slic3d_params(shape, sp_size, regul, spacing)
        want = orc.slic3d(vol, n_seg, compact, spacing)
        res = slic3d_tiled(vol, n_seg, compact, spacing, comm=comm, bands_per_rank=bpr, eng=eng)
        assert not res.fell_back
        assert np.array_equal(eng.to_host(res.d_seg), want), 'rank %d: label volume differs %r' % (comm.rank, shape)
        flags = ('mean', 'std', 'energy')
        got = eng.to_host(gray_stats_tiled(res, vol.dtype, flags, comm=comm, eng=eng)).copy()
        ref = eng.to_host(eng.gray_table(eng.to_device(vol, 'volume_check'), res.d_seg, int(res.nb_bound), list(flags))).copy()
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    vol = _as(_blobs((20, 60, 52), 42), np.uint8)
    hosts, done = eng.download(pl.segment_resident_volume(eng.to_device(vol, 'volume_check'), pl._fit_model(2, True), FEATURES, (2, 1, 1),
                                                          10, 0.3, 0.1))
    done.synchronize()
    segm, soft = (h.numpy() for h in hosts)
    got, got_soft, (lo, hi) = pipe_gray3d_slic_features_model_graphcut_tiled(vol, 2, FEATURES, (2, 1, 1), 10, 0.3, 0.1, comm=comm)
    assert np.array_equal(got, segm[lo:hi]), 'rank %d: segmentation differs' % comm.rank
    np.testing.assert_allclose(got_soft, soft[lo:hi], rtol=1e-9, atol=1e-9)
    full, _, _ = pipe_gray3d_slic_features_model_graphcut_tiled(vol, 2, FEATURES, (2, 1, 1), 10, 0.3, 0.1, comm=comm, want_soft=False,
                                                                gather_segm=True)
    assert np.array_equal(full, segm)
    ok = torch.ones(1, device='cuda')
    dist.all_reduce(ok)
    if comm.rank == 0 and int(ok.item()) == comm.world:
        print('TILED-VOLUME-RANKS-OK world=%d' % comm.world)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
