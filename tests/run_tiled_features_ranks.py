"""
torchrun entry of tests/test_gpu_tiled_features.py::test_two_ranks_nccl_features (and of a run over N GPUs): one process per GPU,
NCCL between them.  Every rank checks the banded colour-space statistics, the banded texture meanGrad and a caller-fitted model's
segmentation against what it computes on the whole image on its own GPU; rank 0 prints TILED-FEATURES-RANKS-OK.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def _close_per_column(got, want, rel, what):
    scale = np.maximum(np.abs(want).max(axis=0), 1e-300)
    err = (np.abs(got - want) / scale).max()
    assert err <= rel, '%s: off by %.3g of a column maximum' % (what, err)


def main():
    import torch
    import torch.distributed as dist
    from conftest import synth_regions
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.descriptors import device_feature_table, native_feature_layout
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.texture import device_lm_materialised
    from pyimsegm_b200.tiled import (GroupComm, banded_raw_margin, features_tiled, segment_color2d_slic_features_model_graphcut_tiled,
                                     slic_tiled)
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
    dist.init_process_group('nccl')
    comm = GroupComm()
    eng = get_engine()
    # colour spaces with meanGrad, one and two bands per rank
    fts = {k: ('mean', 'std', 'energy', 'meanGrad') for k in ('color', 'color_hsv', 'color_luv', 'color_lab', 'color_hed', 'color_xyz')}
    layout, ncol = native_feature_layout(fts)
    img = synth_regions(397, 263, seed=61)[0].astype(np.float32)
    n_seg, compact = slic_params(img.shape[:2], 17, 0.25)
    for bpr in (1, 2):
        res = slic_tiled(img, n_seg, compact, comm=comm, bands_per_rank=bpr, eng=eng)
        got = eng.to_host(features_tiled(res, img.dtype, 3, layout, ncol, comm=comm, eng=eng)[0]).copy()
        want = eng.buf('feat_whole', (int(res.nb_bound), ncol), torch.float64)
        device_feature_table(eng, eng.to_device(img, 'image'), res.d_seg, int(res.nb_bound), fts, want)
        _close_per_column(got, eng.to_host(want).copy(), 1e-12, 'rank %d colour spaces, %d bands per rank' % (comm.rank, bpr))
    # texture meanGrad: the response norms summed over the ranks
    img = synth_regions(2600, 160, seed=33)[0] + 0.05 * np.random.RandomState(3).standard_normal((2600, 160, 3))
    fts = {'tLM_short': ('meanGrad', )}
    layout, ncol = native_feature_layout(fts)
    n_seg, compact = slic_params(img.shape[:2], 24, 0.2)
    res = slic_tiled(img, n_seg, compact, comm=comm, eng=eng, raw_margin=banded_raw_margin(layout))
    got = eng.to_host(features_tiled(res, img.dtype, 3, layout, ncol, comm=comm, eng=eng)[0]).copy()
    want = eng.buf('feat_whole', (int(res.nb_bound), ncol), torch.float64)
    device_lm_materialised(eng, eng.to_device(img, 'image'), res.d_seg, int(res.nb_bound), ['meanGrad'], 'short', want, 0)
    _close_per_column(got, eng.to_host(want).copy(), 1e-9, 'rank %d texture meanGrad' % comm.rank)
    # a caller-fitted group model
    fts = {'color': ('mean', 'meanGrad'), 'color_hsv': ('mean', 'std')}
    model, _ = pl.estim_model_classes_group([synth_regions(384, 320, seed=s)[0] for s in (51, 52)], 3, fts, sp_size=20, sp_regul=0.2)
    img = synth_regions(768, 448, seed=53)[0]
    segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, model, fts, sp_size=20, sp_regul=0.2)
    got, got_soft, (lo, hi) = segment_color2d_slic_features_model_graphcut_tiled(img, model, fts, sp_size=20, sp_regul=0.2, comm=comm)
    assert np.array_equal(got, segm[lo:hi]), 'rank %d: segmentation differs' % comm.rank
    np.testing.assert_allclose(got_soft, soft[lo:hi], rtol=0, atol=1e-9)
    ok = torch.ones(1, device='cuda')
    dist.all_reduce(ok)
    if comm.rank == 0 and int(ok.item()) == comm.world:
        print('TILED-FEATURES-RANKS-OK world=%d' % comm.world)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
