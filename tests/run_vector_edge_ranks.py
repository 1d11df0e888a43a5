"""
torchrun entry of tests/test_gpu_vector_edge_weights.py::test_ranks_agree_on_vector_edge_cuts: the banded 2-D pipelines with
gc_edge_type 'color' and 'features' over two or more processes.  Backend from argv[1]: 'nccl' with one GPU per process, 'gloo' when
the processes share a GPU (the collectives then run through gloo on the same device tensors).  Every rank checks the whole label
map against segment_resident on its own GPU and that every rank holds the same map; rank 0 prints VECTOR-EDGE-RANKS-OK.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def main(backend):
    import torch
    import torch.distributed as dist
    from sklearn.ensemble import RandomForestClassifier

    from conftest import synth_regions
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.tiled import GroupComm, pipe_color2d_slic_features_model_graphcut_tiled, segment_color2d_slic_features_model_graphcut_tiled
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)) % torch.cuda.device_count())
    dist.init_process_group(backend)
    comm = GroupComm()
    eng = get_engine()
    feats = {'color': ['mean', 'std']}
    base = synth_regions(320, 224, seed=51)[0]
    above = base.copy()
    above[-3, 5, 1] = 1.5        # the one sample above 1 lies in the last rank's rows: the others learn it from the all-reduce
    images = {'float_max_in_last_band': above, 'u8': (base * 255).astype(np.uint8)}
    checked = 0
    for name, img in images.items():
        _, features = pl.compute_color2d_superpixels_features(img, feats, sp_size=12, sp_regul=0.2)
        y = np.argsort(np.argsort(features[:, 1])) * 3 // len(features)
        forest = RandomForestClassifier(n_estimators=10, max_depth=6, random_state=0).fit(features, y)
        d_img = eng.to_device(img, 'ranks_img')
        for edge_type in ('color', 'features'):
            want_gmm = eng.to_host(pl.segment_resident(d_img, pl._fit_model(3, True), feats, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                       gc_edge_type=edge_type)[0]).copy()
            want_forest = eng.to_host(pl.segment_resident(d_img, forest, feats, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                          gc_edge_type=edge_type)[0]).copy()
            for bands in (1, 2):
                for what, want, run in (
                        ('gmm', want_gmm, lambda: pipe_color2d_slic_features_model_graphcut_tiled(
                            img, 3, feats, sp_size=12, sp_regul=0.2, gc_regul=2., gc_edge_type=edge_type, comm=comm, bands_per_rank=bands,
                            want_soft=False, gather_segm=True)),
                        ('forest', want_forest, lambda: segment_color2d_slic_features_model_graphcut_tiled(
                            img, forest, feats, sp_size=12, sp_regul=0.2, gc_regul=2., gc_edge_type=edge_type, comm=comm,
                            bands_per_rank=bands, want_soft=False, gather_segm=True))):
                    segm = run()[0]
                    where = 'rank %d, %s, %s, %s, %d bands per rank' % (comm.rank, name, edge_type, what, bands)
                    assert np.array_equal(segm, want), where + ': labels differ from segment_resident'
                    # every rank holds the same map: its elementwise min and max over the ranks are the map itself
                    d = torch.from_numpy(np.ascontiguousarray(segm, dtype=np.int64)).cuda()
                    lo, hi = d.clone(), d.clone()
                    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
                    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
                    assert torch.equal(lo, d) and torch.equal(hi, d), where + ': the ranks hold different labels'
                    checked += 1
    ok = torch.ones(1, device='cuda')
    dist.all_reduce(ok)
    if comm.rank == 0 and int(ok.item()) == comm.world:
        print('VECTOR-EDGE-RANKS-OK world=%d backend=%s cases=%d' % (comm.world, backend, checked))
    dist.destroy_process_group()


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else 'nccl')
