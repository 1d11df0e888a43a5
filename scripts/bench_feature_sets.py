#!/usr/bin/env python
"""
bench_feature_sets.py -- the feature sets the reference's users run (median, meanGrad, colour-space groups) on the resident device
path against the general path and the numpy API.  Prints one JSON line.

    python scripts/bench_feature_sets.py --steps K --warmup W [--texture]

Image: one config-2 image (bench.synth_image: 2048x2048 RGB f64, sp_size 29).  Feature sets: the unsupervised tutorial's
{'color': mean, std, median}, the region-growing notebook's {'color': mean, median}, {'color': all five}, and
{'color_hsv': mean, std, energy; 'color_lab': mean, median}; with --texture also {'tLM_short': mean, meanGrad} and
descriptors.FEATURES_SET_ALL (colour and tLM with all five statistics).  Legs, alternating within every step:
  pipe_resident / pipe_general   pipe_color2d_slic_features_model_graphcut (self-fitted GMM), resident vs. debug_visual={} -- the
                                 general path through the numpy-facing stages (which also fills the small debug_visual arrays; its
                                 features come from compute_color2d_superpixels_features, so from the resident feature table too)
  features_resident / features_numpy  compute_color2d_superpixels_features vs. segment_slic_img2d + compute_selected_features_img2d
                                       -- the numpy API on the label map SLIC gave (the same device feature driver, with one
                                       upload of the image and of the labels and one download of the table)
Parity: max |features resident - numpy API| per set on the same superpixels, and segm equality of the two pipeline paths under
one caller-fitted StandardScaler + GaussianMixture.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402  (the workload constants and image generator of the headline benchmark)
from bench_shared_model import card_info  # noqa: E402

SETS = {
    'tutorial': {'color': ['mean', 'std', 'median']},
    'rg2sp': {'color': ['mean', 'median']},
    'color_all': {'color': ['mean', 'std', 'energy', 'median', 'meanGrad']},
    'hsv_lab': {'color_hsv': ('mean', 'std', 'energy'), 'color_lab': ('mean', 'median')},
}
TEXTURE_SETS = {
    'tlm_short_meangrad': {'tLM_short': ('mean', 'meanGrad')},
    'features_set_all': {'color': ('mean', 'std', 'energy', 'median', 'meanGrad'), 'tLM': ('mean', 'std', 'energy', 'median', 'meanGrad')},
}


def run(steps, warmup, texture):
    import torch
    from sklearn import mixture, pipeline, preprocessing
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    torch.cuda.set_device(bench.dist_env()[2])
    from pyimsegm_b200 import _lib, pipelines
    from pyimsegm_b200.descriptors import compute_selected_features_img2d
    from pyimsegm_b200.superpixels import segment_slic_img2d
    lib = _lib.lib()
    SP, REG, GC, K = bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL, bench.NB_CLASSES
    img = torch.from_numpy(bench.synth_image(6100)).pin_memory().numpy()
    sets = dict(SETS, **(TEXTURE_SETS if texture else {}))

    def legs_of(feats):
        return [('pipe_resident', lambda: pipelines.pipe_color2d_slic_features_model_graphcut(img, K, feats, SP, REG, gc_regul=GC)),
                ('pipe_general', lambda: pipelines.pipe_color2d_slic_features_model_graphcut(img, K, feats, SP, REG, gc_regul=GC,
                                                                                               debug_visual={})),
                ('features_resident', lambda: pipelines.compute_color2d_superpixels_features(img, feats, SP, REG)),
                ('features_numpy', lambda: compute_selected_features_img2d(img, segment_slic_img2d(img, sp_size=SP, relative_compact=REG),
                                                                           feats))]

    nstage = lib.isb_profile_stage_count()
    stage_ids = {lib.isb_profile_stage_name(i).decode(): i for i in range(nstage)}
    result = {}
    for set_name, feats in sets.items():
        legs = legs_of(feats)
        for _, fn in legs:               # warm every leg: buffers sized, graphs captured
            for _ in range(warmup):
                fn()
        # parity: features on the same superpixels, and one caller-fitted model through both pipeline paths
        slic, fts = pipelines.compute_color2d_superpixels_features(img, feats, SP, REG)
        api_fts, _ = compute_selected_features_img2d(img, slic, feats)
        model = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                   ('model', mixture.GaussianMixture(K, covariance_type='full', random_state=0))]).fit(api_fts)
        seg_res, _ = pipelines.segment_color2d_slic_features_model_graphcut(img, model, feats, SP, REG, GC)
        seg_gen, _ = pipelines.segment_color2d_slic_features_model_graphcut(img, model, feats, SP, REG, GC, debug_visual={})
        parity = {'features_max_abs_diff': float(np.max(np.abs(fts - api_fts))), 'n_features': int(fts.shape[1]),
                  'shared_model_segm_identical': bool(np.array_equal(seg_res, seg_gen))}
        del seg_res, seg_gen, fts, api_fts
        per_step = {name: [] for name, _ in legs}
        for _ in range(steps):           # the legs alternate inside every step (the host shares the machine with other work)
            for name, fn in legs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                per_step[name].append((time.perf_counter() - t0) * 1e3)
                del out
        legs_out = {}
        for name, fn in legs:            # device stage timers: a separate untimed pass with eager launches
            pipelines.USE_CUDA_GRAPHS = False
            lib.isb_profile_enable(1)
            fn()
            ms_arr, cnt_arr = (C.c_double * nstage)(), (C.c_longlong * nstage)()
            lib.isb_profile_collect(ms_arr, cnt_arr)
            lib.isb_profile_enable(0)
            pipelines.USE_CUDA_GRAPHS = True
            legs_out[name] = {'ms_per_image': float(np.median(per_step[name])),
                              'ms_per_image_min_max': [min(per_step[name]), max(per_step[name])],
                              'segment_stats_stage_ms': ms_arr[stage_ids['segment_stats']], 'lm_stage_ms': ms_arr[stage_ids['lm_texture']]}
        result[set_name] = {'features': {k: list(v) for k, v in feats.items()}, 'legs': legs_out, 'parity': parity,
                            'speedup_pipe': legs_out['pipe_general']['ms_per_image'] / legs_out['pipe_resident']['ms_per_image'],
                            'speedup_features': legs_out['features_numpy']['ms_per_image'] / legs_out['features_resident']['ms_per_image']}
    return {'metric': 'ms per image, feature sets with median / meanGrad / colour spaces: resident path vs general path and numpy API',
            'unit': 'ms', 'n_gpus': 1, 'steps': steps, 'warmup': warmup, 'higher_is_better': False, 'dtype': 'f64', 'data': 'synthetic',
            'config': {'workload': 'one config-2 image (%dx%d RGB f64), SLIC sp_size=%d, %d-class GMM, GraphCut gc_regul %g'
                                   % (bench.H, bench.W, SP, K, GC),
                       'timed': 'host clock around each call with a device synchronise on both sides; legs alternate within a step; '
                                'ms_per_image = median over the steps; pipe_general also builds the debug_visual arrays'},
            'sets': result, 'card': card_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--texture', action='store_true', help='also the Leung-Malik sets with median / meanGrad')
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup, args.texture)))


if __name__ == '__main__':
    main()
