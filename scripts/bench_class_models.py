#!/usr/bin/env python
"""
bench_class_models.py -- the class model variants of the reference (estim_model, pca_coef) fitted on the device against scikit-learn
on the host.  Prints one JSON line.

    python scripts/bench_class_models.py --steps K --warmup W

Legs, alternating within every step:
  * pipe_color2d_slic_features_model_graphcut on config-2 images (bench.synth_image: 2048x2048 RGB f64, sp_size 29, colour means)
    per variant (GMM, kmeans, BGM, GMM + pca_coef 0.95), with the device fit and with graph_cuts.USE_DEVICE_GMM = False;
  * the fit alone (estim_class_model) at D = 189, N = 5000, K = 4 on seeded synthetic features: BGM and PCA(0.95) + GMM.
Parity fields: the label maps of the device and host legs agree (up to a permutation of the classes) on most pixels -- the two
fits start from different k-means draws, so they are compared by agreement, not equality.
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

import bench  # noqa: E402
from scripts.bench_shared_model import card_info  # noqa: E402

PIPE_VARIANTS = [('GMM', None), ('kmeans', None), ('BGM', None), ('GMM', 0.95)]
FIT_VARIANTS = [('BGM', None), ('GMM', 0.95)]


def _agreement(a, b, K):
    """fraction of pixels on which two label maps agree under the best matching of their classes"""
    import itertools
    best = 0.0
    for perm in itertools.permutations(range(K)):
        best = max(best, float(np.mean(np.asarray(perm)[a] == b)))
    return best


def run(steps, warmup):
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    torch.cuda.set_device(bench.dist_env()[2])
    from pyimsegm_b200 import _lib, graph_cuts, pipelines
    lib = _lib.lib()
    F, SP, REG, GC, K = bench.FEATURES, bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL, bench.NB_CLASSES
    image = torch.from_numpy(bench.synth_image(7000)).pin_memory().numpy()
    rng = np.random.RandomState(189)
    centres = rng.uniform(0, 1, (4, 189))
    feats = centres[rng.randint(0, 4, 5000)] + rng.normal(0, 0.15, (5000, 189))

    def on(device, fn):
        graph_cuts.USE_DEVICE_GMM = device
        try:
            return fn()
        finally:
            graph_cuts.USE_DEVICE_GMM = True

    legs = []
    for v, p in PIPE_VARIANTS:
        name = 'pipe_%s%s' % (v, '' if p is None else '_pca%g' % p)
        for dev in (True, False):
            legs.append(('%s_%s' % (name, 'device' if dev else 'host'), name, dev,
                         (lambda v=v, p=p, dev=dev: on(dev, lambda: pipelines.pipe_color2d_slic_features_model_graphcut(
                             image, K, F, SP, REG, p, True, v, GC, 'model')))))
    for v, p in FIT_VARIANTS:
        name = 'fit189_%s%s' % (v, '' if p is None else '_pca%g' % p)
        for dev in (True, False):
            legs.append(('%s_%s' % (name, 'device' if dev else 'host'), name, dev,
                         (lambda v=v, p=p, dev=dev: on(dev, lambda: graph_cuts.estim_class_model(feats, 4, v, p)))))
    outs = {}
    for name, _, _, fn in legs:
        for _ in range(max(warmup, 1)):
            outs[name] = fn()
    parity = {}
    for name, group, dev, _ in legs:
        if not dev:
            continue
        d, h = outs[name], outs[group + '_host']
        if group.startswith('pipe'):
            parity[group + '_label_agreement'] = _agreement(d[0], h[0], K)
        else:
            ld, lh = d.predict_proba(feats).argmax(1), h.predict_proba(feats).argmax(1)
            parity[group + '_label_agreement'] = _agreement(ld, lh, 4)
            parity[group + '_lower_bound'] = [float(d.steps[-1][1].lower_bound_), float(h.steps[-1][1].lower_bound_)]
            if p_ := dict(d.steps).get('reduce_dim'):
                parity[group + '_n_components'] = [int(p_.n_components_), int(dict(h.steps)['reduce_dim'].n_components_)]
    outs = None
    per_step = {name: [] for name, _, _, _ in legs}
    for _ in range(steps):
        for name, _, _, fn in legs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            per_step[name].append((time.perf_counter() - t0) * 1e3)
            del out
    # class-model stage time (device timers, one untimed pass with eager launches)
    nstage = lib.isb_profile_stage_count()
    stage = [i for i in range(nstage) if lib.isb_profile_stage_name(i).decode() == 'gmm'][0]
    gmm_stage = {}
    pipelines.USE_CUDA_GRAPHS = False
    for name, _, dev, fn in legs:
        if not dev:
            continue
        lib.isb_profile_enable(1)
        fn()
        ms_arr, cnt_arr = (C.c_double * nstage)(), (C.c_longlong * nstage)()
        lib.isb_profile_collect(ms_arr, cnt_arr)
        lib.isb_profile_enable(0)
        gmm_stage[name] = ms_arr[stage]
    pipelines.USE_CUDA_GRAPHS = True
    result = {}
    for name, _, dev, _ in legs:
        result[name] = {'ms': float(np.median(per_step[name])), 'ms_min_max': [min(per_step[name]), max(per_step[name])]}
        if dev:
            result[name]['gmm_stage_ms'] = gmm_stage[name]
    return {'metric': 'ms per call, class model variants fitted on the device vs scikit-learn', 'unit': 'ms', 'n_gpus': 1,
            'steps': steps, 'warmup': max(warmup, 1), 'higher_is_better': False, 'dtype': 'f64', 'data': 'synthetic',
            'config': {'pipe': 'pipe_color2d_slic_features_model_graphcut on one config-2 image (2048x2048 RGB f64, sp_size %d, '
                               'colour means, gc_regul %g, %d classes)' % (SP, GC, K),
                       'fit189': 'estim_class_model on seeded features N=5000, D=189, K=4',
                       'timed': 'host clock around each call with a device synchronise on both sides; legs alternate within a step; '
                                'ms = median over the steps; *_host legs run with graph_cuts.USE_DEVICE_GMM = False'},
            'legs': result, 'parity': parity, 'card': card_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))


if __name__ == '__main__':
    main()
