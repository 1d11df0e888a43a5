#!/usr/bin/env python
"""
bench_edge_types.py -- the GraphCut edge weights 'color' and 'features' on the resident device path against the general path
that pipe_color2d_slic_features_model_graphcut takes for them.  Prints one JSON line.

    python scripts/bench_edge_types.py --steps K --warmup W

Image: the headline benchmark's (bench.synth_image: 2048x2048 RGB f64, sp_size 29, colour means, 3-class GMM fitted on the
device).  Legs, alternating within every step, milliseconds per image (host clock around a call that ends in a device
synchronise; the resident legs download the label map, as a caller would):
  resident_model / resident_color / resident_features   segment_resident with gc_edge_type 'model' / 'color' / 'features'
  general_color / general_features                      pipe_color2d_slic_features_model_graphcut with 'color' / 'features'
                                                        (label map down, edges and weights on the host, graph up)
Parity: the label maps of the resident and the general legs per edge type.
"""
import argparse
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


def run(steps, warmup):
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    torch.cuda.set_device(bench.dist_env()[2])
    from pyimsegm_b200 import pipelines
    from pyimsegm_b200.engine import get_engine
    SP, REG, GC, K, FEATS = bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL, bench.NB_CLASSES, bench.FEATURES
    eng = get_engine()
    img = bench.synth_image(7100)
    d_img = eng.to_device(img, 'bench_edge_img')
    model = pipelines._fit_model(K, True)

    def resident(edge_type):
        def call():
            d_segm, _ = pipelines.segment_resident(d_img, model, FEATS, sp_size=SP, sp_regul=REG, gc_regul=GC, gc_edge_type=edge_type)
            return eng.to_host(d_segm).copy()
        return call

    def general(edge_type):
        def call():
            return pipelines.pipe_color2d_slic_features_model_graphcut(img, K, FEATS, sp_size=SP, sp_regul=REG, gc_regul=GC,
                                                                       gc_edge_type=edge_type)[0]
        return call

    legs = {'resident_model': resident('model'), 'resident_color': resident('color'), 'resident_features': resident('features'),
            'general_color': general('color'), 'general_features': general('features')}
    last = {}
    for _ in range(warmup):
        for name, fn in legs.items():
            last[name] = fn()
    times = {name: [] for name in legs}
    for _ in range(steps):
        for name, fn in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last[name] = fn()
            times[name].append((time.perf_counter() - t0) * 1e3)
    ms = {name: round(float(np.median(t)), 2) for name, t in times.items()}
    return {
        'metric': 'ms_per_image', 'median_ms': ms,
        'spread_ms': {name: [round(float(min(t)), 2), round(float(max(t)), 2)] for name, t in times.items()},
        'speedup_resident_vs_general': {t: round(ms['general_' + t] / ms['resident_' + t], 2) for t in ('color', 'features')},
        'labels_identical': {t: bool(np.array_equal(last['resident_' + t], last['general_' + t])) for t in ('color', 'features')},
        'config': {'image': '%dx%d RGB f64 (bench.synth_image)' % img.shape[:2], 'sp_size': SP, 'sp_regul': REG, 'gc_regul': GC,
                   'nb_classes': K, 'features': FEATS, 'steps': steps, 'warmup': warmup},
        'card': card_info(),
    }


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))
