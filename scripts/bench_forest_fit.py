#!/usr/bin/env python
"""
bench_forest_fit.py -- the fit of the reference's default classifier, RandomForestClassifier(n_estimators=20, min_samples_leaf=2,
min_samples_split=3), on the device (forest_fit.fit_tree_model, csrc/forest_fit.cu) against scikit-learn's fit on the host.  Prints
one JSON line.

    python scripts/bench_forest_fit.py [--steps 5] [--warmup 1]

The data: the labelled superpixels of 8 config-2 images (bench.synth_image with the Voronoi class map of
scripts/bench_shared_model.synth_classes as the annotation, SLIC as bench.py, label purity 0.9), balanced per image by
convert_set_features_labels_2_dataset(balance_type='random'), with colour mean / std / energy (D = 9) and with colour + full
Leung-Malik statistics (D = 189).  Per feature set:
- the device fit: median / min / max over --steps of the wall time (numpy in, fitted estimator out) and of CUDA events around it;
- scikit-learn's fit with n_jobs=-1 and with n_jobs=1 (one run each), and os.cpu_count();
- the accuracy of both forests on the labelled superpixels of 4 other images;
- the levels the device built, and the share of the device's kernel time spent in radix sorts (torch.profiler, a separate run);
- the card's name, power limit and maximum SM clock (nvidia-smi), read in the same run.
There is no CPU fallback: without a CUDA device the script fails.
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_shared_model import card_info, synth_classes  # noqa: E402

FEATURE_SETS = {
    'd9': {'color': ('mean', 'std', 'energy')},
    'd189': {'color': ('mean', 'std', 'energy'), 'tLM': ('mean', 'std', 'energy')},
}
FOREST = dict(n_estimators=20, min_samples_leaf=2, min_samples_split=3)


def stats(ts):
    return {'median': round(float(np.median(ts)), 4), 'min': round(float(np.min(ts)), 4), 'max': round(float(np.max(ts)), 4)}


def image_sets(seeds, features):
    from pyimsegm_b200 import pipelines
    d_fts, d_lbs = {}, {}
    for s in seeds:
        _, fts, lbs = pipelines.wrapper_compute_color2d_slic_features_labels((bench.synth_image(s), synth_classes(s)), bench.SP_SIZE,
                                                                             bench.SP_REGUL, features, 0.9)
        d_fts['%03d' % s], d_lbs['%03d' % s] = np.asarray(fts), np.asarray(lbs)
    return d_fts, d_lbs


def run(steps, warmup):
    import torch
    from sklearn.ensemble import RandomForestClassifier
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    from pyimsegm_b200 import classification as clf
    from pyimsegm_b200 import forest_fit
    levels = []
    device_fit = forest_fit._fit_arrays

    def counting(*args):
        trees = device_fit(*args)
        levels.append(trees[0]['n_levels'])
        return trees
    forest_fit._fit_arrays = counting
    out = {'metric': 'forest_fit', 'cpu_count': os.cpu_count(), 'card': card_info(), 'sets': {}}
    for name, feats in FEATURE_SETS.items():
        random.seed(0)
        X, y, _ = clf.convert_set_features_labels_2_dataset(*image_sets(range(8), feats), drop_labels=[-1], balance_type='random')
        Xh, yh, _ = clf.convert_set_features_labels_2_dataset(*image_sets(range(100, 104), feats), drop_labels=[-1])
        X32 = X.astype(np.float32)
        wall, events = [], []
        for i in range(warmup + steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.record()
            dev = forest_fit.fit_tree_model(RandomForestClassifier(random_state=i, **FOREST), X32, y)
            b.record()
            torch.cuda.synchronize()
            if i >= warmup:
                wall.append(time.perf_counter() - t0)
                events.append(a.elapsed_time(b) / 1e3)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            forest_fit.fit_tree_model(RandomForestClassifier(random_state=0, **FOREST), X32, y)
            torch.cuda.synchronize()
        kern = [(e.key, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0]
        total = sum(t for _, t in kern)
        sort = sum(t for n, t in kern if 'RadixSort' in n or 'Onesweep' in n)
        host = {}
        for jobs in (-1, 1):
            t0 = time.perf_counter()
            ref = RandomForestClassifier(random_state=0, n_jobs=jobs, **FOREST).fit(X32, y)
            host['n_jobs=%d' % jobs] = round(time.perf_counter() - t0, 3)
        out['sets'][name] = {
            'rows': int(len(X)), 'features': int(X.shape[1]), 'classes': int(len(np.unique(y))), 'held_out_rows': int(len(Xh)),
            'device_fit_wall_s': stats(wall), 'device_fit_events_s': stats(events), 'host_fit_s': host,
            'speedup_vs_n_jobs_-1': round(host['n_jobs=-1'] / float(np.median(wall)), 2),
            'held_out_accuracy': {'device': round(float(np.mean(dev.predict(Xh.astype(np.float32)) == yh)), 4),
                                  'scikit-learn': round(float(np.mean(ref.predict(Xh.astype(np.float32)) == yh)), 4)},
            'levels': int(levels[-1]), 'sort_share_of_kernel_time': round(sort / total, 3) if total else None,
            'kernel_time_s': round(total / 1e6, 4),
        }
    forest_fit._fit_arrays = device_fit
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))


if __name__ == '__main__':
    main()
