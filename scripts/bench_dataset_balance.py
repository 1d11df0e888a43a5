#!/usr/bin/env python
"""
bench_dataset_balance.py -- balance_dataset_by_(..., balance_type='kmeans') of imsegm.classification on the device against the host
reference path (scikit-learn KMeans, as the reference calls it).  Prints one JSON line.

    python scripts/bench_dataset_balance.py [--images 8] [--steps 3] [--warmup 1] [--host-max-rows 12000]

The data: the superpixel features and labels of several config-2 images (bench.synth_image with the Voronoi class map of
scripts/bench_shared_model.synth_classes as the annotation, SLIC as bench.py, label purity 0.9, unlabelled superpixels dropped), with
colour mean / std / energy (D = 9) and with colour + full Leung-Malik statistics (D = 189).  The classes are imbalanced, so k (the
smallest class) is in the thousands.  Per feature set:
- the device call end to end (numpy in, numpy out; host clock, the call ends in a host read), median / min / max over --steps;
- one Lloyd run alone (CUDA events around isb_kmeans_lloyd on buffers already on the device) and one assignment alone (the same call
  started from the status of a stopped run: the fused tensor-core assignment plus the inertia sum), with FP64 TFLOP/s by 2 n k D
  per sweep;
- the host reference path (np.argmin(KMeans(k, init='random', n_init=3, max_iter=5).fit_transform(X), axis=0) for every larger
  class) on the first image alone when its rows are at most --host-max-rows, with the device call on the same rows, and for the same
  np.random.seed the number of centres whose kept rows differ and whether each such pair is a rounding tie (oracle/dataset.py
  selection_ties: two rows at the same true distance from a centre, which scikit-learn's expansion and the device's exact
  differences tell apart by rounding only) -- ``parity``;
- the card's name and power limit (nvidia-smi), read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_shared_model import card_info, synth_classes  # noqa: E402
from oracle import dataset as od  # noqa: E402

FEATURE_SETS = {
    'd9': {'color': ('mean', 'std', 'energy')},
    'd189': {'color': ('mean', 'std', 'energy'), 'tLM': ('mean', 'std', 'energy')},
}


def stats(ts):
    return {'median': round(float(np.median(ts)), 4), 'min': round(float(np.min(ts)), 4), 'max': round(float(np.max(ts)), 4)}


def image_rows(seeds, features):
    """[(features, labels)] of the labelled superpixels of every image"""
    from pyimsegm_b200 import pipelines
    out = []
    for s in seeds:
        _, fts, labels = pipelines.wrapper_compute_color2d_slic_features_labels((bench.synth_image(s), synth_classes(s)), bench.SP_SIZE,
                                                                                bench.SP_REGUL, features, 0.9)
        keep = labels >= 0
        out.append((np.asarray(fts)[keep], np.asarray(labels)[keep]))
    return out


def host_reference(X, y, seed):
    """the rows the reference's balance_dataset_by_(X, y, 'kmeans') keeps, through scikit-learn on the host: (rows per class, seconds)"""
    from sklearn.cluster import KMeans
    np.random.seed(seed)
    uq, counts = np.unique(y, return_counts=True)
    k = counts.min()
    rows = {}
    t0 = time.perf_counter()
    for lb in uq:
        idx = np.where(y == lb)[0]
        if len(idx) <= k:
            rows[int(lb)] = idx
            continue
        dist = KMeans(n_clusters=k, init='random', n_init=3, max_iter=5).fit_transform(X[idx])
        rows[int(lb)] = idx[np.argmin(dist, axis=0)]
    return rows, time.perf_counter() - t0


def device_rows(X, y, seed):
    """the same rows through pyimsegm_b200.classification._kmeans_sample (what balance_dataset_by_ calls): (rows per class, seconds)"""
    from pyimsegm_b200 import classification as clf
    np.random.seed(seed)
    uq, counts = np.unique(y, return_counts=True)
    k = counts.min()
    rows, centres = {}, {}
    t0 = time.perf_counter()
    for lb in uq:
        idx = np.where(y == lb)[0]
        if len(idx) <= k:
            rows[int(lb)] = idx
            continue
        sel, _, best = clf._kmeans_sample(X[idx], k)
        rows[int(lb)], centres[int(lb)] = idx[sel], best.centres + X[idx].mean(axis=0)
    return rows, centres, time.perf_counter() - t0


def lloyd_alone(X, k, steps):
    """CUDA-event times of one Lloyd run (5 sweeps at most) and of one assignment on device buffers; sweeps done"""
    import torch
    from pyimsegm_b200 import _lib
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    lib, st = eng.lib, _lib.stream_ptr()
    n, D = X.shape
    Xc = X - X.mean(axis=0)
    tol = float(np.mean(np.var(X, axis=0)) * 1e-4)
    c0 = Xc[np.random.RandomState(0).choice(n, k, replace=False)]
    d_x = eng.to_device(Xc)
    d_c = torch.empty((k, D), dtype=torch.float64, device=eng.device)
    labels = torch.empty(n, dtype=torch.int32, device=eng.device)
    status = torch.empty(4, dtype=torch.int32, device=eng.device)
    sums = torch.empty((k, D), dtype=torch.float64, device=eng.device)
    counts = torch.empty(k, dtype=torch.int32, device=eng.device)
    inertia = torch.empty(1, dtype=torch.float64, device=eng.device)
    ws_bytes = lib.isb_kmeans_workspace_bytes(n, k, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=eng.device)
    c0_dev = torch.from_numpy(c0).to(eng.device)
    out = {}
    for name, st0 in (('run', 0), ('assign', 2)):
        ts, sweeps, code = [], 0, 0
        for _ in range(steps + 1):
            d_c.copy_(c0_dev)
            labels.fill_(-1)
            status.copy_(torch.tensor([st0, 0, 0, 0], dtype=torch.int32))
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            sweeps_enqueued = 5 if st0 == 0 else 0
            _lib.check(lib.isb_kmeans_lloyd(_lib.ptr(d_x), n, D, k, 5, sweeps_enqueued, C.c_double(tol), _lib.ptr(d_c), _lib.ptr(labels),
                                            _lib.ptr(status), _lib.ptr(sums), _lib.ptr(counts), _lib.ptr(inertia), _lib.ptr(ws),
                                            C.c_size_t(ws_bytes), st))
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
            sweeps, code = int(status[1].item()), int(status[0].item())
        ms = float(np.median(ts[1:]))
        # the sweeps, and the final E-step when the run stopped without strict convergence (status 2 or 4)
        passes = sweeps + (code in (2, 4)) if name == 'run' else 1
        out[name] = {'ms': stats(ts[1:]), 'assign_passes': passes, 'fp64_tflops': round(2.0 * n * k * D * passes / (ms * 1e-3) / 1e12, 2)}
        if name == 'run':
            out[name]['sweeps'] = sweeps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=8)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--host-max-rows', type=int, default=12000)
    ap.add_argument('--sets', default='d9,d189')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    from pyimsegm_b200 import classification as clf
    warnings.simplefilter('ignore')
    seeds = [6000 + i for i in range(args.images)]
    result = {'card': card_info(), 'images': args.images, 'sets': {}}
    for set_name in args.sets.split(','):
        per_image = image_rows(seeds, FEATURE_SETS[set_name])
        X = np.concatenate([f for f, _ in per_image])
        y = np.concatenate([lb for _, lb in per_image])
        uq, counts = np.unique(y, return_counts=True)
        k = int(counts.min())
        entry = {'rows': int(len(X)), 'D': int(X.shape[1]), 'class_rows': counts.tolist(), 'k': k}
        ts = []
        for i in range(args.warmup + args.steps):
            np.random.seed(i)
            t0 = time.perf_counter()
            clf.balance_dataset_by_(X, y, balance_type='kmeans')
            ts.append(time.perf_counter() - t0)
        entry['device_balance_s'] = stats(ts[args.warmup:])
        big = counts.argmax()
        entry['lloyd_largest_class'] = dict(lloyd_alone(X[y == uq[big]], k, args.steps), n=int(counts[big]))
        X1, y1 = per_image[0]
        if len(X1) <= args.host_max_rows:
            host, t_host = host_reference(X1, y1, 7)
            dev, centres, t_dev = device_rows(X1, y1, 7)
            ties = [od.selection_ties(X1[y1 == c], centres[c], np.searchsorted(np.where(y1 == c)[0], dev[c]),
                                      np.searchsorted(np.where(y1 == c)[0], host[c])) for c in centres]
            entry['first_image'] = {'rows': int(len(X1)), 'k': int(np.unique(y1, return_counts=True)[1].min()), 'host_s': round(t_host, 3),
                                    'device_s': round(t_dev, 3), 'selected_rows_differing': int(sum(t[0] for t in ties)),
                                    'same_rows_up_to_rounding_ties': all(t[1] for t in ties)}
        result['sets'][set_name] = entry
    result['parity'] = all(e['first_image']['same_rows_up_to_rounding_ties'] for e in result['sets'].values() if 'first_image' in e)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
