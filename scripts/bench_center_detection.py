#!/usr/bin/env python
"""
bench_center_detection.py -- object-centre detection of the reference's ovary experiment (experiments_ovary_centres) on
bench.synth_eggs_image-style images of 1024 x 1280.  Prints one JSON line.

    python scripts/bench_center_detection.py --steps K --warmup W [--images N]

Inputs: N images (4-class label maps from a quantised, smoothed intensity), the experiment's default ``params`` (slic_size 25,
slic_regul 0.3, fts_hist_diams [10, 50, 100, 200, 300], fts_ray_step 15, DBSCAN_max_dist 50) and a RandomForest trained on the
first image (a superpixel centre within 50 px of a true egg centre is a positive).  Legs, alternating in each step, each the median
over steps with min and max:
- ``device``: center_detection.detect_center_candidates_points;
- ``device_pixel_walk``: the same with descriptors.RUN_LENGTH_DISCS off (the discs counted by isb_disc_label_hist's pixel walk);
- ``host``: the host composition (the device SLIC and centres, then the oracle's ring counts and Ray tracer, scikit-learn predict
  and DBSCAN), from tests/center_host_reference.py.
Kernel time of the disc counts alone, old against new, from CUDA events over the same positions: ``isb_ring_label_hist`` (with its
run encoding) and ``isb_disc_label_hist``.  Parity: device and host give identical candidate masks, centres and cluster labels.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True      # the tree may be read-only
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import bench  # noqa: E402
import center_host_reference as chr_  # noqa: E402

H, W = 1024, 1280


def segment(img):
    from scipy import ndimage
    smooth = ndimage.gaussian_filter(img.mean(axis=-1), 2)
    return np.choose(np.digitize(smooth, [0.36, 0.42, 0.5]), [0, 2, 3, 1])


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def kernel_ms(positions, segm, diameters, reps=20):
    """CUDA-event time per call of the disc counts over the same device inputs: (run-length, pixel walk)"""
    import torch
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    d_seg = torch.from_numpy(np.ascontiguousarray(segm, dtype=np.int32)).cuda()
    d_pos = torch.from_numpy(np.ascontiguousarray(positions, dtype=np.int32)).cuda()
    d_diam = torch.from_numpy(np.asarray(diameters, dtype=np.int32)).cuda()
    nb = int(segm.max()) + 1
    hist = torch.empty((len(positions), len(diameters), nb), dtype=torch.float64, device='cuda')
    sizes = torch.empty((len(positions), len(diameters)), dtype=torch.float64, device='cuda')
    ws_bytes = lib.isb_label_runs_workspace_bytes(H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    calls = {
        'run_length': lambda: lib.isb_ring_label_hist(_lib.ptr(d_seg), H, W, _lib.ptr(d_pos), len(positions), _lib.ptr(d_diam), len(diameters),
                                                      nb, _lib.ptr(hist), _lib.ptr(sizes), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()),
        'pixel_walk': lambda: lib.isb_disc_label_hist(_lib.ptr(d_seg), None, H, W, _lib.ptr(d_pos), len(positions), _lib.ptr(d_diam),
                                                      len(diameters), None, 0, 0, nb, _lib.ptr(hist), _lib.ptr(sizes), _lib.stream_ptr()),
    }
    out, results = {}, {}
    for name, call in calls.items():
        _lib.check(call())
        torch.cuda.synchronize()
        results[name] = hist.cpu().numpy().copy()
        n = reps if name == 'run_length' else max(2, reps // 5)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(n):
            _lib.check(call())
        t1.record()
        t1.synchronize()
        out[name + '_ms'] = t0.elapsed_time(t1) / n
    out['equal'] = bool(np.array_equal(results['run_length'], results['pixel_walk']))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--images', type=int, default=2)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device'
    from sklearn.ensemble import RandomForestClassifier
    from pyimsegm_b200 import center_detection as cd
    from pyimsegm_b200 import descriptors as ds

    params = dict(cd.CENTER_PARAMS)
    params.update(cd.CLUSTER_PARAMS)
    data = []
    for i in range(args.images):
        img, _, centres = bench.synth_eggs_image(100 + i, h=H, w=W, n_eggs=8)
        data.append((img, segment(img), centres))
    img0, segm0, centres0 = data[0]
    _, _, points, feats, _ = cd.estim_points_compute_features('train', img0, segm0, params)
    labels = np.asarray(cd.label_close_points([tuple(c) for c in centres0], points, params)).astype(int)
    classif = RandomForestClassifier(n_estimators=50, random_state=0).fit(feats, labels)

    def device():
        return [cd.detect_center_candidates_points(img, segm, classif, params) for img, segm, _ in data]

    def device_pixel_walk():
        ds.RUN_LENGTH_DISCS = False
        try:
            return device()
        finally:
            ds.RUN_LENGTH_DISCS = True

    def host():
        return [chr_.detect_center_candidates_points(img, segm, classif, params) for img, segm, _ in data]

    legs = {'device': device, 'device_pixel_walk': device_pixel_walk, 'host': host}
    times = {k: [] for k in legs}
    results = {}
    for step in range(args.warmup + args.steps):
        for name, fn in legs.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            results[name] = fn()
            torch.cuda.synchronize()
            if step >= args.warmup:
                times[name].append(time.perf_counter() - t)

    def same(a, b):
        return all(np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3]) and np.array_equal(np.asarray(x[4]), np.asarray(y[4]))
                   for x, y in zip(a, b))

    int_pos = [[int(p) for p in q] for q in results['device'][0][0]]
    kern = kernel_ms(int_pos, segm0, params['fts_hist_diams'])
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        'bench': 'center_detection', 'gpu': gpu, 'image': [H, W], 'images': args.images, 'steps': args.steps,
        'points_per_image': [int(len(r[0])) for r in results['device']],
        'candidates_per_image': [int(r[2].sum()) for r in results['device']],
        'centres_per_image': [int(len(r[3])) for r in results['device']],
        'legs': {k: stats(v) for k, v in times.items()},
        'disc_counts_kernel': kern,
        'parity': {'device_vs_host': same(results['device'], results['host']),
                   'pixel_walk_vs_host': same(results['device_pixel_walk'], results['host']),
                   'features_device_vs_host': all(np.array_equal(x[1], y[1]) for x, y in zip(results['device'], results['host']))},
    }))


if __name__ == '__main__':
    main()
