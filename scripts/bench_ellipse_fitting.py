#!/usr/bin/env python
"""
bench_ellipse_fitting.py -- RANSAC ellipse fitting of the reference's egg-segmentation experiment (ellipse_ransac_crit) on a
bench.synth_eggs_image.  Prints one JSON line.

    python scripts/bench_ellipse_fitting.py --steps K --warmup W [--host-steps H]

The image is segmented into 4 classes (a quantised, smoothed intensity: 0 background, 1 egg core, 2-3 the rim); boundary points come
from prepare_boundary_points_ray_edge / _ray_join / _ray_mean about the true egg centres; the experiment's parameters
(slic_size 15, slic_regul 0.1, min_samples 0.35, residual_threshold 25, max_trials 250, table [0.01, 0.95, 0.95, 0.85]).
Legs, each the median over steps with min and max: ransac_segm per centre on the device, ransac_segm_centres over all centres,
and the oracle's host loop (scipy leastsq per point, the process pinned to one core).  Parity per centre: the selected trial and max |d params|.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import ellipse as oe  # noqa: E402

TABLE = [0.01, 0.95, 0.95, 0.85]
SLIC_SIZE, SLIC_REGUL, MIN_SAMPLES, THR, TRIALS = 15, 0.1, 0.35, 25, 250


def segment(img):
    from scipy import ndimage
    smooth = ndimage.gaussian_filter(img.mean(axis=-1), 2)
    return np.choose(np.digitize(smooth, [0.36, 0.42, 0.5]), [0, 2, 3, 1])


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--host-steps', type=int, default=1)
    args = ap.parse_args()
    import torch
    from pyimsegm_b200 import ellipse_fitting as ef
    img, _, centres = bench.synth_eggs_image(0)
    seg = segment(img)
    slic, points_all, labels = ef.get_slic_points_labels(seg, slic_size=SLIC_SIZE, slic_regul=SLIC_REGUL)
    weights = np.bincount(slic.ravel())
    point_sets = []
    for prep in (ef.prepare_boundary_points_ray_edge, ef.prepare_boundary_points_ray_join, ef.prepare_boundary_points_ray_mean):
        point_sets += prep(seg, centres)
    ext = (points_all, weights, labels, TABLE, MIN_SAMPLES, THR, TRIALS)

    def per_centre():
        np.random.seed(0)
        return [ef.ransac_segm(p, ef.EllipseModelSegm, *ext) for p in point_sets]

    def batched():
        np.random.seed(0)
        return ef.ransac_segm_centres(point_sets, ef.EllipseModelSegm, *ext)

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        ts, out = [], None
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return ts, out

    t_loop, res_loop = timed(per_centre, args.steps, args.warmup)
    t_batch, res_batch = timed(batched, args.steps, args.warmup)
    same = all((a[0] is None and b[0] is None) or (a[0] is not None and b[0] is not None and np.array_equal(a[0].params, b[0].params))
               for a, b in zip(res_loop, res_batch))

    # oracle host loop, and parity of the selected trial and the final parameters
    t_host, parity = [], []
    cpus = os.sched_getaffinity(0)
    os.sched_setaffinity(0, {min(cpus)})          # the host leg on one core (BLAS threads included)
    for _ in range(args.host_steps):
        np.random.seed(0)
        t0 = time.perf_counter()
        sel = [oe.ransac_select(p, oe.ransac_trials(p, points_all, weights, labels, TABLE, MIN_SAMPLES, THR, TRIALS)) for p in point_sets]
        t_host.append(time.perf_counter() - t0)
    os.sched_setaffinity(0, cpus)
    np.random.seed(0)
    samples = [[np.random.choice(len(p), int(MIN_SAMPLES * len(p)), replace=False) for _ in range(TRIALS)] for p in point_sets]
    term = ef._label_terms(weights, labels, TABLE)
    for c, p in enumerate(point_sets):
        ok, _, n_inl, crit, _ = ef._run_trials([p], [0] * TRIALS, samples=samples[c], crit_input=(points_all, labels, term), thr=THR)
        idx_d, _ = ef._select(ok, n_inl, crit)
        dev_model = res_batch[c][0]
        dp = None
        if dev_model is not None and sel[c][0] is not None:
            dp = float(np.max(np.abs(np.subtract(dev_model.params, sel[c][0]))))
        parity.append({'centre': c, 'trial_device': -1 if idx_d is None else int(idx_d), 'trial_oracle': int(sel[c][2]),
                       'max_abs_dparams': dp})
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'bench': 'ellipse_fitting', 'gpu': gpu, 'centres': len(point_sets), 'trials_per_centre': TRIALS,
                      'superpixels': int(len(labels)), 'ransac_segm_per_centre': stats(t_loop), 'ransac_segm_centres': stats(t_batch),
                      'oracle_host_loop_one_core': stats(t_host), 'centres_equal_loop': bool(same),
                      'selected_trial_equal': all(p['trial_device'] == p['trial_oracle'] for p in parity), 'parity': parity}))


if __name__ == '__main__':
    main()
