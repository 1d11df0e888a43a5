#!/usr/bin/env python
"""
bench_shared_model.py -- the reference's shared-model entry point (pipelines.py:160-241) on config-2 images: a caller-fitted class
model evaluated on the device against the host round trip.  Prints one JSON line.

    python scripts/bench_shared_model.py --steps K --warmup W

Images: eight config-2 images (bench.synth_image: 2048x2048 RGB f64, sp_size 29, colour means).  Two models, both fitted before
timing -- the group GMM of estim_model_classes_group over the eight images, and StandardScaler + RandomForestClassifier with the
reference's RandForest hyper-parameters (classification.py:101) trained on the superpixel labels of the synthetic class map of
image 0.  Legs, device predict and host predict (graph_cuts.USE_DEVICE_PREDICT = False) alternating in every step:
segment_images_batch over the eight images per model, and segment_resident with each compiled model (CUDA-graph replay).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload constants and image generator of the headline benchmark)

NB_IMAGES = 8


def synth_classes(seed, h=bench.H, w=bench.W, n_classes=bench.NB_CLASSES, cell=64):
    """the class map [h, w] behind bench.synth_image(seed, h, w, n_classes, cell): the same random draws, in the same order, up to the
    Voronoi assignment (the annotation a supervised model is trained on)"""
    rng = np.random.RandomState(seed)
    pts = rng.rand(40, 2) * [h, w]
    cls = rng.randint(0, n_classes, 40)
    gy, gx = np.mgrid[:(h + cell - 1) // cell, :(w + cell - 1) // cell] * cell + cell / 2
    near = ((gy[..., None] - pts[:, 0]) ** 2 + (gx[..., None] - pts[:, 1]) ** 2).argmin(-1)
    return np.kron(cls[near], np.ones((cell, cell), dtype=int))[:h, :w]


def card_info():
    """name, power limit and maximum SM clock of the card the numbers were measured on (nvidia-smi), or None"""
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                              str(bench.dist_env()[2])], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [c.strip() for c in out.split(',')]
        return {'name': name, 'power_limit': power, 'sm_max_clock': clock}
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def run(steps, warmup):
    import torch
    from sklearn import ensemble, pipeline, preprocessing
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    torch.cuda.set_device(bench.dist_env()[2])
    from pyimsegm_b200 import _lib, graph_cuts, pipelines
    lib = _lib.lib()
    F, SP, REG, GC = bench.FEATURES, bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL
    seeds = [6000 + i for i in range(NB_IMAGES)]
    images = [torch.from_numpy(bench.synth_image(s)).pin_memory().numpy() for s in seeds]
    gmm, _ = pipelines.estim_model_classes_group(images, bench.NB_CLASSES, F, sp_size=SP, sp_regul=REG)
    _, fts, labels = pipelines.wrapper_compute_color2d_slic_features_labels((images[0], synth_classes(seeds[0])), SP, REG, F, 0.9)
    sel = labels >= 0
    forest = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                ('classif', ensemble.RandomForestClassifier(n_estimators=20, min_samples_leaf=2, min_samples_split=3,
                                                                            n_jobs=1, random_state=0))]).fit(fts[sel], labels[sel])
    models = {'gmm': gmm, 'forest': forest}
    dev_img = torch.from_numpy(images[0]).cuda()

    def batch(name, device):
        graph_cuts.USE_DEVICE_PREDICT = device
        try:
            return pipelines.segment_images_batch(images, dict_features=F, sp_size=SP, sp_regul=REG, gc_regul=GC, model_pipeline=models[name])
        finally:
            graph_cuts.USE_DEVICE_PREDICT = True

    def resident(name):
        return pipelines.segment_resident(dev_img, models[name], F, SP, REG, GC, 'model')

    legs = [('batch_%s_%s' % (m, 'device' if d else 'host'), (lambda m=m, d=d: batch(m, d)), NB_IMAGES) for m in models for d in (True, False)]
    legs += [('resident_%s_device' % m, (lambda m=m: resident(m)), 1) for m in models]
    outs = {}
    for name, fn, _ in legs:            # warm every leg: buffers sized, graphs captured, model tables uploaded
        for _ in range(max(warmup, 3)):
            outs[name] = fn()
    # parity of the last warm-up call of every leg (graph replays by then); the resident forest leg ran last, so the engine's result
    # buffers still hold its output.  The outputs are dropped before timing so that no leg holds pinned result buffers.
    gd, gh = outs['batch_gmm_device'], outs['batch_gmm_host']
    fd, fh = outs['batch_forest_device'], outs['batch_forest_host']
    rd = [t.cpu().numpy() for t in outs['resident_forest_device']]
    parity = {'forest_segm_identical': all(np.array_equal(a[0], b[0]) for a, b in zip(fd, fh)),
              'forest_segm_soft_identical': all(np.array_equal(a[1], b[1]) for a, b in zip(fd, fh)),
              'forest_resident_segm_identical': bool(np.array_equal(np.asarray(forest.classes_)[rd[0]], fh[0][0])),
              'gmm_segm_identical': all(np.array_equal(a[0], b[0]) for a, b in zip(gd, gh)),
              'gmm_segm_soft_max_abs_diff': float(max(np.abs(a[1] - b[1]).max() for a, b in zip(gd, gh)))}
    del gd, gh, fd, fh, rd
    per_step = {name: [] for name in outs}
    outs = None
    for _ in range(steps):               # the legs alternate inside every step (the host shares the machine with other work)
        for name, fn, n in legs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            per_step[name].append((time.perf_counter() - t0) / n * 1e3)
            del out
    # class-model stage time per image (device timers, a separate untimed pass with eager launches)
    gmm_stage = {}
    nstage = lib.isb_profile_stage_count()
    stage = [i for i in range(nstage) if lib.isb_profile_stage_name(i).decode() == 'gmm'][0]
    pipelines.USE_CUDA_GRAPHS = False
    for name, fn, n in legs:
        lib.isb_profile_enable(1)
        fn()
        ms_arr, cnt_arr = (C.c_double * nstage)(), (C.c_longlong * nstage)()
        lib.isb_profile_collect(ms_arr, cnt_arr)
        lib.isb_profile_enable(0)
        gmm_stage[name] = ms_arr[stage] / n
    pipelines.USE_CUDA_GRAPHS = True
    mpix = bench.H * bench.W / 1e6
    result = {}
    for name, _, _ in legs:
        ms_img = float(np.median(per_step[name]))
        result[name] = {'value': mpix / (ms_img / 1e3), 'unit': 'MPix/s', 'ms_per_image': ms_img,
                        'ms_per_image_min_max': [min(per_step[name]), max(per_step[name])], 'gmm_stage_ms_per_image': gmm_stage[name]}
    return {'metric': 'megapixels/sec, shared-model segmentation (segment_color2d_slic_features_model_graphcut family)',
            'unit': 'MPix/s', 'n_gpus': 1, 'steps': steps, 'warmup': max(warmup, 3), 'higher_is_better': True, 'dtype': 'f64',
            'data': 'synthetic',
            'config': {'workload': 'shared-model: %d config-2 images (2048x2048 RGB f64), SLIC sp_size=%d, colour-mean, GraphCut gc_regul %g; '
                                   'models fitted before timing' % (NB_IMAGES, SP, GC),
                       'models': {'gmm': 'estim_model_classes_group over the %d images (StandardScaler + 3-class full GMM)' % NB_IMAGES,
                                  'forest': 'StandardScaler + RandomForestClassifier(n_estimators=20, min_samples_leaf=2, '
                                            'min_samples_split=3, n_jobs=1) on the superpixel labels of image 0'},
                       'timed': 'host clock around each call with a device synchronise on both sides; legs alternate within a step; '
                                'ms_per_image = median over the steps; batch legs: host images in, host (segm, segm_soft) out; '
                                'resident legs: device image, device results'},
            'legs': result, 'parity': parity, 'card': card_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))


if __name__ == '__main__':
    main()
