#!/usr/bin/env python
"""
bench_neighbour_models.py -- k-nearest-neighbour and logistic-regression models in the shared-model entry point (reference
pipelines.py:160-241) on config-2 images: device predict_proba (isb_knn_predict_proba / isb_linear_predict_proba) against the host
round trip, and the KNN kernel alone.  Prints one JSON line.

    python scripts/bench_neighbour_models.py --steps K --warmup W

Images: eight config-2 images (bench.synth_image: 2048x2048 RGB f64, sp_size 29, colour means).  Two models fitted before timing,
the reference's create_clf_pipeline('KNN') and ('LogistRegr') -- StandardScaler, PCA(0.95), then KNeighborsClassifier() or
LogisticRegression(solver='sag') -- on the superpixel labels (synthetic class maps) of four other config-2 images.  Legs, alternating
in every step: segment_images_batch over the eight images per model with device predict and with host predict
(graph_cuts.USE_DEVICE_PREDICT = False).  Kernel legs: isb_knn_predict_proba alone on 5 000 queries against 40 000 training rows
(k = 5, uniform) at D = 9 and D = 189, timed with CUDA events; achieved FP64 rate = 3 N N_t D / kernel time (a subtraction, a
multiplication and an addition per query, training row and dimension).
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

import bench  # noqa: E402  (the workload constants and image generator of the headline benchmark)
from scripts.bench_shared_model import card_info, synth_classes  # noqa: E402

NB_IMAGES, NB_TRAIN = 8, 4
#: NVIDIA H100 SXM data sheet, FP64 without the tensor cores (a card allowed up to 700 W)
DATASHEET_FP64_TFLOPS = 34.0
KERNEL_N, KERNEL_NT, KERNEL_K = 5000, 40000, 5


def kernel_leg(D, reps=20):
    """isb_knn_predict_proba on random clustered rows: (ms per call, achieved FLOP/s)"""
    import torch
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    rng = np.random.RandomState(D)
    centres = rng.normal(0, 1, (bench.NB_CLASSES, D))
    yt = rng.randint(0, bench.NB_CLASSES, KERNEL_NT)
    fit_x = torch.from_numpy(centres[yt] + rng.normal(0, 0.5, (KERNEL_NT, D))).cuda()
    x = torch.from_numpy(centres[rng.randint(0, bench.NB_CLASSES, KERNEL_N)] + rng.normal(0, 0.5, (KERNEL_N, D))).cuda()
    y = torch.from_numpy(yt.astype(np.int32)).cuda()
    proba = torch.empty((KERNEL_N, bench.NB_CLASSES), dtype=torch.float64, device='cuda')
    wsb = lib.isb_knn_predict_workspace_bytes(KERNEL_N, KERNEL_NT, KERNEL_K)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device='cuda')

    def call():
        _lib.check(lib.isb_knn_predict_proba(_lib.ptr(x), KERNEL_N, None, D, _lib.ptr(fit_x), KERNEL_NT, _lib.ptr(y), KERNEL_K,
                                             bench.NB_CLASSES, 0, _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
    for _ in range(3):
        call()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        call()
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / reps
    flops = 3.0 * KERNEL_N * KERNEL_NT * D / (ms / 1e3)
    return {'ms_per_call': ms, 'fp64_tflops_achieved': flops / 1e12, 'fraction_of_datasheet_fp64': flops / 1e12 / DATASHEET_FP64_TFLOPS,
            'N': KERNEL_N, 'N_t': KERNEL_NT, 'D': D, 'k': KERNEL_K}


def run(steps, warmup):
    import torch
    from sklearn import decomposition, linear_model, neighbors, pipeline, preprocessing
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    torch.cuda.set_device(bench.dist_env()[2])
    from pyimsegm_b200 import graph_cuts, pipelines
    from pyimsegm_b200.class_models import compile_model
    F, SP, REG, GC = bench.FEATURES, bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL
    images = [torch.from_numpy(bench.synth_image(7000 + i)).pin_memory().numpy() for i in range(NB_IMAGES)]
    feats, labels = [], []
    for s in range(7100, 7100 + NB_TRAIN):
        _, f, lab = pipelines.wrapper_compute_color2d_slic_features_labels((bench.synth_image(s), synth_classes(s)), SP, REG, F, 0.9)
        feats.append(f[lab >= 0])
        labels.append(lab[lab >= 0])
    X, y = np.vstack(feats), np.hstack(labels)

    def clf_pipeline(classif):
        return pipeline.Pipeline([('scaler', preprocessing.StandardScaler()), ('reduce_dim', decomposition.PCA(0.95)), ('classif', classif)])
    models = {'knn': clf_pipeline(neighbors.KNeighborsClassifier()).fit(X, y),
              'logistic': clf_pipeline(linear_model.LogisticRegression(solver='sag')).fit(X, y)}
    assert compile_model(models['knn']).kind == 'knn' and compile_model(models['logistic']).kind == 'linear'

    def batch(name, device):
        graph_cuts.USE_DEVICE_PREDICT = device
        try:
            return pipelines.segment_images_batch(images, dict_features=F, sp_size=SP, sp_regul=REG, gc_regul=GC, model_pipeline=models[name])
        finally:
            graph_cuts.USE_DEVICE_PREDICT = True

    legs = [('batch_%s_%s' % (m, 'device' if d else 'host'), (lambda m=m, d=d: batch(m, d))) for m in models for d in (True, False)]
    outs = {}
    for name, fn in legs:
        for _ in range(max(warmup, 3)):
            outs[name] = fn()
    parity = {'%s_segm_identical' % m: all(np.array_equal(a[0], b[0]) for a, b in zip(outs['batch_%s_device' % m], outs['batch_%s_host' % m]))
              for m in models}
    parity['knn_segm_soft_identical'] = all(np.array_equal(a[1], b[1]) for a, b in zip(outs['batch_knn_device'], outs['batch_knn_host']))
    parity['logistic_segm_soft_max_abs_diff'] = float(max(np.abs(a[1] - b[1]).max()
                                                          for a, b in zip(outs['batch_logistic_device'], outs['batch_logistic_host'])))
    outs = None
    per_step = {name: [] for name, _ in legs}
    for _ in range(steps):
        for name, fn in legs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            per_step[name].append((time.perf_counter() - t0) / NB_IMAGES * 1e3)
            del out
    result = {name: {'ms_per_image': float(np.median(v)), 'ms_per_image_min_max': [min(v), max(v)]} for name, v in per_step.items()}
    return {'metric': 'ms per image, shared-model segmentation with KNN / logistic-regression models, device vs host predict_proba',
            'unit': 'ms/image', 'n_gpus': 1, 'steps': steps, 'warmup': max(warmup, 3), 'higher_is_better': False, 'dtype': 'f64',
            'data': 'synthetic',
            'config': {'workload': '%d config-2 images (2048x2048 RGB f64), SLIC sp_size=%d, colour-mean, GraphCut gc_regul %g'
                                   % (NB_IMAGES, SP, GC),
                       'models': 'StandardScaler + PCA(0.95) + KNeighborsClassifier() / LogisticRegression(solver=sag), fitted on '
                                 '%d superpixel rows of %d other images' % (len(X), NB_TRAIN),
                       'timed': 'host clock around each batch call with a device synchronise on both sides; legs alternate within a '
                                'step; median over the steps'},
            'legs': result, 'parity': parity,
            'knn_kernel': {'D9': kernel_leg(9), 'D189': kernel_leg(189),
                           'reference_rate': 'H100 SXM data-sheet FP64 (non-tensor) %.0f TFLOP/s' % DATASHEET_FP64_TFLOPS},
            'card': card_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))


if __name__ == '__main__':
    main()
