#!/usr/bin/env python
"""
bench_tiled_features.py -- the banded path (pyimsegm_b200/tiled.py) with colour spaces, meanGrad and caller-fitted models on one
config-5-style image, against the single-image pipelines.  Prints one JSON line.

    python scripts/bench_tiled_features.py [--size 8192] [--bands 2] [--steps 3] [--warmup 1]
    torchrun --nproc-per-node N scripts/bench_tiled_features.py ...      (bands over N GPUs; rank 0 prints)

Image: bench.synth_image (seeded, RGB f64) of --size x --size, sp_size 29, 3 classes, GraphCut gc_regul 1.  Cases:
  colour_spaces     pipe_..._tiled with {'color': mean, std, meanGrad; 'color_hsv': mean}
  texture_meangrad  pipe_..._tiled with {'tLM_short': mean, meanGrad}
  group_gmm         segment_..._tiled with a GMM from estim_model_classes_group (fitted on two 1024^2 images), {'color': mean, std}
  random_forest     segment_..._tiled with a RandomForestClassifier trained on wrapper_compute_color2d_slic_features_labels output
Legs: 'banded' = --bands bands per rank (all on this process's GPU), 'single' = the single-image pipeline on one GPU (only in a
one-process run).  Host clock around each call with a device synchronise on both sides, the legs alternating within every step;
ms = median over the steps (max over the ranks for the banded leg).  Labels of the two legs are compared once per case.
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

COLOUR = {'color': ['mean', 'std', 'meanGrad'], 'color_hsv': ['mean']}
TEXTURE = {'tLM_short': ['mean', 'meanGrad']}
MODEL_FTS = {'color': ['mean', 'std']}


def run(size, bands, steps, warmup):
    import torch
    import torch.distributed as dist
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    rank, world, local = bench.dist_env()
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl')
    from sklearn.ensemble import RandomForestClassifier
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200 import tiled
    comm = tiled.default_comm()
    SP, REG, GC, K = bench.SP_SIZE, bench.SP_REGUL, bench.GC_REGUL, bench.NB_CLASSES
    img = torch.from_numpy(bench.synth_image(5, size, size)).pin_memory().numpy()
    train = [bench.synth_image(s, 1024, 1024) for s in (6, 7)]
    gmm, _ = pl.estim_model_classes_group(train, K, MODEL_FTS, sp_size=SP, sp_regul=REG)
    feats, labels = [], []
    for s, im in zip((6, 7), train):
        annot = np.array([2, 5, 7])[np.rint((im[..., 0] - 0.2) / 0.3).clip(0, 2).astype(int)]
        _, f, lab = pl.wrapper_compute_color2d_slic_features_labels((im, annot), SP, REG, MODEL_FTS, 0.9)
        feats.append(f[lab >= 0])
        labels.append(lab[lab >= 0])
    forest = RandomForestClassifier(n_estimators=16, max_depth=10, random_state=0).fit(np.vstack(feats), np.hstack(labels))

    def pipe_case(fts):
        return (lambda: tiled.pipe_color2d_slic_features_model_graphcut_tiled(img, K, fts, SP, REG, gc_regul=GC, comm=comm,
                                                                               bands_per_rank=bands),
                lambda: pl.pipe_color2d_slic_features_model_graphcut(img, K, fts, SP, REG, gc_regul=GC))

    def model_case(model):
        return (lambda: tiled.segment_color2d_slic_features_model_graphcut_tiled(img, model, MODEL_FTS, SP, REG, GC, comm=comm,
                                                                                  bands_per_rank=bands),
                lambda: pl.segment_color2d_slic_features_model_graphcut(img, model, MODEL_FTS, SP, REG, GC))

    cases = {'colour_spaces': (COLOUR, pipe_case(COLOUR)), 'texture_meangrad': (TEXTURE, pipe_case(TEXTURE)),
             'group_gmm': (MODEL_FTS, model_case(gmm)), 'random_forest': (MODEL_FTS, model_case(forest))}
    out = {}
    for name, (fts, (banded, single)) in cases.items():
        legs = [('banded', banded)] + ([('single', single)] if world == 1 else [])
        for _, fn in legs:
            for _ in range(warmup):
                fn()
        agree = None
        if world == 1:
            got, want = banded()[0], single()[0]
            agree = float(np.mean(got == want))
        times = {leg: [] for leg, _ in legs}
        for _ in range(steps):
            for leg, fn in legs:
                if world > 1:
                    dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
                if world > 1:
                    t = torch.tensor([ms], device='cuda')
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                    ms = float(t.item())
                times[leg].append(ms)
        res = {leg: {'ms': float(np.median(v)), 'ms_min_max': [min(v), max(v)]} for leg, v in times.items()}
        if 'single' in res:
            res['banded_over_single'] = res['banded']['ms'] / res['single']['ms']
        out[name] = {'features': fts, 'legs': res, 'label_agreement_banded_vs_single': agree}
    card = card_info()
    result = {'metric': 'ms per image, banded path with colour spaces / meanGrad / caller-fitted models vs the single-image pipeline',
              'unit': 'ms', 'n_gpus': world, 'bands_per_rank': bands, 'steps': steps, 'warmup': warmup, 'higher_is_better': False,
              'config': {'workload': 'one %dx%d RGB f64 synthetic image, SLIC sp_size=%d, %d classes, GraphCut gc_regul %g'
                                     % (size, size, SP, K, GC)},
              'cases': out, 'card': card}
    if world > 1:
        dist.destroy_process_group()
    return result if rank == 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=8192)
    ap.add_argument('--bands', type=int, default=2, help='bands per rank')
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    result = run(args.size, args.bands, args.steps, args.warmup)
    if result is not None:
        print(json.dumps(result))


if __name__ == '__main__':
    main()
