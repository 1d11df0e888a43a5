#!/usr/bin/env python
"""
bench_volume_pipeline.py -- the gray-volume pipeline (pipe_gray3d_slic_features_model_graphcut) three ways.  Prints one JSON line.

    python scripts/bench_volume_pipeline.py [--steps K] [--warmup W] [--volumes N] [--depth D] [--size S]

Inputs: N seeded synthetic float32 volumes of D x S x S (default 8 of 64 x 512 x 512: two intensity classes in blocks, a z step
and gaussian noise), spacing (12, 1, 1), sp_size 15, sp_regul 0.2, {'color': ['mean', 'std', 'energy']}, 2 classes fitted per
volume, gc_regul 0.1.  Legs, each the median and the min-max over steps of the time per volume:
- ``stages``: pipe_gray3d_slic_features_model_graphcut on a host volume, labels to the host (the stage functions: label volume
  down, features, host StandardScaler, device mixture fit, host edge weights, cut);
- ``resident``: segment_resident_volume on a volume already on the device, results left there (timed to a device synchronise);
- ``batch``: segment_volumes_batch over the N host volumes, (segm, segm_soft) to the host, total time / N.
Parity: the share of voxels on which ``stages`` and ``resident`` agree, and whether ``batch`` equals ``resident`` on every volume.
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

SPACING, SP_SIZE, SP_REGUL, GC_REGUL, NB_CLASSES = (12, 1, 1), 15, 0.2, 0.1, 2
FEATURES = {'color': ['mean', 'std', 'energy']}


def synth_volume(seed, depth, size):
    rng = np.random.RandomState(seed)
    zz, yy, xx = np.ogrid[:depth, :size, :size]
    cell = size // 8
    vol = 0.3 + 0.35 * (((yy // cell + xx // cell + rng.randint(0, 2)) % 2) ^ (zz > depth // 2))
    return np.clip(vol + rng.normal(0, 0.1, (depth, size, size)), 0, 1).astype(np.float32)


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--volumes', type=int, default=8)
    ap.add_argument('--depth', type=int, default=64)
    ap.add_argument('--size', type=int, default=512)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_volume_pipeline.py needs a CUDA device')
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    vols = [synth_volume(100 + i, args.depth, args.size) for i in range(args.volumes)]
    model = pl._fit_model(NB_CLASSES, True)
    d_vols = [torch.from_numpy(v).cuda() for v in vols]
    torch.cuda.synchronize()

    def stage_leg(i):
        return pl.pipe_gray3d_slic_features_model_graphcut(vols[i], NB_CLASSES, FEATURES, SPACING, SP_SIZE, SP_REGUL, GC_REGUL)

    def resident_leg(i):
        out = pl.segment_resident_volume(d_vols[i], model, FEATURES, SPACING, SP_SIZE, SP_REGUL, GC_REGUL)
        torch.cuda.synchronize()
        return out

    def batch_leg():
        return pl.segment_volumes_batch(vols, nb_classes=NB_CLASSES, dict_features=FEATURES, spacing=SPACING, sp_size=SP_SIZE,
                                        sp_regul=SP_REGUL, gc_regul=GC_REGUL)

    times = {'stages': [], 'resident': [], 'batch': []}
    last = {}
    for step in range(args.warmup + args.steps):
        timed = step >= args.warmup
        for i in range(len(vols)):
            t0 = time.perf_counter()
            segm = stage_leg(i)
            dt = time.perf_counter() - t0
            if timed:
                times['stages'].append(dt)
                last[('stages', i)] = segm
            t0 = time.perf_counter()
            d_segm, _ = resident_leg(i)
            dt = time.perf_counter() - t0
            if timed:
                times['resident'].append(dt)
                last[('resident', i)] = d_segm.cpu().numpy()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = batch_leg()
        dt = time.perf_counter() - t0
        if timed:
            times['batch'].append(dt / len(vols))
            last['batch'] = out
    agree = float(np.mean([np.mean(last[('stages', i)] == last[('resident', i)]) for i in range(len(vols))]))
    batch_equal = all(np.array_equal(last['batch'][i][0], last[('resident', i)]) for i in range(len(vols)))
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({
        'benchmark': 'gray-volume pipeline, ms per volume',
        'gpu': gpu[torch.cuda.current_device()] if gpu else 'unknown',
        'volumes': len(vols), 'shape': [args.depth, args.size, args.size], 'dtype': 'float32', 'spacing': list(SPACING),
        'sp_size': SP_SIZE, 'features': FEATURES, 'nb_classes': NB_CLASSES, 'gc_regul': GC_REGUL, 'steps': args.steps,
        'supervoxels_last_volume': int(eng.to_host(eng.buf('n_labels', (1, ), torch.int32))[0]),
        'stages': stats(times['stages']), 'resident': stats(times['resident']), 'batch': stats(times['batch']),
        'parity': {'stages_vs_resident_voxel_agreement': agree, 'batch_equals_resident': batch_equal},
    }))


if __name__ == '__main__':
    main()
