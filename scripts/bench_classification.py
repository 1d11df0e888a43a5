#!/usr/bin/env python
"""
bench_classification.py -- the scoring functions of imsegm.classification on the device against the host oracle
(oracle/classification.py).  Prints one JSON line.

    python scripts/bench_classification.py [--steps K] [--warmup W] [--sizes 2048,8192] [--oracle-max 2048]

Per size, on a synthetic pair (conftest's synth_regions: a uint8 annotation of 4 classes, an int64 segmentation of 3 classes in
smaller cells, label 0 dropped):
- end-to-end time (numpy in, dict out; host clock, every call ends in a synchronise) of compute_classif_stat_segm_annot with and
  without relabel, and of compute_stat_per_image over 8 pairs;
- the contingency kernels alone (count and write calls on maps already on the device, CUDA events), against their algorithmic
  bytes -- the maps' bytes per pixel times the passes over the pixels: the count call reads both maps twice (the range pass runs
  because the segmentation is 64-bit, then the presence pass), the write call once -- and a device-to-device copy measured in the
  same run;
- the oracle's host time up to --oracle-max;
- the card's name and power limit (nvidia-smi), read in the same run.
Each time is given as median, min and max over the steps.
"""
import argparse
import ctypes as C
import json
import logging
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import synth_regions  # noqa: E402
from oracle import classification as oc  # noqa: E402


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def pair(size, seed):
    _, annot = synth_regions(size, size, n_classes=4, seed=seed)
    _, segm = synth_regions(size, size, n_classes=3, seed=seed + 10, cell=32)
    return annot.astype(np.uint8), segm.astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sizes', default='2048,8192')
    ap.add_argument('--oracle-max', type=int, default=2048)
    args = ap.parse_args()
    warnings.simplefilter('ignore')
    logging.disable(logging.CRITICAL)
    import torch
    from pyimsegm_b200 import _lib
    from pyimsegm_b200 import classification as clf
    from pyimsegm_b200.engine import get_engine
    if not torch.cuda.is_available():
        raise SystemExit('bench_classification.py needs a CUDA device')

    def timed(fn, steps=None):
        for _ in range(args.warmup):
            fn()
        ts = []
        for _ in range(steps or args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return stats(ts)

    def event_ms(fn, reps=20):
        for _ in range(args.warmup + 1):
            fn()
        ts = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b) / reps / 1e3)
        return stats(ts)

    out = {'metric': 'classification_scoring', 'sizes': {}}
    eng = get_engine()
    lib = eng.lib
    for size in [int(s) for s in args.sizes.split(',')]:
        annot, segm = pair(size, 5)
        res = {}
        for relabel in (False, True):
            res['stat_segm_annot' + ('_relabel' if relabel else '')] = timed(
                lambda: clf.compute_classif_stat_segm_annot((annot, segm, 'x'), drop_labels=[0], relabel=relabel))
        pairs = [pair(size, s) for s in range(8)] if size <= 2048 else [(annot, segm)] * 8
        res['stat_per_image_8'] = timed(lambda: clf.compute_stat_per_image([s for _, s in pairs], [a for a, _ in pairs], drop_labels=[0]))

        # the contingency kernels alone, on maps already on the device
        n = annot.size
        d_t, d_p = eng.to_device(annot.ravel(), 'bench_t'), eng.to_device(segm.ravel(), 'bench_p')
        d_drop = eng.to_device(np.zeros(1, np.int64), 'bench_drop')
        dts = (clf._LABEL_DTYPES['uint8'], clf._LABEL_DTYPES['int64'])
        ws_bytes = lib.isb_contingency_workspace_bytes(*dts)
        ws = eng.buf('bench_ws', ws_bytes, torch.uint8)
        info = (C.c_longlong * 6)()
        cargs = (_lib.ptr(d_t), dts[0], _lib.ptr(d_p), dts[1], C.c_longlong(n), _lib.ptr(d_drop), 1)
        st = _lib.stream_ptr()
        _lib.check(lib.isb_contingency_count(*cargs, _lib.ptr(ws), C.c_size_t(ws_bytes), info, st))
        kt, kp = int(info[0]), int(info[1])
        vt, vp = eng.buf('bench_vt', kt, torch.int64), eng.buf('bench_vp', kp, torch.int64)
        counts = eng.buf('bench_counts', kt * kp, torch.int64)

        def count():
            _lib.check(lib.isb_contingency_count(*cargs, _lib.ptr(ws), C.c_size_t(ws_bytes), info, st))

        def write():
            _lib.check(lib.isb_contingency_write(*cargs, info, _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(vt), _lib.ptr(vp),
                                                 _lib.ptr(counts), st))
        px_bytes = annot.itemsize + segm.itemsize
        src = torch.empty(n * px_bytes, dtype=torch.uint8, device='cuda')
        dst = torch.empty_like(src)
        copy = event_ms(lambda: dst.copy_(src))
        copy_gbs = 2 * n * px_bytes / (copy['median_ms'] / 1e3) / 1e9       # read + write
        t_count, t_write = event_ms(count, reps=5), event_ms(write)
        res['kernels'] = {
            'count_ms': t_count, 'write_ms': t_write, 'table': [kt, kp],
            'count_passes': 2, 'write_passes': 1, 'bytes_per_pixel_per_pass': px_bytes,
            'count_GBs': 2 * n * px_bytes / (t_count['median_ms'] / 1e3) / 1e9,
            'write_GBs': n * px_bytes / (t_write['median_ms'] / 1e3) / 1e9,
            'copy_GBs_read_plus_write': copy_gbs,
        }
        if size <= args.oracle_max:
            for relabel in (False, True):
                t0 = time.perf_counter()
                oc.compute_classif_stat_segm_annot((annot, segm, 'x'), drop_labels=[0], relabel=relabel)
                res['oracle_stat_segm_annot' + ('_relabel' if relabel else '') + '_ms'] = (time.perf_counter() - t0) * 1e3
        out['sizes'][str(size)] = res
    try:
        out['gpu'] = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                             text=True).strip()
    except (OSError, subprocess.CalledProcessError) as err:
        out['gpu'] = 'nvidia-smi failed: %s' % err
    print(json.dumps(out))


if __name__ == '__main__':
    main()
