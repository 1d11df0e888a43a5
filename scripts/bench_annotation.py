#!/usr/bin/env python
"""
bench_annotation.py -- imsegm.annotation on the device against the host oracle (oracle/annotation.py).  Prints one JSON line.

    python scripts/bench_annotation.py [--steps K] [--warmup W] [--sizes 2048,8192] [--oracle-max 2048]

Per size, on a synthetic annotation image (conftest's synth_regions classes painted with DICT_COLOURS, 2 % of the pixels set to
colours outside the palette, as anti-aliased strokes leave them):
- end-to-end time (numpy in, numpy out; host clock around calls that end in a synchronise) of unique_image_colors,
  image_frequent_colors, convert_img_colors_to_labels, convert_img_labels_to_colors, image_color_2_labels,
  quantize_image_nearest_color, image_inpaint_pixels and quantize_image_nearest_pixel;
- the oracle's host time for the same calls, at sizes up to --oracle-max (its KD-tree and per-colour passes take minutes beyond);
- the card's name and power limit (nvidia-smi) beside the numbers.
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import synth_regions  # noqa: E402
from oracle import annotation as oa  # noqa: E402


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def annotation_image(size, palette):
    _, cls = synth_regions(size, size, n_classes=len(palette))
    img = np.asarray(palette, dtype=np.uint8)[cls]
    rng = np.random.RandomState(0)
    stray = rng.rand(size, size) < 0.02
    img[stray] = rng.randint(0, 256, (int(stray.sum()), 3))
    return img, cls, ~stray


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sizes', default='2048,8192')
    ap.add_argument('--oracle-max', type=int, default=2048)
    args = ap.parse_args()
    import torch
    from pyimsegm_b200 import annotation as an

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ts = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return stats(ts)

    palette = [an.DICT_COLOURS[k] for k in range(4)]
    lut = {k: palette[k] for k in range(4)}
    results = []
    for size in [int(s) for s in args.sizes.split(',')]:
        img, cls, valid = annotation_image(size, palette)
        clean = np.asarray(palette, dtype=np.uint8)[cls]
        values = cls.astype(np.float64)
        calls = {
            'unique_image_colors': (an.unique_image_colors, oa.unique_image_colors, (img, )),
            'image_frequent_colors': (an.image_frequent_colors, oa.image_frequent_colors, (img, )),
            'convert_img_colors_to_labels': (an.convert_img_colors_to_labels, oa.convert_img_colors_to_labels, (clean, lut)),
            'convert_img_labels_to_colors': (an.convert_img_labels_to_colors, oa.convert_img_labels_to_colors, (cls, lut)),
            'image_color_2_labels': (an.image_color_2_labels, oa.image_color_2_labels, (img, palette)),
            'quantize_image_nearest_color': (an.quantize_image_nearest_color, oa.quantize_image_nearest_color, (img, palette)),
            'image_inpaint_pixels': (an.image_inpaint_pixels, oa.image_inpaint_pixels, (values, valid)),
            'quantize_image_nearest_pixel': (an.quantize_image_nearest_pixel, oa.quantize_image_nearest_pixel, (img, palette)),
        }
        row = {'size': [size, size], 'device_ms': {}, 'oracle_host_ms': {}, 'speedup': {}}
        for name, (dev, host, fargs) in calls.items():
            row['device_ms'][name] = timed(lambda: dev(*fargs))
            if size <= args.oracle_max:
                t0 = time.perf_counter()
                host(*fargs)
                row['oracle_host_ms'][name] = (time.perf_counter() - t0) * 1e3
                row['speedup'][name] = row['oracle_host_ms'][name] / row['device_ms'][name]['median_ms']
        if size > args.oracle_max:
            row['oracle_host_ms'] = 'not run above --oracle-max'
        results.append(row)
        print(json.dumps({'size': size, 'partial': row}), file=sys.stderr)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({'bench': 'annotation', 'gpu': gpu, 'sizes': results}))


if __name__ == '__main__':
    main()
