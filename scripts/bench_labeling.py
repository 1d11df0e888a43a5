#!/usr/bin/env python
"""
bench_labeling.py -- imsegm.labeling on SLIC label maps of conftest's synth_regions image against its annotation.  Prints one JSON line.

    python scripts/bench_labeling.py [--steps K] [--warmup W] [--sizes 2048,8192]

Per size (the SLIC map of segment_slic_img2d(img, 30, 0.2) versus the annotation):
- end-to-end time (numpy in, numpy out) of compute_boundary_distances, compute_distance_map, relabel_max_overlap_unique and
  compute_labels_overlap_matrix, host clock around calls that end in a synchronise;
- device time of the same calls' kernels from CUDA events, with the inputs already on the device (boundary maps + EDT + compaction;
  contour map + EDT; joint histogram + relabel gather; joint histogram);
- the time of every EDT phase (torch.profiler, CUDA activities), its bytes computed from the shape, and the phase's time at the
  device-to-device copy bandwidth measured in the same run;
- the oracle's host time for the same calls (oracle/labeling.py; its per-pixel loops are run at 2048 x 2048 only).
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import synth_regions  # noqa: E402
from oracle import labeling as ol  # noqa: E402

EDT_KERNELS = ('k_edt_bits', 'k_edt_links', 'k_edt_cols', 'k_edt_local', 'k_edt_merge', 'Memset', 'k_edt_marks', 'k_edt_bandmax',
               'k_edt_carry', 'k_edt_fill')


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def edt_phase_bytes(H, W):
    """bytes each EDT phase must move, from the shape: u8 sites, i32 band words and links, i32 column distances gT, i32 list pointers
    (prev, next) and marks, i32 per-(band, row) tables, f64 output.  The merges touch only the junctions of the lists: their per-row
    head / tail tables are counted."""
    nb, nc = (H + 31) // 32, (W + 31) // 32
    px, levels = H * W, max(1, (nc - 1).bit_length())
    return {'k_edt_bits': px + 4 * nb * W, 'k_edt_links': 12 * nb * W, 'k_edt_cols': 12 * nb * W + 4 * px,
            'k_edt_local': 4 * px + 8 * px + 8 * nc * H, 'k_edt_merge': levels * 16 * nc * H, 'Memset': 4 * px,
            'k_edt_marks': 12 * px, 'k_edt_bandmax': 4 * px + 4 * nc * H, 'k_edt_carry': 8 * nc * H, 'k_edt_fill': 4 * px + 8 * px}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--sizes', default='2048,8192')
    args = ap.parse_args()
    import torch
    from pyimsegm_b200 import _lib, labeling as lb, superpixels
    eng = lb.get_engine()
    lib = eng.lib
    st = _lib.stream_ptr

    def timed(fn, steps=args.steps, warmup=args.warmup):
        for _ in range(warmup):
            fn()
        ts = []
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return stats(ts)

    def events(fn, steps=args.steps, warmup=args.warmup):
        for _ in range(warmup):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in ev:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return stats([a.elapsed_time(b) * 1e-3 for a, b in ev])

    # device-to-device copy bandwidth (read + write bytes over time)
    big = torch.empty(1 << 30, dtype=torch.uint8, device='cuda')
    dst = torch.empty_like(big)
    t_copy = events(lambda: dst.copy_(big), steps=20, warmup=3)
    copy_bw = 2 * big.numel() / (t_copy['median_ms'] * 1e-3)
    del big, dst

    results = []
    for size in [int(s) for s in args.sizes.split(',')]:
        img, annot = synth_regions(size, size)
        slic = superpixels.segment_slic_img2d(img, 30, 0.2)
        del img
        H, W = slic.shape
        row = {'size': [H, W], 'superpixels': int(slic.max()) + 1}
        row['end_to_end'] = {
            'compute_boundary_distances': timed(lambda: lb.compute_boundary_distances(annot, slic)),
            'compute_distance_map': timed(lambda: lb.compute_distance_map(annot, 1)),
            'relabel_max_overlap_unique': timed(lambda: lb.relabel_max_overlap_unique(annot, slic, True)),
            'compute_labels_overlap_matrix': timed(lambda: lb.compute_labels_overlap_matrix(slic, annot)),
        }

        # device-resident legs
        d_slic = torch.from_numpy(slic.astype(np.int32)).cuda()
        d_annot = torch.from_numpy(annot.astype(np.int32)).cuda()
        m_a = torch.empty((H, W), dtype=torch.uint8, device='cuda')
        m_b = torch.empty_like(m_a)
        ws_e = lib.isb_edt_workspace_bytes(H, W)
        ws_edt = torch.empty(ws_e, dtype=torch.uint8, device='cuda')
        dist = torch.empty((H, W), dtype=torch.float64, device='cuda')
        ws_c = lib.isb_mask_compact_workspace_bytes(H, W)
        ws_cpt = torch.empty(ws_c, dtype=torch.uint8, device='cuda')
        total = torch.empty(1, dtype=torch.int64, device='cuda')
        P = len(lb.compute_boundary_distances(annot, slic)[1])
        pts = torch.empty((max(P, 1), 2), dtype=torch.int64, device='cuda')
        vals = torch.empty(max(P, 1), dtype=torch.float64, device='cuda')
        nb_s, nb_a = int(slic.max()) + 1, int(annot.max()) + 1
        hist = torch.empty((nb_s, nb_a), dtype=torch.int32, device='cuda')
        hist_t = torch.empty((nb_a, nb_s), dtype=torch.int32, device='cuda')
        lut = torch.arange(nb_s, dtype=torch.int32, device='cuda')
        out = torch.empty((H, W), dtype=torch.int32, device='cuda')
        p = _lib.ptr

        def dev_boundary():
            _lib.check(lib.isb_label_boundary_map(p(d_slic), H, W, p(m_a), st()))
            _lib.check(lib.isb_edt_2d(p(m_a), H, W, p(dist), p(ws_edt), C.c_size_t(ws_e), st()))
            _lib.check(lib.isb_label_boundary_map(p(d_annot), H, W, p(m_b), st()))
            _lib.check(lib.isb_mask_compact_count(p(m_b), H, W, p(ws_cpt), C.c_size_t(ws_c), p(total), st()))
            _lib.check(lib.isb_mask_compact_write(p(m_b), H, W, p(dist), p(ws_cpt), C.c_size_t(ws_c), p(pts), p(vals), st()))

        def dev_distance():
            _lib.check(lib.isb_label_contour_map(p(d_annot), H, W, 1, 0, p(m_a), st()))
            _lib.check(lib.isb_edt_2d(p(m_a), H, W, p(dist), p(ws_edt), C.c_size_t(ws_e), st()))

        def dev_overlap():
            _lib.check(lib.isb_region_label_hist(p(d_slic), p(d_annot), H, W, nb_s, nb_a, p(hist), st()))

        def dev_relabel():
            _lib.check(lib.isb_region_label_hist(p(d_annot), p(d_slic), H, W, nb_a, nb_s, p(hist_t), st()))
            _lib.check(lib.isb_relabel_gather(p(d_slic), C.c_longlong(H * W), p(lut), nb_s, p(out), st()))

        row['device_events'] = {'compute_boundary_distances': events(dev_boundary), 'compute_distance_map': events(dev_distance),
                                'relabel_max_overlap_unique': events(dev_relabel), 'compute_labels_overlap_matrix': events(dev_overlap),
                                'edt_of_the_slic_boundary': events(lambda: _lib.check(lib.isb_edt_2d(p(m_a), H, W, p(dist), p(ws_edt),
                                                                                                      C.c_size_t(ws_e), st())))}

        # EDT phases (profiler run of its own)
        _lib.check(lib.isb_label_boundary_map(p(d_slic), H, W, p(m_a), st()))
        from torch.profiler import ProfilerActivity, profile
        n_prof = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                _lib.check(lib.isb_edt_2d(p(m_a), H, W, p(dist), p(ws_edt), C.c_size_t(ws_e), st()))
            torch.cuda.synchronize()
        per = {k: 0.0 for k in EDT_KERNELS}
        for e in prof.key_averages():
            for k in EDT_KERNELS:
                if k in e.key:
                    per[k] += e.device_time_total / n_prof * 1e-3       # us -> ms
        nbytes = edt_phase_bytes(H, W)
        row['edt_phases'] = {k: {'ms': per[k], 'bytes': nbytes[k], 'ms_at_copy_bandwidth': nbytes[k] / copy_bw * 1e3} for k in EDT_KERNELS}

        if size <= 2048:
            t0 = time.perf_counter()
            ol.compute_boundary_distances(annot, slic)
            t1 = time.perf_counter()
            ol.compute_distance_map(annot, 1)
            t2 = time.perf_counter()
            ol.relabel_max_overlap_unique(annot, slic, True)
            t3 = time.perf_counter()
            ol.compute_labels_overlap_matrix(slic, annot)
            t4 = time.perf_counter()
            row['oracle_host_ms'] = {'compute_boundary_distances': (t1 - t0) * 1e3, 'compute_distance_map': (t2 - t1) * 1e3,
                                     'relabel_max_overlap_unique': (t3 - t2) * 1e3, 'compute_labels_overlap_matrix': (t4 - t3) * 1e3}
        else:
            row['oracle_host_ms'] = 'not run: the literal per-pixel loops take minutes at this size'
        results.append(row)
        del d_slic, d_annot, m_a, m_b, ws_edt, dist, ws_cpt, pts, vals, hist, hist_t, out
        torch.cuda.empty_cache()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'bench': 'labeling', 'gpu': gpu, 'copy_bandwidth_GBps': copy_bw / 1e9, 'sizes': results}))


if __name__ == '__main__':
    main()
