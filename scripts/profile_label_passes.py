"""
Per-kernel GPU times of the three label-map passes that follow SLIC on the benchmark image (2048x2048 f64, sp_size 29): segment
statistics (colour means and centroids, as the benchmark asks for them), the adjacency scan and the final gathers (segm and a K = 3
segm_soft).  Kernel times come from torch.profiler (CUDA activity) in a run of their own, call times (memsets and launch gaps
included) from CUDA events around each call in a separate loop.  GB/s is the bytes each pass must move over its time:

    segment_stats  f64 RGB 24 B/px + label 4 B/px
    adjacency      label 4 B/px
    gather         label 4 + segm 4 + segm_soft 24 B/px

Prints one JSON line with the GPU name and power limit the numbers were taken on.

    python scripts/profile_label_passes.py [--iters 50] [--out DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PASSES = {'segment_stats': ('k_stats_pass1', 'k_stats_finalize'),
          'adjacency': ('k_edge_scan', 'k_edge_offsets', 'k_edge_fill', 'k_edge_emit'),
          'gather': ('k_gather', )}
BYTES_PER_PX = {'segment_stats': 28, 'adjacency': 4, 'gather': 32}


def kernel_key(name):
    """the project's kernel name inside a (demangled) CUDA kernel name, or 'memset'"""
    if 'memset' in name.lower():
        return 'memset'
    kernels = [k for ks in PASSES.values() for k in ks]
    for m in re.finditer(r'(k_\w+)\s*[<(]', name):
        if m.group(1) in kernels:
            return m.group(1)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--out', default=None, help='directory for the JSON result')
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import SP_REGUL, SP_SIZE, synth_image
    from pyimsegm_b200.engine import edge_capacity, get_engine
    from pyimsegm_b200.superpixels import slic_params
    assert torch.cuda.is_available(), 'needs a CUDA device'
    eng = get_engine()
    img = synth_image(2)
    H, W = img.shape[:2]
    n_seg, compact = slic_params((H, W), SP_SIZE, SP_REGUL)
    d_img = torch.from_numpy(img).cuda()
    d_seg, d_n = eng.slic(d_img, n_seg, compact, sigma=1.0)
    d_seg = d_seg.clone()
    nb = eng.slic_label_bound(H, W, n_seg)
    cap = edge_capacity(nb)
    rng = np.random.RandomState(0)
    lut_i = eng.to_device(rng.randint(0, 3, nb).astype(np.int32))
    lut_p = eng.to_device(rng.rand(nb, 3))
    calls = {'segment_stats': lambda: eng.segment_stats(d_img, d_seg, nb, ('mean', ), want_centres=True),
             'adjacency': lambda: eng.adjacency(d_seg, nb, cap),
             'gather': lambda: eng.gather(d_seg, lut_i, lut_p)}
    for fn in calls.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()

    call_us = {}
    for name, fn in calls.items():
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            fn()
        t1.record()
        torch.cuda.synchronize()
        call_us[name] = t0.elapsed_time(t1) * 1e3 / args.iters

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, fn in calls.items():
            for _ in range(args.iters):
                fn()
            torch.cuda.synchronize()
    us = {name: {} for name in calls}
    owner = {k: name for name, ks in PASSES.items() for k in ks}
    memset_us = []
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernel_key(ev.name)
        if k == 'memset':
            memset_us.append(ev.time_range.elapsed_us())
        elif k is not None:
            d = us[owner[k]]
            d[k] = d.get(k, 0.0) + ev.time_range.elapsed_us() / args.iters
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True)
    npx = H * W
    res = {'gpu': smi.stdout.strip(), 'iters': args.iters, 'image': [H, W], 'labels': int(eng.to_host(d_n)[0]), 'passes': {}}
    for name in calls:
        kern = sum(us[name].values())
        res['passes'][name] = {'kernels_us': {k: round(v, 2) for k, v in us[name].items()}, 'kernels_total_us': round(kern, 2),
                               'call_us': round(call_us[name], 2), 'bytes': BYTES_PER_PX[name] * npx,
                               'kernel_GBps': round(BYTES_PER_PX[name] * npx / kern / 1e3, 1) if kern else None,
                               'call_GBps': round(BYTES_PER_PX[name] * npx / call_us[name] / 1e3, 1)}
    res['memsets_per_iter'] = round(len(memset_us) / args.iters, 2)
    res['memset_us_per_iter'] = round(sum(memset_us) / args.iters, 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'label_passes_profile.json'), 'a') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
