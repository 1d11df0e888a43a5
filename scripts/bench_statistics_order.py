"""
How often two launches of the segment and gray statistics differ in their bits, and what the statistics stage costs.

- Reruns: ``isb_segment_stats_2d`` (mean, std, energy) on the benchmark image (2048x2048 f64, config 2, its SLIC labels) and
  ``isb_gray_stats`` on a 128^3 float32 volume of 8^3 supervoxels, ``--reruns`` times each; reports how many launches differ from
  the first in any byte and the share of differing values.
- Stage time: CUDA events around ``Engine.segment_stats`` on grid label maps of ~5 000 superpixels over 2048^2 and ~80 000 over
  8192^2 (f64 RGB), with the benchmark's statistics (mean + centroids) and with mean, std and energy.

``--lib PATH`` loads another build of libimsegm_b200.so (one with the same entry points for these two calls) to compare builds.
Prints one JSON line with the GPU name and power limit the numbers were taken on.

    python scripts/bench_statistics_order.py [--lib PATH] [--reruns 20] [--iters 20] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=None, help='another libimsegm_b200.so to load instead of the in-tree build')
    ap.add_argument('--reruns', type=int, default=20)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None, help='directory for the JSON result')
    args = ap.parse_args()
    import numpy as np
    import torch
    from pyimsegm_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    from bench import SP_REGUL, SP_SIZE, synth_image
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    assert torch.cuda.is_available(), 'needs a CUDA device'
    eng = get_engine()
    lib = _lib.lib()
    st = _lib.stream_ptr
    res = {'gpu': gpu_info(), 'lib': args.lib or 'in-tree'}

    # -- reruns ------------------------------------------------------------------------------------------------------------------
    img = synth_image(2)
    H, W = img.shape[:2]
    n_seg, compact = slic_params((H, W), SP_SIZE, SP_REGUL)
    d_img = torch.from_numpy(img).cuda()
    d_seg, _ = eng.slic(d_img, n_seg, compact, sigma=1.0)
    d_seg = d_seg.clone()
    nb = eng.slic_label_bound(H, W, n_seg)
    wsb = lib.isb_segment_stats_workspace_bytes(nb)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    feat = torch.empty((nb, 9), dtype=torch.float64, device='cuda')
    outs = []
    for _ in range(args.reruns):
        _lib.check(lib.isb_segment_stats_2d(_lib.ptr(d_img), 3, _lib.ptr(d_seg), H, W, nb, 7, _lib.ptr(feat), 9, 0, None, None,
                                            _lib.ptr(ws), C.c_size_t(wsb), st()))
        outs.append(feat.cpu().numpy().view(np.int64).copy())
    diff = [o != outs[0] for o in outs[1:]]
    res['image_reruns'] = {'launches': args.reruns, 'differing_launches': int(sum(d.any() for d in diff)),
                           'differing_value_share': float(np.mean([d.mean() for d in diff])), 'labels': int(nb)}
    rng = np.random.RandomState(0)
    shape = (128, 128, 128)
    vol = torch.from_numpy(rng.rand(*shape).astype(np.float32)).cuda()
    z, y, x = np.indices(shape) // 8
    vseg = torch.from_numpy(np.ascontiguousarray(((z * 16 + y) * 16 + x).astype(np.int32))).cuda()
    vnb = 16 ** 3
    gwsb = lib.isb_gray_stats_workspace_bytes(vnb)
    gws = torch.empty(gwsb, dtype=torch.uint8, device='cuda')
    gfeat = torch.empty((vnb, 3), dtype=torch.float64, device='cuda')
    outs = []
    for _ in range(args.reruns):
        _lib.check(lib.isb_gray_stats(_lib.ptr(vol), 2, _lib.ptr(vseg), C.c_longlong(vol.numel()), vnb, 7, _lib.ptr(gfeat), 3, 0,
                                      _lib.ptr(gws), C.c_size_t(gwsb), st()))
        outs.append(gfeat.cpu().numpy().view(np.int64).copy())
    diff = [o != outs[0] for o in outs[1:]]
    res['volume_reruns'] = {'launches': args.reruns, 'differing_launches': int(sum(d.any() for d in diff)),
                            'differing_value_share': float(np.mean([d.mean() for d in diff])), 'labels': vnb}

    # -- stage time --------------------------------------------------------------------------------------------------------------
    times = {}
    for side, step in ((2048, 29), (8192, 29)):
        g = (side + step - 1) // step
        yy, xx = np.mgrid[:side, :side] // step
        seg = torch.from_numpy(np.ascontiguousarray((yy * g + xx).astype(np.int32))).cuda()
        nbl = g * g
        im = torch.rand((side, side, 3), dtype=torch.float64, device='cuda')
        for name, flags, centres in (('mean+centres', ('mean', ), True), ('mean+std+energy', ('mean', 'std', 'energy'), False)):
            fn = lambda: eng.segment_stats(im, seg, nbl, flags, want_centres=centres)   # noqa: E731
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            times['%d^2 %d labels %s' % (side, nbl, name)] = round(t0.elapsed_time(t1) / args.iters, 4)
        del im, seg
        torch.cuda.empty_cache()
    res['stage_ms'] = times
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_statistics_order.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
