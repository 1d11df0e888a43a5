"""
Per-kernel GPU times of the SLIC pre-pass (k_minmax, k_blur_lab) and of every connectivity kernel on the benchmark image, from
torch.profiler (CUDA activity) over a run of its own.  Prints one JSON line: microseconds per image for each kernel, with the
GPU name and power limit the numbers were taken on.

    python scripts/profile_slic_prepare_connectivity.py [--iters 20] [--out DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ('k_minmax', 'k_minmax_decode', 'k_blur_lab', 'k_ccl_tile', 'k_ccl_seams', 'k_ccl_roots', 'k_ccl_classify',
           'k_ccl_flatten', 'k_oversize_split', 'k_kept_ranks', 'k_small_window', 'k_small_adjacent', 'k_ccl_write')


def kernel_key(name):
    """the project's kernel name inside a (demangled) CUDA kernel name, template arguments dropped"""
    for m in re.finditer(r'(k_\w+)\s*[<(]', name):
        if m.group(1) in KERNELS:
            return m.group(1)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None, help='directory for the JSON result')
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import SP_REGUL, SP_SIZE, synth_image
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    assert torch.cuda.is_available(), 'needs a CUDA device'
    eng = get_engine()
    img = synth_image(2)
    n_seg, compact = slic_params(img.shape[:2], SP_SIZE, SP_REGUL)
    d_img = torch.from_numpy(img).cuda()
    for _ in range(3):
        eng.slic(d_img, n_seg, compact, sigma=1.0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            eng.slic(d_img, n_seg, compact, sigma=1.0)
        torch.cuda.synchronize()
    us = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernel_key(ev.name)
        if k is not None:
            us[k] = us.get(k, 0.0) + ev.time_range.elapsed_us() / args.iters
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    res = {'gpu': smi.stdout.strip(), 'iters': args.iters, 'us_per_image': {k: round(us[k], 2) for k in KERNELS if k in us},
           'slic_prepare_us': round(sum(us.get(k, 0.0) for k in KERNELS[:3]), 2),
           'slic_connectivity_us': round(sum(v for k, v in us.items() if k not in KERNELS[:3]), 2)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'slic_prepare_connectivity_profile.json'), 'a') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
