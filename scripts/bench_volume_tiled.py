#!/usr/bin/env python
"""
bench_volume_tiled.py -- one large gray volume through the z-slab pipeline (tiled.pipe_gray3d_slic_features_model_graphcut_tiled)
and through segment_resident_volume.  Prints one JSON line (from rank 0 under torchrun).

    python scripts/bench_volume_tiled.py [--steps K] [--warmup W] [--depth D] [--size S] [--bands 1,2]
    torchrun --nproc-per-node=N scripts/bench_volume_tiled.py ...      # one slab per GPU (--bands 1)

Input: one seeded synthetic uint16 volume of D x S x S (default 256 x 1024 x 1024, a microscopy-sized stack: two intensity
classes in blocks, a z step and gaussian noise), spacing (12, 1, 1), sp_size 15, sp_regul 0.2, {'color': ['mean', 'std', 'energy']},
2 classes fitted on the device, gc_regul 0.1.  Legs, each the median and the min-max over steps:
- ``resident`` (single process only): segment_resident_volume on the volume already on the device, results left there;
- ``slabs_bpr<n>``: the slab pipeline with ``n`` slabs per GPU, host volume in, the owned slices' labels out (no segm_soft: at K = 2
  it is 16 bytes per voxel of host traffic), timed end to end; with its ms per stage, each timed to a device synchronise in a
  separate pass that runs the stages one after the other as the pipeline does: upload (the raw slabs), prepare (blur), sweeps (10,
  with their exchanges), broadcast (the owned slices of the label volume to every rank), connectivity, statistics, model
  (scaler + mixture fit), cut (graph + energies + alpha-expansion), gather (LUT gather of the owned slices + download).
Peak device memory per rank (torch's allocator) per leg.  Parity: the share of voxels on which each slab leg agrees with
``resident`` (single process) and whether the slab label volume equals the single-GPU one.  The card's name and power limit are
read in the same run.
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
    out = np.empty((depth, size, size), dtype=np.uint16)
    yy, xx = np.ogrid[:size, :size]
    cell = max(size // 8, 1)
    base = ((yy // cell + xx // cell) % 2).astype(np.float32)
    for z in range(depth):          # slice by slice: the float temporaries of the whole volume would not fit a small host
        sl = 0.3 + 0.35 * (base if z <= depth // 2 else 1 - base) + rng.normal(0, 0.1, (size, size)).astype(np.float32)
        out[z] = (np.clip(sl, 0, 1) * 65535).astype(np.uint16)
    return out


def stats(ts):
    return {'median_ms': float(np.median(ts)) * 1e3, 'min_ms': float(np.min(ts)) * 1e3, 'max_ms': float(np.max(ts)) * 1e3}


def stage_times(vol, comm, bpr, eng, torch):
    """the slab pipeline's stages one after the other, each timed to a device synchronise (ms)"""
    from pyimsegm_b200 import graph_cuts, tiled
    from pyimsegm_b200.engine import edge_capacity
    from pyimsegm_b200.pipelines import _volume_flags
    from pyimsegm_b200.superpixels import slic3d_params
    flags = _volume_flags(FEATURES)
    n_seg, compact = slic3d_params(vol.shape, SP_SIZE, SP_REGUL, SPACING)
    D, H, W = vol.shape
    out = {}

    def tick(name, t0):
        torch.cuda.synchronize()
        out[name] = out.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
        return time.perf_counter()

    bands, _, _, _ = tiled.slab_plan(vol.shape, n_seg, SPACING, comm.world * bpr)
    local = range(comm.rank * bpr, (comm.rank + 1) * bpr)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for i, b in enumerate(local):
        eng.to_device(vol[bands[b].raw_lo:bands[b].raw_hi], 'ts%d_raw' % i)
    t = tick('upload', t)
    res = tiled.slic3d_tiled(vol, n_seg, compact, SPACING, max_iter=0, comm=comm, bands_per_rank=bpr, eng=eng, enforce_connectivity=False)
    t = tick('upload+prepare', t)
    res = tiled.slic3d_tiled(vol, n_seg, compact, SPACING, comm=comm, bands_per_rank=bpr, eng=eng, enforce_connectivity=False)
    t = tick('upload+prepare+sweeps+broadcast', t)
    full = res.d_seg
    for bd in bands:
        comm.broadcast(full[bd.own_lo:bd.own_hi], bd.index // bpr)
    t = tick('broadcast', t)
    res.d_seg, res.d_n_labels = eng.enforce_connectivity3d(full, n_seg)
    res.nb_bound = eng.slic_label_bound(D * H * W, 1, n_seg)
    t = tick('connectivity', t)
    feat = tiled.gray_stats_tiled(res, vol.dtype, flags, comm=comm, eng=eng)
    t = tick('statistics', t)
    d_x = eng.standard_scaler(feat, res.d_n_labels)[0]
    kind, n_init, n_iter = graph_cuts.class_model_spec('GMM', NB_CLASSES, 99)
    d_proba = graph_cuts.device_fit_predict(eng, d_x, NB_CLASSES, True, kind, n_init, n_iter, None, d_n=res.d_n_labels)[0]
    t = tick('model', t)
    cap = edge_capacity(res.nb_bound, ndim=3)
    d_labels, _ = graph_cuts.device_graphcut(eng, res.d_seg, None, res.nb_bound, d_proba, GC_REGUL, 'model', res.d_n_labels, cap)
    t = tick('cut', t)
    lo, hi = bands[local[0]].own_lo, bands[local[-1]].own_hi
    d_segm, _ = eng.gather(res.d_seg[lo:hi], d_labels)
    eng.to_host(d_segm)
    tick('gather', t)
    out['prepare'] = out.pop('upload+prepare') - out['upload']
    out['sweeps'] = out.pop('upload+prepare+sweeps+broadcast') - out['upload'] - out['prepare']   # the copies of the owned slices too
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--depth', type=int, default=256)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--bands', default='1,2', help='slabs per GPU of the slab legs, comma separated')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_volume_tiled.py needs a CUDA device')
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200 import tiled
    from pyimsegm_b200.engine import get_engine
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
        dist.init_process_group('nccl')
        comm = tiled.GroupComm()
    else:
        comm = tiled.LoopbackComm()
    eng = get_engine()
    vol = synth_volume(7, args.depth, args.size)
    times, peaks, last, stages = {}, {}, {}, {}

    def timed(name, fn):
        ts = []
        torch.cuda.reset_peak_memory_stats()
        for step in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            if world > 1:
                torch.distributed.barrier()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            if step >= args.warmup:
                ts.append(time.perf_counter() - t0)
        times[name], peaks[name] = stats(ts), torch.cuda.max_memory_allocated() / 2 ** 30
        return out

    if world == 1:
        d_vol = torch.from_numpy(vol).cuda()
        model = pl._fit_model(NB_CLASSES, True)
        d_segm, _ = timed('resident', lambda: pl.segment_resident_volume(d_vol, model, FEATURES, SPACING, SP_SIZE, SP_REGUL, GC_REGUL))
        last['resident'] = d_segm.cpu().numpy()
        from pyimsegm_b200.superpixels import slic3d_params
        n_seg, compact = slic3d_params(vol.shape, SP_SIZE, SP_REGUL, SPACING)
        last['resident_slic'] = eng.to_host(eng.slic3d(d_vol, n_seg, compact, SPACING)[0]).copy()
        del d_vol
        eng._bufs.clear()
        torch.cuda.empty_cache()
    for bpr in [int(b) for b in args.bands.split(',')]:
        name = 'slabs_bpr%d' % bpr
        segm, _, rows = timed(name, lambda: tiled.pipe_gray3d_slic_features_model_graphcut_tiled(
            vol, NB_CLASSES, FEATURES, SPACING, SP_SIZE, SP_REGUL, GC_REGUL, comm=comm, bands_per_rank=bpr, want_soft=False))
        last[name] = (segm, rows)
        if world == 1:
            last[name + '_slic'] = eng.to_host(eng.buf('labels3d', vol.shape, torch.int32)).copy()
        stages[name] = [stage_times(vol, comm, bpr, eng, torch) for _ in range(args.steps)]
        stages[name] = {k: float(np.median([s[k] for s in stages[name]])) for k in stages[name][0]}
        eng._bufs.clear()
        torch.cuda.empty_cache()
    parity = {}
    if world == 1:
        for name in [k for k in last if k.startswith('slabs_') and not k.endswith('_slic')]:
            segm, (lo, hi) = last[name]
            parity[name] = {'voxel_agreement_with_resident': float(np.mean(segm == last['resident'][lo:hi])),
                            'label_volume_equal': bool(np.array_equal(last[name + '_slic'], last['resident_slic']))}
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    rank = comm.rank
    result = {
        'benchmark': 'one gray volume over z-slabs, ms per volume',
        'gpu': gpu[torch.cuda.current_device()] if gpu else 'unknown', 'world': world,
        'shape': list(vol.shape), 'dtype': 'uint16', 'spacing': list(SPACING), 'sp_size': SP_SIZE, 'features': FEATURES,
        'nb_classes': NB_CLASSES, 'gc_regul': GC_REGUL, 'steps': args.steps,
        'legs': times, 'stages_ms': stages, 'peak_device_gib_rank%d' % rank: peaks, 'parity': parity,
    }
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
    if rank == 0:
        print(json.dumps(result))


if __name__ == '__main__':
    main()
