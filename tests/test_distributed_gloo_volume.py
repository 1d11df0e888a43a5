"""
z-slab mode of one gray volume (pyimsegm_b200/tiled.py: slic3d_tiled) on CPU: the exchange protocol with a world-size-2 gloo group.
The slab worker below is a numpy stand-in for the ``isb_slic3d_slab_*`` kernels (same ownership rule, same halo, same 5-word
exchange record of int64 bit patterns), merged by the REAL communicator class; the label volume must be the oracle's whole-volume
k-means, bit for bit.
"""
import os
import sys

import numpy as np
import pytest

from test_distributed_gloo import _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _numpy_slab_sweeps(vol, seeds, steps, step, spacing, slab, halo, comm, max_iter=10):
    """the sweeps of oracle_slic_kmeans3d restricted to the k-means slab [km_lo, km_hi): every alive cluster whose window meets the
    slab assigns its part of the window (strict '<' in cluster order, the oracle's operation order), the owner of a cluster's centre
    slice sums its members in raster order, the records are summed as int64 over the ranks"""
    import torch
    D, H, W = vol.shape
    tz, ty, tx = steps
    sz, sy, sx = spacing
    n = len(seeds)
    cen = np.zeros((n, 4))
    cen[:, :3] = seeds
    alive = np.ones(n, dtype=bool)
    lo, hi = slab.km_lo, slab.km_hi
    labels = np.zeros((hi - lo, H, W), dtype=np.int64)
    sw = 1.0 / (step * step)
    zs = np.arange(lo, hi, dtype=np.float64)[:, None, None]
    ys = np.arange(H, dtype=np.float64)[None, :, None]
    xs = np.arange(W, dtype=np.float64)[None, None, :]
    part = vol[lo:hi]
    for _ in range(max_iter):
        dist = np.full((hi - lo, H, W), np.finfo(np.float64).max)
        for k in range(n):
            if not alive[k]:
                continue
            cz, cy, cx, cv = cen[k]
            z0, z1 = int(max(cz - 2 * tz, 0)), int(min(cz + 2 * tz + 1, D))
            y0, y1 = int(max(cy - 2 * ty, 0)), int(min(cy + 2 * ty + 1, H))
            x0, x1 = int(max(cx - 2 * tx, 0)), int(min(cx + 2 * tx + 1, W))
            a, b = max(z0, lo) - lo, min(z1, hi) - lo
            if a >= b:
                continue
            t_z = sz * (cz - zs[a:b])
            t_y = sy * (cy - ys[:, y0:y1])
            t_x = sx * (cx - xs[:, :, x0:x1])
            dc = ((t_z * t_z + t_y * t_y) + t_x * t_x) * sw
            d0 = part[a:b, y0:y1, x0:x1] - cv
            dc = dc + d0 * d0
            take = dist[a:b, y0:y1, x0:x1] > dc
            dist[a:b, y0:y1, x0:x1][take] = dc[take]
            labels[a:b, y0:y1, x0:x1][take] = k
        xchg = np.zeros((n, 5), dtype=np.int64)
        for k in range(n):
            if not alive[k] or not (slab.own_lo <= int(cen[k, 0]) < slab.own_hi):
                continue
            zz, yy, xx = np.nonzero(labels == k)                # raster order
            if len(zz) == 0:
                continue                                         # died: the record stays zero
            assert (zz + lo).min() >= int(cen[k, 0]) - halo and (zz + lo).max() <= int(cen[k, 0]) + halo
            sums = [float((zz + lo).sum()), float(yy.sum()), float(xx.sum()), np.cumsum(part[zz, yy, xx])[-1]]  # cumsum: in order
            xchg[k, :4] = (np.array(sums) / float(len(zz))).view(np.int64)
            xchg[k, 4] = 1
        t = torch.from_numpy(xchg)
        comm.all_reduce(t, 'sum')
        for k in range(n):
            if xchg[k, 4] == 1:
                cen[k] = xchg[k, :4].view(np.float64)
            else:
                alive[k] = False
    return labels[slab.own_lo - lo:slab.own_hi - lo]


def _slab_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    import oracle as orc
    from pyimsegm_b200.tiled import GroupComm, slab_plan
    comm = GroupComm()
    rng = np.random.RandomState(7)
    for shape, n_seg, compact, spacing in (((15, 22, 20), 24, 5, (2., 1., 1.)), ((13, 18, 16), 12, 3, (1., 1., 1.))):
        zz, yy, xx = np.mgrid[:shape[0], :shape[1], :shape[2]]
        vol = np.clip(0.3 + 0.4 * ((xx > shape[2] // 2) ^ (zz > shape[0] // 3)) + rng.normal(0, 0.1, shape), 0, 1)
        want = orc.slic3d(vol, n_seg, compact, spacing, enforce_conn=False)
        blurred = orc.gaussian_blur3d(vol, np.ones(3) / np.asarray(spacing))
        scaled = np.ascontiguousarray(blurred * (1.0 / compact))
        slabs, seeds, steps, _ = slab_plan(shape, n_seg, spacing, world)
        halo = 2 * steps[0] + 1
        slab = slabs[rank]
        got = _numpy_slab_sweeps(scaled, seeds, steps, float(max(steps)), spacing, slab, halo, comm)
        assert np.array_equal(got, want[slab.own_lo:slab.own_hi]), 'rank %d %r' % (rank, shape)
        np.save(os.path.join(out_dir, 'slab_%d_%d.npy' % (shape[0], rank)), got)
    dist.barrier()
    dist.destroy_process_group()


def test_slab_exchange_world2(tmp_path, oracle):
    import torch.multiprocessing as mp
    mp.spawn(_slab_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    for D in (15, 13):
        assert np.load(tmp_path / ('slab_%d_0.npy' % D)).shape[0] + np.load(tmp_path / ('slab_%d_1.npy' % D)).shape[0] == D
