"""
Census of the SLIC assignment's pruning, counted on the CPU (no GPU needed).

Replays k_assign (pyimsegm_b200/csrc/slic_kmeans.cu) in numpy on the benchmark's image (bench.synth_image, 2048x2048, sp_size 29,
sp_regul 0.2) with the centres the oracle (oracle/slic_oracle.c) has before every sweep, and counts per sweep the (thread,
candidate) pairs that reach each stage of the loop.  A thread owns one column and 8 rows of a 32x32 tile; a pair is one thread and
one cluster whose window meets the thread's tile.

    candidates / tile      clusters in the tile's list
    visited                pairs before the nearest-first loop breaks (the sorted spatial bound exceeds every row's minimum)
    pass spatial           pairs whose float spatial bound does not reject them
    pass colour            of those, pairs that the float colour-box bound does not reject either
    fp64 spatial           pairs that reach the double spatial chain of 8 rows (window column test passed), without and
                           with the colour-box bound
    fp64 colour            4-row groups that reach the double colour chain, without and with the colour-box bound

The float operations are emulated in float32 (round to nearest) and the directed roundings of the colour bound by stepping to the
neighbouring float, so the counts are those of the kernel up to the order of candidates with equal keys, which the kernel takes in
list order.  As a check of the replay, the labels it computes must equal the oracle's after every sweep.  The script also counts
the tiles whose list would overflow the capacity the workspace reserves, at sp_size 29, 10 and 5.

    python scripts/slic_assign_census.py [--size 2048] [--sweeps 10]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE, AROWS = 32, 8
F = np.float32


def tile_cap(step_y, step_x):
    """the list capacity per tile that carve() in slic_kmeans.cu reserves"""
    return ((TILE + 4 * step_y + 2) // step_y + 2) * ((TILE + 4 * step_x + 2) // step_x + 2)


def windows(cent, alive, step_y, step_x, H, W):
    """make_window of slic_kmeans.cu: (y0, y1, x0, x1), empty for dead clusters"""
    cy, cx = cent[:, 0], cent[:, 1]
    y0 = np.maximum(cy - 2 * step_y, 0.0).astype(np.int64)
    y1 = np.minimum(cy + 2 * step_y + 1.0, float(H)).astype(np.int64)
    x0 = np.maximum(cx - 2 * step_x, 0.0).astype(np.int64)
    x1 = np.minimum(cx + 2 * step_x + 1.0, float(W)).astype(np.int64)
    w = np.stack([y0, y1, x0, x1], axis=1)
    w[~alive] = 0
    return w


def tile_pairs(win, H, W):
    """(tile, cluster) for every tile a window meets"""
    ntx = (W + TILE - 1) // TILE
    ok = (win[:, 1] > win[:, 0]) & (win[:, 3] > win[:, 2])
    k = np.nonzero(ok)[0]
    ty0, ty1 = win[k, 0] // TILE, (win[k, 1] - 1) // TILE
    tx0, tx1 = win[k, 2] // TILE, (win[k, 3] - 1) // TILE
    span = int(max((ty1 - ty0).max(), (tx1 - tx0).max())) + 1
    tiles, ks = [], []
    for dy in range(span):
        for dx in range(span):
            m = (ty0 + dy <= ty1) & (tx0 + dx <= tx1)
            tiles.append((ty0[m] + dy) * ntx + tx0[m] + dx)
            ks.append(k[m])
    return np.concatenate(tiles), np.concatenate(ks)


def round_down(x):
    f = x.astype(F)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, F(-np.inf)), f)


def round_up(x):
    f = x.astype(F)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, F(np.inf)), f)


def replay_sweep(lab, cent, alive, prev_labels, step_y, step_x, sw):
    """one k_assign launch; returns the labels and the counts"""
    H, W, _ = lab.shape
    nty, ntx = (H + TILE - 1) // TILE, (W + TILE - 1) // TILE
    win = windows(cent, alive, step_y, step_x, H, W)
    tiles, ks = tile_pairs(win, H, W)
    # nearest-first order of every tile's list: key = float distance of the centre to the tile centre
    ty, tx = tiles // ntx, tiles % ntx
    tcy = (F(0.5) * (ty * TILE + np.minimum(ty * TILE + TILE, H) - 1).astype(F)).astype(F)
    tcx = (F(0.5) * (tx * TILE + np.minimum(tx * TILE + TILE, W) - 1).astype(F)).astype(F)
    fy, fx = cent[ks, 0].astype(F) - tcy, cent[ks, 1].astype(F) - tcx
    key = fy * fy + fx * fx
    o = np.lexsort((ks, key, tiles))
    tiles, ks, key = tiles[o], ks[o], key[o]
    nc = np.bincount(tiles, minlength=nty * ntx)
    first = np.concatenate([[0], np.cumsum(nc)[:-1]])
    rank = np.arange(len(tiles)) - first[tiles]
    maxnc = int(nc.max())
    order = np.full((nty * ntx, maxnc), -1, np.int64)
    order[tiles, rank] = ks
    r = np.sqrt(key) - F(23.5)
    lbv = np.where(r > 0, (r * r * F(0.999)).astype(np.float64) * sw * 0.999, 0.0)
    lb = np.full((nty * ntx, maxnc), np.inf)
    lb[tiles, rank] = lbv

    # threads: (row block of 8, column)
    nrb = (H + AROWS - 1) // AROWS
    rb, x = np.meshgrid(np.arange(nrb), np.arange(W), indexing='ij')
    rb, x = rb.ravel(), x.ravel()
    tid = (rb * AROWS // TILE) * ntx + x // TILE
    T = len(x)
    ys = rb[:, None] * AROWS + np.arange(AROWS)[None, :]            # [T, 8]
    yin = ys < H
    yc = np.minimum(ys, H - 1)
    px = lab[yc, x[:, None], :]                                     # [T, 8, 3]
    # the thread's colour box, rounded outwards (rows inside the image)
    plo = np.where(yin[:, :, None], round_down(px), F(np.inf)).min(axis=1)
    phi = np.where(yin[:, :, None], round_up(px), F(-np.inf)).max(axis=1)
    clo, chi = round_down(cent[:, 2:5]), round_up(cent[:, 2:5])
    cyf, cxf = cent[:, 0].astype(F), cent[:, 1].astype(F)
    xf = x.astype(F)
    ymid = (rb * AROWS).astype(F) + F(0.5 * (AROWS - 1))
    swf = F(sw) * F(0.998)

    best = np.full((T, AROWS), np.finfo(np.float64).max)
    bestk = np.full((T, AROWS), -1, np.int64)
    worst = np.full(T, np.finfo(np.float64).max)
    live = np.ones(T, bool)
    c = dict.fromkeys(('visited', 'pass_spatial', 'pass_colour', 'fp64_spatial', 'fp64_spatial_box', 'fp64_colour_groups',
                       'fp64_colour_groups_box'), 0)
    for ci in range(maxnc):
        k = order[tid, ci]
        live &= (k >= 0) & ~(lb[tid, ci] > worst)
        if not live.any():
            break
        i = np.nonzero(live)[0]
        k = k[i]
        c['visited'] += len(i)
        worstf = round_up(worst[i])
        ax = np.maximum(np.abs(cxf[k] - xf[i]) - F(2e-3), F(0))
        ay = np.maximum(np.abs(cyf[k] - ymid[i]) - F(0.5 * (AROWS - 1) + 2e-3), F(0))
        lbs = (ax * ax + ay * ay) * swf
        sp_ok = ~(lbs > worstf)
        g = np.maximum(np.maximum(round_down(plo[i].astype(np.float64) - chi[k]), round_down(clo[k].astype(np.float64) - phi[i])), F(0))
        gg = round_down(g.astype(np.float64) * g)
        lbc = round_down(round_down(gg[:, 0].astype(np.float64) + gg[:, 1]).astype(np.float64) + gg[:, 2])
        col_ok = ~(round_down(lbc.astype(np.float64) * np.float64(F(0.998)) + lbs) > worstf)
        xin = (x[i] >= win[k, 2]) & (x[i] < win[k, 3])
        c['pass_spatial'] += int(sp_ok.sum())
        c['pass_colour'] += int((sp_ok & col_ok).sum())
        ev = sp_ok & xin
        c['fp64_spatial'] += int(ev.sum())
        c['fp64_spatial_box'] += int((ev & col_ok).sum())
        if not ev.any():
            continue
        e = i[ev]
        ke = k[ev]
        y = ys[e]
        ty_ = cent[ke, 0][:, None] - y
        tx_ = cent[ke, 1] - x[e]
        sp = (ty_ * ty_ + (tx_ * tx_)[:, None]) * sw
        inwin = (y >= win[ke, 0][:, None]) & (y < win[ke, 1][:, None])
        need = inwin & ~(sp > best[e])
        grp = need.reshape(len(e), 2, 4).any(axis=2)
        c['fp64_colour_groups'] += int(grp.sum())
        c['fp64_colour_groups_box'] += int((grp & col_ok[ev][:, None]).sum())
        d = px[e] - cent[ke, 2:5][:, None, :]
        dcol = d[:, :, 0] * d[:, :, 0]
        dcol = dcol + d[:, :, 1] * d[:, :, 1]
        dcol = dcol + d[:, :, 2] * d[:, :, 2]
        dc = sp + dcol
        be, bk = best[e], bestk[e]
        win_ = need & np.repeat(grp, 4, axis=1) & ((dc < be) | ((dc == be) & (bk >= 0) & (ke[:, None] < bk)))
        best[e] = np.where(win_, dc, be)
        bestk[e] = np.where(win_, ke[:, None], bk)
        imp = win_.any(axis=1)
        if imp.any():
            ei = e[imp]
            worst[ei] = np.where(yin[ei], best[ei], 0.0).max(axis=1)
    labels = prev_labels.copy()
    got = bestk >= 0
    yy, xx = ys[got], np.broadcast_to(x[:, None], ys.shape)[got]
    labels[yy, xx] = bestk[got]
    return labels, c, nc


def overflow_census(oracle, img_lab, sp_size, sweeps):
    H, W, _ = img_lab.shape
    n_seg = int(H * W / sp_size ** 2)
    seeds, ty, tx = oracle.slic_seeds(H, W, n_seg)
    cap = tile_cap(ty, tx)
    rows = []
    for s in sweeps:
        if s == 0:
            cent, alive = np.concatenate([seeds, np.zeros((len(seeds), 3))], axis=1), np.ones(len(seeds), bool)
        else:
            lbl, cent = oracle.slic_kmeans(img_lab, n_seg, max_iter=s, return_centroids=True)
            alive = np.bincount(lbl.ravel(), minlength=len(seeds)) > 0
        tiles, _ = tile_pairs(windows(cent, alive, ty, tx, H, W), H, W)
        cnt = np.bincount(tiles)
        rows.append((s, int(cnt.max()), float(cnt.mean()), int((cnt > cap).sum())))
    return len(seeds), ty, tx, cap, rows


def main():
    np.seterr(over='ignore')   # DBL_MAX (the initial minima) rounds up to +inf in float
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--size', type=int, default=2048)
    ap.add_argument('--sweeps', type=int, default=10)
    args = ap.parse_args()
    import bench
    import oracle
    oracle.build()
    sp_size, regul = bench.SP_SIZE, bench.SP_REGUL
    img = bench.synth_image(2, h=args.size, w=args.size)
    lo, hi = img.min(), img.max()
    if lo != 0. or hi != 1.:
        img = (img - lo) / float(hi - lo)

    def lab_for(sp):
        return oracle.rgb2lab_scaled(oracle.gaussian_blur(img, 1.0), 1.0 / (sp * regul) ** 1.5)

    lab = lab_for(sp_size)
    H, W, _ = lab.shape
    n_seg = int(H * W / sp_size ** 2)
    seeds, ty, tx = oracle.slic_seeds(H, W, n_seg)
    n = len(seeds)
    sw = 1.0 / float(max(1, ty, tx)) ** 2
    cent = np.concatenate([seeds, np.zeros((n, 3))], axis=1)
    alive = np.ones(n, bool)
    labels = np.zeros((H, W), np.int64)
    print('image %dx%d, sp_size %d, %d clusters, tile capacity %d' % (H, W, sp_size, n, tile_cap(ty, tx)))
    hdr = ('sweep', 'cand/tile', 'visited', 'pass sp', 'pass col', 'fp64 sp', 'fp64 sp+box', 'col grp', 'col grp+box')
    print(('%5s' + ' %11s' * (len(hdr) - 1)) % hdr)
    tot = None
    for s in range(args.sweeps):
        labels, c, nc = replay_sweep(lab, cent, alive, labels, ty, tx, sw)
        want, cent = oracle.slic_kmeans(lab, n_seg, max_iter=s + 1, return_centroids=True)
        assert np.array_equal(labels, want), 'the replay differs from the oracle in sweep %d' % s
        alive &= np.bincount(want.ravel(), minlength=n) > 0
        vals = [c[k] for k in ('visited', 'pass_spatial', 'pass_colour', 'fp64_spatial', 'fp64_spatial_box', 'fp64_colour_groups',
                               'fp64_colour_groups_box')]
        tot = vals if tot is None else [a + b for a, b in zip(tot, vals)]
        print(('%5d %11.1f' + ' %11d' * len(vals)) % ((s, nc[nc > 0].mean()) + tuple(vals)))
    print(('%5s %11s' + ' %11d' * len(tot)) % (('all', '') + tuple(tot)))
    print('colour-box bound: fp64 spatial chains %.1f %% of before, fp64 colour groups %.1f %% of before'
          % (100.0 * tot[4] / max(tot[3], 1), 100.0 * tot[6] / max(tot[5], 1)))
    for sp in (29, 10, 5):
        n_sp, ty_, tx_, cap, rows = overflow_census(oracle, lab_for(sp), sp, (0, 1, 2, 5, 9))
        print('sp_size %d (%d clusters, step %d): tile capacity %d' % (sp, n_sp, max(ty_, tx_), cap))
        for s, mx, mean, over in rows:
            print('    before sweep %d: list length mean %.1f, max %d, overflowed tiles %d' % (s, mean, mx, over))


if __name__ == '__main__':
    main()
