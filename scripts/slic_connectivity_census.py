"""
Census of the small pieces the SLIC connectivity pass merges on the benchmark image (CPU only, from the oracle).

The small-piece kernel of slic_connectivity.cu runs one thread per 4-connected piece below min_size, and the launch lasts as long
as the BFS of the largest one.  This prints the k-means map's piece count, the size histogram of the small pieces, and the BFS
steps (pixels dequeued) and levels of the largest small piece, replayed from its first pixel in raster order with the kernel's
neighbour order.

    python scripts/slic_connectivity_census.py [--seed 2] [--size 2048]
"""
import argparse
import collections
import os
import sys

import numpy as np
from scipy import ndimage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def bfs_levels(mask, start):
    """BFS over a boolean piece mask from `start` (+x, -x, +y, -y): (steps, levels)"""
    H, W = mask.shape
    level = {start: 0}
    q = collections.deque([start])
    steps = 0
    while q:
        y, x = q.popleft()
        steps += 1
        for ny, nx in ((y, x + 1), (y, x - 1), (y + 1, x), (y - 1, x)):
            if 0 <= ny < H and 0 <= nx < W and mask[ny, nx] and (ny, nx) not in level:
                level[(ny, nx)] = level[(y, x)] + 1
                q.append((ny, nx))
    return steps, max(level.values()) + 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seed', type=int, default=2)
    ap.add_argument('--size', type=int, default=2048)
    args = ap.parse_args()
    import oracle
    from bench import SP_REGUL, SP_SIZE, synth_image
    from pyimsegm_b200.superpixels import slic_params
    oracle.build()
    img = synth_image(args.seed, args.size, args.size)
    n_seg, compact = slic_params(img.shape[:2], SP_SIZE, SP_REGUL)
    lo, hi = img.min(), img.max()
    km = oracle.slic((img - lo) / (hi - lo), n_seg, compact, sigma=1, enforce_conn=False)
    seg = km.shape[0] * km.shape[1] / n_seg
    min_size, max_size = int(0.5 * seg), int(3 * seg)

    four = ndimage.generate_binary_structure(2, 1)
    sizes, small = [], []  # small: (size, first raster pixel, mask slice, mask)
    for lab, sl in enumerate(ndimage.find_objects(km + 1)):
        if sl is None:
            continue
        comp, n = ndimage.label(km[sl] == lab, structure=four)
        for c in range(1, n + 1):
            m = comp == c
            s = int(m.sum())
            sizes.append(s)
            if s < min_size:
                ys, xs = np.nonzero(m)
                first = np.lexsort((xs, ys))[0]
                small.append((s, (int(ys[first]), int(xs[first])), m))
    sizes = np.array(sizes)
    print('image %dx%d seed %d: %d seeds, min_size %d, max_size %d' % (args.size, args.size, args.seed, n_seg, min_size, max_size))
    print('components: %d, oversize (>= max_size): %d, largest %d, median %d'
          % (len(sizes), int((sizes >= max_size).sum()), int(sizes.max()), int(np.median(sizes))))
    ss = np.array([s for s, _, _ in small])
    print('small pieces (< min_size): %d with %d pixels, median size %d, largest %d'
          % (len(ss), int(ss.sum()), int(np.median(ss)), int(ss.max())))
    edges = [1, 2, 3, 5, 9, 17, 33, 65, 129, 257, min_size]
    hist, _ = np.histogram(ss, bins=edges)
    for a, b, h in zip(edges[:-1], edges[1:], hist):
        print('  size %4d-%-4d %5d' % (a, b - 1, h))
    by_levels = []
    for s, start, m in small:
        steps, levels = bfs_levels(m, (start[0], start[1]))
        assert steps == s
        by_levels.append((levels, s))
    s, start, m = max(small, key=lambda t: t[0])
    steps, levels = bfs_levels(m, start)
    print('largest small piece: %d px, %d BFS steps, %d BFS levels' % (s, steps, levels))
    lv, sz = max(by_levels)
    print('most BFS levels: %d (a %d px piece)' % (lv, sz))


if __name__ == '__main__':
    main()
