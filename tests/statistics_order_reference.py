"""numpy restatement of the order in which the per-segment statistics are added, for bit-for-bit comparison with the device.

Colour statistics (``isb_segment_stats_2d`` and the banded ``_accumulate / _deviation``, csrc/segment_stats.cu):
  1. a lane owns one column of a 16-row strip and sums its pixels' float32 terms in float64, in row order, while the label holds;
  2. in a row where runs end, the runs of neighbouring lanes of one warp (32 columns from a multiple of 32) with one label are summed
     by ``seg_sum``: five shuffle-down steps, lane i adding lane i + o (o = 1, 2, 4, 8, 16) while i + o is inside its segment;
  3. each label's total is the correctly rounded sum of those flushed partials (csrc/exact_sum.cuh), which ``math.fsum`` gives; a
     NaN partial, or infinities of both signs, give NaN, one sign of infinity that infinity.
Gray statistics (``isb_gray_stats`` and its banded entries, csrc/native_misc.cu): a thread sums the runs of 16 consecutive voxels
in row order; every run is one partial, then step 3.
A banded call rounds its band's totals and adds them into the caller's accumulator with one float64 add.
"""
import math

import numpy as np

SROWS = 16
GSTRIP = 16
DBL_MAX = np.finfo(np.float64).max


def f32_terms(values):
    """the kernels' load: float32 with NaN as 0 (infinities stay)"""
    v = np.asarray(values).astype(np.float32)
    return np.where(np.isnan(v), np.float32(0), v)


def exact_total(parts):
    """the correctly rounded float64 sum of ``parts`` as the device forms it (+0 for none)"""
    parts = np.asarray(parts, dtype=np.float64)
    if np.isnan(parts).any():
        return np.nan
    pinf, ninf = np.isposinf(parts).any(), np.isneginf(parts).any()
    if pinf and ninf:
        return np.nan
    if pinf or ninf:
        return np.inf if pinf else -np.inf
    return 0.0 + math.fsum(parts.tolist())


def label_totals(labels, parts, nb):
    """[nb, K] exact totals of the partials parts [n, K] grouped by labels [n]"""
    K = parts.shape[1]
    out = np.zeros((nb, K))
    if len(labels) == 0:
        return out
    order = np.argsort(labels, kind='stable')
    lab, par = labels[order], parts[order]
    starts = np.flatnonzero(np.r_[True, lab[1:] != lab[:-1]])
    ends = np.r_[starts[1:], len(lab)]
    single = ends - starts == 1
    out[lab[starts[single]]] = 0.0 + par[starts[single]]
    for s, e in zip(starts[~single], ends[~single]):
        for k in range(K):
            out[lab[s], k] = exact_total(par[s:e, k])
    return out


def _seg_sum(vals, flush, key):
    """the head lanes and their segment sums of one row: vals [..., 32, K], flush / key [..., 32]"""
    lane = np.arange(32)
    prev_fl = np.concatenate([np.zeros_like(flush[..., :1]), flush[..., :-1]], axis=-1)
    prev_key = np.concatenate([key[..., :1], key[..., :-1]], axis=-1)
    head = flush & ~((lane > 0) & prev_fl & (prev_key == key))
    start = ~flush | head
    # end[i] = the first lane above i that starts a segment, 32 when none does
    idx = np.where(start, lane, 32)
    nxt = np.minimum.accumulate(idx[..., ::-1], axis=-1)[..., ::-1]
    end = np.concatenate([nxt[..., 1:], np.full_like(nxt[..., :1], 32)], axis=-1)
    v = vals.copy()
    for o in (1, 2, 4, 8, 16):
        u = np.concatenate([v[..., o:, :], v[..., 32 - o:, :]], axis=-2)   # shfl_down: lanes past 31 read their own value
        v = np.where(((lane + o) < end)[..., None], v + u, v)
    return head, v


def colour_partials(terms, seg, chunk_strips=16):
    """the flushed partials of one image (or band): terms [H, W, K] float64, seg [H, W] -> (labels [n], partials [n, K])"""
    H, W, K = terms.shape
    Wp = (W + 31) // 32 * 32
    S = (H + SROWS - 1) // SROWS
    labs, parts = [], []
    with np.errstate(invalid='ignore', over='ignore'):
        for s0 in range(0, S, chunk_strips):
            s1 = min(S, s0 + chunk_strips)
            rows = slice(s0 * SROWS, min(H, s1 * SROWS))
            n = s1 - s0
            sg = np.full((n * SROWS, Wp), -1, np.int64)
            tm = np.zeros((n * SROWS, Wp, K))
            sg[:rows.stop - rows.start, :W] = seg[rows]
            tm[:rows.stop - rows.start, :W] = terms[rows]
            sg = sg.reshape(n, SROWS, Wp)
            tm = tm.reshape(n, SROWS, Wp, K)
            cur = np.full((n, Wp), -1, np.int64)
            acc = np.zeros((n, Wp, K))
            for r in range(SROWS + 1):
                lab = sg[:, r] if r < SROWS else np.full((n, Wp), -1, np.int64)
                flush = (cur >= 0) & (lab != cur)
                if flush.any():
                    head, v = _seg_sum(acc.reshape(n, Wp // 32, 32, K), flush.reshape(n, -1, 32), cur.reshape(n, -1, 32))
                    labs.append(cur.reshape(n, -1, 32)[head])
                    parts.append(v[head])
                change = lab != cur
                cur = np.where(change, lab, cur)
                acc = np.where(change[..., None], 0.0, acc)
                if r < SROWS:
                    acc = np.where((lab >= 0)[..., None], acc + tm[:, r], acc)
    if not labs:
        return np.zeros(0, np.int64), np.zeros((0, K))
    return np.concatenate(labs), np.concatenate(parts)


def _tidy(v):
    v = np.where(np.isnan(v), 0.0, v)
    v = np.clip(v, -DBL_MAX, DBL_MAX)
    return v + 0.0


def colour_stats(img, seg, nb, bands=None):
    """(mean, std, energy [nb, 3], centres [nb, 2], counts [nb]) as the device computes them, whole image (bands None) or over row
    bands [(lo, hi), ...] accumulated in that order"""
    H, W = seg.shape
    bands = bands or [(0, H)]
    v = f32_terms(img).reshape(H, W, 3)
    seg = np.asarray(seg, np.int64)
    with np.errstate(invalid='ignore', over='ignore'):
        t1 = np.concatenate([v.astype(np.float64), (v * v).astype(np.float64)], axis=2)
        acc = np.zeros((nb, 6))
        for lo, hi in bands:
            acc = acc + label_totals(*colour_partials(t1[lo:hi], seg[lo:hi]), nb)
        cnt = np.bincount(seg.ravel(), minlength=nb).astype(np.float64)
        c = cnt[:, None]
        meanf = np.where(c > 0, acc[:, :3] / np.maximum(c, 1), acc[:, :3]).astype(np.float32)
        d = v - meanf[seg]
        t2 = (d * d).astype(np.float64)
        var = np.zeros((nb, 3))
        for lo, hi in bands:
            var = var + label_totals(*colour_partials(t2[lo:hi], seg[lo:hi]), nb)
        mean = _tidy(np.where(c > 0, acc[:, :3] / np.maximum(c, 1), acc[:, :3]))
        energy = _tidy(np.where(c > 0, acc[:, 3:] / np.maximum(c, 1), acc[:, 3:]))
        std = _tidy(np.sqrt(np.where(c > 0, var / np.maximum(c, 1), var)))
    yy, xx = np.divmod(np.arange(H * W), W)
    s = seg.ravel()
    centres = np.full((nb, 2), -1.0)
    ok = cnt > 0
    centres[ok, 0] = np.bincount(s, weights=yy, minlength=nb)[ok] / cnt[ok]
    centres[ok, 1] = np.bincount(s, weights=xx, minlength=nb)[ok] / cnt[ok]
    return mean, std, energy, centres, cnt.astype(np.int64)


def gray_partials(terms, seg):
    """the flushed partials of one flat volume (or slab): terms [n, K] float64, seg [n] -> (labels, partials [m, K])"""
    n, K = terms.shape
    T = (n + GSTRIP - 1) // GSTRIP
    sg = np.full(T * GSTRIP, -1, np.int64)
    tm = np.zeros((T * GSTRIP, K))
    sg[:n], tm[:n] = seg, terms
    sg, tm = sg.reshape(T, GSTRIP), tm.reshape(T, GSTRIP, K)
    cur = np.full(T, -1, np.int64)
    acc = np.zeros((T, K))
    labs, parts = [], []
    with np.errstate(invalid='ignore', over='ignore'):
        for i in range(GSTRIP + 1):
            lab = sg[:, i] if i < GSTRIP else np.full(T, -1, np.int64)
            change = lab != cur
            fl = change & (cur >= 0)
            labs.append(cur[fl])
            parts.append(acc[fl])
            cur = np.where(change, lab, cur)
            acc = np.where(change[:, None], 0.0, acc)
            if i < GSTRIP:
                acc = np.where((lab >= 0)[:, None], acc + tm[:, i], acc)
    return np.concatenate(labs), np.concatenate(parts)


def gray_stats(vol, seg, nb, slabs=None):
    """(mean, std, energy [nb]) of isb_gray_stats (whole volume when slabs is None, else flat ranges [(lo, hi), ...] in order)"""
    v = f32_terms(vol).ravel()
    s = np.asarray(seg, np.int64).ravel()
    slabs = slabs or [(0, len(v))]
    with np.errstate(invalid='ignore', over='ignore'):
        t1 = np.stack([v.astype(np.float64), (v * v).astype(np.float64)], axis=1)
        acc = np.zeros((nb, 2))
        for lo, hi in slabs:
            acc = acc + label_totals(*gray_partials(t1[lo:hi], s[lo:hi]), nb)
        cnt = np.bincount(s, minlength=nb).astype(np.float64)
        meanf = np.where(cnt > 0, acc[:, 0] / np.maximum(cnt, 1), acc[:, 0]).astype(np.float32)
        d = v - meanf[s]
        t2 = (d * d).astype(np.float64)[:, None]
        var = np.zeros((nb, 1))
        for lo, hi in slabs:
            var = var + label_totals(*gray_partials(t2[lo:hi], s[lo:hi]), nb)

        def fin(x):
            x = np.where(cnt > 0, x / np.maximum(cnt, 1), x)
            return np.where(np.isnan(x), 0.0, x) + 0.0
        return fin(acc[:, 0]), np.where(np.isnan(np.sqrt(fin(var[:, 0]))), 0.0, np.sqrt(fin(var[:, 0]))), fin(acc[:, 1])
