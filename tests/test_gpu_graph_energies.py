"""The adjacency graph, the GraphCut energies and the final gathers (csrc/graph.cu) against float64 references written here, at the
sizes and values where the kernels branch.

- Adjacency (``isb_adjacency_edges`` / ``_3d``): every edge table is compared row for row with :func:`ref_edges` (a < b, sorted by
  (b, a)), which tests/test_graph_energies_host.py holds to ``oracle.adjacency_edges`` and to a pixel loop.  The maps put a
  256-thread block across a row end, every combination of the de-duplication predicate of ``k_edge_scan``, label counts on both
  sides of the 1 024-label rounds of ``k_edge_offsets``, a label of degree 5 000 through the insertion sort of ``k_edge_emit`` and
  tables on both sides of their capacity.
- Energies (``isb_gc_energies``): all five outputs for every entry of ``engine.EDGE_MODES``; see :func:`ref_energies` for the bound
  of the weights and :func:`check_energies` for what is asserted of the integers.
- Gathers (``isb_gather``): bit patterns.

Bound of an edge weight.  With x = d / (2 std(d)^2) the weight is exp(-x) / (s / mean(s)), clamped, times ``edge_cost``.  The
reference takes mean(d), std(d) and mean(s) with ``math.fsum`` (one rounding each); the kernel adds E non-negative terms along a
chain of at most L = ceil(E / 8192) + 5 + 32 + 8 additions (a thread's strided terms, five warp shuffles, the 32 warp partials of
a CTA, the 8 CTAs of the cluster), so each of its sums is within L u of the exact one (u = 2^-53).  An error delta of the mean
enters the variance as E delta^2 only.  For lT and l1 the reference forms d with the kernel's own operations; the l2 sum of squares
could be contracted into fused multiply-adds by a build without -fmad=false, which would move d by up to (K + 2) u and the variance by up to
2 (K + 2) u kappa, kappa = sqrt(1 + mean(d)^2 / var(d)).  So x is within (L + 2 (K + 2) kappa + K + 7) u of the reference's,
exp turns that into x times as much plus its own ulp, and the spatial ratio, the clamp and ``edge_cost`` add L + 10 more u.
Counting the reference's own roundings once more:

    |dw| / w  <=  c u (1 + x),     c = L + 2 K + 24 + [l2] 2 (K + 2) kappa

Measured by this file on an H100 80GB HBM3 at 700 W (``test_worst_figures`` prints the figures of a run): worst |dw| / w 0.060 of
that bound; worst unary 1 ulp from ``oracle.unary_cost`` (CUDA's log is within 1 ulp, not correctly rounded); 2 of 41.2 million
integers within the float bound of an integer, each 1 away or equal, every other one equal.
"""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
F_CANARY, I_CANARY = -12345.625, -777
#: worst figures seen by :func:`check_energies` in this run
WORST = {'unary_ulp': 0.0, 'weight_ratio': 0.0, 'weight_ratio_case': '', 'near_unary': 0, 'near_weight': 0, 'elements': 0}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


# ------------------------------------------------------------------------------------------------------------------------------
# generators (no device; tests/test_graph_energies_host.py checks them)
# ------------------------------------------------------------------------------------------------------------------------------

def voronoi_map(h, w, n_sites, seed):
    """nearest-site label map [h, w] int32 of seeded random sites (exact Euclidean distance transform) and the sites (y, x) in
    label order; labels are a random permutation of 0 .. n - 1, n <= n_sites the number of distinct sites"""
    from scipy import ndimage
    rng = np.random.RandomState(seed)
    flat = np.unique(rng.randint(0, h * w, n_sites))
    ids = rng.permutation(len(flat)).astype(np.int32)
    free = np.ones(h * w, dtype=bool)
    free[flat] = False
    idx = ndimage.distance_transform_edt(free.reshape(h, w), return_distances=False, return_indices=True)
    label_of = np.zeros(h * w, dtype=np.int32)
    label_of[flat] = ids
    seg = label_of[idx[0] * w + idx[1]]
    sites = np.zeros((len(flat), 2))
    sites[ids] = np.stack(np.divmod(flat, w), axis=1)
    return seg, sites


def comb_volume(m):
    """[2, m, m] volume of two families of m slabs, crossed: label i is the column x = i of slice 0, label m + j the row y = j of
    slice 1, so every label of one family touches every label of the other: m^2 + 2 (m - 1) edges over 2 m labels"""
    vol = np.empty((2, m, m), dtype=np.int32)
    vol[0] = np.arange(m)[None, :]
    vol[1] = m + np.arange(m)[:, None]
    return vol


def junction_maps():
    """hand-built maps where the pixel above a pair shares one of its labels but not the other"""
    a = np.array
    maps = {
        'staircase_down': a([[0, 1, 1, 1], [0, 0, 1, 1], [0, 0, 0, 1], [0, 0, 0, 0]]),
        'staircase_up': a([[0, 0, 0, 1], [0, 0, 1, 1], [0, 1, 1, 1], [1, 1, 1, 1]]),
        'diagonal_down': a([[1, 0, 0, 0], [2, 1, 0, 0], [2, 2, 1, 0], [2, 2, 2, 1]]),
        'diagonal_up': a([[0, 0, 0, 1], [0, 0, 1, 2], [0, 1, 2, 2], [1, 2, 2, 2]]),
        't_junction': a([[0, 0, 0, 0], [0, 0, 0, 0], [1, 1, 2, 2], [1, 1, 2, 2]]),
        't_junction_side': a([[0, 0, 1, 1], [0, 0, 1, 1], [0, 0, 2, 2], [0, 0, 2, 2]]),
        'x_junction': a([[0, 0, 1, 1], [0, 0, 1, 1], [2, 2, 3, 3], [2, 2, 3, 3]]),
        'x_junction_swapped': a([[0, 0, 1, 1], [0, 0, 1, 1], [1, 1, 0, 0], [1, 1, 0, 0]]),
        'above_left_only': a([[0, 2], [0, 1]]),               # the pixel above 0|1 is 0 but its right neighbour is not 1
        'above_right_only': a([[2, 1], [0, 1]]),
        'left_upper_only': a([[0, 0], [2, 1]]),               # the pixel left of 0/1 is 0 but the one below it is not 1
        'left_lower_only': a([[2, 0], [1, 1]]),
        'touch_twice': a([[0, 1, 2, 2, 2], [2, 2, 2, 2, 2], [2, 2, 2, 0, 1]]),
        'last_row_right_only': a([[0, 0, 0, 0], [0, 0, 0, 0], [0, 0, 1, 2]]),
        'last_column_down_only': a([[0, 0, 0], [0, 0, 1], [0, 0, 2]]),
        'two_labels_two_pixels': a([[0, 1]]),
        'two_labels_column': a([[1], [0]]),
    }
    return {k: v.astype(np.int32) for k, v in maps.items()}


def random_junction_maps(count=300, seed=11):
    """seeded maps of up to 12 x 12 pixels with 2 to 6 labels: small enough that every combination of a pair with its upper / left
    neighbours occurs many times"""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(count):
        h, w, k = rng.randint(1, 13), rng.randint(1, 13), rng.randint(2, 7)
        seg = rng.randint(0, k, (h, w))
        if rng.rand() < 0.5:            # coarser regions: repeat pixels so that pairs also run along straight boundaries
            seg = np.repeat(np.repeat(seg, 2, axis=0), 2, axis=1)[:h, :w]
        out.append(seg.astype(np.int32))
    return out


def block_grid_map(n_labels, cols=32, block=3):
    """grid of ``block`` x ``block`` squares numbered row by row, ``cols`` per row; the squares past n_labels - 1 join the last"""
    rows = -(-n_labels // cols)
    ids = np.minimum(np.arange(rows * cols).reshape(rows, cols), n_labels - 1)
    return np.kron(ids, np.ones((block, block), dtype=np.int64)).astype(np.int32)


def hub_map(n_islands, hub_is_largest):
    """one background label around ``n_islands`` one-pixel islands: the background is label 0, or the largest label"""
    side = int(math.ceil(math.sqrt(n_islands)))
    seg = np.zeros((2 * side + 1, 2 * side + 1), dtype=np.int32)
    isl = np.arange(1, side * side + 1).reshape(side, side)
    isl[isl > n_islands] = 0
    seg[1::2, 1::2] = isl
    if hub_is_largest:
        seg = np.where(seg == 0, n_islands, seg - 1).astype(np.int32)
    return seg


# ------------------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------------------

def ref_edges(grid):
    """unique pairs (a < b) of labels adjacent along an axis of a 2-D or 3-D label array, sorted by (b, a): int32 [E, 2]"""
    g = np.asarray(grid)
    n = int(g.max()) + 1
    codes = [np.zeros(0, dtype=np.int64)]
    for ax in range(g.ndim):
        lo = g[(slice(None), ) * ax + (slice(None, -1), )].ravel()
        hi = g[(slice(None), ) * ax + (slice(1, None), )].ravel()
        m = lo != hi
        a, b = np.minimum(lo[m], hi[m]).astype(np.int64), np.maximum(lo[m], hi[m]).astype(np.int64)
        codes.append(np.unique(b * n + a))
    code = np.unique(np.concatenate(codes))
    return np.stack([code % n, code // n], axis=1).astype(np.int32)


def ref_energies(proba, edges, centres, mode, edge_cost):
    """float64 reference of the float outputs of ``k_gc_energies``: dict with unary [N, K], the edge weights ``w`` [E], their
    value ``v`` before the clamp, the exponent ``x`` and the relative bound ``bound`` of the module docstring"""
    metric, spatial = mode
    K, E = proba.shape[1], len(edges)
    unary = np.abs(-np.log(np.clip(proba, 0.01, 1 - 0.01)))
    a, b = edges[:, 0].astype(np.int64), edges[:, 1].astype(np.int64)
    x, v, kappa = np.zeros(E), np.ones(E), 0.0
    with np.errstate(all='ignore'):
        if metric and E:
            d = np.zeros(E)
            for k in range(K):                      # the kernel's order of operations
                df = proba[a, k] - proba[b, k]
                d = np.maximum(d, df * df) if metric == 1 else d + (np.abs(df) if metric == 2 else df * df)
            if metric == 3:
                d = np.sqrt(d)
            mean = math.fsum(d) / E
            var = math.fsum((d - mean) ** 2) / E
            sd = math.sqrt(var)
            x = d / np.float64(2 * (sd * sd))
            v = np.exp(-x)
            if metric == 3 and var > 0:
                kappa = math.sqrt(1 + mean * mean / var)
        if spatial and E:
            dy, dx = centres[a, 0] - centres[b, 0], centres[a, 1] - centres[b, 1]
            s = np.sqrt(dy * dy + dx * dx)
            v = v / (s / np.float64(math.fsum(s) / E))
    w = v.copy()
    w[v < 1e-3] = 1e-3
    w[v > 1e3] = 1e3
    w *= edge_cost
    c = (-(-E // 8192) + 45) + 2 * K + 24 + (2 * (K + 2) * kappa if metric == 3 else 0)
    bound = c * U * (1 + np.where(np.isfinite(x), x, 0))
    return {'unary': unary, 'w': w, 'v': v, 'x': x, 'bound': bound}


def pygco_conversion(edge_w, unary, pairwise):
    """pyGCO's float -> int conversion (truncation of the scaled values) with the repository's rule for a NaN weight: left out of
    the factor, capacity 0"""
    ok = ~np.isnan(edge_w)
    wmax = float(np.abs(edge_w[ok]).max()) if ok.any() else 0.0
    dwf = max(float(np.abs(unary).max()), wmax * float(pairwise.max())) + 1e-10
    return ((np.where(ok, edge_w, 0.0) / dwf * 1000).astype(np.intc), (unary / dwf * 100000).astype(np.intc),
            (pairwise * 100).astype(np.intc), dwf)


# ------------------------------------------------------------------------------------------------------------------------------
# device calls
# ------------------------------------------------------------------------------------------------------------------------------

def dev_edges(eng, seg, nb=None, cap=None):
    """(rows of the device table, device count) of ``Engine.adjacency`` (2-D) or ``Engine.graph3d`` (3-D, plus the centres)"""
    seg = np.array(seg, dtype=np.int32, order='C')          # a copy: a flipped view has strides torch does not take
    nb = int(seg.max()) + 1 if nb is None else nb
    d_seg = eng.to_device(seg)
    out = eng.adjacency(d_seg, nb, cap) if seg.ndim == 2 else eng.graph3d(d_seg, nb, cap)
    n = int(eng.to_host(out[1])[0])
    rows = eng.to_host(out[0][:min(n, cap)]).copy() if n else np.zeros((0, 2), dtype=np.int32)
    return (rows, n) if seg.ndim == 2 else (rows, n, eng.to_host(out[3]).copy())


def check_adjacency(eng, seg, nb=None, what=''):
    want = ref_edges(seg)
    got, n = dev_edges(eng, seg, nb, len(want) + 5)
    assert n == len(want), '%s: the device counts %d edges, the map has %d' % (what, n, len(want))
    np.testing.assert_array_equal(got, want, err_msg=what)
    return want


def run_energies(eng, proba, edges, centres, mode, edge_cost, pairwise, n_nodes=None, n_edges=None, canaries=False):
    """host copies of the five outputs of ``Engine.gc_energies``; ``canaries`` fills the output buffers beforehand"""
    torch = eng.torch
    (N, K), E = proba.shape, len(edges)
    d_p = eng.to_device(np.ascontiguousarray(proba, dtype=np.float64))
    d_e = eng.to_device(np.ascontiguousarray(edges if E else np.zeros((1, 2)), dtype=np.int32))
    d_c = eng.to_device(np.ascontiguousarray(centres, dtype=np.float64)) if mode[1] else None
    d_nn = None if n_nodes is None else eng.to_device(np.array([n_nodes], dtype=np.int32))
    d_ne = None if n_edges is None else eng.to_device(np.array([n_edges], dtype=np.int32))
    if canaries:
        for name, shape, dtype, val in (('unary', (N, K), torch.float64, F_CANARY), ('edge_w', (max(E, 1), ), torch.float64, F_CANARY),
                                        ('unary_i', (N, K), torch.int32, I_CANARY), ('edge_wi', (max(E, 1), ), torch.int32, I_CANARY)):
            eng.buf(name, shape, dtype).fill_(val)
    out = eng.gc_energies(d_p, d_e, E, d_ne, d_c, mode, float(edge_cost), pairwise, d_n_nodes=d_nn)
    unary, edge_w, unary_i, edge_wi, smooth_i = (eng.to_host(t).copy() for t in out)
    return unary, edge_w[:E], unary_i, edge_wi[:E], smooth_i


def check_energies(eng, oracle, proba, edges, centres, mode, edge_cost, pairwise, what):
    """all five outputs of one call:
    floats -- unary within 1 ulp of ``oracle.unary_cost``; a weight whose reference lies inside the clamp interval by twice its
      bound within that bound, one outside by twice its bound exactly the clamp value times ``edge_cost``, NaN where the
      reference is NaN;
    integers (a) -- equal to pyGCO's conversion of the kernel's own floats, element for element;
    integers (b) -- equal to ``oracle.integerise`` of the reference floats except where the value before truncation lies within
      the float bound of an integer, and there at most 1 away."""
    pairwise = np.ascontiguousarray(pairwise, dtype=np.float64)
    unary, edge_w, unary_i, edge_wi, smooth_i = run_energies(eng, proba, edges, centres, mode, edge_cost, pairwise)
    ref = ref_energies(proba, edges, centres, mode, edge_cost)
    # ---- floats
    np.testing.assert_array_equal(ref['unary'], oracle.unary_cost(proba), err_msg=what)
    ulps = np.abs(unary - ref['unary']) / np.spacing(ref['unary'])
    WORST['unary_ulp'] = max(WORST['unary_ulp'], float(ulps.max()))
    assert ulps.max() <= 1, '%s: unary %d ulp from the reference' % (what, ulps.max())
    v, w, bound = ref['v'], ref['w'], ref['bound']
    lo, hi = 1e-3 * edge_cost, 1e3 * edge_cost
    with np.errstate(invalid='ignore'):
        nan = np.isnan(v)
        free = (v > 1e-3 * (1 + 2 * bound)) & (v < 1e3 / (1 + 2 * bound))
        low, high = v < 1e-3 / (1 + 2 * bound), v > 1e3 * (1 + 2 * bound)
        err = np.abs(edge_w - w)
    assert np.isnan(edge_w[nan]).all(), '%s: a weight the reference leaves NaN is not NaN' % what
    assert (edge_w[low] == lo).all() and (edge_w[high] == hi).all(), '%s: clamped weights are not the clamp value times edge_cost' % what
    if free.any():
        ratio = err[free] / (w[free] * bound[free])
        if ratio.max() > WORST['weight_ratio']:
            WORST['weight_ratio'], WORST['weight_ratio_case'] = float(ratio.max()), what
        k = int(np.argmax(ratio))
        assert ratio.max() <= 1, '%s: edge %d: weight %r, reference %r, exponent %g: error is %.3g of the bound' % (
            what, np.flatnonzero(free)[k], edge_w[free][k], w[free][k], ref['x'][free][k], ratio.max())
    rest = ~(nan | free | low | high)
    assert ((err[rest] <= 2 * bound[rest] * w[rest]) | (edge_w[rest] == lo) | (edge_w[rest] == hi)).all(), what
    # ---- integers (a): the kernel's own floats through pyGCO's conversion
    own_w, own_u, own_v, _ = pygco_conversion(edge_w, unary, pairwise)
    np.testing.assert_array_equal(unary_i, own_u, err_msg=what + ': unary_i is not the truncation of the kernel\'s unary')
    np.testing.assert_array_equal(edge_wi, own_w, err_msg=what + ': edge_wi is not the truncation of the kernel\'s weights')
    np.testing.assert_array_equal(smooth_i, own_v, err_msg=what + ': smooth_i')
    assert (edge_wi >= 0).all() and (edge_wi[np.isnan(edge_w)] == 0).all()
    # ---- integers (b): the float64 reference through the oracle's conversion
    want_w, want_u, want_v = oracle.integerise(w, ref['unary'], pairwise)
    _, _, _, dwf = pygco_conversion(w, ref['unary'], pairwise)
    np.testing.assert_array_equal(smooth_i, want_v, err_msg=what)
    exact = nan | low | high                                       # weights both sides know exactly
    b_w = np.where(exact, 0.0, 2 * bound)
    ok = ~nan
    near_max = ok & (w >= (w[ok].max() if ok.any() else 0.0) * (1 - 2 * b_w.max(initial=0.0)))
    b_dwf = 4 * U + b_w[near_max].max(initial=0.0)                 # the factor: 1 ulp of log in the largest unary, or the largest weight
    for got, want, t, tol, key in ((unary_i, want_u, ref['unary'] / dwf * 100000, b_dwf + 6 * U, 'near_unary'),
                                   (edge_wi, want_w, np.where(ok, w, 0.0) / dwf * 1000, b_w + b_dwf + 4 * U, 'near_weight')):
        near = np.floor(t * (1 - tol)) != np.floor(t * (1 + tol))
        WORST[key] += int(near.sum())
        WORST['elements'] += near.size
        assert near.sum() <= 2 + near.size // 100, '%s: %d of %d integers are undecided, the comparison says nothing' % (what, near.sum(), near.size)
        np.testing.assert_array_equal(got[~near], want[~near], err_msg='%s: %s differs where the float is not at an integer' % (what, key))
        assert (np.abs(got[near].astype(np.int64) - want[near]) <= 1).all(), what
    return unary, edge_w, unary_i, edge_wi, smooth_i


# ------------------------------------------------------------------------------------------------------------------------------
# inputs of the energy tests
# ------------------------------------------------------------------------------------------------------------------------------

def special_proba(rng, n, k):
    """class probabilities with the values where the clip and the logarithm decide: exactly 0, 0.01, 0.99 and 1, the neighbours of
    0.01 and 0.99, subnormals, and rows that do not sum to 1 or exceed it"""
    p = rng.dirichlet(np.ones(k), n) if k > 1 else rng.rand(n, 1)
    specials = [0.0, 0.01, 0.99, 1.0, np.nextafter(0.01, 0), np.nextafter(0.01, 1), np.nextafter(0.99, 0), np.nextafter(0.99, 1),
                5e-324, 5.5e-309, 1e-300, 1.5, 7.0]
    at = rng.permutation(n * k)[:min(n * k, 4 * len(specials))]
    p.ravel()[at] = np.resize(specials, len(at))
    return p


def random_graph(rng, n, n_edges):
    """about ``n_edges`` distinct pairs a < b over n nodes, sorted by (b, a), int32"""
    if n < 2 or n_edges == 0:
        return np.zeros((0, 2), dtype=np.int32)
    a, b = rng.randint(0, n, n_edges).astype(np.int64), rng.randint(0, n, n_edges).astype(np.int64)
    keep = a != b
    code = np.unique(np.maximum(a, b)[keep] * n + np.minimum(a, b)[keep])
    return np.stack([code % n, code // n], axis=1).astype(np.int32)


def potts(k, regul=1.0):
    return (np.ones((k, k)) - np.eye(k)) * regul


@pytest.fixture(scope='module')
def voronoi_2048():
    seg, sites = voronoi_map(2048, 2048, 5000, 3)
    return seg, sites, ref_edges(seg)


@pytest.fixture(scope='module')
def voronoi_8192():
    seg, sites = voronoi_map(8192, 8192, 80000, 4)
    return seg, sites, ref_edges(seg)


# ------------------------------------------------------------------------------------------------------------------------------
# adjacency, 2-D
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('shape', [(1, 1), (1, 2), (1, 9), (7, 1), (2, 2), (1, 255), (1, 256), (1, 257), (3, 255), (3, 256), (3, 257)])
def test_adjacency_of_small_and_block_straddling_shapes(eng, shape):
    rng = np.random.RandomState(shape[0] * 1000 + shape[1])
    h, w = shape
    maps = {'one label': np.zeros(shape), 'own label': np.arange(h * w).reshape(shape), 'columns': np.tile(np.arange(w) // 2, (h, 1)),
            'random 5': rng.randint(0, 5, shape), 'random 2': rng.randint(0, 2, shape), 'rows': np.tile(np.arange(h)[:, None], (1, w))}
    for name, seg in maps.items():
        seg = seg - seg.min()
        want = check_adjacency(eng, seg.astype(np.int32), what='%s %dx%d' % (name, h, w))
        if name == 'one label':
            assert len(want) == 0
        if name == 'own label':
            assert len(want) == 2 * h * w - h - w


def test_adjacency_of_one_label_a_checkerboard_and_one_label_per_pixel(eng):
    assert len(check_adjacency(eng, np.zeros((64, 96), dtype=np.int32), what='one label')) == 0
    yy, xx = np.mgrid[:97, :130]
    assert check_adjacency(eng, ((yy + xx) % 2).astype(np.int32), what='checkerboard').tolist() == [[0, 1]]
    for h, w in ((64, 64), (65, 63)):
        want = check_adjacency(eng, np.arange(h * w, dtype=np.int32).reshape(h, w), what='own label %dx%d' % (h, w))
        assert len(want) == 2 * h * w - h - w
    # a one-pixel checkerboard of four labels: every pixel has another label above, left and diagonally
    assert len(check_adjacency(eng, ((yy % 2) * 2 + xx % 2).astype(np.int32), what='four-label checkerboard')) == 4


def test_adjacency_of_junction_maps(eng):
    for name, seg in junction_maps().items():
        for variant, m in (('', seg), (' transposed', seg.T), (' flipped', seg[::-1]), (' mirrored', seg[:, ::-1])):
            check_adjacency(eng, np.ascontiguousarray(m), what=name + variant)


def test_adjacency_of_random_small_maps(eng):
    for i, seg in enumerate(random_junction_maps()):
        check_adjacency(eng, seg, what='random map %d %r' % (i, seg.tolist()))


@pytest.mark.parametrize('n_labels', [1023, 1024, 1025, 2049])
def test_adjacency_across_the_rounds_of_the_offset_scan(eng, n_labels):
    seg = block_grid_map(n_labels)
    assert seg.max() + 1 == n_labels
    perm = np.random.RandomState(n_labels).permutation(n_labels).astype(np.int32)
    for name, m, nb in (('in order', seg, None), ('permuted ids', perm[seg], None), ('every other id unused', 2 * perm[seg], None),
                        ('nb = 4 x labels', perm[seg], 4 * n_labels), ('gaps and nb = 4 x', 2 * perm[seg] + 1, 8 * n_labels)):
        want = check_adjacency(eng, m, nb, what='%d labels, %s' % (n_labels, name))
        assert len(want) > n_labels          # a grid graph: the last round of the scan carries edges


@pytest.mark.parametrize('hub_is_largest', [False, True])
def test_adjacency_of_a_hub_of_degree_5000(eng, hub_is_largest):
    """``hub_is_largest``: the hub is the b of every pair, so one thread of ``k_edge_emit`` sorts its 5 000 neighbours"""
    torch = eng.torch
    seg = hub_map(5000, hub_is_largest)
    want = check_adjacency(eng, seg, what='hub')
    assert len(want) == 5000
    d_seg = eng.to_device(seg)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    eng.adjacency(d_seg, 5001, 5005)
    t1.record()
    t1.synchronize()
    WORST['hub %s ms' % ('largest id' if hub_is_largest else 'id 0')] = round(t0.elapsed_time(t1), 3)


def test_adjacency_of_voronoi_maps(eng, voronoi_2048):
    seg, sites, want = voronoi_2048
    assert len(sites) > 4900 and seg.max() + 1 == len(sites)
    got, n = dev_edges(eng, seg, None, len(want) + 5)
    assert n == len(want)
    np.testing.assert_array_equal(got, want)


def test_adjacency_of_a_large_voronoi_map_with_ids_above_65535(eng, voronoi_8192):
    seg, sites, want = voronoi_8192
    assert len(sites) > 79000 and seg.max() > 65535
    got, n = dev_edges(eng, seg, None, len(want) + 5)
    assert n == len(want)
    np.testing.assert_array_equal(got, want)
    # the pipelines pass an upper bound of the label count
    got, n = dev_edges(eng, seg, 3 * len(sites), 2 * len(want))
    assert n == len(want)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('case', ['random', 'own label'])
def test_adjacency_table_at_and_below_its_capacity(eng, case):
    """a table of exactly E rows is complete; a smaller one reports cap + 1 and nothing is written past row cap.  'own label' has
    more edges than the 1 024 slots of the smallest hash table, so with cap = 1 the table itself fills up"""
    from pyimsegm_b200 import _lib
    torch, lib = eng.torch, eng.lib
    seg = np.random.RandomState(5).randint(0, 50, (40, 40)).astype(np.int32) if case == 'random' else np.arange(32 * 32, dtype=np.int32).reshape(32, 32)
    want = ref_edges(seg)
    E, nb = len(want), int(seg.max()) + 1
    assert E > 1024 or case == 'random'
    d_seg = eng.to_device(seg)
    for cap in (E, E - 1, 1):
        edges = torch.full((cap + 8, 2), I_CANARY, dtype=torch.int32, device=eng.device)
        n_edges = torch.full((1, ), I_CANARY, dtype=torch.int32, device=eng.device)
        wsb = lib.isb_adjacency_workspace_bytes(nb, cap)
        ws = torch.empty(wsb, dtype=torch.uint8, device=eng.device)
        _lib.check(lib.isb_adjacency_edges(_lib.ptr(d_seg), seg.shape[0], seg.shape[1], nb, _lib.ptr(edges), cap, _lib.ptr(n_edges), _lib.ptr(ws),
                                           C.c_size_t(wsb), _lib.stream_ptr()))
        n, rows = int(n_edges.cpu()[0]), edges.cpu().numpy()
        assert (rows[cap:] == I_CANARY).all(), 'cap = %d: a row past the capacity was written' % cap
        if cap >= E:
            assert n == E
            np.testing.assert_array_equal(rows[:E], want)
        else:
            assert n == cap + 1, 'cap = %d of %d edges: the device reports %d, not cap + 1' % (cap, E, n)


def test_public_adjacency_keeps_the_callers_label_values(eng, oracle):
    from pyimsegm_b200 import superpixels as sp
    rng = np.random.RandomState(8)
    values = np.array([3, 4, 9, 100, 70000, 70001])
    for seg in (values[rng.randint(0, 6, (33, 47))], np.full((5, 5), 9), block_grid_map(1025).astype(np.int64) * 3 + 2):
        vertices, edges = sp.make_graph_segm_connect_grid2d_conn4(seg)
        v_o, e_o = oracle.adjacency_edges(seg)
        assert np.array_equal(vertices, v_o)
        assert np.asarray(edges, dtype=np.int64).reshape(-1, 2).tolist() == e_o.tolist()


# ------------------------------------------------------------------------------------------------------------------------------
# adjacency and centroids, 3-D
# ------------------------------------------------------------------------------------------------------------------------------

def check_graph3d(eng, vol, nb=None, what=''):
    vol = np.ascontiguousarray(vol, dtype=np.int32)
    nb = int(vol.max()) + 1 if nb is None else nb
    want = ref_edges(vol)
    got, n, centres = dev_edges(eng, vol, nb, len(want) + 5)
    assert n == len(want), what
    np.testing.assert_array_equal(got, want, err_msg=what)
    cnt = np.bincount(vol.ravel(), minlength=nb)
    ref = np.full((nb, 3), -1.0)
    for d, coord in enumerate(np.indices(vol.shape).reshape(3, -1)):
        ref[cnt > 0, d] = np.bincount(vol.ravel(), weights=coord, minlength=nb)[cnt > 0] / cnt[cnt > 0]
    np.testing.assert_array_equal(centres, ref, err_msg=what + ' centres')
    return want


def test_graph3d_shapes_one_voxel_labels_and_gaps(eng):
    rng = np.random.RandomState(2)
    check_graph3d(eng, np.zeros((1, 1, 1)), what='1x1x1')
    check_graph3d(eng, rng.randint(0, 4, (1, 1, 300)), what='1x1xW')
    check_graph3d(eng, rng.randint(0, 4, (300, 1, 1)), what='Dx1x1')
    check_graph3d(eng, rng.randint(0, 4, (1, 300, 1)), what='1xHx1')
    want = check_graph3d(eng, np.arange(16 ** 3).reshape(16, 16, 16), what='one voxel per label')
    assert len(want) == 3 * 16 * 16 * 15
    vol = rng.randint(0, 40, (9, 17, 33))
    check_graph3d(eng, vol, what='random')
    check_graph3d(eng, 3 * vol + 2, nb=4 * 130, what='labels with gaps, nb above the count')
    check_graph3d(eng, np.kron(rng.permutation(1100).reshape(10, 10, 11), np.ones((2, 3, 2), dtype=np.int64)), what='1100 labels')


def test_comb_volume_overflows_the_shipped_capacity_and_comes_back_complete(eng):
    from pyimsegm_b200 import engine, graph_cuts
    m = 64
    vol = comb_volume(m)
    want = ref_edges(vol)
    assert len(want) == m * m + 2 * (m - 1)
    default = engine.EDGE_CAP_PER_NODE
    try:
        assert len(want) > engine.edge_capacity(2 * m, 3), 'the comb no longer overflows the first table'
        d_vol = eng.to_device(vol)
        E, (d_edges, _, cap, _) = eng.edge_table(lambda cap: eng.graph3d(d_vol, 2 * m, cap), 2 * m, ndim=3)
        assert engine.EDGE_CAP_PER_NODE > default, 'the table was never grown'
        assert E == len(want) <= cap
        np.testing.assert_array_equal(eng.to_host(d_edges[:E]), want)
        engine.EDGE_CAP_PER_NODE = default
        edges, weights = graph_cuts.compute_edge_weights(vol, edge_type='')
        np.testing.assert_array_equal(edges, want)
        assert (weights == 1).all()
    finally:
        engine.EDGE_CAP_PER_NODE = default
    check_graph3d(eng, vol, what='comb')


# ------------------------------------------------------------------------------------------------------------------------------
# energies
# ------------------------------------------------------------------------------------------------------------------------------

def _modes():
    from pyimsegm_b200.engine import EDGE_MODES
    return sorted(EDGE_MODES.items())


@pytest.mark.parametrize('n,k', [(1, 1), (1, 3), (2, 2), (2, 64), (3, 8), (1023, 1), (1023, 3), (8193, 2), (8193, 64), (80000, 3), (80000, 8)])
def test_energies_over_sizes_and_every_edge_mode(eng, oracle, n, k):
    rng = np.random.RandomState(n * 100 + k)
    proba = special_proba(rng, n, k)
    edges = random_graph(rng, n, 1 if n == 2 else 3 * n + 17)
    assert n < 1000 or len(edges) % 8192
    centres = rng.rand(n, 2) * 1000
    pairwise = potts(k, 1.5)
    for name, mode in _modes():
        for edge_cost in (1.0, 0.25, 7.0):
            check_energies(eng, oracle, proba, edges, centres, mode, edge_cost, pairwise, 'N=%d K=%d E=%d %r cost %g' % (n, k, len(edges), name, edge_cost))
    # no edge at all: the factor is the largest unary alone
    unary, _, unary_i, _, _ = check_energies(eng, oracle, proba, edges[:0], centres, (1, 1), 1.0, pairwise, 'N=%d K=%d E=0' % (n, k))
    assert unary_i.max() == int(unary.max() / (unary.max() + 1e-10) * 100000)


def test_energies_of_dirichlet_probabilities_inside_the_clamps(eng, oracle):
    """rows near one class each, so that the distances are near 0 or near 1 and their deviation is large: most weights are
    neither clamped nor degenerate and the bound is exercised (Dirichlet rows alone give distances so alike that d / (2 std^2)
    clamps nearly every weight to 1e-3)"""
    rng = np.random.RandomState(12)
    for n, k in ((400, 2), (5000, 3), (5000, 8)):
        proba = 0.8 * np.eye(k)[rng.randint(0, k, n)] + 0.2 * rng.dirichlet(np.ones(k) * 3, n)
        edges = random_graph(rng, n, 3 * n)
        centres = rng.rand(n, 2) * 100
        for name, mode in _modes():
            for edge_cost in (1.0, 0.25, 7.0):
                _, edge_w, _, _, _ = check_energies(eng, oracle, proba, edges, centres, mode, edge_cost, potts(k, 2.0), 'dirichlet N=%d K=%d %r' % (n, k, name))
                assert ((edge_w > 1e-3 * edge_cost) & (edge_w < 1e3 * edge_cost)).mean() > 0.5


@pytest.mark.parametrize('pairwise', [np.zeros((3, 3)), potts(3, 0.004), np.array([[0, 1.7, -9.5], [1.7, 0, 2.25], [-9.5, 2.25, 0]]),
                                      np.array([[0.5, 1e5, 3], [1e5, 0.25, 0.999], [3, 0.999, 0]])])
def test_energies_with_pairwise_tables_of_either_sign(eng, oracle, pairwise):
    """the factor takes the largest pairwise entry, not the largest magnitude; a large table makes the weights, not the unary,
    decide the factor"""
    rng = np.random.RandomState(21)
    proba = special_proba(rng, 600, 3)
    edges = random_graph(rng, 600, 2000)
    for name, mode in _modes():
        check_energies(eng, oracle, proba, edges, rng.rand(600, 2) * 50, mode, 7.0, pairwise, 'pairwise %r %r' % (pairwise.tolist(), name))


def test_energies_of_the_large_voronoi_graph(eng, oracle, voronoi_8192):
    _, sites, edges = voronoi_8192
    rng = np.random.RandomState(30)
    proba = rng.dirichlet(np.ones(3) * 2, len(sites))
    assert len(edges) > 200000 and len(edges) % 8192
    for name, mode in _modes():
        check_energies(eng, oracle, proba, edges, sites, mode, 1.0, potts(3, 1.0), 'Voronoi 8192 %r' % name)


def test_energies_honour_the_device_counts(eng, oracle):
    """``n_nodes_dev`` below N: the rows past it stay unwritten.  ``n_edges_dev`` below E: the edges past it are not read.  Above E
    (an overflowed table): no edge is read, the largest weight is 0 and the unary integers are still written"""
    rng = np.random.RandomState(40)
    N, K, n = 700, 3, 412
    proba = special_proba(rng, N, K)
    centres = rng.rand(N, 2) * 30
    edges = random_graph(rng, n, 1500)                 # only nodes below n: the table a pipeline builds for n real labels
    pairwise = potts(K, 2.0)
    for name, mode in _modes():
        for n_edges in (len(edges), 1000):
            unary, edge_w, unary_i, edge_wi, _ = run_energies(eng, proba, edges, centres, mode, 1.0, pairwise, n_nodes=n, n_edges=n_edges, canaries=True)
            assert (unary[n:] == F_CANARY).all() and (unary_i[n:] == I_CANARY).all(), name
            assert (edge_w[n_edges:] == F_CANARY).all() and (edge_wi[n_edges:] == I_CANARY).all(), name
            ref = ref_energies(proba[:n], edges[:n_edges], centres, mode, 1.0)
            assert (np.abs(unary[:n] - ref['unary']) <= np.spacing(ref['unary'])).all()
            np.testing.assert_allclose(edge_w[:n_edges], ref['w'], rtol=1e-9)
            own_w, own_u, _, _ = pygco_conversion(edge_w[:n_edges], unary[:n], pairwise)
            np.testing.assert_array_equal(unary_i[:n], own_u)
            np.testing.assert_array_equal(edge_wi[:n_edges], own_w)
        unary, edge_w, unary_i, edge_wi, _ = run_energies(eng, proba, edges, centres, mode, 1.0, pairwise, n_nodes=n, n_edges=len(edges) + 1, canaries=True)
        assert (edge_w == F_CANARY).all() and (edge_wi == I_CANARY).all(), '%s: an overflowed table was read' % name
        _, own_u, _, _ = pygco_conversion(np.zeros(0), unary[:n], pairwise)
        np.testing.assert_array_equal(unary_i[:n], own_u)
        assert (unary_i[n:] == I_CANARY).all()


# ------------------------------------------------------------------------------------------------------------------------------
# degenerate edge models and coincident centroids
# ------------------------------------------------------------------------------------------------------------------------------

def ring_map(third=False):
    """a disc (label 1) inside a ring (label 0): the same centroid, bit for bit.  ``third``: the ring is an annulus and a third
    label, whose centroid lies elsewhere, surrounds it"""
    yy, xx = np.mgrid[:41, :(60 if third else 41)]
    r2 = (yy - 20) ** 2 + (xx - 20) ** 2
    seg = np.where(r2 <= 36, 1, 0)
    if third:
        seg[r2 > 196] = 2
    return seg.astype(np.int32)


def centroids(seg):
    n = np.bincount(seg.ravel())
    yy, xx = np.indices(seg.shape)
    return np.stack([np.bincount(seg.ravel(), weights=yy.ravel()) / n, np.bincount(seg.ravel(), weights=xx.ravel()) / n], axis=1)


def degenerate_cases():
    """name -> (label map, probabilities): every edge at the same model distance, or an edge between coincident centroids"""
    two = np.repeat(np.array([[0, 1]], dtype=np.int32), 6, axis=0).repeat(5, axis=1)
    grid = block_grid_map(48, cols=8, block=4)
    rng = np.random.RandomState(3)
    one_hot = np.eye(3)[rng.randint(0, 2, 48)]
    return {
        'two superpixels': (two, np.array([[0.8, 0.2], [0.3, 0.7]])),
        'two equal superpixels': (two, np.array([[0.6, 0.4], [0.6, 0.4]])),
        'uniform probabilities': (grid, np.full((48, 3), 1 / 3.)),
        'identical one-hot rows': (grid, np.tile([0., 1., 0.], (48, 1))),
        'one-hot rows of two classes': (grid, one_hot),
        'disc in a ring': (ring_map(), np.array([[0.9, 0.1], [0.2, 0.8]])),
        'disc in a ring, equal rows': (ring_map(), np.array([[0.5, 0.5], [0.5, 0.5]])),
        'disc in a ring in a frame': (ring_map(True), np.array([[0.9, 0.1], [0.2, 0.8], [0.6, 0.4]])),
        'disc in a ring in a frame, one-hot': (ring_map(True), np.array([[1., 0.], [0., 1.], [1., 0.]])),
        # lT distances 1 and 0.95: the exponent of the first is 2 / 0.05^2 = 800, exp underflows to 0 and 0 / 0 is NaN
        'disc in a ring in a frame, underflow': (ring_map(True), np.array([[1., 0.], [0., 1.], [1 - math.sqrt(0.95), math.sqrt(0.95)]])),
        'equal centroid distances': (np.repeat(np.arange(6, dtype=np.int32)[None, :], 4, axis=0).repeat(3, axis=1), rng.dirichlet(np.ones(2), 6)),
    }


@pytest.mark.parametrize('case', sorted(degenerate_cases()))
def test_degenerate_edge_models_have_one_result_on_the_device(eng, oracle, case):
    seg, proba = degenerate_cases()[case]
    edges, centres = ref_edges(seg), centroids(seg)
    for name, mode in _modes():
        for edge_cost in (1.0, 7.0):
            _, edge_w, _, edge_wi, _ = check_energies(eng, oracle, proba, edges, centres, mode, edge_cost, potts(proba.shape[1], 2.0), '%s %r' % (case, name))
            if case in ('uniform probabilities', 'identical one-hot rows', 'two equal superpixels') and mode[0]:
                assert np.isnan(edge_w).all() and (edge_wi == 0).all()          # -0 / 0: NaN stays NaN, its capacity is 0
            if case.startswith('disc in a ring') and mode[1]:
                assert edges[0].tolist() == [0, 1] and centres[0].tolist() == centres[1].tolist() == [20., 20.]
                if 'frame' not in case:
                    assert np.isnan(edge_w).all() and (edge_wi == 0).all()          # the only distance is 0: 0 / mean = 0 / 0
                elif 'underflow' in case and mode[0]:
                    assert np.isnan(edge_w[0]) and edge_wi[0] == 0                  # exp underflowed: 0 / 0
                else:
                    assert edge_w[0] == 1e3 * edge_cost                             # w / 0 = inf, clamped
            if case == 'equal centroid distances' and mode == (0, 1):
                assert (edge_w == edge_cost).all()


@pytest.mark.parametrize('case', sorted(degenerate_cases()))
def test_degenerate_edge_models_are_cut_the_same_way_by_every_route(eng, oracle, case):
    """'model*', 'spatial' and '' are integerised on the device, 'features' and 'color' by ``graph_cuts.integerise_energies`` on the
    host: both give the oracle's labels, and a NaN weight is capacity 0 on both"""
    from pyimsegm_b200 import graph_cuts as gc
    seg, proba = degenerate_cases()[case]
    n = len(proba)
    rng = np.random.RandomState(6)
    image = np.round(rng.rand(*seg.shape, 3) * 256) / 256.          # exact in float32
    flat_image = np.full(seg.shape + (3, ), 0.5)
    for edge_type in ('model', 'model_lT', 'model_l1', 'model_l2', 'spatial', ''):
        with np.errstate(all='ignore'):
            e_g, w_g = gc.compute_edge_weights(seg, proba=proba, edge_type=edge_type)
            e_o, w_o = oracle.edge_weights(seg, proba, edge_type)
            want = oracle.segment_graph_cut_general(seg, proba, 2., edge_type)
        np.testing.assert_array_equal(e_g, e_o)
        np.testing.assert_array_equal(np.isnan(w_g), np.isnan(w_o), err_msg='%s %s' % (case, edge_type))
        np.testing.assert_allclose(w_g, w_o, rtol=1e-9, err_msg='%s %s' % (case, edge_type))
        got = gc.segment_graph_cut_general(seg, proba, gc_regul=2., edge_type=edge_type)
        np.testing.assert_array_equal(got, want, err_msg='%s %s' % (case, edge_type))
    for edge_type, kw_g, kw_o in (('features', {'features': np.ones((n, 4))}, {'features': np.ones((n, 4))}),
                                  ('features', {'features': rng.rand(n, 4)}, None),
                                  ('color', {'image': flat_image}, {'color_means': np.full((n, 3), 0.5)}),
                                  ('color', {'image': image}, {'color_means': oracle.color2d_mean(image, seg)})):
        kw_o = kw_g if kw_o is None else kw_o
        with np.errstate(all='ignore'):
            _, w_g = gc.compute_edge_weights(seg, proba=proba, edge_type=edge_type, **kw_g)
            _, w_o = oracle.edge_weights(seg, proba, edge_type, **kw_o)
            want = oracle.segment_graph_cut_general(seg, proba, 2., edge_type, **kw_o)
            got = gc.segment_graph_cut_general(seg, proba, gc_regul=2., edge_type=edge_type, **kw_g)
        np.testing.assert_array_equal(np.isnan(w_g), np.isnan(w_o), err_msg='%s %s' % (case, edge_type))
        np.testing.assert_allclose(w_g, w_o, rtol=1e-9, err_msg='%s %s' % (case, edge_type))
        np.testing.assert_array_equal(got, want, err_msg='%s %s' % (case, edge_type))


def test_cut_general_graph_gives_nan_weights_no_capacity(eng, oracle):
    """NaN weights from a caller: the labels are those of the graph without these edges, whatever else the graph holds"""
    from pyimsegm_b200 import graph_cuts as gc
    rng = np.random.RandomState(9)
    proba = rng.dirichlet(np.ones(3), 300)
    edges = random_graph(rng, 300, 900)
    w = rng.rand(len(edges)) * 3
    nan = rng.rand(len(edges)) < 0.3
    unary, pw = gc.compute_unary_cost(proba), gc.compute_pairwise_cost(1.5, proba.shape)
    want = oracle.cut_general_graph(edges[~nan], w[~nan], unary, pw)
    assert np.array_equal(gc.cut_general_graph(edges, np.where(nan, np.nan, w), unary, pw), want)
    assert np.array_equal(oracle.cut_general_graph(edges, np.where(nan, np.nan, w), unary, pw), want)
    all_nan = gc.cut_general_graph(edges, np.full(len(edges), np.nan), unary, pw)
    assert np.array_equal(all_nan, np.argmin(unary, axis=1))


# ------------------------------------------------------------------------------------------------------------------------------
# gathers
# ------------------------------------------------------------------------------------------------------------------------------

def _lut_p(rng, nb, k):
    lut = rng.rand(nb, k)
    specials = [np.nan, -np.nan, np.inf, -np.inf, -0.0, 0.0, 5e-324, -5e-324, 2.2e-308 / 8, np.float64(1.7e308)]
    at = rng.permutation(nb * k)[:min(nb * k, 3 * len(specials))]
    lut.ravel()[at] = np.resize(specials, len(at))
    return lut


@pytest.mark.parametrize('k', [1, 2, 3, 5, 8, 64])
@pytest.mark.parametrize('npx', [1, 255, 256, 257, 1000])
def test_gather_is_the_lookup_bit_for_bit(eng, k, npx):
    rng = np.random.RandomState(k * 1000 + npx)
    nb = 301
    seg = rng.randint(0, nb, (1, npx)).astype(np.int32)
    seg.ravel()[rng.randint(0, npx)] = nb - 1
    seg.ravel()[0] = 0 if npx > 1 else nb - 1
    lut_i = rng.randint(-2 ** 31, 2 ** 31 - 1, nb).astype(np.int32)
    lut_p = _lut_p(rng, nb, k)
    d_seg, d_i, d_p = eng.to_device(seg), eng.to_device(lut_i), eng.to_device(lut_p)
    for want_i, want_p in ((True, False), (False, True), (True, True)):
        out_i, out_p = eng.gather(d_seg, d_i if want_i else None, d_p if want_p else None)
        assert (out_i is not None) == want_i and (out_p is not None) == want_p
        if want_i:
            np.testing.assert_array_equal(eng.to_host(out_i), lut_i[seg])
        if want_p:
            got = eng.to_host(out_p)
            assert got.shape == (1, npx, k)
            np.testing.assert_array_equal(got.view(np.int64), lut_p[seg].view(np.int64))


def test_gather_of_a_4096_square_map(eng):
    rng = np.random.RandomState(77)
    nb = 70000
    seg = rng.randint(0, nb, (4096, 4096)).astype(np.int32)
    seg[0, 0], seg[-1, -1] = nb - 1, 0
    lut_i = rng.randint(0, 8, nb).astype(np.int32)
    lut_p = _lut_p(rng, nb, 3)
    out_i, out_p = eng.gather(eng.to_device(seg), eng.to_device(lut_i), eng.to_device(lut_p))
    np.testing.assert_array_equal(eng.to_host(out_i), lut_i[seg])
    assert np.array_equal(eng.to_host(out_p).view(np.int64), lut_p[seg].view(np.int64))


# ------------------------------------------------------------------------------------------------------------------------------
# public routes
# ------------------------------------------------------------------------------------------------------------------------------

def test_public_routes_on_the_voronoi_map(eng, oracle, voronoi_2048):
    """``compute_edge_weights`` and ``segment_graph_cut_general`` for every ``edge_type``: 'features' and 'color' are integerised on
    the host, the others on the device; ``gc_regul`` as a scalar, a list and a matrix"""
    from pyimsegm_b200 import graph_cuts as gc
    seg, sites, edges = voronoi_2048
    n = len(sites)
    rng = np.random.RandomState(50)
    cls = (sites[:, 0] // 512 + sites[:, 1] // 700).astype(int) % 3                     # coarse class regions
    proba = 0.3 * np.eye(3)[cls] + 0.7 * rng.dirichlet(np.ones(3), n)
    features = np.eye(3)[cls] + rng.normal(0, 0.4, (n, 3))
    image = np.round(np.clip(0.2 + 0.3 * cls[seg][..., None] + rng.normal(0, 0.08, seg.shape + (3, )), 0, 1) * 256) / 256.
    color_means = oracle.color2d_mean(image, seg)
    for edge_type in ('model', 'model_lT', 'model_l1', 'model_l2', 'spatial', '', 'features', 'color'):
        kw_g = {'features': features} if edge_type == 'features' else {'image': image} if edge_type == 'color' else {}
        kw_o = {'features': features} if edge_type == 'features' else {'color_means': color_means} if edge_type == 'color' else {}
        e_g, w_g = gc.compute_edge_weights(seg, proba=proba, edge_type=edge_type, **kw_g)
        e_o, w_o = oracle.edge_weights(seg, proba, edge_type, **kw_o)
        np.testing.assert_array_equal(e_g, edges)
        np.testing.assert_array_equal(e_o, edges)
        np.testing.assert_allclose(w_g, w_o, rtol=1e-6 if edge_type == 'color' else 1e-9, err_msg=edge_type)
        want = oracle.segment_graph_cut_general(seg, proba, 2., edge_type, **kw_o)
        got = gc.segment_graph_cut_general(seg, proba, gc_regul=2., edge_type=edge_type, **kw_g)
        assert got.dtype == np.int32 and 0 < (got != np.argmax(proba, axis=1)).sum(), 'the cut changes nothing: the test shows nothing'
        np.testing.assert_array_equal(got, want, err_msg=edge_type)
        if edge_type in ('model', 'features'):
            un = oracle.unary_cost(proba)
            for regul in ([((0, 1), 2.0), ((1, 2), 0.5)], np.array([[1., 3., 2.], [3., 1., 4.5], [2., 4.5, 1.]])):
                pw = gc.compute_pairwise_cost(regul, proba.shape)
                want = oracle.cut_general_graph(e_o, w_o, un, pw)
                got = gc.segment_graph_cut_general(seg, proba, gc_regul=regul, edge_type=edge_type, **kw_g)
                np.testing.assert_array_equal(got, want, err_msg='%s, gc_regul %r' % (edge_type, regul))


def test_worst_figures(eng):
    """prints what the energy checks of this run measured (pytest -s shows it); the asserts repeat the bounds"""
    name = eng.torch.cuda.get_device_name(eng.device)
    print('\ngraph energies on %s: %r' % (name, WORST))
    if WORST['elements']:
        assert WORST['unary_ulp'] <= 1 and WORST['weight_ratio'] <= 1
