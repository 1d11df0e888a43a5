"""What tests/test_gpu_graph_energies.py rests on, checked without a device: its float64 references against the reference's own
outputs and doctest values, the oracle's adjacency against a pixel loop, the generators of its maps, and the one rule for a NaN
edge weight (DESIGN.md section 2) in the host conversion and in the oracle."""
import os
import warnings

import numpy as np
import pytest

from test_gpu_graph_energies import (U, block_grid_map, comb_volume, hub_map, junction_maps, pygco_conversion, random_junction_maps,
                                     ref_edges, ref_energies, voronoi_map)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_vectors.npz')
INT_MIN = -2 ** 31


def brute_force_edges(grid):
    """every pixel with its right and lower neighbour (and the next slice of a volume), one Python step at a time"""
    grid = np.asarray(grid)
    pairs = set()
    for idx in np.ndindex(*grid.shape):
        for ax in range(grid.ndim):
            nxt = tuple(i + (1 if d == ax else 0) for d, i in enumerate(idx))
            if nxt[ax] < grid.shape[ax] and grid[idx] != grid[nxt]:
                pairs.add((int(min(grid[idx], grid[nxt])), int(max(grid[idx], grid[nxt]))))
    return sorted(pairs, key=lambda p: (p[1], p[0]))


def test_edge_references_agree_on_the_junction_maps(oracle):
    maps = list(junction_maps().values()) + random_junction_maps()
    combos = set()
    for seg in maps:
        want = brute_force_edges(seg)
        assert ref_edges(seg).tolist() == [list(p) for p in want]
        present = np.unique(seg)
        if len(present) == seg.max() + 1:            # the oracle returns the label values, the same thing when none is missing
            assert oracle.adjacency_edges(seg)[1].tolist() == [list(p) for p in want]
        # which states of the de-duplication predicate of k_edge_scan the maps reach: (direction, first neighbour == l, second == other)
        h, w = seg.shape
        for y in range(h):
            for x in range(w):
                if x + 1 < w and seg[y, x] != seg[y, x + 1] and y > 0:
                    combos.add(('right', seg[y - 1, x] == seg[y, x], seg[y - 1, x + 1] == seg[y, x + 1]))
                if y + 1 < h and seg[y, x] != seg[y + 1, x] and x > 0:
                    combos.add(('down', seg[y, x - 1] == seg[y, x], seg[y + 1, x - 1] == seg[y + 1, x]))
    assert len(combos) == 8


def test_edge_reference_on_volumes_and_the_reference_outputs(oracle):
    rng = np.random.RandomState(1)
    for shape in ((1, 1, 7), (5, 1, 1), (3, 4, 5), (2, 2, 2)):
        vol = rng.randint(0, 4, shape)
        assert ref_edges(vol).tolist() == [list(p) for p in brute_force_edges(vol)]
    ref = np.load(GOLD)
    assert ref_edges(ref['color_seg']).tolist() == ref['graph_edges'].tolist()
    # doctest graphs of the reference (superpixels.py:163-168, graph_cuts.py:587-609)
    assert ref_edges(np.array([[0] * 5 + [1] * 5, [2] * 5 + [3] * 5])).tolist() == [[0, 1], [0, 2], [1, 3], [2, 3]]
    segments = np.array([[0] * 3 + [1] * 3 + [2] * 3 + [3] * 3, [4] * 3 + [5] * 3 + [6] * 3 + [7] * 3])
    assert ref_edges(segments).tolist() == [[0, 1], [1, 2], [2, 3], [0, 4], [1, 5], [4, 5], [2, 6], [5, 6], [3, 7], [6, 7]]


def test_energy_reference_against_the_reference_outputs(oracle):
    """the fsum reference = the reference's own unary, edge model (every metric) and spatial normalisation on the stored graph"""
    ref = np.load(GOLD)
    proba, edges, centres = ref['gc_proba'], ref['gc_edges'], ref['gc_centres']
    np.testing.assert_allclose(ref_energies(proba, edges, centres, (0, 0), 1.0)['unary'], ref['gc_unary'], rtol=1e-15)
    for metric, code in (('lT', 1), ('l1', 2), ('l2', 3)):
        got = ref_energies(proba, edges, centres, (code, 0), 1.0)
        want = ref['gc_edge_model_' + metric]
        inside = (want > 1e-3) & (want < 1e3)
        assert inside.any()
        assert (np.abs(got['w'] - want)[inside] <= got['bound'][inside] * want[inside]).all()
        np.testing.assert_array_equal(got['w'][~inside], np.clip(want[~inside], 1e-3, 1e3))
    got = ref_energies(proba, edges, centres, (0, 1), 0.25)
    np.testing.assert_allclose(got['w'], np.clip(1 / ref['gc_spatial_rel'], 1e-3, 1e3) * 0.25, rtol=1e-14)
    for mode, edge_type in (((1, 1), 'model'), ((2, 0), 'model_l1'), ((0, 1), 'spatial'), ((0, 0), '')):
        seg = ref['color_seg']
        p = np.random.RandomState(0).dirichlet(np.ones(3), seg.max() + 1)
        e_o, w_o = oracle.edge_weights(seg, p, edge_type)
        got = ref_energies(p, e_o, oracle.superpixel_centers(seg), mode, 1.0)
        assert (np.abs(got['w'] - w_o) <= np.maximum(got['bound'], 4 * U) * w_o).all()
    # doctest of compute_edge_model (graph_cuts.py:399-413)
    edges = np.array([[0, 1], [1, 2], [0, 3], [2, 3], [2, 4]])
    proba = np.ones((5, 2)) * 0.5
    proba[:2, 0], proba[:2, 1] = 0.9, 0.1
    np.testing.assert_allclose(ref_energies(proba, edges, None, (3, 0), 1.0)['v'], oracle.edge_model(edges, proba, 'l2'), rtol=1e-14)


def test_generators():
    seg, sites = voronoi_map(96, 128, 150, 1)
    assert seg.shape == (96, 128) and seg.dtype == np.int32 and set(np.unique(seg)) == set(range(len(sites)))
    yy, xx = np.mgrid[:96, :128]
    d2 = (yy[..., None] - sites[:, 0]) ** 2 + (xx[..., None] - sites[:, 1]) ** 2
    assert (d2[yy, xx, seg] == d2.min(axis=-1)).all()                 # every pixel carries a nearest site
    assert (seg[sites[:, 0].astype(int), sites[:, 1].astype(int)] == np.arange(len(sites))).all()
    for m in (2, 5, 64):
        vol = comb_volume(m)
        assert vol.shape == (2, m, m) and vol.max() + 1 == 2 * m
        assert len(ref_edges(vol)) == m * m + 2 * (m - 1)
    assert len(ref_edges(comb_volume(5))) == len(brute_force_edges(comb_volume(5)))
    for n in (1023, 1024, 1025, 2049):
        assert set(np.unique(block_grid_map(n))) == set(range(n))
    for largest in (False, True):
        hub = hub_map(5000, largest)
        edges = ref_edges(hub)
        assert hub.max() == 5000 and len(edges) == 5000 and (edges[:, 1 if largest else 0] == (5000 if largest else 0)).all()


# ------------------------------------------------------------------------------------------------------------------------------
# one result for a NaN edge weight
# ------------------------------------------------------------------------------------------------------------------------------

def _degenerate_tables():
    rng = np.random.RandomState(4)
    unary = -np.log(np.clip(rng.dirichlet(np.ones(3), 40), 0.01, 0.99))
    pairwise = (np.ones((3, 3)) - np.eye(3)) * 2.0
    some = rng.rand(60) * 5
    some[::7] = np.nan
    return unary, pairwise, {'all NaN': np.full(60, np.nan), 'some NaN': some, 'one NaN edge': np.array([np.nan]), 'no edge': np.zeros(0),
                             'no NaN': rng.rand(60) * 5}


@pytest.mark.parametrize('case', ['all NaN', 'some NaN', 'one NaN edge', 'no edge', 'no NaN'])
def test_nan_weights_are_left_out_of_the_factor_and_become_capacity_zero(oracle, case):
    from pyimsegm_b200 import graph_cuts as gc
    unary, pairwise, tables = _degenerate_tables()
    w = tables[case]
    want_w, want_u, want_v, dwf = pygco_conversion(w, unary, pairwise)
    ok = ~np.isnan(w)
    assert dwf == max(unary.max(), (w[ok].max() if ok.any() else 0.) * 2.0) + 1e-10
    with warnings.catch_warnings():
        warnings.simplefilter('error')                    # no cast of NaN to int is attempted at all
        for name, (got_w, got_u, got_v) in (('graph_cuts', gc.integerise_energies(w, unary, pairwise)), ('oracle', oracle.integerise(w, unary, pairwise))):
            assert got_w.dtype == got_u.dtype == got_v.dtype == np.intc, name
            np.testing.assert_array_equal(got_w, want_w, err_msg=name)
            np.testing.assert_array_equal(got_u, want_u, err_msg=name)
            np.testing.assert_array_equal(got_v, want_v, err_msg=name)
            assert (got_w >= 0).all() and (got_w[~ok] == 0).all() and got_w.min(initial=0) > INT_MIN, name
            assert got_u.max() == int(unary.max() / dwf * 100000) > 0, name
    if case == 'no NaN':                                  # pyGCO's conversion, unchanged
        f = max(np.abs(unary).max(), np.abs(w).max() * pairwise.max()) + 1e-10
        np.testing.assert_array_equal(gc.integerise_energies(w, unary, pairwise)[0], (w / f * 1000).astype(np.intc))
        np.testing.assert_array_equal(gc.integerise_energies(w, unary, pairwise)[1], (unary / f * 100000).astype(np.intc))


def test_conversion_keeps_a_given_factor_and_the_input_types():
    from pyimsegm_b200 import graph_cuts as gc
    w = np.array([0.5, np.nan, 2.0], dtype=np.float32)
    unary = np.array([[0.25, 1.5]], dtype=np.float32)
    got_w, got_u, got_v = gc.integerise_energies(w, unary, np.array([[0, 1], [1, 0]]), down_weight_factor=1.0)
    assert got_w.tolist() == [500, 0, 2000] and got_u.tolist() == [[25000, 150000]] and got_v.tolist() == [[0, 100], [100, 0]]
    third = np.float32(1) / np.float32(3)
    got = gc.integerise_energies(np.zeros(0, dtype=np.float32), np.array([[third]]), np.zeros((1, 1)), down_weight_factor=np.float32(7))
    assert got[1].tolist() == [[int(third / np.float32(7) * 100000)]]          # float32 arithmetic, as pyGCO does on float32 tables
