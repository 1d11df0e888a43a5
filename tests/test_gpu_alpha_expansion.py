"""Alpha-expansion on the device (csrc/alpha_expansion.cu) against the CPU oracle (oracle/gc_oracle.cpp) on the graphs where
the kernel changes behaviour: the flow state in shared memory or in the global workspace, the smooth-cost table in shared
memory (K <= 16) or in global memory, truncated cycle counts, start labelings, tiny and degenerate graphs, energies with many
minimisers, long augmenting paths, non-submodular moves, large integer energies, and a whole pipeline at that scale.

Every case asks for the oracle's labels exactly and for the oracle's int64 energy, which must also equal a NumPy recomputation
from the returned labels."""
import numpy as np
import pytest

from conftest import synth_regions

pytestmark = pytest.mark.gpu

CS = 8                                    # CTAs of the cluster
DYN_SMEM_BYTES = 227 * 1024 - 8 * 1024    # dynamic shared memory the kernel is launched with


def fits_in_smem(n, edges):
    """the kernel's choice of where the flow state lives: per CTA, 8 bytes (excess) + 4 x 4 bytes (sink capacity, two height
    buffers, scratch) per node of its range and 4 x 4 bytes per arc of the CTA holding the most arcs.  Arcs are grouped by tail
    node, so a CTA's arcs are the degrees of its nodes."""
    npc = (n + CS - 1) // CS
    deg = np.bincount(np.asarray(edges).ravel(), minlength=n) if len(edges) else np.zeros(n, np.int64)
    off = np.concatenate([[0], np.cumsum(deg)])
    apc = int(np.diff(off[np.minimum(np.arange(CS + 1) * npc, n)]).max())
    return 8 * npc + 4 * (4 * npc + 4 * apc) <= DYN_SMEM_BYTES


def energy(edges, w, un, pw, labels):
    labels = np.asarray(labels, dtype=np.int64)
    e = int(np.asarray(un, dtype=np.int64)[np.arange(len(labels)), labels].sum())
    if len(edges):
        e += int((np.asarray(w, dtype=np.int64) * np.asarray(pw, dtype=np.int64)[labels[edges[:, 0]], labels[edges[:, 1]]]).sum())
    return e


def device_solve(edges, w, un, pw, n_iter=-1, init=None):
    """isb_alpha_expansion through the engine: (labels, energy, stats)"""
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    N, K = un.shape
    E = len(edges)
    d_edges = eng.to_device(np.ascontiguousarray(edges if E else np.zeros((1, 2)), dtype=np.int32))
    d_w = eng.to_device(np.ascontiguousarray(w if E else np.zeros(1), dtype=np.int32))
    d_un = eng.to_device(np.ascontiguousarray(un, dtype=np.int32))
    d_pw = eng.to_device(np.ascontiguousarray(pw, dtype=np.int32))
    d_init = None if init is None else eng.to_device(np.ascontiguousarray(init, dtype=np.int32))
    labels, e, stats = eng.alpha_expansion(N, K, E, None, d_edges, d_w, d_un, d_pw, int(n_iter), d_init)
    return eng.to_host(labels).copy(), int(eng.to_host(e)[0]), eng.to_host(stats).copy()


def check(oracle, edges, w, un, pw, n_iter=-1, init=None, smem=None, min_share=None):
    """device == oracle (labels and energy), energy == NumPy; ``smem``: the path the kernel must take, asserted against both
    :func:`fits_in_smem` and stats[5]; ``min_share``: every label must hold at least this share of the nodes"""
    edges = np.asarray(edges, dtype=np.int32).reshape(-1, 2)
    want, e_want, _ = oracle.alpha_expansion_int(edges, w, un, pw, n_iter, return_energy=True, init=init)
    got, e_got, stats = device_solve(edges, w, un, pw, n_iter, init)
    assert np.array_equal(got, want), '%d of %d labels differ' % (int((got != want).sum()), len(want))
    assert e_got == e_want == energy(edges, w, un, pw, got)
    assert stats[6] == 0 and stats[7] == 0
    if smem is not None:
        assert fits_in_smem(len(un), edges) == smem
        assert stats[5] == int(smem)
    if min_share is not None:
        assert np.bincount(got, minlength=un.shape[1]).min() >= min_share * len(got)
    return got, stats


def random_graph(rng, n, deg=3.0):
    m = int(n * deg)
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    keep = a != b
    return np.unique(np.stack([np.minimum(a, b)[keep], np.maximum(a, b)[keep]], 1), axis=0).astype(np.int32)


def potts(k):
    return 1 - np.eye(k)


def truncated_linear(k, t=3):
    lab = np.arange(k)
    return np.minimum(np.abs(lab[:, None] - lab[None, :]), t).astype(float)


def integer_problem(oracle, rng, edges, n, k, regul=1.0, V=None, concentration=0.3):
    """pyGCO's integerisation of -log(Dirichlet probabilities), edge weights in [1e-3, 2] and regul * V"""
    w = rng.random_sample(len(edges)) * 2 + 1e-3
    un = -np.log(np.clip(rng.dirichlet(np.ones(k) * concentration, n), 0.01, 0.99))
    w_i, un_i, pw_i = oracle.integerise(w, un, regul * (potts(k) if V is None else V))
    return w_i, un_i, pw_i


def grid_edges(h, w, diagonal=False):
    idx = np.arange(h * w).reshape(h, w)
    parts = [np.stack([idx[:, :-1].ravel(), idx[:, 1:].ravel()], 1), np.stack([idx[:-1].ravel(), idx[1:].ravel()], 1)]
    if diagonal:
        parts += [np.stack([idx[:-1, :-1].ravel(), idx[1:, 1:].ravel()], 1), np.stack([idx[:-1, 1:].ravel(), idx[1:, :-1].ravel()], 1)]
    return np.concatenate(parts).astype(np.int32)


def region_unary(oracle, rng, h, w, k, edges, regul=1.0, noise=0.35):
    """unaries of a k-class Voronoi map under strong noise, so that the cut has to smooth; every class holds a fair share"""
    pts = rng.rand(4 * k, 2) * [h, w]
    yy, xx = np.mgrid[:h, :w]
    near = ((yy[..., None] - pts[:, 0]) ** 2 + (xx[..., None] - pts[:, 1]) ** 2).argmin(-1)
    cls = (np.arange(4 * k) % k)[near].ravel()
    p = np.full((h * w, k), 0.2 / max(k - 1, 1)) + rng.random_sample((h * w, k)) * noise
    p[np.arange(h * w), cls] += 0.8
    p /= p.sum(1, keepdims=True)
    wgt = 0.5 + rng.random_sample(len(edges))
    return oracle.integerise(wgt, -np.log(np.clip(p, 0.01, 0.99)), regul * potts(k))


# ---------------------------------------------------------------------------------------------------------------------
# shared memory and global workspace
# ---------------------------------------------------------------------------------------------------------------------

def test_random_graph_global_path_and_determinism(oracle):
    rng = np.random.RandomState(40)
    n, k = 40000, 3
    edges = random_graph(rng, n)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=1.0)
    got, _ = check(oracle, edges, w, un, pw, smem=False, min_share=0.05)
    # the flow claims excess with atomics in whatever order the hardware runs them: the labels must not depend on it
    again, _, stats = device_solve(edges, w, un, pw)
    assert np.array_equal(again, got) and stats[5] == 0


def _grid_side_at_threshold():
    """largest square 4-connected grid whose flow state still fits in shared memory"""
    sides = [s for s in range(100, 200) if fits_in_smem(s * s, grid_edges(s, s))]
    return max(sides)


def test_grids_on_either_side_of_the_shared_memory_threshold(oracle):
    s0 = _grid_side_at_threshold()
    assert not fits_in_smem((s0 + 1) ** 2, grid_edges(s0 + 1, s0 + 1))
    for side, smem in ((s0, True), (s0 + 1, False), (150, False)):
        rng = np.random.RandomState(side)
        edges = grid_edges(side, side)
        w, un, pw = region_unary(oracle, rng, side, side, 3, edges)
        check(oracle, edges, w, un, pw, smem=smem, min_share=0.05)


def test_superpixel_like_lattice_with_diagonals_global_path(oracle):
    rng = np.random.RandomState(60)
    h, wd = 200, 300                            # 60 000 raster-ordered nodes, 8 neighbours: almost every arc stays in its CTA
    edges = grid_edges(h, wd, diagonal=True)
    w, un, pw = region_unary(oracle, rng, h, wd, 4, edges, regul=0.7)
    check(oracle, edges, w, un, pw, smem=False, min_share=0.05)


def test_star_hub_global_path(oracle):
    """few nodes but one CTA holds the hub's 20 000 arcs: the arc tables do not fit"""
    rng = np.random.RandomState(20)
    n, k = 20001, 3
    edges = np.stack([np.zeros(n - 1, np.int32), np.arange(1, n, dtype=np.int32)], 1)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=0.3)
    assert fits_in_smem(n, edges[:0])           # the nodes alone would fit
    check(oracle, edges, w, un, pw, smem=False, min_share=0.05)


# ---------------------------------------------------------------------------------------------------------------------
# labels, cycles, start labeling
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('metric', ['potts', 'truncated_linear'])
@pytest.mark.parametrize('k', [2, 16, 17, 33, 64])
def test_label_counts(oracle, k, metric):
    """K <= 16 reads the smooth costs from shared memory, K > 16 from global memory; K = 64 fills the adaptive queue"""
    rng = np.random.RandomState(100 + k)
    n = 1500
    edges = random_graph(rng, n)
    V = potts(k) if metric == 'potts' else truncated_linear(k)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=1.5, V=V)
    got, stats = check(oracle, edges, w, un, pw, smem=True)
    assert len(np.unique(got)) >= min(k, 8) and stats[0] > 0


def test_cycle_counts(oracle):
    rng = np.random.RandomState(5)
    n, k = 3000, 5
    edges = random_graph(rng, n, deg=4.0)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=3.0, V=truncated_linear(k, 2), concentration=1.0)
    results = {}
    for n_iter in (1, 2, 5, -1):
        got, _ = check(oracle, edges, w, un, pw, n_iter=n_iter)
        results[n_iter] = energy(edges, w, un, pw, got)
    assert results[1] > results[2] >= results[5]            # the truncated runs really stop early


def test_init_labels(oracle):
    from pyimsegm_b200 import graph_cuts as gc
    rng = np.random.RandomState(7)
    n, k = 4000, 4
    edges = random_graph(rng, n)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=0.5)
    start = rng.randint(0, k, n).astype(np.int32)
    got, _ = check(oracle, edges, w, un, pw, init=start)
    assert not np.array_equal(got, oracle.alpha_expansion_int(edges, w, un, pw))        # the start matters
    assert np.array_equal(gc.cut_general_graph(edges, w, un, pw, init_labels=start), got)
    # a local minimum: every move fails, the start comes back unchanged
    again, _ = check(oracle, edges, w, un, pw, init=got)
    assert np.array_equal(again, got)
    assert np.array_equal(gc.cut_general_graph(edges, w, un, pw, n_iter=3, init_labels=got), got)


# ---------------------------------------------------------------------------------------------------------------------
# small and degenerate graphs
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [1, 2, 7, 8, 9, 13])
def test_tiny_graphs(oracle, n):
    """fewer nodes than CTAs, or ranges of one or two nodes"""
    rng = np.random.RandomState(n)
    k = 3
    edges = np.array([[i, j] for i in range(n) for j in range(i + 1, n) if rng.rand() < 0.5 or j == i + 1], dtype=np.int32)
    w = rng.randint(1, 60, len(edges)).astype(np.int32)
    un = rng.randint(0, 100, (n, k)).astype(np.int32)
    pw = (potts(k) * 10).astype(np.int32)
    got, _ = check(oracle, edges, w, un, pw)
    best = min(energy(edges, w, un, pw, np.array(np.unravel_index(c, (k,) * n)).reshape(n)) for c in range(k ** n)) if n <= 9 else None
    if best is not None:
        assert energy(edges, w, un, pw, got) <= 2 * best     # expansion's bound for a metric


def test_no_edges_ties_go_to_the_lowest_label(oracle):
    from pyimsegm_b200 import graph_cuts as gc
    rng = np.random.RandomState(3)
    un = rng.randint(0, 2, (5000, 4)).astype(np.int32)
    got, _ = check(oracle, np.zeros((0, 2)), np.zeros(0), un, (potts(4) * 5).astype(np.int32))
    assert np.array_equal(got, np.argmin(un, axis=1))
    assert np.array_equal(gc.cut_general_graph(np.zeros((0, 2), np.int32), np.zeros(0, np.int32), un, potts(4).astype(np.int32)), got)


@pytest.mark.parametrize('case', ['isolated', 'zero_weights', 'two_components'])
def test_degenerate_graphs(oracle, case):
    rng = np.random.RandomState(11)
    n, k = 3000, 3
    edges = random_graph(rng, n)
    if case == 'isolated':       # a block of nodes without edges, across a CTA boundary, and the last node
        lone = (edges >= 300) & (edges < 450) | (edges == n - 1)
        edges = edges[~lone.any(1)]
    elif case == 'two_components':
        half = n // 2
        edges = edges[(edges < half).all(1) | (edges >= half).all(1)]
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=0.5)
    if case == 'zero_weights':
        w[rng.rand(len(w)) < 0.3] = 0
    check(oracle, edges, w, un, pw, min_share=0.2)


def test_duplicate_and_reversed_edges(oracle):
    """cut_general_graph merges parallel edges in either orientation; the oracle takes the raw list"""
    from pyimsegm_b200 import graph_cuts as gc
    rng = np.random.RandomState(13)
    n, k = 2000, 3
    edges = random_graph(rng, n)
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=0.5, V=truncated_linear(k, 2))
    dup, again = rng.rand(len(edges)) < 0.3, rng.rand(len(edges)) < 0.1
    raw = np.concatenate([edges, edges[dup][:, ::-1], edges[again]])
    raw_w = np.concatenate([w, w[dup], w[again]])
    flip = rng.rand(len(raw)) < 0.5
    raw[flip] = raw[flip][:, ::-1]
    want, e_want, _ = oracle.alpha_expansion_int(raw, raw_w, un, pw, return_energy=True)
    got = gc.cut_general_graph(raw, raw_w, un, pw)
    assert np.array_equal(got, want)
    assert energy(raw, raw_w, un, pw, got) == e_want


# ---------------------------------------------------------------------------------------------------------------------
# many minimisers, long paths, non-submodular moves
# ---------------------------------------------------------------------------------------------------------------------

def test_ties_decided_by_sink_reachability(oracle):
    rng = np.random.RandomState(17)
    n, k = 3000, 4
    edges = random_graph(rng, n)
    w = rng.randint(0, 3, len(edges)).astype(np.int32)
    un = rng.randint(0, 3, (n, k)).astype(np.int32)
    pw = potts(k).astype(np.int32)
    check(oracle, edges, w, un, pw)
    # flat: every labeling of the unaries costs the same, only the pairwise term and the tie rule decide
    flat = np.full((n, k), 5, np.int32)
    got, _ = check(oracle, edges, w, flat, pw)
    assert not got.any()


def test_long_chain_needs_many_sweeps(oracle):
    """terminal costs only at the two ends of a 4 000-node path: the flow crosses the whole chain, and the cut can lie on any
    edge -- the tie rule puts it after the first node"""
    n = 4000
    edges = np.stack([np.arange(n - 1), np.arange(1, n)], 1).astype(np.int32)
    w = np.full(n - 1, 10, np.int32)
    un = np.zeros((n, 2), np.int32)
    un[0] = (0, 1000)
    un[-1] = (1000, 0)
    got, stats = check(oracle, edges, w, un, potts(2).astype(np.int32))
    assert got[0] == 0 and got[1:].all()
    assert stats[2] > 96 and stats[3] > 1                    # sweeps, global relabels


def test_non_submodular_moves_are_skipped(oracle):
    rng = np.random.RandomState(19)
    n, k = 2000, 3
    edges = random_graph(rng, n)
    V = np.array([[0, 1, 5], [1, 0, 1], [5, 1, 0]], dtype=float)   # V[0, 2] > V[0, 1] + V[1, 2]: not a metric
    w, un, pw = integer_problem(oracle, rng, edges, n, k, regul=1.0, V=V)
    got, _ = check(oracle, edges, w, un, pw)
    la, lb = got[edges[:, 0]], got[edges[:, 1]]
    assert ((la == 0) & (lb == 2) | (la == 2) & (lb == 0)).any()   # an expansion on 1 meets a non-submodular pair


# ---------------------------------------------------------------------------------------------------------------------
# large integer energies
# ---------------------------------------------------------------------------------------------------------------------

def test_hub_excess_beyond_32_bits(oracle):
    """8 leaves push 2^28 each into the hub in the first sweep: 2^31 in one node"""
    n = 9
    edges = np.stack([np.zeros(8), np.arange(1, 9)], 1).astype(np.int32)
    w = np.full(8, 2 ** 28, np.int32)
    un = np.zeros((n, 2), np.int32)
    un[0] = (0, 2 ** 28)
    un[1:] = (2 ** 28, 0)
    pw = potts(2).astype(np.int32)
    energies = [energy(edges, w, un, pw, (c >> np.arange(n)) & 1) for c in range(2 ** n)]
    best = int(np.argmin(energies))
    assert energies[best] == 2 ** 28 and best == 2 ** n - 1 and energies.count(2 ** 28) == 1
    got, _ = check(oracle, edges, w, un, pw)
    assert got.tolist() == [1] * n


def test_hub_with_mixed_large_weights(oracle):
    """64 leaves: 56 lean to label 1 and push about 2^33 into the hub in the first sweep, 8 lean to label 0 on light edges.
    Every terminal capacity of every move stays below 2^29, so no move is refused."""
    rng = np.random.RandomState(64)
    n = 65
    edges = np.stack([np.zeros(n - 1), np.arange(1, n)], 1).astype(np.int32)
    lean0 = np.arange(1, n) % 8 == 0
    w = np.where(lean0, rng.randint(2 ** 20, 2 ** 24, n - 1), rng.randint(2 ** 26, 2 ** 28, n - 1)).astype(np.int32)
    un = np.zeros((n, 2), np.int32)
    un[0] = (0, 2 ** 28)
    un[1:, 0] = np.where(lean0, 0, rng.randint(2 ** 27, 2 ** 28, n - 1))
    un[1:, 1] = np.where(lean0, rng.randint(2 ** 27, 2 ** 28, n - 1), 0)
    assert np.minimum(un[1:, 0], w)[~lean0].astype(np.int64).sum() >= 2 ** 32
    got, _ = check(oracle, edges, w, un, potts(2).astype(np.int32))
    assert got[0] == 1 and got[1:][~lean0].all() and not got[1:][lean0].any()


def test_capacities_beyond_the_flow_arrays_raise():
    from pyimsegm_b200 import graph_cuts as gc
    edges = np.array([[0, 1], [1, 2]], np.int32)
    un = np.array([[0, 5], [5, 0], [0, 5]], np.int32)
    with pytest.raises(RuntimeError, match=r'2\^30'):
        gc.cut_general_graph(edges, np.full(2, 2 ** 30, np.int32), un, potts(2).astype(np.int32))
    with pytest.raises(RuntimeError, match=r'2\^29'):
        gc.cut_general_graph(edges, np.ones(2, np.int32), un * 2 ** 27, potts(2).astype(np.int32))
    cost = np.full((4, 4), 2e6)                  # x 1000 on the weights and x 100 on V: pair capacities of 4e11
    with pytest.raises(RuntimeError, match=r'2\^30'):
        gc.cut_grid_graph(np.random.RandomState(0).rand(4, 4, 2), potts(2), cost[:-1], cost[:, :-1])


# ---------------------------------------------------------------------------------------------------------------------
# pixel grids and the pipeline at global-path scale
# ---------------------------------------------------------------------------------------------------------------------

def test_cut_grid_graph_matches_oracle(oracle):
    from pyimsegm_b200 import graph_cuts as gc
    rng = np.random.RandomState(256)
    h = wd = 256
    k = 3
    edges = grid_edges(h, wd)
    _, un_i, _ = region_unary(oracle, rng, h, wd, k, edges)
    unary = un_i.reshape(h, wd, k) / 1e5 + rng.random_sample((h, wd, k)) * 0.5
    cost_v, cost_h = rng.random_sample((h - 1, wd)) * 0.5, rng.random_sample((h, wd - 1)) * 0.5
    pw = truncated_linear(k, 1) * 1.3
    got = gc.cut_grid_graph(unary, pw, cost_v, cost_h)
    # the same integerisation with down_weight_factor = 1 and the same edge order
    idx = np.arange(h * wd).reshape(h, wd)
    e = np.concatenate([np.stack([idx[:-1].ravel(), idx[1:].ravel()], 1), np.stack([idx[:, :-1].ravel(), idx[:, 1:].ravel()], 1)])
    w_i = (np.concatenate([cost_v.ravel(), cost_h.ravel()]) * 1000).astype(np.intc)
    u_i = (unary.reshape(-1, k) * 100000).astype(np.intc)
    want = oracle.alpha_expansion_int(e, w_i, u_i, (pw * 100).astype(np.intc))
    assert not fits_in_smem(h * wd, e)
    assert np.array_equal(got, want)
    assert np.bincount(got, minlength=k).min() >= 0.05 * len(got)


def test_pipeline_on_the_global_path_matches_oracle(oracle):
    """2048^2 at sp_size 12: ~23 000 superpixels (29 127 seeds), the device label count below the buffer bound, the global path"""
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic_params
    img, _ = synth_regions(2048, 2048, seed=12)
    feats = {'color': ['mean']}
    segm, soft = pl.pipe_color2d_slic_features_model_graphcut(img, 3, feats, sp_size=12, sp_regul=0.2, gc_regul=1.)
    eng = get_engine()
    stats = eng.to_host(eng.buf('gc_stats', (8,), eng.torch.int32)).copy()
    assert stats[5] == 0 and stats[6] == 0 and stats[7] == 0
    slic, _ = pl.compute_color2d_superpixels_features(img, feats, sp_size=12, sp_regul=0.2)
    nb = int(slic.max()) + 1
    assert nb > 20000 and nb < eng.slic_label_bound(2048, 2048, slic_params((2048, 2048), 12, 0.2)[0])
    _, first = np.unique(slic.ravel(), return_index=True)
    proba = soft.reshape(-1, 3)[first]
    want = oracle.segment_graph_cut_general(slic, proba, 1., 'model')
    assert np.bincount(want, minlength=3).min() >= 0.05 * nb
    assert np.array_equal(segm, want[slic])
    e_g, w_g = gc.compute_edge_weights(slic, proba=proba, edge_type='model')
    e_o, w_o = oracle.edge_weights(slic, proba, 'model')
    assert not fits_in_smem(nb, e_o)
    assert np.array_equal(e_g, e_o)
    np.testing.assert_allclose(w_g, w_o, rtol=1e-9)
