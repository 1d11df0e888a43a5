"""
'color' and 'features' GraphCut edge weights on the device (isb_gc_vector_edge_weights, isb_image_unit_scale, isb_gc_energies
with given weights) against the host route ``graph_cuts.compute_edge_weights`` -- itself pinned to the reference's goldens in
tests/test_oracle_goldens.py --, then the resident and banded pipelines that take these edge types against the general route.
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, synth_disc, synth_regions

pytestmark = pytest.mark.gpu

FEATS = {'color': ['mean', 'std']}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _device_weights(eng, segments, edge_type, image=None, features=None, cap_factor=1):
    """(edges [E, 2], weights [E], (device edge table, count, capacity, centres, weights)) of the device route over a host label map"""
    from pyimsegm_b200.engine import VECTOR_EDGE_METRICS, edge_capacity
    from pyimsegm_b200.graph_cuts import device_edge_vectors
    seg = np.ascontiguousarray(segments, dtype=np.int32)
    nb = int(seg.max()) + 1
    d_seg = eng.to_device(seg, 'vt_seg')
    cap = max(edge_capacity(nb), nb * (nb - 1) // 2) * cap_factor     # a random label map is not planar: room for every pair
    d_edges, d_n_edges, _ = eng.adjacency(d_seg, nb, cap)
    _, d_centres, _ = eng.segment_stats(None, d_seg, nb, (), want_centres=True)
    d_img = None if image is None else eng.to_device(np.ascontiguousarray(image), 'vt_img')
    d_feat = None if features is None else eng.to_device(np.ascontiguousarray(features, dtype=np.float64), 'vt_feat')
    d_n = eng.to_device(np.array([nb], dtype=np.int32), 'vt_n')
    d_vec = device_edge_vectors(eng, edge_type, d_img, d_seg, nb, d_feat, d_n)
    d_w = eng.vector_edge_weights(d_vec, d_edges, cap, d_n_edges, d_centres, VECTOR_EDGE_METRICS[edge_type])
    E = int(eng.to_host(d_n_edges)[0])
    assert E <= cap
    return eng.to_host(d_edges[:E]).copy(), eng.to_host(d_w[:E]).copy(), (d_edges, d_n_edges, cap, d_centres, d_w)


def _sorted(edges, weights):
    edges = np.sort(np.asarray(edges), axis=1)
    order = np.lexsort((edges[:, 0], edges[:, 1]))
    return edges[order], np.asarray(weights)[order]


def _random_map(rng, h, w, n):
    seg = rng.randint(0, n, (h, w))
    seg.flat[rng.permutation(h * w)[:n]] = np.arange(n)      # every label present
    return seg


def _compare(eng, segments, edge_type, image=None, features=None, cap_factor=1):
    from pyimsegm_b200.graph_cuts import compute_edge_weights
    e_d, w_d, table = _device_weights(eng, segments, edge_type, image, features, cap_factor)
    e_h, w_h = compute_edge_weights(np.asarray(segments), image=image, features=features, edge_type=edge_type)
    e_d, w_d = _sorted(e_d, w_d)
    e_h, w_h = _sorted(e_h, w_h)
    assert np.array_equal(e_d, e_h)
    np.testing.assert_allclose(w_d, w_h, rtol=1e-12, atol=0, equal_nan=True)
    return w_h, table


def _cases():
    rng = np.random.RandomState(5)
    img_f = synth_regions(96, 80, seed=3)[0]
    return {
        'random_map_float': (_random_map(rng, 40, 50, 60), rng.rand(40, 50, 3)),
        'random_map_u8_above_1': (_random_map(rng, 33, 47, 25), rng.randint(0, 256, (33, 47, 3)).astype(np.uint8)),
        'u8_max_1': (_random_map(rng, 30, 30, 20), rng.randint(0, 2, (30, 30, 3)).astype(np.uint8)),
        'u16': (_random_map(rng, 30, 30, 20), rng.randint(0, 4000, (30, 30, 3)).astype(np.uint16)),
        'float_above_1': (_random_map(rng, 36, 28, 30), rng.rand(36, 28, 3) * 300),
        'f32': (_random_map(rng, 36, 28, 30), rng.rand(36, 28, 3).astype(np.float32)),
        'slic_float': (None, img_f),
        'slic_u8': (None, (synth_disc(120, 90, seed=4) * 255).astype(np.uint8)),
    }


@pytest.mark.parametrize('case', sorted(_cases()))
def test_color_weights_match_host_route(eng, case):
    from pyimsegm_b200.superpixels import segment_slic_img2d
    segments, image = _cases()[case]
    if segments is None:
        segments = segment_slic_img2d(image, sp_size=10, relative_compact=0.2)
    _compare(eng, segments, 'color', image=image)


def test_color_weights_nan_pixel(eng):
    rng = np.random.RandomState(6)
    segments = _random_map(rng, 30, 40, 30)
    for scale in (1., 200.):
        image = rng.rand(30, 40, 3) * scale
        image[7, 9, 1] = np.nan      # np.max is NaN: NaN > 1 is false, the image is not divided
        _compare(eng, segments, 'color', image=image)


@pytest.mark.parametrize('D', [1, 3, 6, 17, 40])
def test_feature_weights_match_host_route(eng, D):
    rng = np.random.RandomState(D)
    segments = _random_map(rng, 45, 38, 70)
    features = rng.normal(size=(70, D)) * rng.rand(D) * 10 + rng.rand(D) * 100
    _compare(eng, segments, 'features', features=features)
    features[:, 0] = 3.25        # a zero-variance column (StandardScaler's scale 1)
    _compare(eng, segments, 'features', features=features)


def test_feature_weights_of_a_slic_map(eng):
    from pyimsegm_b200.pipelines import compute_color2d_superpixels_features
    img = synth_regions(128, 96, seed=8)[0]
    segments, features = compute_color2d_superpixels_features(img, FEATS, sp_size=12, sp_regul=0.2)
    _compare(eng, segments, 'features', features=features)


@pytest.mark.parametrize('edge_type', ['color', 'features'])
def test_degenerate_graphs(eng, edge_type):
    """std(d) = 0: every vector equal (d = 0, NaN weights) and a single edge (d > 0, exp(-inf) = 0, clamped to 1e-3); a table
    with four times the rows of its edges"""
    two = np.zeros((10, 12), dtype=int)
    two[:, 6:] = 1
    rng = np.random.RandomState(9)
    segments = _random_map(rng, 20, 20, 15)
    flat = np.full((20, 20, 3), 0.4)
    if edge_type == 'color':
        w, _ = _compare(eng, two, 'color', image=rng.rand(10, 12, 3))
        assert np.array_equal(w, [1e-3])
        w, _ = _compare(eng, segments, 'color', image=flat)
        assert np.isnan(w).all()
        _compare(eng, segments, 'color', image=rng.rand(20, 20, 3), cap_factor=4)
    else:
        w, _ = _compare(eng, two, 'features', features=rng.rand(2, 4))
        assert np.array_equal(w, [1e-3])
        w, _ = _compare(eng, segments, 'features', features=np.ones((15, 4)))
        assert np.isnan(w).all()
        _compare(eng, segments, 'features', features=rng.rand(15, 4), cap_factor=4)


@pytest.mark.parametrize('edge_type', ['color', 'features'])
def test_integer_capacities_match_host(eng, edge_type):
    """isb_gc_energies with the given weights against integerise_energies of the host weights: a capacity may differ only where
    the float weight is within 1e-9 of a truncation boundary"""
    from pyimsegm_b200.engine import EDGE_GIVEN
    from pyimsegm_b200.graph_cuts import compute_pairwise_cost, compute_unary_cost, integerise_energies
    from pyimsegm_b200.pipelines import compute_color2d_superpixels_features
    n_near, n_total = 0, 0
    for seed in range(4):
        img = (synth_regions(160, 128, seed=20 + seed)[0] * 255).astype(np.uint8)
        segments, features = compute_color2d_superpixels_features(img, FEATS, sp_size=10, sp_regul=0.2)
        nb = int(segments.max()) + 1
        proba = np.random.RandomState(seed).dirichlet([1, 1, 1], nb)
        w_h, (d_edges, d_n_edges, cap, d_centres, d_w) = _compare(eng, segments, edge_type, image=img, features=features)
        pairwise = compute_pairwise_cost(1.5, proba.shape)
        _, _, unary_i, edge_wi, _ = eng.gc_energies(eng.to_device(proba, 'vt_proba'), d_edges, cap, d_n_edges, d_centres, EDGE_GIVEN,
                                                    1.0, pairwise, edge_w=d_w)
        E = int(eng.to_host(d_n_edges)[0])
        edges_d = eng.to_host(d_edges[:E]).copy()
        wi_d = eng.to_host(edge_wi[:E]).copy()
        un_i_d = eng.to_host(unary_i[:nb]).copy()
        order = np.lexsort((edges_d[:, 0], edges_d[:, 1]))
        wi_h, un_i_h, _ = integerise_energies(w_h, compute_unary_cost(proba), pairwise)
        assert np.array_equal(un_i_d, un_i_h)
        wi_d = wi_d[order]
        diff = wi_d != wi_h
        if diff.any():
            f = max(np.abs(compute_unary_cost(proba)).max(), np.abs(w_h).max() * pairwise.max()) + 1e-10
            v = w_h[diff] / f * 1000
            assert np.all(np.abs(v - np.round(v)) < 1e-9), 'capacities differ away from a truncation boundary'
        n_near += int(diff.sum())
        n_total += E
    print('%s: %d of %d capacities differ, all at a truncation boundary' % (edge_type, n_near, n_total))


def _general_and_resident(eng, img, model_kind, edge_type, nb_classes=3):
    from pyimsegm_b200 import pipelines as pl
    if model_kind == 'gmm':
        segm_g, _ = pl.pipe_color2d_slic_features_model_graphcut(img, nb_classes, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                                gc_edge_type=edge_type)
        model = pl._fit_model(nb_classes, True)
    else:
        from sklearn.ensemble import RandomForestClassifier
        _, features = pl.compute_color2d_superpixels_features(img, FEATS, sp_size=12, sp_regul=0.2)
        y = np.argsort(np.argsort(features[:, 0])) * nb_classes // len(features)
        model = RandomForestClassifier(n_estimators=10, max_depth=6, random_state=0).fit(features, y)
        segm_g, _ = pl.segment_color2d_slic_features_model_graphcut(img, model, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                                   gc_edge_type=edge_type)
    d_img = eng.to_device(img, 'vt_resident_img')
    d_segm, _ = pl.segment_resident(d_img, model, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2., gc_edge_type=edge_type)
    return segm_g, eng.to_host(d_segm).copy(), model


@pytest.mark.parametrize('edge_type', ['color', 'features'])
@pytest.mark.parametrize('model_kind', ['gmm', 'forest'])
@pytest.mark.parametrize('u8', [False, True])
def test_resident_equals_general_route(eng, edge_type, model_kind, u8):
    img = synth_regions(192, 160, seed=31)[0]
    if u8:
        img = (img * 255).astype(np.uint8)
    segm_g, segm_r, _ = _general_and_resident(eng, img, model_kind, edge_type)
    assert np.array_equal(segm_g, segm_r)


def test_resident_differs_from_unit_weights(eng):
    """the regression this edge type had: the resident path ran a unit-weight cut for 'color' / 'features'"""
    from pyimsegm_b200 import pipelines as pl
    img = synth_regions(192, 160, seed=33, noise=0.15)[0]
    d_img = eng.to_device(img, 'vt_resident_img')
    model = pl._fit_model(3, True)
    got = {t: eng.to_host(pl.segment_resident(d_img, model, FEATS, sp_size=8, sp_regul=0.2, gc_regul=5., gc_edge_type=t)[0]).copy()
           for t in ('', 'color', 'features')}
    assert not np.array_equal(got[''], got['color']) or not np.array_equal(got[''], got['features'])


def test_resident_color_replays_a_cuda_graph(eng):
    """three calls with a device-fitted model and colour features: the third replays captured CUDA graphs, which a host read
    inside the captured work would have made impossible"""
    from pyimsegm_b200 import pipelines as pl
    assert pl.USE_CUDA_GRAPHS
    img = synth_regions(160, 144, seed=35)[0]
    d_img = eng.to_device(img, 'vt_graph_img')
    model = pl._fit_model(3, True)
    outs = [eng.to_host(pl.segment_resident(d_img, model, {'color': ['mean']}, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                            gc_edge_type='color')[0]).copy() for _ in range(3)]
    cuts = [v for k, v in pl._GRAPHS.items() if k[0] == 'cut' and k[9] == 'color' and k[10][0] == d_img.data_ptr()]
    assert cuts and all(isinstance(v, tuple) for v in cuts), 'the colour cut was not captured as a CUDA graph'
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])


def test_resident_replays_keep_feature_sets_and_image_dtypes_apart(eng):
    """one image and one device-fitted model, three calls per configuration: 'features' with a 6-, a 3- and again a 6-column
    feature table (the same cached table buffer at another width), and 'color' over images of other dtypes.  After every call the
    edge weights the cut used equal the host route's on the same superpixels, and the labels equal the general route's, so no
    configuration replays the cut captured for another."""
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.graph_cuts import compute_edge_weights
    img = synth_regions(176, 144, seed=43)[0]
    d_img = eng.to_device(img, 'vt_sets_img')
    model = pl._fit_model(3, True)

    def check(image, d_image, feats, edge_type):
        slic, features = pl.compute_color2d_superpixels_features(image, feats, sp_size=12, sp_regul=0.2)
        edges, want_w = _sorted(*compute_edge_weights(slic, image=image, features=features, edge_type=edge_type))
        assert len(edges) > 200, len(edges)
        want = pl.pipe_color2d_slic_features_model_graphcut(image, 3, feats, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                            gc_edge_type=edge_type)[0]
        for call in range(3):
            got = eng.to_host(pl.segment_resident(d_image, model, feats, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                  gc_edge_type=edge_type)[0]).copy()
            used = eng.to_host(eng._bufs['edge_w_given'][:len(edges)]).copy()      # the device table is sorted as _sorted sorts
            np.testing.assert_allclose(used, want_w, rtol=1e-12, atol=0, err_msg='%r %r call %d' % (feats, image.dtype, call))
            assert np.array_equal(got, want), (feats, image.dtype, call)

    for feats in ({'color': ['mean', 'std']}, {'color': ['mean']}, {'color': ['mean', 'std']}):
        check(img, d_img, feats, 'features')
    for image in (img.astype(np.float32), (img * 255).astype(np.uint8), img.astype(np.float32)):
        check(image, eng.to_device(image), FEATS, 'color')


def test_unknown_edge_type_raises_on_every_entry(eng):
    from pyimsegm_b200 import pipelines as pl, tiled
    img = synth_regions(96, 96, seed=37)[0]
    d_img = eng.to_device(img, 'vt_resident_img')
    for name in ('colour', 'model_l3', 'feature'):
        with pytest.raises(ValueError, match='unknown gc_edge_type'):
            pl.segment_resident(d_img, pl._fit_model(2, True), FEATS, sp_size=12, gc_edge_type=name)
        with pytest.raises(ValueError, match='unknown gc_edge_type'):
            tiled.pipe_color2d_slic_features_model_graphcut_tiled(img, 2, FEATS, sp_size=12, gc_edge_type=name)
        with pytest.raises(ValueError, match='unknown gc_edge_type'):
            tiled.segment_color2d_slic_features_model_graphcut_tiled(img, None, FEATS, sp_size=12, gc_edge_type=name)


@pytest.mark.parametrize('edge_type', ['color', 'features'])
@pytest.mark.parametrize('u8', [False, True])
def test_banded_equals_resident(eng, edge_type, u8):
    """one and two bands per rank give the labels of segment_resident on the same image, with the device-fitted GMM and with a
    caller-fitted forest"""
    from sklearn.ensemble import RandomForestClassifier

    from pyimsegm_b200 import pipelines as pl, tiled
    img = synth_regions(256, 192, seed=41)[0]
    if u8:
        img = (img * 255).astype(np.uint8)
    d_img = eng.to_device(img, 'vt_resident_img')
    want_gmm = eng.to_host(pl.segment_resident(d_img, pl._fit_model(3, True), FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                               gc_edge_type=edge_type)[0]).copy()
    _, features = pl.compute_color2d_superpixels_features(img, FEATS, sp_size=12, sp_regul=0.2)
    y = np.argsort(np.argsort(features[:, 1])) * 3 // len(features)
    forest = RandomForestClassifier(n_estimators=10, max_depth=6, random_state=0).fit(features, y)
    want_forest = eng.to_host(pl.segment_resident(d_img, forest, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                  gc_edge_type=edge_type)[0]).copy()
    for bands in (1, 2):
        segm, _, _ = tiled.pipe_color2d_slic_features_model_graphcut_tiled(img, 3, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                                            gc_edge_type=edge_type, bands_per_rank=bands,
                                                                            want_soft=False, gather_segm=True)
        assert np.array_equal(segm, want_gmm), 'GMM, %d bands' % bands
        segm, _, _ = tiled.segment_color2d_slic_features_model_graphcut_tiled(img, forest, FEATS, sp_size=12, sp_regul=0.2, gc_regul=2.,
                                                                               gc_edge_type=edge_type, bands_per_rank=bands,
                                                                               want_soft=False, gather_segm=True)
        assert np.array_equal(segm, want_forest), 'forest, %d bands' % bands


def test_ranks_agree_on_vector_edge_cuts():
    """the banded 'color' / 'features' cuts over two processes: the band maximum and the colour sums all-reduced over the ranks.
    One GPU per process with NCCL when there are two GPUs; otherwise both processes share the GPU and the collectives run through
    gloo.  Every rank must hold the labels of segment_resident."""
    import torch
    backend = 'nccl' if torch.cuda.device_count() >= 2 else 'gloo'
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1',
           '--master-port', str(port), os.path.join(ROOT, 'tests', 'run_vector_edge_ranks.py'), backend]
    out = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = out.stdout.decode(errors='replace')
    assert out.returncode == 0, text[-3000:]
    assert 'VECTOR-EDGE-RANKS-OK world=2' in text, text[-3000:]
