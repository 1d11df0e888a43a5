"""
The resident gray-volume path: the 3-D mode of ``isb_gc_energies``, the bit-exact StandardScaler (``isb_standard_scaler``),
``segment_resident_volume`` and ``segment_volumes_batch``, against the numpy-facing stage functions of
``pipe_gray3d_slic_features_model_graphcut``, which stay the reference.

Whole pipelines are compared bit for bit: ``isb_gray_stats`` rounds each label's sum of its run partials once, so the resident
path and the stage chain give the same statistics on float volumes and with std too.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
EDGE_TYPES = ('', 'spatial', 'model', 'model_l1', 'model_l2')
EXACT_FEATURES = {'color': ['mean', 'energy', 'median']}
#: (shape, seed, noise, dtype, (sp_size, sp_regul, spacing)) -- the volumes of test_gpu_volume.py and a single slice
VOLUMES = {
    'aniso': ((5, 125, 150), 1, 0.08, np.float64, (15, 0.2, (12, 1, 1))),
    'iso': ((24, 40, 36), 2, 0.08, np.float64, (8, 0.3, (1, 1, 1))),
    'thin': ((1, 61, 47), 3, 0.2, np.float64, (9, 0.15, (3, 1, 1))),
    'u8': ((12, 50, 44), 4, 0.08, np.uint8, (10, 0.3, (2, 1, 1))),
    'f32': ((9, 33, 70), 5, 0.08, np.float32, (7, 0.25, (1, 1, 2))),
}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _blobs(shape, seed, noise=0.08):
    rng = np.random.RandomState(seed)
    zz, yy, xx = np.mgrid[:shape[0], :shape[1], :shape[2]]
    vol = 0.3 + 0.4 * ((xx > shape[2] // 2) ^ (yy > shape[1] // 3)) + 0.15 * (zz > shape[0] // 2)
    return np.clip(vol + rng.normal(0, noise, shape), 0, 1)


def _volume(name):
    shape, seed, noise, dtype, args = VOLUMES[name]
    vol = _blobs(shape, seed, noise)
    if dtype == np.uint8:
        vol = (vol * 255).astype(np.uint8)
    return vol.astype(dtype), args


def _u8_volume(shape, seed):
    return (_blobs(shape, seed) * 255).astype(np.uint8)


# ------------------------------------------------------------------ energies -----------------------------------------------------------

def _host_distance(edges, proba, edge_type):
    """the edge model's d of graph_cuts.compute_edge_model (0 when the type has no model)"""
    if not edge_type.startswith('model'):
        return np.zeros(len(edges))
    v1, v2 = proba[edges[:, 0]], proba[edges[:, 1]]
    if edge_type == 'model_l1':
        return np.abs(v1 - v2).sum(axis=1)
    if edge_type == 'model_l2':
        return np.sqrt(np.einsum('ij,ij->i', v1 - v2, v1 - v2))
    return np.max((v1 - v2) ** 2, axis=1)


def _check_volume_energies(eng, slic, proba, edge_type, gc_regul=0.7):
    from pyimsegm_b200 import graph_cuts as gc
    nb, K = int(slic.max()) + 1, proba.shape[1]
    edges_h, w_h = gc._edge_weights_volume(eng, slic, proba, edge_type)
    unary_h = gc.compute_unary_cost(proba)
    pairwise = gc.compute_pairwise_cost(gc_regul, proba.shape)
    d_seg = eng.to_device(slic.astype(np.int32), 'test_seg3d')
    E, (d_edges, _, _, d_centres) = eng.edge_table(lambda cap: eng.graph3d(d_seg, nb, cap), nb, ndim=3)
    assert E == len(edges_h)
    unary, edge_w, unary_i, edge_wi, smooth_i = eng.gc_energies(eng.to_device(proba, 'test_proba3d'), d_edges, E, None, d_centres,
                                                                gc._edge_mode(edge_type), 1.0, pairwise)
    if E:
        assert np.array_equal(eng.to_host(d_edges[:E]), edges_h)
    w_d = eng.to_host(edge_w[:E]).copy() if E else np.zeros(0)
    # floats: the kernel's reductions run in another order than numpy's, and CUDA's exp / log are within an ulp; the bound of
    # test_gpu_graph_energies.py, |dw| / w <= c u (1 + x) with x = d / (2 std(d)^2)
    nan_h = np.isnan(w_h)
    assert np.array_equal(nan_h, np.isnan(w_d)), edge_type
    if E and not nan_h.all():
        d = _host_distance(edges_h, proba, edge_type)
        sd = np.std(d)
        x = d / (2 * sd ** 2) if sd > 0 else np.zeros_like(d)
        c = int(np.ceil(E / 8192)) + 45 + 2 * K + 24 + (2 * (K + 2) * np.sqrt(1 + np.mean(d) ** 2 / max(np.var(d), 1e-300))
                                                        if edge_type == 'model_l2' else 0)
        ok = ~nan_h
        rel = np.abs(w_d[ok] - w_h[ok]) / w_h[ok]
        assert (rel <= c * U * (1 + x[ok])).all(), (edge_type, float((rel / (c * U * (1 + x[ok]))).max()))
    ulps = np.abs(eng.to_host(unary[:nb]) - unary_h) / np.spacing(unary_h)
    assert ulps.max() <= 1, edge_type
    # integers: pyGCO's conversion of the host values; a float within the bound above of an integer boundary may land 1 away
    w_i_h, un_i_h, pw_i_h = gc.integerise_energies(w_h, unary_h, pairwise)
    assert np.array_equal(eng.to_host(smooth_i), pw_i_h)
    for got, want, val in ((eng.to_host(unary_i[:nb]), un_i_h, unary_h), (eng.to_host(edge_wi[:E]) if E else np.zeros(0, np.int32), w_i_h,
                                                                            np.where(nan_h, 0, w_h))):
        diff = got.astype(np.int64) - want
        assert (np.abs(diff) <= 1).all(), edge_type
        if diff.any():
            dwf = max(np.abs(unary_h).max(), (np.abs(w_h[~nan_h]).max() if (~nan_h).any() else 0.) * pairwise.max()) + 1e-10
            scaled = val[diff != 0] / dwf * (100000 if val is unary_h else 1000)
            assert np.all(np.abs(scaled - np.round(scaled)) <= 1e-9 * np.maximum(np.abs(scaled), 1)), edge_type


@pytest.mark.parametrize('edge_type', EDGE_TYPES)
@pytest.mark.parametrize('case', sorted(VOLUMES))
def test_volume_energies_against_host_weights(eng, case, edge_type):
    from pyimsegm_b200 import superpixels as sp
    vol, (sp_size, sp_regul, spacing) = _volume(case)
    slic = sp.segment_slic_img3d_gray(vol, sp_size, sp_regul, spacing)
    rng = np.random.RandomState(len(case) + len(edge_type))
    for K in (2, 3):
        proba = rng.dirichlet(np.ones(K) * 0.7, size=int(slic.max()) + 1)
        _check_volume_energies(eng, slic, proba, edge_type)


@pytest.mark.parametrize('edge_type', EDGE_TYPES)
def test_volume_energies_one_and_two_supervoxels(eng, edge_type):
    one = np.zeros((3, 4, 5), dtype=np.int64)
    _check_volume_energies(eng, one, np.array([[0.3, 0.7]]), edge_type)
    two = np.zeros((3, 4, 5), dtype=np.int64)
    two[:, :, 2:] = 1
    _check_volume_energies(eng, two, np.array([[0.2, 0.8], [0.9, 0.1]]), edge_type)
    # centres apart along z only: the 3-D distance has to take the first coordinate
    two_z = np.zeros((4, 3, 3), dtype=np.int64)
    two_z[2:] = 1
    _check_volume_energies(eng, two_z, np.array([[0.6, 0.4], [0.5, 0.5]]), edge_type)


def test_2d_energies_keep_the_2d_mode(eng):
    """centres [N, 2] still take the 2-D spatial mode through the same entry point"""
    from pyimsegm_b200 import graph_cuts as gc
    seg = np.repeat(np.repeat(np.arange(12).reshape(3, 4), 7, axis=0), 9, axis=1)
    proba = np.random.RandomState(0).dirichlet(np.ones(2), size=12)
    edges, w = gc.compute_edge_weights(seg, proba=proba, edge_type='spatial')
    cy, cx = np.divmod(np.arange(12), 4)
    cent = np.stack([cy * 7 + 3.0, cx * 9 + 4.0], 1)
    dist = np.sqrt(np.einsum('ij,ij->i', cent[edges[:, 0]] - cent[edges[:, 1]], cent[edges[:, 0]] - cent[edges[:, 1]]))
    want = np.clip(1.0 / (dist / dist.mean()), 1e-3, 1e3)
    assert np.allclose(w, want, rtol=1e-13, atol=0)


# ------------------------------------------------------------------ scaler -------------------------------------------------------------

@pytest.mark.parametrize('n, d', [(1, 1), (7, 1), (8, 1), (129, 1), (1000, 1), (4099, 1), (2, 3), (1000, 3), (777, 4), (5000, 8), (300, 40)])
def test_standard_scaler_bit_exact(eng, n, d):
    from sklearn.preprocessing import StandardScaler
    rng = np.random.RandomState(n + d)
    x = rng.standard_normal((n, d)) * rng.choice([1e-3, 1., 1e4], d) + rng.choice([0., 3., -1e5], d)
    if d > 2:
        x[:, 1] = 2.5                       # a constant column: scale 1
    ref = StandardScaler().fit(x)
    table = np.vstack([x, np.full((5, d), np.nan)])     # rows past the real count are not read
    d_n = eng.to_device(np.array([n], np.int32), 'test_scaler_n')
    out, params = eng.standard_scaler(eng.to_device(table, 'test_scaler_in'), d_n)
    params = eng.to_host(params).copy()
    assert np.array_equal(params[:d], ref.mean_) and np.array_equal(params[d:], ref.scale_)
    assert np.array_equal(eng.to_host(out[:n]), ref.transform(x))


# ------------------------------------------------------------------ pipelines ----------------------------------------------------------

def _stage_reference(vol, proba_fn, feats, spacing, sp_size, sp_regul, gc_regul):
    """the stage chain of pipe_gray3d_slic_features_model_graphcut with a given model"""
    from pyimsegm_b200 import descriptors as desc
    from pyimsegm_b200 import graph_cuts as gc
    from pyimsegm_b200 import superpixels as sp
    slic = sp.segment_slic_img3d_gray(vol, sp_size=sp_size, relative_compact=sp_regul, space=spacing)
    features, _ = desc.compute_selected_features_gray3d(vol, slic, feats)
    features[np.isnan(features)] = 0
    features, _ = desc.norm_features(features)
    proba = proba_fn(features)
    labels = gc.segment_graph_cut_general(slic, proba, vol, features, gc_regul)
    return labels[slic], proba[slic], features


def _fitted_models(feats, spacing=(2, 1, 1), sp_size=10, sp_regul=0.3):
    """a GMM pipeline and a random forest fitted by the caller on the standardised features of a training volume"""
    from sklearn import ensemble, mixture, pipeline, preprocessing
    train = _u8_volume((10, 60, 52), 11)
    _, _, x = _stage_reference(train, lambda f: np.ones((len(f), 2)) / 2, feats, spacing, sp_size, sp_regul, 0.)
    gmm = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()),
                             ('model', mixture.GaussianMixture(2, covariance_type='full', random_state=0))]).fit(x)
    y = np.where(x[:, 0] > np.median(x[:, 0]), 7, 3)
    forest = ensemble.RandomForestClassifier(n_estimators=12, max_depth=6, random_state=0).fit(x, y)
    return {'gmm': gmm, 'forest': forest}


def _download(eng, tensors):
    hosts, done = eng.download(tensors)
    done.synchronize()
    return [h.numpy() for h in hosts]


@pytest.mark.parametrize('model_name', ['gmm', 'forest'])
@pytest.mark.parametrize('gc_regul', [0.1, 1.0])
def test_resident_volume_equals_stage_chain_bit_for_bit(eng, model_name, gc_regul):
    from pyimsegm_b200 import class_models
    from pyimsegm_b200 import pipelines as pl
    model = _fitted_models(EXACT_FEATURES)[model_name]
    cm = class_models.compile_model(model)
    assert cm is not None
    for shape, seed, spacing in (((12, 50, 44), 21, (2, 1, 1)), ((5, 125, 150), 22, (12, 1, 1)), ((1, 64, 80), 23, (3, 1, 1))):
        vol = _u8_volume(shape, seed)
        want_segm, want_soft, _ = _stage_reference(vol, cm.predict_proba, EXACT_FEATURES, spacing, 10, 0.3, gc_regul)
        d_segm, d_soft = pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), model, EXACT_FEATURES, spacing, 10, 0.3, gc_regul)
        assert d_segm.dtype == eng.torch.int32 and tuple(d_segm.shape) == shape and tuple(d_soft.shape) == shape + (2, )
        segm, soft = _download(eng, (d_segm, d_soft))
        assert np.array_equal(segm, want_segm), (model_name, shape)
        assert np.array_equal(soft.view(np.int64), want_soft.view(np.int64)), (model_name, shape)


@pytest.mark.parametrize('case', ['aniso', 'f32', 'thin'])
def test_resident_volume_float_statistics(eng, case):
    """float volumes with std: the same labels and the same probabilities, bit for bit (the statistics round each label's sum once)"""
    from pyimsegm_b200 import class_models
    from pyimsegm_b200 import pipelines as pl
    feats = {'color': ['mean', 'std', 'energy', 'median']}
    vol, (sp_size, sp_regul, spacing) = _volume(case)
    model = _fitted_models(feats)['gmm']
    want_segm, want_soft, _ = _stage_reference(vol, class_models.compile_model(model).predict_proba, feats, spacing, sp_size, sp_regul, 0.1)
    segm, soft = _download(eng, pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), model, feats, spacing, sp_size, sp_regul, 0.1))
    assert np.array_equal(segm, want_segm)
    assert np.array_equal(soft.view(np.int64), want_soft.view(np.int64))


def test_resident_volume_device_fit_and_host_model(eng):
    """('fit', K, ...) runs the device mixture on the standardised table; a model compile_model does not take runs on the host"""
    from pyimsegm_b200 import pipelines as pl
    vol = _u8_volume((12, 50, 44), 31)
    segm, soft = _download(eng, pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), pl._fit_model(2, True), EXACT_FEATURES,
                                                           (2, 1, 1), 10, 0.3, 0.1))
    assert soft.shape == vol.shape + (2, ) and np.allclose(soft.sum(-1), 1)
    assert set(np.unique(segm)) == {0, 1}

    def proba_fn(features):          # a plain callable: one round trip
        return np.stack([1 / (1 + np.exp(features[:, 0])), 1 - 1 / (1 + np.exp(features[:, 0]))], 1)
    want_segm, want_soft, _ = _stage_reference(vol, proba_fn, EXACT_FEATURES, (2, 1, 1), 10, 0.3, 0.1)
    segm, soft = _download(eng, pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), proba_fn, EXACT_FEATURES, (2, 1, 1), 10, 0.3,
                                                           0.1))
    assert np.array_equal(segm, want_segm) and np.array_equal(soft, want_soft)


def test_volumes_batch_equals_resident(eng):
    from pyimsegm_b200 import pipelines as pl
    vols = [_u8_volume(s, 40 + i) for i, s in enumerate([(12, 50, 44), (5, 70, 90), (1, 64, 80), (12, 50, 44), (8, 33, 61)])]
    models = _fitted_models(EXACT_FEATURES)
    for kw in ({'model_pipeline': models['forest']}, {'model_pipeline': models['gmm']}, {'nb_classes': 2}):
        got = pl.segment_volumes_batch(vols, dict_features=EXACT_FEATURES, spacing=(2, 1, 1), sp_size=10, sp_regul=0.3, gc_regul=0.1, **kw)
        assert len(got) == len(vols)
        model = kw.get('model_pipeline') or pl._fit_model(2, True)
        classes = getattr(kw.get('model_pipeline'), 'classes_', None)
        for vol, (segm, soft) in zip(vols, got):
            want_segm, want_soft = _download(eng, pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), model, EXACT_FEATURES,
                                                                             (2, 1, 1), 10, 0.3, 0.1))
            if classes is not None:
                want_segm = np.asarray(classes)[want_segm]
            assert segm.shape == vol.shape and soft.shape == vol.shape + (2, )
            assert np.array_equal(segm, want_segm), kw
            assert np.array_equal(soft, want_soft), kw
    assert set(np.unique(np.concatenate([s.ravel() for s, _ in
                                         pl.segment_volumes_batch(vols[:2], model_pipeline=models['forest'], dict_features=EXACT_FEATURES,
                                                                  spacing=(2, 1, 1), sp_size=10, sp_regul=0.3)]))) <= {3, 7}


def test_volume_edge_table_overflow_is_redone(eng, monkeypatch):
    from pyimsegm_b200 import engine
    from pyimsegm_b200 import pipelines as pl
    vols = [_u8_volume((12, 50, 44), 51), _u8_volume((6, 80, 70), 52)]
    model = _fitted_models(EXACT_FEATURES)['forest']
    want = [_download(eng, pl.segment_resident_volume(eng.to_device(v, 'test_volume'), model, EXACT_FEATURES, (2, 1, 1), 10, 0.3, 0.1))
            for v in vols]
    # a table of 64 rows: every volume overflows it, grows x4 and is redone
    monkeypatch.setattr(engine, 'EDGE_CAP_PER_NODE', 1e-3)
    got = _download(eng, pl.segment_resident_volume(eng.to_device(vols[0], 'test_volume'), model, EXACT_FEATURES, (2, 1, 1), 10, 0.3, 0.1))
    assert engine.EDGE_CAP_PER_NODE > 1e-3
    assert np.array_equal(got[0], want[0][0]) and np.array_equal(got[1], want[0][1])
    monkeypatch.setattr(engine, 'EDGE_CAP_PER_NODE', 1e-3)
    got = pl.segment_volumes_batch(vols, model_pipeline=model, dict_features=EXACT_FEATURES, spacing=(2, 1, 1), sp_size=10, sp_regul=0.3,
                                   gc_regul=0.1)
    assert engine.EDGE_CAP_PER_NODE > 1e-3
    for (segm, soft), (w_segm, w_soft) in zip(got, want):
        assert np.array_equal(segm, np.asarray(model.classes_)[w_segm]) and np.array_equal(soft, w_soft)


def test_texture_dictionaries_keep_the_stage_path(eng):
    from pyimsegm_b200 import pipelines as pl
    assert pl._volume_flags({'tLM_short': ['mean']}) is None and pl._volume_flags({'color': ['meanGrad']}) is None
    with pytest.raises(ValueError):
        pl.segment_resident_volume(eng.to_device(_u8_volume((4, 30, 30), 1), 'test_volume'), pl._fit_model(2, True),
                                   {'color': ['mean'], 'tLM_short': ['mean']})
