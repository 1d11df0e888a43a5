"""
Every feature set of the reference on the device feature driver (descriptors.device_feature_table), through the pipelines'
resident table and through the numpy API on a given label map: median, meanGrad, the colour-space groups and the Leung-Malik
responses with median / meanGrad -- against the host composition the numpy API used before it shared that driver, written here from
public pieces: the colour space on the host (color.py), one single-statistic function per statistic, meanGrad by np.gradient in
numpy's dtype, and the Leung-Malik responses by the generic FP64 filter kernels.

The mean / std / energy columns of the host composition add the same terms in another association (one statistic per launch, some
on the host), so they are compared at rtol 1e-12; two device launches over one label map give the same bits, so replays, batches and
single calls are compared bit for bit.  The medians are exact selections and compared bit for bit.
"""
import numpy as np
import pytest

from conftest import synth_regions

pytestmark = pytest.mark.gpu

FLAGS = ('mean', 'std', 'energy', 'median', 'meanGrad')
SPACES = ('hsv', 'luv', 'lab', 'hed', 'xyz')
TUTORIAL = {'color': ['mean', 'std', 'median']}


def _as_dtype(img, dtype):
    if dtype == np.uint8:
        return np.round(img * 255).astype(np.uint8)
    if dtype == np.uint16:
        return np.round(img * 65535).astype(np.uint16)
    return img.astype(dtype)


def _conversion_inputs():
    """greys (delta == 0), primaries and secondaries, zeros, ties of two maxima, the sRGB (0.04045) and L (0.008856) thresholds, and
    random colours, in all four dtypes"""
    rng = np.random.RandomState(3)
    special = [[0, 0, 0], [1, 1, 1], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1], [.5, .5, .5], [.5, .5, .2],
               [.2, .5, .5], [.5, .2, .5], [.04045, .04045, .04045], [.04045, .2, .7], [.1144, .1144, .1144], [.0989, .0989, .0989],
               [1e-7, 0, 0], [0.008856, 0.008856, 0.008856]]
    px = np.concatenate([np.array(special), np.linspace(0, 1, 257)[:, None].repeat(3, 1), rng.rand(400, 3),
                         rng.randint(0, 4, (100, 3)) / 3.])
    img = px[:len(px) // 16 * 16].reshape(16, -1, 3)
    return {np.uint8: _as_dtype(img, np.uint8), np.uint16: _as_dtype(img, np.uint16), np.float32: img.astype(np.float32), np.float64: img}


def test_color_convert_matches_color_py():
    from pyimsegm_b200 import color
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    for dtype, img in _conversion_inputs().items():
        d_img = eng.to_device(np.ascontiguousarray(img))
        for space in SPACES:
            got = eng.to_host(eng.color_convert(d_img, space)).copy()
            want = color.convert_img_color_from_rgb(img, space)
            if space == 'hsv':
                np.testing.assert_array_equal(got, want, err_msg='%s %s' % (dtype.__name__, space))
            else:
                np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12, err_msg='%s %s' % (dtype.__name__, space))


def _compare_group(got, want, space, ncol_native):
    if space in ('color', 'hsv'):
        np.testing.assert_allclose(got[:, :ncol_native], want[:, :ncol_native], rtol=1e-12, atol=0)
        np.testing.assert_array_equal(got[:, ncol_native:ncol_native + 3], want[:, ncol_native:ncol_native + 3])
        np.testing.assert_allclose(got[:, ncol_native + 3:], want[:, ncol_native + 3:], rtol=1e-12, atol=0)
    else:
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12)


def _colour_reference(img, seg, key, flags):
    """one colour group as the host composed it: the image, or its colour space when the key names one (color.py, on the host);
    then per statistic the single-statistic function, the median of np.nan_to_num(x), meanGrad as the mean of
    np.sum(np.gradient(np.nan_to_num(channel)), axis=0) in numpy's dtype"""
    from pyimsegm_b200 import color
    from pyimsegm_b200 import descriptors as ds
    src = color.convert_img_color_from_rgb(img, key.split('_')[-1]) if '_' in key else img
    blocks = []
    for f in [f for f in FLAGS if f in flags]:
        if f == 'median':
            blocks.append(ds.numpy_img2d_color_median(np.nan_to_num(src), seg))
        elif f == 'meanGrad':
            clean = np.nan_to_num(src)
            blocks.append(ds.cython_img2d_color_mean(np.stack([np.sum(np.gradient(clean[..., c]), axis=0) for c in range(3)], -1), seg))
        else:
            blocks.append(getattr(ds, 'cython_img2d_color_' + f)(src, seg))
    return np.nan_to_num(np.hstack(blocks))


def _lm_reference(img, seg, flags, bank_type):
    """the Leung-Malik group with every response in memory, in the reference's sequence (descriptors.py:1078-1098): background
    (sigma 150 on all three axes), per battery the strongest response per channel (FP64, isb_filter_response_2d), clip, log-norm
    scaling, then the colour group's statistics (:func:`_colour_reference`).  Returns (features, names)."""
    from pyimsegm_b200 import descriptors as ds
    from pyimsegm_b200 import texture
    _, _, mix = texture.background_kernel()
    roll = np.ascontiguousarray(np.rollaxis(np.asarray(img, dtype=np.float64), -1, 0))
    smooth = ds._gauss_smooth_slices(roll, texture.BACKGROUND_SIGMA)      # the two image axes ...
    roll = roll - np.tensordot(mix, smooth, axes=(1, 0))                  # ... and the reflected length-3 channel axis
    batteries, battery_names = texture.lm_bank(bank_type)
    features, names = [], []
    for battery, battery_name in zip(batteries, battery_names):
        resp = ds.compute_img_filter_response3d(roll, battery)
        resp[resp > ds.MAX_SIGNAL_RESPONSE] = ds.MAX_SIGNAL_RESPONSE
        norm = np.sqrt(np.sum(resp ** 2))
        resp = np.zeros(resp.shape) if norm == 0 or abs(norm) == np.inf else (resp * (np.log(1 + norm) / 0.03)) / norm
        features.append(_colour_reference(np.rollaxis(resp, 0, 3), seg, 'color', flags))
        names += ['tLM_%s-ch%i_%s' % (battery_name, c + 1, f) for f in FLAGS if f in flags for c in range(3)]
    return np.hstack(features), names


def _reference_table(img, seg, feats):
    """the whole dict in the column order of compute_selected_features_color2d: colour groups, then texture groups"""
    keys = [k for k in feats if k.startswith('color')] + [k for k in feats if k.startswith('tLM')]
    return np.hstack([_colour_reference(img, seg, k, feats[k]) if k.startswith('color')
                      else _lm_reference(img, seg, feats[k], 'short' if k.endswith('_short') else 'normal')[0] for k in keys])


@pytest.mark.parametrize('dtype', [np.uint8, np.uint16, np.float16, np.float32, np.float64])
def test_colour_groups_match_host_route(dtype):
    """the pipeline table and the numpy API on its label map; a float16 image is widened to f64 for every statistic, meanGrad too"""
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.descriptors import compute_selected_features_img2d
    img = _as_dtype(synth_regions(96, 112, seed=71)[0], dtype)
    ref_img = img.astype(np.float64) if dtype == np.float16 else img
    for key in ['color'] + ['color_' + s for s in SPACES]:
        slic, got = pl.compute_color2d_superpixels_features(img, {key: FLAGS}, sp_size=12)
        api, _ = compute_selected_features_img2d(img, slic, {key: FLAGS})
        want = _colour_reference(ref_img, slic, key, FLAGS)
        assert got.shape == api.shape == want.shape == (slic.max() + 1, 15)
        _compare_group(got, want, key.split('_')[-1], 9)
        _compare_group(api, want, key.split('_')[-1], 9)


def test_group_statistics_of_an_image_with_nan_and_inf():
    """the resident group statistics on a caller's label map: NaN / inf pixels go through np.nan_to_num as on the host"""
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    rng = np.random.RandomState(4)
    seg = (np.arange(40)[:, None] // 8) * 6 + np.arange(36)[None, :] // 6
    for dtype in (np.float32, np.float64):
        img = rng.rand(40, 36, 3).astype(dtype)
        img[rng.rand(40, 36) < 0.05, 1] = np.nan
        img[3, 4, 0], img[20, 30, 2] = np.inf, -np.inf
        want = _colour_reference(img, seg, 'color', FLAGS)
        nb = int(seg.max()) + 1
        feat = eng.buf('test_feat', (nb, 15), eng.torch.float64)
        eng.group_stats(eng.to_device(img), eng.to_device(seg.astype(np.int32)), nb, FLAGS, feat, 0)
        got = eng.to_host(feat).copy()
        _compare_group(got, want, 'color', 9)


def _column_scaled_close(got, want, rel=1e-9):
    scale = np.maximum(np.abs(want).max(axis=0), 1e-300)
    assert np.all(np.abs(got - want) <= rel * scale), np.max(np.abs(got - want) / scale)


@pytest.mark.parametrize('key', ['tLM_short', 'tLM'])
def test_texture_median_meangrad_match_host_route_and_oracle(key):
    from oracle import texture as otex
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.descriptors import compute_selected_features_img2d
    img = synth_regions(48, 56, seed=72)[0]
    flags = ('mean', 'std', 'median', 'meanGrad')
    bank = 'short' if key == 'tLM_short' else 'normal'
    slic, got = pl.compute_color2d_superpixels_features(img, {key: flags}, sp_size=10)
    api, names = compute_selected_features_img2d(img, slic, {key: flags})
    want, want_names = _lm_reference(img, slic, flags, bank)
    assert got.shape == api.shape == want.shape == (slic.max() + 1, (15 if key == 'tLM_short' else 20) * 12)
    assert names == want_names
    _column_scaled_close(got, want)
    _column_scaled_close(api, want)
    oracle_fts, _ = otex.texture_desc_lm(img, slic, flags, bank)
    np.testing.assert_allclose(got, oracle_fts, rtol=1e-5, atol=1e-7)


def test_mixed_dict_comes_out_in_host_column_order():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.descriptors import compute_selected_features_img2d
    img = _as_dtype(synth_regions(48, 64, seed=73)[0], np.uint8)
    feats = {'tLM_short': ('meanGrad', ), 'color_hsv': ('median', 'mean'), 'color': ('energy', ), 'color_lab': ('std', 'median')}
    slic, got = pl.compute_color2d_superpixels_features(img, feats, sp_size=10)
    api, _ = compute_selected_features_img2d(img, slic, feats)
    want = _reference_table(img, slic, feats)
    assert got.shape == api.shape == want.shape == (slic.max() + 1, 6 + 3 + 6 + 45)
    for table in (got, api):
        np.testing.assert_allclose(table[:, :9], want[:, :9], rtol=1e-12, atol=0)
        np.testing.assert_allclose(table[:, 9:15], want[:, 9:15], rtol=1e-9, atol=1e-12)
        _column_scaled_close(table[:, 15:], want[:, 15:])


def _host_models(img, feats, sp_size):
    from sklearn import ensemble, mixture, pipeline, preprocessing
    from pyimsegm_b200 import pipelines as pl
    slic, _ = pl.compute_color2d_superpixels_features(img, feats, sp_size=sp_size)
    fts = _reference_table(img, slic, feats)
    gmm = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                             ('model', mixture.GaussianMixture(3, covariance_type='full', random_state=0))]).fit(fts)
    labels = gmm.predict(fts)
    forest = pipeline.Pipeline([('scaler', preprocessing.StandardScaler()),
                                ('classif', ensemble.RandomForestClassifier(n_estimators=10, random_state=0))]).fit(fts, labels)
    return gmm, forest


def test_shared_model_resident_equals_general_path():
    from pyimsegm_b200 import pipelines as pl
    img = synth_regions(96, 112, seed=74)[0]
    gmm, forest = _host_models(img, TUTORIAL, 12)
    for model, soft_tol in ((gmm, 1e-9), (forest, 0)):
        segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, model, TUTORIAL, sp_size=12)
        segm_g, soft_g = pl.segment_color2d_slic_features_model_graphcut(img, model, TUTORIAL, sp_size=12, debug_visual={})
        np.testing.assert_array_equal(segm, segm_g)
        np.testing.assert_allclose(soft, soft_g, rtol=0, atol=soft_tol)


def test_colour_space_set_replays_as_cuda_graph():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    feats = {'color_hsv': ('mean', 'median'), 'color': ('mean', 'meanGrad')}      # D = 12 <= 16: one-kernel device GMM
    img, img2 = synth_regions(88, 104, seed=75)[0], synth_regions(88, 104, seed=76)[0]
    pl.USE_CUDA_GRAPHS = False
    try:
        eager2 = pl.pipe_color2d_slic_features_model_graphcut(img2, 3, feats, sp_size=11)
    finally:
        pl.USE_CUDA_GRAPHS = True
    outs = []
    captured0 = eng.graphs_captured
    for i in range(3):          # eager, capture, replay
        n0 = eng.lib.isb_launch_count()
        outs.append(pl.pipe_color2d_slic_features_model_graphcut(img, 3, feats, sp_size=11))
        if i == 1:
            assert eng.graphs_captured > captured0, 'no CUDA graph was captured'
            captured1 = eng.graphs_captured
        if i == 2:
            assert eng.graphs_captured == captured1, 'the third run captured again instead of replaying'
            assert eng.lib.isb_launch_count() > n0, 'the replay reported no kernels'
    for segm, soft in outs[1:]:
        np.testing.assert_array_equal(segm, outs[0][0])
        np.testing.assert_array_equal(soft.view(np.int64), outs[0][1].view(np.int64))
    segm2, soft2 = pl.pipe_color2d_slic_features_model_graphcut(img2, 3, feats, sp_size=11)
    assert eng.graphs_captured == captured1
    np.testing.assert_array_equal(segm2, eager2[0])
    np.testing.assert_array_equal(soft2.view(np.int64), eager2[1].view(np.int64))


def test_batch_and_group_equal_single_image_calls():
    from pyimsegm_b200 import pipelines as pl
    imgs = [synth_regions(80, 96, seed=s)[0] for s in (77, 78, 79)]
    batch = pl.segment_images_batch(imgs, 3, TUTORIAL, sp_size=11)
    for img, (segm, soft) in zip(imgs, batch):
        want = pl.pipe_color2d_slic_features_model_graphcut(img, 3, TUTORIAL, sp_size=11)
        np.testing.assert_array_equal(segm, want[0])
        np.testing.assert_array_equal(soft.view(np.int64), want[1].view(np.int64))
    _, forest = _host_models(imgs[0], TUTORIAL, 11)
    batch = pl.segment_images_batch(imgs, dict_features=TUTORIAL, sp_size=11, model_pipeline=forest)
    for img, (segm, soft) in zip(imgs, batch):
        want = pl.segment_color2d_slic_features_model_graphcut(img, forest, TUTORIAL, sp_size=11)
        np.testing.assert_array_equal(segm, want[0])
        np.testing.assert_array_equal(soft, want[1])
    _, list_fts = pl.estim_model_classes_group(imgs, 3, TUTORIAL, sp_size=11)
    for img, fts in zip(imgs, list_fts):
        slic, _ = pl.compute_color2d_superpixels_features(img, TUTORIAL, sp_size=11)
        np.testing.assert_allclose(fts, _reference_table(img, slic, TUTORIAL), rtol=1e-12, atol=0)


def test_thin_image_meangrad_raises_and_unknown_groups_take_the_general_path():
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.descriptors import compute_selected_features_color2d
    from pyimsegm_b200.superpixels import segment_slic_img2d
    for shape in ((1, 64, 3), (64, 1, 3)):
        with pytest.raises(ValueError):
            pl.compute_color2d_superpixels_features(np.full(shape, 0.5), {'color': ['meanGrad']}, sp_size=4)
        with pytest.raises(ValueError):
            compute_selected_features_color2d(np.full(shape, 0.5), np.zeros(shape[:2], dtype=int), {'color': ['meanGrad']})
    img = synth_regions(64, 72, seed=80)[0]
    want_slic = segment_slic_img2d(img, sp_size=10, relative_compact=0.2)
    for feats in ({'color_foo': ['mean']}, {'color': ['mean', 'foo']}):
        slic, got = pl.compute_color2d_superpixels_features(img, feats, sp_size=10)
        np.testing.assert_array_equal(slic, want_slic)
        np.testing.assert_allclose(got, _reference_table(img, want_slic, feats), rtol=1e-12, atol=0)
    # keys the pipelines do not take resident, through the numpy API: an unknown colour space and a key without '_' are the image
    # itself, and a texture key without the suffix 'short' is the full bank
    for key, prefix in (('color_foo', 'foo'), ('colorX', 'rgb')):
        got, names = compute_selected_features_color2d(img, want_slic, {key: FLAGS})
        _compare_group(got, _colour_reference(img, want_slic, key, FLAGS), 'color', 9)
        assert names == ['%s-ch%i_%s' % (prefix, c + 1, f) for f in FLAGS for c in range(3)]
    got, names = compute_selected_features_color2d(img, want_slic, {'tLM_long': ('mean', 'median')})
    want, want_names = _lm_reference(img, want_slic, ('mean', 'median'), 'long')
    assert names == want_names and got.shape == (want_slic.max() + 1, 20 * 6)
    _column_scaled_close(got, want)
