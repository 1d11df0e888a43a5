"""
The banded path (pyimsegm_b200/tiled.py) with the colour-space groups, meanGrad, every device-fitted class model and a caller-fitted
model, against the single-image drivers.  Statistics are compared on the same label map (``res.d_seg``); the bands add their own rounded sums, the single image rounds
its whole sums once, so a column may differ in its last bits and keeps a bound.  On one GPU the bands live side by side in one process; the real multi-GPU run
is tests/run_tiled_features_ranks.py under torchrun (spawned by test_two_ranks_nccl_features on a host with two GPUs).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, synth_regions

pytestmark = pytest.mark.gpu

ALL_BANDED = ('mean', 'std', 'energy', 'meanGrad')
COLOUR_GROUPS = {k: ALL_BANDED for k in ('color', 'color_hsv', 'color_luv', 'color_lab', 'color_hed', 'color_xyz')}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _as_dtype(img, dtype):
    if dtype == np.uint8:
        return (img * 255).round().astype(np.uint8)
    if dtype == np.uint16:
        return (img * 65535).round().astype(np.uint16)
    return img.astype(dtype)


def _whole_table(eng, img, res, fts):
    from pyimsegm_b200.descriptors import device_feature_table, native_feature_layout
    nb = int(res.nb_bound)
    feat = eng.buf('feat_whole_test', (nb, native_feature_layout(fts)[1]), eng.torch.float64)
    device_feature_table(eng, eng.to_device(img, 'image'), res.d_seg, nb, fts, feat)
    return eng.to_host(feat).copy()


def _close_per_column(got, want, rel):
    scale = np.maximum(np.abs(want).max(axis=0), 1e-300)
    err = np.abs(got - want) / scale
    assert err.max() <= rel, 'column %d off by %.3g of its largest value' % (int(err.max(axis=0).argmax()), err.max())


@pytest.mark.parametrize('dtype', [np.uint8, np.uint16, np.float32, np.float64])
def test_banded_colour_groups_match_whole_image(eng, dtype):
    """every colour space with mean / std / energy / meanGrad over 2, 3 and 5 bands of a ragged image; an f32 image keeps its
    f32 gradient on both sides"""
    from pyimsegm_b200.descriptors import native_feature_layout
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import features_tiled, slic_tiled
    img = _as_dtype(synth_regions(397, 263, seed=41)[0], dtype)        # 397 rows: no band count divides it
    layout, ncol = native_feature_layout(COLOUR_GROUPS)
    n_seg, compact = slic_params(img.shape[:2], 17, 0.25)
    for n_bands in (2, 3, 5):
        res = slic_tiled(img, n_seg, compact, bands_per_rank=n_bands, eng=eng)
        feat, centres = features_tiled(res, img.dtype, 3, layout, ncol, eng=eng)
        got = eng.to_host(feat).copy()
        got_centres = eng.to_host(centres).copy()
        want = _whole_table(eng, img, res, COLOUR_GROUPS)
        _close_per_column(got, want, 1e-12)
        nb = int(eng.to_host(res.d_n_labels)[0])
        seg = eng.to_host(res.d_seg)
        yy, xx = np.mgrid[:seg.shape[0], :seg.shape[1]]
        cnt = np.bincount(seg.ravel(), minlength=nb)
        np.testing.assert_allclose(got_centres[:nb, 0], np.bincount(seg.ravel(), yy.ravel(), nb) / cnt, rtol=1e-13)
        np.testing.assert_allclose(got_centres[:nb, 1], np.bincount(seg.ravel(), xx.ravel(), nb) / cnt, rtol=1e-13)


def test_banded_colour_groups_with_thin_bands(eng):
    """bands of 6 rows: the gradient's halo row of every band is another band's owned row; the first and last bands end at the
    image borders, where the gradient is one-sided"""
    from pyimsegm_b200.descriptors import native_feature_layout
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import features_tiled, slic_tiled
    img = synth_regions(90, 256, seed=42, cell=16)[0]
    fts = {'color': ('meanGrad', ), 'color_lab': ('mean', 'meanGrad'), 'color_hed': ('std', 'meanGrad')}
    layout, ncol = native_feature_layout(fts)
    n_seg, compact = slic_params(img.shape[:2], 8, 0.2)
    res = slic_tiled(img, n_seg, compact, bands_per_rank=15, eng=eng)
    assert all(b.own_hi - b.own_lo == 6 for b in res.bands)
    got = eng.to_host(features_tiled(res, img.dtype, 3, layout, ncol, eng=eng)[0]).copy()
    _close_per_column(got, _whole_table(eng, img, res, fts), 1e-12)


def _texture_image():
    rng = np.random.RandomState(5)
    return synth_regions(2000, 192, seed=21)[0] + 0.05 * rng.standard_normal((2000, 192, 3))


@pytest.mark.parametrize('bank', ['normal', 'short'])
def test_banded_texture_meangrad_matches_materialised_route(eng, bank):
    """texture meanGrad over 3 bands whose slabs end inside the image against device_lm_materialised; the mean columns of the same
    group still come from the fused kernel"""
    from pyimsegm_b200.descriptors import native_feature_layout
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.texture import device_lm_features, device_lm_materialised
    from pyimsegm_b200.tiled import banded_raw_margin, features_tiled, slic_tiled
    img = _texture_image()
    key = 'tLM_short' if bank == 'short' else 'tLM'
    fts = {key: ('mean', 'meanGrad')}
    layout, ncol = native_feature_layout(fts)
    n_seg, compact = slic_params(img.shape[:2], 24, 0.2)
    res = slic_tiled(img, n_seg, compact, bands_per_rank=3, eng=eng, raw_margin=banded_raw_margin(layout))
    assert res.bands[1].up_lo > 0 and res.bands[1].up_hi < 2000
    got = eng.to_host(features_tiled(res, img.dtype, 3, layout, ncol, eng=eng)[0]).copy().reshape(-1, ncol // 6, 2, 3)
    nb = int(res.nb_bound)
    d_img = eng.to_device(img, 'image')
    mat = eng.buf('feat_mat_test', (nb, ncol), eng.torch.float64)
    device_lm_materialised(eng, d_img, res.d_seg, nb, ['mean', 'meanGrad'], bank, mat, 0)
    want = eng.to_host(mat).copy().reshape(-1, ncol // 6, 2, 3)
    assert np.abs(want[:, :, 1]).max() > 0.01
    _close_per_column(got[:, :, 1].reshape(nb, -1), want[:, :, 1].reshape(nb, -1), 1e-9)
    fused = eng.to_host(device_lm_features(eng, d_img, res.d_seg, nb, ('mean', ), bank)[0]).copy()
    np.testing.assert_allclose(got[:, :, 0].reshape(nb, -1), fused, rtol=1e-7, atol=1e-9)


def test_banded_texture_meangrad_needs_its_extra_row(eng):
    from pyimsegm_b200.superpixels import slic_params
    from pyimsegm_b200.tiled import LM_ROW_MARGIN, slic_tiled, texture_gradient_tiled
    img = _texture_image()
    n_seg, compact = slic_params(img.shape[:2], 24, 0.2)
    res = slic_tiled(img, n_seg, compact, bands_per_rank=3, eng=eng, raw_margin=LM_ROW_MARGIN)
    feat = eng.buf('feat_margin_test', (int(res.nb_bound), 45), eng.torch.float64)
    with pytest.raises(ValueError):
        texture_gradient_tiled(res, img.dtype, 'short', eng=eng, feat=feat)


PIPE_FTS = {'color': ('mean', 'meanGrad'), 'color_hsv': ('mean', 'std'), 'color_lab': ('meanGrad', )}


@pytest.mark.parametrize('model', [dict(), dict(estim_model='kmeans'), dict(estim_model='BGM'), dict(pca_coef=0.95)])
def test_banded_pipeline_colour_spaces_and_models(eng, model):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.tiled import pipe_color2d_slic_features_model_graphcut_tiled
    img = synth_regions(600, 512, seed=17)[0]
    segm, soft = pl.pipe_color2d_slic_features_model_graphcut(img, 3, PIPE_FTS, sp_size=20, sp_regul=0.2, gc_regul=1., **model)
    for n_bands in (1, 3):
        got, got_soft, (lo, hi) = pipe_color2d_slic_features_model_graphcut_tiled(img, 3, PIPE_FTS, sp_size=20, sp_regul=0.2,
                                                                                 bands_per_rank=n_bands, **model)
        assert (lo, hi) == (0, 600)
        assert np.array_equal(got, segm), 'bands=%d' % n_bands
        np.testing.assert_allclose(got_soft, soft, rtol=1e-6, atol=1e-6)


def _group_images():
    return [synth_regions(384, 320, seed=s)[0] for s in (51, 52)], synth_regions(600, 448, seed=53)


def test_banded_segment_with_group_gmm(eng):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.tiled import segment_color2d_slic_features_model_graphcut_tiled
    train, (img, _) = _group_images()
    model, _ = pl.estim_model_classes_group(train, 3, PIPE_FTS, sp_size=20, sp_regul=0.2)
    segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, model, PIPE_FTS, sp_size=20, sp_regul=0.2)
    for n_bands in (1, 3):
        got, got_soft, _ = segment_color2d_slic_features_model_graphcut_tiled(img, model, PIPE_FTS, sp_size=20, sp_regul=0.2,
                                                                              bands_per_rank=n_bands)
        assert np.array_equal(got, segm), 'bands=%d' % n_bands
        np.testing.assert_allclose(got_soft, soft, rtol=0, atol=1e-9)


class _HostOnly(object):
    """a duck-typed model that class_models.compile_model does not take"""

    def __init__(self, model):
        self.model, self.classes_ = model, model.classes_

    def predict_proba(self, features):
        return self.model.predict_proba(features)


def test_banded_segment_with_random_forest_and_host_model(eng):
    from sklearn.ensemble import RandomForestClassifier
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.class_models import compile_model
    from pyimsegm_b200.tiled import segment_color2d_slic_features_model_graphcut_tiled
    train, (img, _) = _group_images()
    feats, labels = [], []
    for i, im in enumerate(train):
        annot = np.array([2, 5, 7])[synth_regions(384, 320, seed=51 + i)[1]]
        _, f, lab = pl.wrapper_compute_color2d_slic_features_labels((im, annot), 20, 0.2, PIPE_FTS, 0.9)
        feats.append(f[lab >= 0])
        labels.append(lab[lab >= 0])
    forest = RandomForestClassifier(n_estimators=12, max_depth=8, random_state=0).fit(np.vstack(feats), np.hstack(labels))
    assert list(forest.classes_) == [2, 5, 7]
    host = _HostOnly(forest)
    assert compile_model(forest) is not None and compile_model(host) is None
    for model, exact in ((forest, True), (host, False)):
        segm, soft = pl.segment_color2d_slic_features_model_graphcut(img, model, PIPE_FTS, sp_size=20, sp_regul=0.2)
        assert set(np.unique(segm)) <= {2, 5, 7}
        for n_bands in (1, 3):
            got, got_soft, _ = segment_color2d_slic_features_model_graphcut_tiled(img, model, PIPE_FTS, sp_size=20, sp_regul=0.2,
                                                                                  bands_per_rank=n_bands)
            assert np.array_equal(got, segm), (type(model).__name__, n_bands)
            if exact:
                assert np.array_equal(got_soft, soft)


def test_two_ranks_nccl_features():
    """the colour-space, texture-meanGrad and caller-fitted-model checks with two processes, one GPU each, over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs (on a host with two: python -m pytest tests -m gpu -k two_ranks)')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1',
           '--master-port', '29573', os.path.join(ROOT, 'tests', 'run_tiled_features_ranks.py')]
    out = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    text = out.stdout.decode(errors='replace')
    assert out.returncode == 0, text[-3000:]
    assert 'TILED-FEATURES-RANKS-OK' in text, text[-3000:]
