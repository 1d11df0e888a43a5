"""
z-slab mode of one gray volume (pyimsegm_b200/tiled.py: slic3d_tiled, gray_stats_tiled and the two volume pipelines) against the
oracle and against the single-GPU volume path.  On one GPU the slabs live side by side in one process (``bands_per_rank``) and are
merged by isb_combine -- the same integer sum the NCCL all_reduce does between GPUs; the real 2-GPU run is
tests/run_tiled_volume_ranks.py under torchrun (spawned by test_two_ranks_nccl_volume when the box has two GPUs).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

FEATURES = {'color': ['mean', 'std', 'energy']}


@pytest.fixture(scope='module')
def eng():
    from pyimsegm_b200.engine import get_engine
    return get_engine()


def _blobs(shape, seed, noise=0.08):
    rng = np.random.RandomState(seed)
    zz, yy, xx = np.mgrid[:shape[0], :shape[1], :shape[2]]
    vol = 0.3 + 0.4 * ((xx > shape[2] // 2) ^ (yy > shape[1] // 3)) + 0.15 * (zz > shape[0] // 2)
    return np.clip(vol + rng.normal(0, noise, shape), 0, 1)


def _as(vol, dtype):
    if dtype == np.uint8:
        return (vol * 255).astype(np.uint8)
    if dtype == np.uint16:
        return (vol * 65535).astype(np.uint16)
    return vol.astype(dtype)


#: case -> (shape, dtype, sp_size, sp_regul, spacing, slab counts)
CASES = {
    'u8_aniso': ((30, 60, 52), np.uint8, 10, 0.3, (12, 1, 1), (2, 3, 4)),
    'u16_iso': ((32, 36, 40), np.uint16, 8, 0.3, (1, 1, 1), (2, 3, 4)),
    'f32_iso': ((27, 40, 30), np.float32, 7, 0.25, (1, 1, 1), (2, 3, 4)),         # D not divisible by 2 or 4
    'f64_aniso': ((41, 50, 44), np.float64, 12, 0.2, (2, 1, 1), (2, 3, 4)),       # D prime
    'thin_slabs': ((24, 30, 30), np.float64, 9, 0.2, (1, 1, 1), (6, 8, 12)),      # slabs of 2-4 slices, halo of 10+
    'blur_border': ((60, 24, 24), np.float32, 6, 0.3, (1, 1, 1), (3, 5)),         # interior slabs whose raw slab ends inside
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_slab_label_volumes_are_bit_exact(oracle, eng, case):
    from pyimsegm_b200.superpixels import slic3d_params
    from pyimsegm_b200.tiled import slic3d_tiled
    shape, dtype, sp_size, regul, spacing, slab_counts = CASES[case]
    vol = _as(_blobs(shape, seed=len(case)), dtype)
    n_seg, compact = slic3d_params(shape, sp_size, regul, spacing)
    want_km = oracle.slic3d(vol, n_seg, compact, spacing, enforce_conn=False)
    want = oracle.slic3d(vol, n_seg, compact, spacing)
    whole_km, _ = eng.slic3d(eng.to_device(vol, 'test_volume'), n_seg, compact, spacing, enforce_connectivity=False)
    assert np.array_equal(eng.to_host(whole_km), want_km)
    whole, _ = eng.slic3d(eng.to_device(vol, 'test_volume'), n_seg, compact, spacing)
    assert np.array_equal(eng.to_host(whole), want)
    for n in slab_counts:
        res = slic3d_tiled(vol, n_seg, compact, spacing, bands_per_rank=n, eng=eng, enforce_connectivity=False)
        assert not res.fell_back
        assert np.array_equal(eng.to_host(res.d_seg), want_km), (case, n)
        if case == 'blur_border' and n == 5:
            # interior slabs: one blurs from the volume's lower border (reflected there), one with both raw ends inside the volume
            ends = [(bd.raw_lo == 0, bd.raw_hi == shape[0]) for bd in res.bands[1:-1]]
            assert (True, False) in ends and (False, False) in ends
        res = slic3d_tiled(vol, n_seg, compact, spacing, bands_per_rank=n, eng=eng)
        assert np.array_equal(eng.to_host(res.d_seg), want), (case, n)
        assert int(eng.to_host(res.d_n_labels)[0]) == want.max() + 1


def test_orphans_beyond_the_halo_fall_back(oracle, eng):
    """NaN voxels have a NaN distance to every centre: no window ever takes them, they keep label 0 -- orphans far from cluster 0's
    centre in the upper slabs.  The device check must notice and the whole-volume sweeps must give the oracle's answer."""
    from pyimsegm_b200.superpixels import slic3d_params
    from pyimsegm_b200.tiled import slic3d_tiled
    shape, spacing = (36, 30, 28), (2, 1, 1)
    vol = _blobs(shape, 3)
    vol[24:, 10:20] = np.nan
    n_seg, compact = slic3d_params(shape, 8, 0.3, spacing)
    want_km = oracle.slic3d(vol, n_seg, compact, spacing, enforce_conn=False)
    assert (want_km[24:, 10:20] == 0).all()
    res = slic3d_tiled(vol, n_seg, compact, spacing, bands_per_rank=3, eng=eng, enforce_connectivity=False)
    assert res.fell_back
    assert np.array_equal(eng.to_host(res.d_seg), want_km)
    res = slic3d_tiled(vol, n_seg, compact, spacing, bands_per_rank=3, eng=eng, enforce_connectivity=False, defer_check=True)
    assert not res.fell_back and int(eng.to_host(res.d_err)[0]) > 0


@pytest.mark.parametrize('dtype', [np.uint8, np.float32, np.float64])
def test_slab_statistics(oracle, eng, dtype):
    """mean / std / energy over the slabs against gray_table on the whole volume and the float64 oracle, NaN voxels counting 0"""
    from pyimsegm_b200.superpixels import slic3d_params
    from pyimsegm_b200.tiled import gray_stats_tiled, slic3d_tiled
    shape, spacing = (33, 48, 40), (12, 1, 1)
    vol = _as(_blobs(shape, 9), dtype)
    if dtype != np.uint8:
        vol[0, :2, :3] = np.nan             # inside cluster 0's reach: unassigned, but no orphan beyond the halo
        vol[20, 30, 31] = np.nan
    n_seg, compact = slic3d_params(shape, 10, 0.3, spacing)
    d_vol = eng.to_device(vol, 'test_volume')
    for n in (1, 3, 4):
        res = slic3d_tiled(vol, n_seg, compact, spacing, bands_per_rank=n, eng=eng)
        seg = eng.to_host(res.d_seg).copy()
        nb = int(seg.max()) + 1
        for flags in (('mean', 'std', 'energy'), ('std', ), ('mean', 'energy')):
            got = eng.to_host(gray_stats_tiled(res, vol.dtype, flags, eng=eng)).copy()
            want = eng.to_host(eng.gray_table(d_vol, res.d_seg, int(res.nb_bound), list(flags))).copy()
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
            assert not np.isnan(got).any() and not np.signbit(got).any()
        img = np.nan_to_num(vol.astype(np.float32))
        mean = oracle.gray3d_stat(img, seg, 0)
        ref = np.stack([mean, np.sqrt(oracle.gray3d_stat(img, seg, 2, mean.astype(np.float32))), oracle.gray3d_stat(img, seg, 1)], 1)
        got = eng.to_host(gray_stats_tiled(res, vol.dtype, ('mean', 'std', 'energy'), eng=eng)).copy()
        np.testing.assert_allclose(got[:nb], ref, rtol=1e-9, atol=1e-9)


def _train_models():
    """a GMM pipeline and a random forest (classes 3 and 7) fitted by the caller on the standardised features of a training volume"""
    from sklearn import ensemble, mixture, pipeline, preprocessing
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    from pyimsegm_b200.superpixels import slic3d_params
    eng = get_engine()
    train = _as(_blobs((16, 60, 52), 11), np.uint8)
    n_seg, compact = slic3d_params(train.shape, 10, 0.3, (2, 1, 1))
    d_seg, d_n = eng.slic3d(eng.to_device(train, 'test_volume'), n_seg, compact, (2, 1, 1))
    n = int(eng.to_host(d_n)[0])
    feat = eng.gray_table(eng.to_device(train, 'test_volume'), d_seg, eng.slic_label_bound(train.size, 1, n_seg), pl._volume_flags(FEATURES))
    x = eng.to_host(eng.standard_scaler(feat, d_n)[0][:n]).copy()
    gmm = pipeline.Pipeline([('std_scaler', preprocessing.StandardScaler()),
                             ('model', mixture.GaussianMixture(2, covariance_type='full', random_state=0))]).fit(x)
    forest = ensemble.RandomForestClassifier(n_estimators=12, max_depth=6, random_state=0).fit(x, np.where(x[:, 0] > np.median(x[:, 0]), 7, 3))
    return {'gmm': gmm, 'forest': forest}


def _resident(eng, vol, model, spacing, sp_size, sp_regul, gc_regul):
    from pyimsegm_b200 import pipelines as pl
    hosts, done = eng.download(pl.segment_resident_volume(eng.to_device(vol, 'test_volume'), model, FEATURES, spacing, sp_size, sp_regul,
                                                          gc_regul))
    done.synchronize()
    return [h.numpy() for h in hosts]


VOLS = (((20, 60, 52), np.uint8, (2, 1, 1), 10, 0.3), ((17, 70, 64), np.float32, (12, 1, 1), 15, 0.2))


@pytest.mark.parametrize('model_name', ['gmm', 'forest'])
def test_caller_model_pipeline_matches_resident_volume(eng, model_name):
    from pyimsegm_b200 import class_models
    from pyimsegm_b200.tiled import segment_gray3d_slic_features_model_graphcut_tiled
    model = _train_models()[model_name]
    assert class_models.compile_model(model) is not None
    classes = getattr(model, 'classes_', None)
    for i, (shape, dtype, spacing, sp_size, regul) in enumerate(VOLS):
        vol = _as(_blobs(shape, 21 + i), dtype)
        want_segm, want_soft = _resident(eng, vol, model, spacing, sp_size, regul, 0.1)
        if classes is not None:
            want_segm = np.asarray(classes)[want_segm]
        for n in (1, 3):
            segm, soft, (lo, hi) = segment_gray3d_slic_features_model_graphcut_tiled(vol, model, FEATURES, spacing, sp_size, regul, 0.1,
                                                                                     bands_per_rank=n)
            assert (lo, hi) == (0, shape[0]) and segm.shape == shape and soft.shape == shape + (2, )
            assert np.array_equal(segm, want_segm), (model_name, shape, n)
            np.testing.assert_allclose(soft, want_soft, rtol=1e-9, atol=1e-9)
    if model_name == 'forest':
        assert set(np.unique(segm)) <= {3, 7}


def test_host_model_pipeline_matches_resident_volume(eng):
    """a model compile_model does not take: its predict_proba runs on the host of every rank"""
    from pyimsegm_b200.tiled import segment_gray3d_slic_features_model_graphcut_tiled

    class Logistic(object):
        classes_ = np.array([5, 9])

        def predict_proba(self, features):
            p = 1 / (1 + np.exp(features[:, 0]))
            return np.stack([p, 1 - p], 1)

    model = Logistic()
    shape, dtype, spacing, sp_size, regul = VOLS[0]
    vol = _as(_blobs(shape, 25), dtype)
    want_segm, want_soft = _resident(eng, vol, model.predict_proba, spacing, sp_size, regul, 0.1)
    segm, soft, _ = segment_gray3d_slic_features_model_graphcut_tiled(vol, model, FEATURES, spacing, sp_size, regul, 0.1, bands_per_rank=3)
    assert np.array_equal(segm, model.classes_[want_segm])
    np.testing.assert_allclose(soft, want_soft, rtol=1e-9, atol=1e-9)


def test_device_fit_pipeline_matches_resident_volume(eng):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.tiled import pipe_gray3d_slic_features_model_graphcut_tiled
    for i, (shape, dtype, spacing, sp_size, regul) in enumerate(VOLS):
        vol = _as(_blobs(shape, 31 + i), dtype)
        want_segm, want_soft = _resident(eng, vol, pl._fit_model(2, True), spacing, sp_size, regul, 0.1)
        for n in (1, 3):
            segm, soft, (lo, hi) = pipe_gray3d_slic_features_model_graphcut_tiled(vol, 2, FEATURES, spacing, sp_size, regul, 0.1,
                                                                                  bands_per_rank=n)
            assert (lo, hi) == (0, shape[0])
            assert np.array_equal(segm, want_segm), (shape, n)
            np.testing.assert_allclose(soft, want_soft, rtol=1e-9, atol=1e-9)
        full, none, _ = pipe_gray3d_slic_features_model_graphcut_tiled(vol, 2, FEATURES, spacing, sp_size, regul, 0.1, bands_per_rank=2,
                                                                       want_soft=False, gather_segm=True)
        assert none is None and np.array_equal(full, want_segm)


def test_pipeline_orphans_redo_the_whole_volume(eng):
    """NaN voxels beyond cluster 0's halo: the pipeline reads the orphan count with its results and redoes the front"""
    from pyimsegm_b200.tiled import segment_gray3d_slic_features_model_graphcut_tiled
    model = _train_models()['forest']
    vol = _blobs((36, 30, 28), 3)
    vol[24:, 10:20] = np.nan
    want_segm, want_soft = _resident(eng, vol, model, (2, 1, 1), 8, 0.3, 0.1)
    segm, soft, _ = segment_gray3d_slic_features_model_graphcut_tiled(vol, model, FEATURES, (2, 1, 1), 8, 0.3, 0.1, bands_per_rank=3)
    assert np.array_equal(segm, model.classes_[want_segm])
    np.testing.assert_allclose(soft, want_soft, rtol=1e-9, atol=1e-9)


def test_two_ranks_nccl_volume():
    """the slab checks with two processes, one GPU each, merged by NCCL all_reduce / broadcast"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs (on a host with two: python -m pytest tests -m gpu -k two_ranks)')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1',
           '--master-port', '29573', os.path.join(ROOT, 'tests', 'run_tiled_volume_ranks.py')]
    out = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = out.stdout.decode(errors='replace')
    assert out.returncode == 0, text[-3000:]
    assert 'TILED-VOLUME-RANKS-OK' in text, text[-3000:]
