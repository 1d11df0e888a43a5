"""
The z-slab path of one gray volume (pyimsegm_b200/tiled.py: slic3d_tiled and the two volume pipelines): which inputs it refuses,
before any engine call, and how it cuts a volume into slabs.  Host logic only.
"""
import numpy as np
import pytest


def _no_engine(monkeypatch):
    from pyimsegm_b200 import tiled

    def no_engine(*args, **kwargs):
        raise AssertionError('the slab path reached the engine')

    monkeypatch.setattr(tiled, 'get_engine', no_engine)
    return tiled


def _both(tiled, volume, fts, **kwargs):
    """the two volume pipelines with the same arguments"""
    yield lambda: tiled.pipe_gray3d_slic_features_model_graphcut_tiled(volume, 2, fts, **kwargs)
    yield lambda: tiled.segment_gray3d_slic_features_model_graphcut_tiled(volume, object(), fts, **kwargs)


@pytest.mark.parametrize('fts', [{'color': ['mean', 'median']}, {'color': ['median']}, {'color': ['mean', 'meanGrad']},
                                 {'tLM_short': ['mean']}, {'color': ['mean'], 'tLM': ['mean']}, {'gray': ['mean']},
                                 {'color': ['mean', 'foo']}, {}, {'color': []}])
def test_unsupported_features_refused_before_any_engine_call(monkeypatch, fts):
    tiled = _no_engine(monkeypatch)
    for call in _both(tiled, np.zeros((8, 32, 32)), fts):
        with pytest.raises(NotImplementedError):
            call()


def test_more_classes_than_the_device_fit_takes_are_refused(monkeypatch):
    tiled = _no_engine(monkeypatch)
    with pytest.raises(NotImplementedError):
        tiled.pipe_gray3d_slic_features_model_graphcut_tiled(np.zeros((8, 32, 32)), 9, {'color': ['mean']})


@pytest.mark.parametrize('case', ['2d', '4d', 'more_slabs_than_slices', 'empty_last_slab', 'regul', 'sp_too_large'])
def test_bad_volumes_refused_before_any_engine_call(monkeypatch, case):
    tiled = _no_engine(monkeypatch)
    volume, kwargs = np.zeros((8, 32, 32)), dict(spacing=(1, 1, 1), sp_size=5)
    if case == '2d':
        volume = np.zeros((32, 32))
    elif case == '4d':
        volume = np.zeros((4, 32, 32, 1))
    elif case == 'more_slabs_than_slices':
        kwargs['bands_per_rank'] = 9
    elif case == 'empty_last_slab':
        volume, kwargs['bands_per_rank'] = np.zeros((7, 32, 32)), 5      # ceil(7 / 5) = 2 slices per slab leaves the fifth empty
    elif case == 'regul':
        kwargs['sp_regul'] = 0.
    else:
        kwargs['sp_size'] = 100
    for call in _both(tiled, volume, {'color': ['mean', 'std']}, **kwargs):
        with pytest.raises(ValueError):
            call()


def _check_plan(shape, n_segments, spacing, n_slabs):
    from pyimsegm_b200.engine import gaussian_half_kernel, slic_seed_grid3d
    from pyimsegm_b200.tiled import slab_plan
    D = shape[0]
    bands, seeds, steps, halves = slab_plan(shape, n_segments, spacing, n_slabs)
    want_seeds, want_steps = slic_seed_grid3d(shape, n_segments)
    assert np.array_equal(seeds, want_seeds) and steps == want_steps
    r_z = gaussian_half_kernel(1.0 / spacing[0])[1]
    assert halves[0][1] == r_z
    halo = 2 * steps[0] + 1
    per = -(-D // n_slabs)
    assert [(b.own_lo, b.own_hi) for b in bands] == [(i * per, min((i + 1) * per, D)) for i in range(n_slabs)]
    for b in bands:
        assert (b.km_lo, b.km_hi) == (max(b.own_lo - halo, 0), min(b.own_hi + halo, D))
        assert (b.raw_lo, b.raw_hi) == (max(b.km_lo - r_z, 0), min(b.km_hi + r_z, D))
        assert (b.up_lo, b.up_hi) == (b.raw_lo, b.raw_hi)
    return bands, steps, r_z


def test_slab_plan_anisotropic_spacing():
    """spacing (12, 1, 1): the z-blur's sigma is 1/12, radius 0 -- the raw slab is the k-means slab"""
    bands, steps, r_z = _check_plan((120, 64, 64), 600, (12, 1, 1), 4)
    assert r_z == 0 and steps[0] == 9
    assert all((b.raw_lo, b.raw_hi) == (b.km_lo, b.km_hi) for b in bands)
    assert (bands[1].own_lo, bands[1].km_lo, bands[1].own_hi, bands[1].km_hi) == (30, 11, 60, 79)


def test_slab_plan_isotropic_spacing():
    """spacing (1, 1, 1): radius 4, interior slabs reach 4 slices past their k-means slab on both sides"""
    bands, steps, r_z = _check_plan((96, 40, 40), 96, (1, 1, 1), 4)
    assert r_z == 4 and steps[0] == 12
    assert (bands[1].own_lo, bands[1].km_lo, bands[1].raw_lo) == (24, 0, 0)
    assert (bands[1].own_hi, bands[1].km_hi, bands[1].raw_hi) == (48, 73, 77)
    assert (bands[2].km_lo, bands[2].raw_lo, bands[2].raw_hi) == (23, 19, 96)


def test_slab_plan_ragged_and_one_slice_slabs():
    bands, _, _ = _check_plan((10, 30, 30), 20, (2, 1, 1), 3)
    assert [(b.own_lo, b.own_hi) for b in bands] == [(0, 4), (4, 8), (8, 10)]
    bands, steps, _ = _check_plan((6, 30, 30), 30, (1, 1, 1), 6)
    assert all(b.own_hi - b.own_lo == 1 for b in bands)
    assert all((b.km_lo, b.km_hi) == (max(b.own_lo - 2 * steps[0] - 1, 0), min(b.own_hi + 2 * steps[0] + 1, 6)) for b in bands)
    with pytest.raises(ValueError):
        _check_plan((6, 30, 30), 30, (1, 1, 1), 7)
