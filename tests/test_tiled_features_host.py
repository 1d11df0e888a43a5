"""
Which feature dictionaries and class models the banded path (pyimsegm_b200/tiled.py) takes, and the raw rows a band keeps for
them.  Host logic only: every refusal happens before any engine call.
"""
import itertools

import numpy as np
import pytest


def _no_engine(monkeypatch):
    from pyimsegm_b200 import tiled

    def no_engine(*args, **kwargs):
        raise AssertionError('the banded path reached the engine')

    monkeypatch.setattr(tiled, 'get_engine', no_engine)
    return tiled


def test_banded_predicate_every_group_and_statistic():
    from pyimsegm_b200.descriptors import NAMES_FEATURE_FLAGS, RESIDENT_FEATURE_GROUPS, flags_are_banded
    for group, flag in itertools.product(RESIDENT_FEATURE_GROUPS, NAMES_FEATURE_FLAGS):
        assert flags_are_banded({group: [flag]}) == (flag != 'median'), (group, flag)
        assert flags_are_banded({group: ['mean', flag]}) == (flag != 'median'), (group, flag)
    assert flags_are_banded({g: [f for f in NAMES_FEATURE_FLAGS if f != 'median'] for g in RESIDENT_FEATURE_GROUPS})
    assert flags_are_banded({'color': ()})
    for refused in ({}, {'color_foo': ['mean']}, {'color': ['mean', 'foo']}, {'tLM_long': ['mean']}, {'gray': ['mean']},
                    {'color': ['mean'], 'tLM_short': ['mean', 'median']}):
        assert not flags_are_banded(refused), refused


def test_native_predicate_keeps_its_answers():
    from pyimsegm_b200.descriptors import flags_are_native
    assert flags_are_native({'color': ['mean', 'std', 'energy'], 'tLM_short': ['mean']})
    assert not flags_are_native({'color': ['median']}) and not flags_are_native({'color_hsv': ['mean']})
    assert not flags_are_native({'color': ['meanGrad']}) and not flags_are_native({'tLM': ['meanGrad']})


@pytest.mark.parametrize('fts', [{'color': ['mean', 'median']}, {'color_hsv': ['median']}, {'tLM': ['mean', 'median']},
                                 {'color_foo': ['mean']}, {'color': ['mean', 'foo']}, {'gray': ['mean']}])
def test_banded_pipelines_refuse_before_any_engine_call(monkeypatch, fts):
    tiled = _no_engine(monkeypatch)
    with pytest.raises(NotImplementedError):
        tiled.pipe_color2d_slic_features_model_graphcut_tiled(np.zeros((32, 32, 3)), 2, fts)
    with pytest.raises(NotImplementedError):
        tiled.segment_color2d_slic_features_model_graphcut_tiled(np.zeros((32, 32, 3)), object(), fts)


@pytest.mark.parametrize('kwargs', [dict(pca_coef='mle'), dict(pca_coef=True), dict(pca_coef=1.5), dict(pca_coef=10),
                                    dict(estim_model=None), dict(nb_classes=9)])
def test_unsupported_class_models_refused_before_any_engine_call(monkeypatch, kwargs):
    tiled = _no_engine(monkeypatch)
    kwargs = dict(kwargs)
    nb_classes = kwargs.pop('nb_classes', 2)
    with pytest.raises(NotImplementedError):
        tiled.pipe_color2d_slic_features_model_graphcut_tiled(np.zeros((32, 32, 3)), nb_classes, {'color': ['mean', 'std']}, **kwargs)


def test_raw_margin_arithmetic():
    from pyimsegm_b200.descriptors import native_feature_layout
    from pyimsegm_b200.tiled import LM_ROW_MARGIN, banded_raw_margin
    assert LM_ROW_MARGIN == 616

    def margin(fts):
        return banded_raw_margin(native_feature_layout(fts)[0])

    assert margin({'tLM_short': ['mean', 'meanGrad']}) == 617
    assert margin({'color': ['mean'], 'tLM': ['meanGrad']}) == 617
    assert margin({'tLM': ['mean', 'std'], 'tLM_short': ['energy', 'meanGrad']}) == 617
    assert margin({'tLM_short': ['mean', 'energy']}) == 616
    assert margin({'color': ['meanGrad'], 'tLM': ['mean']}) == 616
    assert margin({'color': ['mean', 'meanGrad'], 'color_lab': ['meanGrad']}) == 0


def test_band_rows_for_the_gradient():
    from pyimsegm_b200.tiled import gradient_rows, plan_bands
    bands = plan_bands(100, 3, 5, 4)
    assert [gradient_rows(b, 100) for b in bands] == [(0, 35), (33, 69), (67, 100)]
    for b in bands:             # the blur's raw rows always hold the gradient's extra row
        lo, hi = gradient_rows(b, 100)
        assert b.up_lo <= lo and hi <= b.up_hi
