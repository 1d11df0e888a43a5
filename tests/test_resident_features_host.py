"""
Which feature dictionaries the resident single-GPU path takes, and the feature-table layout it fills: the column order of
compute_selected_features_color2d (colour groups first, then texture groups, each in dict order; statistic-major, channel-minor;
texture groups battery-major).  Host logic only.
"""
import pytest


def test_native_feature_layout_mixed_dict():
    from pyimsegm_b200.descriptors import native_feature_layout
    layout, ncol = native_feature_layout({'tLM_short': ('meanGrad', ), 'color_hsv': ('median', 'mean'), 'color': ('energy', )})
    assert layout == [('color_hsv', ['mean', 'median'], 0, 6), ('color', ['energy'], 6, 3), ('tLM_short', ['meanGrad'], 9, 45)]
    assert ncol == 54
    layout, ncol = native_feature_layout({'tLM': ('median', 'std', 'mean'), 'color_lab': ('meanGrad', 'median', 'energy', 'std', 'mean')})
    assert layout == [('color_lab', ['mean', 'std', 'energy', 'median', 'meanGrad'], 0, 15), ('tLM', ['mean', 'std', 'median'], 15, 180)]
    assert ncol == 195
    # the sets that were resident before keep their layout
    assert native_feature_layout({'color': ('mean', 'std', 'energy'), 'tLM': ('mean', )}) == (
        [('color', ['mean', 'std', 'energy'], 0, 9), ('tLM', ['mean'], 9, 60)], 69)


def test_resident_predicate():
    from pyimsegm_b200.descriptors import FEATURES_SET_ALL, NAMES_FEATURE_FLAGS, flags_are_native, flags_are_resident
    admitted = [{'color': ['mean', 'std', 'median']}, {'color': ['mean', 'median']}, {'color': NAMES_FEATURE_FLAGS}, FEATURES_SET_ALL,
                {'color_hsv': ('mean', 'std', 'energy'), 'color_lab': ('mean', 'median')}, {'tLM_short': ('mean', 'meanGrad')},
                {'color_luv': ('std', ), 'color_hed': ('energy', ), 'color_xyz': ('meanGrad', )}, {'color': ()}]
    for d in admitted:
        assert flags_are_resident(d), d
    refused = [{}, {'color_foo': ['mean']}, {'color': ['mean', 'foo']}, {'tLM_long': ['mean']}, {'gray': ['mean']},
               {'color_hsv': ['mean'], 'texture': ['mean']}]
    for d in refused:
        assert not flags_are_resident(d), d
    # the banded path keeps its own, narrower predicate
    assert flags_are_native({'color': ['mean', 'std', 'energy'], 'tLM_short': ['mean']})
    assert not flags_are_native({'color': ['median']}) and not flags_are_native({'color_hsv': ['mean']})


def test_tiled_still_refuses_median_before_any_engine_call(monkeypatch):
    from pyimsegm_b200 import tiled

    def no_engine(*args, **kwargs):
        raise AssertionError('the banded path reached the engine')

    monkeypatch.setattr(tiled, 'get_engine', no_engine)
    import numpy as np
    with pytest.raises(NotImplementedError):
        tiled.pipe_color2d_slic_features_model_graphcut_tiled(np.zeros((32, 32, 3)), 2, {'color': ['median']})
