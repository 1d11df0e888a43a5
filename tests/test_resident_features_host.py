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


def test_native_feature_names():
    from pyimsegm_b200.descriptors import NAMES_FEATURE_FLAGS, _stat_names, native_feature_names

    def chans(prefix, flags):
        return ['%s-ch%i_%s' % (prefix, c, f) for f in flags for c in (1, 2, 3)]

    # compute_image2d_color_statistic's default color_name: the reference doctest (descriptors.py:804-808)
    assert _stat_names('color', NAMES_FEATURE_FLAGS) == [
        'color-ch1_mean', 'color-ch2_mean', 'color-ch3_mean', 'color-ch1_std', 'color-ch2_std', 'color-ch3_std',
        'color-ch1_energy', 'color-ch2_energy', 'color-ch3_energy', 'color-ch1_median', 'color-ch2_median', 'color-ch3_median',
        'color-ch1_meanGrad', 'color-ch2_meanGrad', 'color-ch3_meanGrad']
    # 'color' and keys without '_' are 'rgb', a known or unknown space names itself; duplicate and unknown flags drop out
    assert native_feature_names({'color': ('std', 'mean', 'std', 'foo')}) == chans('rgb', ('mean', 'std'))
    assert native_feature_names({'colorX': ('energy', )}) == chans('rgb', ('energy', ))
    assert native_feature_names({'color_hsv': ('meanGrad', 'median')}) == chans('hsv', ('median', 'meanGrad'))
    assert native_feature_names({'color_foo': ('mean', )}) == chans('foo', ('mean', ))
    # colour groups first, then texture groups, each in dict order; other groups contribute nothing
    assert native_feature_names({'tLM_short': ('mean', ), 'gray': ('mean', ), 'color_lab': ('std', ), 'color': ('mean', )}) == (
        chans('lab', ('std', )) + chans('rgb', ('mean', ))
        + [n for s in ('1.4', '2.0', '4.0') for b in ('edge', 'bar', 'Gauss', 'GaussLap', 'GaussLap2')
           for n in chans('tLM_sigma%s-%s' % (s, b), ('mean', ))])
    # the full bank for 'tLM' and any suffix other than 'short', battery-major (reference descriptors.py:1066-1074)
    full = [n for s in ('1.4', '2.0', '2.8', '4.0') for b in ('edge', 'bar', 'Gauss', 'GaussLap', 'GaussLap2')
            for n in chans('tLM_sigma%s-%s' % (s, b), ('mean', 'std', 'median'))]
    assert native_feature_names({'tLM': ('median', 'mean', 'std')}) == full
    assert native_feature_names({'tLM_long': ('median', 'mean', 'std')}) == full
    assert native_feature_names({}) == [] and native_feature_names({'color': ()}) == []


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
