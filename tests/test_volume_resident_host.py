"""CPU tests of the resident gray-volume path: which feature dictionaries it takes, the SLIC parameters it shares with
segment_slic_img3d_gray, and the argument checks of the two C-ABI entries it adds or extends (no compute call)."""
import ctypes as C

import numpy as np
import pytest


def test_volume_flags_follow_compute_selected_features_gray3d():
    from pyimsegm_b200 import pipelines as pl
    assert pl._volume_flags({'color': ['energy', 'mean']}) == ['mean', 'energy']
    assert pl._volume_flags({'color': ['median', 'std'], 'color_b': ['mean']}) == ['mean', 'std', 'median']
    for feats in ({}, {'color': []}, {'color': ['meanGrad']}, {'tLM': ['mean']}, {'color': ['mean'], 'tLM_short': ['mean']}):
        assert pl._volume_flags(feats) is None, feats


@pytest.mark.parametrize('shape, sp_size, regul, space', [((5, 125, 150), 15, 0.2, (12, 1, 1)), ((64, 512, 512), 15, 0.2, (12, 1, 1)),
                                                          ((24, 40, 36), 8, 0.3, (1, 1, 1)), ((9, 33, 70), 7, 0.25, (1, 1, 2))])
def test_slic3d_params_are_the_reference_formula(shape, sp_size, regul, space):
    from pyimsegm_b200.superpixels import slic3d_params
    size = np.prod(sp_size / np.asarray(space, dtype=np.float32) * min(space))      # reference superpixels.py:97-101
    assert slic3d_params(shape, sp_size, regul, space) == (int(np.prod(shape) / size), int((size * regul) ** 1.5))


def test_standard_scaler_and_3d_energies_reject_bad_arguments():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    buf = C.c_void_p(64)        # never dereferenced: every call below fails its checks first
    assert lib.isb_standard_scaler(None, 10, 3, 3, None, buf, buf, None) == _lib.ISB_ERR_ARG
    assert lib.isb_standard_scaler(buf, 0, 3, 3, None, buf, buf, None) == _lib.ISB_ERR_ARG
    assert lib.isb_standard_scaler(buf, 10, 3, 2, None, buf, buf, None) == _lib.ISB_ERR_ARG
    for spatial in (-1, 4):
        rc = lib.isb_gc_energies(buf, 4, None, 2, buf, 3, None, buf, 1, spatial, 1.0, buf, buf, buf, buf, buf, buf, buf, 1 << 20, None)
        assert rc == _lib.ISB_ERR_ARG and b'spatial' in lib.isb_last_error()
    rc = lib.isb_gc_energies(buf, 4, None, 2, buf, 3, None, None, 1, 3, 1.0, buf, buf, buf, buf, buf, buf, buf, 1 << 20, None)
    assert rc == _lib.ISB_ERR_ARG and b'centres' in lib.isb_last_error()
