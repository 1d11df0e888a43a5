"""
Error behaviour of the C-ABI without a GPU: every entry point validates its arguments BEFORE touching CUDA, returns a negative
isb_status and leaves a message in isb_last_error() (include/imsegm_b200.h; INTEGRATION.md "Ownership, errors, threading").
No compute call is made here.
"""
import ctypes as C

import pytest


@pytest.fixture(scope='module')
def lib():
    from pyimsegm_b200 import _lib
    return _lib.lib()


def _err(lib):
    return lib.isb_last_error().decode(errors='replace')


def test_null_pointers_and_bad_sizes_are_reported(lib):
    from pyimsegm_b200 import _lib
    bad = [
        lambda: lib.isb_slic_prepare(None, 3, 8, 8, 3, None, 0, 1.0, 1, None, None, None),
        lambda: lib.isb_slic_kmeans(None, 8, 8, None, 4, 2, 2, 2.0, 10, 0, None, None, None, 0, None),
        lambda: lib.isb_enforce_connectivity(None, 8, 8, 1, 10, None, None, None, 0, None),
        lambda: lib.isb_segment_stats_2d(None, 3, None, 8, 8, 4, 1, None, 3, 0, None, None, None, 0, None),
        lambda: lib.isb_adjacency_edges(None, 8, 8, 4, None, 16, None, None, 0, None),
        lambda: lib.isb_alpha_expansion(4, None, 2, 3, None, None, None, None, None, -1, None, None, None, None, 0, None),
        lambda: lib.isb_mixture_fit_predict(0, None, 10, 3, 3, None, 2, 1, 10, 1e-3, 1e-6, 1, 0, None, None, None, None, 0, None),
        lambda: lib.isb_slic3d_kmeans(None, 2, 8, 8, None, 4, 1, 2, 2, 2.0, None, 10, None, None, 0, None),
        lambda: lib.isb_enforce_connectivity3d(None, 2, 8, 8, 1, 10, None, None, None, 0, None),
        lambda: lib.isb_disc_label_hist(None, None, 8, 8, None, 1, None, 1, None, 0, 0, 3, None, None, None),
        lambda: lib.isb_filter_response_2d(None, 1, 8, 8, None, 1, 3, 3, None, None),
        lambda: lib.isb_combine(None, None, 4, 0, None),
    ]
    for call in bad:
        rc = call()
        assert rc == _lib.ISB_ERR_ARG, rc
        assert _err(lib), 'an error message must be left behind'
    with pytest.raises(ValueError):
        _lib.check(_lib.ISB_ERR_ARG)


def test_messages_name_the_problem(lib):
    from pyimsegm_b200 import _lib
    one = (C.c_double * 4)()
    p = C.cast(one, C.c_void_p)
    assert lib.isb_slic_prepare(p, 3, 8, 8, 2, None, 0, 1.0, 1, p, p, None) == _lib.ISB_ERR_ARG
    assert 'C must be 1 or 3' in _err(lib)
    assert lib.isb_filter_response_2d(p, 1, 8, 8, p, 1, 4, 3, p, None) == _lib.ISB_ERR_ARG
    assert 'odd' in _err(lib)
    assert lib.isb_mixture_fit_predict(0, p, 10, 300, 300, None, 2, 1, 10, 1e-3, 1e-6, 1, 0, None, p, None, p, 1 << 40, None) == _lib.ISB_ERR_UNSUPPORTED
    assert 'D <=' in _err(lib)
    with pytest.raises(NotImplementedError):
        _lib.check(_lib.ISB_ERR_UNSUPPORTED)
