"""
Host side of the 'color' / 'features' edge weights on the device: the argument checks of isb_gc_vector_edge_weights and
isb_image_unit_scale (every refusal returns ISB_ERR_ARG before a pointer is dereferenced or CUDA is touched), the given-weights
mode of isb_gc_energies, and the edge-type names the device pipelines take.  No GPU is needed.
"""
import ctypes as C

import pytest


@pytest.fixture(scope='module')
def lib():
    from pyimsegm_b200 import _lib
    return _lib.lib()


def _err(lib):
    return lib.isb_last_error().decode(errors='replace')


def _host_ptr():
    buf = (C.c_double * 16)()
    return buf, C.cast(buf, C.c_void_p)


def test_vector_edge_weights_refuses_bad_arguments(lib):
    from pyimsegm_b200 import _lib
    keep, p = _host_ptr()
    ws = C.c_size_t(1 << 20)
    cases = [
        ((None, 4, 3, 3, p, 8, None, p, 2, p, p, ws, None), 'null pointer'),
        ((p, 4, 3, 3, None, 8, None, p, 2, p, p, ws, None), 'null pointer'),
        ((p, 4, 3, 3, p, 8, None, None, 2, p, p, ws, None), 'null pointer'),
        ((p, 4, 3, 3, p, 8, None, p, 2, None, p, ws, None), 'null pointer'),
        ((p, 4, 3, 3, p, 8, None, p, 2, p, None, ws, None), 'null pointer'),
        ((p, 0, 3, 3, p, 8, None, p, 2, p, p, ws, None), 'bad sizes'),
        ((p, 4, 0, 3, p, 8, None, p, 2, p, p, ws, None), 'bad sizes'),
        ((p, 4, 3, 3, p, 0, None, p, 2, p, p, ws, None), 'bad sizes'),
        ((p, 4, 3, 2, p, 8, None, p, 2, p, p, ws, None), 'ld'),
        ((p, 4, 3, 3, p, 8, None, p, 1, p, p, ws, None), 'metric'),
        ((p, 4, 3, 3, p, 8, None, p, 4, p, p, ws, None), 'metric'),
        ((p, 4, 3, 3, p, 8, None, p, 2, p, p, C.c_size_t(8), None), 'workspace'),
    ]
    for args, what in cases:
        assert lib.isb_gc_vector_edge_weights(*args) == _lib.ISB_ERR_ARG, args
        assert what in _err(lib), (args, _err(lib))
    with pytest.raises(ValueError, match='metric'):
        _lib.check(lib.isb_gc_vector_edge_weights(p, 4, 3, 3, p, 8, None, p, 0, p, p, ws, None))
    del keep


def test_unit_scale_refuses_bad_arguments(lib):
    from pyimsegm_b200 import _lib
    keep, p = _host_ptr()
    for args in [(None, 3, 12, p, p, None), (p, 3, 12, None, p, None), (p, 3, 12, p, None, None), (p, 3, 0, p, p, None)]:
        assert lib.isb_image_unit_scale(*args) == _lib.ISB_ERR_ARG, args
        assert _err(lib)
    assert lib.isb_image_unit_scale(p, 7, 12, p, p, None) == _lib.ISB_ERR_ARG
    assert 'dtype' in _err(lib)
    del keep


def test_energies_take_given_weights_only_without_spatial(lib):
    from pyimsegm_b200 import _lib
    keep, p = _host_ptr()
    args = [p, 4, None, 2, p, 3, None, p, 4, 1, 1.0, p, p, p, p, p, p, p, C.c_size_t(1 << 20), None]
    assert lib.isb_gc_energies(*args) == _lib.ISB_ERR_ARG
    assert 'spatial must be 0' in _err(lib)
    args[8] = 5
    assert lib.isb_gc_energies(*args) == _lib.ISB_ERR_ARG
    assert 'metric must be 0..4' in _err(lib)
    del keep


def test_edge_type_names():
    from pyimsegm_b200.graph_cuts import check_edge_type, reference_edge_type
    for name in ('', 'spatial', 'model', 'model_lT', 'model_l1', 'model_l2', 'color', 'features'):
        check_edge_type(name)
        assert reference_edge_type(name) == name
    for name in ('colour', 'feature', 'model_l3', 'Model', 'spatial ', None, 3):
        with pytest.raises(ValueError, match='unknown gc_edge_type'):
            check_edge_type(name)
    # the reference weights an unknown name by ones without the spatial term: the weights of ''
    assert reference_edge_type('colour') == ''
    assert reference_edge_type('model_l3') == ''


def test_unknown_edge_type_is_refused_before_device_work():
    """the banded entries check the name before they upload anything, so this runs without a GPU"""
    import numpy as np

    from pyimsegm_b200 import tiled
    img = np.zeros((64, 64, 3))
    with pytest.raises(ValueError, match='unknown gc_edge_type'):
        tiled.pipe_color2d_slic_features_model_graphcut_tiled(img, 2, gc_edge_type='colour')
    with pytest.raises(ValueError, match='unknown gc_edge_type'):
        tiled.segment_color2d_slic_features_model_graphcut_tiled(img, object(), {'color': ['mean']}, gc_edge_type='feature')
