"""CPU tests of imsegm.annotation: the oracle (oracle/annotation.py) against the reference's own outputs on its doctest inputs
(tests/golden/annotation_reference.npz, made by make_annotation_goldens.py), the host-only table loader, and the argument, dtype and
palette checks that raise before any device work, in Python and in the C entry points (no launch)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import annotation as oa
from pyimsegm_b200 import annotation as an

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

#: every public name of the reference's imsegm/annotation.py
REFERENCE_NAMES = [
    'unique_image_colors', 'convert_img_colors_to_labels', 'convert_img_colors_to_labels_reverted', 'convert_img_labels_to_colors',
    'image_frequent_colors', 'group_images_frequent_colors', 'image_color_2_labels', 'quantize_image_nearest_color',
    'image_inpaint_pixels', 'quantize_image_nearest_pixel', 'load_info_group_by_slices',
]
REFERENCE_CONSTANTS = ['COLUMNS_POSITION', 'SLICE_NAME_GROUPING', 'ANNOT_SLICE_DIST_TOL', 'DICT_COLOURS']


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLDEN, 'annotation_reference.npz')))


def test_every_reference_name_is_importable():
    import importlib
    mod = importlib.import_module('imsegm.annotation')
    for name in REFERENCE_NAMES:
        assert callable(getattr(mod, name)), name
    for name in REFERENCE_CONSTANTS:
        assert getattr(mod, name) is not None, name
    assert mod.COLUMNS_POSITION == ('ant_x', 'ant_y', 'post_x', 'post_y', 'lat_x', 'lat_y')
    assert mod.DICT_COLOURS[3] == (255, 229, 0) and mod.ANNOT_SLICE_DIST_TOL[4] == 3 and mod.SLICE_NAME_GROUPING == 'stack_path'


def test_oracle_reproduces_the_reference(gold):
    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3))
    assert oa.unique_image_colors(img) == [tuple(c) for c in gold['unique_colors'].tolist()]
    assert oa.unique_image_colors(gold['unique_img_rand']) == [tuple(c) for c in gold['unique_colors_rand'].tolist()]
    seg = gold['convert_seg']
    img = np.array([(0.2, 0.2, 0.2), (0.9, 0.9, 0.9)])[seg]
    assert np.array_equal(oa.convert_img_colors_to_labels(img, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)}), gold['convert_labels'])
    assert np.array_equal(oa.convert_img_colors_to_labels_reverted(img, {(0.2, 0.2, 0.2): 0, (0.9, 0.9, 0.9): 1}),
                          gold['convert_labels_reverted'])
    assert np.array_equal(oa.convert_img_labels_to_colors(seg, {0: (0.2, 0.2, 0.2), 1: (0.9, 0.9, 0.9)}), gold['labels_to_colors'])
    np.random.seed(0)
    img = np.random.randint(0, 2, (50, 50, 3)).astype(np.uint8)
    d = oa.image_frequent_colors(img)
    assert list(d) == [tuple(c) for c in gold['frequent_colors'].tolist()] and list(d.values()) == gold['frequent_counts'].tolist()
    assert sorted(d.values()) == [271, 289, 295, 317, 318, 330, 335, 345]
    assert np.array_equal(oa.image_color_2_labels(gold['color_2_labels_img']), gold['color_2_labels'])
    img = gold['quantize_img']
    assert np.array_equal(oa.quantize_image_nearest_color(img, [(0, 0, 0), (1, 1, 1)]), gold['quantize_nearest_color'])
    assert np.array_equal(oa.quantize_image_nearest_pixel(img, [(0, 0, 0), (1, 1, 1)]), gold['quantize_nearest_pixel'])
    assert np.array_equal(oa.image_inpaint_pixels(gold['inpaint_img'], gold['inpaint_valid']), gold['inpaint'])


def test_reference_doctest_values_are_pinned(gold):
    assert gold['convert_labels'][0].tolist() == [0, 1, 1, 0, 1, 1, 1]
    assert gold['labels_to_colors'][1, :, 0].tolist() == [0.9, 0.9, 0.9, 0.9, 0.2, 0.2, 0.9]
    assert gold['color_2_labels'][0].tolist() == [1, 0, 0, 1, 0, 0, 0]
    assert gold['quantize_nearest_color'][0, :, 0].tolist() == [1, 1, 1, 1, 0, 0, 0]
    assert gold['quantize_nearest_pixel'][2, :, 0].tolist() == [1, 1, 1, 1, 1, 0, 0]


def test_load_info_group_by_slices_reproduces_the_doctest():
    df = an.load_info_group_by_slices(os.path.join(GOLDEN, 'info_ovary_images.txt'), [4])
    assert list(df.index) == ['insitu7569']
    row = df.loc['insitu7569']
    want = {'ant_x': [298], 'ant_y': [327], 'lat_x': [673], 'lat_y': [411], 'post_x': [986], 'post_y': [155]}
    assert sorted(df.columns) == sorted(want)
    assert {k: [int(v) for v in row[k]] for k in want} == want
    assert an.load_info_group_by_slices(os.path.join(GOLDEN, 'info_ovary_images.txt'), [42]).empty


def test_arguments_raise_before_any_device_work():
    from pyimsegm_b200.utilities import ImageDimensionError
    img = np.zeros((4, 5, 3), np.uint8)
    with pytest.raises(ValueError):
        an.convert_img_colors_to_labels_reverted(img, {})
    with pytest.raises(ValueError):
        an.convert_img_colors_to_labels(img, {0: (1, 2), 1: (3, 4)})                # 2 components for 3 channels
    with pytest.raises(NotImplementedError, match='1024'):
        an.convert_img_colors_to_labels(img, {i: (i % 256, i // 256, 0) for i in range(1025)})
    with pytest.raises(NotImplementedError, match='1024'):
        an.image_color_2_labels(img, [(i % 256, i // 256, 0) for i in range(1025)])
    with pytest.raises(ValueError):
        an.image_color_2_labels(np.zeros((4, 5, 4), np.uint8), [(0, 0, 0, 0)])
    with pytest.raises(ValueError):
        an.quantize_image_nearest_color(np.zeros((4, 5)), [(0, 0, 0)])
    with pytest.raises(TypeError):
        an.quantize_image_nearest_color(np.zeros((4, 5, 3), complex), [(0, 0, 0)])
    with pytest.raises(ValueError):
        an.quantize_image_nearest_pixel(np.zeros((4, 5, 3, 1)), [(0, 0, 0)])
    with pytest.raises(ValueError):
        an.quantize_image_nearest_pixel(img, [(0, 0, 0), (0, 0)])                   # ragged colours
    with pytest.raises(ImageDimensionError):
        an.image_inpaint_pixels(np.zeros((4, 5)), np.zeros((5, 4), bool))
    with pytest.raises(ValueError, match='2-D'):
        an.image_inpaint_pixels(np.zeros((2, 4, 5)), np.ones((2, 4, 5), bool))
    with pytest.raises(ValueError, match='no valid pixel'):
        an.image_inpaint_pixels(np.zeros((4, 5)), np.zeros((4, 5), bool))
    with pytest.raises(ValueError, match='no valid pixel'):
        an.image_inpaint_pixels(np.zeros((0, 5)), np.zeros((0, 5), bool))
    with pytest.raises(TypeError):
        an.image_inpaint_pixels(np.zeros((4, 5), complex), np.ones((4, 5), bool))
    with pytest.raises(ValueError):
        an.unique_image_colors(np.zeros((4, 5, 2), np.uint8))
    with pytest.raises(ValueError):
        an.convert_img_labels_to_colors(np.zeros((4, 5)) + 0.5, {0: (0, 0, 0)})
    with pytest.raises(ValueError, match='missing'):
        an.convert_img_labels_to_colors(np.zeros((4, 5), int), {0.5: (0, 0, 0)})
    assert an.convert_img_colors_to_labels(np.zeros((0, 3, 3)), {0: (0, 0, 0)}).shape == (0, 3)
    assert an.convert_img_labels_to_colors(np.zeros((0, 3), int), {0: (1, 2, 3)}).shape == (0, 3, 3)
    assert an.unique_image_colors(np.zeros((0, 3, 3), np.uint8)) == [] and an.image_frequent_colors(np.zeros((3, 0, 3), np.uint8)) == {}


def test_annotation_entry_points_reject_bad_arguments():
    from pyimsegm_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    assert lib.isb_abi_version() == 8
    assert lib.isb_color_hist(None, 4, 3, 0, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_color_hist(p, 4, 2, 0, p, None) == _lib.ISB_ERR_ARG and b'channels' in lib.isb_last_error()
    assert lib.isb_color_hist(p, 0, 3, 0, p, None) == _lib.ISB_ERR_ARG
    ws = lib.isb_color_hist_workspace_bytes()
    assert ws > 0
    assert lib.isb_color_hist_compact_count(p, p, ws - 1, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_color_hist_compact_write(p, p, ws, None, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_palette_map(p, 0, 10, 3, p, 1025, 0, None, p, None, None, None) == _lib.ISB_ERR_UNSUPPORTED
    assert b'1024' in lib.isb_last_error()
    assert lib.isb_palette_map(p, 2, 10, 3, p, 4, 0, None, p, None, None, None) == _lib.ISB_ERR_ARG        # float32
    assert lib.isb_palette_map(p, 0, 10, 5, p, 4, 0, None, p, None, None, None) == _lib.ISB_ERR_ARG        # 5 channels
    assert lib.isb_palette_map(p, 0, 10, 3, p, 4, 2, None, p, None, None, None) == _lib.ISB_ERR_ARG        # mode
    assert lib.isb_palette_map(p, 0, 10, 3, p, 0, 0, None, p, None, None, None) == _lib.ISB_ERR_ARG
    assert lib.isb_palette_gather(p, 10, None, 1025, p, 3, p, None, None) == _lib.ISB_ERR_UNSUPPORTED
    assert lib.isb_palette_gather(p, 10, None, 4, p, 33, p, None, None) == _lib.ISB_ERR_ARG
    assert lib.isb_palette_gather(p, 10, None, 4, None, 3, p, None, None) == _lib.ISB_ERR_ARG
    assert lib.isb_gather_at_index(p, 3, p, 10, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_gather_at_index(p, 8, p, 0, p, None) == _lib.ISB_ERR_ARG
    assert lib.isb_edt_index_workspace_bytes(0, 4) == 0
    assert lib.isb_edt_index_workspace_bytes(8, 8) > lib.isb_edt_workspace_bytes(8, 8)
    ws = lib.isb_edt_index_workspace_bytes(40000, 4)
    assert lib.isb_edt_2d_indices(p, 40000, 4, p, p, ws, None) == _lib.ISB_ERR_ARG and b'32768' in lib.isb_last_error()
    assert lib.isb_edt_2d_indices(p, 8, 8, p, p, lib.isb_edt_workspace_bytes(8, 8), None) == _lib.ISB_ERR_ARG
