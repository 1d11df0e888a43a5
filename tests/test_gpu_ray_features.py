"""GPU tests of the Ray tracer (k_ray_features behind descriptors.cython_ray_features_seg2d): every ray bit for bit against the
oracle (oracle.ray_features2d) and, where it was built, against the reference's own module compiled IEEE-strict, at angle steps
that divide 360 and one that does not, both edges, positions on the corners, borders and boundary label and wrapped negative
positions, thin and 4096 x 4096 masks, one launch of more than 1e5 rays, and the two constructed cases that hang on the angle
table and on round half to even.  Then the consumers -- the Ray features of positions, the RG2SP shape model and the ellipse
boundary points -- against the same calls with the host tracer in place of the device one."""
import numpy as np
import pytest

import oracle
from test_ray_features_host import (STEPS, edge_positions, host_tracer, random_positions, ref_trace, smooth_mask, strict_module,
                                    table_case, tie_case)

pytestmark = pytest.mark.gpu

EDGES = {'up': 1, 'down': -1}


@pytest.fixture(scope='module')
def ds():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pyimsegm_b200 import descriptors
    return descriptors


@pytest.fixture(scope='module')
def strict():
    return strict_module()


def _check(ds, strict, mask, positions, step, edge):
    """one launch for all positions; each row equal to the oracle's and the strict module's, bit for bit"""
    got = ds.cython_ray_features_seg2d(mask, positions, step, edge)
    assert got.dtype == np.float32 and got.shape[0] == len(positions)
    for p, g in zip(positions, got):
        want = oracle.ray_features2d(mask, p, step, EDGES[edge])
        assert np.array_equal(g, want), (tuple(p), step, edge, np.nonzero(g != want)[0])
        if strict is not None:
            assert np.array_equal(g, ref_trace(strict, mask, p, step, EDGES[edge])), (tuple(p), step, edge)
    return got


@pytest.mark.parametrize('shape', [(300, 400), (1000, 1200)])
@pytest.mark.parametrize('step', [5, 1])
@pytest.mark.parametrize('edge', ['up', 'down'])
def test_smooth_noise_bit_exact(ds, strict, shape, step, edge):
    mask = smooth_mask(shape, seed=shape[0])
    _check(ds, strict, mask, random_positions(shape, 200, seed=shape[1]), step, edge)


@pytest.mark.parametrize('step', STEPS)
@pytest.mark.parametrize('edge', ['up', 'down'])
def test_every_step_at_corners_borders_and_boundary(ds, strict, step, edge):
    mask = smooth_mask((120, 170), seed=3, sigma=3.)
    got = _check(ds, strict, mask, np.concatenate([edge_positions(mask, negative=False), random_positions(mask.shape, 30, 4)]), step, edge)
    assert got.shape[1] == len(np.arange(0, 360, float(np.float32(step)), dtype=np.float32))
    if edge == 'up':
        assert np.all(got[8] == 0)           # edge_positions' pixel of the boundary label


@pytest.mark.parametrize('step', STEPS)
@pytest.mark.parametrize('edge', ['up', 'down'])
def test_negative_positions_wrap(ds, strict, step, edge):
    """a row in [-H, -1] or a column in [-W, -1] reads the start pixel wrapped and marches from the negative coordinate"""
    mask = smooth_mask((120, 170), seed=3, sigma=3.)
    pos = np.concatenate([edge_positions(mask)[-7:], random_positions(mask.shape, 30, 5, negative=True)])
    _check(ds, strict, mask, pos, step, edge)


def _thin_masks(shape):
    rng = np.random.RandomState(shape[0] * 1000 + shape[1])
    return np.zeros(shape, bool), np.ones(shape, bool), rng.rand(*shape) < 0.2


@pytest.mark.parametrize('shape', [(1, 1), (1, 57), (57, 1), (2, 300), (300, 2)])
@pytest.mark.parametrize('edge', ['up', 'down'])
def test_thin_masks(ds, strict, shape, edge):
    for mask in _thin_masks(shape):
        for step in (1, 7.5, 90):
            _check(ds, strict, mask, edge_positions(mask, negative=False), step, edge)


@pytest.mark.parametrize('shape', [(1, 1), (1, 57), (57, 1), (2, 300), (300, 2)])
@pytest.mark.parametrize('edge', ['up', 'down'])
def test_thin_masks_negative_positions(ds, strict, shape, edge):
    for mask in _thin_masks(shape):
        for step in (1, 7.5, 90):
            _check(ds, strict, mask, edge_positions(mask)[-7:], step, edge)


def test_4096_mask(ds, strict):
    mask = smooth_mask((4096, 4096), seed=7, sigma=24.)
    for step, edge in ((5, 'up'), (5, 'down'), (1, 'down')):
        _check(ds, strict, mask, np.concatenate([edge_positions(mask, negative=False), random_positions(mask.shape, 12, 8)]), step, edge)


def test_4096_mask_negative_positions(ds, strict):
    mask = smooth_mask((4096, 4096), seed=7, sigma=24.)
    _check(ds, strict, mask, np.concatenate([edge_positions(mask)[-7:], random_positions(mask.shape, 8, 9, negative=True)]), 5, 'down')


def test_one_launch_of_more_than_1e5_rays(ds, strict):
    from pyimsegm_b200 import _lib
    mask = smooth_mask((1000, 1200), seed=13)
    pos = random_positions(mask.shape, 300, seed=14)
    before = _lib.lib().isb_launch_count()
    got = _check(ds, strict, mask, pos, 1, 'down')
    assert _lib.lib().isb_launch_count() - before == 1 and got.size == 300 * 360 > 10 ** 5


@pytest.mark.parametrize('edge', ['up', 'down'])
def test_tie_rounds_half_to_even(ds, strict, edge):
    """the only boundary pixel is the one round-half-away reads at the tied step: the reference's ray misses it"""
    up, down, pos, i, roundf_dist = tie_case()
    got = _check(ds, strict, up if edge == 'up' else down, np.array([pos]), 5., edge)
    assert got[0, i] == -1. and roundf_dist > 0


@pytest.mark.parametrize('edge', ['up', 'down'])
def test_table_follows_the_float64_radians(ds, strict, edge):
    """at 345 degrees the reference's direction reads the only boundary pixel; a float32 np.deg2rad table reads the next row"""
    up, down, pos, i, dist = table_case()
    got = _check(ds, strict, up if edge == 'up' else down, np.array([pos]), 5., edge)
    assert got[0, i] == dist > 0


def test_out_of_range_positions_raise_before_any_launch(ds):
    from pyimsegm_b200 import _lib
    mask = smooth_mask((40, 50), seed=5)
    before = _lib.lib().isb_launch_count()
    for position in [(40, 0), (0, 50), (-41, 0), (0, -51), (40, 50), (-41, -51), (1000, 3)]:
        for edge in ('up', 'down'):
            with pytest.raises(IndexError):
                ds.cython_ray_features_seg2d(mask, position, 5., edge)
            with pytest.raises(IndexError):
                ds.cython_ray_features_seg2d(mask, [(3, 4), position, (5, 6)], 5., edge)
    with pytest.raises(IndexError):
        ds.compute_ray_features_positions(mask.astype(int), [(3, 4), (40, 3)], 5.)
    with pytest.raises(ValueError):
        ds.cython_ray_features_seg2d(np.zeros((4, 5, 2), bool), (1, 1), 5.)
    with pytest.raises(ValueError):
        ds.cython_ray_features_seg2d(np.zeros(20, bool), (1, 1), 5.)
    assert _lib.lib().isb_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# consumers: the same calls with the host tracer monkeypatched in
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def eggs():
    from test_gpu_ellipse_fitting import _eggs
    return _eggs(0)


def _host(strict):
    """the strict reference module where it was built, else the oracle (the two agree bit for bit, tests/test_ray_features_host.py)"""
    if strict is not None:
        return host_tracer(lambda seg, p, step, e: ref_trace(strict, seg, p, step, e))
    return host_tracer(oracle.ray_features2d)


def _both(monkeypatch, strict, call):
    """``call()`` through the device tracer, then with the host tracer in every module that holds it by name"""
    from pyimsegm_b200 import descriptors, ellipse_fitting
    got = call()
    with monkeypatch.context() as mp:
        for mod in (descriptors, ellipse_fitting):
            mp.setattr(mod, 'cython_ray_features_seg2d', _host(strict))
        want = call()
    return got, want


@pytest.mark.parametrize('step,edge,segm_open', [(5, 'up', None), (1, 'down', None), (1, 'up', None), (10, 'up', 3)])
def test_ray_features_positions_equal_host_tracer(ds, strict, eggs, monkeypatch, step, edge, segm_open):
    seg, _, centres = eggs
    pos = list(centres) + [tuple(p) for p in random_positions(seg.shape, 20, 21)]
    got, want = _both(monkeypatch, strict, lambda: ds.compute_ray_features_positions(seg, pos, step, border_labels=[0], segm_open=segm_open,
                                                                                      edge=edge))
    assert np.array_equal(got[0], want[0]) and got[1] == want[1] and got[2] == want[2]


@pytest.mark.parametrize('ray_step,interp_order,smooth_coef', [(5, 3, 0), (5, 'spline', 1), (10, None, 0), (1, 3, 0)])
def test_object_shapes_equal_host_tracer(ds, strict, eggs, monkeypatch, ray_step, interp_order, smooth_coef):
    from pyimsegm_b200 import region_growing as rg
    _, annot, centres = eggs
    objects = [annot == i + 1 for i in range(len(centres))] + [annot]
    got, want = _both(monkeypatch, strict, lambda: rg.compute_object_shapes(objects, ray_step, interp_order, smooth_coef))
    assert got == want and len(got[0]) == 2 * len(centres)


@pytest.mark.parametrize('name', ['join', 'edge', 'mean', 'dist'])
def test_ellipse_boundary_points_equal_host_tracer(ds, strict, eggs, monkeypatch, name):
    from pyimsegm_b200 import ellipse_fitting as ef
    seg, _, centres = eggs
    fn = getattr(ef, 'prepare_boundary_points_ray_' + name)
    got, want = _both(monkeypatch, strict, lambda: fn(seg, centres, sel_bg=3, sel_fg=2))
    assert len(got) == len(want) > 0
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
