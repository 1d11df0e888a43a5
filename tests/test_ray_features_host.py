"""The Ray tracer of imsegm/features_cython.pyx:239-282 (computeRayFeaturesBinary2d): the oracle (oracle.ray_features2d,
oracle/stats_oracle.c) against the reference's own module compiled IEEE-strict (oracle/_ref/strict), bit for bit, and against
the module built with the reference's -O3 -ffast-math -march=native to 1e-5.

Two details of the reference decide single pixels and are pinned here: the angle table (each float32 angle is boxed to a Python
float, so np.deg2rad runs in float64 before the store to the C float ``rad``) and the rounding of the marching position (Python's
round(), half to even).  The cases built by ``tie_case`` and ``table_case`` hang on exactly one of them each.  The helpers are
shared with tests/test_gpu_ray_features.py."""
import numpy as np
import pytest
from scipy import ndimage

import oracle

STEPS = [0.5, 1, 5, 7, 7.5, 10, 15, 45, 90, 37.3]


def strict_module():
    oracle.build()
    return oracle.ref_features_cython(strict=True)


def fast_module():
    oracle.build()
    return oracle.ref_features_cython(strict=False)


def ref_trace(module, seg, position, angle_step, edge):
    """the reference module's tracer called as imsegm/descriptors.py:1655-1659 calls it; edge 1 ('up') or -1 ('down')"""
    return np.asarray(module.computeRayFeaturesBinary2d(np.array(seg, dtype=np.int8), np.array(position, dtype=np.int32),
                                                        float(angle_step), int(edge)))


def host_tracer(trace):
    """a drop-in for descriptors.cython_ray_features_seg2d running ``trace(seg, position, step, edge_int)`` per position"""
    def tracer(seg_binary, position, angle_step=5., edge='up'):
        e = {'down': -1, 'up': 1}[edge]
        pos = np.atleast_2d(np.array(position, dtype=np.int32))
        rays = np.array([trace(seg_binary, p, angle_step, e) for p in pos], dtype=np.float32)
        return rays[0] if np.ndim(position) == 1 else rays
    return tracer


def smooth_mask(shape, seed, sigma=4.):
    """blobs of both labels at a scale of ``sigma`` pixels, about half of the pixels set"""
    rng = np.random.RandomState(seed)
    return ndimage.gaussian_filter(rng.rand(*shape), sigma) > 0.5


def edge_positions(mask, negative=True):
    """corners, the middle of every border, a pixel of the boundary label and, ``negative``, rows in [-H, -1] and columns in
    [-W, -1] (the reference starts such a ray from the wrapped pixel)"""
    H, W = mask.shape
    on = np.argwhere(mask)
    pos = [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2), (H - 1, W // 3), (H // 2, 0), (H // 3, W - 1)]
    if len(on):
        pos.append(tuple(on[len(on) // 2]))
    if negative:
        pos += [(-1, min(12, W - 1)), (-1, -1), (-H, -W), (-H, W - 1), (H - 1, -W), (-(H + 1) // 2, W // 2), (H // 2, -1)]
    return np.array(pos, dtype=np.int32)


def random_positions(shape, n, seed, negative=False):
    rng = np.random.RandomState(seed)
    lo = (-shape[0], -shape[1]) if negative else (0, 0)
    return np.stack([rng.randint(lo[0], shape[0], n), rng.randint(lo[1], shape[1], n)], 1).astype(np.int32)


def directions(sin_a, cos_a):
    """the per-step increments of the reference's march: the table divided by its larger component, in float32"""
    gmax = np.maximum(np.abs(sin_a), np.abs(cos_a))
    return sin_a / gmax, cos_a / gmax


def float32_angle_table(angle_step):
    """the table of a tracer that takes np.deg2rad of a np.float32 angle, in float32: one ulp off at some angles"""
    angles = np.arange(0, 360, float(np.float32(angle_step)), dtype=np.float32)
    rads = [float(np.float32(np.deg2rad(a))) for a in angles]
    return np.array([np.sin(r) for r in rads], dtype=np.float32), np.array([np.cos(r) for r in rads], dtype=np.float32)


def march(start, step, n):
    """the float32 positions after 1..n steps of ``pos += grad`` from the integer ``start`` (or [len(start), n] for an array)"""
    acc = np.empty((np.size(start), n + 1), dtype=np.float32)
    acc[:, 0], acc[:, 1:] = np.ravel(start), step
    pos = np.add.accumulate(acc, axis=1)[:, 1:]
    return pos if np.ndim(start) else pos[0]


def _in_bounds(p0, p1, H, W):
    """the number of leading steps that stay inside the image (the reference's break test, with round half to even)"""
    inb = (p0 >= 0) & (np.rint(p0) < H) & (p1 >= 0) & (np.rint(p1) < W)
    return len(inb) if inb.all() else int(np.argmin(inb))


def tie_case(shape=(640, 640), angle_step=5., seed=0):
    """a (position, angle) whose float32 march lands exactly on an even x.5 in one coordinate, and masks whose only boundary
    pixel is the one round-half-away (roundf) reads at that step, x + 1: round half to even reads x, so the reference's ray
    misses it and leaves the image (-1), where a roundf tracer stops on it.  Returns (mask_up, mask_down, position, angle
    index, the distance a roundf tracer reports)."""
    H, W = shape
    n = int(np.sqrt(H * H + W * W))
    g0, g1 = directions(*oracle.ray_angles(angle_step))
    for pr, pc in random_positions(shape, 200, seed):
        for i in range(len(g0)):
            p0, p1 = march(pr, g0[i], n), march(pc, g1[i], n)
            m = _in_bounds(p0, p1, H, W)
            for tied, other in ((p0, p1), (p1, p0)):
                fl = np.floor(tied[:m])
                hit = np.nonzero((tied[:m] - fl == 0.5) & (fl % 2 == 0))[0]
                if not len(hit) or fl[hit[0]] + 1 >= (H if tied is p0 else W):
                    continue
                k = hit[0]
                px = [0, 0]
                px[0 if tied is p0 else 1] = int(fl[k]) + 1          # roundf
                px[1 if tied is p0 else 0] = int(np.rint(other[k]))   # the other coordinate is an exact integer
                up = np.zeros(shape, dtype=bool)
                up[px[0], px[1]] = True
                d0, d1 = np.float32(p0[k] - np.float32(pr)), np.float32(p1[k] - np.float32(pc))
                dist = np.float32(np.sqrt(float(np.float32(d0 * d0 + d1 * d1))))
                return up, ~up, (int(pr), int(pc)), i, dist
    raise AssertionError('no rounding tie found')


def table_case(shape=(1024, 4096), angle_step=5., angle=345.):
    """a ray at 345 degrees whose hit step depends on the one-ulp difference between the reference's angle table and a float32
    np.deg2rad table.  The ray moves one column right and 0.268 rows up a step, so only its row march depends on the table;
    the rays start in column 0 and the first row where the two marches round to different rows at some step is taken.  The
    only boundary pixel is the one the reference's direction reads at that step, so the reference stops there and the
    float32-table ray, one row off in that column, never reads it.  The marches agree to a fraction of a pixel until rows of
    ~15 after ~2600 steps, hence the wide mask.  Returns (mask_up, mask_down, position, angle index, the reference's hit
    distance)."""
    H, W = shape
    n = int(np.sqrt(H * H + W * W))
    i = int(round(angle / angle_step))
    ref_g = [g[i] for g in directions(*oracle.ray_angles(angle_step))]
    f32_g = [g[i] for g in directions(*float32_angle_table(angle_step))]
    assert ref_g[1] == f32_g[1] == 1 and ref_g[0] != f32_g[0], 'the two tables agree at %s degrees' % angle
    rows = np.arange(H)
    r0, f0 = march(rows, ref_g[0], n), march(rows, f32_g[0], n)
    inside = np.logical_and.accumulate((r0 >= 0) & (f0 >= 0) & (np.arange(1, n + 1) < W), axis=1)
    differ = (np.rint(r0) != np.rint(f0)) & inside
    assert differ.any(), 'no table-sensitive ray found'
    pr = int(np.argmax(differ.any(axis=1)))
    k = int(np.argmax(differ[pr]))
    up = np.zeros(shape, dtype=bool)
    up[int(np.rint(r0[pr, k])), k + 1] = True
    d0, d1 = np.float32(r0[pr, k] - np.float32(pr)), np.float32(k + 1)
    dist = np.float32(np.sqrt(float(np.float32(d0 * d0 + d1 * d1))))
    return up, ~up, (pr, 0), i, dist


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the reference module, bit for bit
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def strict():
    mod = strict_module()
    if mod is None:
        pytest.skip('the reference module was not built IEEE-strict (oracle/_ref/strict: set IMSEGM_REFERENCE and build)')
    return mod


def _assert_oracle_is_strict(strict, mask, positions, step, edge):
    for p in positions:
        want = ref_trace(strict, mask, p, step, edge)
        got = oracle.ray_features2d(mask, p, step, edge)
        assert got.dtype == np.float32 and want.dtype == np.float32
        assert np.array_equal(got, want), (tuple(p), step, edge, np.nonzero(got != want)[0])


@pytest.mark.parametrize('shape,n_pos', [((300, 400), 200), ((1000, 1200), 200)])
@pytest.mark.parametrize('step', [5, 1])
@pytest.mark.parametrize('edge', [1, -1])
def test_oracle_equals_strict_module_on_smooth_noise(strict, shape, n_pos, step, edge):
    mask = smooth_mask(shape, seed=shape[0])
    _assert_oracle_is_strict(strict, mask, random_positions(shape, n_pos, seed=shape[1]), step, edge)


@pytest.mark.parametrize('step', STEPS)
@pytest.mark.parametrize('edge', [1, -1])
def test_oracle_equals_strict_module_at_every_step_and_edge_position(strict, step, edge):
    mask = smooth_mask((120, 170), seed=3, sigma=3.)
    _assert_oracle_is_strict(strict, mask, np.concatenate([edge_positions(mask), random_positions(mask.shape, 30, 4, negative=True)]),
                             step, edge)


@pytest.mark.parametrize('shape', [(1, 1), (1, 57), (57, 1), (2, 300), (300, 2)])
@pytest.mark.parametrize('edge', [1, -1])
def test_oracle_equals_strict_module_on_thin_masks(strict, shape, edge):
    rng = np.random.RandomState(shape[0] * 1000 + shape[1])
    for mask in (np.zeros(shape, bool), np.ones(shape, bool), rng.rand(*shape) < 0.2):
        for step in (1, 7.5, 90):
            _assert_oracle_is_strict(strict, mask, edge_positions(mask), step, edge)


def test_oracle_equals_strict_module_on_a_4096_mask(strict):
    mask = smooth_mask((4096, 4096), seed=7, sigma=24.)
    pos = np.concatenate([edge_positions(mask), random_positions(mask.shape, 12, 8, negative=True)])
    for step, edge in ((5, 1), (5, -1), (1, -1)):
        _assert_oracle_is_strict(strict, mask, pos, step, edge)


def test_tie_case_rounds_half_to_even(strict):
    up, down, pos, i, roundf_dist = tie_case()
    assert roundf_dist > 0
    for mask, edge in ((up, 1), (down, -1)):
        want = ref_trace(strict, mask, pos, 5., edge)
        assert want[i] == -1.
        assert np.array_equal(oracle.ray_features2d(mask, pos, 5., edge), want)


def test_table_case_follows_the_float64_radians(strict):
    up, down, pos, i, dist = table_case()
    for mask, edge in ((up, 1), (down, -1)):
        want = ref_trace(strict, mask, pos, 5., edge)
        assert want[i] == dist > 0
        assert np.array_equal(oracle.ray_features2d(mask, pos, 5., edge), want)


def test_angle_tables_are_the_reference_ones():
    """the table differs from a float32 np.deg2rad one at 175, 345, 350, 355 degrees for a 5 degree step (one ulp of ``rad``)"""
    from pyimsegm_b200.descriptors import ray_angle_tables
    for step in STEPS:
        s, c = oracle.ray_angles(step)
        assert len(s) == len(np.arange(0, 360, float(np.float32(step)), dtype=np.float32))
        ds, dc = ray_angle_tables(step)
        assert np.array_equal(s, ds) and np.array_equal(c, dc)
    s, c = oracle.ray_angles(5.)
    s32, c32 = float32_angle_table(5.)
    assert (np.nonzero((s != s32) | (c != c32))[0] * 5).tolist() == [175, 345, 350, 355]


@pytest.mark.parametrize('position', [(40, 0), (0, 50), (-41, 0), (0, -51), (40, 50), (-41, -51), (1000, 3)])
def test_out_of_range_positions_raise(strict, position):
    mask = smooth_mask((40, 50), seed=5)
    with pytest.raises(IndexError):
        ref_trace(strict, mask, position, 5., 1)
    for edge in (1, -1):
        with pytest.raises(IndexError):
            oracle.ray_features2d(mask, position, 5., edge)


# ---------------------------------------------------------------------------------------------------------------------
# the module as the reference builds it: the same rays to 1e-5
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('step', [5, 1, 37.3])
@pytest.mark.parametrize('edge', [1, -1])
def test_oracle_close_to_fast_module(step, edge):
    fast = fast_module()
    if fast is None:
        pytest.skip('the reference module was not built with its own flags (oracle/_ref: set IMSEGM_REFERENCE and build)')
    mask = smooth_mask((300, 400), seed=11)
    for p in np.concatenate([edge_positions(mask), random_positions(mask.shape, 60, 12, negative=True)]):
        np.testing.assert_allclose(oracle.ray_features2d(mask, p, step, edge), ref_trace(fast, mask, p, step, edge), rtol=1e-5, atol=0)
