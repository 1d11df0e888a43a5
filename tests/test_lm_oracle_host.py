"""The per-pixel float64 oracle of the Leung-Malik responses (oracle/texture.py `clipped_responses`, by FFT) and what it can tell apart,
on the host (no GPU):
- it equals the ndimage restatement of the reference (`battery_responses`) on images smaller than the 33-tap kernels, where the
  reflection wraps more than once;
- the per-pixel bound that tests/test_gpu_lm_responses.py puts on the tensor-core contraction, |r_gpu - r| <= 1e-5 M with
  M = max |img - background|, sits far above what the 3xTF32 split itself costs and far below what a split missing one of its
  remainder products costs (a numpy emulation of the split: tf32 roundings as cvt.rna, products and sums in float64);
- a NaN or infinite pixel makes every Leung-Malik feature of the reference 0."""
import numpy as np
import pytest
from scipy import ndimage

BOUND = 1e-5    # tests/test_gpu_lm_responses.py: per-pixel error of a response over max |img - background|


def _textured(h, w, seed):
    """0.5 + 0.2 sin(x / 3) in the lower half, N(0, 0.05) noise everywhere"""
    rng = np.random.RandomState(seed)
    img = np.zeros((h, w, 3))
    img[h // 2:] = 0.5 + 0.2 * np.sin(np.arange(w) / 3.0)[None, :, None]
    return img + rng.normal(0, 0.05, img.shape)


def test_reflect_index_is_ndimage_reflect():
    """ndimage's own padding, read back as the line shifted by k with a one-tap kernel, for pads up to 100 times the axis"""
    from oracle import texture as otex
    for n in (1, 2, 3, 5, 40):
        line = np.arange(n, dtype=np.float64) + 1
        for pad in (0, 1, 16, 100):
            got = line[otex.reflect_index(n, pad)]
            for k in range(-pad, pad + 1):
                w = np.zeros(2 * pad + 1)
                w[pad + k] = 1
                shifted = ndimage.correlate1d(line, w, mode='reflect')
                np.testing.assert_array_equal(got[pad + k:pad + k + n], shifted, err_msg='n %d pad %d shift %d' % (n, pad, k))


@pytest.mark.parametrize('shape', [(1, 7), (5, 5), (6, 300), (17, 40)])
@pytest.mark.parametrize('bank', ['normal', 'short'])
def test_fft_oracle_equals_ndimage_oracle(shape, bank):
    """every axis is 1 or at least 5 pixels long: see test_fft_oracle_on_axes_of_at_most_four_pixels for the others"""
    from oracle import texture as otex
    img = _textured(shape[0], shape[1], seed=shape[0] * 1000 + shape[1])
    want, _ = otex.battery_responses(img, bank)
    sub, resp, norms = otex.clipped_responses(img, bank)
    want_sub = np.rollaxis(img - ndimage.gaussian_filter(img, 150), -1, 0)
    np.testing.assert_array_equal(sub, want_sub)
    got = otex.norm_scale(norms)[:, None, None, None] * resp
    assert got.shape == want.shape == (15 if bank == 'short' else 20, 3) + shape
    scale = np.abs(want).max(axis=(1, 2, 3), keepdims=True)
    assert np.all(np.abs(got - want) <= 1e-12 * scale), np.max(np.abs(got - want) / scale)


@pytest.mark.parametrize('shape', [(5, 3), (3, 300), (2, 129), (4, 4)])
def test_fft_oracle_on_axes_of_at_most_four_pixels(shape):
    """scipy.ndimage's n-D filters (ndimage.convolve, which the reference calls) do not reflect an index of exactly -2n m, m >= 2, on
    an axis of length n: they read the element before the line, outside the image (garbage or NaN at (5, 3) and (3, 300)).  A
    33-tap kernel reaches such an index when n <= 4.  The well-defined answer there, which the device kernels compute, is the
    2n-periodic reflection of ndimage's 1-D filters (test_reflect_index_is_ndimage_reflect); the FFT oracle equals its direct sum."""
    from numpy.lib.stride_tricks import sliding_window_view
    from oracle import texture as otex
    img = _textured(shape[0], shape[1], seed=7)[..., 0]
    bank, _ = otex.filter_bank()
    kernels = np.concatenate([bank[0], bank[1], bank[3], bank[14]])     # odd and even oriented kernels, two Laplacians
    got = otex.convolve_reflect(img, kernels)
    padded = img[otex.reflect_index(shape[0], 16)[:, None], otex.reflect_index(shape[1], 16)[None, :]]
    want = np.einsum('hwab,kab->khw', sliding_window_view(padded, (33, 33)), kernels[:, ::-1, ::-1])
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13)


def test_fft_convolution_of_asymmetric_kernels():
    """the bank's edge kernels are odd: a flipped kernel (correlation instead of convolution) would show here"""
    from oracle import texture as otex
    rng = np.random.RandomState(5)
    planes = rng.rand(2, 9, 23)
    kernels = rng.rand(3, 33, 33) - 0.5
    got = otex.convolve_reflect(planes, kernels)
    assert got.shape == (3, 2, 9, 23)
    for k in range(3):
        for p in range(2):
            np.testing.assert_allclose(got[k, p], ndimage.convolve(planes[p], kernels[k]), rtol=0, atol=1e-12)


def _split(x):
    """a float32 value as tf32 value + tf32 remainder, as k_lm_pad_split and bank_operand_layout form them"""
    from pyimsegm_b200.texture import _round_tf32
    x32 = np.asarray(x, dtype=np.float32)
    hi = _round_tf32(x32)
    lo = _round_tf32((x32 - hi).astype(np.float32))
    return hi.astype(np.float64), lo.astype(np.float64)


def test_per_pixel_bound_separates_3xtf32_from_a_broken_split():
    """the worst per-pixel error over M of the first ten batteries of the full bank, for the split the kernel uses and for the
    splits that drop a remainder product; the FP32 accumulation of the tensor cores is not emulated.  Measured when this test was
    written: 3xTF32 4.2e-8, no a_hi*b_lo 8.0e-5, no a_lo*b_hi 9.9e-5, 1xTF32 1.5e-4."""
    from oracle import texture as otex
    img = _textured(96, 300, seed=11)
    sub = np.rollaxis(img - ndimage.gaussian_filter(img, 150), -1, 0)
    M = np.abs(sub).max()
    a_hi, a_lo = _split(sub)
    bank, _ = otex.filter_bank()
    worst = {'3xTF32': 0., 'no a_hi*b_lo': 0., 'no a_lo*b_hi': 0., '1xTF32': 0.}
    for battery in bank[:10]:
        b_hi, b_lo = _split(battery)
        hh, hl, lh = (otex.convolve_reflect(a, b) for a, b in ((a_hi, b_hi), (a_hi, b_lo), (a_lo, b_hi)))
        want = np.max(otex.convolve_reflect(sub, battery), axis=0)
        variants = {'3xTF32': hh + hl + lh, 'no a_hi*b_lo': hh + lh, 'no a_lo*b_hi': hh + hl, '1xTF32': hh}
        for name, resp in variants.items():
            worst[name] = max(worst[name], np.abs(np.max(resp, axis=0) - want).max() / M)
    msg = ', '.join('%s %.3g' % kv for kv in worst.items())
    assert worst['3xTF32'] <= BOUND / 10, msg
    for name in ('no a_hi*b_lo', 'no a_lo*b_hi', '1xTF32'):
        assert worst[name] > 3 * BOUND, msg


@pytest.mark.parametrize('bank', ['normal', 'short'])
def test_oracle_features_of_an_image_with_nan_or_inf_are_zero(oracle, bank):
    """descriptors.py:1078-1100: the sigma-150 background spreads a NaN (or inf - inf) over the whole image, every battery's norm is
    NaN, and np.nan_to_num makes every feature 0"""
    from oracle import texture as otex
    img = _textured(12, 10, seed=3)
    seg = (np.arange(12)[:, None] // 4) * 2 + np.arange(10)[None, :] // 5
    flags = ('mean', 'std', 'energy')
    clean, _ = otex.texture_desc_lm(img, seg, flags, bank)
    assert np.count_nonzero(clean) > 0.9 * clean.size
    with_nan = img.copy()
    with_nan[5, 7, 1] = np.nan
    with_inf = img.copy()
    with_inf[2, 3, 0], with_inf[9, 1, 2] = np.inf, -np.inf
    for bad in (with_nan, with_inf):
        fts, _ = otex.texture_desc_lm(bad, seg, flags, bank)
        assert fts.shape == clean.shape and not fts.any()
        _, _, norms = otex.clipped_responses(bad, bank)
        assert np.all(np.isnan(norms)) and not otex.norm_scale(norms).any()
