"""Every Leung-Malik response pixel by pixel against the float64 oracle (oracle/texture.py `clipped_responses`), on both device routes.

A label map with one label per pixel (seg = arange(H W)) makes each pixel its own segment, so a pixel's 'mean' feature is a r(y, x):
r the clipped battery response, a = log(1 + ||r||) / 0.03 / ||r|| the log-norm factor of its battery.  Errors are measured against
a M, M = max |img - background|, the scale every response of the image is made from.

- Fused route (mean / std / energy: the tensor-core contraction of csrc/lm_texture.cu, 3xTF32 with FP32 accumulation):
  |mean - a r| <= 1e-5 a M at every pixel, channel and battery.  A split that drops one of its remainder products costs 8e-5 to
  1.5e-4, the split itself 4e-8 (tests/test_lm_oracle_host.py); the rest of the budget is the FP32 accumulation of the tensor
  cores.  Worst ratio measured on an H100 80GB HBM3 at 700 W, over every shape, dtype and the clipped image below: full bank 2.2e-6,
  short bank 2.1e-6.
- Materialised route (median, meanGrad: FP64 direct sums of native_misc.cu): the median within 1e-10 a M; the mean also carries
  the reference's rounding of every response to f32 before its statistics (descriptors.py:233), half an f32 ulp of a r.
- The shapes put the tiles (128 pixels x 3 rows) and the reflections at their edges: W < 128, W = 128, W = 129 (a second tile of one
  pixel), W >= 664; H mod 3 in {0, 1, 2}; both axes shorter than the 16-pixel kernel radius; each axis on either side of the
  background blur's single-reflection branch (taken when the axis has at least 600 + 64 pixels).
- A NaN or infinite pixel zeroes every texture feature on both routes, as np.nan_to_num does on the reference's NaN features.
  float64 images with values beyond the float32 range are out of scope: the fused route narrows the image to float32.

Every assertion names its worst element: battery, channel, pixel, its place in the tile and its distance to the border."""
import functools

import numpy as np
import pytest

from test_gpu_resident_features import FLAGS, _as_dtype, _colour_reference, _compare_group

pytestmark = pytest.mark.gpu

SHAPES = [(7, 5), (2, 129), (35, 128), (64, 300), (97, 257), (663, 131), (664, 40), (40, 700)]
BANKS = ['normal', 'short']
FUSED = ('mean', 'std', 'energy')
MATERIALISED = ('mean', 'median')
FUSED_BOUND = 1e-5
FP64_BOUND = 1e-10


def _image(shape, seed):
    """noise around 0.45, an oblique sine texture in the lower half and a horizontal one in the second channel, within [0, 1]"""
    h, w = shape
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:h, :w]
    img = 0.3 + 0.3 * rng.random_sample((h, w, 3))
    img += (0.2 * np.sin(xx / 3.0 + yy / 5.0) * (yy >= h // 2))[..., None]
    img[..., 1] += 0.1 * np.cos(yy / 4.0)
    return np.clip(img, 0, 1)


@functools.lru_cache(maxsize=None)
def _case(shape, bank, dtype='float64', scale=1.0):
    """(image, clipped responses [n_batt, 3, H, W], a [n_batt], M) of the test image of a shape in a dtype"""
    from oracle import texture as otex
    img = _image(shape, seed=shape[0] * 1000 + shape[1]) * scale
    img = _as_dtype(img, getattr(np, dtype)) if scale == 1.0 else img.astype(getattr(np, dtype))
    sub, resp, norms = otex.clipped_responses(img, bank)
    return img, resp, otex.norm_scale(norms), np.abs(sub).max()


def _key(bank):
    return 'tLM_short' if bank == 'short' else 'tLM'


def _per_pixel(img, bank, flags):
    """the features of one label per pixel as [n_batt, len(flags), 3, H, W]"""
    from pyimsegm_b200.descriptors import compute_selected_features_color2d
    H, W = img.shape[:2]
    seg = np.arange(H * W).reshape(H, W)
    fts, _ = compute_selected_features_color2d(img, seg, {_key(bank): flags})
    return fts.reshape(H, W, -1, len(flags), 3).transpose(2, 3, 4, 0, 1)


def _worst(ratio, bank, what):
    """(worst ratio, a message naming its element) of ratio [n_batt, 3, H, W]; NaN counts as the worst"""
    from pyimsegm_b200.texture import bank_names
    r = np.where(np.isnan(ratio), np.inf, ratio)
    b, c, y, x = np.unravel_index(np.argmax(r), r.shape)
    H, W = r.shape[-2:]
    msg = ('%s, %s bank %dx%d: battery %d (%s), channel %d, (y, x) = (%d, %d), y %% 3 = %d, x %% 128 = %d, distance to the border %d: '
           'ratio %.3g' % (what, bank, H, W, b, bank_names(bank)[b], c, y, x, y % 3, x % 128, min(y, x, H - 1 - y, W - 1 - x), r[b, c, y, x]))
    return r[b, c, y, x], msg


def _check_fused(img, bank, resp, a, M):
    got = _per_pixel(img, bank, FUSED)
    mean, std, energy = got[:, 0], got[:, 1], got[:, 2]
    aM = (a * M)[:, None, None, None]
    worst, msg = _worst(np.abs(mean - a[:, None, None, None] * resp) / aM, bank, 'mean')
    assert worst <= FUSED_BOUND, msg
    rel, msg = _worst(np.abs(energy - mean ** 2) / np.maximum(mean ** 2, 1e-300), bank, 'energy against mean^2')
    assert rel <= 1e-12, msg
    sd, msg = _worst(std / aM, bank, 'std of one pixel')
    assert sd <= 1e-6, msg
    print('fused per-pixel ratio %s %s %s: %.3g' % (bank, img.shape[:2], img.dtype, worst))
    return worst


def _check_materialised(img, bank, resp, a, M):
    got = _per_pixel(img, bank, MATERIALISED)
    want = a[:, None, None, None] * resp
    aM = (a * M)[:, None, None, None]
    excess = np.maximum(np.abs(got[:, 0] - want) - 2.0 ** -24 * np.abs(want) * (1 + 1e-9), 0)
    worst, msg = _worst(excess / aM, bank, 'mean (beyond half an f32 ulp)')
    assert worst <= FP64_BOUND, msg
    worst, msg = _worst(np.abs(got[:, 1] - want) / aM, bank, 'median')
    assert worst <= FP64_BOUND, msg


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('bank', BANKS)
def test_fused_route_per_pixel(shape, bank):
    img, resp, a, M = _case(shape, bank)
    _check_fused(img, bank, resp, a, M)


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('bank', BANKS)
def test_materialised_route_per_pixel(shape, bank):
    img, resp, a, M = _case(shape, bank)
    _check_materialised(img, bank, resp, a, M)


@pytest.mark.parametrize('dtype', ['uint8', 'uint16', 'float32', 'float64'])
def test_fused_route_per_pixel_in_every_dtype(dtype):
    img, resp, a, M = _case((48, 160), 'normal', dtype)
    assert img.dtype == getattr(np, dtype)
    _check_fused(img, 'normal', resp, a, M)


@pytest.mark.parametrize('bank', BANKS)
def test_fused_route_clips_at_1e6(bank):
    """a float32 image scaled by 1e7: many Gauss and LoG responses lie beyond 1e6 (clipped) and below -1e6 (kept)"""
    img, resp, a, M = _case((64, 300), bank, 'float32', 1e7)
    from pyimsegm_b200.texture import bank_names
    gauss = [b for b, n in enumerate(bank_names(bank)) if n.endswith('Gauss')]
    assert np.mean(resp[gauss] == 1e6) > 0.05 and np.mean(resp < -1e6) > 0.01
    _check_fused(img, bank, resp, a, M)


def _fragmented_labels(h, w, seed, n_labels=7):
    """runs of random labels along x, 1 to 47 pixels long; on every other row the label also changes at each multiple of 64
    (the half-row a run-length walker of the fused kernel owns) while on the others runs cross those boundaries"""
    rng = np.random.RandomState(seed)
    seg = np.empty((h, w), dtype=np.int64)
    for y in range(h):
        x = 0
        while x < w:
            run = rng.randint(1, 48)
            seg[y, x:x + run] = rng.randint(n_labels)
            x += run
        if y % 2 == 0:
            for x0 in range(64, w, 64):
                seg[y, x0:] = np.where(seg[y, x0:] == seg[y, x0 - 1], (seg[y, x0:] + 1) % n_labels, seg[y, x0:])
    return seg


@pytest.mark.parametrize('bank', BANKS)
def test_fused_route_on_fragmented_labels(bank):
    """seven labels in short runs over (97, 257): the walker's flushes at label changes, at the ends of its half-row and tile, and
    the atomics that add the pieces of a segment"""
    from pyimsegm_b200.descriptors import compute_selected_features_color2d
    from pyimsegm_b200.texture import bank_names
    img, resp, a, M = _case((97, 257), bank)
    seg = _fragmented_labels(97, 257, seed=5)
    assert np.all(seg[::2, 64::64] != seg[::2, 63:-1:64]) and np.any(seg[1::2, 64::64] == seg[1::2, 63:-1:64])
    fts, _ = compute_selected_features_color2d(img, seg, {_key(bank): FUSED})
    got = fts.reshape(7, len(a), 3, 3)                     # [segment, battery, statistic, channel]
    rmax = np.abs(resp).max(axis=(1, 2, 3))
    names = bank_names(bank)
    for k in range(7):
        mask = seg == k
        r = resp[:, :, mask]
        mean = a[:, None] * r.mean(-1)
        energy = (a ** 2)[:, None] * (r ** 2).mean(-1)
        std = np.sqrt(np.maximum(energy - mean ** 2, 0))
        for i, (want, scale) in enumerate(((mean, a * M), (std, a * M), (energy, 2 * a ** 2 * M * rmax))):
            ratio = np.abs(got[k, :, i] - want) / scale[:, None]
            b, c = np.unravel_index(np.argmax(np.where(np.isnan(ratio), np.inf, ratio)), ratio.shape)
            assert ratio[b, c] <= FUSED_BOUND, '%s, %s bank: segment %d (%d pixels), battery %d (%s), channel %d: ratio %.3g' % (
                FUSED[i], bank, k, mask.sum(), b, names[b], c, ratio[b, c])


@pytest.mark.parametrize('case', ['nan-float32', 'nan-float64', 'inf-float32', 'inf-float64'])
def test_nan_or_inf_pixel_zeroes_every_texture_column(case):
    """one NaN pixel, or one +inf and one -inf: the sigma-150 background carries them over the whole image, so the reference's
    battery norms are NaN and every texture feature is 0 after np.nan_to_num -- on the fused route as on the materialised one.  The
    colour columns are the host's colour statistics of the same image."""
    from pyimsegm_b200.descriptors import compute_selected_features_color2d
    kind, dtype = case.split('-')
    img = _image((40, 36), seed=6).astype(dtype)
    seg = (np.arange(40)[:, None] // 8) * 6 + np.arange(36)[None, :] // 6
    clean = img.copy()
    if kind == 'nan':
        img[17, 20, 1] = np.nan
    else:
        img[3, 4, 0], img[30, 25, 2] = np.inf, -np.inf
    for flags in (FUSED, MATERIALISED):
        feats = {'color': FLAGS, 'tLM_short': flags}
        base, _ = compute_selected_features_color2d(clean, seg, feats)
        assert np.count_nonzero(base[:, 15:]) > 0.9 * base[:, 15:].size
        got, _ = compute_selected_features_color2d(img, seg, feats)
        bad = np.flatnonzero(np.any(got[:, 15:] != 0, axis=0))
        assert bad.size == 0, '%s, %s: %d texture columns are not 0 (first %d, max |x| %g)' % (
            case, flags, bad.size, bad[0] if bad.size else -1, np.abs(got[:, 15:]).max())
        _compare_group(got[:, :15], _colour_reference(img, seg, 'color', FLAGS), 'color', 9)
