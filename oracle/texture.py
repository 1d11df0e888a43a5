"""
oracle/texture.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (numpy + scipy.ndimage, float64, the same library calls the reference makes) of the Leung-Malik
texture descriptors:
    imsegm/descriptors.py:880-948   make_gaussian_filter1d / make_edge_filter2d / create_filter_bank_lm_2d
    imsegm/descriptors.py:951-980   compute_img_filter_response2d / 3d  (ndimage.convolve, max over orientations)
    imsegm/descriptors.py:1041-1106 compute_texture_desc_lm_img2d_clr   (sigma-150 background, clip 1e6, log-norm, statistics)
The reference's doctests pin only SHAPES and NAMES (descriptors.py:911-922, 1052-1074, 1235-1239), but its own functions run in
this container (tests/golden/make_goldens.py): the bank and the descriptors of a textured image are pinned on their outputs
(tests/golden/reference_vectors.npz, tests/test_reference_vectors.py).
"""
import numpy as np
from scipy import ndimage

SIGMAS_FULL = (np.sqrt(2), 2, 2 * np.sqrt(2), 4)
SIGMAS_SHORT = (np.sqrt(2), 2, 4)
MAX_RESPONSE = 1.e6


def _gauss1d(vals, sigma, order=0):
    g = np.exp(-vals ** 2 / (2. * sigma ** 2))
    if order == 1:
        g = -g * vals
    elif order == 2:
        g = g * (vals ** 2 - sigma ** 2)
    return g / np.abs(g).sum()


def _edge2d(sig, phase, pts, sup):
    f = (_gauss1d(pts[0], 3 * sig) * _gauss1d(pts[1], sig, phase)).reshape(sup, sup)
    return f / np.abs(f).sum()


def filter_bank(radius=16, sigmas=SIGMAS_FULL, nb_orient=8):
    sup = 2 * radius + 1
    x, y = np.mgrid[-radius:radius + 1, radius:-radius - 1:-1]
    pts = np.vstack([x.ravel(), y.ravel()])
    delta = np.zeros((sup, sup))
    delta[radius, radius] = 1
    bank, names = [], []
    for sigma in sigmas:
        edge, bar = [], []
        for o in range(nb_orient):
            ang = np.pi * o / nb_orient
            c, s = np.cos(ang), np.sin(ang)
            rot = np.dot(np.array([[c, -s], [s, c]]), pts)
            edge.append(_edge2d(sigma, 1, rot, sup))
            bar.append(_edge2d(sigma, 2, rot, sup))
        bank += [np.asarray(edge), np.asarray(bar), ndimage.gaussian_filter(delta, sigma)[None],
                 ndimage.gaussian_laplace(delta, sigma)[None], ndimage.gaussian_laplace(delta, sigma ** 2)[None]]
        names += ['sigma%.1f-%s' % (sigma, n) for n in ('edge', 'bar', 'Gauss', 'GaussLap', 'GaussLap2')]
    return bank, names


def battery_responses(img, bank_type='normal', background_sigma=150):
    """normalised responses [n_batteries, 3, H, W] float64 (descriptors.py:1078-1094)"""
    img = np.asarray(img)
    img = img - ndimage.gaussian_filter(img.astype(float), background_sigma)
    roll = np.rollaxis(img, -1, 0)
    bank, names = filter_bank(sigmas=SIGMAS_SHORT, nb_orient=4) if bank_type == 'short' else filter_bank()
    out = []
    for battery in bank:
        resp = np.array([np.max([ndimage.convolve(ch, f) for f in battery], axis=0) for ch in roll])
        resp[resp > MAX_RESPONSE] = MAX_RESPONSE
        norm = np.sqrt(np.sum(resp ** 2))
        if norm == 0 or abs(norm) == np.inf:
            resp = np.zeros(resp.shape)
        else:
            resp = (resp * (np.log(1 + norm) / 0.03)) / norm
        out.append(resp)
    return np.array(out), names


def reflect_index(n, pad):
    """indices of an axis of length n padded by ``pad`` on both sides in ndimage's mode 'reflect' (d c b a | a b c d | d c b a), for
    any pad: the 2n-periodic reflection.  np.pad(mode='symmetric') differs from it once the pad is wider than the axis."""
    i = np.arange(-pad, n + pad) % (2 * n)
    return np.where(i < n, i, 2 * n - 1 - i)


def convolve_reflect(planes, kernels):
    """ndimage.convolve(plane, kernel) (mode 'reflect') of every plane [..., H, W] with every odd square kernel [K, k, k], in float64
    by FFT: reflect-pad, then fftconvolve 'valid'.  Returns [K, ..., H, W]."""
    from scipy import signal
    planes = np.asarray(planes, dtype=np.float64)
    kernels = np.asarray(kernels, dtype=np.float64)
    r = kernels.shape[-1] // 2
    H, W = planes.shape[-2:]
    padded = planes[..., reflect_index(H, r)[:, None], reflect_index(W, r)[None, :]]
    kern = kernels.reshape(kernels.shape[:1] + (1, ) * (planes.ndim - 2) + kernels.shape[1:])
    return signal.fftconvolve(padded[None], kern, mode='valid', axes=(-2, -1))


def clipped_responses(img, bank_type='normal', background_sigma=150):
    """the reference's responses before their log-norm scaling (descriptors.py:1078-1092), by FFT in float64:
    (img - background [3, H, W], clipped battery responses [n_batteries, 3, H, W], battery norms [n_batteries]).
    A battery's scaled response is ``a * resp`` with ``a = log(1 + norm) / 0.03 / norm`` (0 when the norm is 0 or infinite)."""
    img = np.asarray(img)
    sub = img - ndimage.gaussian_filter(img.astype(float), background_sigma)
    roll = np.rollaxis(sub, -1, 0)
    bank, _ = filter_bank(sigmas=SIGMAS_SHORT, nb_orient=4) if bank_type == 'short' else filter_bank()
    out = np.empty((len(bank), ) + roll.shape)
    for b, battery in enumerate(bank):
        resp = np.max(convolve_reflect(roll, battery), axis=0)
        resp[resp > MAX_RESPONSE] = MAX_RESPONSE
        out[b] = resp
    return roll, out, np.sqrt(np.sum(out ** 2, axis=(1, 2, 3)))


def norm_scale(norms):
    """the log-norm factor a of every battery (descriptors.py:1090-1094); 0 for a norm of 0, inf or NaN, whose features are 0"""
    norms = np.asarray(norms, dtype=np.float64)
    ok = (norms != 0) & np.isfinite(norms)
    safe = np.where(ok, norms, 1.)
    return np.where(ok, np.log(1 + safe) / 0.03 / safe, 0.)


def texture_desc_lm(img, seg, flags, bank_type='normal', stat_fn=None):
    """features [N, n_batteries * 3 * len(flags)] in the reference's column order, names"""
    import oracle
    resp, names = battery_responses(img, bank_type)
    cols, out_names = [], []
    for r, name in zip(resp, names):
        fts = oracle.image2d_color_statistic(np.rollaxis(r, 0, 3), seg, flags)
        cols.append(fts)
        out_names += ['tLM_%s-ch%i_%s' % (name, c + 1, f) for f in ('mean', 'std', 'energy', 'median', 'meanGrad') if f in flags for c in range(3)]
    fts = np.nan_to_num(np.concatenate(cols, axis=1))
    fts[fts == 0] = 0
    return fts, out_names
