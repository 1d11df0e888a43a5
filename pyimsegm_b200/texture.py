"""
Leung-Malik texture descriptors on the GPU (reference ``imsegm/descriptors.py:880-1106``).

Host side: the filter bank is built with numpy/scipy exactly like the reference does at run time
(``create_filter_bank_lm_2d``, descriptors.py:903-948), then laid out for the tensor-core contraction of
``isb_lm_texture`` (correlation form, oriented batteries first, tf32 hi/lo split, operand layout).  The contraction, the battery max,
the log-norm scaling and the per-superpixel statistics run in CUDA (``csrc/lm_texture.cu``).
"""
import ctypes as C
import functools

import numpy as np

from . import _lib
from .engine import flag_bits, get_engine

#: sigma of the background that is subtracted before filtering (descriptors.py:1078)
BACKGROUND_SIGMA = 150
_KW, _KWP = 33, 40
_BANK_CACHE = {}


def make_gaussian_filter1d(vals, sigma, order=0):
    """ sampled Gaussian (derivative of order 0..2) normalised to unit L1 norm (descriptors.py:880-891) """
    if order > 2:
        raise ValueError("Only orders up to 2 are supported")
    resp = np.exp(-vals ** 2 / (2. * sigma ** 2))
    if order == 1:
        resp = -resp * vals
    elif order == 2:
        resp = resp * (vals ** 2 - sigma ** 2)
    return resp / np.abs(resp).sum()


def make_edge_filter2d(sig, phase, points, sup):
    """ anisotropic (3 sigma x sigma) Gaussian derivative on the rotated grid ``points`` (descriptors.py:894-900) """
    ft = (make_gaussian_filter1d(points[0, :], sigma=3 * sig) * make_gaussian_filter1d(points[1, :], sigma=sig, order=phase))
    ft = ft.reshape(sup, sup)
    return ft / np.abs(ft).sum()


def create_filter_bank_lm_2d(radius=16, sigmas=None, nb_orient=8):
    """ Leung-Malik bank: per sigma 'edge' and 'bar' batteries of ``nb_orient`` rotated kernels, a Gaussian and two
    Laplacians of Gaussian (descriptors.py:903-948)

    :return tuple(list(ndarray),list(str)): batteries [n_kernels, 2r+1, 2r+1] and their names
    """
    from scipy.ndimage import gaussian_filter, gaussian_laplace
    from .descriptors import DEFAULT_FILTERS_SIGMAS
    sigmas = DEFAULT_FILTERS_SIGMAS if sigmas is None else sigmas
    support = 2 * radius + 1
    gx, gy = np.mgrid[-radius:radius + 1, radius:-radius - 1:-1]
    grid = np.vstack([gx.ravel(), gy.ravel()])
    impulse = np.zeros((support, support))
    impulse[radius, radius] = 1
    filters, names = [], []
    for sigma in sigmas:
        edges, bars = [], []
        for k in range(nb_orient):
            angle = np.pi * k / nb_orient  # half turn only: the kernels are symmetric
            rot = np.dot(np.array([[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]]), grid)
            edges.append(make_edge_filter2d(sigma, 1, rot, support))
            bars.append(make_edge_filter2d(sigma, 2, rot, support))
        filters += [np.asarray(edges), np.asarray(bars), gaussian_filter(impulse, sigma)[np.newaxis],
                    gaussian_laplace(impulse, sigma)[np.newaxis], gaussian_laplace(impulse, sigma ** 2)[np.newaxis]]
        names += ['sigma%.1f-%s' % (sigma, n) for n in ('edge', 'bar', 'Gauss', 'GaussLap', 'GaussLap2')]
    return filters, names


def lm_bank(bank_type):
    """:func:`create_filter_bank_lm_2d` of the 'short' bank (3 sigmas x 4 orientations, 15 batteries) or, for any other bank type,
    of the full one (4 x 8, 20 batteries)"""
    from .descriptors import SHORT_FILTERS_SIGMAS
    return create_filter_bank_lm_2d(sigmas=SHORT_FILTERS_SIGMAS, nb_orient=4) if bank_type == 'short' else create_filter_bank_lm_2d()


@functools.lru_cache(maxsize=None)
def bank_names(bank_type):
    """the battery names of :func:`lm_bank`, built once per bank type"""
    return tuple(lm_bank(bank_type)[1])


def _round_tf32(x):
    """cvt.rna.tf32.f32: round a float32 to 10 explicit mantissa bits, ties away from zero"""
    bits = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    out = ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return out


def bank_operand_layout(bank_type):
    """(names, w_tc, NP, orient, n_batt) for 'normal' / 'short' on the HOST.  ``w_tc`` holds, per kernel row, the weights in the operand
    layout of the tensor-core contraction (see isb_lm_texture): float32 [33 kernel rows][hi | lo][10 k-chunks][NP / 8][8 filters][4 taps],
    correlation form (kernels flipped), tf32-rounded value and tf32-rounded remainder, taps 33..39 and the padding filters zero"""
    filters, names = lm_bank(bank_type)
    orient, NP = (4, 48) if bank_type == 'short' else (8, 80)
    n_sig = len(filters) // 5
    cols = []
    for s in range(n_sig):      # oriented batteries first: edge s0 | bar s0 | edge s1 | ...
        cols += list(filters[5 * s]) + list(filters[5 * s + 1])
    for s in range(n_sig):      # then Gauss, LoG(sigma), LoG(sigma^2) per sigma
        cols += [filters[5 * s + 2][0], filters[5 * s + 3][0], filters[5 * s + 4][0]]
    assert len(cols) <= NP
    w = np.zeros((_KW, _KWP, NP), dtype=np.float64)
    for j, f in enumerate(cols):
        w[:, :_KW, j] = f[::-1, ::-1]          # ndimage.convolve == correlation with the flipped kernel
    w32 = w.astype(np.float32)
    hi = _round_tf32(w32)
    lo = _round_tf32((w32 - hi).astype(np.float32))
    # [dy][dx][n] -> [dy][half][dx // 4][n // 8][n % 8][dx % 4]: K-major core matrices of 8 filters x 4 taps (16 bytes)
    both = np.stack([hi, lo], axis=1).reshape(_KW, 2, _KWP // 4, 4, NP // 8, 8)
    w_tc = np.ascontiguousarray(both.transpose(0, 1, 2, 4, 5, 3))
    return names, w_tc, NP, orient, len(filters)


def _device_bank(bank_type):
    """(names, d_w_tc, NP, orient, n_batt) for 'normal' / 'short', cached per device (:func:`bank_operand_layout` uploaded once)"""
    eng = get_engine()
    key = (bank_type, eng.device.index)
    if key in _BANK_CACHE:
        return _BANK_CACHE[key]
    names, w_tc, NP, orient, n_batt = bank_operand_layout(bank_type)
    d_w = eng.torch.from_numpy(w_tc).to(eng.device)
    _BANK_CACHE[key] = (names, d_w, NP, orient, n_batt)
    return _BANK_CACHE[key]


def background_kernel(sigma=BACKGROUND_SIGMA, truncate=4.0):
    """scipy.ndimage's 1-D Gaussian (full, 2r+1 taps) and the same kernel folded onto a reflected length-3 axis (3x3)"""
    radius = int(truncate * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    w = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    w = w / w.sum()
    mix = np.zeros((3, 3))
    for c in range(3):
        idx = (c + x) % 6
        idx = np.where(idx < 3, idx, 5 - idx)        # reflect: (c b a | a b c | c b a)
        for cp in range(3):
            mix[c, cp] = w[idx == cp].sum()
    return np.ascontiguousarray(w), radius, np.ascontiguousarray(mix)


def device_lm_features(eng, d_img, d_seg, nb, flags, bank_type='normal', feat=None, col0=0):
    """run isb_lm_texture on device buffers; returns (feat tensor [nb, ld], names, n_cols)"""
    torch, lib = eng.torch, eng.lib
    names, d_w, NP, orient, n_batt = _device_bank(bank_type)
    bits, cols = flag_bits(flags)
    ncol = n_batt * cols
    if feat is None:
        feat = eng.buf('feat_lm', (nb, ncol), torch.float64)
    H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
    w_bg, radius, mix = background_kernel()
    d_wbg = eng.const_device(w_bg, 'lm_bg_w')
    wsb = lib.isb_lm_workspace_bytes(H, W, int(nb), n_batt)
    ws = eng.buf('ws_lm', (wsb,), torch.uint8)
    code = _lib.dtype_code(d_img.dtype)
    _lib.check(lib.isb_lm_texture(_lib.ptr(d_img), code, _lib.ptr(d_seg), H, W, int(nb), _lib.ptr(d_wbg), radius,
                                  mix.ctypes.data_as(C.POINTER(C.c_double)), _lib.ptr(d_w), NP, orient, n_batt, bits,
                                  _lib.ptr(feat), int(feat.shape[1]), int(col0), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
    return feat, names, ncol


def _device_batteries(eng, bank_type):
    """the batteries of :func:`create_filter_bank_lm_2d` for 'normal' / 'short' as f64 device tensors, uploaded once per device"""
    key = ('batteries', bank_type, eng.device.index)
    if key not in _BANK_CACHE:
        filters, _ = lm_bank(bank_type)
        _BANK_CACHE[key] = [eng.torch.from_numpy(np.ascontiguousarray(f, dtype=np.float64)).to(eng.device) for f in filters]
    return _BANK_CACHE[key]


def device_lm_materialised(eng, d_img, d_seg, nb, flags, bank_type, feat, col0):
    """the reference's own sequence (descriptors.py:1078-1098) with every response in memory, into feat[:, col0:] (battery-major):
    background subtraction (``isb_lm_background``), then per battery the clipped, log-norm scaled responses
    (``isb_lm_battery_response``) and their group statistics (:meth:`~.engine.Engine.group_stats`) -- the route for the statistics
    the fused kernel does not produce (``median``, ``meanGrad``).  Nothing is read back; the buffers are the engine's."""
    from .descriptors import MAX_SIGNAL_RESPONSE
    from .engine import gaussian_half_kernel
    torch, lib = eng.torch, eng.lib
    H, W = int(d_img.shape[0]), int(d_img.shape[1])
    st = _lib.stream_ptr()
    w_half, radius = gaussian_half_kernel(BACKGROUND_SIGMA)
    d_w = eng.const_device(w_half, 'lm_bg_half')
    _, _, mix = background_kernel()
    planar, tmp, smooth = (eng.buf(name, (3, H, W), torch.float64) for name in ('lmm_planar', 'lmm_tmp', 'lmm_smooth'))
    _lib.check(lib.isb_lm_background(_lib.ptr(d_img), _lib.dtype_code(d_img.dtype), H, W, _lib.ptr(d_w), radius,
                                     mix.ctypes.data_as(C.POINTER(C.c_double)), _lib.ptr(planar), _lib.ptr(tmp), _lib.ptr(smooth), st))
    out = eng.buf('lmm_out', (H, W, 3), torch.float64)
    wsb = lib.isb_lm_battery_workspace_bytes()
    ws = eng.buf('ws_lmm', (wsb,), torch.uint8)
    per_battery = 3 * len(flags)
    for b, d_k in enumerate(_device_batteries(eng, bank_type)):
        nk, kh, kw = (int(v) for v in d_k.shape)
        _lib.check(lib.isb_lm_battery_response(_lib.ptr(planar), H, W, _lib.ptr(d_k), nk, kh, kw, C.c_double(MAX_SIGNAL_RESPONSE),
                                               _lib.ptr(tmp), _lib.ptr(out), _lib.ptr(ws), C.c_size_t(wsb), st))
        eng.group_stats(out, d_seg, nb, flags, feat, col0 + b * per_battery)
    return feat


def compute_texture_desc_lm_img2d_clr(img, seg, feature_flags, bank_type='normal'):
    """ texture descriptors of a colour image: statistics of the Leung-Malik filter-bank responses per segment
    (reference descriptors.py:1041-1106), the texture group of :func:`~.descriptors.compute_selected_features_color2d`

    :param ndarray img: image [H, W, 3]
    :param ndarray seg: segmentation [H, W]
    :param list(str) feature_flags: subset of ('mean', 'std', 'energy', 'median', 'meanGrad')
    :param str bank_type: 'normal' (4 sigmas x 8 orientations, 20 batteries) or 'short' (3 x 4, 15 batteries)
    :return tuple(ndarray,list(str)): features [nb_segments, n_batteries * 3 * n_flags], names
    """
    from .descriptors import compute_selected_features_color2d
    return compute_selected_features_color2d(img, seg, {'tLM_short' if bank_type == 'short' else 'tLM': feature_flags})
