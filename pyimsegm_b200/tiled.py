"""
Row-band mode: ONE image cut into horizontal bands, one band (or a few) per GPU -- BASELINE config 5 (a single 8192 x 8192
image over 8 GPUs), SURVEY.md section 8(e) "one huge image".

What shards and what does not (reference call stack ``imsegm/pipelines.py:46-110``):

* pixel-sized work is banded: H2D of the band, min-max / blur / rgb2lab, the 10 SLIC sweeps, the colour statistics, the
  final LUT gathers and their D2H.  Per sweep the bands exchange one buffer of 6 int64 words per cluster (the centroids as
  bit patterns; summed as integers, which is an exact merge because every cluster has exactly one owner) -- the one real
  exchange step of the path, an ``all_reduce`` over NCCL.
* superpixel-sized work is replicated: every GPU gets the whole k-means label map (band broadcasts over NVLink), runs the
  connectivity pass, the adjacency extraction, the class model and the alpha-expansion on it.  These are small next to the
  pixel work and identical on every rank, so nothing has to be sent back.

The label map is bit-identical to the single-GPU path (tests/test_gpu_tiled.py): the pixel-centric assignment does not care
how the pixels are partitioned, and the raster-order sequential centroid sums are formed by the one band that owns the
cluster, over a slab that holds every member (checked on the device; an orphan pixel outside the slab makes every rank fall
back to the whole image on its own GPU).

Several bands may live on one GPU (``bands_per_rank``); the merge between them is the same integer sum done by
``isb_combine`` -- that is also how the single-GPU tests exercise every code path of the exchange.

Features: any group of ``descriptors.RESIDENT_FEATURE_GROUPS`` (the image, its colour spaces, the two Leung-Malik banks) with mean /
std / energy / meanGrad (``descriptors.flags_are_banded``); a median does not decompose over bands and is refused.  ``meanGrad``
takes the gradient of the owned rows +- 1 and keeps the owned rows; the Leung-Malik responses' norms are summed over the bands in
band order between the two halves of the battery step.  Models: :func:`pipe_color2d_slic_features_model_graphcut_tiled` fits any
device ``estim_model`` / ``pca_coef`` on the replicated feature table, :func:`segment_color2d_slic_features_model_graphcut_tiled`
applies a caller-fitted one (on the device when ``class_models.compile_model`` takes it, on every rank's host otherwise).

Slab mode: ONE gray volume cut into z-slabs the same way (:func:`slab_plan` is :func:`plan_bands` along z), for
:func:`pipe_gray3d_slic_features_model_graphcut_tiled` and :func:`segment_gray3d_slic_features_model_graphcut_tiled`:

* slab ``i`` owns slices [own_lo, own_hi); its k-means slab is the owned slices +- ``2 step_z + 1`` (every member the assignment
  gives a cluster lies within ``2 step_z`` slices of its centre), its raw slab the k-means slab +- the z-blur radius; the blur
  reflects z at the volume's borders, not the slab's.  A cluster is owned by the slab whose owned slices hold its centre's z at
  the start of the sweep.
* per sweep the slabs exchange ``5 n + 1`` int64 words (``isb_slic3d_slab_*``): per cluster the bit patterns of (cz, cy, cx, cv)
  and an alive flag, zero in every slab but the owner's, then the orphan counter; the integer sum is an exact merge.  A voxel no
  window reaches, with a label whose centre is beyond the halo, makes every rank redo the sweeps on the whole volume.
* replicated: every rank gets the whole k-means label volume (slab broadcasts) and runs the 3-D connectivity, the statistics'
  finish, the scaler, the class model and the cut on the whole supervoxel graph.  Mean / std / energy are accumulated over the
  owned slices and all-reduced between the calls; a median is refused.
* memory per rank: its raw slabs (dtype + two f64 copies), 16 bytes per k-means-slab voxel, and about 44 bytes per voxel of the
  WHOLE volume (label volume, connectivity workspace and output): slabs share out the voxel-sized blur and sweeps but do not raise
  the largest volume one GPU can take; the connectivity's int voxel indices cap a volume below 2^31 / 4 voxels.
"""
import ctypes as C
import logging

import numpy as np

from . import _lib
from .engine import edge_capacity, edges_fit, flag_bits, gaussian_half_kernel, get_engine, slic_seed_grid, slic_seed_grid3d

OP_SUM_I64, OP_MAX_I64, OP_MIN_F64, OP_MAX_F64, OP_SUM_F64 = 0, 1, 2, 3, 4


class Band(object):
    """rows of one band: owned [own_lo, own_hi), k-means slab [km_lo, km_hi) = owned +- halo, raw slab = k-means slab +-
    blur radius, uploaded rows [up_lo, up_hi) = the raw slab or owned +- ``margin`` (what a descriptor with a wide footprint
    asks for), whichever reaches further (all clipped to the image)"""

    def __init__(self, index, own_lo, own_hi, H, halo, radius, margin=0):
        self.index = index
        self.own_lo, self.own_hi = own_lo, own_hi
        self.km_lo, self.km_hi = max(own_lo - halo, 0), min(own_hi + halo, H)
        self.raw_lo, self.raw_hi = max(self.km_lo - radius, 0), min(self.km_hi + radius, H)
        self.up_lo, self.up_hi = min(self.raw_lo, max(own_lo - margin, 0)), max(self.raw_hi, min(own_hi + margin, H))

    def __repr__(self):
        return 'Band(%d: own %d:%d, slab %d:%d, raw %d:%d)' % (self.index, self.own_lo, self.own_hi, self.km_lo, self.km_hi,
                                                            self.raw_lo, self.raw_hi)


def plan_bands(H, n_bands, halo, radius, margin=0):
    """equal bands of ceil(H / n_bands) rows (the last one takes what is left); every band must own at least one row"""
    rows = -(-int(H) // int(n_bands))
    bands = []
    for b in range(n_bands):
        lo, hi = b * rows, min((b + 1) * rows, H)
        if lo >= hi:
            raise ValueError('an image of %d rows cannot be cut into %d bands of %d rows' % (H, n_bands, rows))
        bands.append(Band(b, lo, hi, H, halo, radius, margin))
    return bands


class LoopbackComm(object):
    """world of one process"""
    rank, world = 0, 1

    def all_reduce(self, t, op):
        pass

    def broadcast(self, t, src):
        pass


class GroupComm(object):
    """torch.distributed process group (NCCL on the GPUs); tensors are reduced in place"""

    def __init__(self, group=None):
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self._ops = {'sum': dist.ReduceOp.SUM, 'max': dist.ReduceOp.MAX, 'min': dist.ReduceOp.MIN}

    def all_reduce(self, t, op):
        self.dist.all_reduce(t, op=self._ops[op], group=self.group)

    def broadcast(self, t, src):
        src = src if self.group is None else self.dist.get_global_rank(self.group, src)
        self.dist.broadcast(t, src=src, group=self.group)


def default_comm(group=None):
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        return GroupComm(group)
    return LoopbackComm()


class TiledSuperpixels(object):
    """device-resident result of :func:`slic_tiled`"""
    shape = bands = local = d_raw = d_seg = d_n_labels = nb_bound = d_feat = d_centres = d_err = None
    fell_back = False


def _combine(lib, dst_ptr, src_ptr, n, op):
    _lib.check(lib.isb_combine(C.c_void_p(dst_ptr), C.c_void_p(src_ptr), C.c_longlong(int(n)), int(op), _lib.stream_ptr()))


def _band_extrema(lib, ptr, code, n, mm, mm_b, first):
    """[min, max] of the ``n`` samples at device ``ptr`` into mm[0:2] (the first band of a rank) or merged into it (the others,
    through ``mm_b``); numpy's rule: a NaN sample makes both NaN (isb_image_minmax, isb_combine)"""
    tgt = mm if first else mm_b
    _lib.check(lib.isb_image_minmax(C.c_void_p(ptr), code, C.c_longlong(int(n)), _lib.ptr(tgt), _lib.stream_ptr()))
    if not first:
        _combine(lib, mm.data_ptr(), mm_b.data_ptr(), 1, OP_MIN_F64)
        _combine(lib, mm.data_ptr() + 8, mm_b.data_ptr() + 8, 1, OP_MAX_F64)


def _rank_extrema(comm, mm):
    """the extrema mm[0:2] of every rank's bands merged over the ranks"""
    if comm.world > 1:
        # a NaN sample makes both extrema NaN (numpy's rule, kept by isb_image_minmax and isb_combine); the collectives' min and
        # max need not keep a NaN, so a flag carries it across the GPUs
        has_nan = mm[0:1].isnan().to(mm.dtype)
        comm.all_reduce(mm[0:1], 'min')
        comm.all_reduce(mm[1:2], 'max')
        comm.all_reduce(has_nan, 'max')
        mm[0:2].masked_fill_(has_nan > 0, float('nan'))


def slic_tiled(image, n_segments, compactness, sigma=1.0, max_iter=10, slic_zero=False, rescale=True, comm=None,
               bands_per_rank=1, eng=None, min_size_factor=0.5, max_size_factor=3, enforce_connectivity=True, defer_check=False,
               force_whole=False, raw_margin=0):
    """ SLIC of one host image over the bands of ``comm`` (every rank passes the same image; it uploads only its rows)

    :param ndarray image: [H, W, C] host array, C in {1, 3}, dtype uint8 / uint16 / float32 / float64
    :return TiledSuperpixels: ``d_seg`` = the whole label map on this GPU (identical on every rank), ``d_raw[i]`` = the raw
        image rows ``bands[local[i]].up_lo:up_hi`` still on the device for the descriptors
    :param bool defer_check: do not synchronise to read the orphan counter ``res.d_err``; the caller reads it with its own
        results and calls again with ``force_whole=True`` when it is not zero
    :param bool force_whole: skip the banded sweeps, every rank runs them on the whole image (the fallback)
    :param int raw_margin: keep at least this many raw rows above and below the owned ones on the device (``d_raw[i]`` then holds
        the rows ``bands[local[i]].up_lo:up_hi``) -- the Leung-Malik descriptor needs its background radius + 16
    """
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    image = np.asarray(image)
    if image.ndim == 2:
        image = image[:, :, None]
    H, W, Cn = int(image.shape[0]), int(image.shape[1]), int(image.shape[2])
    code = _lib.dtype_code(image.dtype)
    itemsize = image.dtype.itemsize
    st = _lib.stream_ptr()
    w_half, radius = gaussian_half_kernel(sigma)
    seeds, ty, tx = slic_seed_grid(H, W, n_segments)
    n_seeds = len(seeds)
    step = float(max(1, ty, tx))
    halo = 2 * ty + 1
    n_bands = comm.world * int(bands_per_rank)
    bands = plan_bands(H, n_bands, halo, radius, int(raw_margin))
    local = list(range(comm.rank * bands_per_rank, (comm.rank + 1) * bands_per_rank))
    owner = lambda b: b // bands_per_rank  # noqa: E731

    res = TiledSuperpixels()
    res.shape, res.bands, res.local = (H, W), bands, local
    d_seeds = eng.to_device(seeds, 'seeds')
    mm = eng.buf('tb_minmax', (4,), torch.float64)
    mm_b = eng.buf('tb_minmax_b', (4,), torch.float64)
    wsb = lib.isb_slic_kmeans_workspace_bytes(H, W, n_seeds, ty, tx)

    # 1) upload the raw rows, extrema of the owned rows
    res.d_raw = []
    for i, b in enumerate(local):
        bd = bands[b]
        raw = eng.to_device(image[bd.up_lo:bd.up_hi], 'tb%d_raw' % i)
        res.d_raw.append(raw)
        if rescale:
            own_ptr = raw.data_ptr() + (bd.own_lo - bd.up_lo) * W * Cn * itemsize
            _band_extrema(lib, own_ptr, code, (bd.own_hi - bd.own_lo) * W * Cn, mm, mm_b, first=i == 0)
    if rescale:
        _rank_extrema(comm, mm)

    # 2) blur + rgb2lab of every raw slab, band descriptors
    descs, keep = [], []
    xchg = [eng.buf('tb%d_xchg' % i, (6 * n_seeds + 1,), torch.int64) for i in range(len(local))]
    mdc = [eng.buf('tb%d_maxdc' % i, (n_seeds,), torch.int64) for i in range(len(local))] if slic_zero else [None] * len(local)
    err = eng.buf('tb_err', (1,), torch.int64)
    err.zero_()
    for i, b in enumerate([] if force_whole else local):
        bd = bands[b]
        hraw = bd.raw_hi - bd.raw_lo
        lab = eng.buf('tb%d_lab' % i, (3, hraw, W), torch.float64)
        raw_ptr = C.c_void_p(res.d_raw[i].data_ptr() + (bd.raw_lo - bd.up_lo) * W * Cn * itemsize)
        _lib.check(lib.isb_slic_prepare(raw_ptr, code, hraw, W, Cn, w_half.ctypes.data_as(C.POINTER(C.c_double)), radius,
                                        C.c_double(1.0 / compactness), 2 if rescale else 0, _lib.ptr(lab), _lib.ptr(mm), st))
        slab_rows = bd.km_hi - bd.km_lo
        labels = eng.buf('tb%d_labels' % i, (slab_rows, W), torch.int32)
        ws = eng.buf('tb%d_ws' % i, (wsb,), torch.uint8)
        d = _lib.SlicBand(slab_rows=slab_rows, width=W, image_rows=H, y_off=bd.km_lo, own_lo=bd.own_lo, own_hi=bd.own_hi, halo=halo,
                          n_seeds=n_seeds, step_y=ty, step_x=tx, slic_zero=int(bool(slic_zero)), step=step,
                          lab_slab=lab.data_ptr() + (bd.km_lo - bd.raw_lo) * W * 8, plane_stride=hraw * W,
                          seeds_yx=d_seeds.data_ptr(), labels_slab=labels.data_ptr(), ws=ws.data_ptr(), ws_bytes=wsb)
        descs.append(d)
        keep.append((lab, labels, ws))
        _lib.check(lib.isb_slic_band_begin(C.byref(d), st))

    # 3) the sweeps: assign, sum the owned clusters, merge, take the merged centroids
    for _ in range(0 if force_whole else int(max_iter)):
        for i, d in enumerate(descs):
            _lib.check(lib.isb_slic_band_assign(C.byref(d), st))
            _lib.check(lib.isb_slic_band_update(C.byref(d), _lib.ptr(xchg[i]), st))
            if i > 0:
                _combine(lib, xchg[0].data_ptr(), xchg[i].data_ptr(), 6 * n_seeds + 1, OP_SUM_I64)
        comm.all_reduce(xchg[0], 'sum')
        _combine(lib, err.data_ptr(), xchg[0].data_ptr() + 8 * 6 * n_seeds, 1, OP_SUM_I64)
        for i, d in enumerate(descs):
            _lib.check(lib.isb_slic_band_import(C.byref(d), _lib.ptr(xchg[0]), _lib.ptr(mdc[i]), st))
            if slic_zero and i > 0:
                _combine(lib, mdc[0].data_ptr(), mdc[i].data_ptr(), n_seeds, OP_MAX_I64)
        if slic_zero:
            comm.all_reduce(mdc[0], 'max')
        for d in descs:
            _lib.check(lib.isb_slic_band_finalize(C.byref(d), _lib.ptr(mdc[0]), st))

    # 4) the whole k-means label map on every GPU
    full = eng.buf('tb_full', (H, W), torch.int32)
    res.d_err = err
    if not force_whole:
        for i, b in enumerate(local):
            bd = bands[b]
            full[bd.own_lo:bd.own_hi].copy_(keep[i][1][bd.own_lo - bd.km_lo:bd.own_hi - bd.km_lo])
        if comm.world > 1:
            for bd in bands:
                comm.broadcast(full[bd.own_lo:bd.own_hi], owner(bd.index))
    if force_whole or (not defer_check and int(eng.to_host(err)[0]) != 0):
        # some pixel kept the label of a cluster centred beyond the halo (no window covers it -- only degenerate inputs do
        # that): the banded sums are not trustworthy, every rank redoes the sweeps on the whole image on its own GPU
        logging.warning('slic_tiled: orphan pixels beyond the halo, redoing the sweeps on the whole image on every GPU')
        res.fell_back = True
        d_img = eng.to_device(image if Cn == 3 else image[:, :, 0], 'image')
        km, _ = eng.slic(d_img, n_segments, compactness, sigma=sigma, max_iter=max_iter, enforce_connectivity=False,
                         slic_zero=slic_zero, rescale=rescale)
        full.copy_(km)
    if not enforce_connectivity:
        res.d_seg = full
        return res
    res.d_seg, res.d_n_labels = eng.enforce_connectivity(full, n_segments, min_size_factor, max_size_factor)
    res.nb_bound = eng.slic_label_bound(H, W, n_segments, min_size_factor)
    return res


def _stats_banded(res, source, flags, feat, col0, centres, comm, eng):
    """statistics ``flags`` (of mean / std / energy) of a banded 3-channel source over ``res.d_seg`` into feat[:, col0:] (and the
    centroids into ``centres`` unless it is None): every band accumulates its owned rows, the accumulators are summed over the GPUs
    between the calls, every GPU finishes the same table.  ``source(i)`` -> (device pointer to the owned rows [rows, W, 3] of local
    band i, isb dtype code); it is called right before each pass over the band, so it may fill a buffer the bands share."""
    torch, lib = eng.torch, eng.lib
    W = res.shape[1]
    nb = int(res.nb_bound)
    st = _lib.stream_ptr()
    bits, _ = flag_bits(flags)
    acc = eng.buf('tb_acc', (nb, 6), torch.float64)
    iacc = eng.buf('tb_iacc', (nb, 3), torch.int64)
    acc.zero_()
    iacc.zero_()

    def rows(i, b):
        bd = res.bands[b]
        ptr, code = source(i)
        return bd, C.c_void_p(ptr), code, C.c_void_p(res.d_seg.data_ptr() + bd.own_lo * W * 4)

    for i, b in enumerate(res.local):
        bd, img_ptr, code, seg_ptr = rows(i, b)
        _lib.check(lib.isb_segment_stats_accumulate(img_ptr, code, seg_ptr, bd.own_hi - bd.own_lo, W, bd.own_lo, nb, _lib.ptr(acc),
                                                    _lib.ptr(iacc), st))
    comm.all_reduce(acc, 'sum')
    comm.all_reduce(iacc, 'sum')
    var = None
    if bits & 2:
        var = eng.buf('tb_var', (nb, 3), torch.float64)
        meanf = eng.buf('tb_meanf', (nb, 3), torch.float32)
        var.zero_()
        for i, b in enumerate(res.local):
            bd, img_ptr, code, seg_ptr = rows(i, b)
            _lib.check(lib.isb_segment_stats_deviation(img_ptr, code, seg_ptr, bd.own_hi - bd.own_lo, W, nb, _lib.ptr(acc), _lib.ptr(iacc),
                                                       _lib.ptr(meanf), _lib.ptr(var), st))
        comm.all_reduce(var, 'sum')
    _lib.check(lib.isb_segment_stats_finish(nb, bits, _lib.ptr(acc), _lib.ptr(var), _lib.ptr(iacc), _lib.ptr(feat), int(feat.shape[1]),
                                            int(col0), _lib.ptr(centres), None, st))


def _raw_rows(res, i, lo, hi, itemsize, what):
    """device pointer to the raw image rows [lo, hi) of local band i; ValueError when the band did not keep them"""
    bd = res.bands[res.local[i]]
    if lo < bd.up_lo or hi > bd.up_hi:
        raise ValueError('the band keeps the raw rows %d:%d, %s needs %d:%d (slic_tiled raw_margin)' % (bd.up_lo, bd.up_hi, what, lo, hi))
    return res.d_raw[i].data_ptr() + (lo - bd.up_lo) * res.shape[1] * 3 * itemsize


def color_stats_tiled(res, image_dtype, channels, flags, comm=None, eng=None, feat=None, col0=0):
    """colour statistics + centroids of the banded image over ``res.d_seg``: every band accumulates its owned rows, the
    accumulators are summed over the GPUs, every GPU finishes the same [nb, 3*len(flags)] table"""
    eng = eng or get_engine()
    comm = comm or default_comm()
    if channels != 3:
        raise ValueError('the colour statistics need a 3-channel image')
    code = _lib.dtype_code(np.dtype(image_dtype))
    itemsize = np.dtype(image_dtype).itemsize
    nb = int(res.nb_bound)
    if feat is None:
        feat = eng.buf('feat', (nb, max(flag_bits(flags)[1], 1)), eng.torch.float64)
    centres = eng.buf('centres', (nb, 2), eng.torch.float64)

    def source(i):
        bd = res.bands[res.local[i]]
        return _raw_rows(res, i, bd.own_lo, bd.own_hi, itemsize, 'the colour statistics'), code

    _stats_banded(res, source, flags, feat, col0, centres, comm, eng)
    res.d_feat, res.d_centres = feat, centres
    return feat, centres


def gradient_rows(bd, H):
    """the rows [lo, hi) whose np.gradient gives the owned rows of band ``bd`` their whole-image values: one more row on each side
    that is not an image border (there the gradient is one-sided, as it is for the whole image)"""
    return max(bd.own_lo - 1, 0), min(bd.own_hi + 1, H)


def color_group_tiled(res, image_dtype, key, flags, comm=None, eng=None, feat=None, col0=0, centres=None):
    """the statistics ``flags`` (mean / std / energy / meanGrad) of one colour group of ``native_feature_layout`` -- the image, or
    its conversion when ``key`` ends in '_<space>' of DICT_CONVERT_COLOR_FROM_RGB -- over ``res.d_seg`` into feat[:, col0:], the
    centroids into ``centres`` when given.  A band converts its owned rows (plus the gradient's one row on each interior side)
    into an f64 buffer of its own; ``meanGrad`` is the mean of ``isb_gradient_sum_2d`` of those rows (f32 for an f32 image that
    is not converted, as on the single-image path), of which only the owned rows are accumulated."""
    from .color import DICT_CONVERT_COLOR_FROM_RGB
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    H, W = res.shape
    st = _lib.stream_ptr()
    space = key.split('_')[-1]
    convert = space in DICT_CONVERT_COLOR_FROM_RGB
    grad = 'meanGrad' in flags
    native = [f for f in ('mean', 'std', 'energy') if f in flags]
    code, itemsize = _lib.dtype_code(np.dtype(image_dtype)), np.dtype(image_dtype).itemsize
    srcs = []       # per local band: (pointer to rows [lo, hi), dtype code, item size, lo, hi)
    for i, b in enumerate(res.local):
        bd = res.bands[b]
        lo, hi = gradient_rows(bd, H) if grad else (bd.own_lo, bd.own_hi)
        ptr = _raw_rows(res, i, lo, hi, itemsize, 'the colour group %r' % key)
        if convert:
            conv = eng.buf('tb%d_conv' % i, (hi - lo, W, 3), torch.float64)
            _lib.check(lib.isb_color_convert(C.c_void_p(ptr), code, C.c_longlong((hi - lo) * W), eng.COLOR_SPACES[space], _lib.ptr(conv), st))
            srcs.append((conv.data_ptr(), _lib.dtype_code(np.dtype(np.float64)), 8, lo, hi))
        else:
            srcs.append((ptr, code, itemsize, lo, hi))

    def owned(i, ptr, isz, lo):
        return ptr + (res.bands[res.local[i]].own_lo - lo) * W * 3 * isz

    col = col0
    if native:
        _stats_banded(res, lambda i: (owned(i, srcs[i][0], srcs[i][2], srcs[i][3]), srcs[i][1]), native, feat, col, centres, comm, eng)
        centres = None
        col += 3 * len(native)
    if grad:
        f32 = srcs[0][1] == _lib.dtype_code(np.dtype(np.float32))
        gdtype, gcode, gsize = (torch.float32, srcs[0][1], 4) if f32 else (torch.float64, _lib.dtype_code(np.dtype(np.float64)), 8)

        def gradient(i):
            ptr, c, _, lo, hi = srcs[i]
            out = eng.buf('tb_grad', (hi - lo, W, 3), gdtype)
            _lib.check(lib.isb_gradient_sum_2d(C.c_void_p(ptr), c, hi - lo, W, 3, _lib.ptr(out), st))
            return owned(i, out.data_ptr(), gsize, lo), gcode

        _stats_banded(res, gradient, ('mean', ), feat, col, centres, comm, eng)
    return feat


LM_ROW_MARGIN = 616     # rows of the Leung-Malik descriptor's footprint: sigma-150 background (radius 600) + half a 33 x 33 kernel


def texture_stats_tiled(res, image_dtype, flags, bank_type='normal', comm=None, eng=None, feat=None, col0=0):
    """Leung-Malik texture statistics (reference descriptors.py:1041-1106) of the banded image over ``res.d_seg``: every band runs
    the background subtraction and the filter-bank contraction on its rows + ``LM_ROW_MARGIN`` rows of halo (``slic_tiled`` must
    have been called with ``raw_margin=LM_ROW_MARGIN``) and accumulates the sums of the rows it owns; the accumulators -- the
    per-superpixel sums and the per-battery response norms of the WHOLE image -- are summed over the GPUs, every GPU finishes
    the same [nb, n_batteries * 3 * len(flags)] block of ``feat``"""
    from .texture import _device_bank, background_kernel
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    H, W = res.shape
    code = _lib.dtype_code(np.dtype(image_dtype))
    itemsize = np.dtype(image_dtype).itemsize
    nb = int(res.nb_bound)
    st = _lib.stream_ptr()
    bits, cols = flag_bits(flags)
    _, d_w, NP, orient, n_batt = _device_bank(bank_type)
    w_bg, radius, mix = background_kernel()
    d_wbg = eng.const_device(w_bg, 'lm_bg_w')
    acc = eng.buf('tb_lm_acc', (int(lib.isb_lm_acc_doubles(nb, n_batt)),), torch.float64)
    counts = eng.buf('tb_lm_counts', (nb,), torch.int32)
    acc.zero_()
    counts.zero_()
    for i, b in enumerate(res.local):
        bd = res.bands[b]
        lo, hi = max(bd.own_lo - LM_ROW_MARGIN, 0), min(bd.own_hi + LM_ROW_MARGIN, H)
        if lo < bd.up_lo or hi > bd.up_hi:
            raise ValueError('the band keeps the raw rows %d:%d, the texture descriptor needs %d:%d (slic_tiled raw_margin)'
                             % (bd.up_lo, bd.up_hi, lo, hi))
        img_ptr = C.c_void_p(res.d_raw[i].data_ptr() + (lo - bd.up_lo) * W * 3 * itemsize)
        seg_ptr = C.c_void_p(res.d_seg.data_ptr() + lo * W * 4)
        wsb = lib.isb_lm_workspace_bytes(hi - lo, W, nb, n_batt)
        ws = eng.buf('ws_lm', (wsb,), torch.uint8)
        _lib.check(lib.isb_lm_texture_accumulate(img_ptr, code, seg_ptr, hi - lo, W, bd.own_lo - lo, bd.own_hi - lo, nb, _lib.ptr(d_wbg), radius,
                                                 mix.ctypes.data_as(C.POINTER(C.c_double)), _lib.ptr(d_w), NP, orient, n_batt,
                                                 _lib.ptr(acc), _lib.ptr(counts), _lib.ptr(ws), C.c_size_t(wsb), st))
    comm.all_reduce(acc, 'sum')
    comm.all_reduce(counts, 'sum')
    ncol = n_batt * cols
    if feat is None:
        feat = eng.buf('feat_lm', (nb, ncol), torch.float64)
    _lib.check(lib.isb_lm_texture_finish(nb, n_batt, bits, _lib.ptr(acc), _lib.ptr(counts), _lib.ptr(feat), int(feat.shape[1]), int(col0), st))
    return feat


def texture_gradient_tiled(res, image_dtype, bank_type='normal', comm=None, eng=None, feat=None, col0=0, stride=3):
    """``meanGrad`` of every Leung-Malik battery of the banded image over ``res.d_seg``: battery b's three columns go to
    feat[:, col0 + b * stride:].  The route of ``texture.device_lm_materialised`` split at the response norm: every band subtracts
    the background of its rows + ``LM_ROW_MARGIN + 1`` rows of halo (``slic_tiled`` must have kept them, see
    :func:`banded_raw_margin`); then per battery every band computes its responses and the sum of their squares over its owned rows
    (``isb_lm_battery_partial``), the ranks exchange those sums and add them in band order -- the same bits on every rank and in
    every run --, and every band scales its owned rows +- 1 with that norm (``isb_lm_battery_scale``), takes their gradient and
    accumulates the owned rows."""
    from .descriptors import MAX_SIGNAL_RESPONSE
    from .texture import BACKGROUND_SIGMA, _device_batteries, background_kernel
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    H, W = res.shape
    st = _lib.stream_ptr()
    code, itemsize = _lib.dtype_code(np.dtype(image_dtype)), np.dtype(image_dtype).itemsize
    f64 = _lib.dtype_code(np.dtype(np.float64))
    margin = LM_ROW_MARGIN + 1
    w_half, radius = gaussian_half_kernel(BACKGROUND_SIGMA)
    d_w = eng.const_device(w_half, 'lm_bg_half')
    _, _, mix = background_kernel()
    slabs = []      # per local band: (slab rows [lo, hi), its background-subtracted planar copy, its responses)
    for i, b in enumerate(res.local):
        bd = res.bands[b]
        lo, hi = max(bd.own_lo - margin, 0), min(bd.own_hi + margin, H)
        ptr = _raw_rows(res, i, lo, hi, itemsize, 'the texture meanGrad')
        planar = eng.buf('tb%d_lmm_planar' % i, (3, hi - lo, W), torch.float64)
        tmp, smooth = (eng.buf(name, (3, hi - lo, W), torch.float64) for name in ('lmm_tmp', 'lmm_smooth'))
        _lib.check(lib.isb_lm_background(C.c_void_p(ptr), code, hi - lo, W, _lib.ptr(d_w), radius, mix.ctypes.data_as(C.POINTER(C.c_double)),
                                         _lib.ptr(planar), _lib.ptr(tmp), _lib.ptr(smooth), st))
        slabs.append((lo, hi, planar, eng.buf('tb%d_lmm_resp' % i, (3, hi - lo, W), torch.float64)))
    n_bands = len(res.bands)
    sums = eng.buf('tb_lmm_sumsq', (n_bands + 1, ), torch.float64)     # one slot per band, then their total
    wsb = lib.isb_lm_battery_workspace_bytes()
    ws = eng.buf('ws_lmm', (wsb, ), torch.uint8)
    for bt, d_k in enumerate(_device_batteries(eng, bank_type)):
        nk, kh, kw = (int(v) for v in d_k.shape)
        sums.zero_()
        for i, b in enumerate(res.local):
            bd, (lo, hi, planar, resp) = res.bands[b], slabs[i]
            _lib.check(lib.isb_lm_battery_partial(_lib.ptr(planar), hi - lo, W, _lib.ptr(d_k), nk, kh, kw, C.c_double(MAX_SIGNAL_RESPONSE),
                                                  bd.own_lo - lo, bd.own_hi - lo, _lib.ptr(resp), C.c_void_p(sums.data_ptr() + 8 * b),
                                                  _lib.ptr(ws), C.c_size_t(wsb), st))
        comm.all_reduce(sums, 'sum')    # an all-gather: every slot has one writer, the other ranks add +0
        for b in range(n_bands):
            _combine(lib, sums.data_ptr() + 8 * n_bands, sums.data_ptr() + 8 * b, 1, OP_SUM_F64)

        def gradient(i):
            bd, (lo, hi, planar, resp) = res.bands[res.local[i]], slabs[i]
            g_lo, g_hi = gradient_rows(bd, H)
            scaled = eng.buf('tb_lmm_out', (g_hi - g_lo, W, 3), torch.float64)
            _lib.check(lib.isb_lm_battery_scale(_lib.ptr(resp), hi - lo, W, g_lo - lo, g_hi - lo, C.c_double(MAX_SIGNAL_RESPONSE),
                                                C.c_void_p(sums.data_ptr() + 8 * n_bands), _lib.ptr(scaled), st))
            grad = eng.buf('tb_grad', (g_hi - g_lo, W, 3), torch.float64)
            _lib.check(lib.isb_gradient_sum_2d(_lib.ptr(scaled), f64, g_hi - g_lo, W, 3, _lib.ptr(grad), st))
            return grad.data_ptr() + (bd.own_lo - g_lo) * W * 3 * 8, f64

        _stats_banded(res, gradient, ('mean', ), feat, col0 + bt * stride, None, comm, eng)
    return feat


def banded_raw_margin(layout):
    """raw rows a band keeps above and below its owned ones (``slic_tiled(raw_margin=...)``) for the feature groups of ``layout``
    (``native_feature_layout``): none beyond the blur's for colour groups, whose gradient needs one row that the blur radius
    already covers; the Leung-Malik footprint ``LM_ROW_MARGIN`` for a texture group, one row more when it asks for ``meanGrad``
    (the gradient of the responses one row beyond the owned ones)"""
    texture = [flags for key, flags, _, _ in layout if key.startswith('tLM')]
    if not texture:
        return 0
    return LM_ROW_MARGIN + (1 if any('meanGrad' in flags for flags in texture) else 0)


def features_tiled(res, image_dtype, channels, layout, ncol, comm=None, eng=None):
    """the [nb, ncol] feature table of ``native_feature_layout`` over the banded image (``res.d_feat``) + the centroids, which come
    from the first statistics of a colour group (or from a pass over the image when there is none).  ``layout`` may hold any group
    of RESIDENT_FEATURE_GROUPS with any statistic but 'median' (``descriptors.flags_are_banded``)."""
    eng = eng or get_engine()
    torch = eng.torch
    nb = int(res.nb_bound)
    feat = eng.buf('feat', (nb, max(ncol, 1)), torch.float64)
    centres = None
    for key, flags, col0, n in layout:
        if key.startswith('color'):
            if centres is None and flags:
                centres = eng.buf('centres', (nb, 2), torch.float64)
                color_group_tiled(res, image_dtype, key, flags, comm=comm, eng=eng, feat=feat, col0=col0, centres=centres)
            else:
                color_group_tiled(res, image_dtype, key, flags, comm=comm, eng=eng, feat=feat, col0=col0)
            continue
        bank = 'short' if key.endswith('_short') else 'normal'
        if 'meanGrad' not in flags:
            texture_stats_tiled(res, image_dtype, flags, bank, comm=comm, eng=eng, feat=feat, col0=col0)
            continue
        # battery-major columns: the fused kernel's mean / std / energy, then the gradient mean of the materialised responses
        native = [f for f in ('mean', 'std', 'energy') if f in flags]
        n_batt, per_battery = n // (3 * len(flags)), 3 * len(flags)
        if native:
            part = texture_stats_tiled(res, image_dtype, native, bank, comm=comm, eng=eng)
            block = feat[:, col0:col0 + n].view(nb, n_batt, per_battery)
            block[:, :, :3 * len(native)].copy_(part[:nb, :n_batt * 3 * len(native)].reshape(nb, n_batt, 3 * len(native)))
        texture_gradient_tiled(res, image_dtype, bank, comm=comm, eng=eng, feat=feat, col0=col0 + 3 * len(native), stride=per_battery)
    if centres is None:
        _, centres = color_stats_tiled(res, image_dtype, channels, (), comm=comm, eng=eng, feat=eng.buf('feat_none', (nb, 1), torch.float64))
    res.d_feat, res.d_centres = feat, centres
    return feat, centres




def banded_edge_vectors(res, image_dtype, edge_type, comm=None, eng=None):
    """the vectors of ``graph_cuts.device_edge_vectors`` for the banded image, the same on every rank: 'features' standardises the
    replicated feature table ``res.d_feat``; 'color' takes the image's maximum as the bands' maxima merged over the ranks, scales the
    owned rows of every band by it (``Engine.unit_scaled_image``'s rule) and sums their mean colours over the ranks.  None for the
    edge types that need no vectors."""
    from .graph_cuts import device_edge_vectors
    eng = eng or get_engine()
    comm = comm or default_comm()
    if edge_type != 'color':
        return device_edge_vectors(eng, edge_type, None, res.d_seg, int(res.nb_bound), res.d_feat, res.d_n_labels)
    if int(res.d_raw[0].shape[-1]) != 3:
        raise ValueError("gc_edge_type 'color' needs an RGB image [H, W, 3]")
    torch, lib = eng.torch, eng.lib
    W = res.shape[1]
    code, itemsize = _lib.dtype_code(np.dtype(image_dtype)), np.dtype(image_dtype).itemsize
    f64 = _lib.dtype_code(np.dtype(np.float64))
    mm = eng.buf('tb_edge_minmax', (4,), torch.float64)
    mm_b = eng.buf('tb_edge_minmax_b', (4,), torch.float64)
    for i, b in enumerate(res.local):
        bd = res.bands[b]
        ptr = _raw_rows(res, i, bd.own_lo, bd.own_hi, itemsize, "gc_edge_type 'color'")
        _band_extrema(lib, ptr, code, (bd.own_hi - bd.own_lo) * W * 3, mm, mm_b, first=i == 0)
    _rank_extrema(comm, mm)

    def scaled(i):
        bd = res.bands[res.local[i]]
        out = eng.buf('tb_edge_img', (bd.own_hi - bd.own_lo, W, 3), torch.float64)
        _lib.check(lib.isb_image_unit_scale(C.c_void_p(_raw_rows(res, i, bd.own_lo, bd.own_hi, itemsize, "gc_edge_type 'color'")), code,
                                            C.c_longlong(out.numel()), _lib.ptr(mm), _lib.ptr(out), _lib.stream_ptr()))
        return out.data_ptr(), f64

    vec = eng.buf('edge_vec', (int(res.nb_bound), 3), torch.float64)
    _stats_banded(res, scaled, ('mean', ), vec, 0, None, comm, eng)
    return vec


def _admit(dict_features):
    """(layout, ncol, raw margin) of a feature dictionary the banded path takes; NotImplementedError for any other, before any
    device work"""
    from .descriptors import flags_are_banded, native_feature_layout
    layout, ncol = native_feature_layout(dict_features)
    if not layout or not flags_are_banded(dict_features):
        raise NotImplementedError('the banded path computes mean / std / energy / meanGrad of the colour, colour-space and Leung-Malik '
                                  'groups; a median does not decompose over row bands (got %r)' % (dict_features, ))
    return layout, ncol, banded_raw_margin(layout)


def _prepare_image(image, layout, sp_size, sp_regul):
    """(host image in a device dtype, n_segments, compactness) with the single-image pipelines' argument errors"""
    from .descriptors import _check_gradient_size
    from .superpixels import _as_rgb_like, _supported_dtype, slic_params
    image = _supported_dtype(_as_rgb_like(np.asarray(image)))
    H, W = int(image.shape[0]), int(image.shape[1])
    _check_gradient_size((H, W), [flags for _, flags, _, _ in layout])
    n_seg, compact = slic_params((H, W), sp_size, sp_regul)
    if n_seg < 1:
        raise ValueError('superpixel size %r is larger than the image %r' % (sp_size, tuple(image.shape)))
    return image, n_seg, compact


def _banded_segment(eng, shape, comm, bands_per_rank, front, gc_regul, gc_edge_type, want_soft, gather_segm, edge_vectors=None):
    """the tail the banded pipelines share, for an image [H, W] cut into row bands or a volume [D, H, W] cut into z-slabs:
    ``front(force_whole)`` -> (res, d_proba) runs the banded SLIC (``defer_check``), the feature table and the class probabilities;
    then the soft segmentation of the owned rows (slices), the graph cut on the replicated superpixel graph (4-connected in 2-D,
    6-connected in 3-D: :func:`~.graph_cuts.device_graphcut`), the LUT gather of the owned rows and one download.  Orphan pixels
    beyond the halo redo the front on the whole image, an edge table that was too small redoes the cut.  ``edge_vectors(res)`` gives
    the per-superpixel vectors of a 'color' / 'features' cut (:func:`banded_edge_vectors`).  Returns (segm,
    segm_soft or None, (lo, hi)) on the host, the rows (slices) [lo, hi) of this rank."""
    from . import graph_cuts
    torch = eng.torch
    force_whole, redo_front = False, True
    while True:
        if redo_front:
            res, d_proba = front(force_whole)
            d_vec = edge_vectors(res) if edge_vectors is not None else None
            redo_front = False
        lo, hi = res.bands[res.local[0]].own_lo, res.bands[res.local[-1]].own_hi
        soft = eng.early_soft(res.d_seg[lo:hi], d_proba) if want_soft else None
        cap = edge_capacity(res.nb_bound, ndim=len(shape))
        d_labels, d_n_edges = graph_cuts.device_graphcut(eng, res.d_seg, res.d_centres, res.nb_bound, d_proba, gc_regul, gc_edge_type,
                                                         res.d_n_labels, cap, edge_vectors=d_vec)
        # 5) LUT gather of the owned rows
        d_full = eng.buf('segm', tuple(shape), torch.int32) if gather_segm else None
        d_segm, _ = eng.gather(res.d_seg[lo:hi], d_labels, out_i=d_full[lo:hi] if gather_segm else None)
        if gather_segm and comm.world > 1:
            for r in range(comm.world):
                blo = res.bands[r * bands_per_rank].own_lo
                bhi = res.bands[(r + 1) * bands_per_rank - 1].own_hi
                comm.broadcast(d_full[blo:bhi], r)
        (h_segm, n_edges, err), done = eng.download((d_full if gather_segm else d_segm, d_n_edges, res.d_err))
        done.synchronize()
        if soft is not None:
            soft[1].synchronize()
        if int(err[0]) != 0 and not force_whole:
            # orphan pixels beyond the halo (see slic_tiled): same answer on every rank, so every rank takes this branch
            logging.warning('banded SLIC met orphan pixels beyond the halo, redoing the sweeps on the whole image on every GPU')
            force_whole = redo_front = True
            continue
        if edges_fit(n_edges[0], cap):
            break
    return h_segm.numpy(), (soft[0].numpy() if want_soft else None), (lo, hi)


def _segment_banded_image(image, n_seg, compact, layout, ncol, margin, model, gc_regul, gc_edge_type, comm, bands_per_rank, want_soft,
                          gather_segm):
    """the banded image pipeline after the argument checks (:func:`_admit`, :func:`_prepare_image`): banded SLIC, the feature table
    of ``layout``, the class probabilities of ``model`` (a model of :func:`~.pipelines._device_proba`, on the replicated table of
    every rank) and the tail of :func:`_banded_segment`"""
    from .pipelines import _device_proba
    eng = get_engine()
    comm = comm or default_comm()

    def front(force_whole):
        res = slic_tiled(image, n_seg, compact, sigma=1.0, comm=comm, bands_per_rank=bands_per_rank, eng=eng, defer_check=True,
                         force_whole=force_whole, raw_margin=margin)
        features_tiled(res, image.dtype, int(image.shape[2]), layout, ncol, comm=comm, eng=eng)
        return res, _device_proba(eng, model, res.d_feat, res.d_n_labels, res.nb_bound)

    return _banded_segment(eng, image.shape[:2], comm, bands_per_rank, front, gc_regul, gc_edge_type, want_soft, gather_segm,
                           lambda res: banded_edge_vectors(res, image.dtype, gc_edge_type, comm, eng))


def pipe_color2d_slic_features_model_graphcut_tiled(image, nb_classes, dict_features=None, sp_size=30, sp_regul=0.2, use_scaler=True,
                                                    gc_regul=1., gc_edge_type='model', max_iter=99, comm=None, bands_per_rank=1,
                                                    want_soft=True, gather_segm=False, estim_model='GMM', pca_coef=None):
    """ ``pipe_color2d_slic_features_model_graphcut`` (reference pipelines.py:46-110) for one image banded over the GPUs of
    ``comm``.  Every rank passes the same host image and gets the rows it owns.  The features may be any group of
    RESIDENT_FEATURE_GROUPS with mean / std / energy / meanGrad (not median); the class model is fitted on the GPU on the
    replicated feature table, every ``estim_model`` variant and ``pca_coef`` that ``graph_cuts.device_gmm_applicable`` takes.

    :return tuple: (segm [rows, W] int32, segm_soft [rows, W, K] float64 or None, (row_lo, row_hi)); with ``gather_segm``
        ``segm`` is the whole [H, W] map on every rank (``segm_soft`` stays banded: it is 8*K bytes per pixel)
    """
    from . import graph_cuts
    from .pipelines import _fit_model
    graph_cuts.check_edge_type(gc_edge_type)
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    dict_features = {'color': ['mean']} if dict_features is None else dict_features
    layout, ncol, margin = _admit(dict_features)
    if not graph_cuts.device_gmm_applicable(ncol, nb_classes, estim_model, pca_coef):
        raise NotImplementedError('the banded path fits the class model on the GPU, which does not take estim_model=%r, pca_coef=%r with '
                                  '%d features and %d classes' % (estim_model, pca_coef, ncol, nb_classes))
    # the default 'GMM' gives (GMM, sqrt(max_iter) restarts, max_iter): the mixture fit the banded path has always made
    model = _fit_model(int(nb_classes), use_scaler, estim_model, pca_coef, max_iter)
    image, n_seg, compact = _prepare_image(image, layout, sp_size, sp_regul)
    return _segment_banded_image(image, n_seg, compact, layout, ncol, margin, model, gc_regul, gc_edge_type, comm, bands_per_rank, want_soft,
                                 gather_segm)


def segment_color2d_slic_features_model_graphcut_tiled(image, model_pipeline, dict_features, sp_size=30, sp_regul=0.2, gc_regul=1.,
                                                       gc_edge_type='model', comm=None, bands_per_rank=1, want_soft=True,
                                                       gather_segm=False):
    """ ``segment_color2d_slic_features_model_graphcut`` (reference pipelines.py:160-241) for one image banded over the GPUs of
    ``comm``: a caller-fitted model -- typically the group model of ``estim_model_classes_group`` -- applied to an image too large
    for one pass.  A model that ``class_models.compile_model`` takes (and whose feature count matches the banded table) is evaluated
    on the device on every rank; any other model's ``predict_proba`` runs on the host of every rank, on the same replicated feature
    table, and its probabilities are uploaded.  The labels are mapped through the model's ``classes_``.

    :return tuple: (segm [rows, W], segm_soft [rows, W, K] float64 or None, (row_lo, row_hi)) as
        :func:`pipe_color2d_slic_features_model_graphcut_tiled`
    """
    from .graph_cuts import check_edge_type
    from .pipelines import _device_model
    check_edge_type(gc_edge_type)
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    layout, ncol, margin = _admit(dict_features)
    image, n_seg, compact = _prepare_image(image, layout, sp_size, sp_regul)
    model = _device_model(model_pipeline.predict_proba, ncol)
    segm, soft, rows = _segment_banded_image(image, n_seg, compact, layout, ncol, margin, model, gc_regul, gc_edge_type, comm, bands_per_rank,
                                             want_soft, gather_segm)
    classes = getattr(model_pipeline, 'classes_', None)
    if classes is not None:
        segm = np.asarray(classes)[segm]
    return segm, soft, rows


# ---------------------------------------------------------------------------------------------------------------------
# z-slab mode: ONE gray volume cut into slabs of slices, one slab (or a few) per GPU
# ---------------------------------------------------------------------------------------------------------------------

def slab_plan(shape, n_segments, spacing, n_slabs, sigma=1.0):
    """the z-slabs of the 3-D SLIC of a volume ``shape`` = (D, H, W): (:func:`plan_bands` along z with a halo of ``2 step_z + 1``
    slices and the z-blur's radius, seeds (z, y, x), steps (z, y, x), the half kernels (weights, radius) of the z, y, x blurs)"""
    halves = [gaussian_half_kernel(s) for s in np.array([sigma, sigma, sigma], dtype=np.float64) / np.asarray(spacing, dtype=np.float64)]
    seeds, steps = slic_seed_grid3d(tuple(shape), n_segments)
    return plan_bands(shape[0], n_slabs, 2 * steps[0] + 1, halves[0][1]), seeds, steps, halves


def slic3d_tiled(volume, n_segments, compactness, spacing, sigma=1.0, max_iter=10, comm=None, bands_per_rank=1, eng=None,
                 min_size_factor=0.5, max_size_factor=3, enforce_connectivity=True, defer_check=False, force_whole=False):
    """ 3-D SLIC of one host gray volume over the z-slabs of ``comm`` (every rank passes the same volume; it uploads only the raw
    slices of its slabs).  The slabs are :func:`plan_bands` along z: owned slices, k-means slab = owned +- ``2 step_z + 1``, raw
    slab = k-means slab +- the z-blur radius.  Per sweep the slabs exchange 5 int64 words per cluster (``isb_slic3d_slab_*``).

    :param ndarray volume: [D, H, W] host array, dtype uint8 / uint16 / float32 / float64
    :return TiledSuperpixels: ``d_seg`` = the whole label volume on this GPU (identical on every rank), ``d_raw[i]`` = the raw slices
        ``bands[local[i]].raw_lo:raw_hi`` still on the device for the statistics
    :param bool defer_check: do not synchronise to read the orphan counter ``res.d_err``; the caller reads it with its own
        results and calls again with ``force_whole=True`` when it is not zero
    :param bool force_whole: skip the banded sweeps, every rank runs them on the whole volume (the fallback)
    """
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    volume = np.asarray(volume)
    D, H, W = (int(v) for v in volume.shape)
    code = _lib.dtype_code(volume.dtype)
    st = _lib.stream_ptr()
    spacing = np.ascontiguousarray(spacing, dtype=np.float64)
    bands, seeds, (tz, ty, tx), halves = slab_plan((D, H, W), n_segments, spacing, comm.world * int(bands_per_rank), sigma)
    d_w = [eng.const_device(w, 'slic3d_w%d' % axis) for axis, (w, _) in enumerate(halves)]
    n_seeds = len(seeds)
    halo = 2 * tz + 1
    local = list(range(comm.rank * bands_per_rank, (comm.rank + 1) * bands_per_rank))
    owner = lambda b: b // bands_per_rank  # noqa: E731

    res = TiledSuperpixels()
    res.shape, res.bands, res.local = (D, H, W), bands, local
    res.d_raw = [eng.to_device(volume[bands[b].raw_lo:bands[b].raw_hi], 'ts%d_raw' % i) for i, b in enumerate(local)]
    d_seeds = eng.const_device(seeds, 'seeds3d')
    xchg = [eng.buf('ts%d_xchg' % i, (5 * n_seeds + 1,), torch.int64) for i in range(len(local))]
    err = eng.buf('ts_err', (1,), torch.int64)
    err.zero_()

    # 1) blur of every raw slab, slab descriptors
    descs, keep = [], []
    for i, b in enumerate([] if force_whole else local):
        bd = bands[b]
        S, slab = bd.raw_hi - bd.raw_lo, bd.km_hi - bd.km_lo
        tmp = eng.buf('ts_tmp', (S, H, W), torch.float64)
        prep = eng.buf('ts%d_vol' % i, (S, H, W), torch.float64)
        _lib.check(lib.isb_slic3d_prepare_slab(_lib.ptr(res.d_raw[i]), code, S, H, W, bd.raw_lo, D, _lib.ptr(d_w[0]), halves[0][1],
                                               _lib.ptr(d_w[1]), halves[1][1], _lib.ptr(d_w[2]), halves[2][1], C.c_double(1.0 / compactness),
                                               _lib.ptr(tmp), _lib.ptr(prep), st))
        labels = eng.buf('ts%d_labels' % i, (slab, H, W), torch.int32)
        wsb = lib.isb_slic3d_kmeans_workspace_bytes(slab, H, W, n_seeds)
        ws = eng.buf('ts%d_ws' % i, (wsb,), torch.uint8)
        d = _lib.Slic3dSlab(depth=D, height=H, width=W, z_off=bd.km_lo, slab_slices=slab, own_lo=bd.own_lo, own_hi=bd.own_hi, halo=halo,
                            n_seeds=n_seeds, step_z=tz, step_y=ty, step_x=tx, step=float(max(tz, ty, tx)), spacing=(C.c_double * 3)(*spacing),
                            vol_slab=prep.data_ptr() + (bd.km_lo - bd.raw_lo) * H * W * 8, seeds_zyx=d_seeds.data_ptr(),
                            labels_slab=labels.data_ptr(), ws=ws.data_ptr(), ws_bytes=wsb)
        descs.append(d)
        keep.append((prep, labels, ws))
        _lib.check(lib.isb_slic3d_slab_begin(C.byref(d), st))

    # 2) the sweeps: assign, sum the owned clusters, merge, take the merged centres
    for _ in range(0 if force_whole else int(max_iter)):
        for i, d in enumerate(descs):
            _lib.check(lib.isb_slic3d_slab_assign(C.byref(d), st))
            _lib.check(lib.isb_slic3d_slab_update(C.byref(d), _lib.ptr(xchg[i]), st))
            if i > 0:
                _combine(lib, xchg[0].data_ptr(), xchg[i].data_ptr(), 5 * n_seeds + 1, OP_SUM_I64)
        comm.all_reduce(xchg[0], 'sum')
        _combine(lib, err.data_ptr(), xchg[0].data_ptr() + 8 * 5 * n_seeds, 1, OP_SUM_I64)
        for d in descs:
            _lib.check(lib.isb_slic3d_slab_import(C.byref(d), _lib.ptr(xchg[0]), st))

    # 3) the whole k-means label volume on every GPU
    full = eng.buf('ts_full', (D, H, W), torch.int32)
    res.d_err = err
    if not force_whole:
        for i, b in enumerate(local):
            bd = bands[b]
            full[bd.own_lo:bd.own_hi].copy_(keep[i][1][bd.own_lo - bd.km_lo:bd.own_hi - bd.km_lo])
        if comm.world > 1:
            for bd in bands:
                comm.broadcast(full[bd.own_lo:bd.own_hi], owner(bd.index))
    if force_whole or (not defer_check and int(eng.to_host(err)[0]) != 0):
        # some voxel kept the label of a cluster centred beyond the halo (no window covers it): the slab sums are not trustworthy,
        # every rank redoes the sweeps on the whole volume on its own GPU
        logging.warning('slic3d_tiled: orphan voxels beyond the halo, redoing the sweeps on the whole volume on every GPU')
        res.fell_back = True
        km, _ = eng.slic3d(eng.to_device(volume, 'volume'), n_segments, compactness, spacing, sigma=sigma, max_iter=max_iter,
                           enforce_connectivity=False)
        full.copy_(km)
    if not enforce_connectivity:
        res.d_seg = full
        return res
    res.d_seg, res.d_n_labels = eng.enforce_connectivity3d(full, n_segments, min_size_factor, max_size_factor)
    res.nb_bound = eng.slic_label_bound(D * H * W, 1, n_segments, min_size_factor)
    return res


def gray_stats_tiled(res, volume_dtype, flags, comm=None, eng=None):
    """statistics ``flags`` (of mean / std / energy, in that order) of the slab-cut volume over ``res.d_seg``, one column each, as
    :meth:`~.engine.Engine.gray_table` lays them out: every slab accumulates its owned slices, the accumulators are summed over the
    GPUs between the calls, every GPU finishes the same [nb, len(flags)] table"""
    eng = eng or get_engine()
    torch, lib = eng.torch, eng.lib
    comm = comm or default_comm()
    D, H, W = res.shape
    code, itemsize = _lib.dtype_code(np.dtype(volume_dtype)), np.dtype(volume_dtype).itemsize
    nb = int(res.nb_bound)
    st = _lib.stream_ptr()
    bits, _ = flag_bits(flags)
    acc = eng.buf('ts_gacc', (nb, 2), torch.float64)
    cnt = eng.buf('ts_gcnt', (nb,), torch.int64)
    acc.zero_()
    cnt.zero_()

    def slices(i):
        bd = res.bands[res.local[i]]
        n = (bd.own_hi - bd.own_lo) * H * W
        return (C.c_void_p(res.d_raw[i].data_ptr() + (bd.own_lo - bd.raw_lo) * H * W * itemsize),
                C.c_void_p(res.d_seg.data_ptr() + bd.own_lo * H * W * 4), C.c_longlong(n))

    for i in range(len(res.local)):
        img, seg, n = slices(i)
        _lib.check(lib.isb_gray_stats_accumulate(img, code, seg, n, nb, _lib.ptr(acc), _lib.ptr(cnt), st))
    comm.all_reduce(acc, 'sum')
    comm.all_reduce(cnt, 'sum')
    var = None
    if bits & 2:
        var = eng.buf('ts_gvar', (nb,), torch.float64)
        meanf = eng.buf('ts_gmeanf', (nb,), torch.float32)
        var.zero_()
        for i in range(len(res.local)):
            img, seg, n = slices(i)
            _lib.check(lib.isb_gray_stats_deviation(img, code, seg, n, nb, _lib.ptr(acc), _lib.ptr(cnt), _lib.ptr(meanf), _lib.ptr(var), st))
        comm.all_reduce(var, 'sum')
    feat = eng.buf('feat3d', (nb, len(flags)), torch.float64)
    _lib.check(lib.isb_gray_stats_finish(nb, bits, _lib.ptr(acc), _lib.ptr(var), _lib.ptr(cnt), _lib.ptr(feat), len(flags), 0, st))
    res.d_feat = feat
    return feat


def _admit_volume(dict_features):
    """the statistic columns of a feature dictionary the slab path takes (``color`` groups' mean / std / energy, in
    compute_selected_features_gray3d's order); NotImplementedError for any other, before any device work"""
    from .pipelines import _volume_flags
    flags = _volume_flags(dict_features)
    if flags is None or 'median' in flags:
        raise NotImplementedError('the slab path computes mean / std / energy of "color" groups of a gray volume; a median does not '
                                  'decompose over slabs, texture and meanGrad have no volume form (got %r)' % (dict_features, ))
    return flags


def _prepare_volume(volume, sp_size, sp_regul, spacing, n_slabs):
    """(host volume in a device dtype, n_segments, compactness) with the volume pipelines' argument errors"""
    from .superpixels import _supported_dtype, slic3d_params
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    volume = np.asarray(volume)
    if volume.ndim != 3:
        raise ValueError('expected a gray volume [D, H, W], got shape %r' % (volume.shape, ))
    plan_bands(volume.shape[0], n_slabs, 1, 0)          # ValueError: more slabs than slices
    n_seg, compact = slic3d_params(volume.shape, sp_size, sp_regul, spacing)
    if n_seg < 1 or compact < 1:
        raise ValueError('superpixel size %r / compactness do not fit the volume %r' % (sp_size, volume.shape))
    return _supported_dtype(volume), n_seg, compact


def _segment_banded_volume(volume, n_seg, compact, spacing, flags, model, gc_regul, comm, bands_per_rank, want_soft, gather_segm):
    """the slab volume pipeline after the argument checks (:func:`_admit_volume`, :func:`_prepare_volume`): slab SLIC, the statistics
    table and norm_features (the device StandardScaler), the class probabilities of ``model`` (a model of
    :func:`~.pipelines._device_proba`, on the replicated standardised table of every rank) and the tail of :func:`_banded_segment`"""
    from .pipelines import _device_proba
    eng = get_engine()

    def front(force_whole):
        res = slic3d_tiled(volume, n_seg, compact, spacing, sigma=1.0, comm=comm, bands_per_rank=bands_per_rank, eng=eng, defer_check=True,
                           force_whole=force_whole)
        d_x = eng.standard_scaler(gray_stats_tiled(res, volume.dtype, flags, comm=comm, eng=eng), res.d_n_labels)[0]
        return res, _device_proba(eng, model, d_x, res.d_n_labels, res.nb_bound)

    return _banded_segment(eng, volume.shape, comm, bands_per_rank, front, gc_regul, 'model', want_soft, gather_segm)


def pipe_gray3d_slic_features_model_graphcut_tiled(volume, nb_classes, dict_features, spacing=(12, 1, 1), sp_size=15, sp_regul=0.2,
                                                   gc_regul=0.1, use_scaler=True, max_iter=99, comm=None, bands_per_rank=1, want_soft=True,
                                                   gather_segm=False):
    """ ``pipe_gray3d_slic_features_model_graphcut`` (reference pipelines.py:382-431) for one gray volume cut into z-slabs over the
    GPUs of ``comm``.  Every rank passes the same host volume and gets the slices it owns.  The features are mean / std / energy of
    ``color`` groups (not median); the class model (GaussianMixture, ``sqrt(max_iter)`` restarts) is fitted on the GPU on the
    replicated, standardised feature table, as :func:`~.pipelines.segment_resident_volume` does.

    :return tuple: (segm [slices, H, W] int32, segm_soft [slices, H, W, K] float64 or None, (z_lo, z_hi)); with ``gather_segm``
        ``segm`` is the whole [D, H, W] volume on every rank (``segm_soft`` stays sliced: it is 8*K bytes per voxel)
    """
    from . import graph_cuts
    from .pipelines import _fit_model
    flags = _admit_volume(dict_features)
    if not graph_cuts.device_gmm_applicable(len(flags), nb_classes):
        raise NotImplementedError('the slab path fits the class model on the GPU, which does not take %d classes' % nb_classes)
    model = _fit_model(int(nb_classes), use_scaler, 'GMM', None, max_iter)
    comm = comm or default_comm()
    volume, n_seg, compact = _prepare_volume(volume, sp_size, sp_regul, spacing, comm.world * int(bands_per_rank))
    return _segment_banded_volume(volume, n_seg, compact, spacing, flags, model, gc_regul, comm, bands_per_rank, want_soft, gather_segm)


def segment_gray3d_slic_features_model_graphcut_tiled(volume, model_pipeline, dict_features, spacing=(12, 1, 1), sp_size=15, sp_regul=0.2,
                                                      gc_regul=0.1, comm=None, bands_per_rank=1, want_soft=True, gather_segm=False):
    """ the volume pipeline with a caller-fitted model (fitted on standardised supervoxel features, as the reference's
    pipe_gray3d_slic_features_model_graphcut feeds its model) for one gray volume cut into z-slabs over the GPUs of ``comm``.  A
    model that ``class_models.compile_model`` takes is evaluated on the device on every rank; any other model's ``predict_proba``
    runs on the host of every rank, on the same replicated table.  The labels are mapped through the model's ``classes_``.

    :return tuple: (segm [slices, H, W], segm_soft [slices, H, W, K] float64 or None, (z_lo, z_hi)) as
        :func:`pipe_gray3d_slic_features_model_graphcut_tiled`
    """
    from .pipelines import _device_model
    flags = _admit_volume(dict_features)
    comm = comm or default_comm()
    volume, n_seg, compact = _prepare_volume(volume, sp_size, sp_regul, spacing, comm.world * int(bands_per_rank))
    model = _device_model(model_pipeline.predict_proba, len(flags))
    segm, soft, rows = _segment_banded_volume(volume, n_seg, compact, spacing, flags, model, gc_regul, comm, bands_per_rank, want_soft,
                                              gather_segm)
    classes = getattr(model_pipeline, 'classes_', None)
    if classes is not None:
        segm = np.asarray(classes)[segm]
    return segm, soft, rows
