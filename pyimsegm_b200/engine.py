"""
Device-resident driver of the SLIC -> descriptors -> GraphCut hot path.

Everything here is plumbing: torch tensors are used purely as device-memory containers and every computation is
a call into ``libimsegm_b200.so`` through the C-ABI (``include/imsegm_b200.h``).  No torch op touches the data
path.  The numpy-facing modules (``superpixels``, ``descriptors``, ``graph_cuts``, ``pipelines``) are thin
wrappers over this class.
"""
import ctypes as C

import numpy as np

from . import _lib

FLAG_BITS = {'mean': 1, 'std': 2, 'energy': 4}
#: edge_type -> (metric, spatial) of isb_gc_energies; only 'model' and 'spatial' are spatially normalised
#: (reference graph_cuts.py:646)
EDGE_MODES = {'': (0, 0), 'model': (1, 1), 'model_lT': (1, 0), 'model_l1': (2, 0), 'model_l2': (3, 0), 'spatial': (0, 1)}
#: edge_type -> metric of isb_gc_vector_edge_weights, which compares per-label vectors (the mean colours: L1, the standardised
#: features: L2) into weights that isb_gc_energies then takes as given (:data:`EDGE_GIVEN`)
VECTOR_EDGE_METRICS = {'color': 2, 'features': 3}
EDGE_GIVEN = (4, 0)

#: initial capacity of a device edge table, in edges per node (per upper bound of the label count) of a 2-D label map, twice
#: that for a volume; grown x4 whenever a table overflows.  The device then reports cap + 1 edges and writes no row past cap.
EDGE_CAP_PER_NODE = 8


def edge_capacity(nb, ndim=2):
    """rows of a new device edge table for ``nb`` nodes of a ``ndim``-D label map"""
    return max(64, int(EDGE_CAP_PER_NODE * (ndim - 1) * int(nb)))


def edges_fit(n_edges, cap):
    """whether a table of ``cap`` rows held all ``n_edges`` the device counted; if not, the capacity grows x4 and the caller redoes
    the work that filled it"""
    global EDGE_CAP_PER_NODE
    if int(n_edges) <= cap:
        return True
    EDGE_CAP_PER_NODE *= 4
    return False


def flag_bits(flags):
    """statistic names -> (bit mask of the C-ABI, columns per 3-channel source: three per statistic)"""
    bits = 0
    for f in flags:
        bits |= FLAG_BITS[f]
    return bits, 3 * bin(bits).count('1')


def gaussian_half_kernel(sigma, truncate=4.0):
    """half of scipy.ndimage's normalised 1-D Gaussian: [w0, w1 .. wr], radius r = int(truncate * sigma + 0.5); ``sigma <= 0``
    gives the identity [1] of radius 0 (no blur, as scipy skips such an axis)"""
    if sigma <= 0:
        return np.ones(1), 0
    radius = int(truncate * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    phi = phi / phi.sum()
    return np.ascontiguousarray(phi[radius:], dtype=np.float64), radius


def regular_grid_steps(shape, n_points):
    """(start, step) per axis of skimage.util.regular_grid for an array of ``shape`` and ``n_points`` seeds"""
    shape = np.asarray(shape)
    ndim = len(shape)
    rank = np.argsort(np.argsort(shape))
    dims = np.sort(shape)
    space = float(np.prod(shape))
    if space <= n_points:
        return [(0, 1)] * ndim
    steps = np.full(ndim, (space / n_points) ** (1.0 / ndim))
    if (dims < steps).any():
        for d in range(ndim):
            steps[d] = dims[d]
            space = float(np.prod(dims[d + 1:]))
            steps[d + 1:] = (space / n_points) ** (1.0 / (ndim - d - 1))
            if (dims >= steps).all():
                break
    starts = (steps // 2).astype(int)
    steps = np.round(steps).astype(int)
    pairs = [(int(a), int(b)) for a, b in zip(starts, steps)]
    return [pairs[i] for i in rank]


def slic_seed_grid(H, W, n_segments):
    (_, _), (sy, ty), (sx, tx) = regular_grid_steps((1, H, W), n_segments)
    gy, gx = np.meshgrid(np.arange(sy, H, ty), np.arange(sx, W, tx), indexing='ij')
    seeds = np.stack([gy.ravel(), gx.ravel()], axis=1).astype(np.float64)
    return np.ascontiguousarray(seeds), int(ty), int(tx)


def slic_seed_grid3d(shape, n_segments):
    """seeds (z, y, x) of skimage's regular grid over a volume and the per-axis steps"""
    (sz, tz), (sy, ty), (sx, tx) = regular_grid_steps(shape, n_segments)
    gz, gy, gx = np.meshgrid(np.arange(sz, shape[0], tz), np.arange(sy, shape[1], ty), np.arange(sx, shape[2], tx), indexing='ij')
    seeds = np.stack([gz.ravel(), gy.ravel(), gx.ravel()], axis=1).astype(np.float64)
    return np.ascontiguousarray(seeds), (int(tz), int(ty), int(tx))


class Engine(object):
    """owns the device buffers for one image shape at a time and sequences the C-ABI calls on the current stream"""

    def __init__(self, device=None):
        self.torch = _lib.require_cuda()
        self.lib = _lib.lib()
        self.device = self.torch.device('cuda', self.torch.cuda.current_device() if device is None else device)
        self._bufs = {}
        self._consts = {}
        self._stage = None
        self._side = None
        #: CUDA graphs captured on this engine's buffers: once there is one, an outgrown buffer is retired instead of freed
        self.graphs_captured = 0
        self._retired = []

    # -- memory helpers ------------------------------------------------------------------------------------------
    def buf(self, name, shape, dtype):
        """cached device buffer (grown on demand, never shrunk)"""
        torch = self.torch
        if torch.cuda.current_device() != self.device.index:
            # the C-ABI calls launch on the CURRENT device's stream: an engine must only be driven with its own device current
            raise RuntimeError('Engine of cuda:%d used while cuda:%d is the current device' % (self.device.index, torch.cuda.current_device()))
        shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        n = int(np.prod(shape)) if shape else 1
        cur = self._bufs.get(name)
        if cur is None or cur.dtype != dtype or cur.numel() < n:
            if cur is not None and self.graphs_captured:
                # a captured CUDA graph may hold the address of the old block: keep it alive instead of returning it to the allocator
                self._retired.append(cur)
            cur = torch.empty(max(n, 1), dtype=dtype, device=self.device)
            self._bufs[name] = cur
        return cur[:n].view(shape)

    #: host arrays at least this large that are NOT page-locked go through the staged upload below
    STAGE_MIN_BYTES = 4 << 20
    STAGE_CHUNK = 4 << 20
    STAGE_SLOTS = 8

    def to_device(self, arr, name=None):
        """host ndarray -> device tensor through the current stream (pinned sources copy asynchronously; large pageable sources
        are staged, see :meth:`_staged_upload`)"""
        torch = self.torch
        arr = np.ascontiguousarray(arr)
        src = torch.from_numpy(arr)
        if name is None:
            return src.to(self.device, non_blocking=True)
        dst = self.buf(name, arr.shape, src.dtype)
        if arr.nbytes >= self.STAGE_MIN_BYTES and not src.is_pinned():
            self._staged_upload(dst, arr)
        else:
            dst.copy_(src, non_blocking=True)
        return dst

    def _staged_upload(self, dst, arr):
        """upload of a large PAGEABLE array (what a caller of the numpy API normally holds): the driver would bounce it through
        its own small staging buffer at a fraction of the PCIe rate.  Here worker threads copy 4 MB chunks into a ring of pinned
        buffers (numpy releases the GIL while copying) and every chunk is sent by an asynchronous DMA as soon as it is complete, so
        the host copies overlap the transfers."""
        torch = self.torch
        if self._stage is None:
            from concurrent.futures import ThreadPoolExecutor
            slots = [torch.empty(self.STAGE_CHUNK, dtype=torch.uint8, pin_memory=True) for _ in range(self.STAGE_SLOTS)]
            self._stage = (slots, [t.numpy() for t in slots], [torch.cuda.Event() for _ in slots], [False] * len(slots),
                           ThreadPoolExecutor(self.STAGE_SLOTS))
        slots, views, events, used, pool = self._stage
        src = arr.reshape(-1).view(np.uint8)
        out = dst.view(torch.uint8).reshape(-1)
        n, ch = src.shape[0], self.STAGE_CHUNK
        nchunks = (n + ch - 1) // ch

        def fill(slot, lo, hi):
            np.copyto(views[slot][:hi - lo], src[lo:hi])

        def submit(c):
            slot = c % len(slots)
            if used[slot]:
                events[slot].synchronize()      # the DMA that last read this slot has finished
            return pool.submit(fill, slot, c * ch, min(n, (c + 1) * ch))

        futs = {c: submit(c) for c in range(min(len(slots), nchunks))}
        for c in range(nchunks):
            slot = c % len(slots)
            futs.pop(c).result()
            lo, hi = c * ch, min(n, (c + 1) * ch)
            out[lo:hi].copy_(slots[slot][:hi - lo], non_blocking=True)
            events[slot].record()
            used[slot] = True
            if c + len(slots) < nchunks:
                futs[c + len(slots)] = submit(c + len(slots))

    def const_device(self, arr, name, digest=None):
        """small host array that rarely changes between calls (seed grid, pairwise table, filter taps): every distinct content gets
        its OWN device tensor, uploaded once and never overwritten -- no copy in steady state, and a captured CUDA graph that read
        one of them keeps reading the right values whatever other configurations run in between.  ``digest``: a content digest the
        caller already holds (it must change whenever ``arr`` does), which saves hashing a large table on every call"""
        import hashlib
        arr = np.ascontiguousarray(arr)
        key = (name, arr.shape, arr.dtype.str, digest if digest is not None else hashlib.blake2b(arr.tobytes(), digest_size=16).digest())
        hit = self._consts.get(key)
        if hit is not None:
            return hit
        if self.torch.cuda.is_current_stream_capturing():
            raise RuntimeError('constant %r is new while a CUDA graph is being captured' % name)
        dst = self.torch.from_numpy(arr).to(self.device)
        self._consts[key] = dst
        return dst

    def pinned_empty(self, shape, dtype):
        """pinned host tensor (torch's caching host allocator recycles the blocks once the result is dropped)"""
        return self.torch.empty(tuple(shape), dtype=dtype, pin_memory=True)

    def download(self, tensors):
        """enqueue D2H copies of device tensors into pinned host tensors on the current stream and record one event after them:
        returns (host tensors, event); the host tensors hold the data once the event has completed"""
        hosts = []
        for t in tensors:
            h = self.pinned_empty(t.shape, t.dtype)
            h.copy_(t, non_blocking=True)
            hosts.append(h)
        done = self.torch.cuda.Event()
        done.record()
        return hosts, done

    def to_host(self, t):
        (out, ), done = self.download((t, ))
        done.synchronize()
        return out.numpy()

    def side_stream(self):
        """a second CUDA stream of this engine (copies that may overlap the kernels of the main stream)"""
        if self._side is None:
            self._side = self.torch.cuda.Stream(device=self.device)
        return self._side

    def early_soft(self, d_seg, d_proba):
        """segm_soft = proba[seg] needs only the class probabilities: gather it and start its (large) download on the side stream,
        so that both overlap what the current stream does next (building and cutting the graph).  Returns (pinned host tensor,
        event); nothing may overwrite ``d_seg`` or ``d_proba`` before the event has completed"""
        torch = self.torch
        side = self.side_stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            _, d_soft = self.gather(d_seg, None, d_proba)
            (host, ), done = self.download((d_soft, ))
        return host, done

    def edge_table(self, build, nb, ndim=2):
        """``build(cap) -> (edges, n_edges device int32[1], ...)`` with a table of :func:`edge_capacity` rows, redone larger until
        the table holds every edge (one synchronisation per attempt): returns (E, what ``build`` returned)"""
        while True:
            cap = edge_capacity(nb, ndim)
            out = build(cap)
            E = int(self.to_host(out[1])[0])
            if edges_fit(E, cap):
                return E, out

    def _ck(self, rc):
        _lib.check(rc)

    # -- (i) SLIC -------------------------------------------------------------------------------------------------
    def slic(self, d_img, n_segments, compactness, sigma=1.0, max_iter=10, enforce_connectivity=True,
             min_size_factor=0.5, max_size_factor=3, slic_zero=False, rescale=True):
        """device SLIC on a [H,W,C] device tensor; returns (labels int32 [H,W] device, n_labels device int32[1] or None)"""
        torch, lib = self.torch, self.lib
        H, W = int(d_img.shape[0]), int(d_img.shape[1])
        Cn = 1 if d_img.dim() == 2 else int(d_img.shape[2])
        code = _lib.dtype_code(d_img.dtype)
        st = _lib.stream_ptr()
        lab = self.buf('lab', (3, H, W), torch.float64)
        mm = self.buf('minmax', (4,), torch.float64)
        w_half, radius = gaussian_half_kernel(sigma)
        self._ck(lib.isb_slic_prepare(_lib.ptr(d_img), code, H, W, Cn, w_half.ctypes.data_as(C.POINTER(C.c_double)), radius,
                                      C.c_double(1.0 / compactness), int(bool(rescale)), _lib.ptr(lab), _lib.ptr(mm), st))
        seeds, ty, tx = slic_seed_grid(H, W, n_segments)
        n_seeds = len(seeds)
        step = float(max(1, ty, tx))
        d_seeds = self.const_device(seeds, 'seeds')
        wsb = lib.isb_slic_kmeans_workspace_bytes(H, W, n_seeds, ty, tx)
        ws = self.buf('ws_kmeans', (wsb,), torch.uint8)
        km = self.buf('labels_km', (H, W), torch.int32)
        self._ck(lib.isb_slic_kmeans(_lib.ptr(lab), H, W, _lib.ptr(d_seeds), n_seeds, ty, tx, C.c_double(step), int(max_iter),
                                     int(bool(slic_zero)), _lib.ptr(km), None, _lib.ptr(ws), C.c_size_t(wsb), st))
        if not enforce_connectivity:
            return km, None
        return self.enforce_connectivity(km, n_segments, min_size_factor, max_size_factor)

    def enforce_connectivity(self, d_km, n_segments, min_size_factor=0.5, max_size_factor=3):
        """connectivity pass over a k-means label map [H,W] (device): returns (labels int32 [H,W] device, n_labels device int32[1])"""
        torch, lib = self.torch, self.lib
        H, W = int(d_km.shape[0]), int(d_km.shape[1])
        segment_size = 1 * H * W / n_segments
        min_size, max_size = int(min_size_factor * segment_size), int(max_size_factor * segment_size)
        cwsb = lib.isb_connectivity_workspace_bytes(H, W)
        cws = self.buf('ws_conn', (cwsb,), torch.uint8)
        out = self.buf('labels', (H, W), torch.int32)
        n_labels = self.buf('n_labels', (1,), torch.int32)
        self._ck(lib.isb_enforce_connectivity(_lib.ptr(d_km), H, W, min_size, max_size, _lib.ptr(out), _lib.ptr(n_labels),
                                              _lib.ptr(cws), C.c_size_t(cwsb), _lib.stream_ptr()))
        return out, n_labels

    def slic3d(self, d_vol, n_segments, compactness, spacing=(1, 1, 1), sigma=1.0, max_iter=10, enforce_connectivity=True,
               min_size_factor=0.5, max_size_factor=3):
        """device SLIC of a single-channel volume [D, H, W] (csrc/slic3d.cu); returns (labels int32 [D,H,W], n_labels or None)"""
        torch, lib = self.torch, self.lib
        D, H, W = (int(v) for v in d_vol.shape)
        code = _lib.dtype_code(d_vol.dtype)
        st = _lib.stream_ptr()
        spacing = np.ascontiguousarray(spacing, dtype=np.float64)
        halves = []
        for axis, sig in enumerate(np.array([sigma, sigma, sigma], dtype=np.float64) / spacing):
            w_half, radius = gaussian_half_kernel(sig)
            halves.append((self.to_device(w_half, 'slic3d_w%d' % axis), radius))
        tmp = self.buf('slic3d_tmp', (D, H, W), torch.float64)
        scaled = self.buf('slic3d_vol', (D, H, W), torch.float64)
        self._ck(lib.isb_slic3d_prepare(_lib.ptr(d_vol), code, D, H, W, _lib.ptr(halves[0][0]), halves[0][1], _lib.ptr(halves[1][0]),
                                        halves[1][1], _lib.ptr(halves[2][0]), halves[2][1], C.c_double(1.0 / compactness), _lib.ptr(tmp),
                                        _lib.ptr(scaled), st))
        seeds, steps = slic_seed_grid3d((D, H, W), n_segments)
        n_seeds = len(seeds)
        d_seeds = self.to_device(seeds, 'seeds3d')
        wsb = lib.isb_slic3d_kmeans_workspace_bytes(D, H, W, n_seeds)
        ws = self.buf('ws_kmeans3d', (wsb,), torch.uint8)
        km = self.buf('labels_km3d', (D, H, W), torch.int32)
        self._ck(lib.isb_slic3d_kmeans(_lib.ptr(scaled), D, H, W, _lib.ptr(d_seeds), n_seeds, steps[0], steps[1], steps[2],
                                       C.c_double(float(max(steps))), spacing.ctypes.data_as(C.POINTER(C.c_double)), int(max_iter),
                                       _lib.ptr(km), _lib.ptr(ws), C.c_size_t(wsb), st))
        if not enforce_connectivity:
            return km, None
        return self.enforce_connectivity3d(km, n_segments, min_size_factor, max_size_factor)

    def enforce_connectivity3d(self, d_km, n_segments, min_size_factor=0.5, max_size_factor=3):
        """connectivity pass over a k-means label volume [D,H,W] (device): returns (labels int32 [D,H,W], n_labels device int32[1])"""
        torch, lib = self.torch, self.lib
        D, H, W = (int(v) for v in d_km.shape)
        st = _lib.stream_ptr()
        segment_size = D * H * W / n_segments
        min_size, max_size = int(min_size_factor * segment_size), int(max_size_factor * segment_size)
        cwsb = lib.isb_connectivity3d_workspace_bytes(D, H, W, max(max_size, 1))
        cws = self.buf('ws_conn3d', (cwsb,), torch.uint8)
        out = self.buf('labels3d', (D, H, W), torch.int32)
        n_labels = self.buf('n_labels', (1,), torch.int32)
        self._ck(lib.isb_enforce_connectivity3d(_lib.ptr(d_km), D, H, W, min_size, max_size, _lib.ptr(out), _lib.ptr(n_labels), _lib.ptr(cws),
                                                C.c_size_t(cwsb), st))
        return out, n_labels

    def graph3d(self, d_seg, nb, cap):
        """6-connected label pairs and centres (z, y, x) of a device label volume: (edges [cap,2], n_edges dev, cap, centres [nb,3])"""
        torch, lib = self.torch, self.lib
        D, H, W = (int(v) for v in d_seg.shape)
        wsb = lib.isb_adjacency_workspace_bytes(int(nb), int(cap))
        ws = self.buf('ws_adj', (wsb,), torch.uint8)
        edges = self.buf('edges', (cap, 2), torch.int32)
        n_edges = self.buf('n_edges', (1,), torch.int32)
        self._ck(lib.isb_adjacency_edges_3d(_lib.ptr(d_seg), D, H, W, int(nb), _lib.ptr(edges), int(cap), _lib.ptr(n_edges), _lib.ptr(ws),
                                            C.c_size_t(wsb), _lib.stream_ptr()))
        centres = self.buf('centres3d', (nb, 3), torch.float64)
        cws = self.buf('ws_centres3d', (4 * int(nb),), torch.int64)
        self._ck(lib.isb_centroids_3d(_lib.ptr(d_seg), D, H, W, int(nb), _lib.ptr(centres), _lib.ptr(cws), C.c_size_t(32 * int(nb)),
                                      _lib.stream_ptr()))
        return edges, n_edges, cap, centres

    def gray_table(self, d_vol, d_seg, nb, flags):
        """the statistics ``flags`` (in :data:`~.descriptors.NAMES_FEATURE_FLAGS` order, any of mean / std / energy / median) of a
        gray volume [D,H,W] over its label volume, one column each, as compute_image3d_gray_statistic lays them out: feat [nb, len(flags)]
        f64 (cached buffer; NaN voxels count as 0, NaN and -0 results are written as +0)"""
        torch, lib = self.torch, self.lib
        D, H, W = (int(v) for v in d_vol.shape)
        code = _lib.dtype_code(d_vol.dtype)
        st = _lib.stream_ptr()
        feat = self.buf('feat3d', (nb, len(flags)), torch.float64)
        native = [f for f in flags if f in FLAG_BITS]
        if native:
            wsb = lib.isb_gray_stats_workspace_bytes(int(nb))
            ws = self.buf('ws_gray', (wsb,), torch.uint8)
            self._ck(lib.isb_gray_stats(_lib.ptr(d_vol), code, _lib.ptr(d_seg), C.c_longlong(D * H * W), int(nb), flag_bits(native)[0],
                                        _lib.ptr(feat), len(flags), 0, _lib.ptr(ws), C.c_size_t(wsb), st))
        if 'median' in flags:
            wsb = lib.isb_segment_median_workspace_bytes(C.c_longlong(D * H * W), int(nb))
            ws = self.buf('ws_median', (wsb,), torch.uint8)
            self._ck(lib.isb_segment_median_2d(_lib.ptr(d_vol), code, _lib.ptr(d_seg), D * H, W, 1, int(nb), _lib.ptr(feat), len(flags),
                                               list(flags).index('median'), _lib.ptr(ws), C.c_size_t(wsb), st))
        return feat

    def standard_scaler(self, d_feat, d_n=None, names=('feat_scaled', 'scaler_params')):
        """sklearn StandardScaler().fit_transform of device features [N, D] bit for bit (isb_standard_scaler; the real row count
        from the device ``d_n``): returns (scaled [N, D], mean_ | scale_ [2 D]) device tensors, in the cached buffers ``names``"""
        torch = self.torch
        N, D = int(d_feat.shape[0]), int(d_feat.shape[1])
        out = self.buf(names[0], (N, D), torch.float64)
        params = self.buf(names[1], (2 * D, ), torch.float64)
        self._ck(self.lib.isb_standard_scaler(_lib.ptr(d_feat), N, D, int(d_feat.stride(0)), _lib.ptr(d_n), _lib.ptr(params), _lib.ptr(out),
                                              _lib.stream_ptr()))
        return out, params

    def slic_label_bound(self, H, W, n_segments, min_size_factor=0.5):
        """upper bound on the number of labels after connectivity enforcement (each kept label has >= min_size px)"""
        min_size = max(1, int(min_size_factor * (H * W / n_segments)))
        return H * W // min_size + 1

    # -- (ii) descriptors -----------------------------------------------------------------------------------------
    def segment_stats(self, d_img, d_seg, nb, flags, feat=None, col0=0, want_centres=False, want_counts=False):
        """colour statistics (+centroids) of a [H,W,3] device image over labels [H,W] int32 in [0, nb)"""
        torch, lib = self.torch, self.lib
        H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
        code = 0 if d_img is None else _lib.dtype_code(d_img.dtype)
        bits, ncol = flag_bits(flags)
        if feat is None and ncol:
            feat = self.buf('feat', (nb, ncol), torch.float64)
        ld = int(feat.shape[1]) if feat is not None else 0
        centres = self.buf('centres', (nb, 2), torch.float64) if want_centres else None
        counts = self.buf('counts', (nb,), torch.int32) if want_counts else None
        wsb = lib.isb_segment_stats_workspace_bytes(nb)
        ws = self.buf('ws_stats', (wsb,), torch.uint8)
        self._ck(lib.isb_segment_stats_2d(_lib.ptr(d_img), code, _lib.ptr(d_seg), H, W, int(nb), bits, _lib.ptr(feat), ld, int(col0),
                                          _lib.ptr(centres), _lib.ptr(counts), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
        return feat, centres, counts

    #: isb_color_space codes of the ``color_<space>`` feature groups
    COLOR_SPACES = {'hsv': 0, 'luv': 1, 'lab': 2, 'hed': 3, 'xyz': 4}

    def color_convert(self, d_img, space):
        """a [H,W,3] device RGB image in ``space`` (pyimsegm_b200.color), f64 [H,W,3] in one cached buffer that the next conversion
        overwrites"""
        H, W = int(d_img.shape[0]), int(d_img.shape[1])
        out = self.buf('color_conv', (H, W, 3), self.torch.float64)
        self._ck(self.lib.isb_color_convert(_lib.ptr(d_img), _lib.dtype_code(d_img.dtype), C.c_longlong(H * W), self.COLOR_SPACES[space],
                                            _lib.ptr(out), _lib.stream_ptr()))
        return out

    def gradient_sum(self, d_img):
        """np.sum(np.gradient(np.nan_to_num(channel)), axis=0) of every channel of a [H,W,C] device image: f32 for an f32 image, f64
        otherwise (cached buffer)"""
        torch = self.torch
        H, W, Cn = (int(v) for v in d_img.shape)
        dtype = torch.float32 if d_img.dtype == torch.float32 else torch.float64
        out = self.buf('grad_' + str(dtype)[6:], (H, W, Cn), dtype)
        self._ck(self.lib.isb_gradient_sum_2d(_lib.ptr(d_img), _lib.dtype_code(d_img.dtype), H, W, Cn, _lib.ptr(out), _lib.stream_ptr()))
        return out

    def segment_median(self, d_img, d_seg, nb, feat, col0=0):
        """per-label median of every channel of a [H,W,C] device image (np.nan_to_num'd pixels) into feat[:nb, col0:col0 + C]"""
        torch, lib = self.torch, self.lib
        H, W, Cn = (int(v) for v in d_img.shape)
        wsb = lib.isb_segment_median_workspace_bytes(C.c_longlong(H * W), int(nb))
        ws = self.buf('ws_median', (wsb,), torch.uint8)
        self._ck(lib.isb_segment_median_2d(_lib.ptr(d_img), _lib.dtype_code(d_img.dtype), _lib.ptr(d_seg), H, W, Cn, int(nb), _lib.ptr(feat),
                                           int(feat.shape[1]), int(col0), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
        return feat

    def group_stats(self, d_src, d_seg, nb, flags, feat, col0, want_centres=False):
        """the statistics ``flags`` of one feature group over a [H,W,3] device source into feat[:, col0:], statistic-major in the
        order mean, std, energy, median, meanGrad and channel-minor, as compute_image2d_color_statistic lays them out.  With
        ``want_centres`` the first stats launch of the group also forms the centroids: returns them, or None when the group has no
        such launch"""
        native = [f for f in ('mean', 'std', 'energy') if f in flags]
        centres = None
        col = col0
        if native:
            _, centres, _ = self.segment_stats(d_src, d_seg, nb, native, feat=feat, col0=col, want_centres=want_centres)
            col += 3 * len(native)
        if 'median' in flags:
            self.segment_median(d_src, d_seg, nb, feat, col)
            col += 3
        if 'meanGrad' in flags:
            _, grad_centres, _ = self.segment_stats(self.gradient_sum(d_src), d_seg, nb, ('mean', ), feat=feat, col0=col,
                                                    want_centres=want_centres and centres is None)
            centres = grad_centres if centres is None else centres
        return centres

    # -- (iii) graph, energies, alpha-expansion ---------------------------------------------------------------------
    def adjacency(self, d_seg, nb, cap):
        """unique 4-connected label pairs; returns (edges int32 [cap,2] device, n_edges device int32[1], cap)"""
        torch, lib = self.torch, self.lib
        H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
        wsb = lib.isb_adjacency_workspace_bytes(int(nb), int(cap))
        ws = self.buf('ws_adj', (wsb,), torch.uint8)
        edges = self.buf('edges', (cap, 2), torch.int32)
        n_edges = self.buf('n_edges', (1,), torch.int32)
        self._ck(lib.isb_adjacency_edges(_lib.ptr(d_seg), H, W, int(nb), _lib.ptr(edges), int(cap), _lib.ptr(n_edges), _lib.ptr(ws),
                                         C.c_size_t(wsb), _lib.stream_ptr()))
        return edges, n_edges, cap

    def gc_energies(self, d_proba, d_edges, E, d_n_edges, d_centres, edge_mode, edge_cost, pairwise, d_n_nodes=None, edge_w=None):
        """isb_gc_energies; centres [N, 3] (z, y, x) of a label volume take its 3-D spatial mode, centres [N, 2] the 2-D one.
        :data:`EDGE_GIVEN` integerises the weights ``edge_w`` [>= E] (:meth:`vector_edge_weights`), which it then scales in place."""
        torch, lib = self.torch, self.lib
        if (tuple(edge_mode) == EDGE_GIVEN) != (edge_w is not None):
            raise ValueError('the given-weights mode %r takes the weights as edge_w, and only it does' % (EDGE_GIVEN, ))
        if edge_w is not None and (edge_w.dtype != torch.float64 or not edge_w.is_contiguous() or edge_w.numel() < max(int(E), 1)):
            raise ValueError('edge_w must be a contiguous float64 tensor of at least %d weights' % max(int(E), 1))
        spatial = int(edge_mode[1])
        if spatial and d_centres is not None and d_centres.dim() == 2 and int(d_centres.shape[1]) == 3:
            spatial = 3
        N, K = int(d_proba.shape[0]), int(d_proba.shape[1])
        d_pw = self.const_device(np.ascontiguousarray(pairwise, dtype=np.float64), 'pairwise')
        unary = self.buf('unary', (N, K), torch.float64)
        if edge_w is None:
            edge_w = self.buf('edge_w', (max(E, 1),), torch.float64)
        unary_i = self.buf('unary_i', (N, K), torch.int32)
        edge_wi = self.buf('edge_wi', (max(E, 1),), torch.int32)
        smooth_i = self.buf('smooth_i', (K, K), torch.int32)
        wsb = lib.isb_gc_energies_workspace_bytes(N, K, int(E))
        ws = self.buf('ws_energy', (wsb,), torch.uint8)
        self._ck(lib.isb_gc_energies(_lib.ptr(d_proba), N, _lib.ptr(d_n_nodes), K, _lib.ptr(d_edges), int(E), _lib.ptr(d_n_edges), _lib.ptr(d_centres),
                                     int(edge_mode[0]), spatial, C.c_double(edge_cost), _lib.ptr(d_pw), _lib.ptr(unary), _lib.ptr(edge_w),
                                     _lib.ptr(unary_i), _lib.ptr(edge_wi), _lib.ptr(smooth_i), _lib.ptr(ws), C.c_size_t(wsb),
                                     _lib.stream_ptr()))
        return unary, edge_w, unary_i, edge_wi, smooth_i

    def unit_scaled_image(self, d_img):
        """np.array(image, dtype=float), divided by 255 when np.max(image) > 1, of a device image: the image whose mean colours
        compute_edge_weights compares for 'color'.  The maximum is reduced on the device (isb_image_minmax, numpy's NaN rule) and
        never read back.  Returns an f64 cached buffer of the image's shape."""
        torch, lib = self.torch, self.lib
        n, code, st = C.c_longlong(int(d_img.numel())), _lib.dtype_code(d_img.dtype), _lib.stream_ptr()
        mm = self.buf('edge_minmax', (4,), torch.float64)
        out = self.buf('edge_img', tuple(d_img.shape), torch.float64)
        self._ck(lib.isb_image_minmax(_lib.ptr(d_img), code, n, _lib.ptr(mm), st))
        self._ck(lib.isb_image_unit_scale(_lib.ptr(d_img), code, n, _lib.ptr(mm), _lib.ptr(out), st))
        return out

    def vector_edge_weights(self, d_vec, d_edges, cap, d_n_edges, d_centres, metric):
        """isb_gc_vector_edge_weights of the per-label vectors ``d_vec`` [nb, D] over the edge table (``cap`` rows, device count
        ``d_n_edges``): returns the weights [cap] (cached buffer), which :meth:`gc_energies` takes as ``edge_w`` under
        :data:`EDGE_GIVEN`"""
        torch, lib = self.torch, self.lib
        nb, D = int(d_vec.shape[0]), int(d_vec.shape[1])
        edge_w = self.buf('edge_w_given', (max(int(cap), 1),), torch.float64)
        wsb = lib.isb_gc_energies_workspace_bytes(nb, 1, int(cap))
        ws = self.buf('ws_energy', (wsb,), torch.uint8)
        self._ck(lib.isb_gc_vector_edge_weights(_lib.ptr(d_vec), nb, D, int(d_vec.stride(0)), _lib.ptr(d_edges), int(cap), _lib.ptr(d_n_edges),
                                                _lib.ptr(d_centres), int(metric), _lib.ptr(edge_w), _lib.ptr(ws), C.c_size_t(wsb),
                                                _lib.stream_ptr()))
        return edge_w

    # -- supervised training data ----------------------------------------------------------------------------------
    def train_labels(self, d_seg, nb, d_annot, label_purity, d_n=None):
        """isb_superpixel_train_labels: the training label of every superpixel of ``d_seg`` [H, W] (labels below ``nb``) from the
        annotation ``d_annot`` [H, W] int32 (negative = unknown); returns int64 [nb] (cached buffer), -1 where no label is kept"""
        torch, lib = self.torch, self.lib
        H, W = int(d_seg.shape[0]), int(d_seg.shape[1])
        labels = self.buf('train_labels', (int(nb),), torch.int64)
        wsb = lib.isb_train_labels_workspace_bytes(H, W, int(nb))
        ws = self.buf('ws_train_labels', (max(wsb, 1),), torch.uint8)
        self._ck(lib.isb_superpixel_train_labels(_lib.ptr(d_seg), H, W, int(nb), _lib.ptr(d_n), _lib.ptr(d_annot), C.c_double(label_purity),
                                                 _lib.ptr(labels), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
        return labels

    def nan_free_table(self, d_feat, D, d_n=None):
        """the first ``D`` columns of ``d_feat`` [N, ld] f64 as a dense [N, D] copy with NaN -> 0 (``features[np.isnan(features)] = 0``
        of the pipelines), rows from the optional device count ``d_n`` on left unwritten: isb_class_transform without scaler or PCA"""
        N = int(d_feat.shape[0])
        out = self.buf('feat_nan_free', (N, int(D)), self.torch.float64)
        self._ck(self.lib.isb_class_transform(_lib.ptr(d_feat), N, int(d_feat.stride(0)), _lib.ptr(d_n), int(D), None, None, None, None, None,
                                              int(D), _lib.ptr(out), None, C.c_size_t(0), _lib.stream_ptr()))
        return out

    def unique_rows(self, d_feat, d_labels, D, d_n=None):
        """isb_unique_rows_rounded of the first ``D`` columns of ``d_feat`` [N, ld] f64 and their labels ``d_labels`` [N] int64: returns
        (rows [N, D] f64, labels [N] int64, count int64 [1]) cached buffers, the first ``count`` rows written; a count of -1 means the
        table held a NaN"""
        torch, lib = self.torch, self.lib
        N = int(d_feat.shape[0])
        rows = self.buf('unique_rows', (N, int(D)), torch.float64)
        labels = self.buf('unique_labels', (N,), torch.int64)
        count = self.buf('unique_count', (1,), torch.int64)
        wsb = lib.isb_unique_rows_workspace_bytes(N, int(D))
        ws = self.buf('ws_unique_rows', (max(wsb, 1),), torch.uint8)
        self._ck(lib.isb_unique_rows_rounded(_lib.ptr(d_feat), N, int(D), int(d_feat.stride(0)), _lib.ptr(d_n), _lib.ptr(d_labels),
                                             _lib.ptr(rows), _lib.ptr(labels), _lib.ptr(count), _lib.ptr(ws), C.c_size_t(wsb),
                                             _lib.stream_ptr()))
        return rows, labels, count

    def alpha_expansion(self, N, K, E, d_n_edges, d_edges, edge_wi, unary_i, smooth_i, n_iter=-1, init_labels=None,
                        d_n_nodes=None):
        torch, lib = self.torch, self.lib
        labels = self.buf('gc_labels', (N,), torch.int32)
        if init_labels is None:
            self._ck(lib.isb_fill_i32(_lib.ptr(labels), C.c_longlong(int(N)), 0, _lib.stream_ptr()))
        else:
            labels.copy_(init_labels)  # device-to-device memcpy of a caller-supplied labeling
        energy = self.buf('gc_energy', (1,), torch.int64)
        stats = self.buf('gc_stats', (8,), torch.int32)
        wsb = lib.isb_alpha_expansion_workspace_bytes(int(N), int(K), int(E))
        ws = self.buf('ws_gc', (wsb,), torch.uint8)
        self._ck(lib.isb_alpha_expansion(int(N), _lib.ptr(d_n_nodes), int(K), int(E), _lib.ptr(d_n_edges), _lib.ptr(d_edges), _lib.ptr(edge_wi),
                                         _lib.ptr(unary_i), _lib.ptr(smooth_i), int(n_iter), _lib.ptr(labels), _lib.ptr(energy),
                                         _lib.ptr(stats), _lib.ptr(ws), C.c_size_t(wsb), _lib.stream_ptr()))
        return labels, energy, stats

    #: isb_mixture_fit_predict kinds
    MIXTURE_KINDS = {'GMM': 0, 'BGM': 1}
    #: the params buffer of each kind: a captured CUDA graph holds the address of the one it writes, so a fit of the other kind
    #: (with a longer params vector) must not grow it
    _MIXTURE_PARAMS = {'GMM': 'gmm_params', 'BGM': 'mixture_params'}

    def mixture_fit_predict(self, d_feat, K, n_init, max_iter, use_scaler=True, seed=0, d_n=None, init_labels=None, tol=1e-3,
                            reg_covar=1e-6, kind='GMM'):
        """device class model of either kind ('GMM' = GaussianMixture, 'BGM' = BayesianGaussianMixture): returns
        (proba [N,K] device, params device vector; see isb_mixture_fit_predict)"""
        torch, lib = self.torch, self.lib
        code = self.MIXTURE_KINDS[kind]
        N, D = int(d_feat.shape[0]), int(d_feat.shape[1])
        proba = self.buf('proba', (N, K), torch.float64)
        params = self.buf(self._MIXTURE_PARAMS[kind], (lib.isb_mixture_fit_params_len(code, D, K),), torch.float64)
        wsb = lib.isb_mixture_fit_workspace_bytes(code, N, D, int(K), int(n_init))
        ws = self.buf('ws_gmm', (wsb,), torch.uint8)
        d_init = None
        if init_labels is not None:
            d_init = self.to_device(np.ascontiguousarray(init_labels, dtype=np.int32), 'gmm_init')
        self._ck(lib.isb_mixture_fit_predict(code, _lib.ptr(d_feat), N, D, int(d_feat.stride(0)), _lib.ptr(d_n), int(K), int(n_init),
                                             int(max_iter), C.c_double(tol), C.c_double(reg_covar), int(bool(use_scaler)),
                                             C.c_ulonglong(int(seed)), _lib.ptr(d_init), _lib.ptr(proba), _lib.ptr(params), _lib.ptr(ws),
                                             C.c_size_t(wsb), _lib.stream_ptr()))
        return proba, params

    def pca_fit_transform(self, d_feat, use_scaler, pca_coef, d_n=None):
        """scaler + PCA(pca_coef) fitted on features [N, D] (device; isb_pca_fit) and applied to them by isb_class_transform: returns
        (transformed [N, D'] device, params device vector, D').  A float ``pca_coef`` makes D' depend on the data: it is read back
        (4 bytes, one synchronisation); an int fixes it."""
        torch, lib = self.torch, self.lib
        N, D = int(d_feat.shape[0]), int(d_feat.shape[1])
        ld = int(d_feat.stride(0))
        params = self.buf('pca_params', (lib.isb_pca_params_len(D),), torch.float64)
        n_comp = self.buf('pca_n_comp', (1,), torch.int32)
        wsb = lib.isb_pca_workspace_bytes(N, D)
        ws = self.buf('ws_pca', (wsb,), torch.uint8)
        is_int = isinstance(pca_coef, (int, np.integer))
        st = _lib.stream_ptr()
        self._ck(lib.isb_pca_fit(_lib.ptr(d_feat), N, D, ld, _lib.ptr(d_n), int(bool(use_scaler)), C.c_double(0.0 if is_int else pca_coef),
                                 int(pca_coef) if is_int else 0, _lib.ptr(params), _lib.ptr(n_comp), _lib.ptr(ws), C.c_size_t(wsb), st))
        dims = int(pca_coef) if is_int else int(self.to_host(n_comp)[0])
        comp = params[3 * D:3 * D + dims * D]
        mproj = params[3 * D + D * D + 3 * D:3 * D + D * D + 3 * D + dims]
        x = self.buf('pca_x', (N, dims), torch.float64)
        twsb = lib.isb_class_transform_workspace_bytes(N, D, 1)
        tws = self.buf('ws_pca_transform', (twsb,), torch.uint8)
        self._ck(lib.isb_class_transform(_lib.ptr(d_feat), N, ld, _lib.ptr(d_n), D, _lib.ptr(params[:D]) if use_scaler else None,
                                         _lib.ptr(params[D:2 * D]) if use_scaler else None, _lib.ptr(comp), _lib.ptr(mproj), None, dims,
                                         _lib.ptr(x), _lib.ptr(tws), C.c_size_t(twsb), st))
        return x, params, dims

    def class_model_predict(self, d_feat, cm, d_n=None):
        """predict_proba of a compiled caller-fitted model (class_models.CompiledModel) on features [N, >= n_features_in] (device):
        returns proba [N, K] device, asynchronous; the model's tables are device constants keyed on its digest"""
        torch, lib = self.torch, self.lib
        N, ld = int(d_feat.shape[0]), int(d_feat.stride(0))
        t = {name: self.const_device(arr, 'cm_' + name, digest=cm.digest) for name, arr in cm.tables.items()}
        st = _lib.stream_ptr()
        x = self.buf('cm_x', (N, cm.n_dims), torch.float64)
        wsb = lib.isb_class_transform_workspace_bytes(N, cm.n_features_in, int('pca_comp' in t))
        ws = self.buf('ws_cm', (max(wsb, 1),), torch.uint8)
        self._ck(lib.isb_class_transform(_lib.ptr(d_feat), N, ld, _lib.ptr(d_n), cm.n_features_in, _lib.ptr(t.get('sc_mean')),
                                         _lib.ptr(t.get('sc_scale')), _lib.ptr(t.get('pca_comp')), _lib.ptr(t.get('pca_mean')),
                                         _lib.ptr(t.get('pca_scale')), cm.n_dims, _lib.ptr(x), _lib.ptr(ws), C.c_size_t(wsb), st))
        K = cm.n_classes
        proba = self.buf('proba', (N, K), torch.float64)
        if cm.kind == 'mixture':
            wsb = lib.isb_mixture_predict_workspace_bytes(N, cm.n_dims, K)
            ws = self.buf('ws_cm_predict', (max(wsb, 1),), torch.uint8)
            self._ck(lib.isb_mixture_predict_proba(_lib.ptr(x), N, _lib.ptr(d_n), cm.n_dims, K, _lib.ptr(t['prec_chol']), _lib.ptr(t['bvec']),
                                                   _lib.ptr(t['log_const']), _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb), st))
        elif cm.kind == 'knn':
            n_fit, k = len(cm.tables['y']), cm.params['n_neighbors']
            wsb = lib.isb_knn_predict_workspace_bytes(N, n_fit, k)
            ws = self.buf('ws_cm_predict', (max(wsb, 1),), torch.uint8)
            self._ck(lib.isb_knn_predict_proba(_lib.ptr(x), N, _lib.ptr(d_n), cm.n_dims, _lib.ptr(t['fit_x']), n_fit, _lib.ptr(t['y']), k, K,
                                               cm.params['weights'], _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb), st))
        elif cm.kind == 'linear':
            wsb = lib.isb_linear_predict_workspace_bytes(N, len(cm.tables['intercept']))
            ws = self.buf('ws_cm_predict', (max(wsb, 1),), torch.uint8)
            self._ck(lib.isb_linear_predict_proba(_lib.ptr(x), N, _lib.ptr(d_n), cm.n_dims, _lib.ptr(t['coef']), _lib.ptr(t['intercept']),
                                                  len(cm.tables['intercept']), _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb), st))
        else:
            n_trees, n_nodes = len(cm.tables['roots']), len(cm.tables['left'])
            wsb = lib.isb_forest_predict_workspace_bytes(N, n_trees)
            ws = self.buf('ws_cm_predict', (max(wsb, 1),), torch.uint8)
            self._ck(lib.isb_forest_predict_proba(_lib.ptr(x), N, _lib.ptr(d_n), cm.n_dims, n_trees, _lib.ptr(t['roots']), _lib.ptr(t['feature']),
                                                  _lib.ptr(t['threshold']), _lib.ptr(t['left']), _lib.ptr(t['right']), n_nodes,
                                                  _lib.ptr(t['value']), K, int(cm.average), _lib.ptr(proba), _lib.ptr(ws), C.c_size_t(wsb), st))
        return proba

    def gather(self, d_seg, lut_i=None, lut_p=None, out_i=None):
        """``lut_i[d_seg]`` (into ``out_i`` when given, a contiguous int32 tensor of the label map's shape) and ``lut_p[d_seg]`` of a
        contiguous label map [H,W] or label volume [D,H,W] (device, one launch): returns (segm or None, segm_soft [..., K] or None)"""
        torch, lib = self.torch, self.lib
        shape = tuple(int(v) for v in d_seg.shape)
        if lut_i is not None and out_i is None:
            out_i = self.buf('segm', shape, torch.int32)
        K = int(lut_p.shape[1]) if lut_p is not None else 0
        out_p = self.buf('segm_soft', shape + (K, ), torch.float64) if lut_p is not None else None
        self._ck(lib.isb_gather(_lib.ptr(d_seg), C.c_longlong(int(np.prod(shape))), _lib.ptr(lut_i), _lib.ptr(lut_p), K, _lib.ptr(out_i),
                                _lib.ptr(out_p), _lib.stream_ptr()))
        return out_i, out_p


_ENGINES = {}


def get_engine(device=None):
    """one engine per device (buffers are cached inside)"""
    torch = _lib.require_cuda()
    idx = torch.cuda.current_device() if device is None else int(device)
    if idx not in _ENGINES:
        _ENGINES[idx] = Engine(idx)
    return _ENGINES[idx]
