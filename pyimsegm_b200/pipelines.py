"""
Segmentation pipelines: SLIC -> per-superpixel features -> class model -> GraphCut, resident on the GPU.

Mirror of the reference module ``imsegm/pipelines.py`` for the unsupervised hot path (same names, arguments
and return values):

* :func:`pipe_color2d_slic_features_model_graphcut`     (reference pipelines.py:46-110)
* :func:`estim_model_classes_group`                     (reference pipelines.py:113-157)
* :func:`segment_color2d_slic_features_model_graphcut`  (reference pipelines.py:160-241)
* :func:`compute_color2d_superpixels_features`          (reference pipelines.py:244-270)

The image goes to the device once; label map, features, class model, graph, energies and the cut never leave it and the
host synchronises ONCE, when the results are downloaded.  A caller-fitted mixture or tree model is compiled to device tables
(:mod:`.class_models`) and evaluated there too; any other model, or a self-fitted one the device GMM does not cover, costs one
round trip: features [N, D] down, probabilities [N, K] up.

The supervised training of the reference (``train_classif_color2d_slic_features``, pipelines.py:293-379) is
:func:`train_classif_images_batch`: per annotated image, SLIC, the feature table, one training label per superpixel
(``isb_superpixel_train_labels``) and the distinct rounded rows of each class for ``feature_balance='unique'``
(``isb_unique_rows_rounded``) run on the device over CUDA streams, then the classifier is fitted by
``classification.create_classif_search_train_export``.  :func:`wrapper_compute_color2d_slic_features_labels` is its one-image data
step.  The reference's name itself still raises NotImplementedError.

Gray volumes have the same resident form: :func:`segment_resident_volume` (a device volume in, device results out) and
:func:`segment_volumes_batch` (host volumes over CUDA streams) run ``pipe_gray3d_slic_features_model_graphcut``'s stages on the device.
"""
import logging

import numpy as np

from .class_models import CompiledModel, compile_model
from .descriptors import (FEATURES_SET_COLOR, _check_gradient_size, compute_selected_features_img2d, device_feature_table,
                          flags_are_resident, native_feature_layout)
from .engine import edge_capacity, edges_fit, get_engine
from .graph_cuts import class_model_spec, device_gmm_applicable, estim_class_model, reference_edge_type, segment_graph_cut_general
from .superpixels import _as_rgb_like, _supported_dtype, slic_params

#: basic features extracted from superpixels (reference pipelines.py:35)
FTS_SET_SIMPLE = FEATURES_SET_COLOR
#: default classifier of the supervised path (reference classification.py:54)
CLASSIF_NAME = 'RandForest'
#: default clustering for unsupervised segmentation (reference pipelines.py:39 -> classification.DEFAULT_CLUSTERING)
CLUSTER_METHOD = 'kMeans'
#: images left out during cross-validation training (reference pipelines.py:41)
CROSS_VAL_LEAVE_OUT = 2
#: default number of workers of the reference's process pool (pipelines.py:43); the GPU path shards images over
#: devices instead, the value is kept for signature compatibility
NB_WORKERS = 1


class DeviceSuperpixels(object):
    """device-resident result of SLIC + descriptors for one image or volume: ``d_feat`` is the table the class model reads,
    ``d_centres`` None for a volume (its 6-connected graph takes the centroids from the label volume)"""
    __slots__ = ('d_img', 'd_seg', 'd_n_labels', 'nb_bound', 'd_feat', 'd_centres', 'shape')


def _device_slic_features(eng, image, dict_features, sp_size, sp_regul):
    """H2D, SLIC, the feature table of ``native_feature_layout`` + centroids; everything stays on the device"""
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    on_device = hasattr(image, 'is_cuda')
    if not on_device:
        image = _supported_dtype(_as_rgb_like(image))
    H, W = int(image.shape[0]), int(image.shape[1])
    _check_gradient_size((H, W), dict_features.values())      # before SLIC: the feature table would refuse this image
    n_seg, compact = slic_params((H, W), sp_size, sp_regul)
    if n_seg < 1:
        raise ValueError('superpixel size %r is larger than the image %r' % (sp_size, tuple(image.shape)))
    res = DeviceSuperpixels()
    res.shape = (H, W)
    res.d_img = image if on_device else eng.to_device(image, 'image')
    res.d_seg, res.d_n_labels = eng.slic(res.d_img, n_seg, compact, sigma=1.0)
    res.nb_bound = eng.slic_label_bound(H, W, n_seg)
    res.d_feat = eng.buf('feat', (res.nb_bound, max(native_feature_layout(dict_features)[1], 1)), eng.torch.float64)
    res.d_centres = device_feature_table(eng, res.d_img, res.d_seg, res.nb_bound, dict_features, res.d_feat, want_centres=True)
    if res.d_centres is None:
        _, res.d_centres, _ = eng.segment_stats(None, res.d_seg, res.nb_bound, (), want_centres=True)
    return res


def compute_color2d_superpixels_features(image, dict_features, sp_size=30, sp_regul=0.2):
    """ segment the image into superpixels and estimate features per superpixel (reference pipelines.py:244-270)

    :return tuple(ndarray,ndarray): superpixel map [H, W], features [N, D]
    """
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    image = np.asarray(image)
    eng = get_engine()
    if image.ndim == 3 and flags_are_resident(dict_features):
        res = _device_slic_features(eng, image, dict_features, sp_size, sp_regul)
        nb = int(eng.to_host(res.d_n_labels)[0])
        slic = eng.to_host(res.d_seg).astype(np.int64)
        features = eng.to_host(res.d_feat[:nb]).copy()
    else:
        from .superpixels import segment_slic_img2d
        slic = segment_slic_img2d(image, sp_size=sp_size, relative_compact=sp_regul)
        features, _ = compute_selected_features_img2d(image, slic, dict_features)
    features[np.isnan(features)] = 0
    return slic, features


def _argmin_labels_device(eng, proba):
    graph_labels = np.argmin(np.abs(-np.log(np.clip(proba, 0.01, 0.99))), axis=-1).astype(np.int32)
    return eng.to_device(graph_labels, 'gc_labels_in')


#: replay the device part of the path as CUDA graphs once a configuration has been seen twice (the ~70 kernel launches of an image
#: cost more host time than the GPU needs for them when images are processed back to back, and the gaps between them add up)
USE_CUDA_GRAPHS = True
_GRAPHS = {}


def _graph_call(eng, key, fn):
    """``fn()`` -- a sequence of C-ABI launches that never touches the host and writes into the engine's cached buffers -- run
    eagerly the first time ``key`` is seen (this also sizes every buffer), captured as a CUDA graph the second time, replayed
    afterwards.  Returns what ``fn`` returned (device tensors that every replay refills)."""
    if not USE_CUDA_GRAPHS:
        return fn()
    entry = _GRAPHS.get(key)
    if entry is None:
        _GRAPHS[key] = 'seen'
        return fn()
    torch = eng.torch
    if entry == 'seen':
        graph = torch.cuda.CUDAGraph()
        n0 = eng.lib.isb_launch_count()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream(device=eng.device)
        side.wait_stream(cur)
        with torch.cuda.graph(graph, stream=side):
            out = fn()
        cur.wait_stream(side)
        eng.graphs_captured += 1      # from now on the engine never frees a buffer it outgrows
        entry = _GRAPHS[key] = (graph, out, int(eng.lib.isb_launch_count() - n0))
    graph, out, n_kernels = entry
    graph.replay()
    eng.lib.isb_note_graph_replay(n_kernels)
    return out


def _features_key(dict_features):
    return tuple(sorted((k, tuple(v)) for k, v in dict_features.items()))


def _resident_width(dict_features):
    """the column count of the resident feature table of ``dict_features``, or None when the dictionary is not resident"""
    return native_feature_layout(dict_features)[1] if flags_are_resident(dict_features) else None


def _device_model(model, n_features):
    """``model`` in the form :func:`_device_proba` runs: a resident fit tuple (:func:`_fit_model`) and a
    :class:`~.class_models.CompiledModel` stay as they are; a fitted model (or its bound ``predict_proba``) is compiled to device
    tables when :func:`~.class_models.compile_model` takes it and its feature count is ``n_features`` (None: the table is not
    resident, never compile); anything else is the host callable proba_fn(features) -- ``model`` itself when it is callable, else
    its ``predict_proba``"""
    from . import graph_cuts
    if isinstance(model, (tuple, CompiledModel)):
        return model
    if graph_cuts.USE_DEVICE_PREDICT and n_features is not None:
        fitted = model.__self__ if getattr(model, '__name__', None) == 'predict_proba' and hasattr(model, '__self__') else model
        cm = compile_model(fitted)
        if cm is not None and cm.n_features_in == n_features:
            return cm
    return model if callable(model) else model.predict_proba


def _fit_model(nb_classes, use_scaler, estim_model='GMM', pca_coef=None, max_iter=99):
    """the resident model tuple of a device-fitted class model: ('fit', nb_classes, use_scaler, 99) for the default 'GMM' with
    ``max_iter`` 99, ('fit', nb_classes, use_scaler, max_iter, kind, n_init, pca_coef) for any other variant
    (graph_cuts.class_model_spec).  It is part of the CUDA-graph key, so a configuration never replays the graph of another."""
    kind, n_init, max_iter = class_model_spec(estim_model, nb_classes, max_iter)
    if kind == 'GMM' and n_init == max(1, int(np.sqrt(max_iter))) and max_iter == 99 and pca_coef is None:
        return ('fit', nb_classes, use_scaler, max_iter)
    return ('fit', nb_classes, use_scaler, max_iter, kind, n_init, pca_coef)


def _fit_spec(model):
    """(nb_classes, use_scaler, max_iter, kind, n_init, pca_coef) of a resident model tuple (:func:`_fit_model`)"""
    _, nb_classes, use_scaler, max_iter, *rest = model
    kind, n_init, pca_coef = rest if rest else ('GMM', max(1, int(np.sqrt(max_iter))), None)
    return nb_classes, use_scaler, max_iter, kind, n_init, pca_coef


def _device_proba(eng, model, d_feat, d_n, nb):
    """class probabilities [nb, K] (device) of the first ``d_n`` (device count) rows of the feature table ``d_feat`` [nb, D] under
    a model of :func:`_device_model`: a fit tuple is fitted on the GPU and a CompiledModel evaluated there, neither syncs with the
    host (a float pca_coef reads its component count back, and D > 16 features read one flag per EM iteration); a host callable
    costs one round trip -- the rows down with NaN set to 0, its probabilities up, padded with zero rows to the label bound ``nb``
    as a device model leaves them"""
    from . import graph_cuts
    if isinstance(model, CompiledModel):
        return eng.class_model_predict(d_feat, model, d_n=d_n)
    if isinstance(model, tuple):
        nb_classes, use_scaler, max_iter, kind, n_init, pca_coef = _fit_spec(model)
        return graph_cuts.device_fit_predict(eng, d_feat, nb_classes, use_scaler, kind, n_init, max_iter, pca_coef, d_n=d_n)[0]
    n = int(eng.to_host(d_n)[0])
    features = eng.to_host(d_feat[:n]).copy()
    features[np.isnan(features)] = 0
    proba = np.asarray(model(features), dtype=np.float64)
    logging.debug('list of probabilities: %r', proba.shape)
    padded = np.zeros((int(nb), proba.shape[1]))
    padded[:n] = proba
    return eng.to_device(padded, 'proba')


def _run_resident(eng, front, model, gc_regul, gc_edge_type, graph_key=None, early_soft=False):
    """the hot path on the device after the caller's argument checks: ``front()`` -> :class:`DeviceSuperpixels`, the class
    probabilities of ``model`` (:func:`_device_proba`), then the argmin of the probabilities when ``gc_regul`` <= 0 (read on the
    host) or the graph cut over the superpixel graph (4-connected in 2-D, 6-connected in 3-D) and the LUT gathers.  With a fit
    tuple or a CompiledModel nothing syncs with the host until the results are ready.
    With ``graph_key`` (the caller's key of the front and the model) and a cut, the two halves -- front + probabilities,
    probabilities -> cut and LUT gathers -- are CUDA-graph replays (:func:`_graph_call`).
    Returns (d_segm, soft, check): ``soft`` is the device segm_soft, or with ``early_soft`` and a graph cut the (pinned host tensor,
    event) of :meth:`~.engine.Engine.early_soft`; ``check`` is None or (d_n_edges, edge_cap) still to be verified by the caller
    (:func:`~.engine.edges_fit`)."""
    from . import graph_cuts
    no_cut = (not isinstance(gc_regul, (list, np.ndarray))) and gc_regul <= 0
    graphed = graph_key is not None and not no_cut

    def first_half():
        res = front()
        return res, _device_proba(eng, model, res.d_feat, res.d_n_labels, res.nb_bound)

    res, d_proba = _graph_call(eng, graph_key, first_half) if graphed else first_half()
    nb = res.nb_bound
    if no_cut:
        proba = eng.to_host(d_proba[:int(eng.to_host(res.d_n_labels)[0])])
        return eng.gather(res.d_seg, _argmin_labels_device(eng, proba), d_proba) + (None, )
    cap = edge_capacity(nb, ndim=len(res.shape))
    soft = eng.early_soft(res.d_seg, d_proba) if early_soft else None

    def second_half():
        d_vec = graph_cuts.device_edge_vectors(eng, gc_edge_type, res.d_img, res.d_seg, nb, res.d_feat, res.d_n_labels)
        d_labels, d_n_edges = graph_cuts.device_graphcut(eng, res.d_seg, res.d_centres, nb, d_proba, gc_regul, gc_edge_type, res.d_n_labels,
                                                         cap, edge_vectors=d_vec)
        return eng.gather(res.d_seg, d_labels, None if early_soft else d_proba) + (d_n_edges, )

    if graphed:
        # 'color' and 'features' also read the image and the feature table: the captured launches hold their addresses, the
        # image's dtype and the table's shape and row stride, so all of these are part of the key
        vec_src = None
        if gc_edge_type in ('color', 'features'):
            vec_src = (res.d_img.data_ptr(), str(res.d_img.dtype), tuple(res.d_img.shape), res.d_feat.data_ptr(), tuple(res.d_feat.shape),
                       int(res.d_feat.stride(0)))
        key2 = ('cut', id(eng), res.d_seg.data_ptr(), d_proba.data_ptr(), res.d_centres.data_ptr(), res.shape, res.nb_bound,
                int(d_proba.shape[1]), float(gc_regul), gc_edge_type, vec_src, cap, not early_soft)
        d_segm, d_soft, d_n_edges = _graph_call(eng, key2, second_half)
    else:
        d_segm, d_soft, d_n_edges = second_half()
    return d_segm, (soft if early_soft else d_soft), (d_n_edges, cap)


def _run_resident_image(eng, image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type, early_soft=False):
    """:func:`_run_resident` for one colour image (host, or a device tensor that is used where it is), with SLIC and the feature
    table of :func:`_device_slic_features` as the front.  With a fit tuple or a CompiledModel and colour features the path is a
    CUDA-graph replay; the image then has to sit in one of the engine's cached buffers."""
    from . import graph_cuts
    graph_cuts.check_edge_type(gc_edge_type)
    if not hasattr(image, 'is_cuda'):
        image = eng.to_device(_supported_dtype(_as_rgb_like(np.asarray(image))), 'image')
    graphable = USE_CUDA_GRAPHS and all(k.startswith('color') for k in dict_features) and flags_are_resident(dict_features)
    model_key = None
    if graphable and isinstance(model, CompiledModel):
        model_key = ('compiled', model.digest)
    elif (graphable and isinstance(model, tuple) and _fit_spec(model)[5] is None
          and native_feature_layout(dict_features)[1] <= graph_cuts.DEVICE_GMM_SINGLE_KERNEL_MAX_FEATURES):
        model_key = model
    key1 = None
    if model_key is not None:
        key1 = ('probabilities', id(eng), image.data_ptr(), tuple(image.shape), str(image.dtype), model_key, _features_key(dict_features),
                sp_size, sp_regul)
    return _run_resident(eng, lambda: _device_slic_features(eng, image, dict_features, sp_size, sp_regul), model, gc_regul, gc_edge_type,
                         key1, early_soft)


def _segment(image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type, debug_visual, classes=None):
    image = np.asarray(image)
    eng = get_engine()
    native = image.ndim == 3 and flags_are_resident(dict_features) and gc_edge_type not in ('color', 'features')
    if not native or debug_visual is not None:
        # general path: every stage still runs on the device, but through the numpy-facing stage functions
        if isinstance(model, CompiledModel):
            proba_fn = model.predict_proba
        elif callable(model):
            proba_fn = model
        elif len(model) == 4:
            proba_fn = lambda f: estim_class_model(f, model[1], 'GMM', None, model[2], model[3]).predict_proba(f)  # noqa: E731
        else:
            from .graph_cuts import fit_class_model_device
            nb_classes, use_scaler, max_iter, kind, n_init, pca_coef = _fit_spec(model)
            proba_fn = lambda f: fit_class_model_device(f, nb_classes, use_scaler, kind, n_init, max_iter,  # noqa: E731
                                                        pca_coef).predict_proba(f)
        slic, features = compute_color2d_superpixels_features(image, dict_features, sp_size=sp_size, sp_regul=sp_regul)
        if debug_visual is not None:
            img3 = image if image.ndim == 3 else np.stack([image] * 3, axis=-1)
            debug_visual['image'] = img3
            debug_visual['slic'] = slic
            means = np.stack([np.bincount(slic.ravel(), weights=img3[..., c].ravel()) for c in range(3)], 1)
            debug_visual['slic_mean'] = (means / np.maximum(np.bincount(slic.ravel()), 1)[:, None])[slic]
        proba = proba_fn(features)
        segm_soft = proba[slic]
        graph_labels = segment_graph_cut_general(slic, proba, image, features, gc_regul, gc_edge_type, debug_visual=debug_visual)
        if classes is not None:
            graph_labels = classes[graph_labels]
        return graph_labels[slic], segm_soft
    gc_edge_type = reference_edge_type(gc_edge_type)
    while True:
        d_segm, soft, check = _run_resident_image(eng, image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type,
                                                  early_soft=True)
        if check is None:   # no graph cut: both gathers were done at the end of the main stream
            (segm, soft), done = eng.download((d_segm, soft))
            done.synchronize()
            break
        (segm, n_edges), done = eng.download((d_segm, check[0]))
        done.synchronize()
        soft, soft_done = soft
        soft_done.synchronize()
        # the next call reuses the buffers the side stream has just read: nothing of this call is left in flight
        if edges_fit(n_edges[0], check[1]):
            break
    segm, soft = segm.numpy(), soft.numpy()
    if classes is not None:
        segm = np.asarray(classes)[segm]
    return segm, soft


_BATCH_ENGINES = {}


def _batch_engines(nb_streams):
    """independent Engine instances (own buffers) with one CUDA stream each, cached per device"""
    from .engine import Engine
    torch = get_engine().torch
    dev = torch.cuda.current_device()
    pool = _BATCH_ENGINES.setdefault(dev, [])
    while len(pool) < nb_streams:
        pool.append((Engine(dev), torch.cuda.Stream(device=dev)))
    return pool[:nb_streams]


def _over_streams(list_images, nb_streams, max_in_flight, launch, finish):
    """``launch(eng, image) -> (pinned host tensors, event, extra)`` for consecutive images alternating over ``nb_streams`` CUDA
    streams with their own engines, at most ``max_in_flight`` images ahead of ``finish(index, host tensors, extra)``, which runs in
    input order once the event has completed: returns what ``finish`` returned, per image"""
    engines = _batch_engines(nb_streams)
    torch = engines[0][0].torch
    results, pending = [None] * len(list_images), []

    def flush(limit):
        while len(pending) > limit:
            idx, (hosts, done, extra) = pending.pop(0)
            done.synchronize()
            results[idx] = finish(idx, hosts, extra)

    caller_stream = torch.cuda.current_stream()
    for i, image in enumerate(list_images):
        eng, stream = engines[i % nb_streams]
        stream.wait_stream(caller_stream)
        with torch.cuda.stream(stream):
            pending.append((i, launch(eng, np.asarray(image))))
        flush(max_in_flight)
    flush(0)
    return results


def _resident_batch(items, nb_streams, max_in_flight, run, redo, classes):
    """``run(eng, item)`` -> :func:`_run_resident`'s (d_segm, d_soft, check) for every item of a batch over :func:`_over_streams`,
    each item's results downloaded with its edge count; an item whose edge table overflowed is redone by ``redo(index)`` -> host
    (segm, segm_soft).  Returns (segm mapped through ``classes`` unless it is None, segm_soft) per item, in input order"""
    def launch(eng, item):
        d_segm, d_soft, check = run(eng, item)
        return eng.download((d_segm, d_soft) + ((check[0], ) if check is not None else ())) + (check, )

    def finish(idx, hosts, check):
        if check is not None and not edges_fit(hosts[2][0], check[1]):
            segm, soft = redo(idx)
        else:
            segm, soft = hosts[0].numpy(), hosts[1].numpy()
        return (segm if classes is None else np.asarray(classes)[segm]), soft

    return _over_streams(items, nb_streams, max_in_flight, launch, finish)


def segment_images_batch(list_images, nb_classes=None, dict_features=FTS_SET_SIMPLE, sp_size=30, sp_regul=0.2, use_scaler=True,
                         gc_regul=1., gc_edge_type='model', model_pipeline=None, nb_streams=3, max_in_flight=6, estim_model='GMM',
                         pca_coef=None):
    """ the hot path over a LIST of images, the way the reference's experiment scripts run it through a process pool
    (``run_segm_slic_model_graphcut.py:461-466``): here consecutive images alternate over ``nb_streams`` CUDA streams with
    their own buffers, so the upload of image i+1 and the download of image i-1 overlap the kernels of image i.

    :param int nb_classes: fit the class model per image on the GPU (as ``pipe_color2d_slic_features_model_graphcut``, with its
        ``estim_model`` and ``pca_coef``), or
    :param model_pipeline: a fitted model used for every image (as ``segment_color2d_slic_features_model_graphcut``)
    :return list(tuple(ndarray,ndarray)): (segm, segm_soft) per image, in input order
    """
    if (nb_classes is None) == (model_pipeline is None):
        raise ValueError('give either nb_classes (per-image GMM) or model_pipeline')
    native = flags_are_resident(dict_features) and gc_edge_type not in ('color', 'features')
    nb_fts = native_feature_layout(dict_features)[1] if native else 10 ** 6
    if model_pipeline is None and not (native and device_gmm_applicable(nb_fts, nb_classes, estim_model, pca_coef)):
        return [pipe_color2d_slic_features_model_graphcut(im, nb_classes, dict_features, sp_size, sp_regul, pca_coef, use_scaler,
                                                          estim_model, gc_regul, gc_edge_type) for im in list_images]
    if not native:
        return [segment_color2d_slic_features_model_graphcut(im, model_pipeline, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type)
                for im in list_images]
    if model_pipeline is None:
        model = _fit_model(nb_classes, use_scaler, estim_model, pca_coef)
    else:
        model = _device_model(model_pipeline.predict_proba, nb_fts)
    gc_edge_type = reference_edge_type(gc_edge_type)

    def run(eng, image):
        return _run_resident_image(eng, image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type)

    def redo(idx):      # through the single-image path
        return _segment(list_images[idx], model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type, None)

    return _resident_batch(list_images, nb_streams, max_in_flight, run, redo, getattr(model_pipeline, 'classes_', None))


def compute_features_batch(list_images, dict_features, sp_size=30, sp_regul=0.2, nb_streams=3, max_in_flight=6):
    """ superpixel features of a LIST of images (the per-image half of ``estim_model_classes_group``, which the reference hands to
    a process pool, pipelines.py:139-147): consecutive images alternate over ``nb_streams`` CUDA streams with their own buffers,
    nothing synchronises with the host until an image's feature table is downloaded

    :return list(ndarray): features [N_i, D] per image, in input order
    """
    if not flags_are_resident(dict_features) or any(np.ndim(im) != 3 for im in list_images):
        return [compute_color2d_superpixels_features(im, dict_features, sp_size=sp_size, sp_regul=sp_regul)[1] for im in list_images]
    def launch(eng, image):
        res = _device_slic_features(eng, image, dict_features, sp_size, sp_regul)
        return eng.download((res.d_feat, res.d_n_labels)) + (None, )

    def finish(idx, hosts, _):
        features = hosts[0].numpy()[:int(hosts[1][0])].copy()
        features[np.isnan(features)] = 0
        return features

    return _over_streams(list_images, nb_streams, max_in_flight, launch, finish)


def train_annotation(image, annot):
    """ the annotation as the supervised data step reads it: ``astype(int)`` as the reference casts it (floats truncate toward zero,
    bools become 0 / 1), then int32 with every negative value as -1 (unknown).  Raises ImageDimensionError when its shape is not the
    image's [H, W], ValueError for a label above 2^31 - 1, and the reference's ValueError when every value is below -1 (its unknown
    label ``max(annot) + 1`` is then itself negative)

    :return ndarray: int32 [H, W]
    """
    from .utilities import ImageDimensionError
    annot = np.asarray(annot).astype(int)
    if np.shape(image)[:2] != annot.shape[:2] or annot.ndim != 2:
        raise ImageDimensionError('image %r and annot %r should match' % (np.shape(image), annot.shape))
    if annot.size and int(annot.max()) > np.iinfo(np.int32).max:
        raise ValueError('annotation label %d is above 2^31 - 1' % int(annot.max()))
    if annot.size and int(annot.max()) < -1:
        raise ValueError('only positive labels are allowed')
    return np.maximum(annot, -1).astype(np.int32)


def _train_data(list_images, list_annots, dict_features, sp_size, sp_regul, label_purity, unique, nb_streams, max_in_flight):
    """ the per-image data step of the supervised training on annotations that :func:`train_annotation` has checked: per image
    (slic int64 [H, W], features [N, D] with NaN -> 0, labels int64 [N], balanced) where ``balanced`` is the image's
    ``balance_dataset_by_(features[labels != -1], labels[labels != -1], 'unique')`` as (rows, labels) when ``unique`` and the image
    took the resident path, else None.  Colour images with a dictionary of the resident feature table alternate over
    ``nb_streams`` CUDA streams as in :func:`compute_features_batch` (SLIC, features, labels and unique rows on the device, one
    download); other images compute their superpixels and features through :func:`compute_color2d_superpixels_features` and
    their labels on the device. """
    D = native_feature_layout(dict_features)[1] if flags_are_resident(dict_features) else 0
    if D == 0 or any(np.ndim(im) != 3 for im in list_images):
        eng = get_engine()
        out = []
        for image, annot in zip(list_images, list_annots):
            slic, features = compute_color2d_superpixels_features(image, dict_features, sp_size=sp_size, sp_regul=sp_regul)
            n = int(slic.max()) + 1
            d_seg = eng.to_device(slic.astype(np.int32), 'train_slic')
            labels = eng.to_host(eng.train_labels(d_seg, n, eng.to_device(annot, 'train_annot'), label_purity)).copy()
            out.append((slic, features, labels, None))
        return out

    def launch(eng, idx):        # _over_streams walks the image indices: the annotation goes with its image
        res = _device_slic_features(eng, np.asarray(list_images[int(idx)]), dict_features, sp_size, sp_regul)
        d_labels = eng.train_labels(res.d_seg, res.nb_bound, eng.to_device(list_annots[int(idx)], 'train_annot'), label_purity,
                                    d_n=res.d_n_labels)
        d_x = eng.nan_free_table(res.d_feat, D, res.d_n_labels)
        outs = (res.d_n_labels, res.d_seg, d_x, d_labels)
        if unique:
            outs += eng.unique_rows(d_x, d_labels, D, d_n=res.d_n_labels)
        return eng.download(outs) + (None, )

    def finish(idx, hosts, _):
        n = int(hosts[0][0])
        balanced = None
        if unique:
            m = int(hosts[6][0])
            if m < 0:
                raise ValueError('the feature table of image %d holds NaN' % idx)
            balanced = (hosts[4].numpy()[:m].copy(), hosts[5].numpy()[:m].copy())
        return hosts[1].numpy().astype(np.int64), hosts[2].numpy()[:n].copy(), hosts[3].numpy()[:n].copy(), balanced

    return _over_streams(range(len(list_images)), nb_streams, max_in_flight, launch, finish)


def wrapper_compute_color2d_slic_features_labels(img_annot, sp_size, sp_regul, dict_features, label_purity):
    """ superpixels, their features and one training label per superpixel from an annotated image -- the data step of the
    supervised path (reference pipelines.py:272-290): a superpixel takes the annotation label that covers most of it, or -1
    when that share is below ``label_purity`` (or the winner is the negative / unknown label).  A one-image call of the data step
    of :func:`train_classif_images_batch`; the labels come from ``isb_superpixel_train_labels``.

    :param tuple(ndarray,ndarray) img_annot: image and its annotation (negative values = unknown)
    :return tuple(ndarray,ndarray,ndarray): slic [H, W], features [N, D], labels [N]
    """
    img, annot = img_annot
    annot = train_annotation(img, annot)
    return _train_data([img], [annot], dict_features, sp_size, sp_regul, label_purity, False, 1, 1)[0][:3]


def train_classif_images_batch(list_images, list_annots, dict_features, sp_size=30, sp_regul=0.2, clf_name=CLASSIF_NAME, label_purity=0.9,
                               feature_balance='unique', pca_coef=None, nb_classif_search=1, nb_hold_out=CROSS_VAL_LEAVE_OUT, nb_workers=1,
                               nb_streams=3, max_in_flight=6):
    """ train a superpixel classifier on annotated images: the reference's ``train_classif_color2d_slic_features``
    (pipelines.py:293-379) with the per-image data step on the GPU.  Consecutive images alternate over ``nb_streams`` CUDA streams
    with their own buffers; for each the device runs SLIC, the feature table, the training label of every superpixel
    (``isb_superpixel_train_labels``) and, for ``feature_balance='unique'``, the image's distinct rounded rows per class
    (``isb_unique_rows_rounded``), and the host downloads them once.  Then as the reference: 'random', 'kmeans' and unknown names
    balance every image with ``balance_dataset_by_`` in image order (so the global RNGs are drawn from in the reference's order),
    None keeps every labelled row; an image without a labelled superpixel raises the reference's ValueError unless
    ``feature_balance`` is None; the images' rows are concatenated and ``create_classif_search_train_export`` fits the classifier,
    cross-validated over the images by ``CrossValidateGroups`` when there are more than ``5 * nb_hold_out`` of them.
    Dictionaries outside the resident feature table and gray images compute their superpixels and features through
    :func:`compute_color2d_superpixels_features` and are balanced on the host.

    :return tuple: (classif, list_slic int64 [H, W], list_features f64 [N, D], list_labels int64 [N])
    """
    from .classification import CrossValidateGroups, _rows_array, balance_dataset_by_, create_classif_search_train_export
    logging.info('TRAIN Superpixels-Features-Classifier')
    if len(list_images) != len(list_annots):
        raise ValueError('size of images (%i) and annotations (%i) should match' % (len(list_images), len(list_annots)))
    annots = [train_annotation(img, annot) for img, annot in zip(list_images, list_annots)]
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    unique = feature_balance is not None and feature_balance.lower() == 'unique'
    data = _train_data(list_images, annots, dict_features, sp_size, sp_regul, label_purity, unique, nb_streams, max_in_flight)
    list_slic, list_features, list_labels = [d[0] for d in data], [d[1] for d in data], [d[2] for d in data]
    blocks, labels_all, sizes = [], [], []
    for _, features, labels, balanced in data:
        keep = labels != -1
        if feature_balance is None:
            features, labels = features[keep], labels[keep]
        elif balanced is not None and keep.any():
            features, labels = balanced
        else:
            features, labels = balance_dataset_by_(features[keep], labels[keep], balance_type=feature_balance)
        blocks.append(features)
        labels_all += np.asarray(labels).tolist()
        sizes.append(len(labels))
    features = np.nan_to_num(_rows_array(blocks))
    labels = np.array(labels_all, dtype=int)
    cv = CrossValidateGroups(sizes, nb_hold_out=nb_hold_out) if len(sizes) > nb_hold_out * 5 else 10
    classif, _ = create_classif_search_train_export(clf_name, features, labels, pca_coef=pca_coef, cross_val=cv,
                                                    nb_search_iter=nb_classif_search, nb_workers=nb_workers)
    return classif, list_slic, list_features, list_labels


def train_classif_color2d_slic_features(list_images, list_annots, dict_features, sp_size=30, sp_regul=0.2, clf_name=CLASSIF_NAME,
                                        label_purity=0.9, feature_balance='unique', pca_coef=None, nb_classif_search=1,
                                        nb_hold_out=CROSS_VAL_LEAVE_OUT, nb_workers=1):
    """ the supervised training wrapper of the reference (pipelines.py:293-379).  Not provided under this name: the same training,
    with the per-image data step on the GPU, is :func:`train_classif_images_batch` """
    raise NotImplementedError('use pipelines.train_classif_images_batch, which trains the classifier as the reference\'s '
                              'train_classif_color2d_slic_features does, with the data step on the GPU')


def pipe_gray3d_slic_features_model_graphcut(image, nb_classes, dict_features, spacing=(12, 1, 1), sp_size=15, sp_regul=0.2,
                                             gc_regul=0.1):
    """ the pipeline for a gray VOLUME: 3-D SLIC supervoxels, their features, a class model, GraphCut over the 6-connected
    supervoxel graph (reference pipelines.py:382-431)

    :param ndarray image: gray volume [D, H, W]
    :param tuple(int,int,int) spacing: voxel spacing (z, y, x)
    :return ndarray: class per voxel [D, H, W]
    """
    from .descriptors import compute_selected_features_gray3d, norm_features
    from .superpixels import segment_slic_img3d_gray
    image = np.asarray(image)
    slic = segment_slic_img3d_gray(image, sp_size=sp_size, relative_compact=sp_regul, space=spacing)
    features, _ = compute_selected_features_gray3d(image, slic, dict_features)
    features[np.isnan(features)] = 0
    features, _ = norm_features(features)
    model = estim_class_model(features, nb_classes)
    proba = model.predict_proba(features)
    graph_labels = segment_graph_cut_general(slic, proba, image, features, gc_regul)
    return graph_labels[slic]


#: statistics of a gray volume that the resident volume path computes on the device (compute_image3d_gray_statistic's columns)
RESIDENT_VOLUME_FLAGS = ('mean', 'std', 'energy', 'median')


def _volume_flags(dict_features):
    """the statistic columns of the resident volume feature table, in compute_selected_features_gray3d's order (the union of the
    ``color*`` groups' flags), or None when the dictionary needs the stage path (``tLM*`` groups, ``meanGrad``)"""
    from .descriptors import NAMES_FEATURE_FLAGS
    if not dict_features or not all(k.startswith('color') for k in dict_features):
        return None
    flags = set(f for v in dict_features.values() for f in v)
    if not flags or not flags <= set(RESIDENT_VOLUME_FLAGS):
        return None
    return [f for f in NAMES_FEATURE_FLAGS if f in flags]


def _device_slic3d_features(eng, d_vol, dict_features, spacing, sp_size, sp_regul):
    """pipe_gray3d_slic_features_model_graphcut's front on the device: 3-D SLIC, the gray statistics into a device table and
    norm_features (StandardScaler, bit for bit), whose standardised table is ``d_feat``.  ``d_vol``: a gray volume [D, H, W] on the
    device or on the host (uploaded)."""
    from .superpixels import slic3d_params
    flags = _volume_flags(dict_features)
    if flags is None:
        raise ValueError('the resident volume path computes the statistics %r of "color" groups, got %r'
                         % (RESIDENT_VOLUME_FLAGS, dict_features))
    if sp_regul <= 0.:
        raise ValueError('slic. regularisation must be positive')
    if not hasattr(d_vol, 'is_cuda'):
        d_vol = eng.to_device(_supported_dtype(np.asarray(d_vol)), 'volume')
    if d_vol.dim() != 3:
        raise ValueError('expected a gray volume [D, H, W], got shape %r' % (tuple(d_vol.shape), ))
    shape = tuple(int(v) for v in d_vol.shape)
    n_seg, compact = slic3d_params(shape, sp_size, sp_regul, spacing)
    if n_seg < 1 or compact < 1:
        raise ValueError('superpixel size %r / compactness do not fit the volume %r' % (sp_size, shape))
    res = DeviceSuperpixels()
    res.shape, res.d_img, res.d_centres = shape, d_vol, None
    res.d_seg, res.d_n_labels = eng.slic3d(d_vol, n_seg, compact, spacing, sigma=1.0)
    res.nb_bound = eng.slic_label_bound(int(np.prod(shape)), 1, n_seg)
    res.d_feat = eng.standard_scaler(eng.gray_table(d_vol, res.d_seg, res.nb_bound, flags), res.d_n_labels)[0]
    return res


def segment_resident_volume(d_vol, model, dict_features, spacing=(12, 1, 1), sp_size=15, sp_regul=0.2, gc_regul=0.1):
    """ pipe_gray3d_slic_features_model_graphcut with the gray volume ALREADY on the device (a cuda tensor [D, H, W]) and the
    results left there: returns (segm int32 [D, H, W], segm_soft float64 [D, H, W, K]) device tensors.  ``model`` is a fitted model
    (or its bound ``predict_proba``) -- evaluated on the device when :func:`~.class_models.compile_model` supports it --, a callable
    proba_fn(features), or ('fit', nb_classes, use_scaler, max_iter) (:func:`_fit_model`) for the class model fitted on the GPU.  The
    model sees the standardised features, as in the reference.  ``dict_features``: ``color`` groups of mean / std / energy / median.
    The indices in ``segm`` are not mapped through the model's ``classes_``.
    A volume's supervoxel graph has no planar bound on its edges, so the call reads the edge count back (4 bytes) once the cut is
    enqueued and redoes the volume with a larger table when it overflowed; nothing else synchronises with the host. """
    eng = get_engine()
    flags = _volume_flags(dict_features)
    model = _device_model(model, len(flags) if flags else None)
    while True:
        d_segm, d_soft, check = _run_resident(eng, lambda: _device_slic3d_features(eng, d_vol, dict_features, spacing, sp_size, sp_regul),
                                              model, gc_regul, 'model')
        if check is None or edges_fit(eng.to_host(check[0])[0], check[1]):
            return d_segm, d_soft


def _segment_volume_stages(volume, proba_fn, dict_features, spacing, sp_size, sp_regul, gc_regul):
    """the volume pipeline through the numpy-facing stage functions (any feature dictionary): (segm [D, H, W], segm_soft [D, H, W, K])"""
    from .descriptors import compute_selected_features_gray3d, norm_features
    from .superpixels import segment_slic_img3d_gray
    volume = np.asarray(volume)
    slic = segment_slic_img3d_gray(volume, sp_size=sp_size, relative_compact=sp_regul, space=spacing)
    features, _ = compute_selected_features_gray3d(volume, slic, dict_features)
    features[np.isnan(features)] = 0
    features, _ = norm_features(features)
    proba = proba_fn(features)
    graph_labels = segment_graph_cut_general(slic, proba, volume, features, gc_regul)
    return graph_labels[slic].astype(np.int32), proba[slic]


def segment_volumes_batch(list_volumes, nb_classes=None, model_pipeline=None, dict_features=FTS_SET_SIMPLE, spacing=(12, 1, 1),
                          sp_size=15, sp_regul=0.2, gc_regul=0.1, use_scaler=True, nb_streams=3, max_in_flight=6):
    """ pipe_gray3d_slic_features_model_graphcut over a LIST of gray volumes: consecutive volumes alternate over ``nb_streams`` CUDA
    streams with their own buffers, so the upload of volume i+1 and the download of volume i-1 overlap the kernels of volume i (as
    :func:`segment_images_batch` does for colour images).  Dictionaries with ``tLM*`` groups or ``meanGrad`` go through the stage
    functions, one volume after the other.

    :param int nb_classes: fit the class model per volume on the GPU (the reference's ``estim_class_model(features, nb_classes)``), or
    :param model_pipeline: a fitted model used for every volume; its ``classes_`` relabel the result
    :return list(tuple(ndarray,ndarray)): (segm int32 [D, H, W], segm_soft [D, H, W, K]) per volume, in input order
    """
    if (nb_classes is None) == (model_pipeline is None):
        raise ValueError('give either nb_classes (per-volume GMM) or model_pipeline')
    flags = _volume_flags(dict_features)
    if model_pipeline is None:
        if flags is None or not device_gmm_applicable(len(flags), nb_classes):
            def proba_fn(features):
                return estim_class_model(features, nb_classes, use_scaler=use_scaler).predict_proba(features)
            return [_segment_volume_stages(v, proba_fn, dict_features, spacing, sp_size, sp_regul, gc_regul) for v in list_volumes]
        model = _fit_model(nb_classes, use_scaler)
    else:
        model = _device_model(model_pipeline, len(flags)) if flags is not None else model_pipeline.predict_proba
    classes = getattr(model_pipeline, 'classes_', None)
    if flags is None:
        out = [_segment_volume_stages(v, model, dict_features, spacing, sp_size, sp_regul, gc_regul) for v in list_volumes]
        return [(segm if classes is None else np.asarray(classes)[segm], soft) for segm, soft in out]

    def run(eng, volume):
        return _run_resident(eng, lambda: _device_slic3d_features(eng, volume, dict_features, spacing, sp_size, sp_regul), model, gc_regul,
                             'model')

    def redo(idx):      # on the caller's stream with the grown table
        eng = get_engine()
        d_segm, d_soft = segment_resident_volume(eng.to_device(_supported_dtype(np.asarray(list_volumes[idx])), 'volume'), model,
                                                 dict_features, spacing, sp_size, sp_regul, gc_regul)
        (segm, soft), done = eng.download((d_segm, d_soft))
        done.synchronize()
        return segm.numpy(), soft.numpy()

    return _resident_batch(list_volumes, nb_streams, max_in_flight, run, redo, classes)


def segment_resident(d_image, model, dict_features, sp_size=30, sp_regul=0.2, gc_regul=1., gc_edge_type='model'):
    """ the same hot path with the image ALREADY on the device (a cuda tensor [H, W, 3]) and the results left
    there: returns (segm int32 [H, W], segm_soft float64 [H, W, K]) device tensors.  ``model`` is a callable
    proba_fn(features), a fitted model (or its bound ``predict_proba``) -- evaluated on the device when
    :func:`~.class_models.compile_model` supports it -- or ('fit', nb_classes, use_scaler, max_iter) for the GPU-fitted default GMM
    (``_fit_model`` gives the tuple of the other ``estim_model`` variants and of ``pca_coef``).
    The indices in ``segm`` are not mapped through the model's ``classes_``.  ``gc_edge_type`` is any edge type of
    ``graph_cuts.compute_edge_weights`` -- 'color' and 'features' weigh the edges on the device too --; an unknown name raises
    ValueError.
    Nothing here waits for the device, so the edge count of the graph cut is not checked against its table as the host-facing
    pipelines do: after the connectivity pass every superpixel is connected, the region graph of a 2-D map is planar with at most
    3N - 6 edges, and the table holds 8 per node of an upper bound of N. """
    model = _device_model(model, _resident_width(dict_features))
    return _run_resident_image(get_engine(), d_image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type)[:2]


def pipe_color2d_slic_features_model_graphcut(image, nb_classes, dict_features, sp_size=30, sp_regul=0.2, pca_coef=None,
                                              use_scaler=True, estim_model='GMM', gc_regul=1., gc_edge_type='model',
                                              debug_visual=None):
    """ complete pipeline: superpixels, features, class model estimated on this image, GraphCut
    (reference pipelines.py:46-110)

    :param ndarray image: input RGB image
    :param int nb_classes: number of classes to be segmented
    :param dict dict_features: {'color': [...], ...}
    :return tuple(ndarray,ndarray): segmentation [H, W] int32, soft segmentation [H, W, nb_classes] float64
    """
    logging.info('PIPELINE Superpixels-Features-GMM-GraphCut')
    nb_fts = native_feature_layout(dict_features)[1] if flags_are_resident(dict_features) else 10 ** 6
    if flags_are_resident(dict_features) and device_gmm_applicable(nb_fts, nb_classes, estim_model, pca_coef):
        model = _fit_model(nb_classes, use_scaler, estim_model, pca_coef)
    else:
        def model(features):
            return estim_class_model(features, nb_classes, estim_model, pca_coef, use_scaler).predict_proba(features)
    return _segment(image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type, debug_visual)


def estim_model_classes_group(list_images, nb_classes, dict_features, sp_size=30, sp_regul=0.2, use_scaler=True,
                              pca_coef=None, model_type='GMM', nb_workers=NB_WORKERS):
    """ one class model from the superpixel features of a sequence of images (reference pipelines.py:113-157);
    the per-image work that the reference spreads over a process pool runs back to back on the GPU

    :return tuple(model, list(ndarray)): fitted sklearn pipeline, list of per-image features
    """
    list_features = compute_features_batch(list_images, dict_features, sp_size=sp_size, sp_regul=sp_regul)
    features = np.nan_to_num(np.concatenate(tuple(list_features), axis=0))
    model = estim_class_model(features, nb_classes, model_type, pca_coef, use_scaler)
    return model, list_features


def segment_color2d_slic_features_model_graphcut(image, model_pipeline, dict_features, sp_size=30, sp_regul=0.2, gc_regul=1.,
                                                 gc_edge_type='model', debug_visual=None):
    """ complete pipeline with a given (already fitted) model (reference pipelines.py:160-241)

    :return tuple(ndarray,ndarray): segmentation [H, W], soft segmentation [H, W, K]
    """
    logging.info('PIPELINE Superpixels-Features-Model-GraphCut')
    classes = getattr(model_pipeline, 'classes_', None)
    model = model_pipeline.predict_proba
    if debug_visual is None and np.ndim(image) == 3 and gc_edge_type not in ('color', 'features'):
        model = _device_model(model, _resident_width(dict_features))
    return _segment(image, model, dict_features, sp_size, sp_regul, gc_regul, gc_edge_type, debug_visual, classes=classes)
