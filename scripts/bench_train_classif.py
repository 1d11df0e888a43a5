#!/usr/bin/env python
"""
bench_train_classif.py -- supervised training of the superpixel classifier (the reference's train_classif_color2d_slic_features):
pipelines.train_classif_images_batch against the composition of the stage functions it replaces.  Prints one JSON line.

    python scripts/bench_train_classif.py [--images 16] [--steps 1] [--warmup 1] [--sets d9,d189]

The data: --images config-2 images (bench.synth_image, 2048 x 2048) annotated with the Voronoi class map of
scripts/bench_shared_model.synth_classes, SLIC as bench.py, label purity 0.9, feature_balance 'unique', the default 'RandForest', with
colour mean / std / energy (D = 9) and with colour + full Leung-Malik statistics (D = 189).  Per feature set:
- ``driver_s``: train_classif_images_batch end to end (host clock; the call ends in host reads);
- ``composition_s``: per image the data step as it was before the device labels (compute_color2d_superpixels_features, the dense
  histogram of histogram_regions_labels_norm and the host argmax / purity), convert_set_features_labels_2_dataset with the host
  'unique' balancing, and create_classif_search_train_export, on the same seed;
- ``stages``: the same three stages of both (features + labels, unique rows, classifier fit), host clock;
- ``kernels_ms``: isb_superpixel_train_labels and isb_unique_rows_rounded alone on the first image's device data (CUDA events, median
  of 20 launches);
- ``parity``: the two training sets are equal and every fitted tree's arrays are equal;
- the card's name and power limit (nvidia-smi), read in the same run.
"""
import argparse
import json
import os
import random
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_shared_model import card_info, synth_classes  # noqa: E402

FEATURE_SETS = {
    'd9': {'color': ['mean', 'std', 'energy']},
    'd189': {'color': ['mean', 'std', 'energy'], 'tLM': ['mean', 'std', 'energy']},
}
PURITY = 0.9


def stage_labels(image, annot, features):
    """the data step as the stage functions composed it: superpixels and features, then the label of the dense histogram"""
    from pyimsegm_b200 import pipelines
    from pyimsegm_b200.labeling import histogram_regions_labels_norm
    annot = np.asarray(annot).astype(int)
    slic, fts = pipelines.compute_color2d_superpixels_features(image, features, sp_size=bench.SP_SIZE, sp_regul=bench.SP_REGUL)
    neg_label = int(np.max(annot)) + 1 if np.any(annot < 0) else None
    if neg_label is not None:
        annot = np.where(annot < 0, neg_label, annot)
    hist = histogram_regions_labels_norm(slic, annot)
    labels = np.argmax(hist, axis=1)
    if neg_label is not None:
        labels[labels == neg_label] = -1
    labels[np.max(hist, axis=1) < PURITY] = -1
    return slic, fts, labels


def composition(images, annots, features):
    from pyimsegm_b200 import classification as cls
    t = {}
    t0 = time.perf_counter()
    data = [stage_labels(im, an, features) for im, an in zip(images, annots)]
    t['features_labels'] = time.perf_counter() - t0
    t0 = time.perf_counter()
    X, y, sizes = cls.convert_set_features_labels_2_dataset(dict(enumerate(d[1] for d in data)), dict(enumerate(d[2] for d in data)),
                                                            balance_type='unique', drop_labels=[-1])
    X = np.nan_to_num(X)
    t['unique_rows'] = time.perf_counter() - t0
    t0 = time.perf_counter()
    cv = cls.CrossValidateGroups(sizes, nb_hold_out=2) if len(sizes) > 10 else 10
    classif, _ = cls.create_classif_search_train_export('RandForest', X, y, pca_coef=None, cross_val=cv, nb_search_iter=1, nb_workers=1)
    t['fit'] = time.perf_counter() - t0
    return classif, (X, y), t


def driver(images, annots, features):
    """train_classif_images_batch with its create_classif_search_train_export timed apart (and its training set kept)"""
    from pyimsegm_b200 import classification as cls
    from pyimsegm_b200 import pipelines
    fit, seen = cls.create_classif_search_train_export, {}

    def timed_fit(*args, **kw):
        seen['set'] = (args[1], args[2])
        t0 = time.perf_counter()
        out = fit(*args, **kw)
        seen['fit'] = time.perf_counter() - t0
        return out

    cls.create_classif_search_train_export = timed_fit
    try:
        t0 = time.perf_counter()
        classif = pipelines.train_classif_images_batch(images, annots, features, sp_size=bench.SP_SIZE, sp_regul=bench.SP_REGUL,
                                                       label_purity=PURITY)[0]
        total = time.perf_counter() - t0
    finally:
        cls.create_classif_search_train_export = fit
    return classif, seen['set'], total, seen['fit']


def data_step(images, annots, features):
    """the driver's data step alone (features + labels + unique rows on the device, over streams): seconds"""
    from pyimsegm_b200 import pipelines
    t0 = time.perf_counter()
    pipelines._train_data(images, [pipelines.train_annotation(im, an) for im, an in zip(images, annots)], features, bench.SP_SIZE,
                          bench.SP_REGUL, PURITY, True, 3, 6)
    return time.perf_counter() - t0


def kernels_alone(image, annot, features):
    import torch
    from pyimsegm_b200 import pipelines
    from pyimsegm_b200.descriptors import native_feature_layout
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    res = pipelines._device_slic_features(eng, image, features, bench.SP_SIZE, bench.SP_REGUL)
    d_annot = eng.to_device(pipelines.train_annotation(image, annot))
    D = native_feature_layout(features)[1]
    d_x = eng.nan_free_table(res.d_feat, D, res.d_n_labels)
    d_lab = eng.train_labels(res.d_seg, res.nb_bound, d_annot, PURITY, d_n=res.d_n_labels)
    out = {}
    for name, fn in (('train_labels', lambda: eng.train_labels(res.d_seg, res.nb_bound, d_annot, PURITY, d_n=res.d_n_labels)),
                     ('unique_rows', lambda: eng.unique_rows(d_x, d_lab, D, d_n=res.d_n_labels))):
        fn()
        ts = []
        for _ in range(20):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = round(float(np.median(ts)), 4)
    out['superpixels'] = int(eng.to_host(res.d_n_labels)[0])
    return out


def same_trees(a, b):
    ta, tb = a.steps[-1][1].estimators_, b.steps[-1][1].estimators_
    return len(ta) == len(tb) and all(np.array_equal(getattr(x.tree_, f), getattr(y.tree_, f)) for x, y in zip(ta, tb)
                                      for f in ('feature', 'threshold', 'children_left', 'children_right', 'value'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=16)
    ap.add_argument('--steps', type=int, default=1)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sets', default='d9,d189')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    warnings.simplefilter('ignore')
    seeds = [6000 + i for i in range(args.images)]
    images = [bench.synth_image(s) for s in seeds]
    annots = [synth_classes(s) for s in seeds]
    result = {'card': card_info(), 'images': args.images, 'shape': list(images[0].shape[:2]), 'sets': {}}
    for set_name in args.sets.split(','):
        features = FEATURE_SETS[set_name]
        entry = {'D': None, 'driver_s': [], 'composition_s': [], 'stages': {'driver': [], 'composition': []}}
        parity = True
        for step in range(args.warmup + args.steps):
            random.seed(step)
            np.random.seed(step)
            clf_d, set_d, t_d, fit_d = driver(images, annots, features)
            t_data = data_step(images, annots, features)
            random.seed(step)
            np.random.seed(step)
            t0 = time.perf_counter()
            clf_c, set_c, t_c = composition(images, annots, features)
            t_comp = time.perf_counter() - t0
            parity = parity and np.array_equal(set_d[0], set_c[0]) and np.array_equal(set_d[1], set_c[1]) and same_trees(clf_d, clf_c)
            if step >= args.warmup:
                entry['D'] = int(set_d[0].shape[1])
                entry['rows'] = int(len(set_d[1]))
                entry['driver_s'].append(round(t_d, 3))
                entry['composition_s'].append(round(t_comp, 3))
                entry['stages']['driver'].append({'features_labels_unique': round(t_data, 3), 'fit': round(fit_d, 3)})
                entry['stages']['composition'].append({k: round(v, 3) for k, v in t_c.items()})
        entry['kernels_ms'] = kernels_alone(images[0], annots[0], features)
        entry['parity'] = bool(parity)
        result['sets'][set_name] = entry
    result['parity'] = all(e['parity'] for e in result['sets'].values())
    print(json.dumps(result))


if __name__ == '__main__':
    main()
