#!/usr/bin/env python
"""
bench_cross_validation.py -- the cross-validation of the reference's supervised experiment (``load_train_classifier``):
``eval_classif_cross_val_scores`` with the four METRIC_SCORING scorings and ``eval_classif_cross_val_roc`` of
``create_clf_pipeline('RandForest', None)`` over ``CrossValidateGroups(sizes, 2)``, i.e. 8 folds x (4 + 1) = 40 forests of 20 trees.
Prints one JSON line.

    python scripts/bench_cross_validation.py [--steps 3] [--warmup 1]

The data: the labelled superpixels of 16 config-2 images (as scripts/bench_forest_fit.py), balanced per image with 'random', with
colour mean / std / energy (D = 9) and with colour + full Leung-Malik statistics (D = 189).  Per feature set, the wall time of
scores + ROC (median / min / max over --steps) on three routes:
- grouped: every forest of the scores in one grouped device fit, those of the ROC in another (forest_fit.TreeBatch);
- per fold: the same with one fit_tree_model call per fold (classification._fit_folds replaced here);
- scikit-learn: its own cross_val_score and fit per fold (one run);
the kernel time of the grouped route (torch.profiler, a separate run), the levels built, whether the grouped and per-fold routes gave
identical score DataFrames (and ROC / AUC), and the card's name, power limit and maximum SM clock, read in the same run.  There is no CPU fallback:
without a CUDA device the script fails.
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

from bench_forest_fit import FEATURE_SETS, image_sets, stats  # noqa: E402
from bench_shared_model import card_info  # noqa: E402


def per_fold_fits(classif, features, labels, fold_lists, catch=True):
    """classification._fit_folds with one fit_tree_model call per fold (through _fit_pipeline)"""
    from sklearn.base import clone
    from pyimsegm_b200 import classification as clf
    out = []
    for folds in fold_lists:
        out.append([clf._fit_pipeline(clone(classif), features[train], labels[train]) for train, _ in folds])
    return out


def run(steps, warmup):
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    from pyimsegm_b200 import classification as clf
    from pyimsegm_b200 import forest_fit
    grouped_fit_folds = clf._fit_folds
    levels = []
    device_fit = forest_fit._fit_arrays_groups

    def counting(*args):
        trees = device_fit(*args)
        levels.append(max(t['n_levels'] for t in trees))
        return trees
    forest_fit._fit_arrays_groups = counting

    def both(X, y, sizes, seed):
        classif = clf.create_clf_pipeline('RandForest', None)
        cv = clf.CrossValidateGroups(sizes, 2)
        np.random.seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        df = clf.eval_classif_cross_val_scores('RandForest', classif, X, y, cross_val=cv)
        roc, auc = clf.eval_classif_cross_val_roc('RandForest', classif, X, y, cv)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, df, roc, auc

    out = {'metric': 'cross_validation', 'cpu_count': os.cpu_count(), 'card': card_info(), 'sets': {}}
    warnings.simplefilter('ignore')
    for name, feats in FEATURE_SETS.items():
        random.seed(0)
        X, y, sizes = clf.convert_set_features_labels_2_dataset(*image_sets(range(16), feats), drop_labels=[-1], balance_type='random')
        n_folds = len(clf.CrossValidateGroups(sizes, 2))
        res = {}
        for route, fit_folds in (('grouped', grouped_fit_folds), ('per_fold', per_fold_fits)):
            clf._fit_folds = fit_folds
            wall = []
            for i in range(warmup + steps):
                t, df, roc, auc = both(X, y, sizes, seed=0)
                if i >= warmup:
                    wall.append(t)
            res[route] = (wall, df, roc, auc)
        clf._fit_folds = grouped_fit_folds
        del levels[:]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            both(X, y, sizes, seed=0)
        kern = [(e.key, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0]
        kernel_s = sum(t for _, t in kern) / 1e6
        forest_fit._fit_arrays_groups = device_fit
        orig = clf._device_folds
        clf._device_folds = lambda c: False
        t_host, df_h, _, auc_h = both(X, y, sizes, seed=0)
        clf._device_folds = orig
        forest_fit._fit_arrays_groups = counting
        g, p = res['grouped'], res['per_fold']
        out['sets'][name] = {
            'rows': int(len(X)), 'features': int(X.shape[1]), 'classes': int(len(np.unique(y))), 'images': len(sizes), 'folds': n_folds,
            'forests': n_folds * (len(clf.METRIC_SCORING) + 1),
            'wall_s': {'grouped': stats(g[0]), 'per_fold': stats(p[0]), 'scikit-learn': round(t_host, 3)},
            'speedup_grouped_vs_per_fold': round(float(np.median(p[0]) / np.median(g[0])), 2),
            'speedup_grouped_vs_scikit-learn': round(float(t_host / np.median(g[0])), 2),
            'grouped_kernel_time_s': round(kernel_s, 4), 'levels_per_grouped_call': [int(v) for v in levels],
            # the ROC is compared too, but the default forest's predict_proba (n_jobs=-1) adds its trees in thread order
            'grouped_equals_per_fold': {'scores': bool(g[1].equals(p[1])), 'roc_and_auc': bool(g[2].equals(p[2]) and g[3] == p[3])},
            'mean_scores': {'grouped': {k: round(float(v), 4) for k, v in g[1].mean().items()},
                            'scikit-learn': {k: round(float(v), 4) for k, v in df_h.mean().items()}},
            'auc': {'grouped': round(float(g[3]), 4), 'scikit-learn': round(float(auc_h), 4)},
        }
    forest_fit._fit_arrays_groups = device_fit
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    print(json.dumps(run(args.steps, args.warmup)))


if __name__ == '__main__':
    main()
