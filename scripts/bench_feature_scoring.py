"""
Benchmark of ``classification.feature_scoring_selection`` (the reference's feature ranking: ``ExtraTreesClassifier(n_estimators=125,
random_state=0)`` importances plus three scikit-learn scores) on seeded superpixel-like training tables: n rows of K classes, each
class a cloud of its own around a per-class centre with a per-feature spread, D = 15 (the colour feature set) and D = 189 (colour +
Leung-Malik texture, config 3).

Per table it times, after warm-up and with a device synchronise:
  - ``feature_scoring_selection`` on the device (the extra-trees fit of ``csrc/extra_trees_fit.cu`` plus the host scores);
  - the device fit alone (``forest_fit._fit_arrays_extra``), also at each ``--small-rows`` value (the warp-path threshold);
  - the reference's route on the same host: scikit-learn's ``ExtraTreesClassifier(n_estimators=125, random_state=0).fit`` with
    ``n_jobs=None`` (one core), all 125 trees, and its three scores;
and checks that the device and scikit-learn importances are bit-equal.  Prints one JSON line with the card's name and power limit,
read in the same run.  There is no CPU fallback: without a CUDA device the script stops.

    python scripts/bench_feature_scoring.py --rows 150000 --dims 15 189 --steps 3 --warmup 1
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_shared_model import card_info  # noqa: E402


def table(n, D, K, seed=0):
    """superpixel-like features: K classes of unequal size, each around its own centre, with a per-feature spread"""
    rng = np.random.RandomState(seed)
    sizes = rng.dirichlet(np.full(K, 2.0)) * n
    labels = np.repeat(np.arange(K), np.diff(np.round(np.concatenate([[0], np.cumsum(sizes)])).astype(int)))[:n]
    labels = np.concatenate([labels, np.full(n - len(labels), K - 1)]).astype(int)
    centres = rng.uniform(0, 1, (K, D))
    spread = rng.uniform(0.5, 2.0, D)
    X = centres[labels] + rng.normal(size=(n, D)) * spread
    perm = rng.permutation(n)
    return X[perm], labels[perm]


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times, out = [], None
    for _ in range(steps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return times, out


def stats(v):
    return {'median': round(float(np.median(v)), 4), 'min': round(float(np.min(v)), 4), 'max': round(float(np.max(v)), 4)}


def run(n, dims, K, steps, warmup, small_rows, sklearn):
    import torch
    assert torch.cuda.is_available(), 'the benchmark needs a CUDA device (there is no CPU fallback)'
    from sklearn import feature_selection
    from sklearn.ensemble import ExtraTreesClassifier
    from pyimsegm_b200 import classification as clf
    from pyimsegm_b200 import forest_fit
    warnings.simplefilter('ignore')
    out = {'benchmark': 'feature_scoring_selection', 'card': card_info(), 'rows': n, 'classes': K, 'trees': 125, 'sets': {}}
    for D in dims:
        X, y = table(n, D, K, seed=D)
        res = {'features': D}
        t_api, (_, df) = timed(lambda: clf.feature_scoring_selection(X, y), steps, warmup)
        res['device_feature_scoring_s'] = stats(t_api)
        prep = forest_fit._prepare(ExtraTreesClassifier(n_estimators=125, random_state=0), X, y, admit=forest_fit._supported_extra)
        states = forest_fit._rand_r_states(prep.seeds)

        def fit(s=0):
            return forest_fit._fit_arrays_extra(prep.X, prep.y, prep.K, prep.counts, states, prep.max_features, prep.mss, prep.msl,
                                                prep.max_depth, prep.mid, small_rows=s)
        t_fit, trees = timed(fit, steps, warmup)
        res['device_fit_s'] = stats(t_fit)
        res['nodes_per_tree'] = int(np.mean([t['node_count'] for t in trees]))
        # one CTA builds a tree's nodes one after another, and the trees run side by side: fit time over one tree's nodes
        res['device_fit_us_per_node'] = round(float(np.median(t_fit)) * 1e6 / res['nodes_per_tree'], 3)
        res['device_fit_by_small_rows_s'] = {str(s): stats(timed(lambda: fit(s), steps, 1)[0]) for s in small_rows}
        if sklearn:
            t0 = time.perf_counter()
            ref = ExtraTreesClassifier(n_estimators=125, random_state=0).fit(X, y)
            t_sk_fit = time.perf_counter() - t0
            feature_selection.f_regression(X, y)
            feature_selection.SelectKBest(feature_selection.f_classif, k='all').fit(X, y)
            feature_selection.VarianceThreshold().fit(X, y)
            res['scikit-learn_fit_s'] = round(t_sk_fit, 3)
            res['scikit-learn_feature_scoring_s'] = round(time.perf_counter() - t0, 3)
            res['importances_bit_equal'] = df['ExtTree'].to_numpy().tobytes() == ref.feature_importances_.tobytes()
            res['speedup_feature_scoring'] = round(res['scikit-learn_feature_scoring_s'] / float(np.median(t_api)), 1)
        else:
            res['scikit-learn_fit_s'] = 'not measured'
        out['sets']['D%d' % D] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=150000)
    ap.add_argument('--dims', type=int, nargs='+', default=[15, 189])
    ap.add_argument('--classes', type=int, default=4)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--small-rows', type=int, nargs='*', default=[16, 32, 64, 128])
    ap.add_argument('--no-sklearn', action='store_true', help='skip the scikit-learn timing')
    args = ap.parse_args()
    print(json.dumps(run(args.rows, args.dims, args.classes, args.steps, args.warmup, args.small_rows, not args.no_sklearn)))


if __name__ == '__main__':
    main()
