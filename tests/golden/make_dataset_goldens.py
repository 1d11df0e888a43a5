"""
Generate tests/golden/dataset_reference.npz by RUNNING THE REFERENCE'S imsegm/classification.py on the inputs of the doctests of its
training-set functions (:1027-1262) and on small sets for every balance type, seeded.

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_dataset_goldens.py

The reference is imported as make_classification_goldens.py does (real scikit-learn, numpy and scipy; inert stubs for the imports no
function called here touches).  Nothing of the reference is copied: this script calls it and stores the inputs and outputs.  Every value
is stored by ``pack``: arrays as npz arrays, lists of numbers as an array plus the Python type names of their items, dicts and tuples
as JSON structure with their keys and key types, so that a test can check types as well as values.  ``np_seed`` / ``py_seed`` are
the seeds of numpy's and Python's global RNGs set right before the call.
"""
import json
import os
import random
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_classification_goldens import import_reference  # noqa: E402


def main():
    clf = import_reference()
    warnings.simplefilter('ignore')
    arrays, cases = {}, []

    def pack(prefix, v):
        if isinstance(v, np.ndarray):
            arrays[prefix] = v
            return {'type': 'ndarray', 'key': prefix}
        if isinstance(v, dict):
            items = []
            for i, (k, x) in enumerate(v.items()):
                key = int(k) if isinstance(k, (int, np.integer)) else str(k)
                items.append([key, type(k).__name__, pack('%s/%d' % (prefix, i), x)])
            return {'type': 'dict', 'items': items}
        if isinstance(v, (list, tuple)):
            if all(isinstance(x, (int, float, np.integer, np.floating)) for x in v):
                arrays[prefix] = np.array(v)
                return {'type': type(v).__name__, 'key': prefix, 'elem': sorted({type(x).__name__ for x in v})}
            return {'type': type(v).__name__, 'items': [pack('%s/%d' % (prefix, i), x) for i, x in enumerate(v)]}
        return {'type': type(v).__name__, 'value': v.item() if isinstance(v, np.generic) else v}

    def add(func, name, args, kwargs=None, np_seed=None, py_seed=None):
        kwargs = kwargs or {}
        case = dict(name=name, func=func, kwargs=kwargs, np_seed=np_seed, py_seed=py_seed,
                    args=[pack('%s/in%d' % (name, i), a) for i, a in enumerate(args)])
        if np_seed is not None:
            np.random.seed(np_seed)
        if py_seed is not None:
            random.seed(py_seed)
        try:
            case['out'] = pack(name + '/out', getattr(clf, func)(*args, **kwargs))
        except Exception as err:                      # the type and message are what the test checks
            case['raises'] = [type(err).__name__, str(err)]
        cases.append(case)

    # the doctests of :1027-1262 (their inputs drawn as the doctests draw them)
    np.random.seed(0)
    fts, lbs = np.random.random((5, 2)), np.random.randint(0, 2, 5)
    add('shuffle_features_labels', 'doc_shuffle', [fts, lbs], np_seed=1)
    np.random.seed(0)
    add('down_sample_dict_features_random', 'doc_random', [{'a': np.random.random((100, 3))}, 5], py_seed=0)
    np.random.seed(0)
    add('down_sample_dict_features_kmean', 'doc_kmean', [{'a': np.random.random((100, 3))}, 5], np_seed=0)
    np.random.seed(0)
    add('down_sample_dict_features_unique', 'doc_unique', [{'a': np.random.random((100, 3))}])
    np.random.seed(0)
    fts, lbs = np.random.random((25, 3)), np.random.randint(0, 2, 25)
    for bt in ('random', 'unique', 'kmeans'):
        add('balance_dataset_by_', 'doc_balance_' + bt, [fts, lbs], {'balance_type': bt}, np_seed=0, py_seed=0)
    np.random.seed(0)
    d_fts = {'a': np.random.random((25, 3)), 'b': np.random.random((30, 3))}
    d_lbs = {'a': np.random.randint(0, 2, 25), 'b': np.random.randint(0, 2, 30)}
    add('convert_set_features_labels_2_dataset', 'doc_convert_set', [d_fts, d_lbs])

    # the plain conversions, with integer, float32 and empty blocks
    add('convert_dict_label_features_2_vectors', 'vectors_mixed', [{2: np.ones((2, 3)), 0: np.arange(3.)[None], 1: np.zeros((0, 3))}])
    add('convert_dict_label_features_2_vectors', 'vectors_int', [{0: np.arange(6).reshape(2, 3), 1: np.arange(3).reshape(1, 3)}])
    add('convert_dict_label_features_2_vectors', 'vectors_f32', [{5: np.ones((2, 2), np.float32) / 3}])
    add('convert_dict_label_features_2_vectors', 'vectors_empty', [{}])
    rng = np.random.RandomState(3)
    add('compose_dict_label_features', 'compose', [rng.rand(12, 2), np.array([3, 1, 3, 0, 1, 1, 3, 0, 0, 3, 1, 1])])
    add('compose_dict_label_features', 'compose_list', [rng.rand(5, 2).tolist(), [1, 0, 1, 1, 0]])
    add('shuffle_features_labels', 'shuffle_seeded', [rng.rand(9, 2), np.arange(9)], np_seed=5)
    add('shuffle_features_labels', 'shuffle_mismatch', [rng.rand(4, 2), np.arange(3)])

    # 'unique': rows that round together, -0.0 against 0.0, rows with NaN
    unq = np.array([[0.1234, 1.], [0.12341, 1.], [-0.0001, 2.], [0.0, 2.], [np.nan, 3.], [np.nan, 3.], [5., -1.], [0.1234, 0.9996]])
    add('unique_rows', 'unique_rows', [np.round(unq, 3)])
    add('down_sample_dict_features_unique', 'unique_quirks', [{7: unq, 1: unq[::-1].copy()}])

    # 'random' and 'kmeans' on imbalanced small sets; 'kmeans' on well separated blobs
    rng = np.random.RandomState(11)
    centres = rng.randn(6, 5) * 10
    lab = np.r_[np.zeros(90, int), np.ones(30, int), np.full(55, 2)]
    rng.shuffle(lab)
    blob = rng.randint(0, 6, len(lab))
    X = centres[blob] + rng.randn(len(lab), 5) * 0.5
    for bt in ('random', 'unique', 'kmeans', 'Kmeans', 'none'):
        add('balance_dataset_by_', 'balance_' + bt, [X, lab], {'balance_type': bt}, np_seed=4, py_seed=4)
    add('balance_dataset_by_', 'balance_kmeans_min', [X, lab], {'balance_type': 'kmeans', 'min_samples': 12}, np_seed=9)
    add('down_sample_dict_features_kmean', 'kmean_dict', [{0: X[:80], 1: X[80:110], 2: X[110:]}, 25], np_seed=2)

    # convert_set_features_labels_2_dataset with drop_labels=[-1] for each balance type
    imgs_fts, imgs_lbs = {}, {}
    for i, name in enumerate(('img_b', 'img_a', 'img_c')):
        n = 60 + 17 * i
        blob = rng.randint(0, 6, n)
        imgs_fts[name] = centres[blob] + rng.randn(n, 5) * 0.5
        imgs_lbs[name] = np.where(rng.rand(n) < 0.15, -1, (rng.rand(n) < 0.35 + 0.1 * i).astype(int)).astype(float)
    for bt in (None, 'random', 'unique', 'kmeans'):
        add('convert_set_features_labels_2_dataset', 'set_%s' % bt, [imgs_fts, imgs_lbs], {'drop_labels': [-1], 'balance_type': bt},
            np_seed=6, py_seed=6)
    add('convert_set_features_labels_2_dataset', 'set_missing', [imgs_fts, {'img_a': imgs_lbs['img_a']}])

    np.savez_compressed(os.path.join(HERE, 'dataset_reference.npz'), cases=np.array(json.dumps(cases)), **arrays)
    print('%d cases, %d arrays' % (len(cases), len(arrays)))


if __name__ == '__main__':
    main()
