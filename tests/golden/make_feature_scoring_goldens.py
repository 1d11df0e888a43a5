"""
Generate tests/golden/feature_scoring_reference.npz by RUNNING THE REFERENCE'S ``feature_scoring_selection`` (imsegm/classification.py)
on its two doctest cases, on given feature names, on list input and on a multi-class table with a constant column.

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_feature_scoring_goldens.py

The reference builds its table with ``DataFrame.append``, which pandas 2 removed; this script gives pandas a ``DataFrame.append`` that
concatenates one row, and otherwise imports the reference as make_classification_goldens.py does.  Nothing of the reference is copied:
per case the file stores the inputs, the indices, the table's columns, index labels and values, and the CSV text it writes.
"""
import json
import os
import sys
import tempfile
import warnings

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_classification_goldens import import_reference  # noqa: E402


def _append(self, other, ignore_index=False):
    return pd.concat([self, pd.DataFrame([other])], ignore_index=ignore_index)


def cases():
    """(name, features, labels, names, as_lists)"""
    from sklearn.datasets import make_classification
    fts, lbs = make_classification(n_samples=250, n_features=5, n_informative=3, n_redundant=0, n_repeated=0, n_classes=2,
                                   random_state=0, shuffle=False)
    yield 'doctest', fts.copy(), lbs, None, False
    const = fts.copy()
    const[:, 2] = 1
    yield 'doctest_constant_lists', const, lbs, None, True
    yield 'names', fts.copy(), lbs, ['r', 'g', 'b', 'h', 's'], False
    yield 'short_names', fts.copy(), lbs, ['r', 'g'], False
    rng = np.random.RandomState(7)
    small = np.round(rng.normal(size=(60, 3)), 2)
    yield 'lists', small, (small[:, 0] > 0).astype(int), None, True
    multi, mlbs = make_classification(n_samples=400, n_features=8, n_informative=4, n_redundant=1, n_classes=4, random_state=3)
    multi[:, 5] = -2.5
    yield 'multiclass_constant', multi, mlbs, ['f%d' % i for i in range(8)], False


def main():
    clf = import_reference()
    pd.DataFrame.append = _append
    warnings.simplefilter('ignore')
    arrays, meta = {}, []
    for name, fts, lbs, names, as_lists in cases():
        with tempfile.TemporaryDirectory() as path_out:
            indices, df = clf.feature_scoring_selection(fts.tolist() if as_lists else fts, lbs.tolist() if as_lists else lbs,
                                                        names=names, path_out=path_out)
            csv = open(os.path.join(path_out, clf.NAME_CSV_FEATURES_SELECT)).read()
        arrays[name + '/features'] = np.asarray(fts)
        arrays[name + '/labels'] = np.asarray(lbs)
        arrays[name + '/indices'] = np.asarray(indices)
        arrays[name + '/values'] = df.to_numpy(dtype=np.float64)
        meta.append(dict(name=name, names=names, as_lists=as_lists, columns=[str(c) for c in df.columns],
                         index=[str(i) for i in df.index], index_name=df.index.name, csv=csv))
    arrays['meta'] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(HERE, 'feature_scoring_reference.npz'), **arrays)
    print('wrote %d cases' % len(meta))


if __name__ == '__main__':
    main()
