"""
Generate tests/golden/classification_reference.npz by RUNNING THE REFERENCE'S imsegm/classification.py on the inputs of the doctests
of its scoring functions and on a few more cases (drop labels, relabelling, negative labels, the [-1, 0] pair).

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_classification_goldens.py

scikit-learn, pandas and scipy are the real packages (``scipy.interp`` is read as ``np.interp``); the reference's other imports that
are not installable here (scikit-image, nibabel, tqdm, matplotlib, yaml, gco, the OLE readers) are inert stubs, which no function
called below touches.  Nothing of the reference is copied: this script calls it and stores the inputs and, as one JSON string, the
outputs (dicts, DataFrame rows as dicts, tuples; NaN as NaN, None as null) or the name of the exception raised.
"""
import importlib
import json
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ['IMSEGM_REFERENCE']


def import_reference():
    import scipy
    for name, val in (('int', int), ('product', np.prod), ('float', float), ('bool', bool)):
        if not hasattr(np, name):       # NumPy-2 removed aliases the reference still uses
            setattr(np, name, val)
    if not hasattr(scipy, 'interp'):
        scipy.interp = np.interp

    class Stub(types.ModuleType):
        __path__ = []

        def __getattr__(self, k):
            if k.startswith('__'):
                raise AttributeError(k)
            m = Stub(self.__name__ + '.' + k)
            setattr(self, k, m)
            sys.modules[self.__name__ + '.' + k] = m
            return m

        def __call__(self, *a, **k):
            return Stub('call')

        def __getitem__(self, k):
            return 'agg'

    for root in ('skimage', 'nibabel', 'tqdm', 'matplotlib', 'olefile', 'OleFileIO_PL', 'yaml', 'gco'):
        sys.modules.setdefault(root, Stub(root))
    for sub in ('skimage.color', 'skimage.exposure', 'skimage.io', 'skimage.measure', 'skimage.morphology', 'skimage.filters',
                'skimage.segmentation', 'skimage.draw', 'skimage.transform', 'matplotlib.pyplot', 'tqdm.auto'):
        root, leaf = sub.split('.', 1)
        getattr(sys.modules[root], leaf)
    sys.path.insert(0, REF)
    return importlib.import_module('imsegm.classification')


def plain(v):
    """JSON-able form of an output"""
    if isinstance(v, dict):
        return {str(k): plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [plain(x) for x in v]
    if isinstance(v, np.ndarray):
        return plain(v.tolist())
    if isinstance(v, (np.integer, )):
        return int(v)
    if isinstance(v, (np.floating, float)):
        return float(v)
    return v


def main():
    clf = import_reference()
    warnings.simplefilter('ignore')
    arrays, cases = {}, []

    def add(func, name, inputs, **kwargs):
        """one call of func on the named input arrays"""
        for key, arr in inputs.items():
            arrays[key] = arr
        args = [arrays[k] for k in inputs]
        if func == 'compute_classif_stat_segm_annot':
            args = [(args[0], args[1], name)]
        try:
            out = getattr(clf, func)(*args, **kwargs)
            if func == 'compute_stat_per_image':
                out = {str(idx): row.to_dict() for idx, row in out.iterrows()}
            res = {'value': plain(out)}
        except Exception as err:                      # the type is what the test checks
            res = {'raises': type(err).__name__}
        cases.append(dict(name=name, func=func, inputs=list(inputs), kwargs=kwargs, **res))

    np.random.seed(0)
    y_true = np.random.randint(0, 3, 25) * 2
    y_pred = np.random.randint(0, 2, 25) * 2
    add('compute_classif_metrics', 'metrics_true_true', {'m_true': y_true, 'm_true2': y_true})
    add('compute_classif_metrics', 'metrics_true_pred', {'m_true': y_true, 'm_pred': y_pred})
    add('compute_classif_metrics', 'metrics_pred_pred', {'m_pred': y_pred, 'm_pred2': y_pred})
    add('compute_classif_metrics', 'metrics_averages', {'m_true': y_true, 'm_pred': y_pred},
        metric_averages=['macro', 'weighted', 'micro', 'binary', 'samples'])
    add('compute_classif_metrics', 'metrics_neg_quirk', {'q_true': np.array([-1, 0, 0, -1, 0]), 'q_pred': np.array([0, 0, -1, -1, 0])})

    np.random.seed(0)
    annot = np.random.randint(0, 2, (5, 10))
    segm = np.random.randint(0, 2, (5, 10))
    add('compute_classif_stat_segm_annot', 'stat_same', {'s_annot': annot, 's_annot2': annot}, relabel=True, drop_labels=[5])
    add('compute_classif_stat_segm_annot', 'stat_relabel', {'s_annot': annot, 's_segm': segm}, relabel=True, drop_labels=[5])
    add('compute_classif_stat_segm_annot', 'stat_drop0', {'s_annot': annot, 's_segm1': segm + 1}, relabel=False, drop_labels=[0])

    np.random.seed(0)
    img_true = np.random.randint(0, 3, (50, 100))
    img_pred = np.random.randint(0, 2, (50, 100))
    add('compute_stat_per_image', 'per_image_same', {'p_true': [img_true], 'p_true2': [img_true]}, relabel=True)
    add('compute_stat_per_image', 'per_image_drop', {'p_pred': [img_pred], 'p_true': [img_true]}, drop_labels=[-1])

    np.random.seed(0)
    annot = np.random.randint(0, 2, (5, 7)) * 9
    segm = np.random.randint(0, 2, (5, 7)) * 9
    add('compute_tp_tn_fp_fn', 'tp_same', {'t_annot': annot, 't_annot2': annot})
    add('compute_tp_tn_fp_fn', 'tp_segm', {'t_annot': annot, 't_segm': segm})
    add('compute_tp_tn_fp_fn', 'tp_ones', {'t_annot': annot, 't_ones': np.ones((5, 7))})
    add('compute_tp_tn_fp_fn', 'tp_zeros', {'t_zeros': np.zeros((5, 7)), 't_zeros2': np.zeros((5, 7))})

    np.random.seed(0)
    annot = np.random.randint(0, 2, (50, 75)) * 3
    segm = np.random.randint(0, 2, (50, 75)) * 3
    for func in ('compute_metric_fpfn_tpfn', 'compute_metric_tpfp_tpfn'):
        add(func, func + '_segm', {'r_annot': annot, 'r_segm': segm})
        add(func, func + '_same', {'r_annot': annot, 'r_annot2': annot})
        add(func, func + '_ones', {'r_annot': annot, 'r_ones': np.ones((50, 75))})
        add(func, func + '_zeros', {'r_annot': annot, 'r_zeros': np.zeros((50, 75))})

    rng = np.random.RandomState(7)
    a4 = rng.randint(0, 4, (40, 60))
    s4 = (a4 + (rng.rand(40, 60) < 0.2) * rng.randint(1, 4, (40, 60))) % 4 * 3 + 1
    add('compute_classif_stat_segm_annot', 'x_relabel4', {'x_annot': a4, 'x_segm': s4}, relabel=True)
    add('compute_classif_stat_segm_annot', 'x_drop', {'x_annot': a4, 'x_segm': s4}, drop_labels=[0, 7])
    neg = a4 - 1
    add('compute_classif_stat_segm_annot', 'x_negative', {'x_neg': neg, 'x_segm_neg': s4 - 5})
    add('compute_classif_stat_segm_annot', 'x_negative_drop', {'x_neg': neg, 'x_segm_neg': s4 - 5}, drop_labels=[-1])
    add('compute_classif_stat_segm_annot', 'x_quirk', {'q_true2': np.array([[-1, 0], [0, -1]]), 'q_pred2': np.array([[0, 0], [-1, 0]])})
    add('compute_classif_stat_segm_annot', 'x_all_dropped', {'x_annot': a4, 'x_segm': s4}, drop_labels=[0, 1, 2, 3])

    arrays = {k: np.asarray(v) for k, v in arrays.items()}
    np.savez_compressed(os.path.join(HERE, 'classification_reference.npz'), cases=np.array(json.dumps(cases)), **arrays)
    print('%d cases, %d arrays' % (len(cases), len(arrays)))


if __name__ == '__main__':
    main()
