"""
The reference's ``imsegm/classification.py``: the metrics between annotations and segmentations, the preparation of class-balanced
training sets, the classifiers, their cross-validation and the feature scoring.

Every number comes from one contingency table -- the pixels of every (annotation value, segmentation value) pair after the
``drop_labels`` mask -- counted on the device (``csrc/classification.cu``, one upload of the two maps and three passes over them).
Everything else runs on the host over the table's nonzero cells, never over the pixels again: the confusion matrix, the accuracy,
the adjusted Rand score (scikit-learn's pair-confusion formula in integers), precision / recall / F1 / support (scikit-learn's own
``precision_recall_fscore_support`` on the cells weighted by their counts, which gives the same float64 divisions, warnings and
exceptions as on the pixel arrays), the ``relabel=True`` table of ``labeling.relabel_max_overlap_unique`` and the binary ratios.
There is no CPU fallback.

Label maps are integer or bool arrays of any shape; float arrays holding integers are cast on the host, other floats raise the
``ValueError`` scikit-learn raises for continuous targets.  The values of a map of 32 or 64 bits must span fewer than 2^26 values
(``NotImplementedError`` above), and a table of more than 2^28 cells raises ``MemoryError``.

Behaviour of the reference that is kept:

- With two or fewer distinct labels, ``compute_classif_metrics`` renumbers them as the reference's ``relabel_sequential`` does,
  including its wrap of a negative label into the end of its look-up table, so -1 and 0 become one class:
  ``compute_classif_metrics([-1, 0, 0, -1, 0], [0, 0, -1, -1, 0])`` has accuracy 1.0 and confusion ``[[5]]``.  In that case float
  maps raise ``TypeError`` (the reference sizes its table with a float), and so does ``relabel=True`` on float maps.
- An average that scikit-learn rejects (``'binary'`` on more than two labels, ``'samples'``) gives -1 for its four entries.

Differences from the reference:

- Bool maps count as 0 / 1 integers; the reference's ``relabel_sequential`` indexes with them as masks and raises ``IndexError``.
- ``relabel=True`` keeps negative labels as ``labeling.relabel_max_overlap_unique`` of this package does.
- ``compute_stat_per_image`` runs the pairs one after the other on the device (the upload of a pair overlaps the counting of the
  previous one) and ignores ``nb_workers``; it shows no progress bar.

The training sets: per-image superpixel features and labels into one class-balanced set (``compose_dict_label_features`` ..
``convert_set_features_labels_2_dataset``).  ``balance_type='kmeans'`` runs scikit-learn's ``KMeans(init='random', n_init=3,
max_iter=5)`` of every larger class on the device (``csrc/kmeans_sample.cu``); ``'random'`` and ``'unique'`` stay on the host with
the reference's exact ``random`` / numpy semantics.  The k-means follows scikit-learn 1.9's ``fit``: the features centred on their
column mean, ``tol = mean(var(X, axis=0)) * 1e-4``, the starting rows of the three runs drawn in order from numpy's global RNG (so a
given ``np.random.seed`` gives scikit-learn's starts), Lloyd sweeps on the device with the host relocating empty clusters as
``_relocate_empty_clusters_dense`` does, the best run by scikit-learn's rule, and its ``ConvergenceWarning``.  Then the row nearest
to each centre.  The labels come from ``|c|^2 - 2 x.c`` in float64 as scikit-learn's, and the nearest rows from exact squared
differences, so the selected rows can differ from scikit-learn's only where two distances agree to within rounding.  Features are
clustered in float64 (scikit-learn clusters float32 features in float32), with at most 256 columns (``NotImplementedError``
above).

The classifiers: the reference's zoo (``create_classifiers``), pipelines, parameter grids and distributions, searches, and saving and
loading.  ``create_classif_search_train_export`` fits the final pipeline's StandardScaler and PCA on the host with scikit-learn, casts
the transformed features to float32 and fits a ``'RandForest'`` or ``'DecTree'`` classifier on the device (``forest_fit.fit_tree_model``,
``csrc/forest_fit.cu``): exact splits with scikit-learn 1.9's rules and its bootstrap draws, the features each node draws differing
(see ``forest_fit``).  The other classifiers, parameters the device does not compute, and the parameter search itself
(``GridSearchCV`` / ``RandomizedSearchCV``) stay on scikit-learn; after a search the refit of the best pipeline goes to the device.

The cross-validation: the reference's fold generators (``HoldOut``, ``CrossValidate``, ``CrossValidateGroups``; pure host code), and
``eval_classif_cross_val_scores`` / ``eval_classif_cross_val_roc`` with the reference's folds, relabelling, per-scoring error handling
and files.  For a ``'RandForest'`` or ``'DecTree'`` classifier (alone or ending a Pipeline) the transforms are fitted fold by fold on
the host and the forests of every (scoring, fold) pair are built in one grouped device fit (``forest_fit.TreeBatch``,
``isb_forest_fit_groups``); each tree is the one ``fit_tree_model`` builds for that fold alone, the global RNG is consumed in
scikit-learn's order, and the scores and ROC are scikit-learn's scorers and ``roc_curve`` on the fitted pipelines.  Other classifiers
go through scikit-learn's ``cross_val_score``.

The feature scoring: ``feature_scoring_selection`` ranks the features by the importances of ``ExtraTreesClassifier(n_estimators=125,
random_state=0)`` fitted on the device (``forest_fit.fit_extra_trees``, ``csrc/extra_trees_fit.cu``): one CTA per tree replays
scikit-learn 1.9's depth-first build and every draw of its splitter, so the trees, importances and ranking are scikit-learn's bits.
Features that are not finite as float32, or a table above the kernel's limits, are fitted by scikit-learn.  The F-test
(``f_regression``), k-Best (``SelectKBest(f_classif)``) and variance (``VarianceThreshold``) scores are scikit-learn on the host,
called as the reference calls them.  ``create_pipeline_neuron_net`` is the reference's unfitted BernoulliRBM + LogisticRegression
pipeline.  Differences: the score table is built in one step (the reference's ``DataFrame.append`` is gone from pandas 2), and of
more ``names`` than features the first D are used (the reference raises ``IndexError``).
"""
import collections
import ctypes as C
import logging
import os
import pickle
import random
import warnings

import numpy as np
from scipy.stats import randint as sp_randint
from scipy.stats import uniform as sp_random
from sklearn import decomposition, ensemble, linear_model, metrics, neighbors, neural_network, pipeline, preprocessing, svm, tree
from sklearn.exceptions import ConvergenceWarning
from sklearn.model_selection import GridSearchCV, RandomizedSearchCV

from . import _lib
from .engine import get_engine
from .utilities import ImageDimensionError

#: name template for exporting trained classifier (adding classifier name and version)
TEMPLATE_NAME_CLF = 'classifier_{}.pkl'
#: default (recommended) classifier for supervised segmentation
DEFAULT_CLASSIF_NAME = 'RandForest'
#: default (recommended) clustering for unsupervised segmentation
DEFAULT_CLUSTERING = 'kMeans'
#: file name of exported evaluation on feature quality
NAME_CSV_FEATURES_SELECT = 'feature_selection.csv'
#: exporting partial results about trained classifier
NAME_CSV_CLASSIF_CV_SCORES = 'classif_{}_cross-val_scores-{}.csv'
#: exporting partial results about trained classifier - Receiver Operating Characteristics
NAME_CSV_CLASSIF_CV_ROC = 'classif_{}_cross-val_ROC-{}.csv'
#: exporting partial results about trained classifier - Area Under Curve
NAME_TXT_CLASSIF_CV_AUC = 'classif_{}_cross-val_AUC-{}.txt'
#: default number of workers of a parameter search: half of the CPUs
NB_WORKERS_SERACH = max(1, int((os.cpu_count() or 1) * 0.5))
#: default types of computed metrics
METRIC_AVERAGES = ('macro', 'weighted')
#: default computed metrics
METRIC_SCORING = ('f1_macro', 'accuracy', 'precision_macro', 'recall_macro')
#: mapping of metrics names to used functions
DICT_SCORING = {
    'f1': metrics.f1_score,
    'accuracy': metrics.accuracy_score,
    'precision': metrics.precision_score,
    'recall': metrics.recall_score,
}

#: decimal digits of the features before ``down_sample_dict_features_unique`` looks for equal rows
ROUND_UNIQUE_FTS_DIGITS = 3
# the k-means of down_sample_dict_features_kmean: KMeans(n_clusters=nb_samples, init='random', n_init=3, max_iter=5), tol 1e-4
_KMEANS_N_INIT, _KMEANS_MAX_ITER, _KMEANS_TOL = 3, 5, 1e-4

#: largest contingency table (cells)
TABLE_MAX_CELLS = 1 << 28
# enum isb_dtype of include/imsegm_b200.h for the label maps
_LABEL_DTYPES = {'bool': 9, 'uint8': 0, 'int8': 4, 'uint16': 1, 'int16': 5, 'int32': 6, 'uint32': 7, 'int64': 8}
_I64 = np.iinfo(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# contingency table (device)
# ---------------------------------------------------------------------------------------------------------------------

def _labels(arr):
    """(flat contiguous label array of a device dtype, whether it was float) of a map"""
    arr = np.asarray(arr)
    kind = arr.dtype.kind
    if kind == 'f':
        if arr.size and not (np.all(np.isfinite(arr)) and np.all(np.floor(arr) == arr)):
            raise ValueError("Classification metrics can't handle continuous targets")
        if arr.size and (arr.min() < _I64.min or arr.max() >= 2.0 ** 63):
            raise ValueError('labels must fit in int64')
        return arr.astype(np.int64).ravel(), True
    if kind not in 'biu':
        raise TypeError('label maps must hold integers, got %s' % arr.dtype)
    if arr.dtype.name not in _LABEL_DTYPES:
        if arr.size and arr.max() > _I64.max:
            raise ValueError('labels must fit in int64')
        arr = arr.astype(np.int64)
    return np.ascontiguousarray(arr).ravel(), False


def _drop_list(drop_labels):
    """ascending int64 values of ``drop_labels`` that an integer map can hold"""
    ints = set()
    for v in ([] if drop_labels is None else np.asarray(list(drop_labels), dtype=object).ravel().tolist()):
        try:
            iv = int(v)
        except (TypeError, ValueError, OverflowError):
            continue
        if iv == v and _I64.min <= iv <= _I64.max:
            ints.add(iv)
    return np.array(sorted(ints), dtype=np.int64)


class _Pending(object):
    """one contingency table in flight on an engine's current stream: the count has run, the write and download are enqueued"""

    def __init__(self, eng, y_true, y_pred, drop):
        torch, lib, st = eng.torch, eng.lib, _lib.stream_ptr()
        self.dtypes = (_LABEL_DTYPES[y_true.dtype.name], _LABEL_DTYPES[y_pred.dtype.name])
        n = y_true.size
        d_true = eng.to_device(y_true.view(np.uint8) if y_true.dtype == bool else y_true, 'clf_true')
        d_pred = eng.to_device(y_pred.view(np.uint8) if y_pred.dtype == bool else y_pred, 'clf_pred')
        d_drop = eng.to_device(drop, 'clf_drop') if len(drop) else None
        ws_bytes = lib.isb_contingency_workspace_bytes(*self.dtypes)
        ws = eng.buf('clf_ws', ws_bytes, torch.uint8)
        info = (C.c_longlong * 6)()
        args = (_lib.ptr(d_true), self.dtypes[0], _lib.ptr(d_pred), self.dtypes[1], C.c_longlong(n), _lib.ptr(d_drop), len(drop))
        _lib.check(lib.isb_contingency_count(*args, _lib.ptr(ws), C.c_size_t(ws_bytes), info, st))
        self.k = (int(info[0]), int(info[1]))
        if self.k[0] * self.k[1] > TABLE_MAX_CELLS:
            raise MemoryError('a contingency table of %d x %d cells is above the limit of %d' % (self.k + (TABLE_MAX_CELLS, )))
        self.done = None
        if self.k[0] and self.k[1]:
            v_true = eng.buf('clf_values_true', self.k[0], torch.int64)
            v_pred = eng.buf('clf_values_pred', self.k[1], torch.int64)
            counts = eng.buf('clf_counts', self.k, torch.int64)
            _lib.check(lib.isb_contingency_write(*args, info, _lib.ptr(ws), C.c_size_t(ws_bytes), _lib.ptr(v_true), _lib.ptr(v_pred),
                                                 _lib.ptr(counts), st))
            self.hosts, self.done = eng.download([v_true[:self.k[0]], v_pred[:self.k[1]], counts[:self.k[0], :self.k[1]]])

    def result(self):
        """(true values [K_true], pred values [K_pred], counts [K_true, K_pred]) int64"""
        if self.done is None:
            return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 0), np.int64)
        self.done.synchronize()
        return tuple(h.numpy().copy() for h in self.hosts)


def _contingency(y_true, y_pred, drop=()):
    """(true values, pred values, counts [K_true, K_pred]) of two flat label arrays of device dtypes, pixels with a value in the
    ascending int64 ``drop`` in either map left out"""
    drop = np.ascontiguousarray(drop, dtype=np.int64)
    if y_true.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 0), np.int64)
    return _Pending(get_engine(), y_true, y_pred, drop).result()


# ---------------------------------------------------------------------------------------------------------------------
# metrics from the table (host)
# ---------------------------------------------------------------------------------------------------------------------

class _Table(object):
    """the nonzero cells of a contingency table: true value a, pred value b, pixel count w (int64 arrays)"""

    def __init__(self, a, b, w, is_float=False):
        self.a, self.b, self.w, self.is_float = a, b, w, is_float

    @classmethod
    def from_dense(cls, v_true, v_pred, counts, is_float=False):
        r, c = np.nonzero(counts)
        return cls(v_true[r], v_pred[c], counts[r, c], is_float)

    def merged(self, a, b):
        """the cells with their values replaced by a, b and equal pairs summed"""
        if len(a) == 0:
            return _Table(a, b, self.w, self.is_float)
        pairs, inv = np.unique(np.stack([a, b], 1), axis=0, return_inverse=True)
        w = np.bincount(inv.ravel(), weights=self.w, minlength=len(pairs)).astype(np.int64)
        return _Table(pairs[:, 0], pairs[:, 1], w, self.is_float)

    def labels(self):
        return np.union1d(self.a, self.b)


def _sequential(table):
    """the cells renumbered as the reference's relabel_sequential over the union of labels (at most two): a table of max + 1 entries
    filled in order, negative labels wrapping as numpy indices do"""
    uq = table.labels()
    if len(uq) == 0:
        raise ValueError('zero-size array to reduction operation maximum which has no identity')
    if table.is_float:
        raise TypeError("'numpy.float64' object cannot be interpreted as an integer")
    size = int(uq.max()) + 1

    def slot(v):
        if not -size <= v < size:
            raise IndexError('index %d is out of bounds for axis 0 with size %d' % (v, size))
        return v % size

    lut = {}
    for i, lb in enumerate(uq.tolist()):
        lut[slot(lb)] = i
    remap = {lb: lut[slot(lb)] for lb in uq.tolist()}
    get = np.vectorize(remap.__getitem__, otypes=[np.int64])
    return table.merged(get(table.a), get(table.b))


def _adjusted_rand(table):
    """scikit-learn's adjusted_rand_score from the pair confusion of the table, in integers"""
    w = table.w
    n = int(w.sum())
    _, ia = np.unique(table.a, return_inverse=True)
    _, ib = np.unique(table.b, return_inverse=True)
    n_c = np.bincount(ia.ravel(), weights=w).astype(np.int64)
    n_k = np.bincount(ib.ravel(), weights=w).astype(np.int64)
    sum_squares = int((w * w).sum())
    tp = sum_squares - n
    fp = int((w * n_k[ib.ravel()]).sum()) - sum_squares
    fn = int((w * n_c[ia.ravel()]).sum()) - sum_squares
    tn = n * n - fp - fn - sum_squares
    if fn == 0 and fp == 0:
        return 1.0
    return 2.0 * (tp * tn - fn * fp) / ((tp + fn) * (fn + tn) + (tp + fp) * (fp + tn))


def _confusion(table):
    """confusion matrix over the sorted union of labels, as lists of Python ints"""
    uq = table.labels()
    conf = np.zeros((len(uq), len(uq)), dtype=np.int64)
    np.add.at(conf, (np.searchsorted(uq, table.a), np.searchsorted(uq, table.b)), table.w)
    return conf.tolist()


def _classif_metrics(table, metric_averages, ndim=1):
    """compute_classif_metrics of the pixels the table counts, taken from arrays of ``ndim`` dimensions"""
    if len(table.labels()) <= 2:
        table = _sequential(table)
    if ndim != 1:                                   # scikit-learn's clustering scores take label vectors
        raise ValueError('labels_true must be 1D: %d dimensions given' % ndim)
    y_true, y_pred, weight = table.a, table.b, table.w
    eval_str = 'EVALUATION: {:<2} PRE: {:.3f} REC: {:.3f} F1: {:.3f} S: {:>6}'
    try:
        p, r, f, s = metrics.precision_recall_fscore_support(y_true, y_pred, sample_weight=weight)
        for lb, _ in enumerate(p):
            logging.debug(eval_str.format(lb, p[lb], r[lb], f[lb], s[lb]))
    except Exception:
        logging.exception('metrics.precision_recall_fscore_support')
    n = int(weight.sum())
    dict_metrics = {
        'ARS': _adjusted_rand(table),
        'accuracy': float(np.float64(int(weight[y_true == y_pred].sum())) / np.float64(n)),
        'confusion': _confusion(table),
    }
    names = ['precision', 'recall', 'f1', 'support']
    for avg in metric_averages:
        try:
            mtr = metrics.precision_recall_fscore_support(y_true, y_pred, average=avg, sample_weight=weight)
            res = dict(zip(['{}_{}'.format(nm, avg) for nm in names], mtr))
        except Exception:
            logging.exception('metrics.precision_recall_fscore_support')
            res = dict(zip(['{}_{}'.format(nm, avg) for nm in names], [-1] * 4))
        dict_metrics.update(res)
    return dict_metrics


def _tp_tn_fp_fn(table, label_positive=None):
    """compute_tp_tn_fp_fn of the pixels the table counts"""
    uq_labels = table.labels().tolist()
    if len(uq_labels) > 2:
        logging.debug('too many labels: %r', uq_labels)
        return np.nan, np.nan, np.nan, np.nan
    if len(uq_labels) < 2:
        logging.debug('only one label: %r', uq_labels)
        return int(table.w.sum()), 0, 0, 0
    if label_positive is None or label_positive not in uq_labels:
        label_positive = uq_labels[-1]
    uq_labels.remove(label_positive)
    neg = uq_labels[0]

    def count(a, b):
        return np.int64(table.w[(table.a == a) & (table.b == b)].sum())
    # the reference's orientation: FP is annotated positive and segmented negative
    return count(label_positive, label_positive), count(neg, neg), count(label_positive, neg), count(neg, label_positive)


def _ratio_fpfn_tpfn(tp, fp, fn):
    if (fp + fn) == 0:
        return 0.
    return float(fp + fn) / float(tp + fn)


def _ratio_tpfp_tpfn(tp, fp, fn):
    if (tp + fn) == 0:
        return 0.
    return float(tp + fp) / float(tp + fn)


def _unique_lut(rows, cols, counts, n_lut, keep_bg, query):
    """the look-up table of labeling.max_overlap_unique_lut at the columns ``query`` from the positive cells (rows, cols, counts) of
    the overlap matrix, without building the matrix:
    - greedy: cells by count descending, ties by row then column (row-major order), skipping a used row or column;
    - first fill: an unmatched column i takes i when no matched row is i;
    - second fill: the unmatched columns that are also matched rows, ascending, take the matched columns that are not matched rows,
      descending (the largest free value first); once those run out the rest stay -1."""
    rows, cols, counts = (np.asarray(x, dtype=np.int64) for x in (rows, cols, counts))
    match = {}
    if keep_bg:
        if n_lut == 0:
            raise IndexError('list assignment index out of range')
        match[0] = 0
        keep = (rows != 0) & (cols != 0)
        rows, cols, counts = rows[keep], cols[keep], counts[keep]
    keep = counts > 0
    rows, cols, counts = rows[keep], cols[keep], counts[keep]
    order = np.lexsort((cols, rows, -counts))
    used_r = set(match.values())
    n_r, n_c = len(np.unique(rows)), len(np.unique(cols))
    for r, c in zip(rows[order].tolist(), cols[order].tolist()):
        if r in used_r or c in match:
            continue
        used_r.add(r)
        match[c] = r
        if len(used_r) >= n_r + keep_bg or len(match) >= n_c + keep_bg:
            break
    matched_rows = set(match.values())
    pending = sorted(r for r in matched_rows if 0 <= r < n_lut and r not in match)
    free = sorted((c for c in match if c not in matched_rows), reverse=True)
    second = dict(zip(pending, free))
    out = []
    for q in np.asarray(query, dtype=np.int64).tolist():
        if q in match:
            out.append(match[q])
        elif q not in matched_rows:
            out.append(q)
        else:
            out.append(second.get(q, -1))
    return np.array(out, dtype=np.int64)


def _relabel_unique(table):
    """the table after ``y_pred = relabel_max_overlap_unique(y_true, y_pred, keep_bg=False)`` (labeling.py of this package):
    negative labels kept"""
    if table.is_float:
        raise TypeError('label maps must be integer arrays, got float64')
    a, b, w = table.a, table.b, table.w
    if len(a) == 0:
        raise ValueError('zero-size array to reduction operation maximum which has no identity')
    n_rows, n_lut = int(a.max()) + 1, int(b.max()) + 1
    if n_rows < 0 or n_lut < 0:                     # numpy's ValueError of the overlap matrix's np.zeros
        raise ValueError('negative dimensions are not allowed')
    lo = int(b.min())
    if lo < -n_lut:                                 # numpy's IndexError of lut[seg] in labeling.relabel_max_overlap_unique
        raise IndexError('index %d is out of bounds for axis 0 with size %d' % (lo, n_lut))
    pos = (a >= 0) & (b >= 0)
    uq_b = np.unique(b[b >= 0])
    lut = _unique_lut(a[pos], b[pos], w[pos], n_lut, False, uq_b)
    new_b = b.copy()
    sel = b >= 0
    new_b[sel] = lut[np.searchsorted(uq_b, b[sel])]
    return table.merged(a, new_b)


def _stat_segm_annot(table, name, relabel):
    """compute_classif_stat_segm_annot of the pixels the table counts (after the drop mask)"""
    if relabel:
        table = _relabel_unique(table)
    dict_stat = _classif_metrics(table, ['macro'])
    if len(np.unique(table.b)) == 2:
        tp, _, fp, fn = _tp_tn_fp_fn(table)
        dict_stat['(FP+FN)/(TP+FN)'] = _ratio_fpfn_tpfn(tp, fp, fn)
        dict_stat['(TP+FP)/(TP+FN)'] = _ratio_tpfp_tpfn(tp, fp, fn)
    dict_stat['name'] = name
    return dict_stat


def _table_of(y_true, y_pred, drop=()):
    (t, ft), (p, fp) = _labels(y_true), _labels(y_pred)
    return _Table.from_dense(*_contingency(t, p, drop), is_float=ft or fp)


# ---------------------------------------------------------------------------------------------------------------------
# public functions
# ---------------------------------------------------------------------------------------------------------------------

def compute_classif_metrics(y_true, y_pred, metric_averages=METRIC_AVERAGES):
    """ standard metrics of a multi-class classification (reference classification.py:305-371): ARS, accuracy, confusion matrix
    and precision / recall / F1 / support for every average of ``metric_averages`` (-1 each when scikit-learn rejects the average)

    >>> np.random.seed(0)
    >>> y_true = np.random.randint(0, 3, 25) * 2
    >>> y_pred = np.random.randint(0, 2, 25) * 2
    >>> d = compute_classif_metrics(y_true, y_true)
    >>> d['accuracy']
    1.0
    >>> d['confusion']
    [[10, 0, 0], [0, 10, 0], [0, 0, 5]]
    >>> d = compute_classif_metrics(y_true, y_pred)
    >>> d['accuracy']  # doctest: +ELLIPSIS
    0.32...
    >>> d['confusion']
    [[3, 7, 0], [5, 5, 0], [1, 4, 0]]
    """
    y_true, y_pred = np.array(y_true), np.array(y_pred)
    if y_true.shape != y_pred.shape:
        raise ValueError('prediction (%i) and annotation (%i) should be equal' % (len(y_true), len(y_pred)))
    return _classif_metrics(_table_of(y_true, y_pred), metric_averages, y_true.ndim)


def compute_classif_stat_segm_annot(annot_segm_name, drop_labels=None, relabel=False):
    """ classification statistic between an annotation and a segmentation (reference classification.py:374-421): the pixels with a
    value of ``drop_labels`` in either map are left out, ``relabel`` matches the segmentation's classes to the annotation's first
    (``labeling.relabel_max_overlap_unique``), and a segmentation of two classes adds the two binary ratios

    >>> np.random.seed(0)
    >>> annot = np.random.randint(0, 2, (5, 10))
    >>> segm = np.random.randint(0, 2, (5, 10))
    >>> d = compute_classif_stat_segm_annot((annot, segm, 'ttt'), relabel=True, drop_labels=[5])
    >>> d['(FP+FN)/(TP+FN)']  # doctest: +ELLIPSIS
    0.846...
    >>> d = compute_classif_stat_segm_annot((annot, segm + 1, 'ttt'), relabel=False, drop_labels=[0])
    >>> d['confusion']
    [[13, 17], [0, 0]]
    """
    annot, segm, name = annot_segm_name
    annot, segm = np.asarray(annot), np.asarray(segm)
    if segm.shape != annot.shape:
        raise ImageDimensionError('dimension do not match for segm: %r - annot: %r' % (segm.shape, annot.shape))
    return _stat_segm_annot(_table_of(annot, segm, _drop_list(drop_labels)), name, relabel)


def compute_stat_per_image(segms, annots, names=None, nb_workers=2, drop_labels=None, relabel=False):
    """ ``compute_classif_stat_segm_annot`` of every (annotation, segmentation) pair as a DataFrame indexed by ``name`` (reference
    classification.py:424-471).  The pairs alternate over two CUDA streams: the upload and counting passes of pair i + 1 overlap
    the final counting pass of pair i.  ``nb_workers`` is accepted and ignored.

    >>> np.random.seed(0)
    >>> img_true = np.random.randint(0, 3, (50, 100))
    >>> img_pred = np.random.randint(0, 2, (50, 100))
    >>> df = compute_stat_per_image([img_true], [img_pred], drop_labels=[-1])
    >>> df.round(4).iloc[0]['accuracy']
    0.3384
    """
    import pandas as pd
    from .pipelines import _batch_engines
    if len(segms) != len(annots):
        raise RuntimeError('size of segment. (%i) amd annot. (%i) should be equal' % (len(segms), len(annots)))
    if not names:
        names = map(str, range(len(segms)))
    drop = _drop_list(drop_labels)
    engines = _batch_engines(2)
    torch = engines[0][0].torch
    caller = torch.cuda.current_stream()
    list_stat, prev = [], None

    def finish(job):
        kind, payload, name = job
        if kind == 'error':
            raise payload
        table = payload[0] if kind == 'host' else _Table.from_dense(*payload[0].result(), is_float=payload[1])
        list_stat.append(_stat_segm_annot(table, name, relabel))

    for i, (annot, segm, name) in enumerate(zip(annots, segms, names)):
        annot, segm = np.asarray(annot), np.asarray(segm)
        if segm.shape != annot.shape:
            job = ('error', ImageDimensionError('dimension do not match for segm: %r - annot: %r' % (segm.shape, annot.shape)), name)
        else:
            (t, ft), (p, fp) = _labels(annot), _labels(segm)
            if t.size == 0:
                job = ('host', (_Table(t.astype(np.int64), p.astype(np.int64), np.zeros(0, np.int64), ft or fp), ), name)
            else:
                eng, stream = engines[i % 2]
                stream.wait_stream(caller)
                with torch.cuda.stream(stream):
                    job = ('device', (_Pending(eng, t, p, drop), ft or fp), name)
        if prev is not None:
            finish(prev)
        prev = job
    if prev is not None:
        finish(prev)
    for _, stream in engines:
        caller.wait_stream(stream)
    df_stat = pd.DataFrame(list_stat)
    df_stat.set_index('name', inplace=True)
    return df_stat


def relabel_sequential(labels, uq_labels=None):
    """ labels renumbered 0, 1, ... in the order of ``uq_labels`` (default: the sorted unique labels), as a list (reference
    classification.py:635-653); the table has max(uq_labels) + 1 entries, so a negative label wraps as a numpy index

    >>> relabel_sequential([0, 0, 0, 5, 5, 5, 0, 5])
    [0, 0, 0, 1, 1, 1, 0, 1]
    """
    labels = np.asarray(labels)
    uq = np.unique(labels) if uq_labels is None else np.asarray(uq_labels)
    lut = np.zeros(np.max(uq) + 1)
    lut[uq] = np.arange(len(uq))
    return lut[labels].astype(labels.dtype).tolist()


def compute_tp_tn_fp_fn(annot, segm, label_positive=None):
    """ (TP, TN, FP, FN) of two binary maps (reference classification.py:1265-1310): NaN each for more than two labels, (pixels, 0, 0,
    0) for one; FP counts annotated-positive pixels segmented negative, as in the reference

    >>> np.random.seed(0)
    >>> annot = np.random.randint(0, 2, (5, 7)) * 9
    >>> segm = np.random.randint(0, 2, (5, 7)) * 9
    >>> compute_tp_tn_fp_fn(annot, annot)
    (20, 15, 0, 0)
    >>> compute_tp_tn_fp_fn(annot, segm)
    (9, 5, 11, 10)
    >>> compute_tp_tn_fp_fn(annot, np.ones((5, 7)))
    (nan, nan, nan, nan)
    """
    annot, segm = np.asarray(annot), np.asarray(segm)
    if annot.size != segm.size:
        raise ValueError('annotation (%i) and segmentation (%i) should have the same size' % (annot.size, segm.size))
    if annot.size == 0:
        return 0, 0, 0, 0
    return _tp_tn_fp_fn(_table_of(annot, segm), label_positive)


def compute_metric_fpfn_tpfn(annot, segm, label_positive=None):
    """ (FP + FN) / (TP + FN) (reference classification.py:1313-1337)

    >>> np.random.seed(0)
    >>> annot = np.random.randint(0, 2, (50, 75)) * 3
    >>> segm = np.random.randint(0, 2, (50, 75)) * 3
    >>> compute_metric_fpfn_tpfn(annot, segm)  # doctest: +ELLIPSIS
    1.02...
    >>> compute_metric_fpfn_tpfn(annot, annot)
    0.0
    """
    tp, _, fp, fn = compute_tp_tn_fp_fn(annot, segm, label_positive)
    return _ratio_fpfn_tpfn(tp, fp, fn)


def compute_metric_tpfp_tpfn(annot, segm, label_positive=None):
    """ (TP + FP) / (TP + FN) (reference classification.py:1340-1366)

    >>> np.random.seed(0)
    >>> annot = np.random.randint(0, 2, (50, 75)) * 3
    >>> segm = np.random.randint(0, 2, (50, 75)) * 3
    >>> compute_metric_tpfp_tpfn(annot, segm)  # doctest: +ELLIPSIS
    1.03...
    >>> compute_metric_tpfp_tpfn(annot, annot)
    1.0
    """
    tp, _, fp, fn = compute_tp_tn_fp_fn(annot, segm, label_positive)
    return _ratio_tpfp_tpfn(tp, fp, fn)


# ---------------------------------------------------------------------------------------------------------------------
# training sets: class-balanced features (k-means on the device)
# ---------------------------------------------------------------------------------------------------------------------

def _rows_array(blocks):
    """the rows of the 2-D blocks stacked as ``np.array`` builds them from their ``tolist()``: floats as float64, integers as int64,
    and ``np.array([])`` when there are no rows"""
    blocks = [np.asarray(b) for b in blocks]
    if sum(len(b) for b in blocks) == 0:
        return np.array([])
    rows = np.concatenate([b for b in blocks if len(b)])
    if rows.dtype.kind == 'f':
        return rows.astype(np.float64)
    if rows.dtype.kind in 'iu' and (rows.dtype.kind == 'i' or rows.dtype.itemsize < 8):
        return rows.astype(np.int64)
    return np.array(rows.tolist())


def shuffle_features_labels(features, labels):
    """ features [n, D] and labels [n] permuted together by one ``np.random.shuffle`` of the row indices (reference
    classification.py:1027-1051)

    >>> np.random.seed(0)
    >>> fts = np.random.random((5, 2))
    >>> lbs = np.random.randint(0, 2, 5)
    >>> fts_new, lbs_new = shuffle_features_labels(fts, lbs)
    >>> np.array_equal(fts, fts_new)
    False
    >>> np.array_equal(lbs, lbs_new)
    False
    """
    if len(features) != len(labels):
        raise ValueError('features (%i) and labels (%i) should have equal length' % (len(features), len(labels)))
    order = list(range(len(labels)))
    np.random.shuffle(order)
    return features[order, :], np.asarray(labels)[order]


def convert_dict_label_features_2_vectors(dict_features):
    """ {label: features [n_label, D]} -> (features [n, D] in the dict's order, list of the label of every row) (reference
    classification.py:1054-1065)

    >>> fts, lbs = convert_dict_label_features_2_vectors({1: np.ones((2, 3)), 0: np.zeros((1, 3))})
    >>> fts.shape, lbs
    ((3, 3), [1, 1, 0])
    """
    labels = []
    for label, fts in dict_features.items():
        labels.extend([label] * len(fts))
    return _rows_array([dict_features[k] for k in dict_features]), labels


def compose_dict_label_features(features, labels):
    """ features [n, D] and labels [n] -> {label: its rows}, keys in the order of ``np.unique(labels)`` (reference
    classification.py:1068-1080)

    >>> d = compose_dict_label_features(np.arange(8).reshape(4, 2), np.array([1, 0, 1, 1]))
    >>> sorted(d), d[0].tolist()
    ([0, 1], [[2, 3]])
    """
    features = np.array(features)
    dict_features = {}
    for label in np.unique(labels):
        dict_features[label] = features[labels == label, :]
    return dict_features


def down_sample_dict_features_random(dict_features, nb_samples):
    """ at most ``nb_samples`` rows of every class: the first ``nb_samples`` of a ``random.shuffle`` (Python's global RNG) of its row
    indices; smaller classes are copied (reference classification.py:1083-1107)

    >>> np.random.seed(0)
    >>> d_fts = {'a': np.random.random((100, 3))}
    >>> d_fts = down_sample_dict_features_random(d_fts, 5)
    >>> d_fts['a'].shape
    (5, 3)
    """
    dict_features_new = {}
    for label, features in dict_features.items():
        if len(features) <= nb_samples:
            dict_features_new[label] = features.copy()
            continue
        order = list(range(len(features)))
        random.shuffle(order)
        dict_features_new[label] = np.array(features)[order[:nb_samples], :]
    return dict_features_new


class _LloydRun(object):
    """one Lloyd run: labels [n] int32, inertia, centres [k, D] (centred), sweeps"""

    def __init__(self, labels, inertia, centres, n_iter):
        self.labels, self.inertia, self.centres, self.n_iter = labels, inertia, centres, n_iter


def _kmeans_seeds(n_samples, n_clusters):
    """the starting rows of one run of KMeans(init='random') with unit weights, drawn from numpy's global RNG as
    ``_init_centroids`` draws them"""
    weight = np.ones(n_samples)
    return np.random.choice(n_samples, size=n_clusters, replace=False, p=weight / weight.sum())


def _relocate_empty_clusters(X, centres_old, sums, weights, labels):
    """scikit-learn's _relocate_empty_clusters_dense (unit weights), in place on the member sums [k, D] and weights [k]: every empty
    cluster takes one of the rows farthest from their centres, which leaves its cluster"""
    empty = np.where(weights == 0)[0]
    if len(empty) == 0:
        return
    dist = ((X - centres_old[labels]) ** 2).sum(axis=1)
    far = np.argpartition(dist, -len(empty))[:-len(empty) - 1:-1]
    if np.max(dist) == 0:                   # more clusters than distinct rows: nothing to move
        return
    for new_id, far_idx in zip(empty.tolist(), far.tolist()):
        old_id = labels[far_idx]
        sums[old_id] -= X[far_idx]
        sums[new_id] = X[far_idx]
        weights[new_id] = 1.
        weights[old_id] -= 1.


def _average_centres(sums, weights):
    """scikit-learn's _average_centers: sum * (1 / weight); a cluster still empty takes the row of the heaviest cluster as it is at
    that point of scikit-learn's in-place loop (averaged when the heaviest comes first, its sum otherwise)"""
    heaviest = int(np.argmax(weights))
    full = weights > 0
    centres = sums.copy()
    centres[full] = sums[full] * (1.0 / weights[full])[:, None]
    empty = np.where(~full)[0]
    centres[empty] = np.where((empty < heaviest)[:, None], sums[heaviest], centres[heaviest])
    return centres


def _same_clustering(labels1, labels2, n_clusters):
    """scikit-learn's _is_same_clustering: every cluster of labels1 maps onto one cluster of labels2"""
    mapping = np.full(n_clusters, -1, dtype=np.int64)
    uq, first = np.unique(labels1, return_index=True)
    mapping[uq] = labels2[first]
    return bool(np.all(mapping[labels1] == labels2))


def _lloyd(eng, d_x, X, centres, max_iter, tol):
    """_kmeans_single_lloyd of scikit-learn from ``centres`` [k, D] on the centred rows X [n, D] (host) = d_x (device), unit
    weights.  The sweeps run on the device; a sweep that leaves a cluster empty comes back here for the relocation."""
    torch, lib, st = eng.torch, eng.lib, _lib.stream_ptr()
    n, D = X.shape
    k = len(centres)
    d_c = eng.to_device(np.ascontiguousarray(centres, dtype=np.float64), 'km_centres')
    labels = eng.buf('km_labels', n, torch.int32)
    _lib.check(lib.isb_fill_i32(_lib.ptr(labels), n, -1, st))
    status = eng.to_device(np.zeros(4, np.int32), 'km_status')
    sums = eng.buf('km_sums', (k, D), torch.float64)
    counts = eng.buf('km_counts', k, torch.int32)
    inertia = eng.buf('km_inertia', 1, torch.float64)
    ws_bytes = lib.isb_kmeans_workspace_bytes(n, k, D)
    ws = eng.buf('km_ws', max(ws_bytes, 1), torch.uint8)
    sweeps = max_iter
    while True:
        _lib.check(lib.isb_kmeans_lloyd(_lib.ptr(d_x), n, D, k, max_iter, sweeps, C.c_double(tol), _lib.ptr(d_c), _lib.ptr(labels), _lib.ptr(status),
                                        _lib.ptr(sums), _lib.ptr(counts), _lib.ptr(inertia), _lib.ptr(ws), C.c_size_t(ws_bytes), st))
        stat = eng.to_host(status).copy()
        if stat[0] != 3:
            break
        # a cluster went empty: this sweep's update on the host, as lloyd_iter_chunked_dense does it
        lab = eng.to_host(labels).copy()
        c_old = eng.to_host(d_c).copy()
        s = eng.to_host(sums).copy()
        w = eng.to_host(counts).astype(np.float64)
        _relocate_empty_clusters(X, c_old, s, w, lab)
        c_new = _average_centres(s, w)
        shift_tot = (np.sqrt(((c_new - c_old) ** 2).sum(axis=1)) ** 2).sum()
        done = int(stat[1]) + 1
        code = 1 if stat[2] == 0 else 2 if shift_tot <= tol else 4 if done >= max_iter else 0
        d_c = eng.to_device(c_new, 'km_centres')
        status = eng.to_device(np.array([code, done, 0, 0], np.int32), 'km_status')
        sweeps = max_iter - done if code == 0 else 0
    return _LloydRun(eng.to_host(labels).copy(), float(eng.to_host(inertia)[0]), eng.to_host(d_c).copy(), int(stat[1]))


def _nearest_rows(eng, d_x, n, D, centres):
    """for every centre the row of least exact squared distance, lowest row on ties (int64 [k])"""
    torch, lib = eng.torch, eng.lib
    k = len(centres)
    d_c = eng.to_device(np.ascontiguousarray(centres, dtype=np.float64), 'km_centres')
    nearest = eng.buf('km_nearest', k, torch.int32)
    ws_bytes = lib.isb_kmeans_workspace_bytes(n, k, D)
    ws = eng.buf('km_ws', max(ws_bytes, 1), torch.uint8)
    _lib.check(lib.isb_kmeans_nearest(_lib.ptr(d_x), n, D, _lib.ptr(d_c), k, _lib.ptr(nearest), _lib.ptr(ws), C.c_size_t(ws_bytes),
                                      _lib.stream_ptr()))
    return eng.to_host(nearest).astype(np.int64)


def _kmeans_sample(features, nb_samples, n_init=_KMEANS_N_INIT, max_iter=_KMEANS_MAX_ITER):
    """np.argmin(KMeans(nb_samples, init='random', n_init, max_iter).fit_transform(features), axis=0) on the device:
    (selected rows int64 [nb_samples], the runs in order, the best run)"""
    X0 = np.asarray(features, dtype=np.float64)
    if X0.ndim != 2:
        raise ValueError('Expected 2D array, got %dD array instead' % X0.ndim)
    if not np.all(np.isfinite(X0)):
        raise ValueError('Input X contains NaN or infinity.')
    n, D = X0.shape
    if not 1 <= nb_samples <= n:
        raise ValueError('n_samples=%d should be >= n_clusters=%d.' % (n, nb_samples))
    tol = np.mean(np.var(X0, axis=0)) * _KMEANS_TOL
    X_mean = X0.mean(axis=0)
    X = X0 - X_mean
    eng = get_engine()
    d_x = eng.to_device(X, 'km_x')
    runs, best = [], None
    for _ in range(n_init):
        run = _lloyd(eng, d_x, X, X[_kmeans_seeds(n, nb_samples)], max_iter, tol)
        runs.append(run)
        if best is None or (run.inertia < best.inertia and not _same_clustering(run.labels, best.labels, nb_samples)):
            best = run
    distinct = len(np.unique(best.labels))
    if distinct < nb_samples:
        warnings.warn('Number of distinct clusters ({}) found smaller than n_clusters ({}). Possibly due to duplicate points '
                      'in X.'.format(distinct, nb_samples), ConvergenceWarning, stacklevel=3)
    d_x0 = eng.to_device(X0, 'km_x')
    return _nearest_rows(eng, d_x0, n, D, best.centres + X_mean), runs, best


def down_sample_dict_features_kmean(dict_features, nb_samples):
    """ ``nb_samples`` rows of every class: the rows nearest to the centres of KMeans(n_clusters=nb_samples, init='random',
    n_init=3, max_iter=5) of its features, run on the device; the starts come from numpy's global RNG; smaller classes are copied
    (reference classification.py:1110-1134)

    >>> np.random.seed(0)
    >>> d_fts = {'a': np.random.random((100, 3))}
    >>> d_fts = down_sample_dict_features_kmean(d_fts, 5)  # doctest: +SKIP
    >>> d_fts['a'].shape  # doctest: +SKIP
    (5, 3)
    """
    dict_features_new = {}
    for label, features in dict_features.items():
        if len(features) <= nb_samples:
            dict_features_new[label] = features.copy()
            continue
        selected, _, _ = _kmeans_sample(features, nb_samples)
        dict_features_new[label] = features[selected, :]
    return dict_features_new


def unique_rows(data):
    """ the distinct rows of a 2-D array, sorted lexicographically over the columns (numpy's structured-row ``np.unique``: rows
    holding NaN never merge, -0.0 equals 0.0) (reference classification.py:1146-1156)

    >>> unique_rows(np.array([[1, 2], [0, 5], [1, 2]]))
    array([[0, 5],
           [1, 2]])
    """
    data = np.array(data, order='C')
    as_records = data.view(np.dtype([('f%d' % i, data.dtype) for i in range(data.shape[1])]))
    return np.unique(as_records).view(data.dtype).reshape(-1, data.shape[1])


def down_sample_dict_features_unique(dict_features):
    """ the distinct rows of every class after rounding to ``ROUND_UNIQUE_FTS_DIGITS`` decimals (reference
    classification.py:1159-1180)

    >>> np.random.seed(0)
    >>> d_fts = {'a': np.random.random((100, 3))}
    >>> d_fts = down_sample_dict_features_unique(d_fts)
    >>> d_fts['a'].shape
    (100, 3)
    """
    dict_features_new = {}
    for label in dict_features:
        features = np.round(dict_features[label], ROUND_UNIQUE_FTS_DIGITS)
        unique_fts = np.array(unique_rows(features))
        if features.ndim != unique_fts.ndim:
            raise ValueError('feature dim matching')
        if features.shape[1] != unique_fts.shape[1]:
            raise ValueError('features: %i <> %i' % (features.shape[1], unique_fts.shape[1]))
        dict_features_new[label] = unique_fts
    return dict_features_new


def balance_dataset_by_(features, labels, balance_type='random', min_samples=None):
    """ the same number of rows per class (reference classification.py:1183-1216): ``'random'``, ``'kmeans'`` (down to
    ``min_samples``, default the smallest class) or ``'unique'`` (the distinct rounded rows); another name logs a warning and keeps
    every row.  Returns (features [n, D], list of labels) grouped by class in the order of ``np.unique(labels)``.

    >>> np.random.seed(0)
    >>> fts, lbs = balance_dataset_by_(np.random.random((25, 3)), np.random.randint(0, 2, 25))
    >>> fts.shape
    (24, 3)
    >>> lbs
    [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1]
    """
    logging.debug('balance dataset using "%s"', balance_type)
    if not min_samples:
        min_samples = min(collections.Counter(labels).values())
    dict_features = compose_dict_label_features(features, labels)
    kind = balance_type.lower()
    if kind == 'random':
        dict_features = down_sample_dict_features_random(dict_features, min_samples)
    elif kind == 'kmeans':
        dict_features = down_sample_dict_features_kmean(dict_features, min_samples)
    elif kind == 'unique':
        dict_features = down_sample_dict_features_unique(dict_features)
    else:
        logging.warning('not defined balancing method "%s"', balance_type)
    return convert_dict_label_features_2_vectors(dict_features)


def convert_set_features_labels_2_dataset(imgs_features, imgs_labels, drop_labels=None, balance_type=None):
    """ the features and labels of every image (dicts by image name, taken in sorted name order) in one training set
    (reference classification.py:1219-1262): rows whose label is in ``drop_labels`` left out, each image balanced by
    ``balance_dataset_by_`` when ``balance_type`` is given.  Returns (features [n, D], labels int [n], rows per image).

    >>> np.random.seed(0)
    >>> d_fts = {'a': np.random.random((25, 3)),
    ...          'b': np.random.random((30, 3)), }
    >>> d_lbs = {'a': np.random.randint(0, 2, 25),
    ...          'b': np.random.randint(0, 2, 30)}
    >>> fts, lbs, sizes = convert_set_features_labels_2_dataset(d_fts, d_lbs)
    >>> fts.shape
    (55, 3)
    >>> lbs.shape
    (55,)
    >>> sizes
    [25, 30]
    """
    logging.debug('convert set of features and labels to single one')
    if not all(k in imgs_labels for k in imgs_features):
        raise ValueError('missing some items of %r' % imgs_labels.keys())
    drop_labels = [] if drop_labels is None else drop_labels
    blocks, labels_all, sizes = [], [], []
    for name in sorted(imgs_features.keys()):
        features = np.array(imgs_features[name])
        labels = np.array(imgs_labels[name].astype(int))
        for lb in drop_labels:
            keep = labels != lb
            features, labels = features[keep], labels[keep]
        if balance_type is not None:
            features, labels = balance_dataset_by_(features, labels, balance_type=balance_type)
        blocks.append(features)
        labels_all += np.asarray(labels).tolist()
        sizes.append(len(labels))
    return _rows_array(blocks), np.array(labels_all, dtype=int), sizes


# ---------------------------------------------------------------------------------------------------------------------
# classifiers: the reference's zoo, searches, training (trees and forests on the device), export
# ---------------------------------------------------------------------------------------------------------------------

def create_classifiers(nb_workers=-1):
    """ every classifier of the reference with its default parameters (reference classification.py:86-124)

    >>> classifs = create_classifiers()
    >>> sorted(classifs)
    ['AdaBoost', 'DecTree', 'GradBoost', 'KNN', 'LogistRegr', 'RandForest', 'SVM']
    >>> sum([isinstance(create_clf_param_search_grid(k), dict) for k in classifs.keys()])
    7
    >>> sum([isinstance(create_clf_param_search_distrib(k), dict) for k in classifs.keys()])
    7
    """
    return {
        'RandForest': ensemble.RandomForestClassifier(n_estimators=20, min_samples_leaf=2, min_samples_split=3, n_jobs=nb_workers),
        'GradBoost': ensemble.GradientBoostingClassifier(subsample=0.25, warm_start=False, max_depth=6, min_samples_leaf=6,
                                                         n_estimators=200, min_samples_split=7),
        'LogistRegr': linear_model.LogisticRegression(solver='sag', n_jobs=nb_workers),
        'KNN': neighbors.KNeighborsClassifier(n_jobs=nb_workers),
        'SVM': svm.SVC(kernel='rbf', probability=True, tol=2e-3, max_iter=5000),
        'DecTree': tree.DecisionTreeClassifier(),
        'AdaBoost': ensemble.AdaBoostClassifier(n_estimators=5),
    }


def create_clf_pipeline(name_classif=DEFAULT_CLASSIF_NAME, pca_coef=0.95):
    """ StandardScaler, an optional PCA(pca_coef) and the named classifier (reference classification.py:127-143)

    >>> create_clf_pipeline()  # doctest: +ELLIPSIS
    Pipeline(...)
    """
    components = [('scaler', preprocessing.StandardScaler())]
    if pca_coef is not None:
        components += [('reduce_dim', decomposition.PCA(pca_coef))]
    components += [('classif', create_classifiers()[name_classif])]
    return pipeline.Pipeline(components)


def create_clf_param_search_grid(name_classif=DEFAULT_CLASSIF_NAME):
    """ parameter grid of a grid search (reference classification.py:146-208); {} and a warning for an unknown name

    >>> create_clf_param_search_grid('RandForest') # doctest: +ELLIPSIS
    {'classif__...': ...}
    >>> dict_classif = create_classifiers()
    >>> all(len(create_clf_param_search_grid(k)) > 0 for k in dict_classif)
    True
    >>> create_clf_param_search_grid('none')
    {}
    """

    def _log_space(b, e, n):
        return np.unique(np.logspace(b, e, n).astype(int)).tolist()

    clf_params = {
        'RandForest': {
            'classif__n_estimators': _log_space(0, 2, 40),
            'classif__min_samples_split': [2, 3, 5, 7, 9],
            'classif__min_samples_leaf': [1, 2, 4, 6, 9],
            'classif__criterion': ('gini', 'entropy'),
        },
        'KNN': {
            'classif__n_neighbors': _log_space(0, 2, 20),
            'classif__algorithm': ('ball_tree', 'kd_tree'),
            'classif__weights': ('uniform', 'distance'),
            'classif__leaf_size': _log_space(0, 1.5, 10),
        },
        'SVM': {
            'classif__C': np.linspace(0.2, 1., 8).tolist(),
            'classif__kernel': ('poly', 'rbf', 'sigmoid'),
            'classif__degree': [1, 2, 4, 6, 9],
        },
        'DecTree': {
            'classif__criterion': ('gini', 'entropy'),
            'classif__min_samples_split': [2, 3, 5, 7, 9],
            'classif__min_samples_leaf': range(1, 7, 2),
        },
        'GradBoost': {
            'classif__n_estimators': _log_space(0, 2, 25),
            'classif__max_depth': range(1, 7, 2),
            'classif__min_samples_split': [2, 3, 5, 7, 9],
            'classif__min_samples_leaf': range(1, 7, 2),
        },
        'LogistRegr': {
            'classif__C': np.linspace(0., 1., 5).tolist(),
            'classif__solver': ('lbfgs', 'sag'),
        },
        'AdaBoost': {
            'classif__n_estimators': _log_space(0, 2, 20),
        }
    }
    if name_classif not in clf_params:
        clf_params[name_classif] = {}
        logging.warning('not defined classifier name "%s"', name_classif)
    return clf_params[name_classif]


def create_clf_param_search_distrib(name_classif=DEFAULT_CLASSIF_NAME):
    """ parameter distributions of a random search (reference classification.py:211-268); {} for an unknown name

    >>> create_clf_param_search_distrib()  # doctest: +ELLIPSIS
    {...}
    >>> dict_classif = create_classifiers()
    >>> all(len(create_clf_param_search_distrib(k)) > 0 for k in dict_classif)
    True
    >>> create_clf_param_search_distrib('none')
    {}
    """
    clf_params = {
        'RandForest': {
            'classif__n_estimators': sp_randint(2, 25),
            'classif__min_samples_split': sp_randint(2, 9),
            'classif__min_samples_leaf': sp_randint(1, 7),
        },
        'KNN': {
            'classif__n_neighbors': sp_randint(5, 25),
            'classif__algorithm': ('ball_tree', 'kd_tree'),
            'classif__weights': ('uniform', 'distance'),
        },
        'SVM': {
            'classif__C': sp_random(0., 1.),
            'classif__kernel': ('poly', 'rbf', 'sigmoid'),
            'classif__degree': sp_randint(2, 9),
        },
        'DecTree': {
            'classif__criterion': ('gini', 'entropy'),
            'classif__min_samples_split': sp_randint(2, 9),
            'classif__min_samples_leaf': sp_randint(1, 7),
        },
        'GradBoost': {
            'classif__n_estimators': sp_randint(10, 200),
            'classif__max_depth': sp_randint(1, 7),
            'classif__min_samples_split': sp_randint(2, 9),
            'classif__min_samples_leaf': sp_randint(1, 7),
        },
        'LogistRegr': {
            'classif__C': sp_random(0., 1.),
            'classif__solver': ('newton-cg', 'lbfgs', 'sag'),
        },
        'AdaBoost': {
            'classif__n_estimators': sp_randint(2, 100),
        }
    }
    return clf_params.get(name_classif, {})


def create_pipeline_neuron_net():
    """ a BernoulliRBM feeding a LogisticRegression, unfitted (reference classification.py:271-283); fitted by scikit-learn

    >>> create_pipeline_neuron_net()  # doctest: +ELLIPSIS
    Pipeline(...)
    """
    logistic = linear_model.LogisticRegression()
    rbm = neural_network.BernoulliRBM(learning_rate=0.05, n_components=35, n_iter=299, verbose=False)
    return pipeline.Pipeline(steps=[('rbm', rbm), ('logistic', logistic)])


def search_params_cut_down_max_nb_iter(clf_parameters, nb_iter):
    """ ``nb_iter`` capped at the number of combinations when every parameter is a list (reference classification.py:953-977)

    >>> clf_params = create_clf_param_search_grid(DEFAULT_CLASSIF_NAME)
    >>> search_params_cut_down_max_nb_iter(clf_params, 100)
    100
    >>> search_params_cut_down_max_nb_iter(clf_params, 1e6)
    1450
    """
    counts = []
    for k in clf_parameters:
        vals = clf_parameters[k]
        if hasattr(vals, '__iter__'):
            counts.append(len(vals))
        else:
            return nb_iter
    count = int(np.prod(counts))
    if count < nb_iter:
        nb_iter = count
    return nb_iter


def create_classif_search(name_clf, clf_pipeline, nb_labels, search_type='random', cross_val=10, eval_metric='f1', nb_iter=250,
                          nb_workers=5):
    """ scikit-learn's GridSearchCV (``search_type='grid'``) or RandomizedSearchCV of the pipeline, scored by ``eval_metric`` with
    the weighted average for more than two labels (reference classification.py:980-1024)"""
    score_weight = 'weighted' if nb_labels > 2 else 'binary'
    scoring = metrics.make_scorer(DICT_SCORING[eval_metric.lower()], average=score_weight)
    if search_type == 'grid':
        clf_parameters = create_clf_param_search_grid(name_clf)
        logging.info('init Grid search...')
        return GridSearchCV(clf_pipeline, clf_parameters, scoring=scoring, cv=cross_val, n_jobs=nb_workers, verbose=1, refit=True)
    clf_parameters = create_clf_param_search_distrib(name_clf)
    nb_iter = search_params_cut_down_max_nb_iter(clf_parameters, nb_iter)
    logging.info('init Randomized search...')
    return RandomizedSearchCV(clf_pipeline, clf_parameters, scoring=scoring, cv=cross_val, n_jobs=nb_workers, n_iter=nb_iter, verbose=1,
                              refit=True)


def save_classifier(path_out, classif, clf_name, params, feature_names=None, label_names=None):
    """ pickle {'params', 'name', 'clf_pipeline', 'features', 'label_names'} to ``path_out/classifier_<name>.pkl`` and return its path
    (reference classification.py:547-586)

    >>> import tempfile
    >>> clf = create_classifiers()['RandForest']
    >>> with tempfile.TemporaryDirectory() as tmp:
    ...     p_clf = save_classifier(tmp, clf, 'TESTINNG', {})
    ...     d_clf = load_classifier(p_clf)
    >>> os.path.basename(p_clf)
    'classifier_TESTINNG.pkl'
    >>> sorted(d_clf.keys())
    ['clf_pipeline', 'features', 'label_names', 'name', 'params']
    >>> d_clf['clf_pipeline']  # doctest: +ELLIPSIS
    RandomForestClassifier(...)
    """
    if not os.path.isdir(path_out):
        raise FileNotFoundError('missing folder: %s' % path_out)
    dict_classif = {
        'params': params,
        'name': clf_name,
        'clf_pipeline': classif,
        'features': feature_names,
        'label_names': label_names,
    }
    path_clf = os.path.join(path_out, TEMPLATE_NAME_CLF.format(clf_name))
    logging.info('export classif. of %s to "%s"', dict_classif, path_clf)
    with open(path_clf, 'wb') as f:
        pickle.dump(dict_classif, f)
    return path_clf


def load_classifier(path_classif):
    """ the dictionary ``save_classifier`` wrote, or None when the file does not exist (reference classification.py:589-605)

    >>> load_classifier('none.abc')
    """
    logging.info('import classifier from "%s"', path_classif)
    if not os.path.isfile(path_classif):
        logging.debug('classifier does not exist')
        return None
    with open(path_classif, 'rb') as f:
        dict_clf = pickle.load(f)
    logging.debug('load classifier: %r', dict_clf.keys())
    return dict_clf


def export_results_clf_search(path_out, clf_name, clf_search):
    """ the search's ``cv_results_`` and best parameters as ``classif_<name>_search_params_{scores,best}.txt`` (reference
    classification.py:608-632)"""
    if not os.path.isdir(path_out):
        raise FileNotFoundError('missing folder: %s' % path_out)

    def _fn_path_out(s):
        return os.path.join(path_out, 'classif_%s_%s.txt' % (clf_name, s))

    with open(_fn_path_out('search_params_scores'), 'w') as fp:
        results = 'no results'
        if hasattr(clf_search, 'cv_results_'):
            results = '\n'.join(['"%s": %r' % (k, clf_search.cv_results_[k]) for k in clf_search.cv_results_])
        fp.write(results)
    with open(_fn_path_out('search_params_best'), 'w') as fp:
        params = clf_search.best_params_
        rows = ['{:30s} {}'.format('"{}":'.format(k), params[k]) for k in params]
        fp.write('\n'.join(rows))


def feature_scoring_selection(features, labels, names=None, path_out=''):
    """ score every feature and rank them by the importances of ``ExtraTreesClassifier(n_estimators=125, random_state=0)`` (reference
    classification.py:474-544); the forest is fitted on the device (``forest_fit.fit_extra_trees``), node for node scikit-learn's

    :param ndarray features: np.array<nb_samples, nb_features>
    :param ndarray labels: np.array<nb_samples, 1>
    :param list(str) names: the feature names ('1' .. 'D' when None or shorter than the features)
    :param str path_out: a directory to write ``NAME_CSV_FEATURES_SELECT`` into, when it exists
    :return tuple(list(int),DF): indices of decreasing importance, DataFrame of the scores

    >>> from sklearn.datasets import make_classification
    >>> features, labels = make_classification(
    ...     n_samples=250, n_features=5, n_informative=3, n_redundant=0, n_repeated=0,
    ...     n_classes=2, random_state=0, shuffle=False)
    >>> indices, df_scoring = feature_scoring_selection(features, labels)  # doctest: +ELLIPSIS
    >>> indices
    array([1, 0, 2, 3, 4]...)
    >>> df_scoring.sort_index(axis=1)  # doctest: +NORMALIZE_WHITESPACE +ELLIPSIS
             ExtTree    F-test    k-Best variance
    feature
    1        0.24...   0.75...   0.75...  2.49...
    2        0.33...  58.94...  58.94...  1.85...
    3        0.22...   2.24...   2.24...  1.54...
    4        0.10...   4.02...   4.02...  0.96...
    5        0.09...   0.02...   0.02...  1.01...
    >>> features[:, 2] = 1
    >>> path_out = 'test_fts-select'
    >>> os.mkdir(path_out)
    >>> indices, df_scoring = feature_scoring_selection(features.tolist(), labels.tolist(), path_out=path_out)
    >>> indices  # doctest: +ELLIPSIS
    array([1, 0, 3, 4, 2]...)
    >>> import shutil
    >>> shutil.rmtree(path_out, ignore_errors=True)
    """
    import pandas as pd
    from sklearn import feature_selection
    from .forest_fit import fit_extra_trees
    logging.info('Feature selection for %s', names)
    features = np.array(features) if not isinstance(features, np.ndarray) else features
    labels = np.array(labels) if not isinstance(labels, np.ndarray) else labels
    logging.debug('Features: %r and labels: %r', features.shape, labels.shape)
    forest = fit_extra_trees(ensemble.ExtraTreesClassifier(n_estimators=125, random_state=0), features, labels)
    if forest is None:
        forest = ensemble.ExtraTreesClassifier(n_estimators=125, random_state=0).fit(features, labels)
    f_test, _ = feature_selection.f_regression(features, labels)
    k_best = feature_selection.SelectKBest(feature_selection.f_classif, k='all')
    k_best.fit(features, labels)
    variances = feature_selection.VarianceThreshold().fit(features, labels)
    imp = collections.OrderedDict([('ExtTree', forest.feature_importances_), ('k-Best', k_best.scores_),
                                   ('variance', variances.variances_), ('F-test', f_test)])
    indices = np.argsort(forest.feature_importances_)[::-1]
    nb_features = features.shape[1]
    if names is None or len(names) < nb_features:
        names = [str(i) for i in range(1, nb_features + 1)]
    names = list(names)[:nb_features]
    df_scoring = pd.DataFrame({k: [v[i] for i in range(nb_features)] for k, v in imp.items()},
                              index=pd.Index(names, name='feature'))
    logging.debug(df_scoring)
    if os.path.exists(path_out):
        path_csv = os.path.join(path_out, NAME_CSV_FEATURES_SELECT)
        logging.debug('export Feature scoting to "%s"', path_csv)
        df_scoring.to_csv(path_csv)
    return indices, df_scoring


def _fit_pipeline(clf_pipeline, features, labels):
    """``clf_pipeline.fit(features, labels)`` with a tree or forest as the final step fitted on the device: the transforms are fitted on
    the host by scikit-learn, their output cast to float32 and the classifier fitted by ``forest_fit.fit_tree_model``.  Any other
    classifier, or parameters the device does not compute, keep scikit-learn's fit."""
    from sklearn.base import clone
    from .forest_fit import _supported, fit_tree_model
    steps = clf_pipeline.steps
    name, final = steps[-1]
    if type(clf_pipeline) is not pipeline.Pipeline or _supported(final) is None:
        return clf_pipeline.fit(features, labels)
    Xt = np.asarray(features)
    for _, step in steps[:-1]:
        if step is None or (isinstance(step, str) and step == 'passthrough'):
            continue
        Xt = step.fit_transform(Xt, labels)
    fitted = fit_tree_model(clone(final), np.asarray(Xt, dtype=np.float32), labels)
    if fitted is None:
        fitted = clone(final).fit(Xt, labels)
    clf_pipeline.steps[-1] = (name, fitted)
    return clf_pipeline


def create_classif_search_train_export(clf_name, features, labels, cross_val=10, nb_search_iter=100, search_type='random',
                                       eval_metric='f1', nb_workers=NB_WORKERS_SERACH, path_out=None, params=None, pca_coef=0.98,
                                       feature_names=None, label_names=None):
    """ the pipeline ``create_clf_pipeline(clf_name, pca_coef)``, its parameters searched when ``nb_search_iter > 1`` or
    ``search_type == 'grid'``, fitted on all features and exported to ``path_out`` when that is a directory (reference
    classification.py:656-759).  Returns (fitted pipeline, path of the exported classifier or ``path_out``).  The final fit of a
    ``'RandForest'`` / ``'DecTree'`` pipeline runs on the device (see the module's description).

    >>> np.random.seed(0)
    >>> lbs = np.random.randint(0, 3, 150)
    >>> fts = np.random.random((150, 5)) + np.tile(lbs, (5, 1)).T
    >>> _, _ = create_classif_search_train_export('LogistRegr', fts, lbs, nb_search_iter=0)
    """
    if not list(labels):
        raise RuntimeError('some labels has to be given')
    features = np.nan_to_num(features)
    if len(features) != len(labels):
        raise ValueError('features (%i) and labels (%i) should have equal length' % (len(features), len(labels)))
    if not (features.ndim == 2 and features.shape[1] > 0):
        raise ValueError('at least one feature is required')
    logging.debug('training data: %r, labels (%i): %r', features.shape, len(labels), collections.Counter(labels))
    logging.info('create Classifier: %s', clf_name)
    clf_pipeline = create_clf_pipeline(clf_name, pca_coef)
    if nb_search_iter > 1 or search_type == 'grid':
        logging.debug('Performing param search...')
        nb_labels = len(np.unique(labels))
        clf_search = create_classif_search(clf_name, clf_pipeline, nb_labels=nb_labels, search_type=search_type, cross_val=cross_val,
                                           eval_metric=eval_metric, nb_iter=nb_search_iter, nb_workers=nb_workers)
        clf_search.fit(features, relabel_sequential(labels))
        logging.info('Best score: %r', clf_search.best_score_)
        clf_pipeline = clf_search.best_estimator_
        logging.info('Best parameters set: \n %r', clf_pipeline.get_params())
        if path_out is not None and os.path.isdir(path_out):
            export_results_clf_search(path_out, clf_name, clf_search)
    clf_pipeline = _fit_pipeline(clf_pipeline, features, labels)
    if path_out is not None and os.path.isdir(path_out):
        path_classif = save_classifier(path_out, clf_pipeline, clf_name, params, feature_names, label_names)
    else:
        path_classif = path_out
    return clf_pipeline, path_classif


# ---------------------------------------------------------------------------------------------------------------------
# cross-validation: the fold generators, scores and mean ROC (every fold's tree or forest in one grouped device fit)
# ---------------------------------------------------------------------------------------------------------------------

def _device_folds(classif):
    """whether the folds of ``classif`` are fitted through forest_fit.TreeBatch: a supported tree / forest, or a Pipeline ending in one"""
    from .forest_fit import _supported
    final = classif.steps[-1][1] if type(classif) is pipeline.Pipeline else classif
    return _supported(final) is not None


def _fit_folds(classif, features, labels, fold_lists, catch=True):
    """one fitted clone of ``classif`` per (train, test) of every list of ``fold_lists`` (None where its fit raised), as scikit-learn's
    ``cross_val_score`` fits them one after the other: per fold the transforms of a Pipeline are fitted on the host by scikit-learn
    (``fit_transform`` of the training rows, as ``Pipeline.fit``) and the final tree or forest is prepared, and every tree of every fold
    is built in one grouped device fit.  ``fold_lists`` may be a generator: each list is split only after the folds before it are
    prepared, so a splitter that draws from numpy's global RNG draws at scikit-learn's place.  ``catch=False`` raises the error of a
    failing fit."""
    from sklearn.base import clone
    from .forest_fit import TreeBatch
    X = np.asarray(features)
    y = np.asarray(labels)
    batch = TreeBatch(y)
    out = []
    for folds in fold_lists:
        models = []
        for train, _ in folds:
            model = clone(classif)
            train = np.asarray(train)
            if train.dtype == bool:
                train = np.nonzero(train)[0]
            try:
                if type(model) is pipeline.Pipeline:
                    Xt = X[train]
                    for _, step in model.steps[:-1]:
                        if step is None or (isinstance(step, str) and step == 'passthrough'):
                            continue
                        Xt = step.fit_transform(Xt, y[train])
                    batch.add(model.steps[-1][1], Xt, train)
                else:
                    batch.add(model, X[train], train)
            except Exception:
                if not catch:
                    raise
                logging.exception('fit of a cross-validation fold')
                model = None
            models.append(model)
        out.append(models)
    fitted = iter(batch.fit())
    for models in out:
        for j, model in enumerate(models):
            if model is None:
                continue
            final = next(fitted)
            if type(model) is pipeline.Pipeline:
                model.steps[-1] = (model.steps[-1][0], final)
            else:
                models[j] = final
    return out


def _fold_scores(models, folds, scorer, features, labels):
    """scikit-learn's ``cross_val_score`` of the fitted ``models`` (``error_score=nan``): NaN and a warning where a fit or a score
    failed, ValueError when every fit failed"""
    from sklearn.exceptions import FitFailedWarning
    X = np.asarray(features)
    y = np.asarray(labels)
    if all(m is None for m in models):
        raise ValueError('All the %d fits failed.' % len(models))
    if any(m is None for m in models):
        warnings.warn('%d fits failed out of a total of %d; their score is nan' % (sum(m is None for m in models), len(models)),
                      FitFailedWarning)
    scores = []
    for model, (_, test) in zip(models, folds):
        score = np.nan
        if model is not None:
            try:
                score = scorer(model, X[test], y[test])
            except Exception:
                warnings.warn('Scoring failed. The score on this train-test partition for these parameters will be set to nan.',
                              UserWarning)
        scores.append(score)
    return np.asarray(scores, dtype=np.float64)


def eval_classif_cross_val_scores(clf_name, classif, features, labels, cross_val=10, path_out=None, scorings=METRIC_SCORING):
    """ the cross-validation scores of ``classif`` for every scoring of ``scorings``, one row per fold (reference
    classification.py:762-850), as a DataFrame, written to ``path_out`` as ``NAME_CSV_CLASSIF_CV_SCORES`` 'all-folds' and, with more
    than one row, 'statistic' (``describe()``).

    As the reference: the folds come from ``check_cv(cross_val, labels, classifier=True)`` -- an int gives ``StratifiedKFold``, an
    iterable of (train, test) such as :class:`CrossValidateGroups` is used as it is -- the labels are renumbered with
    ``relabel_sequential`` when there are two or fewer, each scoring refits every fold, a failing scoring leaves its column out, and a
    failing fit or score gives NaN.  A ``'RandForest'`` / ``'DecTree'`` classifier, alone or at the end of a Pipeline, has the trees of
    all (scoring, fold) pairs built in one grouped device fit (``forest_fit.TreeBatch``) with the transforms fitted fold by fold on the
    host; every score is scikit-learn's scorer of the fitted pipeline on the held-out rows.  Other classifiers go through
    scikit-learn's ``cross_val_score``.

    >>> labels = np.array([0] * 150 + [1] * 100 + [2] * 50)
    >>> data = np.tile(labels, (6, 1)).T.astype(float)
    >>> data += 0.5 - np.random.random(data.shape)
    >>> from sklearn.model_selection import StratifiedKFold
    >>> cv = StratifiedKFold(n_splits=5, random_state=0, shuffle=True)
    >>> df = eval_classif_cross_val_scores('KNN', create_classifiers()['KNN'], data, labels, cv)
    >>> df.round(decimals=1).values.tolist()[0]
    [1.0, 1.0, 1.0, 1.0]
    """
    import pandas as pd
    from sklearn.model_selection import check_cv, cross_val_score
    df_scoring = pd.DataFrame()
    if _device_folds(classif):
        prepared = []

        def _folds_of_each_scoring():
            lbs = labels
            for scoring in scorings:
                try:
                    uq_labels = np.unique(lbs)
                    if len(uq_labels) <= 2:
                        lbs = relabel_sequential(lbs, uq_labels)
                    scorer = metrics.check_scoring(classif, scoring=scoring)
                    folds = list(check_cv(cross_val, lbs, classifier=True).split(features, lbs))
                except Exception:
                    logging.exception('model_selection.cross_val_score')
                    continue
                prepared.append((scoring, scorer, folds, lbs))
                yield folds
        try:    # the labels every scoring trains on: relabel_sequential is the same for each
            labels_fit = relabel_sequential(labels, np.unique(labels)) if len(np.unique(labels)) <= 2 else labels
        except Exception:
            labels_fit = labels                         # every scoring fails on the same relabelling, nothing is fitted
        fitted = _fit_folds(classif, features, np.asarray(labels_fit), _folds_of_each_scoring())
        for (scoring, scorer, folds, lbs), models in zip(prepared, fitted):
            try:
                scores = _fold_scores(models, folds, scorer, features, lbs)
                logging.info('Cross-Val score (%s = %f):\n %r', scoring, np.mean(scores), scores)
                df_scoring[scoring] = scores
            except Exception:
                logging.exception('model_selection.cross_val_score')
    else:
        for scoring in scorings:
            try:
                uq_labels = np.unique(labels)
                if len(uq_labels) <= 2:
                    labels = relabel_sequential(labels, uq_labels)
                scores = cross_val_score(classif, features, labels, cv=cross_val, scoring=scoring)
                logging.info('Cross-Val score (%s = %f):\n %r', scoring, np.mean(scores), scores)
                df_scoring[scoring] = scores
            except Exception:
                logging.exception('model_selection.cross_val_score')

    if path_out is not None:
        if not os.path.exists(path_out):
            raise FileNotFoundError('missing: "%s"' % path_out)
        df_scoring.to_csv(os.path.join(path_out, NAME_CSV_CLASSIF_CV_SCORES.format(clf_name, 'all-folds')))
    if len(df_scoring) > 1:
        df_stat = df_scoring.describe()
        logging.info('cross_val scores: \n %r', df_stat)
        if path_out is not None:
            df_stat.to_csv(os.path.join(path_out, NAME_CSV_CLASSIF_CV_SCORES.format(clf_name, 'statistic')))
    else:
        logging.warning('no statistic collected')
    return df_scoring


def eval_classif_cross_val_roc(clf_name, classif, features, labels, cross_val, path_out=None, nb_steps=100):
    """ the mean ROC curve over the folds of ``cross_val`` and every label (one-vs-rest), as a DataFrame of ``nb_steps`` (FP, TP)
    rows, and its AUC (reference classification.py:853-950); written to ``path_out`` as ``NAME_CSV_CLASSIF_CV_ROC`` and
    ``NAME_TXT_CLASSIF_CV_AUC`` ('mean').  As the reference: labels must be non-negative, ``cross_val`` is an iterable of (train, test)
    or has ``split``, the i-th unique label is scored with ``predict_proba(...)[:, i]``, each fold's curve is closed by (0, 0) and
    (1, 1) and interpolated (``np.interp``) at ``linspace(0, 1, nb_steps)``, and the mean curve starts at 0 and ends at 1.  The trees
    of a ``'RandForest'`` / ``'DecTree'`` classifier (alone or ending a Pipeline) of every fold are built in one grouped device fit.

    >>> np.random.seed(0)
    >>> labels = np.array([0] * 150 + [1] * 100 + [3] * 50)
    >>> data = np.tile(labels, (6, 1)).T.astype(float)
    >>> data += np.random.random(data.shape)
    >>> from sklearn.model_selection import StratifiedKFold
    >>> cv = StratifiedKFold(n_splits=5, random_state=0, shuffle=True)
    >>> fp_tp, auc = eval_classif_cross_val_roc('KNN', create_classifiers()['KNN'], data, labels, cv, nb_steps=11)
    >>> fp_tp.shape, round(auc, 2)
    ((11, 2), 0.94)
    """
    import pandas as pd
    from sklearn.base import clone
    uq_labels = np.unique(labels)
    if np.any(uq_labels < 0):
        raise ValueError('some labels are negative: %r' % uq_labels)
    # one-vs-rest targets, column i for the i-th unique label
    targets = (np.asarray(labels).reshape(-1, 1) == uq_labels.reshape(1, -1)).astype(np.float64)
    folds = cross_val if hasattr(cross_val, '__iter__') else cross_val.split(features, labels)
    if _device_folds(classif):
        folds = list(folds)
        fitted = _fit_folds(classif, features, labels, [folds], catch=False)[0]
    else:
        fitted = None
    grid = np.linspace(0, 1, nb_steps)
    tpr_sum, n_curves = np.zeros(nb_steps), 0
    for k, (train, test) in enumerate(folds):
        if fitted is None:
            model = clone(classif).fit(np.copy(features[train], order='C'), np.copy(labels[train], order='C'))
        else:
            model = fitted[k]
        proba = model.predict_proba(np.copy(features[test], order='C'))
        for i in range(len(uq_labels)):
            fpr, tpr, _ = metrics.roc_curve(targets[test, i], proba[:, i])
            # the curve closed by (0, 0) and (1, 1), sampled on the grid; the sum is taken curve by curve
            tpr_sum += np.interp(grid, [0.] + fpr.tolist() + [1.], [0.] + tpr.tolist() + [1.])
            n_curves += 1
    mean_tpr = tpr_sum / float(n_curves)
    mean_tpr[0], mean_tpr[-1] = 0.0, 1.0
    df_roc = pd.DataFrame(np.array([grid, mean_tpr]).T, columns=['FP', 'TP'])
    auc = metrics.auc(grid, mean_tpr)
    if path_out is not None:
        if not os.path.exists(path_out):
            raise FileNotFoundError('missing: "%s"' % path_out)
        df_roc.to_csv(os.path.join(path_out, NAME_CSV_CLASSIF_CV_ROC.format(clf_name, 'mean')))
        with open(os.path.join(path_out, NAME_TXT_CLASSIF_CV_AUC.format(clf_name, 'mean')), 'w') as fp:
            fp.write(str(auc))
    logging.debug('cross_val ROC: \n %r', df_roc)
    return df_roc, auc


class HoldOut(object):
    """ one split: the first ``hold_out`` indices train, the rest test; with ``rand_seed`` (default 0; None or False: keep the order)
    the indices are shuffled after ``np.random.seed(rand_seed)`` (reference classification.py:1401-1453)

    >>> ho = HoldOut(10, 7, rand_seed=None)
    >>> len(ho), list(ho)
    (1, [([0, 1, 2, 3, 4, 5, 6], [7, 8, 9])])
    >>> list(HoldOut(10, 7, rand_seed=0))
    [([2, 8, 4, 9, 1, 6, 7], [3, 0, 5])]
    """

    def __init__(self, nb_samples, hold_out, rand_seed=0):
        if nb_samples <= hold_out:
            raise ValueError('total %i should be higher than hold Idx %i' % (nb_samples, hold_out))
        self._total = nb_samples
        self.hold_out = hold_out
        self._indexes = list(range(nb_samples))
        if rand_seed is not None and rand_seed is not False:
            np.random.seed(rand_seed)
            np.random.shuffle(self._indexes)

    def __iter__(self):
        yield self._indexes[:self.hold_out], self._indexes[self.hold_out:]

    def __len__(self):
        return 1


class CrossValidate(object):
    """ folds of ``nb_hold_out`` test samples (a count, or a fraction of ``nb_samples`` when below 1) walking over ``indexes`` (shuffled
    after ``np.random.seed(rand_seed)`` when a seed is given), the rest training (reference classification.py:1456-1604).

    - A fold that would start fewer than ``ignore_overflow`` samples (a count, or a fraction when below 1) before the end is dropped.
    - A last fold that runs past the end by more than ``ignore_overflow`` takes its missing test samples from the first indices, and
      trains on the samples between; by less, it is kept short.
    - When more than half is held out, the folds are built for the complement and train and test are swapped ("reverse mode").

    >>> cv = CrossValidate(7, 3, rand_seed=0)
    >>> list(cv)  # doctest: +NORMALIZE_WHITESPACE
    [([3, 0, 5, 4], [6, 2, 1]),
     ([6, 2, 1, 4], [3, 0, 5]),
     ([1, 3, 0, 5], [4, 6, 2])]
    >>> len(CrossValidate(340, 0.33, ignore_overflow=0.0)), len(CrossValidate(340, 0.33, ignore_overflow=0.05))
    (4, 3)
    """

    def __init__(self, nb_samples, nb_hold_out, rand_seed=None, ignore_overflow=0.01):
        if nb_samples <= nb_hold_out:
            raise ValueError('Number of holdout has to be smaller then total size.')
        if nb_hold_out <= 0:
            raise ValueError('Number of holdout has to be positive number.')
        self._nb_samples = nb_samples
        self._nb_hold_out = int(np.round(nb_samples * nb_hold_out)) if nb_hold_out < 1 else nb_hold_out
        ignore_overflow = abs(ignore_overflow)
        self._ignore_overflow = int(np.round(nb_samples * ignore_overflow)) if ignore_overflow < 1 else ignore_overflow
        if self._nb_hold_out <= self._ignore_overflow:
            raise ValueError('The tolerance of overflowing (%i) the split has to be larger than the number of hold out samples (%i).'
                             % (self._ignore_overflow, self._nb_hold_out))
        # more held out than kept: build the folds of the complement and swap train and test
        self._revert = self._nb_hold_out > self._nb_samples / 2.
        if self._revert:
            self._nb_hold_out = self._nb_samples - self._nb_hold_out
        self.indexes = list(range(self._nb_samples))
        self._shuffle = rand_seed is not None and rand_seed is not False
        if self._shuffle:
            np.random.seed(rand_seed)
            np.random.shuffle(self.indexes)
        self.iter = 0

    def _starts(self):
        """the first position of every fold, without those starting within ``ignore_overflow`` of the end"""
        return [i for i in range(0, self._nb_samples, self._nb_hold_out) if self._nb_samples - i >= self._ignore_overflow]

    def __iter__(self):
        for begin in self._starts():
            end = begin + self._nb_hold_out
            test = self.indexes[begin:end]
            train = self.indexes[:begin] + self.indexes[end:]
            over = end - self._nb_samples
            if over > self._ignore_overflow:
                # the last fold runs past the end: its test wraps onto the first indices, its training set is what lies between
                test += self.indexes[:over]
                train = self.indexes[over:begin]
            if self._revert:
                train, test = test, train
            yield train, test

    def __len__(self):
        return len(self._starts())


class CrossValidateGroups(CrossValidate):
    """ :class:`CrossValidate` over groups of consecutive samples (``set_sizes``: the samples of each group, e.g. the superpixels of
    each image): ``nb_hold_out`` counts groups, and a fold yields the sample indices of its groups in fold order (reference
    classification.py:1607-1705).

    >>> cv = CrossValidateGroups([2, 2, 1, 2, 1], 2, rand_seed=0)
    >>> cv.set_indexes, cv.indexes
    ([[0, 1], [2, 3], [4], [5, 6], [7]], [2, 0, 1, 3, 4])
    >>> list(cv)  # doctest: +NORMALIZE_WHITESPACE
    [([2, 3, 5, 6, 7], [4, 0, 1]),
     ([4, 0, 1, 7], [2, 3, 5, 6]),
     ([0, 1, 2, 3, 5, 6], [7, 4])]
    """

    def __init__(self, set_sizes, nb_hold_out, rand_seed=None, ignore_overflow=0.01):
        super(CrossValidateGroups, self).__init__(len(set_sizes), nb_hold_out, rand_seed, ignore_overflow)
        self._set_sizes = list(set_sizes)
        ends = np.cumsum([0] + self._set_sizes).tolist()
        self.set_indexes = [list(range(b, e)) for b, e in zip(ends[:-1], ends[1:])]

    def _samples(self, groups):
        return [i for g in groups for i in self.set_indexes[g]]

    def __iter__(self):
        for train, test in super(CrossValidateGroups, self).__iter__():
            yield self._samples(train), self._samples(test)
