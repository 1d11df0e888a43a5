"""
Host oracle of the scoring functions of ``imsegm/classification.py`` (test infrastructure, never imported by the product).

Each function composes scikit-learn on the raw pixel arrays in the reference's order; the ``relabel`` step is the labeling oracle's
``relabel_max_overlap_unique``.  Slow by design: it is what the device path is checked against.
"""
import logging

import numpy as np
import pandas as pd
from sklearn import metrics

from oracle.labeling import ImageDimensionError, relabel_max_overlap_unique


def relabel_sequential(labels, uq_labels=None):
    labels = np.asarray(labels)
    uq = np.unique(labels) if uq_labels is None else uq_labels
    table = np.zeros(np.max(uq) + 1)
    for idx, value in enumerate(uq):
        table[value] = idx
    return table[labels].astype(labels.dtype).tolist()


def compute_classif_metrics(y_true, y_pred, metric_averages=('macro', 'weighted')):
    y_true, y_pred = np.array(y_true), np.array(y_pred)
    if y_true.shape != y_pred.shape:
        raise ValueError('shapes %r and %r differ' % (y_true.shape, y_pred.shape))
    uq = np.unique(np.hstack((y_true, y_pred)))
    if len(uq) <= 2:
        y_true, y_pred = relabel_sequential(y_true, uq), relabel_sequential(y_pred, uq)
    try:
        metrics.precision_recall_fscore_support(y_true, y_pred)
    except Exception:
        logging.debug('per-class scores failed')
    out = {
        'ARS': metrics.adjusted_rand_score(y_true, y_pred),
        'accuracy': metrics.accuracy_score(y_true, y_pred),
        'confusion': metrics.confusion_matrix(y_true, y_pred).tolist(),
    }
    keys = ('precision', 'recall', 'f1', 'support')
    for avg in metric_averages:
        try:
            vals = metrics.precision_recall_fscore_support(y_true, y_pred, average=avg)
        except Exception:
            vals = [-1] * 4
        out.update({'%s_%s' % (k, avg): v for k, v in zip(keys, vals)})
    return out


def compute_tp_tn_fp_fn(annot, segm, label_positive=None):
    y_true, y_pred = np.asarray(annot).ravel(), np.asarray(segm).ravel()
    uq = np.unique([y_true, y_pred]).tolist()
    if len(uq) > 2:
        return np.nan, np.nan, np.nan, np.nan
    if len(uq) < 2:
        return len(y_true), 0, 0, 0
    pos = label_positive if label_positive is not None and label_positive in uq else uq[-1]
    neg = [v for v in uq if v != pos][0]
    tp = np.sum((y_true == pos) & (y_pred == pos))
    tn = np.sum((y_true == neg) & (y_pred == neg))
    fp = np.sum((y_true == pos) & (y_pred == neg))
    fn = np.sum((y_true == neg) & (y_pred == pos))
    return tp, tn, fp, fn


def compute_metric_fpfn_tpfn(annot, segm, label_positive=None):
    tp, _, fp, fn = compute_tp_tn_fp_fn(annot, segm, label_positive)
    return 0. if (fp + fn) == 0 else float(fp + fn) / float(tp + fn)


def compute_metric_tpfp_tpfn(annot, segm, label_positive=None):
    tp, _, fp, fn = compute_tp_tn_fp_fn(annot, segm, label_positive)
    return 0. if (tp + fn) == 0 else float(tp + fp) / float(tp + fn)


def compute_classif_stat_segm_annot(annot_segm_name, drop_labels=None, relabel=False):
    annot, segm, name = annot_segm_name
    if segm.shape != annot.shape:
        raise ImageDimensionError('shapes %r and %r differ' % (segm.shape, annot.shape))
    y_true, y_pred = annot.ravel(), segm.ravel()
    if drop_labels is not None:
        keep = np.ones(y_true.shape, dtype=bool)
        for lb in drop_labels:
            keep &= (y_true != lb) & (y_pred != lb)
        y_true, y_pred = y_true[keep], y_pred[keep]
    if relabel:
        y_pred = relabel_max_overlap_unique(y_true, y_pred, keep_bg=False)
    stat = compute_classif_metrics(y_true, y_pred, metric_averages=['macro'])
    if len(np.unique(y_pred)) == 2:
        stat['(FP+FN)/(TP+FN)'] = compute_metric_fpfn_tpfn(y_true, y_pred)
        stat['(TP+FP)/(TP+FN)'] = compute_metric_tpfp_tpfn(y_true, y_pred)
    stat['name'] = name
    return stat


def compute_stat_per_image(segms, annots, names=None, nb_workers=2, drop_labels=None, relabel=False):
    if len(segms) != len(annots):
        raise RuntimeError('%i segmentations and %i annotations' % (len(segms), len(annots)))
    names = names or [str(i) for i in range(len(segms))]
    rows = [compute_classif_stat_segm_annot((a, s, n), drop_labels, relabel) for a, s, n in zip(annots, segms, names)]
    return pd.DataFrame(rows).set_index('name')
