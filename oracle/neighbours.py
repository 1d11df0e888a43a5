"""
Host oracle of the k-nearest-neighbour and logistic-regression ``predict_proba`` evaluated by ``isb_knn_predict_proba`` /
``isb_linear_predict_proba`` (test infrastructure, never imported by the product).

The definitions, restated in numpy:

- the squared distance of a query x to a training row t is sum_d (x_d - t_d)^2, added in feature order onto zero, every step
  rounded: the bits of a left-to-right float64 loop;
- the neighbours are the k smallest by (squared distance, training index): among equal distances the lower index wins;
- uniform weights give the class counts / k; distance weights give w = 1 / sqrt(d^2), or the indicator d^2 == 0 when a row has any
  zero distance (scikit-learn's ``_get_weights``), added per class in ascending neighbour order and divided by the row sum;
- logistic regression: d = x . coef_k + intercept_k; one coefficient row gives [1 - expit(d), expit(d)], more give the softmax
  (subtract the row maximum, exp, divide by the row sum).
"""
import numpy as np

#: queries per block of the distance loop (bounds the [block, N_t] temporary)
_BLOCK_BYTES = 1 << 26


def squared_distances(x, fit_x):
    """[N, N_t] squared distances, each summed over the features left to right"""
    x, fit_x = np.asarray(x, dtype=np.float64), np.asarray(fit_x, dtype=np.float64)
    out = np.empty((len(x), len(fit_x)))
    step = max(1, _BLOCK_BYTES // (8 * max(len(fit_x), 1)))
    for a in range(0, len(x), step):
        xb = x[a:a + step]
        acc = np.zeros((len(xb), len(fit_x)))
        for d in range(x.shape[1]):
            diff = xb[:, d, None] - fit_x[None, :, d]
            acc += diff * diff
        out[a:a + step] = acc
    return out


def kneighbours(x, fit_x, k):
    """(squared distances [N, k], training indices [N, k]) of the k nearest by (squared distance, index), ascending"""
    d2 = squared_distances(x, fit_x)
    kth = np.partition(d2, k - 1, axis=1)[:, k - 1:k]
    rows, cols = np.nonzero(d2 <= kth)                       # every row has >= k candidates, more only on ties with the k-th
    order = np.lexsort((cols, d2[rows, cols], rows))         # by row, then squared distance, then training index
    start = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=len(d2)))[:-1]])
    take = order[start[:, None] + np.arange(k)[None]]
    idx = cols[take]
    return np.take_along_axis(d2, idx, axis=1), idx


def knn_predict_proba(x, fit_x, y, k, n_classes, weights='uniform'):
    """KNeighborsClassifier.predict_proba (Euclidean) by the definitions above; y: class indices [N_t] in [0, n_classes)"""
    d2, idx = kneighbours(x, fit_x, k)
    labels = np.asarray(y)[idx]
    if weights == 'uniform':
        w = np.ones_like(d2)
    elif weights == 'distance':
        with np.errstate(divide='ignore'):
            w = 1.0 / np.sqrt(d2)
        zero = d2[:, 0] == 0.0                               # sorted: a zero distance, if any, comes first
        w[zero] = (d2[zero] == 0.0)
    else:
        raise ValueError('weights must be uniform or distance, not %r' % (weights, ))
    rows = np.arange(len(x))
    proba = np.zeros((len(x), n_classes))
    for j in range(k):
        proba[rows, labels[:, j]] += w[:, j]
    norm = np.zeros(len(x))
    for c in range(n_classes):                               # the row sum, class by class
        norm += proba[:, c]
    norm[norm == 0.0] = 1.0
    return proba / norm[:, None]


def linear_predict_proba(x, coef, intercept):
    """LogisticRegression.predict_proba from coef_ [1 or K, D] and intercept_"""
    dec = np.asarray(x, dtype=np.float64) @ np.asarray(coef, dtype=np.float64).T + np.asarray(intercept, dtype=np.float64)
    if dec.shape[1] == 1:
        e = 1.0 / (1.0 + np.exp(-dec[:, 0]))
        return np.stack([1.0 - e, e], axis=1)
    dec = dec - dec.max(axis=1, keepdims=True)
    dec = np.exp(dec)
    return dec / dec.sum(axis=1, keepdims=True)
