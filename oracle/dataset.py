"""
Float64 oracle of the k-means down-sampling of ``balance_dataset_by_(..., 'kmeans')`` (pyimsegm_b200/classification.py): one Lloyd sweep
with exact differences, the per-sample assignment margin, and scikit-learn's own KMeans runs for a seed.
"""
import numpy as np


def sq_distances(X, centres):
    """exact squared distances [n, k]: sum over the features of (x - c)^2, the differences taken first"""
    X, centres = np.asarray(X, np.float64), np.asarray(centres, np.float64)
    return ((X[:, None, :] - centres[None, :, :]) ** 2).sum(axis=2)


def assign(X, centres, chunk=2048):
    """(labels [n] int64, best distance [n], margin [n]) of the rows against the centres: the nearest centre (lowest index on ties),
    its exact squared distance, and the second-least minus the least squared distance (inf with one centre)"""
    X = np.asarray(X, np.float64)
    labels = np.empty(len(X), np.int64)
    best = np.empty(len(X))
    margin = np.full(len(X), np.inf)
    for lo in range(0, len(X), chunk):
        d = sq_distances(X[lo:lo + chunk], centres)
        lab = np.argmin(d, axis=1)
        labels[lo:lo + chunk] = lab
        best[lo:lo + chunk] = d[np.arange(len(d)), lab]
        if d.shape[1] > 1:
            part = np.partition(d, 1, axis=1)
            margin[lo:lo + chunk] = part[:, 1] - part[:, 0]
    return labels, best, margin


def member_means(X, labels, k):
    """centres [k, D] = the mean of each cluster's rows (NaN rows for empty clusters) and the counts [k]"""
    X = np.asarray(X, np.float64)
    counts = np.bincount(labels, minlength=k)
    sums = np.zeros((k, X.shape[1]))
    np.add.at(sums, labels, X)
    with np.errstate(invalid='ignore', divide='ignore'):
        return sums / counts[:, None], counts


def lloyd_sweep(X, centres):
    """one Lloyd sweep: (labels, new centres, margin of every row) from the given centres"""
    labels, _, margin = assign(X, centres)
    new, _ = member_means(X, labels, len(centres))
    return labels, new, margin


def sklearn_runs(X, k, seed, n_init=3, max_iter=5):
    """scikit-learn's KMeans(k, init='random', n_init, max_iter) of the rows taken apart: the (labels, inertia, centres) of every run,
    in order, from starts drawn by a RandomState(seed) shared by the runs, and the rows that
    np.argmin(KMeans(...).fit_transform(X), axis=0) selects with np.random.seed(seed)"""
    from sklearn.cluster import KMeans
    from sklearn.cluster._kmeans import _kmeans_single_lloyd, _tolerance
    X = np.asarray(X, np.float64)
    tol = _tolerance(X, 1e-4)
    Xc = X - X.mean(axis=0)
    w = np.ones(len(X))
    rs = np.random.RandomState(seed)
    runs = []
    for _ in range(n_init):
        seeds = rs.choice(len(X), size=k, replace=False, p=w / w.sum())
        labels, inertia, centres, _ = _kmeans_single_lloyd(Xc, w, Xc[seeds], max_iter=max_iter, tol=tol)
        runs.append((labels, inertia, centres))
    np.random.seed(seed)
    selected = np.argmin(KMeans(n_clusters=k, init='random', n_init=n_init, max_iter=max_iter).fit_transform(X), axis=0)
    return runs, selected


def selection_ties(X, centres, got, want):
    """(number of centres whose selected rows differ, whether every difference is a rounding tie): for centre j, rows got[j] and
    want[j] are a tie when both lie within tol_j of the least exact squared distance to the centre, tol_j = 8 gamma_(D+2)
    (max_i |x_i|^2 + |c_j|^2) -- what |c|^2 - 2 x.c + |x|^2 in float64 (scikit-learn's euclidean_distances) can get wrong"""
    X, centres = np.asarray(X, np.float64), np.asarray(centres, np.float64)
    u = 2.0 ** -53
    gamma = (X.shape[1] + 2) * u / (1 - (X.shape[1] + 2) * u)
    scale = (X ** 2).sum(axis=1).max()
    diff = np.where(np.asarray(got) != np.asarray(want))[0]
    ok = True
    for j in diff:
        d = ((X - centres[j]) ** 2).sum(axis=1)
        tol = 8 * gamma * (scale + (centres[j] ** 2).sum())
        ok &= bool(d[got[j]] <= d.min() + tol and d[want[j]] <= d.min() + tol)
    return len(diff), ok
