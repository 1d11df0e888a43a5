"""
Float64 oracle of the device class-model fit (``isb_mixture_fit_predict``, pyimsegm_b200/csrc/gmm.cu): scikit-learn's
GaussianMixture / BayesianGaussianMixture started from a given hard assignment, sklearn's rule for choosing among restarts, and the
device's own k-means++ / Lloyd start restated in numpy, with the margins that say when its draws and labels are decided beyond
rounding.  numpy and scikit-learn only.
"""
import numpy as np
from sklearn import mixture

MASK64 = (1 << 64) - 1


class SplitMix64:
    """the device's counter-based generator (``Rng`` of gmm.cu): SplitMix64 over a 64-bit state"""

    def __init__(self, state):
        self.s = int(state) & MASK64

    def next(self):
        self.s = (self.s + 0x9E3779B97F4A7C15) & MASK64
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)

    def uniform(self):
        """a double in [0, 1) from the top 53 bits"""
        return float(self.next() >> 11) * 2.0 ** -53


def start_state(seed, init):
    """generator state of restart ``init`` for ``seed``: seed * 0x100000001B3 + 1469598103934665603 * (init + 1) mod 2^64"""
    return (int(seed) * 0x100000001B3 + 1469598103934665603 * (int(init) + 1)) & MASK64


def _sq_dist(Z, centres):
    """exact squared distances [N, k], the differences taken first"""
    return ((Z[:, None, :] - centres[None, :, :]) ** 2).sum(axis=2)


def _relative_gap(d):
    """per row of squared distances [N, k]: (second least - least) / second least; inf with one centre"""
    if d.shape[1] < 2:
        return np.full(len(d), np.inf)
    part = np.partition(d, 1, axis=1)
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.where(part[:, 1] > 0, (part[:, 1] - part[:, 0]) / part[:, 1], 0.0)


def kmeanspp_labels(Z, K, seed, init, max_rounds=300):
    """the hard start of restart ``init`` that the device draws when no ``init_labels`` are given (``k_gmm_fit`` / ``k_big_init``):
    k-means++ seeding with D^2-weighted draws, then Lloyd rounds.

    Returns ``(labels [N] int32, margins)``; ``margins`` is a dict of
      ``draws``: per draw of a further centre, the distance of the threshold from the nearest prefix sum, over the total;
      ``labels``: the least relative gap between the nearest and the second-nearest centre over every assignment round that counts;
      ``shift``: the least relative distance of a round's centre shift from the 1e-4 stop, over the rounds that changed a label.
    The device adds its sums in another order, so only starts whose margins are well above rounding (~1e-9) are reproducible.
    """
    Z = np.asarray(Z, dtype=np.float64)
    N = len(Z)
    rng = SplitMix64(start_state(seed, init))
    first = min(int(rng.uniform() * N), N - 1)
    centres = [Z[first]]
    d2 = ((Z - Z[first]) ** 2).sum(axis=1)
    draw_margins = []
    for _ in range(1, K):
        total = d2.sum()
        thr = rng.uniform() * total
        prefix = np.cumsum(d2)
        pick = int(np.searchsorted(prefix, thr, side='left'))     # the first index whose running sum is >= thr
        bounds = np.concatenate([[0.0], prefix])
        draw_margins.append(float(np.abs(bounds - thr).min() / total) if total > 0 else 0.0)
        pick = min(pick, N - 1)
        centres.append(Z[pick])
        d2 = np.minimum(d2, ((Z - Z[pick]) ** 2).sum(axis=1))
    centres = np.array(centres)
    labels = np.full(N, -1, dtype=np.int64)
    label_gap, shift_gap = np.inf, np.inf
    for _ in range(max_rounds):
        d = _sq_dist(Z, centres)
        new = np.argmin(d, axis=1)                                  # lowest index on ties, as the strict < of the kernels
        changed = bool((new != labels).any())
        labels = new
        label_gap = min(label_gap, float(_relative_gap(d).min()))
        counts = np.bincount(labels, minlength=K).astype(np.float64)
        sums = np.zeros_like(centres)
        np.add.at(sums, labels, Z)
        has = counts > 0
        moved = centres.copy()
        moved[has] = sums[has] / counts[has, None]
        shift = float(((moved[has] - centres[has]) ** 2).sum())
        centres = moved
        if changed:
            shift_gap = min(shift_gap, abs(shift - 1e-4) / 1e-4)
        if not changed or shift <= 1e-4:
            break
    return labels.astype(np.int32), {'draws': draw_margins, 'labels': label_gap, 'shift': shift_gap}


def kmeanspp_starts(Z, K, seed, n_init):
    """``kmeanspp_labels`` of restarts 0 .. n_init - 1 stacked [n_init, N], and the least margin of each kind over them"""
    rows, least = [], {'draws': np.inf, 'labels': np.inf, 'shift': np.inf}
    for r in range(n_init):
        lab, m = kmeanspp_labels(Z, K, seed, r)
        rows.append(lab)
        least['draws'] = min([least['draws']] + list(m['draws']))
        least['labels'] = min(least['labels'], m['labels'])
        least['shift'] = min(least['shift'], m['shift'])
    return np.stack(rows), least


class SharedStartGMM(mixture.GaussianMixture):
    """GaussianMixture started from a given hard assignment ``y0`` (scikit-learn 1.9's _initialize_parameters)"""

    def __init__(self, y0=None, **kw):
        super().__init__(**kw)
        self.y0 = y0

    def _initialize_parameters(self, X, random_state, xp=None):
        self._initialize(X, np.eye(self.n_components)[self.y0])


class SharedStartBGM(mixture.BayesianGaussianMixture):
    """BayesianGaussianMixture started from a given hard assignment ``y0`` (scikit-learn 1.9's _initialize_parameters)"""

    def __init__(self, y0=None, **kw):
        super().__init__(**kw)
        self.y0 = y0

    def _initialize_parameters(self, X, random_state, xp=None):
        self._initialize(X, np.eye(self.n_components)[self.y0])


def shared_start_fit(Z, y0, K, kind='GMM', max_iter=99, reg_covar=1e-6, tol=1e-3):
    """scikit-learn's mixture of ``kind`` ('GMM': GaussianMixture, 'BGM': BayesianGaussianMixture, full covariances, one restart)
    fitted on the (already scaled) features ``Z`` from the hard assignment ``y0``.  Both start through the model's own
    _initialize(X, one_hot): the parameters of the one-hot responsibilities (nk + 10 eps, reg_covar on the covariance diagonal, the
    precision Cholesky factor of the covariance), which is the device's first M-step.  (weights_init / means_init / precisions_init
    would invert the covariance first; scikit-learn rejects that inverse for a component with fewer members than features.)
    Raises what scikit-learn raises (a start whose covariance is not positive definite: ValueError)."""
    Z = np.asarray(Z, dtype=np.float64)
    y0 = np.asarray(y0).astype(np.int64)
    cls = {'GMM': SharedStartGMM, 'BGM': SharedStartBGM}[kind]
    return cls(y0=y0, n_components=K, covariance_type='full', n_init=1, max_iter=max_iter, reg_covar=reg_covar, tol=tol).fit(Z)


def shared_start_best(Z, Y0, K, kind='GMM', max_iter=99, reg_covar=1e-6, tol=1e-3):
    """one ``shared_start_fit`` per start row of ``Y0`` [n_init, N]; returns (index of the winner, its fitted model, the lower bound
    of every start).  The winner is scikit-learn's: the largest lower bound, the first start on a tie (its strict >)."""
    best, best_model, lowers = -1, None, []
    for r, y0 in enumerate(np.atleast_2d(Y0)):
        m = shared_start_fit(Z, y0, K, kind, max_iter, reg_covar, tol)
        lowers.append(float(m.lower_bound_))
        if best < 0 or m.lower_bound_ > lowers[best]:
            best, best_model = r, m
    return best, best_model, lowers


def tol_margin(model, tol=1e-3):
    """how far the fit's stopping decisions were from rounding: the least | |change of the lower bound| - tol | over its
    iterations after the first (inf when there is only one)"""
    lb = np.asarray(getattr(model, 'lower_bounds_', []), dtype=np.float64)
    if len(lb) < 2:
        return np.inf
    return float(np.abs(np.abs(np.diff(lb)) - tol).min())
