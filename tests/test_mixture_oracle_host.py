"""The float64 oracle of the device mixture fit (oracle/mixture.py) against known values and its own invariants (no GPU needed):
the generator, the k-means++ / Lloyd start, and the restart choice of the shared-start fits."""
import numpy as np

from oracle import mixture as om


def test_generator_is_splitmix64():
    g = om.SplitMix64(0)
    assert g.next() == 0xE220A8397B1DCDAF
    assert om.start_state(0, 0) == 0x14650FB0739D0383
    assert om.SplitMix64(om.start_state(0, 0)).uniform() == 0.30713388322638424
    # the state wraps modulo 2^64 and every restart of a seed starts elsewhere
    assert om.start_state(2 ** 64 - 1, 8) < 2 ** 64
    assert len({om.start_state(s, r) for s in (0, 1, 7) for r in range(9)}) == 27
    assert all(0.0 <= om.SplitMix64(s).uniform() < 1.0 for s in range(1000))


def _blobs(D, K, n, seed, spread=0.05):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(-3, 3, (K, D))
    y = rng.randint(0, K, n)
    return centres[y] + rng.normal(0, spread, (n, D)), y


def test_lloyd_labels_are_a_fixed_point():
    rng = np.random.RandomState(0)
    Z = rng.normal(size=(700, 4))                      # no cluster structure: Lloyd has to move the centres
    for K in (1, 2, 5, 8):
        lab, m = om.kmeanspp_labels(Z, K, seed=3, init=1)
        assert lab.dtype == np.int32 and lab.min() >= 0 and lab.max() < K
        assert len(m['draws']) == K - 1
        cent = np.array([Z[lab == k].mean(0) for k in range(K) if (lab == k).any()])
        ks = np.array([k for k in range(K) if (lab == k).any()])
        d = ((Z[:, None, :] - cent[None]) ** 2).sum(-1)
        # stopped on "no label changed": every sample is labelled with its nearest final centre
        assert np.array_equal(ks[np.argmin(d, axis=1)], lab)


def test_kmeanspp_recovers_far_apart_blobs():
    for D, K in ((3, 3), (40, 3), (2, 8)):
        X, y = _blobs(D, K, 2000, seed=D + K)
        for init in range(3):
            lab, m = om.kmeanspp_labels(X, K, seed=0, init=init)
            conf = np.zeros((K, K), dtype=int)
            np.add.at(conf, (lab, y), 1)
            # a permutation: each label holds exactly one blob (k-means++ may still put two centres into one blob for K = 8, so
            # the bijection is required only where every blob was reached)
            if (conf > 0).sum(0).max() == 1 and (conf > 0).sum(1).max() == 1:
                assert sorted(np.argmax(conf, axis=0)) == list(range(K))
            else:
                assert K == 8
            assert m['labels'] > 0.5                     # blob members are far closer to their own centre


def test_draws_follow_the_prefix_rule():
    """the first centre is int(u N); each further one the first index whose running D^2 sum reaches u * total"""
    rng = np.random.RandomState(5)
    Z = rng.normal(size=(50, 2))
    g = om.SplitMix64(om.start_state(4, 2))
    first = int(g.uniform() * 50)
    d2 = ((Z - Z[first]) ** 2).sum(1)
    thr = g.uniform() * d2.sum()
    second = int(np.argmax(np.cumsum(d2) >= thr))
    # K = 2 with a single Lloyd-free check: the two seeds are the first two centres, so the labels split Z by them at round 0
    lab, m = om.kmeanspp_labels(Z, 2, seed=4, init=2, max_rounds=1)
    d = ((Z[:, None, :] - Z[[first, second]][None]) ** 2).sum(-1)
    assert np.array_equal(lab, np.argmin(d, axis=1))
    assert 0 < m['draws'][0] < 1


def test_shared_start_best_takes_the_first_of_a_tie():
    X, y = _blobs(3, 3, 600, seed=1, spread=0.3)
    rng = np.random.RandomState(2)
    bad = rng.randint(0, 3, len(X))
    Y0 = np.stack([bad, y, y, bad])
    best, model, lowers = om.shared_start_best(X, Y0, 3, 'GMM', max_iter=20)
    assert lowers[1] == lowers[2] and lowers[0] == lowers[3]
    assert best == (1 if lowers[1] >= lowers[0] else 0)
    assert model.lower_bound_ == lowers[best]
    again = om.shared_start_fit(X, Y0[best], 3, 'GMM', max_iter=20)
    np.testing.assert_array_equal(model.means_, again.means_)
    # BGM through its own _initialize
    best, model, lowers = om.shared_start_best(X, Y0[1:3], 3, 'BGM', max_iter=20)
    assert best == 0 and lowers[0] == lowers[1]


def test_shared_start_gmm_first_m_step_is_the_hard_start():
    """max_iter = 1: one E-step from the start and one M-step, so the fit is the M-step of the start's own E-step"""
    X, y = _blobs(4, 3, 500, seed=9, spread=0.5)
    m = om.shared_start_fit(X, y, 3, 'GMM', max_iter=1)
    assert m.n_iter_ == 1 and not m.converged_
    assert om.tol_margin(m) == np.inf
    m = om.shared_start_fit(X, y, 3, 'GMM', max_iter=50)
    assert m.converged_ and om.tol_margin(m) > 0
