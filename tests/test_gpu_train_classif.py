"""GPU tests of the supervised training on the device: isb_superpixel_train_labels against the reference's label formula (dense
histogram, np.argmax, purity), isb_unique_rows_rounded against balance_dataset_by_(..., 'unique'), and
pipelines.train_classif_images_batch against the composition of the existing stage functions under the same seeds."""
import random

import numpy as np
import pytest

from test_train_classif_host import reference_labels

pytestmark = pytest.mark.gpu

FEATS = {'color': ['mean', 'std', 'energy']}


def device_labels(slic, annot, purity):
    from pyimsegm_b200 import pipelines as pl
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    nb = int(slic.max()) + 1
    d_seg = eng.to_device(np.ascontiguousarray(slic, dtype=np.int32))
    d_annot = eng.to_device(pl.train_annotation(slic, annot))
    return eng.to_host(eng.train_labels(d_seg, nb, d_annot, purity)).copy()


def block_map(h, w, bh, bw, seed):
    """superpixels as bh x bw blocks, numbered in a random order"""
    rng = np.random.RandomState(seed)
    ids = np.arange(((h + bh - 1) // bh) * ((w + bw - 1) // bw))
    rng.shuffle(ids)
    grid = ids.reshape((h + bh - 1) // bh, (w + bw - 1) // bw)
    return np.repeat(np.repeat(grid, bh, 0), bw, 1)[:h, :w]


def _label_cases():
    rng = np.random.RandomState(3)
    blocks = block_map(20, 24, 5, 2, 0)                            # 48 superpixels of 10 pixels
    pair = np.zeros_like(blocks)
    pair[:, 1::2] = 4
    yield 'tie of two labels', blocks, pair + 1, 0.0
    yield 'tie with unknown', blocks, np.where(pair == 4, -1, 6), 0.0
    yield 'unknown largest', blocks, np.where(rng.rand(*blocks.shape) < 0.7, -1, 2), 0.0
    nine = np.zeros_like(blocks)
    for s in range(48):
        nine.ravel()[np.flatnonzero(blocks.ravel() == s)[0]] = 1
    for purity in (0.9, np.nextafter(0.9, 1.0), 0.0, 1.0):
        yield 'purity %r' % purity, blocks, nine, purity
    yield 'mask 0/255', blocks, np.where(rng.rand(*blocks.shape) < 0.35, 255, 0), 0.6
    yield 'near 2^31-1', blocks, rng.randint(2 ** 31 - 3, 2 ** 31, blocks.shape), 0.3
    yield 'float -0.5', blocks, rng.choice([-0.5, -1.5, 0.5, 1.25, 2.0], blocks.shape), 0.3
    yield 'bool', blocks, rng.rand(*blocks.shape) < 0.5, 0.6
    yield 'all -1', blocks, -np.ones(blocks.shape), 0.0
    yield 'one superpixel', np.zeros((37, 53), int), rng.randint(0, 4, (37, 53)), 0.2
    yield 'random labels', rng.randint(0, 50, (64, 80)), rng.randint(-2, 9, (64, 80)), 0.2
    for h, w in ((1, 1), (1, 37), (41, 1), (5, 3), (257, 259)):
        yield '%dx%d' % (h, w), block_map(h, w, 3, 4, h), rng.randint(-1, 3, (h, w)), 0.5
    yield '2048^2', block_map(2048, 2048, 29, 31, 1), rng.randint(0, 3, (2048, 2048)) * (rng.rand(2048, 2048) < 0.9), 0.5


@pytest.mark.parametrize('name, slic, annot, purity', list(_label_cases()), ids=[c[0] for c in _label_cases()])
def test_label_kernel_is_the_reference_formula(name, slic, annot, purity):
    np.testing.assert_array_equal(device_labels(slic, annot, purity), reference_labels(slic, annot, purity))


def test_label_kernel_at_8192_squared():
    slic = block_map(8192, 8192, 61, 67, 2)
    yy, xx = np.mgrid[:8192, :8192]
    annot = np.where((yy - 4000) ** 2 + (xx - 4100) ** 2 < 3000 ** 2, 255, 0)
    annot[::7, ::5] = -1
    got = device_labels(slic, annot, 0.9)
    # the dense histogram of the reference over the three values (0, 255, unknown as 256)
    a = np.where(annot < 0, 256, annot)
    hist = np.bincount(slic.ravel() * 257 + a.ravel(), minlength=(slic.max() + 1) * 257).reshape(-1, 257).astype(float)
    hist = hist / hist.sum(1, keepdims=True)
    want = np.argmax(hist, 1)
    want[want == 256] = -1
    want[hist.max(1) < 0.9] = -1
    np.testing.assert_array_equal(got, want)
    assert (want == 255).any() and (want == 0).any() and (want == -1).any()


def test_wrapper_labels_follow_the_reference_formula():
    """the data step on SLIC maps of colour and gray images (the gray one takes the host superpixels)"""
    from conftest import synth_regions
    from pyimsegm_b200 import pipelines as pl
    img, truth = synth_regions(150, 190, seed=4)
    annot = np.where(np.random.RandomState(0).rand(*truth.shape) < 0.2, -1, truth * 3)
    for image in (img, img[..., 0]):
        slic, fts, labels = pl.wrapper_compute_color2d_slic_features_labels((image, annot), 12, 0.2, FEATS, 0.7)
        slic_c, fts_c = pl.compute_color2d_superpixels_features(image, FEATS, 12, 0.2)
        np.testing.assert_array_equal(slic, slic_c)
        assert np.array_equal(fts, fts_c, equal_nan=True) and not np.isnan(fts).any()
        assert labels.dtype == np.int64
        np.testing.assert_array_equal(labels, reference_labels(slic, annot, 0.7))


def device_unique(table, labels, D=None):
    from pyimsegm_b200.engine import get_engine
    eng = get_engine()
    D = table.shape[1] if D is None else D
    d_feat = eng.to_device(np.ascontiguousarray(table, dtype=np.float64))[:, :D]
    rows, lab, count = eng.unique_rows(d_feat, eng.to_device(np.asarray(labels, dtype=np.int64)), D)
    m = int(eng.to_host(count)[0])
    if m < 0:
        return None
    return eng.to_host(rows[:m]).copy(), eng.to_host(lab[:m]).copy()


def check_unique(table, labels, D=None):
    from pyimsegm_b200.classification import balance_dataset_by_
    D = table.shape[1] if D is None else D
    keep = labels != -1
    rows, lab = device_unique(table, labels, D)
    want_rows, want_lab = balance_dataset_by_(table[keep][:, :D], labels[keep], 'unique')
    assert np.array_equal(rows, want_rows)                       # -0 equals +0
    np.testing.assert_array_equal(lab, want_lab)
    got_counts = np.unique(lab, return_counts=True)
    want_counts = np.unique(want_lab, return_counts=True)
    for g, w in zip(got_counts, want_counts):
        np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize('D', [1, 9, 189])
def test_unique_rows_match_the_host_balancing(D):
    rng = np.random.RandomState(D)
    n = 3000
    table = rng.randint(-3, 4, (n, D)) / 2000.0 + rng.choice([0.0, 1e-5, -4e-4], (n, D))   # half-way points and near-duplicates
    table[rng.rand(n, D) < 0.05] = -0.0
    table[0, 0], table[1, 0], table[2, -1], table[3, -1] = np.inf, -np.inf, 1e308, -1e308
    labels = rng.choice([-1, 0, 2, 5, 2 ** 31 - 1], n, p=[0.2, 0.3, 0.3, 0.1, 0.1])
    labels[10] = 7                                                # a class of one row
    check_unique(table, labels)


def test_unique_rows_edge_classes_and_stride():
    rng = np.random.RandomState(5)
    table = rng.rand(400, 12)
    labels = np.repeat([3, -1, 0, 9], 100)
    table[200:300] = table[200]                                   # a class whose rows are all one row
    check_unique(table, labels, D=7)                              # a row stride of 12 for 7 columns
    one = np.zeros((1, 4))
    check_unique(one, np.array([2]))
    assert device_unique(table, np.full(400, -1))[0].shape == (0, 12)


def test_unique_rows_at_the_superpixels_of_8192_squared():
    rng = np.random.RandomState(6)
    n = 8192 * 8192 // 29 ** 2
    table = np.round(rng.rand(n, 9) * 3, 2) + rng.choice([0, 4e-4, 6e-4], (n, 9))
    labels = rng.randint(-1, 4, n)
    check_unique(table, labels)


def test_unique_rows_refuse_nan():
    table = np.zeros((20, 3))
    table[4, 1] = np.nan
    assert device_unique(table, np.zeros(20, int)) is None
    labels = np.zeros(20, int)
    labels[4] = -1                                                # a dropped row may hold NaN
    assert device_unique(table, labels)[0].shape == (1, 3)


# ---- the driver against the composition of the stage functions ------------------------------------------------------------

def synth_set(n_images, seed, h=96, w=128):
    from conftest import synth_regions
    images, annots = [], []
    for i in range(n_images):
        img, truth = synth_regions(h, w, seed=seed + i)
        annot = truth.copy()
        annot[:6] = -1
        images.append(img)
        annots.append(annot)
    return images, annots


def composition(images, annots, balance, clf_name, pca_coef, sp=12, reg=0.2, purity=0.9, hold_out=2):
    """the reference's train_classif_color2d_slic_features through this package's stage functions"""
    from pyimsegm_b200 import classification as cls
    from pyimsegm_b200 import pipelines as pl
    slics, fts, lbs = [], [], []
    for img, annot in zip(images, annots):
        slic, features = pl.compute_color2d_superpixels_features(img, FEATS, sp, reg)
        slics.append(slic)
        fts.append(features)
        lbs.append(reference_labels(slic, annot, purity))
    features, labels, sizes = cls.convert_set_features_labels_2_dataset(dict(enumerate(fts)), dict(enumerate(lbs)), balance_type=balance,
                                                                        drop_labels=[-1])
    features = np.nan_to_num(features)
    cv = cls.CrossValidateGroups(sizes, nb_hold_out=hold_out) if len(sizes) > hold_out * 5 else 10
    classif, _ = cls.create_classif_search_train_export(clf_name, features, labels, pca_coef=pca_coef, cross_val=cv, nb_search_iter=1,
                                                        nb_workers=1)
    return classif, slics, fts, lbs, (features, labels)


def driver(images, annots, balance, clf_name, pca_coef, nb_streams, monkeypatch):
    from pyimsegm_b200 import classification as cls
    from pyimsegm_b200 import pipelines as pl
    seen = {}
    fit = cls.create_classif_search_train_export

    def capture(clf_name, features, labels, **kw):
        seen['set'] = (features, labels)
        return fit(clf_name, features, labels, **kw)

    monkeypatch.setattr(cls, 'create_classif_search_train_export', capture)
    out = pl.train_classif_images_batch(images, annots, FEATS, sp_size=12, sp_regul=0.2, clf_name=clf_name, feature_balance=balance,
                                        pca_coef=pca_coef, nb_streams=nb_streams)
    monkeypatch.undo()
    return out + (seen['set'], )


def same_estimator(a, b):
    est_a, est_b = a.steps[-1][1], b.steps[-1][1]
    trees_a = [e.tree_ for e in getattr(est_a, 'estimators_', [])] or ([est_a.tree_] if hasattr(est_a, 'tree_') else [])
    trees_b = [e.tree_ for e in getattr(est_b, 'estimators_', [])] or ([est_b.tree_] if hasattr(est_b, 'tree_') else [])
    assert len(trees_a) == len(trees_b)
    for ta, tb in zip(trees_a, trees_b):
        for name in ('feature', 'threshold', 'children_left', 'children_right', 'value'):
            np.testing.assert_array_equal(getattr(ta, name), getattr(tb, name))
    if not trees_a:
        np.testing.assert_array_equal(est_a.coef_, est_b.coef_)
        np.testing.assert_array_equal(est_a.intercept_, est_b.intercept_)


def run_and_compare(n_images, balance, clf_name, pca_coef, monkeypatch, seed=20):
    from pyimsegm_b200 import pipelines as pl
    images, annots = synth_set(n_images, seed)
    np.random.seed(7)
    random.seed(7)
    want = composition(images, annots, balance, clf_name, pca_coef)
    held_out, _ = synth_set(1, seed + 100)
    _, fts_h = pl.compute_color2d_superpixels_features(held_out[0], FEATS, 12, 0.2)
    for nb_streams in (1, 3):
        np.random.seed(7)
        random.seed(7)
        got = driver(images, annots, balance, clf_name, pca_coef, nb_streams, monkeypatch)
        for g, w in zip(got[1:4], want[1:4]):
            assert len(g) == len(w)
            for a, b in zip(g, w):
                assert a.dtype == b.dtype and np.array_equal(a, b)
        assert np.array_equal(got[4][0], want[4][0]) and np.array_equal(got[4][1], want[4][1])
        same_estimator(got[0], want[0])
        for clf in (got[0], want[0]):       # a forest's threaded predict_proba adds the trees in a varying order
            if hasattr(clf.steps[-1][1], 'estimators_'):
                clf.steps[-1][1].n_jobs = None
        np.testing.assert_array_equal(got[0].predict_proba(fts_h), want[0].predict_proba(fts_h))
    return got


@pytest.mark.parametrize('balance', ['unique', 'random', 'kmeans', None])
@pytest.mark.parametrize('clf_name', ['RandForest', 'DecTree', 'LogistRegr'])
@pytest.mark.parametrize('pca_coef', [None, 0.95])
def test_driver_equals_the_composition(balance, clf_name, pca_coef, monkeypatch):
    run_and_compare(3, balance, clf_name, pca_coef, monkeypatch)


@pytest.mark.parametrize('balance', ['unique', 'random', 'kmeans', None])
def test_driver_equals_the_composition_with_group_folds(balance, monkeypatch):
    run_and_compare(11, balance, 'RandForest', None, monkeypatch, seed=40)       # 11 > 5 * nb_hold_out: CrossValidateGroups


@pytest.mark.parametrize('balance', ['unique', 'random', None])
def test_image_without_labelled_superpixel(balance):
    from pyimsegm_b200 import pipelines as pl
    images, annots = synth_set(3, 60)
    annots[1] = -np.ones_like(annots[1])
    if balance is None:
        np.random.seed(1)
        random.seed(1)
        _, _, _, labels = pl.train_classif_images_batch(images, annots, FEATS, sp_size=12, feature_balance=None)
        assert (labels[1] == -1).all()
        return
    with pytest.raises(ValueError):
        composition(images, annots, balance, 'RandForest', None)
    with pytest.raises(ValueError):
        pl.train_classif_images_batch(images, annots, FEATS, sp_size=12, feature_balance=balance)


def test_trained_classifier_segments_as_the_single_image_pipeline():
    from pyimsegm_b200 import pipelines as pl
    images, annots = synth_set(4, 80, h=128, w=160)
    np.random.seed(2)
    random.seed(2)
    classif, _, _, _ = pl.train_classif_images_batch(images[:3], annots[:3], FEATS, sp_size=12)
    batch = pl.segment_images_batch(images, dict_features=FEATS, sp_size=12, model_pipeline=classif)
    for img, (segm, soft) in zip(images, batch):
        want_segm, want_soft = pl.segment_color2d_slic_features_model_graphcut(img, classif, FEATS, sp_size=12)
        np.testing.assert_array_equal(segm, want_segm)
        np.testing.assert_array_equal(soft, want_soft)
