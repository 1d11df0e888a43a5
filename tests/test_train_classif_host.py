"""CPU tests of the supervised training data step: the closed-form superpixel label rule that isb_superpixel_train_labels implements
against the reference's formula (dense histogram, np.argmax, purity), the rounding rule of isb_unique_rows_rounded against np.round,
the argument errors of pipelines.train_classif_images_batch, and the argument checks of the two entries -- none of it needs a GPU."""
import numpy as np
import pytest

from pyimsegm_b200.utilities import ImageDimensionError


def reference_labels(slic, annot, label_purity):
    """wrapper_compute_color2d_slic_features_labels of the reference (pipelines.py:272-290) with histogram_regions_labels_norm
    (labeling.py:245-278) in numpy; annotation values are ranked through np.unique, which keeps their order and the argmax ties"""
    annot = np.asarray(annot).astype(int)
    neg_label = np.max(annot) + 1 if np.sum(annot < 0) > 0 else None
    if neg_label is not None:
        annot = annot.copy()
        annot[annot < 0] = neg_label
    values, inv = np.unique(annot, return_inverse=True)
    hist = np.bincount(slic.ravel() * len(values) + inv.ravel(), minlength=(slic.max() + 1) * len(values))
    hist = hist.reshape(slic.max() + 1, len(values)).astype(float)
    sums = np.tile(np.sum(hist, axis=1), (hist.shape[1], 1)).T
    sums[sums == 0] = -1.
    hist = np.nan_to_num(hist / sums)
    hist[hist == 0] = 0
    labels = values[np.argmax(hist, axis=1)]
    purity = np.max(hist, axis=1)
    if neg_label is not None:
        labels[labels == neg_label] = -1
    labels[purity < label_purity] = -1
    return labels


def closed_form_labels(slic, annot, label_purity):
    """the rule of isb_superpixel_train_labels: l* (the smallest label of the largest known count c*) when c* >= u (unknown pixels)
    and c* / n is not below label_purity, else -1"""
    annot = np.asarray(annot).astype(int)
    nb = slic.max() + 1
    n = np.bincount(slic.ravel(), minlength=nb)
    unknown = annot.ravel() < 0
    u = np.bincount(slic.ravel()[unknown], minlength=nb)
    out = np.full(nb, -1, dtype=np.int64)
    known_sp, known_lab = slic.ravel()[~unknown], annot.ravel()[~unknown]
    pairs, counts = np.unique(np.stack([known_sp, known_lab]), axis=1, return_counts=True)
    for s in range(nb):
        sel = pairs[0] == s
        if not sel.any():
            continue
        c = counts[sel].max()
        lab = pairs[1][sel][counts[sel] == c].min()
        if c >= u[s] and not (np.float64(c) / np.float64(n[s]) < label_purity):
            out[s] = lab
    return out


def _cases():
    rng = np.random.RandomState(0)
    yield 'random', rng.randint(0, 40, (30, 37)), rng.randint(-1, 5, (30, 37)), 0.5
    blocks = np.kron(np.arange(12).reshape(3, 4), np.ones((5, 2), dtype=int))        # 12 superpixels of 10 pixels
    tie = np.zeros_like(blocks)
    tie[:, 1::2] = 3
    yield 'tie between labels', blocks, tie, 0.0
    yield 'tie with unknown', blocks, np.where(tie == 3, -1, 7), 0.0
    unk = np.where(rng.rand(*blocks.shape) < 0.7, -4, 2)
    yield 'unknown largest', blocks, unk, 0.0
    nine = np.zeros_like(blocks)
    nine.ravel()[np.flatnonzero(blocks.ravel() == 5)[0]] = 1                         # 9 of 10 pixels of superpixel 5 are 0
    for purity in (0.9, 0.9000001, 0.0, 1.0, -1.0, 1.5):
        yield 'purity %r' % purity, blocks, nine, purity
    yield 'mask 0/255', blocks, np.where(rng.rand(*blocks.shape) < 0.4, 255, 0), 0.9
    yield 'labels near 2^31', blocks, rng.randint(2 ** 31 - 4, 2 ** 31, blocks.shape), 0.2
    yield 'float with -0.5', blocks, rng.choice([-0.5, 0.3, 1.7, -2.2], blocks.shape), 0.3
    yield 'bool', blocks, rng.rand(*blocks.shape) < 0.5, 0.6
    yield 'all -1', blocks, -np.ones_like(blocks), 0.0
    yield 'one superpixel', np.zeros((9, 11), dtype=int), rng.randint(0, 3, (9, 11)), 0.2
    yield '1x1', np.zeros((1, 1), dtype=int), np.ones((1, 1), dtype=int), 0.9


@pytest.mark.parametrize('name, slic, annot, purity', list(_cases()), ids=[c[0] for c in _cases()])
def test_closed_form_label_rule_is_the_reference_formula(name, slic, annot, purity):
    np.testing.assert_array_equal(closed_form_labels(slic, annot, purity), reference_labels(slic, annot, purity))


def test_hand_made_label_cases():
    blocks = np.kron(np.arange(4), np.ones((1, 10), dtype=int))
    annot = np.array([[1] * 5 + [2] * 5 + [4] * 5 + [-1] * 5 + [-1] * 6 + [3] * 4 + [0] * 9 + [1]])
    # tie 1/2 -> 1; tie 4 / unknown -> 4 (purity 0.5); unknown largest -> -1; 9 of 10 at 0.9 kept
    np.testing.assert_array_equal(closed_form_labels(blocks, annot, 0.5), [1, 4, -1, 0])
    np.testing.assert_array_equal(closed_form_labels(blocks, annot, 0.9), [-1, -1, -1, 0])


def test_rounding_rule_is_np_round():
    rng = np.random.RandomState(1)
    x = np.concatenate([rng.randn(200000) * 10.0 ** rng.randint(-4, 6, 200000), (np.arange(-20000, 20000) + 0.5) / 1000.,
                        [0., -0., np.inf, -np.inf, 1e308, -1e308, 5e-324, 0.0005, -0.0005, 0.0015, 2.5e-4]])
    np.testing.assert_array_equal(np.rint(x * 1000.0) / 1000.0, np.round(x, 3))
    assert np.round(1e308, 3) == np.inf


def test_train_annotation_checks():
    from pyimsegm_b200.pipelines import train_annotation
    img = np.zeros((4, 5, 3))
    out = train_annotation(img, np.array([[-0.5, 1.7, -3, 2 ** 31 - 1, 0]] * 4))
    assert out.dtype == np.int32 and out[0].tolist() == [0, 1, -1, 2 ** 31 - 1, 0]
    assert train_annotation(img, np.ones((4, 5), bool)).tolist() == np.ones((4, 5), int).tolist()
    assert (train_annotation(img, -np.ones((4, 5))) == -1).all()
    with pytest.raises(ImageDimensionError):
        train_annotation(img, np.zeros((5, 4)))
    with pytest.raises(ImageDimensionError):
        train_annotation(img, np.zeros((4, 5, 1)))
    with pytest.raises(ValueError):
        train_annotation(img, np.full((4, 5), 2 ** 31))
    with pytest.raises(ValueError):
        train_annotation(img, np.full((4, 5), -3))       # the reference's unknown label max + 1 = -2 is negative


def test_driver_argument_errors_before_any_launch():
    from pyimsegm_b200 import pipelines as pl
    img = np.zeros((16, 16, 3))
    with pytest.raises(ValueError):
        pl.train_classif_images_batch([img, img], [np.zeros((16, 16))], {'color': ['mean']})
    with pytest.raises(ImageDimensionError):
        pl.train_classif_images_batch([img, img], [np.zeros((16, 16)), np.zeros((16, 15))], {'color': ['mean']})
    with pytest.raises(ValueError):
        pl.train_classif_images_batch([img], [np.full((16, 16), 2 ** 33)], {'color': ['mean']})
    with pytest.raises(ValueError):
        pl.train_classif_images_batch([img], [np.zeros((16, 16))], {'color': ['mean']}, sp_regul=0.)
    with pytest.raises(NotImplementedError):
        pl.train_classif_color2d_slic_features([img], [np.zeros((16, 16))], {'color': ['mean']})


def test_entries_check_arguments_without_a_gpu():
    from pyimsegm_b200 import _lib, build
    build.build()
    lib = _lib.lib()
    assert lib.isb_abi_version() == 8
    assert lib.isb_train_labels_workspace_bytes(0, 5, 3) == 0 and lib.isb_train_labels_workspace_bytes(64, 64, 10) >= 18 * 64 * 64
    rc = lib.isb_superpixel_train_labels(None, 4, 4, 2, None, None, 0.9, None, None, 0, None)
    assert rc == _lib.ISB_ERR_ARG and b'null' in lib.isb_last_error()
    fake = 1 << 20                                                  # never dereferenced: the checks come first
    rc = lib.isb_superpixel_train_labels(fake, 0, 4, 2, None, fake, 0.9, fake, fake, 1 << 30, None)
    assert rc == _lib.ISB_ERR_ARG and b'bad sizes' in lib.isb_last_error()
    rc = lib.isb_superpixel_train_labels(fake, 4, 4, 2, None, fake, 0.9, fake, fake, 16, None)
    assert rc == _lib.ISB_ERR_ARG and b'workspace' in lib.isb_last_error()
    assert lib.isb_unique_rows_workspace_bytes(0, 3) == 0
    rc = lib.isb_unique_rows_rounded(None, 10, 3, 3, None, None, None, None, None, None, 0, None)
    assert rc == _lib.ISB_ERR_ARG and b'null' in lib.isb_last_error()
    rc = lib.isb_unique_rows_rounded(fake, 10, 3, 2, None, fake, fake, fake, fake, fake, 1 << 30, None)
    assert rc == _lib.ISB_ERR_ARG and b'bad sizes' in lib.isb_last_error()
    rc = lib.isb_unique_rows_rounded(fake, 10, 3, 3, None, fake, fake, fake, fake, fake, 8, None)
    assert rc == _lib.ISB_ERR_ARG and b'workspace' in lib.isb_last_error()
