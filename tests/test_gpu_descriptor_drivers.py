"""
The Python drivers of imsegm/descriptors.py around the native kernels -- label histograms about positions (:1288-1528),
Ray features of many positions (:1805-1884), gray-volume statistics (:679-784) -- against the reference's own doctest values
and against the oracle on random inputs.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _disk_px(cx, cy, r, shape):
    """skimage.draw.disk as the reference's _draw_disk wraps it (utilities/drawing.py:874-900): (dx^2 + dy^2) < r^2"""
    xx, yy = np.mgrid[:shape[0], :shape[1]]
    return np.nonzero((xx - cx) ** 2 + (yy - cy) ** 2 < r ** 2)


def test_label_histograms_positions_reference_doctests_and_oracle(oracle):
    from pyimsegm_b200 import descriptors as ds
    segm = np.zeros((10, 10), dtype=int)
    segm[1:9, 2:8] = 1
    segm[3:7, 4:6] = 2
    points = [[3, 3], [4, 4], [2, 7], [6, 6]]
    hists, names = ds.compute_label_histograms_positions(segm, points, [1, 2, 4])
    assert names == ['hist-d_%i-lb_%i' % (d, lb) for d in (1, 2, 4) for lb in range(3)] and hists.shape == (4, 9)
    want = np.array([[0., 0.8, 0.2, 0.12, 0.62, 0.25, 0.44, 0.41, 0.15], [0., 0.2, 0.8, 0., 0.62, 0.38, 0.22, 0.75, 0.03],
                     [0.2, 0.8, 0., 0.5, 0.5, 0., 0.46, 0.33, 0.21], [0., 0.8, 0.2, 0.12, 0.62, 0.25, 0.44, 0.41, 0.15]])
    assert np.array_equal(np.round(hists, 2), want)
    proba = np.zeros((10, 10, 2), dtype=int)
    proba[3:7, 4:6, 1] = 1
    proba[:, :, 0] = 1 - proba[:, :, 0]
    hists, _ = ds.compute_label_histograms_positions(proba, points, [1, 2, 4])
    want = np.array([[1., 0.2, 1., 0.25, 1., 0.15], [1., 0.8, 1., 0.38, 1., 0.03], [1., 0., 1., 0., 1., 0.21], [1., 0.2, 1., 0.25, 1., 0.15]])
    assert np.array_equal(np.round(hists, 2), want)
    # compute_label_hist_segm :1406-1424, compute_label_hist_proba :1511-1516
    hist, size = ds.compute_label_hist_segm(segm, [6, 6], np.ones((3, 3)), 3)
    assert hist.tolist() == [0., 7., 2.] and size == 9.0
    hist, size = ds.compute_label_hist_segm(segm, [4, 4], np.ones((5, 5)), 3)
    assert hist.tolist() == [0., 17., 8.] and size == 25.0
    seg = np.zeros((50, 50, 2), dtype=float)
    seg[15:35, 20:40, 1] = 1
    seg[:, :, 0] = 1 - seg[:, :, 1]
    hist, size = ds.compute_label_hist_proba(seg, (15, 20), np.ones((12, 13), dtype=int))
    assert hist.tolist() == [114., 42.] and size == 156
    # random segmentation, default diameters, positions at the borders too
    rng = np.random.RandomState(5)
    big = rng.randint(0, 5, (90, 120))
    pts = [(0, 0), (89, 119), (45, 60), (3, 117), (88, 2)] + [tuple(p) for p in rng.randint(0, 90, (20, 2))]
    got, _ = ds.compute_label_histograms_positions(big, pts)
    np.testing.assert_allclose(got, oracle.label_histograms_positions(big, pts, ds.HIST_CIRCLE_DIAGONALS), rtol=1e-12, atol=1e-15)
    soft = rng.dirichlet(np.ones(4), (90, 120))
    got, _ = ds.compute_label_histograms_positions(soft, pts, [3, 7, 15])
    np.testing.assert_allclose(got, oracle.label_histograms_positions(soft, pts, [3, 7, 15]), rtol=1e-10)
    with pytest.raises(ValueError):
        ds.compute_label_hist_segm(segm, [6, 6, 1], np.ones((3, 3)), 3)


def test_ray_features_positions_reference_doctest(oracle):
    """imsegm/descriptors.py:1830-1845: rays of three positions, 20 degree steps, phase shift"""
    from pyimsegm_b200 import descriptors as ds
    seg = np.zeros((100, 100), dtype=int)
    seg[_disk_px(45, 55, 30, seg.shape)] = 1
    seg[_disk_px(55, 45, 10, seg.shape)] = 2
    points = [(50, 50), (60, 40), (44, 55)]
    ray_dist, shift, names = ds.compute_ray_features_positions(seg, points, 20)
    assert [int(s * 10) for s in shift] == [3143, 3147, 900]
    assert ray_dist.astype(int).tolist() == [[37, 37, 35, 32, 30, 27, 25, 24, 23, 23, 24, 25, 26, 30, 31, 33, 35, 38],
                                             [50, 47, 41, 31, 23, 17, 13, 10, 9, 9, 9, 11, 14, 19, 27, 37, 45, 50],
                                             [31, 31, 31, 30, 30, 29, 30, 30, 29, 29, 30, 30, 29, 30, 30, 31, 31, 31]]
    assert names[:3] == ['ray-lb_0-agl_0', 'ray-lb_0-agl_20', 'ray-lb_0-agl_40'] and len(names) == 18
    # one position through the single-position driver == the batched row before shifting; both against the oracle tracer
    single = ds.compute_ray_features_segm_2d(seg == 0, points[1], 20)
    rows, _, _ = ds.compute_ray_features_positions(seg, points, 20, shifting=False)
    assert np.array_equal(single, rows[1])
    np.testing.assert_allclose(single, oracle.ray_features2d(seg == 0, points[1], 20., 1), rtol=1e-6)
    smooth = ds.compute_ray_features_segm_2d(seg == 0, points[0], 10, smooth_coef=2)
    assert smooth.shape == (36, ) and np.all(np.abs(np.diff(smooth)) < 4)
    # descriptors.py:1846-1858: salt noise on the mask, removed by the opening with a disc of radius 10 (device morphology)
    np.random.seed(0)
    noise_pos = np.random.randint(10, 80, (2, 300))
    seg[noise_pos[0], noise_pos[1]] = 0
    ray_dist, shift, names = ds.compute_ray_features_positions(seg, points, 45, segm_open=10)
    assert names == ['ray-lb_0-agl_%d' % a for a in range(0, 360, 45)]
    assert [int(round(s)) for s in shift] == [315, 315, 90]
    assert ray_dist.astype(int).tolist() == [[38, 35, 29, 25, 24, 25, 29, 35], [52, 41, 21, 11, 9, 11, 21, 41], [31, 31, 30, 29, 29, 29, 30, 31]]


def test_gray_volume_statistics_reference_doctest():
    """imsegm/descriptors.py:714-735 and :1117-1127"""
    from pyimsegm_b200 import descriptors as ds
    image = np.zeros((2, 3, 8))
    image[0, :, 2:6] = 1
    image[1, :, 3:7] = 3
    segm = np.array([[[0, 0, 0, 0, 1, 1, 1, 1]] * 3, [[2, 2, 2, 2, 5, 5, 5, 5]] * 3])
    features, names = ds.compute_image3d_gray_statistic(image, segm)
    assert names == ['gray_mean', 'gray_std', 'gray_energy', 'gray_median', 'gray_meanGrad'] and features.shape == (6, 5)
    want = np.array([[0.5, 0.5, 0.5, 0.5, 0.25], [0.5, 0.5, 0.5, 0.5, -0.25], [0.75, 1.299, 2.25, 0., 0.75], [0., 0., 0., 0., 0.],
                     [0., 0., 0., 0., 0.], [2.25, 1.299, 6.75, 3., -1.125]])
    np.testing.assert_allclose(np.round(features, 3), want)
    rng = np.random.RandomState(0)
    img = rng.random_sample((2, 10, 15))
    slic = np.zeros((2, 10, 15), dtype=int)
    slic[:, :, :7] += 1
    slic[1, :, :] += 2
    fts, names = ds.compute_selected_features_gray3d(img, slic, {'color': ('mean', 'std', 'median')})
    assert fts.shape == (4, 3) and names == ['gray_mean', 'gray_std', 'gray_median']
    for k, fn in enumerate((ds.numpy_img3d_gray_mean, ds.numpy_img3d_gray_std, ds.numpy_img3d_gray_median)):
        np.testing.assert_allclose(fts[:, k], fn(img, slic), rtol=1e-6)
    fts, names = ds.compute_selected_features_gray3d(img, slic, {'tLM_short': ('mean', 'std', 'energy')})
    assert fts.shape == (4, 45) and names[0] == 'tLM_sigma1.4-edge_mean' and names[-1] == 'tLM_sigma4.0-GaussLap2_energy'


def test_generic_filter_response_and_gray_volume_texture_match_scipy():
    """compute_img_filter_response2d/3d (:951-983), image_subtract_gauss_smooth (:986-1000), compute_texture_desc_lm_img3d_val
    (:1003-1038): the device FP64 utilities against scipy.ndimage, which is what the reference calls"""
    from scipy import ndimage
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(4)
    vol = rng.random_sample((3, 37, 52))
    bank, bank_names = ds.create_filter_bank_lm_2d(sigmas=ds.SHORT_FILTERS_SIGMAS, nb_orient=4)
    for battery in (bank[0], bank[2], rng.normal(0, 1, (3, 5, 7))):
        want = np.array([np.max([ndimage.convolve(sl, k) for k in battery], axis=0) for sl in vol])
        np.testing.assert_allclose(ds.compute_img_filter_response3d(vol, battery), want, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(ds.compute_img_filter_response2d(vol[1], battery), want[1], rtol=1e-12, atol=1e-14)
    for sigma in (1.5, 150):
        want = vol - np.array([ndimage.gaussian_filter(sl, sigma) for sl in vol])
        np.testing.assert_allclose(ds.image_subtract_gauss_smooth(vol, sigma), want, rtol=1e-11, atol=1e-13)
    with pytest.raises(ValueError):
        ds.compute_img_filter_response2d(vol[0], bank[0][0])
    # the whole gray-volume texture descriptor against a scipy restatement of the reference's steps
    seg = np.zeros(vol.shape, dtype=int)
    seg[:, :, 26:] = 1
    seg[2] += 2
    got, names = ds.compute_texture_desc_lm_img3d_val(vol, seg, ('mean', 'std', 'energy'), 'short')
    hp = vol - np.array([ndimage.gaussian_filter(sl, 150) for sl in vol])
    cols = []
    for battery in bank:
        resp = np.array([np.max([ndimage.convolve(sl, k) for k in battery], axis=0) for sl in hp])
        resp[resp > ds.MAX_SIGNAL_RESPONSE] = ds.MAX_SIGNAL_RESPONSE
        norm = np.sqrt(np.sum(resp ** 2))
        resp = resp * (np.log(1 + norm) / 0.03) / norm
        cols.append(np.stack([ds.numpy_img3d_gray_mean(resp, seg), ds.numpy_img3d_gray_std(resp, seg), ds.numpy_img3d_gray_energy(resp, seg)], 1))
    want = np.concatenate(cols, axis=1)
    assert got.shape == want.shape == (4, 45) and len(names) == 45
    np.testing.assert_allclose(got, want, rtol=2e-5, atol=1e-7)    # the native statistics read the responses as f32 (features_cython.pyx)


def test_supervised_data_step_labels_follow_the_annotation():
    """wrapper_compute_color2d_slic_features_labels (imsegm/pipelines.py:272-290)"""
    from conftest import synth_regions
    from pyimsegm_b200 import pipelines as pl
    img, truth = synth_regions(200, 260, seed=8)
    annot = truth.copy()
    annot[:20] = -1                                           # an unknown strip
    slic, fts, labels = pl.wrapper_compute_color2d_slic_features_labels((img, annot), 15, 0.25, {'color': ['mean']}, 0.9)
    assert slic.shape == truth.shape and fts.shape == (slic.max() + 1, 3) and labels.shape == (slic.max() + 1, )
    inside = np.array([np.bincount(truth[slic == k], minlength=3).argmax() for k in range(slic.max() + 1)])
    known = labels >= 0
    assert known.mean() > 0.7 and np.array_equal(labels[known], inside[known])
    assert np.all(labels[np.unique(slic[:8])] == -1)          # superpixels inside the unknown strip
    with pytest.raises(NotImplementedError):
        pl.train_classif_color2d_slic_features([img], [annot], {'color': ['mean']})


def test_binary_opening_equals_scipy_grey_opening():
    """binary_opening_disk: erosion then dilation with a disc, reflected borders (what skimage.morphology.opening does on a
    boolean image through scipy.ndimage.grey_erosion / grey_dilation); a non-integer radius against the oracle's opening"""
    from scipy import ndimage
    from oracle import ellipse as oe
    from pyimsegm_b200 import descriptors as ds
    rng = np.random.RandomState(3)
    mask = ndimage.gaussian_filter(rng.random_sample((70, 95)), 2) > 0.5
    for radius in (1, 3, 6):
        yy, xx = np.mgrid[-radius:radius + 1, -radius:radius + 1]
        disk = (yy ** 2 + xx ** 2) <= radius ** 2
        want = ndimage.grey_dilation(ndimage.grey_erosion(mask.astype(np.uint8), footprint=disk), footprint=disk).astype(bool)
        assert np.array_equal(ds.binary_opening_disk(mask, radius), want)
    assert np.array_equal(ds.binary_opening_disk(mask, 1.5), oe.opening(mask.astype(np.uint8), oe.disk(1.5)).astype(bool))


def test_segment_median_on_the_device(oracle):
    """isb_segment_median against np.median per label (reference descriptors.py:420-455, 651-676), odd and even counts, every dtype,
    an absent label; and the reference's doctest values (:429-437)"""
    from pyimsegm_b200 import descriptors as ds
    image = np.zeros((2, 10, 3))
    image[:, 2:6, 0] = 1
    image[:, 3:8, 1] = 3
    image[:, 4:9, 2] = 2
    segm = np.array([[0, 0, 0, 0, 1, 1, 1, 1, 1, 1]] * 2)
    np.testing.assert_allclose(ds.numpy_img2d_color_median(image, segm), [[0.5, 0., 0.], [0., 3., 2.]])
    rng = np.random.RandomState(5)
    seg = rng.randint(0, 41, (60, 77))
    seg[seg == 17] = 18                      # label 17 is absent -> NaN
    for dtype in (np.float64, np.float32, np.uint8, np.uint16):
        img = (rng.random_sample((60, 77, 3)) * 200).astype(dtype)
        got = ds.numpy_img2d_color_median(img, seg)
        want = oracle.color2d_median(img, seg)
        assert np.isnan(got[17]).all()
        np.testing.assert_array_equal(np.delete(got, 17, 0), np.delete(want, 17, 0))
    img3 = np.array([[[0] * 3 + [1] * 3 + [2] * 2] * 3] * 2, dtype=float)[:, :, :8]          # doctest volume of descriptors.py:698-715
    seg3 = np.array([[[0] * 2 + [1] * 2 + [2] * 2 + [5] * 2] * 3] * 2)
    np.testing.assert_allclose(ds.numpy_img3d_gray_median(img3, seg3)[[0, 1, 2, 5]], [0., 0.5, 1., 2.])
    vol = rng.random_sample((4, 20, 30))
    vseg = rng.randint(0, 9, vol.shape)
    want = np.array([np.median(vol[vseg == k]) for k in range(9)])
    np.testing.assert_array_equal(ds.numpy_img3d_gray_median(vol, vseg), want)
