"""
Generate tests/golden/reference_vectors.npz by RUNNING THE REFERENCE ITSELF where that is possible in this container.

    IMSEGM_REFERENCE=<reference checkout> python tests/golden/make_goldens.py   (needs oracle/_ref/features_cython, i.e. `make -C oracle ref`)

What runs: the reference's own modules imported from $IMSEGM_REFERENCE -- imsegm.descriptors, imsegm.graph_cuts, imsegm.labeling,
imsegm.superpixels -- with its only native module (features_cython.pyx) compiled unchanged into oracle/_ref.  Packages that are
not installable here (scikit-image, gco, matplotlib, nibabel, ...) are replaced by inert stubs, so only functions that never touch
them can be called: the colour / gray statistics and their drivers, the Leung-Malik bank and the whole texture descriptor (scipy +
features_cython), the label histogram and Ray kernels, the GraphCut energies (unary, pairwise, edge model, spatial distances), the
region/annotation histogram, the grid graph.  SLIC (scikit-image) and the max-flow (gco) cannot run: their parity stays "unpinned"
(oracle headers, DESIGN.md section 2).  Nothing of the reference is copied: this script calls it and stores inputs and outputs.
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ['IMSEGM_REFERENCE']


def import_reference():
    for name, val in (('int', int), ('float', float), ('bool', bool), ('Inf', np.inf), ('NaN', np.nan), ('row_stack', np.vstack)):
        if not hasattr(np, name):       # NumPy-2 removed aliases the reference still uses
            setattr(np, name, val)

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

        def __iter__(self):
            return iter(())

        def __mro_entries__(self, bases):
            return (object, )

    for root in ('skimage', 'matplotlib', 'nibabel', 'gco', 'planar', 'olefile', 'OleFileIO_PL', 'PIL'):
        sys.modules.setdefault(root, Stub(root))
    for sub in ('skimage.segmentation', 'skimage.measure', 'skimage.morphology', 'skimage.filters', 'skimage.color', 'skimage.io',
                'skimage.draw', 'skimage.transform', 'matplotlib.pyplot', 'matplotlib.cm', 'matplotlib.colors', 'matplotlib.patches',
                'matplotlib.pylab', 'matplotlib.backends', 'matplotlib.gridspec', 'matplotlib.path', 'matplotlib.figure', 'PIL.Image',
                'PIL.ImageDraw'):
        root, leaf = sub.split('.', 1)
        getattr(sys.modules[root], leaf)
    sys.path.insert(0, ROOT)
    import oracle
    oracle.build()
    fc = oracle.ref_features_cython()
    assert fc is not None, 'oracle/_ref/features_cython is missing: run `make -C oracle ref`'
    sys.path.insert(0, REF)
    import imsegm
    sys.modules['imsegm.features_cython'] = fc
    imsegm.features_cython = fc
    mods = {m: importlib.import_module('imsegm.' + m) for m in ('descriptors', 'graph_cuts', 'labeling', 'superpixels')}
    assert mods['descriptors'].USE_CYTHON, 'the reference fell back to its NumPy variants'
    return mods


def main():
    ref = import_reference()
    ds, gc, lb, sp = ref['descriptors'], ref['graph_cuts'], ref['labeling'], ref['superpixels']
    rng = np.random.RandomState(20240923)
    out = {}
    # ---- colour statistics over block-like segments (descriptors.py:209-296, 787-863)
    img = rng.random_sample((48, 64, 3))
    img[:, 32:] *= 0.5
    seg = (np.arange(48)[:, None] // 12) * 4 + (np.arange(64)[None, :] // 16)
    seg = seg + (rng.rand(48, 64) < 0.05)                           # ragged borders, all labels 0..16 present or not
    seg = seg.astype(int)
    out.update(color_img=img, color_seg=seg,
               color_mean=ds.cython_img2d_color_mean(img, seg), color_energy=ds.cython_img2d_color_energy(img, seg),
               color_std=ds.cython_img2d_color_std(img, seg))
    fts, names = ds.compute_image2d_color_statistic(img, seg, ('mean', 'std', 'energy', 'median', 'meanGrad'))
    out.update(color_statistic=fts, color_statistic_names=np.array(names))
    # ---- gray volume statistics (descriptors.py:458-551, 679-784)
    vol = rng.random_sample((4, 20, 24))
    vseg = (np.arange(20)[None, :, None] // 7) * 3 + (np.arange(24)[None, None, :] // 8) + 9 * (np.arange(4)[:, None, None] // 2)
    vseg = np.ascontiguousarray(np.broadcast_to(vseg, vol.shape)).astype(int)
    out.update(gray_vol=vol, gray_seg=vseg, gray_mean=ds.cython_img3d_gray_mean(vol, vseg), gray_energy=ds.cython_img3d_gray_energy(vol, vseg),
               gray_std=ds.cython_img3d_gray_std(vol, vseg))
    fts, names = ds.compute_image3d_gray_statistic(vol, vseg)
    out.update(gray_statistic=fts, gray_statistic_names=np.array(names))
    # ---- Leung-Malik bank and the texture descriptor of a colour image (descriptors.py:880-1106) -- scipy + features_cython
    bank, bank_names = ds.create_filter_bank_lm_2d(sigmas=ds.SHORT_FILTERS_SIGMAS, nb_orient=4)
    out.update(lm_short_bank=np.concatenate(bank, axis=0), lm_short_names=np.array(bank_names))
    timg = rng.random_sample((40, 56, 3))
    yy, xx = np.mgrid[:40, :56]
    timg[..., 0] += 0.5 * np.sin(xx / 2.0)
    timg[..., 1] += 0.5 * np.sin((xx + yy) / 3.0) * (xx > 28)
    tseg = ((yy // 20) * 2 + (xx // 28)).astype(int)
    fts, names = ds.compute_texture_desc_lm_img2d_clr(timg, tseg, ('mean', 'std', 'energy'), 'short')
    out.update(lm_img=timg, lm_seg=tseg, lm_short_features=fts, lm_short_feature_names=np.array(names))
    resp = ds.compute_img_filter_response2d(timg[..., 0], bank[0])
    out.update(lm_response_edge0=resp)
    # ---- label histogram / Ray kernels (features_cython.pyx:222-282 through descriptors.py:1479, :1628)
    hseg = rng.randint(0, 4, (15, 17))
    selem = (rng.rand(15, 17) < 0.6).astype(int)
    out.update(hist_seg=hseg, hist_selem=selem, hist=ds.cython_label_hist_seg2d(hseg.astype(float), selem, 4))
    rseg = np.zeros((60, 70), dtype=int)
    rseg[(yy[:60, :70] if False else np.mgrid[:60, :70][0] - 28) ** 2 + (np.mgrid[:60, :70][1] - 33) ** 2 >= 20 ** 2] = 1
    rseg[10:14, 30:40] = 1
    pos = [(28, 33), (20, 40), (35, 25)]
    out.update(ray_seg=rseg, ray_pos=np.array(pos), ray_up=np.array([ds.cython_ray_features_seg2d(rseg, p, 15., 'up') for p in pos]),
               ray_down=np.array([ds.cython_ray_features_seg2d(1 - rseg, p, 15., 'down') for p in pos]))
    # ---- GraphCut energies (graph_cuts.py:303-336, 383-439, 442-555)
    proba = rng.dirichlet(np.ones(3) * 0.7, 30)
    edges = np.array(sorted({tuple(sorted(e)) for e in rng.randint(0, 30, (80, 2)) if e[0] != e[1]}))
    centres = rng.random_sample((30, 2)) * 100
    out.update(gc_proba=proba, gc_edges=edges, gc_centres=centres, gc_unary=gc.compute_unary_cost(proba),
               gc_pairwise_potts=gc.compute_pairwise_cost(2.5, proba.shape),
               gc_pairwise_list=gc.compute_pairwise_cost([((0, 1), 2.0), ((1, 2), 0.5)], proba.shape),
               gc_edge_model_lT=gc.compute_edge_model(edges, proba, 'lT'), gc_edge_model_l1=gc.compute_edge_model(edges, proba, 'l1'),
               gc_edge_model_l2=gc.compute_edge_model(edges, proba, 'l2'),
               gc_spatial=gc.compute_spatial_dist(centres, edges), gc_spatial_rel=gc.compute_spatial_dist(centres, edges, relative=True))
    # ---- grid graph and region / annotation histogram (superpixels.py:115-177, labeling.py:208-283)
    _, g_edges = sp.make_graph_segm_connect_grid2d_conn4(seg)
    annot = (img[..., 0] > 0.35).astype(int) + (img[..., 1] > 0.6)
    out.update(graph_edges=np.array(g_edges), annot=annot, region_hist_norm=lb.histogram_regions_labels_norm(seg, annot))
    return out


if __name__ == '__main__':
    vectors = main()
    path = os.path.join(HERE, 'reference_vectors.npz')
    np.savez_compressed(path, **vectors)
    print('wrote %s: %d arrays, %.0f KB' % (path, len(vectors), os.path.getsize(path) / 1024))
