"""
Drop-in alias: ``import imsegm.pipelines`` (``superpixels``, ``descriptors``, ``graph_cuts``) resolves to the
H100-native implementation in ``pyimsegm_b200`` for the SLIC -> features -> GraphCut hot path of Borda/pyImSegm and for the
region growing (RG2SP) built on it, and for ``labeling``, ``ellipse_fitting``, ``annotation`` and ``classification``.  Of
``classification`` the scoring (segmentations against annotations), the training-set preparation (class balancing, k-means
down-sampling on the device), the classifier training (random forests and decision trees fitted on the device) and the
cross-validation (the fold generators, scores and mean ROC, every fold's forest built in one grouped device fit) and the feature
scoring (the extra-trees importances fitted on the device, node for node scikit-learn's) are provided: every public name of the
reference's module.  ``center_detection`` is the object-centre detection of the reference's experiments (point features at the
superpixel centres, the candidate classifier and the DBSCAN clustering of the candidates).
"""
import sys

import pyimsegm_b200
from pyimsegm_b200 import annotation, center_detection, classification, descriptors, ellipse_fitting, graph_cuts, labeling, pipelines, region_growing, superpixels, tiled, utilities

for _name in ('annotation', 'center_detection', 'classification', 'descriptors', 'ellipse_fitting', 'graph_cuts', 'labeling', 'pipelines', 'region_growing', 'superpixels', 'tiled', 'utilities'):
    sys.modules[__name__ + '.' + _name] = getattr(pyimsegm_b200, _name)

__version__ = '0.1.9+b200'
