"""
Drop-in alias: ``import imsegm.pipelines`` (``superpixels``, ``descriptors``, ``graph_cuts``) resolves to the
H100-native implementation in ``pyimsegm_b200`` for the SLIC -> features -> GraphCut hot path of Borda/pyImSegm and for the
region growing (RG2SP) built on it.  Modules of the reference outside that path (classification, annotation, ...) are not provided.
"""
import sys

import pyimsegm_b200
from pyimsegm_b200 import descriptors, graph_cuts, labeling, pipelines, region_growing, superpixels, tiled, utilities

for _name in ('descriptors', 'graph_cuts', 'labeling', 'pipelines', 'region_growing', 'superpixels', 'tiled', 'utilities'):
    sys.modules[__name__ + '.' + _name] = getattr(pyimsegm_b200, _name)

__version__ = '0.1.9+b200'
