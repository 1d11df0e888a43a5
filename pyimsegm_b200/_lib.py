"""
ctypes binding of ``libimsegm_b200.so`` (the C-ABI declared in ``include/imsegm_b200.h``).

There is NO fallback: if the shared library is missing or a CUDA device is absent the calls raise.
torch is used only for device memory (tensors as containers) and streams.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libimsegm_b200.so')

_lib = None

ISB_OK, ISB_ERR_ARG, ISB_ERR_CUDA, ISB_ERR_CAPACITY, ISB_ERR_UNSUPPORTED = 0, -1, -2, -3, -4
DTYPE_CODES = {'uint8': 0, 'uint16': 1, 'float32': 2, 'float64': 3}

_vp, _i, _d, _sz, _ll = C.c_void_p, C.c_int, C.c_double, C.c_size_t, C.c_longlong



class SlicBand(C.Structure):
    """isb_slic_band_t of include/imsegm_b200.h"""
    _fields_ = [('slab_rows', C.c_int32), ('width', C.c_int32), ('image_rows', C.c_int32), ('y_off', C.c_int32),
                ('own_lo', C.c_int32), ('own_hi', C.c_int32), ('halo', C.c_int32),
                ('n_seeds', C.c_int32), ('step_y', C.c_int32), ('step_x', C.c_int32), ('slic_zero', C.c_int32),
                ('step', C.c_double), ('lab_slab', C.c_void_p), ('plane_stride', C.c_size_t), ('seeds_yx', C.c_void_p),
                ('labels_slab', C.c_void_p), ('ws', C.c_void_p), ('ws_bytes', C.c_size_t)]


class Slic3dSlab(C.Structure):
    """isb_slic3d_slab_t of include/imsegm_b200.h"""
    _fields_ = [('depth', C.c_int32), ('height', C.c_int32), ('width', C.c_int32), ('z_off', C.c_int32), ('slab_slices', C.c_int32),
                ('own_lo', C.c_int32), ('own_hi', C.c_int32), ('halo', C.c_int32),
                ('n_seeds', C.c_int32), ('step_z', C.c_int32), ('step_y', C.c_int32), ('step_x', C.c_int32),
                ('step', C.c_double), ('spacing', C.c_double * 3), ('vol_slab', C.c_void_p), ('seeds_zyx', C.c_void_p),
                ('labels_slab', C.c_void_p), ('ws', C.c_void_p), ('ws_bytes', C.c_size_t)]


_bp = C.POINTER(SlicBand)
_sp = C.POINTER(Slic3dSlab)

#: every symbol declared in include/imsegm_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    'isb_last_error': (C.c_char_p, []),
    'isb_abi_version': (_i, []),
    'isb_launch_count': (_ll, []),
    'isb_note_graph_replay': (_i, [_ll]),
    'isb_profile_enable': (_i, [_i]),
    'isb_profile_stage_count': (_i, []),
    'isb_profile_stage_name': (C.c_char_p, [_i]),
    'isb_profile_collect': (_i, [C.POINTER(_d), C.POINTER(_ll)]),
    'isb_slic_prepare': (_i, [_vp, _i, _i, _i, _i, C.POINTER(_d), _i, _d, _i, _vp, _vp, _vp]),
    'isb_image_minmax': (_i, [_vp, _i, _ll, _vp, _vp]),
    'isb_slic_band_begin': (_i, [_bp, _vp]),
    'isb_slic_band_assign': (_i, [_bp, _vp]),
    'isb_slic_band_update': (_i, [_bp, _vp, _vp]),
    'isb_slic_band_import': (_i, [_bp, _vp, _vp, _vp]),
    'isb_slic_band_finalize': (_i, [_bp, _vp, _vp]),
    'isb_segment_stats_accumulate': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    'isb_segment_stats_deviation': (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'isb_segment_stats_finish': (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'isb_slic_kmeans_workspace_bytes': (_sz, [_i, _i, _i, _i, _i]),
    'isb_slic_kmeans': (_i, [_vp, _i, _i, _vp, _i, _i, _i, _d, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_slic_set_tile_cap': (_i, [_i]),
    'isb_slic_full_scan_tiles': (_ll, []),
    'isb_slic3d_prepare': (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _d, _vp, _vp, _vp]),
    'isb_slic3d_prepare_slab': (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _d, _vp, _vp, _vp]),
    'isb_slic3d_slab_begin': (_i, [_sp, _vp]),
    'isb_slic3d_slab_assign': (_i, [_sp, _vp]),
    'isb_slic3d_slab_update': (_i, [_sp, _vp, _vp]),
    'isb_slic3d_slab_import': (_i, [_sp, _vp, _vp]),
    'isb_slic3d_kmeans_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'isb_slic3d_kmeans': (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _i, _d, C.POINTER(_d), _i, _vp, _vp, _sz, _vp]),
    'isb_connectivity3d_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'isb_enforce_connectivity3d': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_connectivity_workspace_bytes': (_sz, [_i, _i]),
    'isb_enforce_connectivity': (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_segment_stats_workspace_bytes': (_sz, [_i]),
    'isb_segment_stats_2d': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_adjacency_workspace_bytes': (_sz, [_i, _i]),
    'isb_adjacency_edges': (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_adjacency_edges_3d': (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_centroids_3d': (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_gc_energies_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_standard_scaler': (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'isb_gc_energies': (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _d, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_gc_vector_edge_weights': (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_image_unit_scale': (_i, [_vp, _i, _ll, _vp, _vp, _vp]),
    'isb_alpha_expansion_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_alpha_expansion': (_i, [_i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_mixture_fit_workspace_bytes': (_sz, [_i, _i, _i, _i, _i]),
    'isb_mixture_fit_params_len': (_i, [_i, _i, _i]),
    'isb_mixture_fit_predict': (_i, [_i, _vp, _i, _i, _i, _vp, _i, _i, _i, _d, _d, _i, C.c_ulonglong, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_pca_workspace_bytes': (_sz, [_i, _i]),
    'isb_pca_params_len': (_i, [_i]),
    'isb_pca_fit': (_i, [_vp, _i, _i, _i, _vp, _i, _d, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_class_transform_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_class_transform': (_i, [_vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_mixture_predict_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_mixture_predict_proba': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_forest_predict_workspace_bytes': (_sz, [_i, _i]),
    'isb_forest_predict_proba': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_knn_predict_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_knn_predict_proba': (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_linear_predict_workspace_bytes': (_sz, [_i, _i]),
    'isb_linear_predict_proba': (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_lm_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'isb_lm_acc_doubles': (_sz, [_i, _i]),
    'isb_lm_texture_accumulate': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _i, C.POINTER(_d), _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_lm_texture_finish': (_i, [_i, _i, _i, _vp, _vp, _vp, _i, _i, _vp]),
    'isb_lm_texture': (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _i, C.POINTER(_d), _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _sz, _vp]),
    'isb_wgmma_selftest': (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    'isb_fill_i32': (_i, [_vp, _ll, _i, _vp]),
    'isb_combine': (_i, [_vp, _vp, _ll, _i, _vp]),
    'isb_gray_stats_workspace_bytes': (_sz, [_i]),
    'isb_gray_stats': (_i, [_vp, _i, _vp, _ll, _i, _i, _vp, _i, _i, _vp, _sz, _vp]),
    'isb_gray_stats_accumulate': (_i, [_vp, _i, _vp, _ll, _i, _vp, _vp, _vp]),
    'isb_gray_stats_deviation': (_i, [_vp, _i, _vp, _ll, _i, _vp, _vp, _vp, _vp, _vp]),
    'isb_gray_stats_finish': (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    'isb_label_hist_2d': (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    'isb_ray_features_2d': (_i, [_vp, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp]),
    'isb_filter_response_2d': (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp]),
    'isb_gaussian_filter_2d': (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp]),
    'isb_disc_label_hist': (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    'isb_label_runs_workspace_bytes': (_sz, [_i, _i]),
    'isb_ring_label_hist': (_i, [_vp, _i, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_dbscan_workspace_bytes': (_sz, [_i]),
    'isb_dbscan': (_i, [_vp, _i, _d, _i, _vp, _vp, C.POINTER(_i), _vp, _sz, _vp]),
    'isb_region_label_hist': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'isb_train_labels_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_superpixel_train_labels': (_i, [_vp, _i, _i, _i, _vp, _vp, _d, _vp, _vp, _sz, _vp]),
    'isb_unique_rows_workspace_bytes': (_sz, [_i, _i]),
    'isb_unique_rows_rounded': (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_gather': (_i, [_vp, _ll, _vp, _vp, _i, _vp, _vp, _vp]),
    'isb_segment_median_workspace_bytes': (_sz, [_ll, _i]),
    'isb_segment_median': (_i, [_vp, _i, _vp, _ll, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_color_convert': (_i, [_vp, _i, _ll, _i, _vp, _vp]),
    'isb_gradient_sum_2d': (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    'isb_segment_median_2d': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _sz, _vp]),
    'isb_lm_background': (_i, [_vp, _i, _i, _i, _vp, _i, C.POINTER(_d), _vp, _vp, _vp, _vp]),
    'isb_lm_battery_workspace_bytes': (_sz, []),
    'isb_lm_battery_response': (_i, [_vp, _i, _i, _vp, _i, _i, _i, _d, _vp, _vp, _vp, _sz, _vp]),
    'isb_lm_battery_partial': (_i, [_vp, _i, _i, _vp, _i, _i, _i, _d, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    'isb_lm_battery_scale': (_i, [_vp, _i, _i, _i, _i, _d, _vp, _vp, _vp]),
    'isb_ellipse_ransac': (_i, [_i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _d, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'isb_ellipse_overlap': (_i, [_vp, _i, _i, _i, C.POINTER(C.c_int32), C.POINTER(_d), _vp, _vp, _vp]),
    'isb_binary_morph_footprint': (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp]),
    'isb_label_boundary_map': (_i, [_vp, _i, _i, _vp, _vp]),
    'isb_label_contour_map': (_i, [_vp, _i, _i, C.c_int32, _i, _vp, _vp]),
    'isb_edt_workspace_bytes': (_sz, [_i, _i]),
    'isb_edt_2d': (_i, [_vp, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_mask_compact_workspace_bytes': (_sz, [_i, _i]),
    'isb_mask_compact_count': (_i, [_vp, _i, _i, _vp, _sz, _vp, _vp]),
    'isb_mask_compact_write': (_i, [_vp, _i, _i, _vp, _vp, _sz, _vp, _vp, _vp]),
    'isb_relabel_gather': (_i, [_vp, _ll, _vp, _i, _vp, _vp]),
    'isb_edt_index_workspace_bytes': (_sz, [_i, _i]),
    'isb_edt_2d_indices': (_i, [_vp, _i, _i, _vp, _vp, _sz, _vp]),
    'isb_color_hist': (_i, [_vp, _ll, _i, _i, _vp, _vp]),
    'isb_color_hist_workspace_bytes': (_sz, []),
    'isb_color_hist_compact_count': (_i, [_vp, _vp, _sz, _vp, _vp]),
    'isb_color_hist_compact_write': (_i, [_vp, _vp, _sz, _vp, _vp, _vp]),
    'isb_palette_map': (_i, [_vp, _i, _ll, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'isb_palette_gather': (_i, [_vp, _ll, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    'isb_gather_at_index': (_i, [_vp, _i, _vp, _ll, _vp, _vp]),
    'isb_contingency_workspace_bytes': (_sz, [_i, _i]),
    'isb_contingency_count': (_i, [_vp, _i, _vp, _i, _ll, _vp, _i, _vp, _sz, C.POINTER(_ll), _vp]),
    'isb_contingency_write': (_i, [_vp, _i, _vp, _i, _ll, _vp, _i, C.POINTER(_ll), _vp, _sz, _vp, _vp, _vp, _vp]),
    'isb_kmeans_workspace_bytes': (_sz, [_i, _i, _i]),
    'isb_kmeans_lloyd': (_i, [_vp, _i, _i, _i, _i, _i, _d, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'isb_kmeans_nearest': (_i, [_vp, _i, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    'isb_forest_fit_workspace_bytes': (_sz, [_i, _i, _i, _i, _i]),
    'isb_forest_fit': (_i, [_vp, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _d, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                            C.POINTER(_i), _vp, _sz, _vp]),
    'isb_forest_fit_groups_workspace_bytes': (_sz, [_i, _i, _i, _i, _i, _i]),
    'isb_forest_fit_groups': (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _d, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _vp, _vp, C.POINTER(_i), _vp, _sz, _vp]),
    'isb_extra_trees_fit_workspace_bytes': (_sz, [_i, _i, _i, _i, _i]),
    'isb_extra_trees_fit': (_i, [_vp, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _d, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp, _sz, _vp]),
}


class NativeLibraryError(RuntimeError):
    pass


def lib():
    """load the CUDA extension; raises (never falls back) when it has not been built"""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise NativeLibraryError(
                'pyimsegm_b200: %s is missing -- build it with `python -m pyimsegm_b200.build` '
                '(there is no CPU fallback)' % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError here = header / library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status):
    if status != ISB_OK:
        msg = lib().isb_last_error().decode(errors='replace')
        if status == ISB_ERR_ARG:
            raise ValueError('imsegm_b200: ' + msg)
        if status == ISB_ERR_UNSUPPORTED:
            raise NotImplementedError('imsegm_b200: ' + msg)
        raise RuntimeError('imsegm_b200 (status %d): %s' % (status, msg))


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise NativeLibraryError('pyimsegm_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback')
    return torch


def dtype_code(dtype):
    """DTYPE_CODES entry of a numpy or torch dtype"""
    return DTYPE_CODES[str(dtype).replace('torch.', '')]


def ptr(t):
    """device pointer of a torch tensor (or None)"""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
