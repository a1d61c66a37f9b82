"""ctypes mirror of include/mulls_b200/abi.h (the C-ABI of the H100 registration hot path).

The PODs here are byte-for-byte the structs of abi.h; `load_library()` opens the in-tree
`mulls_b200/csrc/libmulls_b200.so` and fails loudly when it is missing — there is no CPU fallback
in the product path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

NUM_CLASSES = 6
GROUND, PILLAR, FACADE, BEAM, ROOF, VERTEX = range(6)
CLASS_NAMES = ("ground", "pillar", "facade", "beam", "roof", "vertex")
MAX_TRACE_ITERS = 64

E_CUDA, E_ARG, E_CAPACITY, E_UNSUPPORTED, E_COMM = -100, -101, -102, -103, -104


class CloudView(C.Structure):
    _fields_ = [("aos48", C.POINTER(C.c_float)), ("n", C.c_size_t)]


class IcpParams(C.Structure):
    _fields_ = [
        ("max_iter_num", C.c_int32),
        ("dis_thre_unit", C.c_float),
        ("converge_translation", C.c_float),
        ("converge_rotation_d", C.c_float),
        ("dis_thre_min", C.c_float),
        ("dis_thre_update_rate", C.c_float),
        ("used_feature_type", C.c_char * 8),
        ("weight_strategy", C.c_char * 8),
        ("z_xy_balanced_ratio", C.c_float),
        ("pt2pt_residual_window", C.c_float),
        ("pt2pl_residual_window", C.c_float),
        ("pt2li_residual_window", C.c_float),
        ("apply_intersection_filter", C.c_int32),
        ("apply_motion_undistortion_while_registration", C.c_int32),
        ("normal_shooting_on", C.c_int32),
        ("normal_bearing", C.c_float),
        ("use_more_points", C.c_int32),
        ("keep_less_source_points", C.c_int32),
        ("sigma_thre", C.c_float),
        ("min_neccessary_corr_ratio", C.c_float),
        ("max_bearable_rotation_d", C.c_float),
        ("target_bound", C.c_double * 6),
        ("random_seed", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


class IcpResult(C.Structure):
    _fields_ = [
        ("T", C.c_double * 16),
        ("info", C.c_double * 36),
        ("sigma", C.c_float),
        ("confidence", C.c_float),
        ("code", C.c_int32),
        ("iters", C.c_int32),
        ("n_corr", C.c_uint32 * 6),
        ("n_src", C.c_uint32 * 6),
    ]


class IcpTrace(C.Structure):
    _fields_ = [
        ("n_iter", C.c_int32),
        ("_pad", C.c_int32),
        ("atpa", (C.c_double * 36) * MAX_TRACE_ITERS),
        ("atpb", (C.c_double * 6) * MAX_TRACE_ITERS),
        ("x", (C.c_double * 6) * MAX_TRACE_ITERS),
        ("n_corr", (C.c_uint32 * 6) * MAX_TRACE_ITERS),
        ("n_src", (C.c_uint32 * 6) * MAX_TRACE_ITERS),
    ]


class TeaserInfo(C.Structure):
    """mulls_teaser_info"""
    _fields_ = [("n_edges", C.c_int64), ("max_core", C.c_int), ("clique_size", C.c_int), ("rotation_inliers", C.c_int),
                ("gnc_iterations", C.c_int), ("search_launches", C.c_int), ("pad", C.c_int)]


class RunStats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64),
        ("algorithmic_bytes", C.c_uint64),
        ("iterations", C.c_uint64),
        ("search_launches", C.c_uint64),
        ("ms_ingest", C.c_float),
        ("ms_iterate", C.c_float),
        ("ms_search", C.c_float),
        ("ms_total", C.c_float),
        ("ms_search_iter", C.c_float * MAX_TRACE_ITERS),
        ("ms_host_pack", C.c_float),
        ("ms_h2d", C.c_float),
        ("ms_host_call", C.c_float),
        ("ms_host_upload", C.c_float),
    ]


class PcaOut(C.Structure):
    _fields_ = [
        ("eigenvalues", C.POINTER(C.c_float)),
        ("principal", C.POINTER(C.c_float)),
        ("normal", C.POINTER(C.c_float)),
        ("pt_num", C.POINTER(C.c_int32)),
    ]


class NdtResult(C.Structure):
    """mulls_ndt_result: Trans1_2, the code omp_ndt returns, the walk's iteration count and convergence, the fitness score
    and the point counts after the intersection filter."""
    _fields_ = [
        ("trans", C.c_double * 16),
        ("code", C.c_int),
        ("iterations", C.c_int),
        ("converged", C.c_int),
        ("n_target", C.c_int),
        ("n_source", C.c_int),
        ("fitness", C.c_double),
    ]


class NdtIter(C.Structure):
    """mulls_ndt_iter: one Newton iteration of the NDT walk (pose vector after the step, step length, score, reversal)."""
    _fields_ = [("p", C.c_double * 6), ("step", C.c_double), ("score", C.c_double), ("reversed", C.c_int)]


class GicpResult(C.Structure):
    """mulls_gicp_result: Trans1_2, the code omp_gicp returns, the walk's step count and convergence, the point counts
    after the prologue, the fitness score and the walk's start point x0 (so3, translation)."""
    _fields_ = [
        ("trans", C.c_double * 16),
        ("code", C.c_int),
        ("iterations", C.c_int),
        ("converged", C.c_int),
        ("n_target", C.c_int),
        ("n_source", C.c_int),
        ("fitness", C.c_double),
        ("x0", C.c_float * 6),
    ]


class GicpIter(C.Structure):
    """mulls_gicp_iter: one Gauss-Newton step of the VGICP walk (point after the step, the step, correspondences,
    whether the step was the random fallback)."""
    _fields_ = [("x", C.c_float * 6), ("delta", C.c_float * 6), ("n_corr", C.c_int), ("random_step", C.c_int)]


GicpPclResult = NdtResult  # mulls_gicp_pcl_result is a typedef of mulls_ndt_result


class GicpPclIter(C.Structure):
    """mulls_gicp_pcl_iter: one outer iteration of the point-wise GICP (the solver's state after it, the change of the
    transformation, correspondences, BFGS steps, the BFGS status, functor calls)."""
    _fields_ = [
        ("x", C.c_double * 6),
        ("delta", C.c_double),
        ("n_corr", C.c_int),
        ("inner_iterations", C.c_int),
        ("status", C.c_int),
        ("evaluations", C.c_int),
    ]


class SorStats(C.Structure):
    """mulls_sor_stats: what pcl::StatisticalOutlierRemoval computed (mean, stddev, threshold) and the point counts."""
    _fields_ = [
        ("mean", C.c_double),
        ("stddev", C.c_double),
        ("threshold", C.c_double),
        ("n_valid", C.c_uint64),
        ("n_kept", C.c_uint64),
    ]


class MapParams(C.Structure):
    """mulls_map_params: the arguments of MapManager::update_local_map (include/pgo/map_manager.h:22-32)."""
    _fields_ = [
        ("local_map_radius", C.c_float),
        ("max_num_pts", C.c_int32),
        ("kept_vertex_num", C.c_int32),
        ("last_frame_reliable_radius", C.c_float),
        ("map_based_dynamic_removal_on", C.c_int32),
        ("used_feature_type", C.c_char * 8),
        ("dynamic_removal_center_radius", C.c_float),
        ("dynamic_dist_thre_min", C.c_float),
        ("dynamic_dist_thre_max", C.c_float),
        ("near_dist_thre", C.c_float),
        ("recalculate_feature_on", C.c_int32),
        ("random_seed", C.c_uint32),
    ]


class MapInfo(C.Structure):
    _fields_ = [
        ("pose_lo", C.c_double * 16),
        ("local_bound", C.c_double * 6),
        ("bound", C.c_double * 6),
        ("n", C.c_uint32 * NUM_CLASSES),
        ("n_appended", C.c_uint32 * NUM_CLASSES),
        ("feature_point_num", C.c_int32),
        ("ms_update", C.c_float),
    ]


OUT_NAMES = ("pillar", "beam", "facade", "roof", "pillar_down", "beam_down", "facade_down", "roof_down", "vertex",
             "unground")
OUT_COUNT = len(OUT_NAMES)


class ClassifyParams(C.Structure):
    """mulls_classify_params: the arguments of CFilter::classify_nground_pts (cfilter.hpp:2070-2081)."""
    _fields_ = [
        ("neighbor_searching_radius", C.c_float),
        ("neighbor_k", C.c_int32),
        ("neigh_k_min", C.c_int32),
        ("pca_down_rate", C.c_int32),
        ("edge_thre", C.c_float),
        ("planar_thre", C.c_float),
        ("edge_thre_down", C.c_float),
        ("planar_thre_down", C.c_float),
        ("extract_vertex_points_method", C.c_int32),
        ("curvature_thre", C.c_float),
        ("vertex_curvature_non_max_radius", C.c_float),
        ("linear_vertical_sin_high_thre", C.c_float),
        ("linear_vertical_sin_low_thre", C.c_float),
        ("planar_vertical_sin_high_thre", C.c_float),
        ("planar_vertical_sin_low_thre", C.c_float),
        ("fixed_num_downsampling", C.c_int32),
        ("pillar_down_fixed_num", C.c_int32),
        ("facade_down_fixed_num", C.c_int32),
        ("beam_down_fixed_num", C.c_int32),
        ("roof_down_fixed_num", C.c_int32),
        ("unground_down_fixed_num", C.c_int32),
        ("beam_height_max", C.c_float),
        ("roof_height_min", C.c_float),
        ("feature_pts_ratio_guess", C.c_float),
        ("sharpen_with_nms", C.c_int32),
        ("use_distance_adaptive_pca", C.c_int32),
        ("random_seed", C.c_uint32),
        ("pca_unit_distance", C.c_float),
    ]


class ClassifyOut(C.Structure):
    _fields_ = [
        ("rows", C.POINTER(C.c_float) * OUT_COUNT),
        ("cap", C.c_size_t),
        ("n", C.c_size_t * OUT_COUNT),
    ]


class GroundParams(C.Structure):
    """mulls_ground_params: the arguments of CFilter::fast_ground_filter (cfilter.hpp:1658-1672)."""
    _fields_ = [
        ("min_grid_pt_num", C.c_int32),
        ("grid_resolution", C.c_float),
        ("max_height_difference", C.c_float),
        ("neighbor_height_diff", C.c_float),
        ("max_ground_height", C.c_float),
        ("ground_random_down_rate", C.c_int32),
        ("ground_random_down_down_rate", C.c_int32),
        ("nonground_random_down_rate", C.c_int32),
        ("reliable_neighbor_grid_num_thre", C.c_int32),
        ("estimate_ground_normal_method", C.c_int32),
        ("normal_estimation_radius", C.c_float),
        ("distance_weight_downsampling_method", C.c_int32),
        ("standard_distance", C.c_float),
        ("fixed_num_downsampling", C.c_int32),
        ("down_ground_fixed_num", C.c_int32),
        ("intensity_thre", C.c_float),
        ("apply_grid_wise_outlier_filter", C.c_int32),
        ("outlier_std_scale", C.c_float),
        ("random_seed", C.c_uint32),
    ]


class GroundOut(C.Structure):
    _fields_ = [
        ("ground", C.POINTER(C.c_float)),
        ("ground_down", C.POINTER(C.c_float)),
        ("unground", C.POINTER(C.c_float)),
        ("cap", C.c_size_t),
        ("n_ground", C.c_size_t),
        ("n_ground_down", C.c_size_t),
        ("n_unground", C.c_size_t),
    ]


class ExtractParams(C.Structure):
    """mulls_extract_params: CFilter::extract_semantic_pts (cfilter.hpp:2295-2413) = voxel filter + ground filter + classification."""
    _fields_ = [("vf_downsample_resolution", C.c_float), ("ground", GroundParams), ("classify", ClassifyParams)]


class ExtractOut(C.Structure):
    _fields_ = [
        ("pc_down", C.POINTER(C.c_float)),
        ("pc_ground", C.POINTER(C.c_float)),
        ("pc_ground_down", C.POINTER(C.c_float)),
        ("cap", C.c_size_t),
        ("n_down", C.c_size_t),
        ("n_ground", C.c_size_t),
        ("n_ground_down", C.c_size_t),
        ("cls", ClassifyOut),
    ]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p)

# every symbol include/mulls_b200/abi.h declares
EXPORTED_SYMBOLS = (
    "mulls_create",
    "mulls_destroy",
    "mulls_last_error",
    "mulls_icp_default_params",
    "mulls_icp_run",
    "mulls_icp_run_batch",
    "mulls_batch_upload",
    "mulls_batch_run_resident",
    "mulls_get_stats",
    "mulls_icp_run_sharded",
    "mulls_pca_features",
    "mulls_pca_features_adaptive",
    "mulls_map_default_params",
    "mulls_map_create",
    "mulls_map_destroy",
    "mulls_map_set",
    "mulls_map_update",
    "mulls_map_get_info",
    "mulls_map_download",
    "mulls_icp_run_to_map",
    "mulls_classify_default_params",
    "mulls_classify_nground",
    "mulls_set_tunable",
    "mulls_nn_query",
    "mulls_nccl_unique_id",
    "mulls_nccl_init",
    "mulls_icp_run_sharded_nccl",
    "mulls_pack_rows",
    "mulls_ground_default_params",
    "mulls_fast_ground_filter",
    "mulls_voxel_downsample",
    "mulls_extract_semantic_pts",
    "mulls_sor_filter",
    "mulls_vertical_intrinsic_calibration",
    "mulls_timestamp_ratio",
    "mulls_motion_compensation",
    "mulls_ncc_correspondences",
    "mulls_coarse_reg_ransac",
    "mulls_coarse_reg_teaser",
    "mulls_non_max_suppress",
    "mulls_omp_ndt",
    "mulls_omp_ndt_kdtree",
    "mulls_omp_ndt_batch",
    "mulls_omp_gicp",
    "mulls_omp_gicp_pcl",
    "mulls_scan_probe",
    "mulls_scan_read",
    "mulls_pose_write",
    "mulls_host_alloc",
    "mulls_host_free",
)

_LIB = None
LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libmulls_b200.so")


def load_library() -> C.CDLL:
    """Open the CUDA library. Raises (never falls back) if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C mulls_b200/csrc`). mulls_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.mulls_create.restype = vp
    lib.mulls_create.argtypes = [C.c_int, C.c_size_t, C.c_size_t, C.c_size_t]
    lib.mulls_destroy.restype = None
    lib.mulls_destroy.argtypes = [vp]
    lib.mulls_last_error.restype = C.c_char_p
    lib.mulls_last_error.argtypes = [vp]
    lib.mulls_icp_default_params.restype = None
    lib.mulls_icp_default_params.argtypes = [C.POINTER(IcpParams)]
    lib.mulls_icp_run.restype = C.c_int
    lib.mulls_icp_run.argtypes = [vp, C.POINTER(CloudView), C.POINTER(CloudView), C.POINTER(IcpParams),
                                  C.POINTER(C.c_double), C.POINTER(IcpResult), C.POINTER(IcpTrace)]
    lib.mulls_icp_run_batch.restype = C.c_int
    lib.mulls_icp_run_batch.argtypes = [vp, C.c_size_t, C.POINTER(CloudView), C.POINTER(CloudView),
                                        C.POINTER(IcpParams), C.POINTER(C.c_double), C.POINTER(IcpResult),
                                        C.POINTER(IcpTrace)]
    lib.mulls_batch_upload.restype = C.c_int
    lib.mulls_batch_upload.argtypes = [vp, C.c_size_t, C.POINTER(CloudView), C.POINTER(CloudView),
                                       C.POINTER(IcpParams), C.POINTER(C.c_double)]
    lib.mulls_batch_run_resident.restype = C.c_int
    lib.mulls_batch_run_resident.argtypes = [vp, C.POINTER(IcpResult), C.POINTER(IcpTrace)]
    lib.mulls_get_stats.restype = C.c_int
    lib.mulls_get_stats.argtypes = [vp, C.POINTER(RunStats)]
    lib.mulls_icp_run_sharded.restype = C.c_int
    lib.mulls_icp_run_sharded.argtypes = [vp, C.POINTER(CloudView), C.POINTER(CloudView),
                                          C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(IcpParams),
                                          C.POINTER(C.c_double), ALLREDUCE_FN, vp, C.POINTER(IcpResult),
                                          C.POINTER(IcpTrace)]
    lib.mulls_icp_run_sharded_nccl.restype = C.c_int
    lib.mulls_icp_run_sharded_nccl.argtypes = [vp, vp, C.POINTER(CloudView), C.POINTER(CloudView), C.POINTER(C.c_uint32),
                                               C.POINTER(C.c_uint32), C.POINTER(IcpParams), C.POINTER(C.c_double),
                                               C.POINTER(IcpResult), C.POINTER(IcpTrace)]
    lib.mulls_pca_features.restype = C.c_int
    lib.mulls_pca_features.argtypes = [vp, CloudView, C.c_float, C.c_int, C.c_int, C.POINTER(PcaOut)]
    lib.mulls_pca_features_adaptive.restype = C.c_int
    lib.mulls_pca_features_adaptive.argtypes = [vp, CloudView, C.c_float, C.c_int, C.c_int, C.c_float, C.POINTER(PcaOut)]
    lib.mulls_ground_default_params.restype = None
    lib.mulls_ground_default_params.argtypes = [C.POINTER(GroundParams)]
    lib.mulls_fast_ground_filter.restype = C.c_int
    lib.mulls_fast_ground_filter.argtypes = [vp, CloudView, C.POINTER(GroundParams), C.POINTER(GroundOut)]
    lib.mulls_voxel_downsample.restype = C.c_int
    lib.mulls_voxel_downsample.argtypes = [vp, CloudView, C.c_float, C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_size_t)]
    lib.mulls_extract_semantic_pts.restype = C.c_int
    lib.mulls_extract_semantic_pts.argtypes = [vp, CloudView, C.POINTER(ExtractParams), C.POINTER(ExtractOut)]
    lib.mulls_sor_filter.restype = C.c_int
    lib.mulls_sor_filter.argtypes = [vp, CloudView, C.c_int, C.c_double, C.POINTER(C.c_uint8), C.POINTER(C.c_float),
                                     C.POINTER(SorStats)]
    lib.mulls_vertical_intrinsic_calibration.restype = C.c_int
    lib.mulls_vertical_intrinsic_calibration.argtypes = [vp, CloudView, C.c_double, C.c_int, C.POINTER(C.c_float),
                                                         C.POINTER(C.c_int)]
    lib.mulls_timestamp_ratio.restype = C.c_int
    lib.mulls_timestamp_ratio.argtypes = [vp, CloudView, C.c_int, C.c_double, C.c_float, C.POINTER(C.c_float)]
    lib.mulls_motion_compensation.restype = C.c_int
    lib.mulls_motion_compensation.argtypes = [vp, C.POINTER(CloudView), C.c_int, C.POINTER(C.c_double), C.c_float,
                                              C.POINTER(C.POINTER(C.c_float))]
    lib.mulls_ncc_correspondences.restype = C.c_int
    lib.mulls_ncc_correspondences.argtypes = [vp, CloudView, CloudView, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
    lib.mulls_coarse_reg_teaser.restype = C.c_int
    lib.mulls_coarse_reg_teaser.argtypes = [vp, CloudView, CloudView, C.c_float, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int),
                                            C.POINTER(TeaserInfo)]
    lib.mulls_coarse_reg_ransac.restype = C.c_int
    lib.mulls_coarse_reg_ransac.argtypes = [vp, CloudView, CloudView, C.c_float, C.c_int, C.c_int, C.POINTER(C.c_double),
                                            C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.mulls_non_max_suppress.restype = C.c_int
    lib.mulls_non_max_suppress.argtypes = [vp, CloudView, C.c_float, C.POINTER(C.c_int32), C.POINTER(C.c_size_t),
                                           C.POINTER(C.c_int)]
    lib.mulls_omp_ndt.restype = C.c_int
    lib.mulls_omp_ndt.argtypes = [vp, CloudView, CloudView, C.c_float, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_float,
                                  C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(NdtResult), C.POINTER(NdtIter), C.c_int]
    lib.mulls_omp_ndt_kdtree.restype = C.c_int
    lib.mulls_omp_ndt_kdtree.argtypes = [vp, CloudView, CloudView, C.c_float, C.POINTER(C.c_double), C.c_int, C.c_float,
                                         C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(NdtResult), C.POINTER(NdtIter),
                                         C.c_int]
    lib.mulls_omp_ndt_batch.restype = C.c_int
    lib.mulls_omp_ndt_batch.argtypes = [vp, C.c_size_t, C.POINTER(CloudView), C.POINTER(CloudView), C.c_float, C.c_int,
                                        C.POINTER(C.c_double), C.c_int, C.c_float, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                        C.POINTER(NdtResult), C.POINTER(NdtIter), C.c_int]
    lib.mulls_omp_gicp.restype = C.c_int
    lib.mulls_omp_gicp.argtypes = [vp, CloudView, CloudView, C.c_int, C.c_float, C.POINTER(C.c_double), C.c_int, C.c_float,
                                   C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(GicpResult), C.POINTER(GicpIter),
                                   C.c_int]
    lib.mulls_omp_gicp_pcl.restype = C.c_int
    lib.mulls_omp_gicp_pcl.argtypes = [vp, CloudView, CloudView, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_float,
                                       C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(GicpPclResult),
                                       C.POINTER(GicpPclIter), C.c_int]
    lib.mulls_pack_rows.restype = C.c_int
    lib.mulls_pack_rows.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_int, C.POINTER(C.c_float)]
    lib.mulls_scan_probe.restype = C.c_int
    lib.mulls_scan_probe.argtypes = [C.c_char_p, C.POINTER(C.c_size_t)]
    lib.mulls_scan_read.restype = C.c_int
    lib.mulls_scan_read.argtypes = [C.c_char_p, C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_double), C.c_int]
    lib.mulls_pose_write.restype = C.c_int
    lib.mulls_pose_write.argtypes = [C.c_char_p, C.POINTER(C.c_double), C.c_int]
    lib.mulls_host_alloc.restype = C.c_void_p
    lib.mulls_host_alloc.argtypes = [C.c_size_t]
    lib.mulls_host_free.restype = None
    lib.mulls_host_free.argtypes = [C.c_void_p]
    lib.mulls_nccl_unique_id.restype = C.c_int
    lib.mulls_nccl_unique_id.argtypes = [C.c_char_p]
    lib.mulls_nccl_init.restype = C.c_int
    lib.mulls_nccl_init.argtypes = [vp, C.c_int, C.c_int, C.c_char_p]
    lib.mulls_nn_query.restype = C.c_int
    lib.mulls_nn_query.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_float)]
    lib.mulls_set_tunable.restype = C.c_int
    lib.mulls_set_tunable.argtypes = [vp, C.c_char_p, C.c_int]
    lib.mulls_map_default_params.restype = None
    lib.mulls_map_default_params.argtypes = [C.POINTER(MapParams)]
    lib.mulls_map_create.restype = vp
    lib.mulls_map_create.argtypes = [vp, C.c_size_t]
    lib.mulls_map_destroy.restype = None
    lib.mulls_map_destroy.argtypes = [vp]
    lib.mulls_map_set.restype = C.c_int
    lib.mulls_map_set.argtypes = [vp, C.POINTER(CloudView), C.POINTER(C.c_double)]
    lib.mulls_map_update.restype = C.c_int
    lib.mulls_map_update.argtypes = [vp, C.POINTER(CloudView), C.POINTER(C.c_double), C.POINTER(MapParams),
                                     C.POINTER(MapInfo)]
    lib.mulls_map_get_info.restype = C.c_int
    lib.mulls_map_get_info.argtypes = [vp, C.POINTER(MapInfo)]
    lib.mulls_map_download.restype = C.c_int
    lib.mulls_map_download.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_size_t)]
    lib.mulls_icp_run_to_map.restype = C.c_int
    lib.mulls_icp_run_to_map.argtypes = [vp, vp, C.POINTER(CloudView), C.POINTER(IcpParams), C.POINTER(C.c_double),
                                         C.POINTER(IcpResult), C.POINTER(IcpTrace)]
    lib.mulls_classify_default_params.restype = None
    lib.mulls_classify_default_params.argtypes = [C.POINTER(ClassifyParams)]
    lib.mulls_classify_nground.restype = C.c_int
    lib.mulls_classify_nground.argtypes = [vp, CloudView, C.POINTER(ClassifyParams), C.POINTER(ClassifyOut)]
    _LIB = lib
    return lib


# ---------------------------------------------------------------------------------------------
# helpers shared by the host-side mirror, the tests and the bench
# ---------------------------------------------------------------------------------------------
def as_aos48(points: np.ndarray) -> np.ndarray:
    """(n,7) [x y z nx ny nz intensity] or (n,12) float32 -> C-contiguous (n,12) pcl::PointXYZINormal rows."""
    points = np.asarray(points, dtype=np.float32)
    if points.ndim != 2:
        raise ValueError("point array must be 2-D")
    if points.shape[1] == 12:
        return np.ascontiguousarray(points)
    if points.shape[1] != 7:
        raise ValueError("expected (n,7) or (n,12) float32")
    out = np.zeros((points.shape[0], 12), dtype=np.float32)
    out[:, 0:3] = points[:, 0:3]
    out[:, 3] = 1.0
    out[:, 4:7] = points[:, 3:6]
    out[:, 8] = points[:, 6]
    return out


def cloud_view(arr: np.ndarray) -> CloudView:
    """View of an (n,12) float32 C-contiguous array (keep `arr` alive while the view is in use)."""
    assert arr.dtype == np.float32 and arr.flags["C_CONTIGUOUS"] and (arr.size == 0 or arr.shape[1] == 12)
    return CloudView(arr.ctypes.data_as(C.POINTER(C.c_float)), arr.shape[0])


def default_params() -> IcpParams:
    """The defaults of mm_lls_icp (cregistration.hpp:1115-1123) — pure Python, no library needed."""
    p = IcpParams()
    p.max_iter_num = 20
    p.dis_thre_unit = 1.5
    p.converge_translation = 0.002
    p.converge_rotation_d = 0.01
    p.dis_thre_min = 0.4
    p.dis_thre_update_rate = 1.1
    p.used_feature_type = b"111110"
    p.weight_strategy = b"1101"
    p.z_xy_balanced_ratio = 1.0
    p.pt2pt_residual_window = 0.1
    p.pt2pl_residual_window = 0.1
    p.pt2li_residual_window = 0.1
    p.apply_intersection_filter = 1
    p.apply_motion_undistortion_while_registration = 0
    p.normal_shooting_on = 0
    p.normal_bearing = 45.0
    p.use_more_points = 0
    p.keep_less_source_points = 0
    p.sigma_thre = 0.5
    p.min_neccessary_corr_ratio = 0.03
    p.max_bearable_rotation_d = 45.0
    big = 1.7976931348623157e308
    p.target_bound[:] = [-big, -big, -big, big, big, big]
    p.random_seed = 0
    return p


def result_to_dict(r: IcpResult) -> dict:
    return {
        "T": np.array(r.T[:], dtype=np.float64).reshape(4, 4),
        "info": np.array(r.info[:], dtype=np.float64).reshape(6, 6),
        "sigma": float(r.sigma),
        "confidence": float(r.confidence),
        "code": int(r.code),
        "iters": int(r.iters),
        "n_corr": [int(v) for v in r.n_corr],
        "n_src": [int(v) for v in r.n_src],
    }


def trace_to_dict(t: IcpTrace) -> dict:
    n = int(t.n_iter)
    return {
        "n_iter": n,
        "atpa": np.ctypeslib.as_array(t.atpa)[:n].reshape(n, 6, 6).copy(),
        "atpb": np.ctypeslib.as_array(t.atpb)[:n].copy(),
        "x": np.ctypeslib.as_array(t.x)[:n].copy(),
        "n_corr": np.ctypeslib.as_array(t.n_corr)[:n].copy(),
        "n_src": np.ctypeslib.as_array(t.n_src)[:n].copy(),
    }


def default_map_params() -> MapParams:
    """The defaults of MapManager::update_local_map (include/pgo/map_manager.h:22-32) — pure Python."""
    p = MapParams()
    p.local_map_radius = 80.0
    p.max_num_pts = 20000
    p.kept_vertex_num = 800
    p.last_frame_reliable_radius = 60.0
    p.map_based_dynamic_removal_on = 0
    p.used_feature_type = b"111110"
    p.dynamic_removal_center_radius = 30.0
    p.dynamic_dist_thre_min = 0.3
    p.dynamic_dist_thre_max = 3.0
    p.near_dist_thre = 0.03
    p.recalculate_feature_on = 0
    p.random_seed = 0
    return p


def map_info_to_dict(info: MapInfo) -> dict:
    return {
        "pose_lo": np.array(info.pose_lo[:], dtype=np.float64).reshape(4, 4),
        "local_bound": np.array(info.local_bound[:], dtype=np.float64),
        "bound": np.array(info.bound[:], dtype=np.float64),
        "n": np.array(info.n[:], dtype=np.int64),
        "n_appended": np.array(info.n_appended[:], dtype=np.int64),
        "feature_point_num": int(info.feature_point_num),
        "ms_update": float(info.ms_update),
    }


def default_classify_params() -> ClassifyParams:
    """Defaults of classify_nground_pts (cfilter.hpp:2070-2081) / extract_semantic_pts (:2295-2318) — pure Python."""
    p = ClassifyParams()
    p.neighbor_searching_radius = 1.0
    p.neighbor_k = 50
    p.neigh_k_min = 8
    p.pca_down_rate = 1
    p.edge_thre = 0.65
    p.planar_thre = 0.65
    p.edge_thre_down = 0.75
    p.planar_thre_down = 0.75
    p.extract_vertex_points_method = 2
    p.curvature_thre = 0.12
    p.vertex_curvature_non_max_radius = 1.5
    p.linear_vertical_sin_high_thre = 0.94
    p.linear_vertical_sin_low_thre = 0.17
    p.planar_vertical_sin_high_thre = 0.98
    p.planar_vertical_sin_low_thre = 0.34
    p.fixed_num_downsampling = 0
    p.pillar_down_fixed_num = 200
    p.facade_down_fixed_num = 800
    p.beam_down_fixed_num = 200
    p.roof_down_fixed_num = 100
    p.unground_down_fixed_num = 20000
    p.beam_height_max = float(np.finfo(np.float32).max)
    p.roof_height_min = -float(np.finfo(np.float32).max)
    p.feature_pts_ratio_guess = 0.3
    p.sharpen_with_nms = 1
    p.use_distance_adaptive_pca = 0
    p.random_seed = 0
    p.pca_unit_distance = 0.0
    return p


def classify_call(fn, handle, cloud: np.ndarray, params: ClassifyParams) -> dict:
    """Shared marshalling of mulls_classify_nground / its CPU restatement: returns {name: (n,12) float32}."""
    cloud = as_aos48(cloud)
    n = cloud.shape[0]
    bufs = [np.zeros((max(n, 1), 12), np.float32) for _ in range(OUT_COUNT)]
    out = ClassifyOut()
    for k in range(OUT_COUNT):
        out.rows[k] = bufs[k].ctypes.data_as(C.POINTER(C.c_float))
    out.cap = max(n, 1)
    args = ([handle] if handle is not None else []) + [cloud_view(cloud), C.byref(params), C.byref(out)]
    rc = fn(*args)
    if rc != 0:
        return {"rc": rc}
    return {OUT_NAMES[k]: np.ascontiguousarray(bufs[k][: out.n[k]]) for k in range(OUT_COUNT)}


def default_ground_params() -> GroundParams:
    """Defaults of fast_ground_filter as extract_semantic_pts is called by test/mulls_slam.cpp (gflags :78-104) — pure Python."""
    p = GroundParams()
    p.min_grid_pt_num = 10
    p.grid_resolution = 3.0
    p.max_height_difference = 0.3
    p.neighbor_height_diff = 1.5
    p.max_ground_height = 5.0
    p.ground_random_down_rate = 15
    p.ground_random_down_down_rate = 2
    p.nonground_random_down_rate = 3
    p.reliable_neighbor_grid_num_thre = 0
    p.estimate_ground_normal_method = 3
    p.normal_estimation_radius = 2.0
    p.distance_weight_downsampling_method = 2
    p.standard_distance = 15.0
    p.fixed_num_downsampling = 0
    p.down_ground_fixed_num = 300
    p.intensity_thre = 3.4028234663852886e38
    p.apply_grid_wise_outlier_filter = 0
    p.outlier_std_scale = 3.0
    p.random_seed = 0
    return p


def ground_call(fn, handle, cloud: np.ndarray, params: GroundParams) -> dict:
    """Shared marshalling of mulls_fast_ground_filter / its CPU restatement: {"ground", "ground_down", "unground"}."""
    cloud = as_aos48(cloud)
    n = max(cloud.shape[0], 1)
    bufs = [np.zeros((n, 12), np.float32) for _ in range(3)]
    fp = C.POINTER(C.c_float)
    out = GroundOut(bufs[0].ctypes.data_as(fp), bufs[1].ctypes.data_as(fp), bufs[2].ctypes.data_as(fp), n, 0, 0, 0)
    args = ([handle] if handle is not None else []) + [cloud_view(cloud), C.byref(params), C.byref(out)]
    rc = fn(*args)
    if rc != 0:
        return {"rc": rc}
    return {"ground": np.ascontiguousarray(bufs[0][: out.n_ground]),
            "ground_down": np.ascontiguousarray(bufs[1][: out.n_ground_down]),
            "unground": np.ascontiguousarray(bufs[2][: out.n_unground])}
