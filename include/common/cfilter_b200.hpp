// Drop-in shims: lo::CFilter<PointT>::classify_nground_pts (include/common/cfilter.hpp:2058-2290), fast_ground_filter
// (:1658-2036), voxel_downsample (:83-165), sor_filter (:203-247), non_max_suppress (:1183-1240), scanner_filter
// (:914-929) and the raw-scan corrections
// vertical_intrinsic_calibration (:250-291), get_pts_timestamp_ratio_in_frame (:412-467), apply_motion_compensation and
// batch_apply_motion_compensation (:470-549) over the mulls_b200 C-ABI. A MULLS maintainer replaces the BODY of classify_nground_pts by
//
//     return lo::b200::classify_nground_pts<PointT>(cloud_in, cloud_pillar, ... );      // all arguments forwarded
//
// and CFilter::extract_semantic_pts (:2295-2413) keeps calling it unchanged. Same names, order, types and defaults as
// :2060-2081. The output clouds are expected empty at the call (as extract_semantic_pts passes them): results are
// appended. Differences (INTEGRATION.md §6): every random_downsample_pcl inside is a reproducible uniform sample;
// std::sort's unspecified order of equal NMS scores is fixed to "first pushed first".
#ifndef MULLS_B200_CFILTER_SHIM_HPP
#define MULLS_B200_CFILTER_SHIM_HPP

#include <cfloat>
#include <cstdint>
#include <vector>

#include "common/cregistration_b200.hpp" // thread_context, view_of
#include "mulls_b200/abi.h"

namespace lo {
namespace b200 {

template <typename PointT>
bool classify_nground_pts(typename pcl::PointCloud<PointT>::Ptr &cloud_in, typename pcl::PointCloud<PointT>::Ptr &cloud_pillar,
                          typename pcl::PointCloud<PointT>::Ptr &cloud_beam, typename pcl::PointCloud<PointT>::Ptr &cloud_facade,
                          typename pcl::PointCloud<PointT>::Ptr &cloud_roof, typename pcl::PointCloud<PointT>::Ptr &cloud_pillar_down,
                          typename pcl::PointCloud<PointT>::Ptr &cloud_beam_down, typename pcl::PointCloud<PointT>::Ptr &cloud_facade_down,
                          typename pcl::PointCloud<PointT>::Ptr &cloud_roof_down, typename pcl::PointCloud<PointT>::Ptr &cloud_vertex,
                          float neighbor_searching_radius, int neighbor_k, int neigh_k_min, int pca_down_rate, float edge_thre,
                          float planar_thre, float edge_thre_down, float planar_thre_down, int extract_vertex_points_method,
                          float curvature_thre, float vertex_curvature_non_max_radius, float linear_vertical_sin_high_thre,
                          float linear_vertical_sin_low_thre, float planar_vertical_sin_high_thre,
                          float planar_vertical_sin_low_thre, bool fixed_num_downsampling = false, int pillar_down_fixed_num = 200,
                          int facade_down_fixed_num = 800, int beam_down_fixed_num = 200, int roof_down_fixed_num = 100,
                          int unground_down_fixed_num = 20000, float beam_height_max = FLT_MAX, float roof_height_min = -FLT_MAX,
                          float feature_pts_ratio_guess = 0.3, bool sharpen_with_nms = true,
                          bool use_distance_adaptive_pca = false) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    static thread_local uint32_t call_seed = 0;
    mulls_classify_params p;
    mulls_classify_default_params(&p);
    p.neighbor_searching_radius = neighbor_searching_radius;
    p.neighbor_k = neighbor_k;
    p.neigh_k_min = neigh_k_min;
    p.pca_down_rate = pca_down_rate;
    p.edge_thre = edge_thre;
    p.planar_thre = planar_thre;
    p.edge_thre_down = edge_thre_down;
    p.planar_thre_down = planar_thre_down;
    p.extract_vertex_points_method = extract_vertex_points_method;
    p.curvature_thre = curvature_thre;
    p.vertex_curvature_non_max_radius = vertex_curvature_non_max_radius;
    p.linear_vertical_sin_high_thre = linear_vertical_sin_high_thre;
    p.linear_vertical_sin_low_thre = linear_vertical_sin_low_thre;
    p.planar_vertical_sin_high_thre = planar_vertical_sin_high_thre;
    p.planar_vertical_sin_low_thre = planar_vertical_sin_low_thre;
    p.fixed_num_downsampling = fixed_num_downsampling;
    p.pillar_down_fixed_num = pillar_down_fixed_num;
    p.facade_down_fixed_num = facade_down_fixed_num;
    p.beam_down_fixed_num = beam_down_fixed_num;
    p.roof_down_fixed_num = roof_down_fixed_num;
    p.unground_down_fixed_num = unground_down_fixed_num;
    p.beam_height_max = beam_height_max;
    p.roof_height_min = roof_height_min;
    p.feature_pts_ratio_guess = feature_pts_ratio_guess;
    p.sharpen_with_nms = sharpen_with_nms;
    p.use_distance_adaptive_pca = use_distance_adaptive_pca;
    p.pca_unit_distance = 30.0f; // the unit classify_nground_pts hands get_pc_pca_feature (cfilter.hpp:2093)
    p.random_seed = call_seed++;

    const size_t n = cloud_in->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<std::vector<PointT>> rows(MULLS_OUT_COUNT, std::vector<PointT>(n ? n : 1));
    mulls_classify_out out;
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) out.rows[k] = reinterpret_cast<float *>(rows[k].data()), out.n[k] = 0;
    out.cap = n ? n : 1;
    if (!ctx || mulls_classify_nground(ctx, view_of<PointT>(cloud_in), &p, &out) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    typename pcl::PointCloud<PointT>::Ptr *dst[MULLS_OUT_COUNT] = {&cloud_pillar,      &cloud_beam,        &cloud_facade,
                                                                   &cloud_roof,        &cloud_pillar_down, &cloud_beam_down,
                                                                   &cloud_facade_down, &cloud_roof_down,   &cloud_vertex,
                                                                   &cloud_in};
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) {
        if (k == MULLS_OUT_UNGROUND) (*dst[k])->points.clear(); // cloud_in is rewritten in place by the reference
        (*dst[k])->points.insert((*dst[k])->points.end(), rows[k].begin(), rows[k].begin() + out.n[k]);
    }
    return true;
}

// lo::CFilter<PointT>::fast_ground_filter (include/common/cfilter.hpp:1658-2036), same names, order, types and defaults
// as :1658-1672. cloud_curb / detect_curb_or_not are accepted and unused (the reference's curb code is `#if 0`, :1987).
// The output clouds are appended to, as the reference does. estimate_ground_normal_method 1 / 2 return false.
template <typename PointT>
bool fast_ground_filter(const typename pcl::PointCloud<PointT>::Ptr &cloud_in, typename pcl::PointCloud<PointT>::Ptr &cloud_ground,
                        typename pcl::PointCloud<PointT>::Ptr &cloud_ground_down, typename pcl::PointCloud<PointT>::Ptr &cloud_unground,
                        typename pcl::PointCloud<PointT>::Ptr &cloud_curb, int min_grid_pt_num, float grid_resolution,
                        float max_height_difference, float neighbor_height_diff, float max_ground_height,
                        int ground_random_down_rate, int ground_random_down_down_rate, int nonground_random_down_rate,
                        int reliable_neighbor_grid_num_thre, int estimate_ground_normal_method, float normal_estimation_radius,
                        int distance_weight_downsampling_method, float standard_distance, bool fixed_num_downsampling = false,
                        int down_ground_fixed_num = 1000, bool detect_curb_or_not = false, float intensity_thre = FLT_MAX,
                        bool apply_grid_wise_outlier_filter = false, float outlier_std_scale = 3.0) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    static thread_local uint32_t call_seed = 0;
    (void)cloud_curb;
    (void)detect_curb_or_not;
    mulls_ground_params p;
    mulls_ground_default_params(&p);
    p.min_grid_pt_num = min_grid_pt_num;
    p.grid_resolution = grid_resolution;
    p.max_height_difference = max_height_difference;
    p.neighbor_height_diff = neighbor_height_diff;
    p.max_ground_height = max_ground_height;
    p.ground_random_down_rate = ground_random_down_rate;
    p.ground_random_down_down_rate = ground_random_down_down_rate;
    p.nonground_random_down_rate = nonground_random_down_rate;
    p.reliable_neighbor_grid_num_thre = reliable_neighbor_grid_num_thre;
    p.estimate_ground_normal_method = estimate_ground_normal_method;
    p.normal_estimation_radius = normal_estimation_radius;
    p.distance_weight_downsampling_method = distance_weight_downsampling_method;
    p.standard_distance = standard_distance;
    p.fixed_num_downsampling = fixed_num_downsampling;
    p.down_ground_fixed_num = down_ground_fixed_num;
    p.intensity_thre = intensity_thre;
    p.apply_grid_wise_outlier_filter = apply_grid_wise_outlier_filter;
    p.outlier_std_scale = outlier_std_scale;
    p.random_seed = call_seed++;
    const size_t n = cloud_in->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<PointT> g(n ? n : 1), gd(n ? n : 1), u(n ? n : 1);
    mulls_ground_out out;
    out.ground = reinterpret_cast<float *>(g.data()), out.ground_down = reinterpret_cast<float *>(gd.data());
    out.unground = reinterpret_cast<float *>(u.data());
    out.cap = n ? n : 1;
    out.n_ground = out.n_ground_down = out.n_unground = 0;
    if (!ctx || mulls_fast_ground_filter(ctx, view_of<PointT>(cloud_in), &p, &out) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    cloud_ground->points.insert(cloud_ground->points.end(), g.begin(), g.begin() + out.n_ground);
    cloud_ground_down->points.insert(cloud_ground_down->points.end(), gd.begin(), gd.begin() + out.n_ground_down);
    cloud_unground->points.insert(cloud_unground->points.end(), u.begin(), u.begin() + out.n_unground);
    return true;
}

// lo::CFilter<PointT>::voxel_downsample (include/common/cfilter.hpp:83-165)
template <typename PointT>
bool voxel_downsample(const typename pcl::PointCloud<PointT>::Ptr &cloud_in, typename pcl::PointCloud<PointT>::Ptr &cloud_out,
                      float voxel_size) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    if (voxel_size < 0.001) { // :89-97: the reference shares the input cloud and reports "disabled"
        cloud_out = cloud_in;
        return false;
    }
    const size_t n = cloud_in->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<PointT> rows(n ? n : 1);
    size_t n_out = 0;
    if (!ctx || mulls_voxel_downsample(ctx, view_of<PointT>(cloud_in), voxel_size, reinterpret_cast<float *>(rows.data()),
                                       rows.size(), &n_out) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    cloud_out->points.insert(cloud_out->points.end(), rows.begin(), rows.begin() + n_out);
    return true;
}

// lo::CFilter<PointT>::sor_filter (include/common/cfilter.hpp:203-222): pcl::StatisticalOutlierRemoval with mean_k and
// n_std (mulls_sor_filter). cloud_out's points become the kept rows of cloud_in, all 48 bytes of each, in input order —
// what PCL's filter() copies; cloud_out may be cloud_in. Returns false (cloud_out untouched) when the call is refused:
// at most mean_k finite points, mean_k outside 1..63, no device.
template <typename PointT>
bool sor_filter(typename pcl::PointCloud<PointT>::Ptr &cloud_in, typename pcl::PointCloud<PointT>::Ptr &cloud_out, int mean_k,
                double n_std) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    const size_t n = cloud_in->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<uint8_t> keep((n + 7) / 8 + 1, 0);
    if (!ctx || mulls_sor_filter(ctx, view_of<PointT>(cloud_in), mean_k, n_std, keep.data(), nullptr, nullptr) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    std::vector<PointT> kept;
    kept.reserve(n);
    for (size_t i = 0; i < n; ++i)
        if ((keep[i >> 3] >> (i & 7)) & 1u) kept.push_back(cloud_in->points[i]);
    cloud_out->points.swap(kept);
    return true;
}

// lo::CFilter<PointT>::sor_filter, the in-place overload (include/common/cfilter.hpp:224-247)
template <typename PointT>
bool sor_filter(typename pcl::PointCloud<PointT>::Ptr &cloud_in_out, int mean_k, double n_std) {
    return sor_filter<PointT>(cloud_in_out, cloud_in_out, mean_k, n_std);
}

// lo::CFilter<PointT>::non_max_suppress, the in-place overload (include/common/cfilter.hpp:1183-1240) with
// kd_tree_already_built = false (mulls_non_max_suppress): the cloud's points become its kept rows, all 48 bytes of each,
// in the reference's order (score descending; abi.h states the readings). width and height are not touched, as in the
// reference. Returns false with the cloud untouched for fewer than 10 points, as the reference, or when the call is
// refused (no device).
template <typename PointT>
bool non_max_suppress(typename pcl::PointCloud<PointT>::Ptr &cloud_in_out, float non_max_radius) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    const size_t n = cloud_in_out->points.size();
    if (n < 10) return false;
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<int32_t> idx(n);
    size_t n_kept = 0;
    int performed = 0;
    if (!ctx || mulls_non_max_suppress(ctx, view_of<PointT>(cloud_in_out), non_max_radius, idx.data(), &n_kept, &performed) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    std::vector<PointT> kept;
    kept.reserve(n_kept);
    for (size_t k = 0; k < n_kept; ++k) kept.push_back(cloud_in_out->points[idx[k]]);
    cloud_in_out->points.swap(kept);
    return performed != 0;
}

// lo::CFilter<PointT>::scanner_filter (include/common/cfilter.hpp:914-929) in float, on the host: drops the points within
// self_radius of the scanner axis (the ego vehicle) or below z_min_thre_global, and the points within ghost_radius that
// lie at or below z_min_thre_ghost (underground ghosts). The kept rows stay in input order; the cloud shrinks in place.
template <typename PointT>
bool scanner_filter(const typename pcl::PointCloud<PointT>::Ptr &cloud_in_out, float self_radius, float ghost_radius,
                    float z_min_thre_ghost, float z_min_thre_global) {
    std::vector<PointT> kept;
    kept.reserve(cloud_in_out->points.size());
    for (const PointT &p : cloud_in_out->points) {
        const float dis_square = p.x * p.x + p.y * p.y;
        if (dis_square > self_radius * self_radius && p.z > z_min_thre_global)
            if (dis_square > ghost_radius * ghost_radius || p.z > z_min_thre_ghost) kept.push_back(p);
    }
    cloud_in_out->points.swap(kept);
    return true;
}

// lo::CFilter<PointT>::extract_semantic_pts (include/common/cfilter.hpp:2295-2413): same names, order, types and
// defaults as :2295-2318. With apply_scanner_filter (and no semantic_assisted) pc_raw first goes through scanner_filter
// as at :2334-2343, and shrinks in place as in the reference. Covers :2346-2399 — voxel_downsample, pc_sketch, fast_ground_filter, classify_nground_pts and
// the feature count — with the three heavy stages chained in HBM (mulls_extract_semantic_pts): replace those lines of
// the member by a call forwarding every argument. The semantic-mask pre-filter (:2331-2332) and
// update_parameters_self_adaptive (:2406-2410) are CFilter members and stay where they are, before / after the call.
template <typename PointT, typename BlockPtr>
bool extract_semantic_pts(BlockPtr in_block, float vf_downsample_resolution, float gf_grid_resolution, float gf_max_grid_height_diff,
                          float gf_neighbor_height_diff, float gf_max_ground_height, int &gf_down_rate_ground,
                          int &gf_downsample_rate_nonground, float pca_neighbor_radius, int pca_neighbor_k, float edge_thre,
                          float planar_thre, float curvature_thre, float edge_thre_down, float planar_thre_down,
                          bool use_distance_adaptive_pca = false, int distance_inverse_sampling_method = 0,
                          float standard_distance = 15.0, int estimate_ground_normal_method = 3,
                          float normal_estimation_radius = 2.0, bool use_adpative_parameters = false,
                          bool apply_scanner_filter = false, bool extract_curb_or_not = false,
                          int extract_vertex_points_method = 2, int gf_grid_pt_num_thre = 8,
                          int gf_reliable_neighbor_grid_thre = 0, int gf_down_down_rate_ground = 2, int pca_neighbor_k_min = 8,
                          int pca_down_rate = 1, float intensity_thre = FLT_MAX, float linear_vertical_sin_high_thre = 0.94,
                          float linear_vertical_sin_low_thre = 0.17, float planar_vertical_sin_high_thre = 0.98,
                          float planar_vertical_sin_low_thre = 0.34, bool sharpen_with_nms_on = true,
                          bool fixed_num_downsampling = false, int ground_down_fixed_num = 500, int pillar_down_fixed_num = 200,
                          int facade_down_fixed_num = 800, int beam_down_fixed_num = 200, int roof_down_fixed_num = 200,
                          int unground_down_fixed_num = 20000, float beam_height_max = FLT_MAX, float roof_height_min = 0.0,
                          float approx_scanner_height = 2.0, float underground_thre = -7.0, float feature_pts_ratio_guess = 0.3,
                          bool semantic_assisted = false, bool apply_roi_filtering = false, float roi_min_y = 0.0,
                          float roi_max_y = 0.0) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    static thread_local uint32_t call_seed = 0;
    (void)use_adpative_parameters, (void)extract_curb_or_not;
    (void)apply_roi_filtering, (void)roi_min_y, (void)roi_max_y;
    if (!semantic_assisted && apply_scanner_filter) { // :2331-2343 (the semantic mask branch is not covered)
        float self_ring_radius = 1.75;
        float ghost_radius = 20.0;
        float z_min = -approx_scanner_height - 4.0;
        float z_min_min = -approx_scanner_height + underground_thre;
        scanner_filter<PointT>(in_block->pc_raw, self_ring_radius, ghost_radius, z_min, z_min_min);
    }
    mulls_extract_params P;
    P.vf_downsample_resolution = vf_downsample_resolution;
    mulls_ground_default_params(&P.ground);
    P.ground.min_grid_pt_num = gf_grid_pt_num_thre;
    P.ground.grid_resolution = gf_grid_resolution;
    P.ground.max_height_difference = gf_max_grid_height_diff;
    P.ground.neighbor_height_diff = gf_neighbor_height_diff;
    P.ground.max_ground_height = gf_max_ground_height;
    P.ground.ground_random_down_rate = gf_down_rate_ground;
    P.ground.ground_random_down_down_rate = gf_down_down_rate_ground;
    P.ground.nonground_random_down_rate = gf_downsample_rate_nonground;
    P.ground.reliable_neighbor_grid_num_thre = gf_reliable_neighbor_grid_thre;
    P.ground.estimate_ground_normal_method = estimate_ground_normal_method;
    P.ground.normal_estimation_radius = normal_estimation_radius;
    P.ground.distance_weight_downsampling_method = distance_inverse_sampling_method;
    P.ground.standard_distance = standard_distance;
    P.ground.fixed_num_downsampling = fixed_num_downsampling;
    P.ground.down_ground_fixed_num = ground_down_fixed_num;
    P.ground.intensity_thre = intensity_thre;
    P.ground.apply_grid_wise_outlier_filter = apply_scanner_filter; // the argument extract_semantic_pts passes there (:2361)
    P.ground.random_seed = call_seed;
    mulls_classify_default_params(&P.classify);
    P.classify.neighbor_searching_radius = pca_neighbor_radius;
    P.classify.neighbor_k = pca_neighbor_k;
    P.classify.neigh_k_min = pca_neighbor_k_min;
    P.classify.pca_down_rate = pca_down_rate;
    P.classify.edge_thre = edge_thre;
    P.classify.planar_thre = planar_thre;
    P.classify.edge_thre_down = edge_thre_down;
    P.classify.planar_thre_down = planar_thre_down;
    P.classify.extract_vertex_points_method = extract_vertex_points_method;
    P.classify.curvature_thre = curvature_thre;
    P.classify.vertex_curvature_non_max_radius = 1.5 * pca_neighbor_radius; // :2363
    P.classify.linear_vertical_sin_high_thre = linear_vertical_sin_high_thre;
    P.classify.linear_vertical_sin_low_thre = linear_vertical_sin_low_thre;
    P.classify.planar_vertical_sin_high_thre = planar_vertical_sin_high_thre;
    P.classify.planar_vertical_sin_low_thre = planar_vertical_sin_low_thre;
    P.classify.fixed_num_downsampling = fixed_num_downsampling;
    P.classify.pillar_down_fixed_num = pillar_down_fixed_num;
    P.classify.facade_down_fixed_num = facade_down_fixed_num;
    P.classify.beam_down_fixed_num = beam_down_fixed_num;
    P.classify.roof_down_fixed_num = roof_down_fixed_num;
    P.classify.unground_down_fixed_num = unground_down_fixed_num;
    P.classify.beam_height_max = beam_height_max;
    P.classify.roof_height_min = roof_height_min;
    P.classify.feature_pts_ratio_guess = feature_pts_ratio_guess;
    P.classify.sharpen_with_nms = sharpen_with_nms_on;
    P.classify.use_distance_adaptive_pca = use_distance_adaptive_pca;
    P.classify.pca_unit_distance = 30.0f; // cfilter.hpp:2093
    P.classify.random_seed = call_seed++;

    const size_t n = in_block->pc_raw->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    const size_t cap = n ? n : 1;
    std::vector<PointT> down(cap), ground(cap), ground_down(cap);
    std::vector<std::vector<PointT>> rows(MULLS_OUT_COUNT, std::vector<PointT>(cap));
    mulls_extract_out out;
    out.pc_down = reinterpret_cast<float *>(down.data());
    out.pc_ground = reinterpret_cast<float *>(ground.data());
    out.pc_ground_down = reinterpret_cast<float *>(ground_down.data());
    out.cap = cap;
    out.n_down = out.n_ground = out.n_ground_down = 0;
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) out.cls.rows[k] = reinterpret_cast<float *>(rows[k].data()), out.cls.n[k] = 0;
    out.cls.cap = cap;
    if (!ctx || mulls_extract_semantic_pts(ctx, view_of<PointT>(in_block->pc_raw), &P, &out) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    auto append = [](typename pcl::PointCloud<PointT>::Ptr &dst, const std::vector<PointT> &src, size_t cnt) {
        dst->points.insert(dst->points.end(), src.begin(), src.begin() + cnt);
    };
    if (vf_downsample_resolution < 0.001) in_block->pc_down = in_block->pc_raw; // :92 the reference shares the cloud
    else append(in_block->pc_down, down, out.n_down);
    {   // :2348 random_downsample(pc_down, pc_sketch, size / 1024 + 1): every k-th point (:713-728)
        const int ratio = (int)(in_block->pc_down->points.size() / 1024 + 1);
        if (ratio > 1) {
            in_block->pc_sketch->points.clear();
            for (size_t i = 0; i < in_block->pc_down->points.size(); i += (size_t)ratio)
                in_block->pc_sketch->points.push_back(in_block->pc_down->points[i]);
        }
    }
    append(in_block->pc_ground, ground, out.n_ground);
    append(in_block->pc_ground_down, ground_down, out.n_ground_down);
    typename pcl::PointCloud<PointT>::Ptr *dst[MULLS_OUT_COUNT] = {
        &in_block->pc_pillar,      &in_block->pc_beam,      &in_block->pc_facade,      &in_block->pc_roof,   &in_block->pc_pillar_down,
        &in_block->pc_beam_down,   &in_block->pc_facade_down, &in_block->pc_roof_down, &in_block->pc_vertex, &in_block->pc_unground};
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) append(*dst[k], rows[k], out.cls.n[k]);
    in_block->down_feature_point_num = in_block->pc_ground_down->points.size() + in_block->pc_pillar_down->points.size() +
                                       in_block->pc_beam_down->points.size() + in_block->pc_facade_down->points.size() +
                                       in_block->pc_roof_down->points.size() + in_block->pc_vertex->points.size(); // :2398-2399
    return true;
}

// ---- raw-scan corrections (mulls_vertical_intrinsic_calibration, mulls_timestamp_ratio, mulls_motion_compensation):
// the cloud's rows go to the device, the changed column comes back and is scattered into points[i]. A refused call (no
// device) logs the error and leaves the cloud as it was.

// lo::CFilter<PointT>::vertical_intrinsic_calibration (include/common/cfilter.hpp:250-291), same defaults
template <typename PointT>
bool vertical_intrinsic_calibration(typename pcl::PointCloud<PointT>::Ptr &cloud_in_out, double var_vertical_ang_d = 0.0,
                                    bool inverse_z = false) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    if (var_vertical_ang_d == 0) return false; // :252-253
    const size_t n = cloud_in_out->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<float> xyz(3 * n + 1);
    int applied = 0;
    if (!ctx || mulls_vertical_intrinsic_calibration(ctx, view_of<PointT>(cloud_in_out), var_vertical_ang_d, inverse_z ? 1 : 0,
                                                     xyz.data(), &applied) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    for (size_t i = 0; i < n; ++i) {
        PointT &p = cloud_in_out->points[i];
        p.x = xyz[3 * i], p.y = xyz[3 * i + 1], p.z = xyz[3 * i + 2];
    }
    return applied != 0;
}

// lo::CFilter<PointT>::get_pts_timestamp_ratio_in_frame (include/common/cfilter.hpp:412-467), same defaults: the
// curvature of every point becomes its timestamp ratio in the frame
template <typename PointT>
bool get_pts_timestamp_ratio_in_frame(typename pcl::PointCloud<PointT>::Ptr &cloud_in_out, bool timestamp_availiable = true,
                                      double scan_begin_ang_anticlock_x_positive_deg = 180.0, float scan_duration_ms = 100) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    const size_t n = cloud_in_out->points.size();
    mulls_ctx *ctx = thread_context(1, n);
    std::vector<float> ratio(n + 1);
    if (!ctx || mulls_timestamp_ratio(ctx, view_of<PointT>(cloud_in_out), timestamp_availiable ? 1 : 0,
                                      scan_begin_ang_anticlock_x_positive_deg, scan_duration_ms, ratio.data()) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    for (size_t i = 0; i < n; ++i) cloud_in_out->points[i].curvature = ratio[i];
    return true;
}

// apply_motion_compensation over n_clouds (in[k] -> out[k]) pairs in one device call; out[k] may be in[k]. When two
// pairs share a cloud the reference's sequential order matters, and the pairs are run one call each, in order.
template <typename PointT>
bool motion_compensation(const typename pcl::PointCloud<PointT>::Ptr *in, const typename pcl::PointCloud<PointT>::Ptr *out,
                         int n_clouds, const Eigen::Matrix4d &Tran, float s_ambigous_thre) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    for (int a = 0; a < n_clouds; ++a)
        for (int b = a + 1; b < n_clouds; ++b)
            if (in[a].get() == in[b].get() || in[a].get() == out[b].get() || out[a].get() == in[b].get() ||
                out[a].get() == out[b].get()) {
                bool ok = true;
                for (int k = 0; k < n_clouds; ++k) ok = motion_compensation<PointT>(in + k, out + k, 1, Tran, s_ambigous_thre) && ok;
                return ok;
            }
    double T[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) T[4 * r + c] = Tran(r, c);
    mulls_cloud_view views[MULLS_NUM_CLASSES];
    std::vector<float> xyz[MULLS_NUM_CLASSES];
    float *dst[MULLS_NUM_CLASSES];
    size_t total = 0;
    for (int k = 0; k < n_clouds; ++k) {
        views[k] = view_of<PointT>(in[k]);
        xyz[k].resize(3 * views[k].n + 1);
        dst[k] = xyz[k].data();
        total += views[k].n;
    }
    mulls_ctx *ctx = thread_context(1, total);
    if (!ctx || mulls_motion_compensation(ctx, views, n_clouds, T, s_ambigous_thre, dst) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    for (int k = 0; k < n_clouds; ++k) {
        if (out[k].get() != in[k].get()) *out[k] = *in[k]; // :496
        for (size_t i = 0; i < views[k].n; ++i) {
            PointT &p = out[k]->points[i];
            p.x = xyz[k][3 * i], p.y = xyz[k][3 * i + 1], p.z = xyz[k][3 * i + 2];
        }
    }
    return true;
}

// lo::CFilter<PointT>::apply_motion_compensation, in place (include/common/cfilter.hpp:470-491)
template <typename PointT>
void apply_motion_compensation(typename pcl::PointCloud<PointT>::Ptr pc_in_out, Eigen::Matrix4d &Tran, float s_ambigous_thre = 0.000) {
    motion_compensation<PointT>(&pc_in_out, &pc_in_out, 1, Tran, s_ambigous_thre);
}

// lo::CFilter<PointT>::apply_motion_compensation, pc_in -> pc_out (include/common/cfilter.hpp:493-516)
template <typename PointT>
void apply_motion_compensation(const typename pcl::PointCloud<PointT>::Ptr pc_in, typename pcl::PointCloud<PointT>::Ptr pc_out,
                               Eigen::Matrix4d &Tran, float s_ambigous_thre = 0.0) {
    motion_compensation<PointT>(&pc_in, &pc_out, 1, Tran, s_ambigous_thre);
}

// lo::CFilter<PointT>::batch_apply_motion_compensation, in place (include/common/cfilter.hpp:519-531): five or six
// clouds in one call, with the threshold 0 of the calls it makes
template <typename PointT>
void batch_apply_motion_compensation(typename pcl::PointCloud<PointT>::Ptr pc_ground, typename pcl::PointCloud<PointT>::Ptr pc_pillar,
                                     typename pcl::PointCloud<PointT>::Ptr pc_beam, typename pcl::PointCloud<PointT>::Ptr pc_facade,
                                     typename pcl::PointCloud<PointT>::Ptr pc_roof, typename pcl::PointCloud<PointT>::Ptr pc_vertex,
                                     Eigen::Matrix4d &Tran, bool undistort_keypoints_or_not = false) {
    const typename pcl::PointCloud<PointT>::Ptr c[6] = {pc_ground, pc_pillar, pc_beam, pc_facade, pc_roof, pc_vertex};
    motion_compensation<PointT>(c, c, undistort_keypoints_or_not ? 6 : 5, Tran, 0.0f);
}

// lo::CFilter<PointT>::batch_apply_motion_compensation, into the *_undistort clouds (include/common/cfilter.hpp:534-549)
template <typename PointT>
void batch_apply_motion_compensation(
    const typename pcl::PointCloud<PointT>::Ptr pc_ground, const typename pcl::PointCloud<PointT>::Ptr pc_pillar,
    const typename pcl::PointCloud<PointT>::Ptr pc_beam, const typename pcl::PointCloud<PointT>::Ptr pc_facade,
    const typename pcl::PointCloud<PointT>::Ptr pc_roof, const typename pcl::PointCloud<PointT>::Ptr pc_vertex,
    typename pcl::PointCloud<PointT>::Ptr pc_ground_undistort, typename pcl::PointCloud<PointT>::Ptr pc_pillar_undistort,
    typename pcl::PointCloud<PointT>::Ptr pc_beam_undistort, typename pcl::PointCloud<PointT>::Ptr pc_facade_undistort,
    typename pcl::PointCloud<PointT>::Ptr pc_roof_undistort, typename pcl::PointCloud<PointT>::Ptr pc_vertex_undistort,
    Eigen::Matrix4d &Tran, bool undistort_keypoints_or_not = false) {
    const typename pcl::PointCloud<PointT>::Ptr in[6] = {pc_ground, pc_pillar, pc_beam, pc_facade, pc_roof, pc_vertex};
    const typename pcl::PointCloud<PointT>::Ptr out[6] = {pc_ground_undistort, pc_pillar_undistort, pc_beam_undistort,
                                                          pc_facade_undistort, pc_roof_undistort, pc_vertex_undistort};
    motion_compensation<PointT>(in, out, undistort_keypoints_or_not ? 6 : 5, Tran, 0.0f);
}

} // namespace b200
} // namespace lo
#endif
