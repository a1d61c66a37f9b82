// DROP-IN replacement of lo::CFilter<PointT> (reference: include/common/cfilter.hpp). Same mechanism as
// dropin/cregistration.hpp: this directory goes BEFORE the reference's include/common on the include path; the
// reference's own cfilter.hpp is pulled in with its class renamed to CFilter_reference, and lo::CFilter<PointT> is
// defined here as a class derived from it whose extract_semantic_pts (cfilter.hpp:2295-2318: same name, argument
// order, types and defaults — all fifty of them), voxel_downsample (:83), fast_ground_filter (:1658-1672),
// classify_nground_pts (:2058-2081), both sor_filter overloads (:204, :225), the in-place non_max_suppress (:1183) without
// a prebuilt tree, vertical_intrinsic_calibration (:250), get_pts_timestamp_ratio_in_frame (:412) and every overload of
// apply_motion_compensation (:470, :493) and batch_apply_motion_compensation (:519, :534) run on the GPU through the C-ABI.
// Every other member (dist_filter, the in-place non_max_suppress with kd_tree_already_built, the non_max_suppress
// overloads of :1243 and :1314, random_downsample, get_cloud_bbx, ... SURVEY.md section 8b) is inherited from the
// reference. test/mulls_slam.cpp:360-377, :462, :1008-1009 and test/mulls_reg.cpp:134-149 compile unchanged.
#ifndef MULLS_B200_DROPIN_CFILTER_HPP
#define MULLS_B200_DROPIN_CFILTER_HPP

#define CFilter CFilter_reference
#include_next "cfilter.hpp"
#undef CFilter

#include <cstddef>
#include <utility>
#include <vector>

#include "common/cfilter_b200.hpp"

namespace lo {

template <typename PointT>
class CFilter : public CFilter_reference<PointT> {
    typedef typename pcl::PointCloud<PointT>::Ptr CloudPtr;

  public:
    // cfilter.hpp:2295-2318
    bool extract_semantic_pts(cloudblock_Ptr in_block, float vf_downsample_resolution, float gf_grid_resolution,
                              float gf_max_grid_height_diff, float gf_neighbor_height_diff, float gf_max_ground_height,
                              int &gf_down_rate_ground, int &gf_downsample_rate_nonground, float pca_neighbor_radius,
                              int pca_neighbor_k, float edge_thre, float planar_thre, float curvature_thre, float edge_thre_down,
                              float planar_thre_down, bool use_distance_adaptive_pca = false,
                              int distance_inverse_sampling_method = 0, float standard_distance = 15.0,
                              int estimate_ground_normal_method = 3, float normal_estimation_radius = 2.0,
                              bool use_adpative_parameters = false, bool apply_scanner_filter = false,
                              bool extract_curb_or_not = false, int extract_vertex_points_method = 2,
                              int gf_grid_pt_num_thre = 8, int gf_reliable_neighbor_grid_thre = 0,
                              int gf_down_down_rate_ground = 2, int pca_neighbor_k_min = 8, int pca_down_rate = 1,
                              float intensity_thre = FLT_MAX, float linear_vertical_sin_high_thre = 0.94,
                              float linear_vertical_sin_low_thre = 0.17, float planar_vertical_sin_high_thre = 0.98,
                              float planar_vertical_sin_low_thre = 0.34, bool sharpen_with_nms_on = true,
                              bool fixed_num_downsampling = false, int ground_down_fixed_num = 500,
                              int pillar_down_fixed_num = 200, int facade_down_fixed_num = 800, int beam_down_fixed_num = 200,
                              int roof_down_fixed_num = 200, int unground_down_fixed_num = 20000, float beam_height_max = FLT_MAX,
                              float roof_height_min = 0.0, float approx_scanner_height = 2.0, float underground_thre = -7.0,
                              float feature_pts_ratio_guess = 0.3, bool semantic_assisted = false,
                              bool apply_roi_filtering = false, float roi_min_y = 0.0, float roi_max_y = 0.0) {
        return b200::extract_semantic_pts<PointT>(
            in_block, vf_downsample_resolution, gf_grid_resolution, gf_max_grid_height_diff, gf_neighbor_height_diff,
            gf_max_ground_height, gf_down_rate_ground, gf_downsample_rate_nonground, pca_neighbor_radius, pca_neighbor_k, edge_thre,
            planar_thre, curvature_thre, edge_thre_down, planar_thre_down, use_distance_adaptive_pca,
            distance_inverse_sampling_method, standard_distance, estimate_ground_normal_method, normal_estimation_radius,
            use_adpative_parameters, apply_scanner_filter, extract_curb_or_not, extract_vertex_points_method, gf_grid_pt_num_thre,
            gf_reliable_neighbor_grid_thre, gf_down_down_rate_ground, pca_neighbor_k_min, pca_down_rate, intensity_thre,
            linear_vertical_sin_high_thre, linear_vertical_sin_low_thre, planar_vertical_sin_high_thre,
            planar_vertical_sin_low_thre, sharpen_with_nms_on, fixed_num_downsampling, ground_down_fixed_num,
            pillar_down_fixed_num, facade_down_fixed_num, beam_down_fixed_num, roof_down_fixed_num, unground_down_fixed_num,
            beam_height_max, roof_height_min, approx_scanner_height, underground_thre, feature_pts_ratio_guess, semantic_assisted,
            apply_roi_filtering, roi_min_y, roi_max_y);
    }
    // cfilter.hpp:83
    bool voxel_downsample(const CloudPtr &cloud_in, CloudPtr &cloud_out, float voxel_size) {
        return b200::voxel_downsample<PointT>(cloud_in, cloud_out, voxel_size);
    }
    // cfilter.hpp:204 and :225 (test/mulls_slam.cpp:1009 runs the in-place one on the merged map)
    bool sor_filter(CloudPtr &cloud_in, CloudPtr &cloud_out, int mean_k, double n_std) {
        return b200::sor_filter<PointT>(cloud_in, cloud_out, mean_k, n_std);
    }
    bool sor_filter(CloudPtr &cloud_in_out, int mean_k, double n_std) { return b200::sor_filter<PointT>(cloud_in_out, mean_k, n_std); }
    // cfilter.hpp:1183 (test/mulls_reg.cpp:147-148, test/mulls_slam.cpp:462), same defaults. A prebuilt tree indexes the
    // cloud as it was before the sort: that form stays with the reference member. The tree's pointer type is a template
    // parameter (its default the reference's NULL), so the reference member is named only when that form is compiled.
    bool non_max_suppress(CloudPtr &cloud_in_out, float non_max_radius) {
        return b200::non_max_suppress<PointT>(cloud_in_out, non_max_radius);
    }
    template <typename TreePtr = std::nullptr_t>
    bool non_max_suppress(CloudPtr &cloud_in_out, float non_max_radius, bool kd_tree_already_built,
                          const TreePtr &built_tree = TreePtr()) {
        if (kd_tree_already_built)
            return CFilter_reference<PointT>::non_max_suppress(cloud_in_out, non_max_radius, kd_tree_already_built, built_tree);
        return b200::non_max_suppress<PointT>(cloud_in_out, non_max_radius);
    }
    // The other two overloads, :1243 into cloud_out and :1314 on pca_feature_t, stay the reference's. Declaring the
    // in-place one hides them, so they are forwarded.
    template <typename... Args>
    bool non_max_suppress(CloudPtr &cloud_in, CloudPtr &cloud_out, Args &&...args) {
        return CFilter_reference<PointT>::non_max_suppress(cloud_in, cloud_out, std::forward<Args>(args)...);
    }
    template <typename Feature, typename IndicesPtr>
    bool non_max_suppress(std::vector<Feature> &features, IndicesPtr &indices, float nms_radius) {
        return CFilter_reference<PointT>::non_max_suppress(features, indices, nms_radius);
    }
    // cfilter.hpp:250 (test/mulls_slam.cpp:362, :407, :967)
    bool vertical_intrinsic_calibration(CloudPtr &cloud_in_out, double var_vertical_ang_d = 0.0, bool inverse_z = false) {
        return b200::vertical_intrinsic_calibration<PointT>(cloud_in_out, var_vertical_ang_d, inverse_z);
    }
    // cfilter.hpp:412 (test/mulls_slam.cpp:410-412, :972-974)
    bool get_pts_timestamp_ratio_in_frame(CloudPtr &cloud_in_out, bool timestamp_availiable = true,
                                          double scan_begin_ang_anticlock_x_positive_deg = 180.0, float scan_duration_ms = 100) {
        return b200::get_pts_timestamp_ratio_in_frame<PointT>(cloud_in_out, timestamp_availiable,
                                                              scan_begin_ang_anticlock_x_positive_deg, scan_duration_ms);
    }
    // cfilter.hpp:470 and :493 (test/mulls_slam.cpp:707, :980, :1001). Both overloads: declaring one hides the other.
    void apply_motion_compensation(CloudPtr pc_in_out, Eigen::Matrix4d &Tran, float s_ambigous_thre = 0.000) {
        b200::apply_motion_compensation<PointT>(pc_in_out, Tran, s_ambigous_thre);
    }
    void apply_motion_compensation(const CloudPtr pc_in, CloudPtr pc_out, Eigen::Matrix4d &Tran, float s_ambigous_thre = 0.0) {
        b200::apply_motion_compensation<PointT>(pc_in, pc_out, Tran, s_ambigous_thre);
    }
    // cfilter.hpp:519 and :534 (test/mulls_slam.cpp:708-711): the five or six clouds in one device call
    void batch_apply_motion_compensation(CloudPtr pc_ground, CloudPtr pc_pillar, CloudPtr pc_beam, CloudPtr pc_facade, CloudPtr pc_roof,
                                         CloudPtr pc_vertex, Eigen::Matrix4d &Tran, bool undistort_keypoints_or_not = false) {
        b200::batch_apply_motion_compensation<PointT>(pc_ground, pc_pillar, pc_beam, pc_facade, pc_roof, pc_vertex, Tran,
                                                      undistort_keypoints_or_not);
    }
    void batch_apply_motion_compensation(const CloudPtr pc_ground, const CloudPtr pc_pillar, const CloudPtr pc_beam,
                                         const CloudPtr pc_facade, const CloudPtr pc_roof, const CloudPtr pc_vertex,
                                         CloudPtr pc_ground_undistort, CloudPtr pc_pillar_undistort, CloudPtr pc_beam_undistort,
                                         CloudPtr pc_facade_undistort, CloudPtr pc_roof_undistort, CloudPtr pc_vertex_undistort,
                                         Eigen::Matrix4d &Tran, bool undistort_keypoints_or_not = false) {
        b200::batch_apply_motion_compensation<PointT>(pc_ground, pc_pillar, pc_beam, pc_facade, pc_roof, pc_vertex,
                                                      pc_ground_undistort, pc_pillar_undistort, pc_beam_undistort,
                                                      pc_facade_undistort, pc_roof_undistort, pc_vertex_undistort, Tran,
                                                      undistort_keypoints_or_not);
    }
};

} // namespace lo
#endif
