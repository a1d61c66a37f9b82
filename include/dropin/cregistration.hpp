// DROP-IN replacement of lo::CRegistration<PointT> (reference: include/common/cregistration.hpp:56-3384).
//
// Put this directory BEFORE the reference's include/common on the include path and link -lmulls_b200:
//
//     g++ ... -I<mulls_b200>/include/dropin -I<mulls_b200>/include -I<MULLS>/include/common -I<MULLS>/include/... \
//         test/mulls_reg.cpp ... -L<mulls_b200>/mulls_b200/csrc -lmulls_b200
//
// Neither the reference's headers nor test/mulls_reg.cpp / test/mulls_slam.cpp are edited: they go on writing
// `#include "cregistration.hpp"` and `CRegistration<Point_T> creg; creg.mm_lls_icp(reg_con, ...)`. What happens:
//   * `#include_next` pulls in the reference's own cregistration.hpp with its class renamed (one macro) to
//     CRegistration_reference — every member the reference defines stays available, unchanged;
//   * lo::CRegistration<PointT> is then defined HERE as a class derived from it whose mm_lls_icp
//     (cregistration.hpp:1114-1123: same name, argument order, types and defaults) and mm_lls_icp_4dof_global
//     (:1584-1592), find_feature_correspondence_ncc (:409-411), coarse_reg_ransac (:605-607), coarse_reg_teaser
//     (:664-666), omp_ndt (:945-947) and omp_gicp (:1024-1027) run on the GPU through the C-ABI
//     (include/mulls_b200/abi.h); coarse_reg_teaser runs whether or not the reference was built with TEASER_ON. All
//     other public members the callers use — determine_source_target_cloud, assign_source_target_cloud,
//     ... (SURVEY.md section 8b) — are inherited from the reference; every overload of
//     coarse_reg_ransac the reference class declares stays visible next to the device one.
// Differences in contract are listed in INTEGRATION.md (block1->tree_* are not populated: use mulls_nn_query or
// the drop-in lo::MapManager of dropin/map_manager.h, which does not need them).
#ifndef MULLS_B200_DROPIN_CREGISTRATION_HPP
#define MULLS_B200_DROPIN_CREGISTRATION_HPP

#define CRegistration CRegistration_reference
#include_next "cregistration.hpp"
#undef CRegistration

#include "common/cregistration_b200.hpp"
#include "pgo/map_manager_b200.hpp"

namespace lo {

template <typename PointT>
class CRegistration : public CRegistration_reference<PointT> {
  public:
    // cregistration.hpp:1114-1123
    int mm_lls_icp(constraint_t &registration_cons, // cblock_1 (target point cloud), cblock_2 (source point cloud)
                   int max_iter_num = 20, float dis_thre_unit = 1.5, float converge_translation = 0.002,
                   float converge_rotation_d = 0.01, float dis_thre_min = 0.4, float dis_thre_update_rate = 1.1,
                   std::string used_feature_type = "111110", std::string weight_strategy = "1101",
                   float z_xy_balanced_ratio = 1.0, float pt2pt_residual_window = 0.1, float pt2pl_residual_window = 0.1,
                   float pt2li_residual_window = 0.1, Eigen::Matrix4d initial_guess = Eigen::Matrix4d::Identity(),
                   bool apply_intersection_filter = true, bool apply_motion_undistortion_while_registration = false,
                   bool normal_shooting_on = false, float normal_bearing = 45.0, bool use_more_points = false,
                   bool keep_less_source_points = false, float sigma_thre = 0.5, float min_neccessary_corr_ratio = 0.03,
                   float max_bearable_rotation_d = 45.0) {
        // the target is a local map that lo::MapManager::update_local_map keeps in HBM (test/mulls_slam.cpp:669-685):
        // register against that copy — nothing but the scan's feature clouds crosses PCIe
        if (b200::MapManagerB200 *resident = b200::resident_map_if_current(registration_cons.block1.get()))
            return resident->mm_lls_icp(registration_cons, max_iter_num, dis_thre_unit, converge_translation, converge_rotation_d,
                                        dis_thre_min, dis_thre_update_rate, used_feature_type, weight_strategy, z_xy_balanced_ratio,
                                        pt2pt_residual_window, pt2pl_residual_window, pt2li_residual_window, initial_guess,
                                        apply_intersection_filter, apply_motion_undistortion_while_registration, normal_shooting_on,
                                        normal_bearing, use_more_points, keep_less_source_points, sigma_thre,
                                        min_neccessary_corr_ratio, max_bearable_rotation_d);
        return b200::mm_lls_icp<PointT>(registration_cons, max_iter_num, dis_thre_unit, converge_translation, converge_rotation_d,
                                        dis_thre_min, dis_thre_update_rate, used_feature_type, weight_strategy, z_xy_balanced_ratio,
                                        pt2pt_residual_window, pt2pl_residual_window, pt2li_residual_window, initial_guess,
                                        apply_intersection_filter, apply_motion_undistortion_while_registration, normal_shooting_on,
                                        normal_bearing, use_more_points, keep_less_source_points, sigma_thre,
                                        min_neccessary_corr_ratio, max_bearable_rotation_d);
    }
    // cregistration.hpp:1584-1592
    bool mm_lls_icp_4dof_global(constraint_t &registration_con, float heading_step_d, int max_iter_num = 20,
                                float dis_thre_unit = 1.5, float converge_translation = 0.005,
                                float converge_rotation_d = 0.05, float dis_thre_min = 0.5,
                                float dis_thre_update_rate = 1.05, float max_bearable_rotation_d = 15.0) {
        return b200::mm_lls_icp_4dof_global<PointT>(registration_con, heading_step_d, max_iter_num, dis_thre_unit, converge_translation,
                                                    converge_rotation_d, dis_thre_min, dis_thre_update_rate, max_bearable_rotation_d);
    }
    // cregistration.hpp:409-411
    bool find_feature_correspondence_ncc(const typename pcl::PointCloud<PointT>::Ptr &target_kpts,
                                         const typename pcl::PointCloud<PointT>::Ptr &source_kpts,
                                         typename pcl::PointCloud<PointT>::Ptr &target_corrs,
                                         typename pcl::PointCloud<PointT>::Ptr &source_corrs, bool fixed_num_corr = false,
                                         int corr_num = 2000, bool reciprocal_on = true) {
        return b200::find_feature_correspondence_ncc<PointT>(target_kpts, source_kpts, target_corrs, source_corrs, fixed_num_corr,
                                                             corr_num, reciprocal_on);
    }
    // cregistration.hpp:605-607
    using CRegistration_reference<PointT>::coarse_reg_ransac;
    int coarse_reg_ransac(const typename pcl::PointCloud<PointT>::Ptr &target_pts, const typename pcl::PointCloud<PointT>::Ptr &source_pts,
                          Eigen::Matrix4d &tran_mat, float noise_bound = 0.2, int min_inlier_num = 8, int max_iter_num = 20000) {
        return b200::coarse_reg_ransac<PointT>(target_pts, source_pts, tran_mat, noise_bound, min_inlier_num, max_iter_num);
    }
    // cregistration.hpp:664-666 (the reference declares one overload)
    int coarse_reg_teaser(const typename pcl::PointCloud<PointT>::Ptr &target_pts, const typename pcl::PointCloud<PointT>::Ptr &source_pts,
                          Eigen::Matrix4d &tran_mat, float noise_bound = 0.2, int min_inlier_num = 8) {
        return b200::coarse_reg_teaser<PointT>(target_pts, source_pts, tran_mat, noise_bound, min_inlier_num);
    }
    // cregistration.hpp:945-947. The device runs the DIRECT7 neighbourhood; KDTREE (use_direct_search = false) is the
    // reference member. A template on the guess type, so that the class compiles against a reference build that does
    // not declare omp_ndt as long as nobody calls the KDTREE form.
    template <typename Matrix4 = Eigen::Matrix4d>
    int omp_ndt(constraint_t &registration_cons, float ndt_resolution = 1.0, bool use_direct_search = true,
                Matrix4 initial_guess = Matrix4::Identity(), bool apply_intersection_filter = true, float fitness_score_thre = 10.0) {
        if (!use_direct_search)
            return CRegistration_reference<PointT>::omp_ndt(registration_cons, ndt_resolution, use_direct_search, initial_guess,
                                                            apply_intersection_filter, fitness_score_thre);
        return b200::omp_ndt<PointT>(registration_cons, ndt_resolution, initial_guess, apply_intersection_filter, fitness_score_thre);
    }
    // cregistration.hpp:1024-1027. The device runs the voxelized GICP (FastVGICP), where max_iter_num and dis_thre_unit
    // have no effect; using_voxel_gicp = false (PCL-style GICP) and the calls the library refuses (fewer than 20
    // points in a cloud) are the reference member. A template on the guess type, as omp_ndt.
    template <typename Matrix4 = Eigen::Matrix4d>
    int omp_gicp(constraint_t &registration_cons, int max_iter_num = 20, float dis_thre_unit = 1.5, bool using_voxel_gicp = true,
                 float voxel_size = 1.0, Matrix4 initial_guess = Matrix4::Identity(), bool apply_intersection_filter = false,
                 float fitness_score_thre = 10.0) {
        bool unsupported = !using_voxel_gicp;
        int code = -3;
        if (using_voxel_gicp)
            code = b200::omp_gicp<PointT>(registration_cons, voxel_size, initial_guess, apply_intersection_filter, fitness_score_thre,
                                          &unsupported);
        if (unsupported)
            return CRegistration_reference<PointT>::omp_gicp(registration_cons, max_iter_num, dis_thre_unit, using_voxel_gicp,
                                                             voxel_size, initial_guess, apply_intersection_filter,
                                                             fitness_score_thre);
        return code;
    }
};

} // namespace lo
#endif
