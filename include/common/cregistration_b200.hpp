// Drop-in shim: lo::CRegistration<PointT>::mm_lls_icp over the mulls_b200 C-ABI.
//
// A MULLS maintainer keeps include/common/cregistration.hpp as it is and replaces the BODY of
// mm_lls_icp (cregistration.hpp:1125-1440) by
//
//     return lo::b200::mm_lls_icp<PointT>(registration_cons, max_iter_num, dis_thre_unit, ... );
//
// (all 23 arguments forwarded unchanged) or calls lo::b200::mm_lls_icp directly. The signature below
// is the reference's (cregistration.hpp:1114-1123): same names, order, types and defaults, so
// test/mulls_reg.cpp:194-195 and test/mulls_slam.cpp:477-482, :560-566, :642-648, :679-685 compile
// unchanged. Needs PCL + Eigen (for the types only) and -lmulls_b200.
//
// Contract differences (see INTEGRATION.md): block1->tree_* are not populated; options
// keep_less_source_points uses a reproducible uniform sample instead of the reference's time-seeded pcl::RandomSample.
#ifndef MULLS_B200_CREGISTRATION_SHIM_HPP
#define MULLS_B200_CREGISTRATION_SHIM_HPP

#include <cfloat>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "mulls_b200/abi.h"
#include "utility.hpp" // lo::constraint_t, lo::cloudblock_t, Matrix6d, Point_T

namespace lo {
namespace b200 {

// Contexts are kept per host thread (mm_lls_icp is called from the app's main thread, SURVEY 8b "Threading"), grown
// when a call needs more room, and destroyed when the thread ends.
struct ThreadContext {
    mulls_ctx *ctx = nullptr;
    size_t cap_pairs = 0, cap_src = 0, cap_tgt = 0;
    ~ThreadContext() {
        if (ctx) mulls_destroy(ctx);
    }
    mulls_ctx *get(size_t pairs, size_t need_src, size_t need_tgt) {
        if (!ctx || pairs > cap_pairs || need_src > cap_src || need_tgt > cap_tgt) {
            if (ctx) mulls_destroy(ctx);
            cap_pairs = pairs > cap_pairs ? pairs : cap_pairs;
            cap_src = need_src > cap_src ? need_src * 2 : cap_src;
            cap_tgt = need_tgt > cap_tgt ? need_tgt * 2 : cap_tgt;
            ctx = mulls_create(/*device*/ 0, cap_pairs ? cap_pairs : 1, cap_src ? cap_src : 1, cap_tgt ? cap_tgt : 1);
        }
        return ctx;
    }
};
inline mulls_ctx *thread_context(size_t need_src, size_t need_tgt) {
    static thread_local ThreadContext tc;
    return tc.get(1, need_src, need_tgt);
}
inline mulls_ctx *thread_batch_context(size_t pairs, size_t need_src, size_t need_tgt) {
    static thread_local ThreadContext tc;
    return tc.get(pairs, need_src, need_tgt);
}

template <typename PointT>
inline mulls_cloud_view view_of(const typename pcl::PointCloud<PointT>::Ptr &cloud) {
    static_assert(sizeof(PointT) == 48, "the C-ABI consumes pcl::PointXYZINormal rows (48 bytes)");
    mulls_cloud_view v;
    v.aos48 = cloud->points.empty() ? nullptr : reinterpret_cast<const float *>(cloud->points.data());
    v.n = cloud->points.size();
    return v;
}

template <typename PointT>
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
    cloudblock_t &b1 = *registration_cons.block1; // target
    cloudblock_t &b2 = *registration_cons.block2; // source
    // clone_feature(..., false) for the target, clone_feature(..., !use_more_points) for the source
    // (cregistration.hpp:1180-1181, utility.hpp:524-550): the library copies, the caller's clouds stay intact.
    mulls_cloud_view tgt[MULLS_NUM_CLASSES] = {view_of<PointT>(b1.pc_ground), view_of<PointT>(b1.pc_pillar),
                                               view_of<PointT>(b1.pc_facade), view_of<PointT>(b1.pc_beam),
                                               view_of<PointT>(b1.pc_roof),   view_of<PointT>(b1.pc_vertex)};
    // the undistortion variant reads block2->pc_*_down whatever use_more_points says (cregistration.hpp:1251-1253)
    const bool down = !use_more_points || apply_motion_undistortion_while_registration;
    mulls_cloud_view src[MULLS_NUM_CLASSES] = {
        view_of<PointT>(down ? b2.pc_ground_down : b2.pc_ground), view_of<PointT>(down ? b2.pc_pillar_down : b2.pc_pillar),
        view_of<PointT>(down ? b2.pc_facade_down : b2.pc_facade), view_of<PointT>(down ? b2.pc_beam_down : b2.pc_beam),
        view_of<PointT>(down ? b2.pc_roof_down : b2.pc_roof),     view_of<PointT>(b2.pc_vertex)};

    mulls_icp_params p;
    mulls_icp_default_params(&p);
    p.max_iter_num = max_iter_num;
    p.dis_thre_unit = dis_thre_unit;
    p.converge_translation = converge_translation;
    p.converge_rotation_d = converge_rotation_d;
    p.dis_thre_min = dis_thre_min;
    p.dis_thre_update_rate = dis_thre_update_rate;
    std::strncpy(p.used_feature_type, used_feature_type.c_str(), 7);
    std::strncpy(p.weight_strategy, weight_strategy.c_str(), 7);
    p.z_xy_balanced_ratio = z_xy_balanced_ratio;
    p.pt2pt_residual_window = pt2pt_residual_window;
    p.pt2pl_residual_window = pt2pl_residual_window;
    p.pt2li_residual_window = pt2li_residual_window;
    p.apply_intersection_filter = apply_intersection_filter;
    p.apply_motion_undistortion_while_registration = apply_motion_undistortion_while_registration;
    p.normal_shooting_on = normal_shooting_on;
    p.normal_bearing = normal_bearing;
    p.use_more_points = use_more_points;
    p.keep_less_source_points = keep_less_source_points;
    p.sigma_thre = sigma_thre;
    p.min_neccessary_corr_ratio = min_neccessary_corr_ratio;
    p.max_bearable_rotation_d = max_bearable_rotation_d;
    const bounds_t &lb = b1.local_bound; // read at cregistration.hpp:2916
    p.target_bound[0] = lb.min_x, p.target_bound[1] = lb.min_y, p.target_bound[2] = lb.min_z;
    p.target_bound[3] = lb.max_x, p.target_bound[4] = lb.max_y, p.target_bound[5] = lb.max_z;

    double init[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) init[4 * r + c] = initial_guess(r, c);

    size_t ns = 0, nt = 0;
    for (int c = 0; c < MULLS_NUM_CLASSES; ++c) ns += src[c].n, nt += tgt[c].n;
    mulls_ctx *ctx = thread_context(ns, nt);
    mulls_icp_result out;
    if (!ctx || mulls_icp_run(ctx, tgt, src, &p, init, &out, nullptr) != MULLS_OK) {
        // An infrastructure failure (no device, capacity, CUDA error) must look like a FAILED registration to the
        // callers, which only test `< 0` and then read Trans1_2 (test/mulls_slam.cpp:650, :686): leave what the
        // reference leaves when no iteration ran — the initial guess, an identity information matrix — with a
        // sigma no acceptance test passes, and return a negative code of our own (-4: device path failed).
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        registration_cons.Trans1_2 = initial_guess;
        registration_cons.information_matrix.setIdentity();
        registration_cons.sigma = FLT_MAX;
        registration_cons.confidence = 0.0f;
        return -4;
    }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) registration_cons.Trans1_2(r, c) = out.T[4 * r + c];     // :1405
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) registration_cons.information_matrix(r, c) = out.info[6 * r + c]; // :1418
    registration_cons.sigma = out.sigma;           // :1419
    registration_cons.confidence = out.confidence; // :1420
    return out.code;                               // :1439
}

// lo::CRegistration<PointT>::mm_lls_icp_4dof_global (cregistration.hpp:1584-1681), same signature. The reference
// tries the headings one after the other; the trials are independent registrations of the same clouds, so here
// they are ONE mulls_icp_run_batch call.
template <typename PointT>
bool mm_lls_icp_4dof_global(constraint_t &registration_con, float heading_step_d, int max_iter_num = 20,
                            float dis_thre_unit = 1.5, float converge_translation = 0.005,
                            float converge_rotation_d = 0.05, float dis_thre_min = 0.5,
                            float dis_thre_update_rate = 1.05, float max_bearable_rotation_d = 15.0) {
    (void)converge_rotation_d, (void)max_bearable_rotation_d; // not forwarded by the reference either (:1636-1638)
    cloudblock_t &b1 = *registration_con.block1;
    cloudblock_t &b2 = *registration_con.block2;
    std::vector<double> guesses;
    std::vector<float> headings;
    for (float heading_d = 0.0f; heading_d < 360.0; heading_d += heading_step_d) { // float accumulation as :1604, :1654
        const float heading_rad = heading_d * M_PI / 180.0;
        const double c = cos(heading_rad), s = sin(heading_rad);
        const double sx = b2.local_station.x, sy = b2.local_station.y, sz = b2.local_station.z;
        // tran_mat_s2g * rot_z * tran_mat_g2s (:1621-1630), written out
        const double R[16] = {c, s, 0, sx - c * sx - s * sy, -s, c, 0, sy + s * sx - c * sy, 0, 0, 1, sz - sz, 0, 0, 0, 1};
        guesses.insert(guesses.end(), R, R + 16);
        headings.push_back(heading_d);
    }
    const size_t n = headings.size();
    mulls_cloud_view tgt1[MULLS_NUM_CLASSES] = {view_of<PointT>(b1.pc_ground), view_of<PointT>(b1.pc_pillar),
                                                view_of<PointT>(b1.pc_facade), view_of<PointT>(b1.pc_beam),
                                                view_of<PointT>(b1.pc_roof),   view_of<PointT>(b1.pc_vertex)};
    mulls_cloud_view src1[MULLS_NUM_CLASSES] = {view_of<PointT>(b2.pc_ground_down), view_of<PointT>(b2.pc_pillar_down),
                                                view_of<PointT>(b2.pc_facade_down), view_of<PointT>(b2.pc_beam_down),
                                                view_of<PointT>(b2.pc_roof_down),   view_of<PointT>(b2.pc_vertex)};
    mulls_icp_params p;
    mulls_icp_default_params(&p);
    p.max_iter_num = max_iter_num;
    p.dis_thre_unit = dis_thre_unit;
    p.converge_translation = converge_translation;
    p.converge_rotation_d = converge_translation; // sic, :1636-1637
    p.dis_thre_min = dis_thre_min;
    p.dis_thre_update_rate = dis_thre_update_rate;
    std::strncpy(p.used_feature_type, "111110", 7);
    std::strncpy(p.weight_strategy, "1001", 7);
    const bounds_t &lb = b1.local_bound;
    p.target_bound[0] = lb.min_x, p.target_bound[1] = lb.min_y, p.target_bound[2] = lb.min_z;
    p.target_bound[3] = lb.max_x, p.target_bound[4] = lb.max_y, p.target_bound[5] = lb.max_z;
    std::vector<mulls_cloud_view> tgt(n * MULLS_NUM_CLASSES), src(n * MULLS_NUM_CLASSES);
    std::vector<mulls_icp_params> params(n, p);
    for (size_t i = 0; i < n; ++i)
        for (int c = 0; c < MULLS_NUM_CLASSES; ++c) tgt[i * MULLS_NUM_CLASSES + c] = tgt1[c], src[i * MULLS_NUM_CLASSES + c] = src1[c];
    size_t ns = 0, nt = 0;
    for (int c = 0; c < MULLS_NUM_CLASSES; ++c) ns += src1[c].n, nt += tgt1[c].n;
    mulls_ctx *ctx = thread_batch_context(n, ns, nt); // kept per thread: a heading search per frame re-uses it
    std::vector<mulls_icp_result> out(n);
    const bool ran = ctx && mulls_icp_run_batch(ctx, n, tgt.data(), src.data(), params.data(), guesses.data(), out.data(), nullptr) == MULLS_OK;
    if (!ran) LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
    if (!ran) return false;
    float current_best_score = 0;
    bool successful_reg = false;
    for (size_t i = 0; i < n; ++i) {
        if (out[i].code > 0) {
            const float cur_score = out[i].confidence / out[i].sigma;
            if (cur_score > current_best_score) {
                for (int r = 0; r < 4; ++r)
                    for (int c = 0; c < 4; ++c) registration_con.Trans1_2(r, c) = out[i].T[4 * r + c];
                for (int r = 0; r < 6; ++r)
                    for (int c = 0; c < 6; ++c) registration_con.information_matrix(r, c) = out[i].info[6 * r + c];
                registration_con.sigma = out[i].sigma;
                registration_con.confidence = out[i].confidence;
                current_best_score = cur_score;
            }
            successful_reg = true;
        }
    }
    return successful_reg;
}

// lo::CRegistration<PointT>::find_feature_correspondence_ncc (cregistration.hpp:409-601), same arguments and defaults
// (test/mulls_reg.cpp:173-174, test/mulls_slam.cpp:534-535): the keypoint matching runs on the device
// (mulls_ncc_correspondences, readings in abi.h); the matched rows are appended to the output clouds here, as the
// reference appends them. Returns false where the reference does (fewer than 10 keypoints in a cloud). A library error
// is logged and also returns false, with both output clouds left as they were.
template <typename PointT>
bool find_feature_correspondence_ncc(const typename pcl::PointCloud<PointT>::Ptr &target_kpts,
                                     const typename pcl::PointCloud<PointT>::Ptr &source_kpts,
                                     typename pcl::PointCloud<PointT>::Ptr &target_corrs,
                                     typename pcl::PointCloud<PointT>::Ptr &source_corrs, bool fixed_num_corr = false,
                                     int corr_num = 2000, bool reciprocal_on = true) {
    const size_t nt = target_kpts->points.size(), ns = source_kpts->points.size();
    const size_t cap = fixed_num_corr ? 7 * (nt < ns ? nt : ns) : nt; // at most 7 pairs per keypoint / one per target row
    std::vector<int32_t> ti(cap ? cap : 1), si(cap ? cap : 1);
    size_t n = 0;
    int performed = 0;
    mulls_ctx *ctx = thread_context(0, nt > ns ? nt : ns);
    if (!ctx || mulls_ncc_correspondences(ctx, view_of<PointT>(target_kpts), view_of<PointT>(source_kpts), fixed_num_corr ? 1 : 0,
                                          corr_num, reciprocal_on ? 1 : 0, ti.data(), si.data(), cap, &n, &performed) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return false;
    }
    if (!performed) {
        LOG(WARNING) << "Too few key points\n"; // :423
        return false;
    }
    for (size_t k = 0; k < n; ++k) {
        target_corrs->points.push_back(target_kpts->points[ti[k]]);
        source_corrs->points.push_back(source_kpts->points[si[k]]);
    }
    return true;
}

// lo::CRegistration<PointT>::coarse_reg_ransac (cregistration.hpp:604-661), same arguments and defaults
// (test/mulls_reg.cpp:170-195, test/mulls_slam.cpp:532-560): the RANSAC rejector over the correspondences i <-> i runs on
// the device (mulls_coarse_reg_ransac, readings in abi.h). Returns 1 (reliable), 0 (need check) or -1 (failed) as the
// reference does, with tran_mat written only on 1 or 0. A library error is logged and returns -1 with tran_mat left as
// it was, so the callers fall back to their odometry guess.
template <typename PointT>
int coarse_reg_ransac(const typename pcl::PointCloud<PointT>::Ptr &target_pts, const typename pcl::PointCloud<PointT>::Ptr &source_pts,
                      Eigen::Matrix4d &tran_mat, float noise_bound = 0.2, int min_inlier_num = 8, int max_iter_num = 20000) {
    const size_t n = target_pts->points.size();
    double T[16];
    int status = -1, n_inliers = 0, n_hypotheses = 0;
    mulls_ctx *ctx = thread_context(0, n);
    if (!ctx || mulls_coarse_reg_ransac(ctx, view_of<PointT>(target_pts), view_of<PointT>(source_pts), noise_bound, min_inlier_num,
                                        max_iter_num, T, &status, &n_inliers, &n_hypotheses) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return -1;
    }
    LOG(INFO) << "[" << n_inliers << "] inlier correspondences found."; // :640
    if (status < 0) {
        LOG(WARNING) << "RANSAC failed"; // :658
        return -1;
    }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) tran_mat(r, c) = T[4 * r + c];
    return status;
}

// lo::CRegistration<PointT>::omp_ndt (cregistration.hpp:945-1021) with use_direct_search (DIRECT7), same arguments and
// defaults (test/mulls_slam.cpp:634-636, :671-673): target = block1->pc_down, source = block2->pc_down, their
// local_bounds, on the device (mulls_omp_ndt, readings in abi.h). Returns 1, or -3 when the fitness exceeds
// fitness_score_thre, and writes Trans1_2, as the reference does. A library error is logged and returns -3 with Trans1_2
// left as it was.
template <typename PointT>
int omp_ndt(constraint_t &registration_cons, float ndt_resolution = 1.0, Eigen::Matrix4d initial_guess = Eigen::Matrix4d::Identity(),
            bool apply_intersection_filter = true, float fitness_score_thre = 10.0) {
    const typename pcl::PointCloud<PointT>::Ptr &t = registration_cons.block1->pc_down, &s = registration_cons.block2->pc_down;
    double guess[16], tb[6], sb[6];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) guess[4 * r + c] = initial_guess(r, c);
    const bounds_t &b1 = registration_cons.block1->local_bound, &b2 = registration_cons.block2->local_bound;
    const double tb_[6] = {b1.min_x, b1.min_y, b1.min_z, b1.max_x, b1.max_y, b1.max_z};
    const double sb_[6] = {b2.min_x, b2.min_y, b2.min_z, b2.max_x, b2.max_y, b2.max_z};
    std::memcpy(tb, tb_, sizeof(tb));
    std::memcpy(sb, sb_, sizeof(sb));
    mulls_ndt_result res;
    mulls_ctx *ctx = thread_context(s->points.size(), t->points.size());
    if (!ctx || mulls_omp_ndt(ctx, view_of<PointT>(t), view_of<PointT>(s), ndt_resolution, 1, guess, apply_intersection_filter ? 1 : 0,
                              fitness_score_thre, tb, sb, &res, nullptr, 0) != MULLS_OK) {
        LOG(ERROR) << "mulls_b200: " << mulls_last_error(ctx);
        return -3;
    }
    LOG(INFO) << "fitness score: " << res.fitness; // base_align, :779
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) registration_cons.Trans1_2(r, c) = res.trans[4 * r + c];
    return res.code;
}

} // namespace b200
} // namespace lo
#endif
