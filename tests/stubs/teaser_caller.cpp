// test/mulls_reg.cpp:170-186 (--teaser_on=true) and test/mulls_slam.cpp:532-556 (--teaser_based_global_registration_on)
// (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759) against the DROP-IN headers (include/dropin), with the
// reference's own header and class names and nothing edited. Include path order as for dropin_caller.cpp:
// include/dropin, include, tests/stubs/ref, tests/stubs. The stand-in reference class does not declare
// coarse_reg_teaser: the drop-in's member does not need the reference's (nor TEASER_ON).
//   teaser_caller                                      both call sites on a small scene (without a GPU every call
//                                                      reports the missing device, returns -1 and leaves tran_mat alone)
//   teaser_caller tgt.bin src.bin out.bin noise_bound min_inlier_num
//                                                      48-byte rows in; the return value and the 16 entries of tran_mat
//                                                      (row-major, started from a marker matrix) out as doubles
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "cregistration.hpp"

using namespace lo;

typedef pcl::PointCloud<Point_T>::Ptr pcTPtr;

static bool read_rows(const char *path, pcTPtr &c) {
    FILE *f = std::fopen(path, "rb");
    if (!f) return false;
    Point_T p;
    while (std::fread(&p, sizeof(p), 1, f) == 1) c->points.push_back(p);
    std::fclose(f);
    return true;
}

static void marker(Eigen::Matrix4d &m) {
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) m(r, c) = 100.0 + 4 * r + c;
}

int main(int argc, char **argv) {
    CRegistration<Point_T> creg;
    int failures = 0;
    if (argc == 6) {
        pcTPtr t(new pcl::PointCloud<Point_T>()), s(new pcl::PointCloud<Point_T>());
        if (!read_rows(argv[1], t) || !read_rows(argv[2], s)) return 2;
        Eigen::Matrix4d tran_mat;
        marker(tran_mat);
        const int ret = creg.coarse_reg_teaser(t, s, tran_mat, (float)std::atof(argv[4]), std::atoi(argv[5]));
        double out[17];
        out[0] = ret;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) out[1 + 4 * r + c] = tran_mat(r, c);
        FILE *f = std::fopen(argv[3], "wb");
        if (!f || std::fwrite(out, sizeof(double), 17, f) != 17) ++failures;
        if (f) std::fclose(f);
        std::printf("teaser drop-in: returned %d for %zu correspondences; failures %d\n", ret, t->points.size(), failures);
        return failures;
    }
    // ---- a stand-in scene: 60 keypoint pairs, the source shifted by (1, -2, 0.5) from the target, 10 outliers ----
    pcTPtr target_cor(new pcl::PointCloud<Point_T>()), source_cor(new pcl::PointCloud<Point_T>());
    for (int i = 0; i < 60; ++i) {
        Point_T p = {};
        p.x = (float)((i * 37) % 61) - 30.f, p.y = (float)((i * 53) % 59) - 29.f, p.z = 0.5f * (float)((i * 17) % 13);
        Point_T q = p;
        q.x -= 1.f, q.y += 2.f, q.z -= 0.5f;
        q.x += 0.01f * (float)((i * 7) % 5 - 2), q.y += 0.01f * (float)((i * 3) % 5 - 2);
        q.z += 0.01f * (float)((i * 11) % 5 - 2);
        if (i % 6 == 5) q.z += 20.f + i; // outliers
        target_cor->points.push_back(p);
        source_cor->points.push_back(q);
    }
    // test/mulls_reg.cpp:176-177 (--teaser_on=true; the run script's keypoint_nms_radius 0.25)
    Eigen::Matrix4d init_mat;
    marker(init_mat);
    const float keypoint_nms_radius = 0.25f;
    const bool teaser_on = true;
    int a = -2;
    if (teaser_on)
        a = creg.coarse_reg_teaser(target_cor, source_cor, init_mat, 4.0 * keypoint_nms_radius);
    // test/mulls_slam.cpp:541-543: the noise bound is pca_neigh_r, the minimum from the flags; the odometry guess is kept on -1
    Eigen::Matrix4d tran_mat = Eigen::Matrix4d::Identity();
    const float pca_neigh_r = 0.6f;
    const int FLAGS_global_reg_min_inlier_count = 8;
    const int b = creg.coarse_reg_teaser(target_cor, source_cor, tran_mat, pca_neigh_r, FLAGS_global_reg_min_inlier_count);
    // too few correspondences: -1, tran_mat untouched
    pcTPtr few_t(new pcl::PointCloud<Point_T>()), few_s(new pcl::PointCloud<Point_T>());
    few_t->points.assign(target_cor->points.begin(), target_cor->points.begin() + 3);
    few_s->points.assign(source_cor->points.begin(), source_cor->points.begin() + 3);
    Eigen::Matrix4d untouched;
    marker(untouched);
    const int c = creg.coarse_reg_teaser(few_t, few_s, untouched);
    if (!creg.coarse_reg_ransac(7)) ++failures; // an inherited member of the stand-in, still visible
    if (a != b || c != -1) ++failures;
    if (untouched(0, 0) != 100.0 || untouched(3, 3) != 115.0) ++failures;
    if (a == 1) { // the shift back: x + 1, y - 2, z + 0.5
        if (std::fabs(init_mat(0, 3) - 1.0) > 0.05 || std::fabs(init_mat(1, 3) + 2.0) > 0.05 || std::fabs(init_mat(2, 3) - 0.5) > 0.05 ||
            std::fabs(tran_mat(0, 3) - 1.0) > 0.05 || init_mat(3, 3) != 1.0)
            ++failures;
    } else if (a != -1 || init_mat(0, 0) != 100.0 || tran_mat(0, 0) != 1.0) {
        ++failures; // a failed call leaves tran_mat as it was
    }
    std::printf("teaser drop-in compiled and linked; ran on a device: %d; failures %d\n", a == 1 ? 1 : 0, failures);
    return failures;
}
