// test/mulls_reg.cpp:173-174 and test/mulls_slam.cpp:534-535 (CRegistration::find_feature_correspondence_ncc,
// cregistration.hpp:409-601) against the DROP-IN headers (include/dropin), with the reference's own header and class
// names and nothing edited. Include path order as for dropin_caller.cpp: include/dropin, include, tests/stubs/ref,
// tests/stubs. The stand-in reference class (tests/stubs/ref/cregistration.hpp) has no find_feature_correspondence_ncc, so
// this file compiles only because the drop-in lo::CRegistration defines the member: every call below is the device path.
//   ncc_caller                                         both call sites on small keypoint clouds (without a GPU every call
//                                                      reports the missing device and returns false)
//   ncc_caller tgt.bin src.bin tcor.bin scor.bin fixed corr_num reciprocal
//                                                      48-byte rows in; the rows appended to target_cor / source_cor out
//                                                      (tests/test_gpu_ncc.py)
#include <cstdio>
#include <cstdlib>
#include <string>

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
static bool write_rows(const char *path, const pcTPtr &c) {
    FILE *f = std::fopen(path, "wb");
    if (!f) return false;
    const size_t w = c->points.empty() ? 0 : std::fwrite(c->points.data(), sizeof(Point_T), c->points.size(), f);
    std::fclose(f);
    return w == c->points.size();
}

int main(int argc, char **argv) {
    CRegistration<Point_T> creg;
    int failures = 0;
    if (argc == 8) {
        pcTPtr tk(new pcl::PointCloud<Point_T>()), sk(new pcl::PointCloud<Point_T>());
        pcTPtr target_cor(new pcl::PointCloud<Point_T>()), source_cor(new pcl::PointCloud<Point_T>());
        if (!read_rows(argv[1], tk) || !read_rows(argv[2], sk)) return 2;
        const bool fixed = std::atoi(argv[5]) != 0, reciprocal = std::atoi(argv[7]) != 0;
        const int corr_num = std::atoi(argv[6]);
        const bool ok = creg.find_feature_correspondence_ncc(tk, sk, target_cor, source_cor, fixed, corr_num, reciprocal);
        if (!write_rows(argv[3], target_cor) || !write_rows(argv[4], source_cor)) ++failures;
        std::printf("ncc drop-in: returned %d, %zu x %zu keypoints -> %zu pairs; failures %d\n", ok ? 1 : 0, tk->points.size(),
                    sk->points.size(), target_cor->points.size(), failures);
        return failures;
    }
    // ---- stand-in vertex clouds of two blocks: encoded neighbourhood categories, curvature, height, intensity ----
    cloudblock_Ptr block1(new cloudblock_t), block2(new cloudblock_t);
    for (int i = 0; i < 40; ++i) {
        Point_T p = {};
        p.x = 0.5f * i;
        p.normal_x = (float)((i % 7) * 1000000 + (i % 5) * 10000 + (i % 3) * 100 + i % 11);
        p.normal_y = (float)((i % 4) * 1000000 + (i % 9) * 100);
        p.pad1 = 0.01f * (i % 13); // normal[3]: curvature
        p.pad0 = 0.1f * (i % 6);   // data[3]: height above ground
        p.intensity = (float)(i * 3 % 40);
        block1->pc_vertex->points.push_back(p);
        p.x += 0.25f;
        p.intensity = (float)((i * 7 + 3) % 40);
        block2->pc_vertex->points.push_back(p);
    }
    constraint_t reg_con;
    reg_con.block1 = block1, reg_con.block2 = block2;
    // test/mulls_reg.cpp:170-174 (the run script's flags: fixed_num_corr_on false, reciprocal_corr_on false)
    const bool FLAGS_fixed_num_corr_on = false, FLAGS_reciprocal_corr_on = false;
    const int feature_correspondence_num = 1000;
    pcTPtr target_cor(new pcl::PointCloud<Point_T>()), source_cor(new pcl::PointCloud<Point_T>());
    const bool a = creg.find_feature_correspondence_ncc(reg_con.block1->pc_vertex, reg_con.block2->pc_vertex, target_cor, source_cor,
                                                        FLAGS_fixed_num_corr_on, feature_correspondence_num, FLAGS_reciprocal_corr_on);
    // test/mulls_slam.cpp:531-535 (best_n_feature_match_on true, feature_corr_num 1000, reciprocal_feature_match_on true)
    std::vector<constraint_t> current_registration_edges(1, reg_con);
    const bool FLAGS_best_n_feature_match_on = true, FLAGS_reciprocal_feature_match_on = true;
    const int FLAGS_feature_corr_num = 1000;
    const size_t j = 0;
    pcTPtr target_cor2(new pcl::PointCloud<Point_T>()), source_cor2(new pcl::PointCloud<Point_T>());
    const bool b = creg.find_feature_correspondence_ncc(current_registration_edges[j].block1->pc_vertex, current_registration_edges[j].block2->pc_vertex,
                                                        target_cor2, source_cor2, FLAGS_best_n_feature_match_on, FLAGS_feature_corr_num, FLAGS_reciprocal_feature_match_on);
    // too few keypoints: false, nothing appended
    pcTPtr few(new pcl::PointCloud<Point_T>());
    few->points.assign(block1->pc_vertex->points.begin(), block1->pc_vertex->points.begin() + 9);
    const bool c = creg.find_feature_correspondence_ncc(few, block2->pc_vertex, target_cor2, source_cor2);
    if (a != b || c) ++failures;
    if (target_cor->points.size() != source_cor->points.size() || target_cor2->points.size() != source_cor2->points.size()) ++failures;
    if (a && (target_cor->points.empty() || target_cor->points.size() > 40 || target_cor2->points.empty())) ++failures;
    if (!a && (!target_cor->points.empty() || !target_cor2->points.empty())) ++failures; // a failed call leaves them as they were
    std::printf("ncc drop-in compiled and linked; ran on a device: %d; %zu and %zu pairs; failures %d\n", a ? 1 : 0,
                target_cor->points.size(), target_cor2->points.size(), failures);
    return failures;
}
