// test/mulls_reg.cpp:145-149 and the in-place CFilter::non_max_suppress (cfilter.hpp:1183) in its call forms against the
// DROP-IN headers (include/dropin), with the reference's own header and class names and nothing edited. Include path
// order as for dropin_caller.cpp, with the stand-in that declares the reference's three overloads: include/dropin,
// include, tests/stubs/nms_ref, tests/stubs.
//   nms_caller                              the reference's calls on two small stand-in vertex clouds (without a GPU
//                                           they report the missing device and return false)
//   nms_caller in.bin a.bin b.bin radius    48-byte rows in; the rows left by non_max_suppress(cloud, r) and by
//                                           non_max_suppress(cloud, r, false, tree) out (tests/test_gpu_nms.py)
// Both modes also check that non_max_suppress(cloud, r, true, tree) and the overloads of :1243 and :1314 reach the
// reference members.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "cfilter.hpp"

using namespace lo;

typedef pcl::PointCloud<Point_T>::Ptr CloudPtr;

static bool read_rows(const char *path, CloudPtr &c) {
    FILE *f = std::fopen(path, "rb");
    if (!f) return false;
    Point_T p;
    while (std::fread(&p, sizeof(p), 1, f) == 1) c->points.push_back(p);
    std::fclose(f);
    return true;
}
static bool write_rows(const char *path, const CloudPtr &c) {
    FILE *f = std::fopen(path, "wb");
    if (!f) return false;
    const size_t w = c->points.empty() ? 0 : std::fwrite(c->points.data(), sizeof(Point_T), c->points.size(), f);
    std::fclose(f);
    return w == c->points.size();
}

// kd_tree_already_built = true, and the overloads into cloud_out (:1243) and on pca_feature_t (:1314): the reference
// members run, the library is not asked
static int reference_forms(CFilter<Point_T> &cfilter, const CloudPtr &cloud) {
    int failures = 0;
    CloudPtr c(new pcl::PointCloud<Point_T>()), out(new pcl::PointCloud<Point_T>());
    c->points = cloud->points;
    pcl::search::KdTree<Point_T>::Ptr tree(new pcl::search::KdTree<Point_T>());
    cfilter.non_max_suppress(c, 0.25f, true, tree);
    if (cfilter.reference_nms_ran != 1183) ++failures;
    cfilter.non_max_suppress(c, out, 0.25f);
    if (cfilter.reference_nms_ran != 1243) ++failures;
    std::vector<pca_feature_t> features;
    pcl::PointIndicesPtr indices(new pcl::PointIndices());
    cfilter.non_max_suppress(features, indices, 0.25f);
    if (cfilter.reference_nms_ran != 1314) ++failures;
    cfilter.reference_nms_ran = 0;
    return failures;
}

int main(int argc, char **argv) {
    CFilter<Point_T> cfilter;
    int failures = 0;
    if (argc == 5) {
        CloudPtr a(new pcl::PointCloud<Point_T>()), b(new pcl::PointCloud<Point_T>());
        if (!read_rows(argv[1], a)) return 2;
        b->points = a->points;
        const float r = (float)std::atof(argv[4]);
        pcl::search::KdTree<Point_T>::Ptr tree(new pcl::search::KdTree<Point_T>());
        const bool ra = cfilter.non_max_suppress(a, r);
        const bool rb = cfilter.non_max_suppress(b, r, false, tree);
        if (cfilter.reference_body_ran || cfilter.reference_nms_ran) ++failures; // the device forms only
        if (!ra || !rb || !write_rows(argv[2], a) || !write_rows(argv[3], b)) ++failures;
        failures += reference_forms(cfilter, a);
        std::printf("nms drop-in: %zu / %zu rows kept; failures %d\n", a->points.size(), b->points.size(), failures);
        return failures;
    }
    // ---- test/mulls_reg.cpp:145-149 on two stand-in vertex clouds: 6 x 6 x 2 lattices at 0.125 m, scores by index ----
    cloudblock_Ptr cblock_1(new cloudblock_t()), cblock_2(new cloudblock_t());
    for (int b = 0; b < 2; ++b)
        for (int i = 0; i < 72; ++i) {
            Point_T p = {};
            p.x = 0.125f * (i % 6) + b, p.y = 0.125f * ((i / 6) % 6), p.z = 0.125f * (i / 36);
            p.pad1 = (float)(i % 7); // normal[3]: the score
            (b ? cblock_2 : cblock_1)->pc_vertex->points.push_back(p);
        }
    const size_t n1 = cblock_1->pc_vertex->points.size(), n2 = cblock_2->pc_vertex->points.size();
    const float pca_neigh_r = 1.0f;
    const float keypoint_nms_radius = 0.25 * pca_neigh_r;
    const bool global_registration_on = true;
    bool a = false, b = false;
    if (global_registration_on) //refine keypoints
    {
        a = cfilter.non_max_suppress(cblock_1->pc_vertex, keypoint_nms_radius);
        b = cfilter.non_max_suppress(cblock_2->pc_vertex, keypoint_nms_radius);
    }
    if (cfilter.reference_body_ran || cfilter.reference_nms_ran) ++failures, std::printf("FAIL: a reference CFilter body ran\n");
    if (a != b) ++failures;
    if (a && (cblock_1->pc_vertex->points.size() >= n1 || cblock_2->pc_vertex->points.size() >= n2)) ++failures;
    if (!a && (cblock_1->pc_vertex->points.size() != n1 || cblock_2->pc_vertex->points.size() != n2)) ++failures;
    failures += reference_forms(cfilter, cblock_1->pc_vertex);
    std::printf("nms drop-in compiled and linked; ran on a device: %d; %zu -> %zu points; failures %d\n", a ? 1 : 0, n1,
                cblock_1->pc_vertex->points.size(), failures);
    return failures;
}
