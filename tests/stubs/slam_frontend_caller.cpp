// test/mulls_slam.cpp:418-428, the SLAM driver's per-frame feature extraction, against the DROP-IN headers
// (include/dropin), with the reference's own header and class names and nothing edited. The call passes `true` as
// argument 16, use_distance_adaptive_pca, as the driver does at start-up (:363-377) and on every frame; the other
// arguments are the values the driver passes by default. Include path order as for dropin_caller.cpp: include/dropin,
// include, tests/stubs/ref, tests/stubs.
//   slam_frontend_caller [raw.bin]   48-byte rows of one raw scan (none: an empty scan). Prints what the call returned
//                                    and the sizes of the feature clouds it appended.
#include <cstdio>

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

int main(int argc, char **argv) {
    CFilter<Point_T> cfilter;
    cloudblock_Ptr cblock_source(new cloudblock_t());
    if (argc > 1 && !read_rows(argv[1], cblock_source->pc_raw)) return 2;
    int ground_down_rate = 15, nonground_down_rate = 3;
    const bool ok = cfilter.extract_semantic_pts(cblock_source, 0.05f, 3.0f, 0.3f, 1.5f, 5.0f, ground_down_rate, nonground_down_rate,
                                                 1.0f, 50, 0.65f, 0.65f, 0.12f, 0.75f, 0.75f, true, 2, 15.0f, 3, 2.0f, false, false,
                                                 false, 2, 10, 0, 2, 8, 1, FLT_MAX, 0.94f, 0.17f, 0.98f, 0.34f, true, false, 300, 200,
                                                 800, 200, 100, 10000, FLT_MAX, 0.0f, 2.0f, -7.0f, 0.3f, false, false, 0.0f, 0.0f);
    int failures = 0;
    if (cfilter.reference_body_ran) ++failures, std::printf("FAIL: the reference's extract_semantic_pts body ran\n");
    std::printf("slam front end: raw %zu returned %d pillar %zu beam %zu facade %zu roof %zu vertex %zu ground %zu ground_down %zu; "
                "failures %d\n",
                cblock_source->pc_raw->points.size(), ok ? 1 : 0, cblock_source->pc_pillar->points.size(),
                cblock_source->pc_beam->points.size(), cblock_source->pc_facade->points.size(), cblock_source->pc_roof->points.size(),
                cblock_source->pc_vertex->points.size(), cblock_source->pc_ground->points.size(),
                cblock_source->pc_ground_down->points.size(), failures);
    return failures;
}
