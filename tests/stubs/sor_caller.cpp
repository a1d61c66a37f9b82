// test/mulls_slam.cpp:1008-1009 and both CFilter::sor_filter overloads (cfilter.hpp:204, :225) against the DROP-IN
// headers (include/dropin), with the reference's own header and class names and nothing edited. Include path order as
// for dropin_caller.cpp: include/dropin, include, tests/stubs/ref, tests/stubs.
//   sor_caller                                   the reference's call on a small merged map (without a GPU both calls
//                                                report the missing device and return false)
//   sor_caller in.bin out.bin inplace.bin k std  48-byte rows in; the rows of the cloud_out overload and of the in-place
//                                                overload out (tests/test_gpu_sor.py)
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

int main(int argc, char **argv) {
    CFilter<Point_T> cfilter;
    int failures = 0;
    if (argc == 6) {
        CloudPtr in(new pcl::PointCloud<Point_T>()), out(new pcl::PointCloud<Point_T>()), inout(new pcl::PointCloud<Point_T>());
        if (!read_rows(argv[1], in)) return 2;
        inout->points = in->points;
        const int mean_k = std::atoi(argv[4]);
        const double n_std = std::atof(argv[5]);
        const bool a = cfilter.sor_filter(in, out, mean_k, n_std);
        const bool b = cfilter.sor_filter(inout, mean_k, n_std);
        if (cfilter.reference_body_ran) ++failures;
        if (!a || !b || !write_rows(argv[2], out) || !write_rows(argv[3], inout)) ++failures;
        std::printf("sor drop-in: %zu -> %zu / %zu rows; failures %d\n", in->points.size(), out->points.size(),
                    inout->points.size(), failures);
        return failures;
    }
    // ---- test/mulls_slam.cpp:1008-1009 on a stand-in merged map: a 12 x 12 x 4 lattice and two far points ----
    CloudPtr pc_map_merged(new pcl::PointCloud<Point_T>());
    for (int i = 0; i < 12; ++i)
        for (int j = 0; j < 12; ++j)
            for (int k = 0; k < 4; ++k) {
                Point_T p = {};
                p.x = 0.5f * i, p.y = 0.5f * j, p.z = 0.5f * k;
                pc_map_merged->points.push_back(p);
            }
    Point_T far = {};
    far.x = 300.0f;
    pc_map_merged->points.push_back(far);
    far.y = -250.0f;
    pc_map_merged->points.push_back(far);
    const size_t n0 = pc_map_merged->points.size();
    CloudPtr pc_filtered(new pcl::PointCloud<Point_T>());
    const bool a = cfilter.sor_filter(pc_map_merged, pc_filtered, 20, 2.0);
    const bool FLAGS_map_filter_on = true;
    bool b = false;
    if (FLAGS_map_filter_on)                        //TODO: add more map based operation //1.generate 2D geo-referenced image //2.intensity generalization
        b = cfilter.sor_filter(pc_map_merged, 20, 2.0); //sor filtering before output
    if (cfilter.reference_body_ran) ++failures, std::printf("FAIL: a reference CFilter body ran\n");
    if (a != b) ++failures;
    if (a && (pc_filtered->points.size() != n0 - 2 || pc_map_merged->points.size() != n0 - 2)) ++failures;
    if (!a && pc_map_merged->points.size() != n0) ++failures; // a refused call leaves the cloud as it was
    std::printf("sor drop-in compiled and linked; ran on a device: %d; %zu -> %zu points; failures %d\n", a ? 1 : 0, n0,
                pc_map_merged->points.size(), failures);
    return failures;
}
