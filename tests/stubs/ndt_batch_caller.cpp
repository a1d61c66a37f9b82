// lo::b200::omp_ndt_batch (include/common/cregistration_b200.hpp) with the argument order and defaults of the reference's
// omp_ndt, over a std::vector<constraint_t>, with stand-in PCL/Eigen types (tests/stubs/utility.hpp).
//   ndt_batch_caller                                   a stand-in scene registered scan to scan and scan to map in one
//                                                      batch (without a GPU: every code -3, every Trans1_2 untouched)
//   ndt_batch_caller out.bin res t0 s0 [t1 s1 ...]     48-byte rows in (block1 / block2 ->pc_down, local_bound their
//                                                      bboxes), one pair per (t, s); per pair the code and Trans1_2
//                                                      (row-major) out as 17 doubles
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "utility.hpp"
#include "common/cregistration_b200.hpp"

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
static void bbox(const pcTPtr &c, bounds_t &b) { // CloudUtility::get_cloud_bbx
    b.min_x = b.min_y = b.min_z = 1e300;
    b.max_x = b.max_y = b.max_z = -1e300;
    for (const Point_T &p : c->points) {
        if (p.x < b.min_x) b.min_x = p.x;
        if (p.y < b.min_y) b.min_y = p.y;
        if (p.z < b.min_z) b.min_z = p.z;
        if (p.x > b.max_x) b.max_x = p.x;
        if (p.y > b.max_y) b.max_y = p.y;
        if (p.z > b.max_z) b.max_z = p.z;
    }
}

int main(int argc, char **argv) {
    int failures = 0;
    if (argc >= 5 && argc % 2 == 1) {
        std::vector<constraint_t> cons((argc - 3) / 2);
        for (size_t i = 0; i < cons.size(); ++i) {
            if (!read_rows(argv[3 + 2 * i], cons[i].block1->pc_down) || !read_rows(argv[4 + 2 * i], cons[i].block2->pc_down)) return 2;
            bbox(cons[i].block1->pc_down, cons[i].block1->local_bound);
            bbox(cons[i].block2->pc_down, cons[i].block2->local_bound);
        }
        const std::vector<int> codes = lo::b200::omp_ndt_batch<Point_T>(cons, (float)std::atof(argv[2]));
        FILE *f = std::fopen(argv[1], "wb");
        for (size_t i = 0; i < cons.size() && f; ++i) {
            double out[17];
            out[0] = codes[i];
            for (int r = 0; r < 4; ++r)
                for (int c = 0; c < 4; ++c) out[1 + 4 * r + c] = cons[i].Trans1_2(r, c);
            if (std::fwrite(out, sizeof(double), 17, f) != 17) ++failures;
        }
        if (!f) ++failures;
        else std::fclose(f);
        std::printf("ndt batch shim: %zu pairs; failures %d\n", cons.size(), failures);
        return failures;
    }
    // a stand-in scene: a noisy ground grid with two walls; the source is the target shifted by (0.2, -0.1, 0)
    cloudblock_Ptr cblock_target(new cloudblock_t), cblock_source(new cloudblock_t), cblock_local_map(new cloudblock_t);
    for (int i = 0; i < 4000; ++i) {
        Point_T p = {};
        const float u = (float)((i * 37) % 400) * 0.1f - 20.f, v = (float)((i * 53) % 397) * 0.1f - 20.f;
        const float e = 0.01f * (float)((i * 7) % 11 - 5);
        if (i % 3 == 0) p.x = u, p.y = v, p.z = e;
        else if (i % 3 == 1) p.x = 20.f + e, p.y = u, p.z = (float)(i % 60) * 0.1f;
        else p.x = u, p.y = 20.f + e, p.z = (float)(i % 60) * 0.1f;
        cblock_target->pc_down->points.push_back(p);
        cblock_local_map->pc_down->points.push_back(p);
        p.x -= 0.2f, p.y += 0.1f;
        cblock_source->pc_down->points.push_back(p);
    }
    bbox(cblock_target->pc_down, cblock_target->local_bound);
    bbox(cblock_local_map->pc_down, cblock_local_map->local_bound);
    bbox(cblock_source->pc_down, cblock_source->local_bound);
    std::vector<constraint_t> cons(2);
    cons[0].block1 = cblock_target, cons[0].block2 = cblock_source;    // scan to scan
    cons[1].block1 = cblock_local_map, cons[1].block2 = cblock_source; // scan to map
    const float FLAGS_reg_voxel_size = 1.0f;
    const bool FLAGS_ndt_searching_method = true, FLAGS_reg_intersection_filter_on = true;
    Eigen::Matrix4d initial_guess_tran = Eigen::Matrix4d::Identity();
    const std::vector<int> codes = lo::b200::omp_ndt_batch<Point_T>(cons, FLAGS_reg_voxel_size, FLAGS_ndt_searching_method,
                                                                     initial_guess_tran, FLAGS_reg_intersection_filter_on);
    const std::vector<int> codes2 = lo::b200::omp_ndt_batch<Point_T>(cons); // defaults only
    int ran = 0;
    if (codes.size() != 2 || codes2.size() != 2) ++failures;
    else if (codes[0] == 1 && codes[1] == 1 && codes2 == codes) { // on a device: the shift recovered to within the walk's last step
        ran = 1;
        for (const constraint_t &c : cons)
            if (std::abs(c.Trans1_2(0, 3) - 0.2) > 0.1 || std::abs(c.Trans1_2(1, 3) + 0.1) > 0.1) ++failures;
    } else if (codes[0] != -3 || codes[1] != -3 || cons[0].Trans1_2(0, 3) != 0.0 || cons[1].Trans1_2(0, 3) != 0.0) {
        ++failures; // no device: -3, Trans1_2 untouched
    }
    std::printf("ndt batch shim compiled and linked; ran on a device: %d; failures %d\n", ran, failures);
    return failures;
}
