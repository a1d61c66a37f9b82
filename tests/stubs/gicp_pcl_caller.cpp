// test/mulls_slam.cpp:637-639 and :674-676 (CRegistration::omp_gicp, cregistration.hpp:1024-1098) with
// --voxel_gicp_on=false, through lo::b200::omp_gicp_pcl (include/common/cregistration_b200.hpp) with the reference's
// arguments (but using_voxel_gicp and voxel_size), with stand-in PCL/Eigen types (tests/stubs/utility.hpp).
//   gicp_pcl_caller                                   both call sites on a stand-in scene (without a GPU: -3 and
//                                                     Trans1_2 untouched), then a 19-point source, which the library
//                                                     refuses (*unsupported set)
//   gicp_pcl_caller tgt.bin src.bin out.bin max_iter  48-byte rows in (block1 / block2 ->pc_down, local_bound their
//                                                     bboxes), the filter on as at the call sites; the return value
//                                                     and Trans1_2 (row-major) out as 17 doubles
#include <cmath>
#include <cstdio>
#include <cstdlib>

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
    const bool FLAGS_reg_intersection_filter_on = true;
    const float FLAGS_reg_dis_thre_unit = 1.0f;
    Eigen::Matrix4d initial_guess_tran = Eigen::Matrix4d::Identity();
    if (argc == 5) {
        constraint_t scan2scan_reg_con;
        if (!read_rows(argv[1], scan2scan_reg_con.block1->pc_down) || !read_rows(argv[2], scan2scan_reg_con.block2->pc_down)) return 2;
        bbox(scan2scan_reg_con.block1->pc_down, scan2scan_reg_con.block1->local_bound);
        bbox(scan2scan_reg_con.block2->pc_down, scan2scan_reg_con.block2->local_bound);
        const int max_iteration_num_s2s = std::atoi(argv[4]);
        const int ret = lo::b200::omp_gicp_pcl<Point_T>(scan2scan_reg_con, max_iteration_num_s2s, FLAGS_reg_dis_thre_unit,
                                                       initial_guess_tran, FLAGS_reg_intersection_filter_on);
        double out[17];
        out[0] = ret;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) out[1 + 4 * r + c] = scan2scan_reg_con.Trans1_2(r, c);
        FILE *f = std::fopen(argv[3], "wb");
        if (!f || std::fwrite(out, sizeof(double), 17, f) != 17) ++failures;
        if (f) std::fclose(f);
        std::printf("gicp_pcl shim: returned %d; failures %d\n", ret, failures);
        return failures;
    }
    // a stand-in scene: a noisy ground with two walls, spread by an additive recurrence (a lattice would leave the
    // point-to-point matches ambiguous by its spacing); the source is the target shifted by (0.2, -0.1, 0)
    constraint_t scan2scan_reg_con, scan2map_reg_con, few_reg_con;
    for (constraint_t *c : {&scan2scan_reg_con, &scan2map_reg_con})
        for (int i = 0; i < 4000; ++i) {
            Point_T p = {};
            const float u = (float)(40.0 * std::fmod(i * 0.7548776662466927, 1.0) - 20.0);
            const float v = (float)(40.0 * std::fmod(i * 0.5698402909980532, 1.0) - 20.0);
            const float e = 0.01f * (float)((i * 7) % 11 - 5);
            if (i % 3 == 0) p.x = u, p.y = v, p.z = e;
            else if (i % 3 == 1) p.x = 20.f + e, p.y = u, p.z = (float)(i % 60) * 0.1f;
            else p.x = u, p.y = 20.f + e, p.z = (float)(i % 60) * 0.1f;
            c->block1->pc_down->points.push_back(p);
            p.x -= 0.2f, p.y += 0.1f;
            c->block2->pc_down->points.push_back(p);
        }
    for (int i = 0; i < 19; ++i) few_reg_con.block2->pc_down->points.push_back(scan2scan_reg_con.block2->pc_down->points[i]);
    few_reg_con.block1->pc_down->points = scan2scan_reg_con.block1->pc_down->points;
    for (constraint_t *c : {&scan2scan_reg_con, &scan2map_reg_con, &few_reg_con}) {
        bbox(c->block1->pc_down, c->block1->local_bound);
        bbox(c->block2->pc_down, c->block2->local_bound);
    }
    const int max_iteration_num_s2s = 15;
    // :637-639 scan to scan, every argument
    const int a = lo::b200::omp_gicp_pcl<Point_T>(scan2scan_reg_con, max_iteration_num_s2s, FLAGS_reg_dis_thre_unit,
                                                 initial_guess_tran, FLAGS_reg_intersection_filter_on);
    // :674-676 scan to map, the defaults after max_iter_num
    const int b = lo::b200::omp_gicp_pcl<Point_T>(scan2map_reg_con, max_iteration_num_s2s);
    int ran = 0;
    if (a == 1 && b == 1) { // on a device: the shift recovered
        ran = 1;
        for (const constraint_t *c : {&scan2scan_reg_con, &scan2map_reg_con})
            if (std::abs(c->Trans1_2(0, 3) - 0.2) > 0.02 || std::abs(c->Trans1_2(1, 3) + 0.1) > 0.02) ++failures;
    } else if (a != -3 || b != -3 || scan2scan_reg_con.Trans1_2(0, 3) != 0.0) { // no device: -3, Trans1_2 untouched
        ++failures;
    }
    // 19 source points: refused (on a device MULLS_E_UNSUPPORTED sets *unsupported)
    bool unsupported = false;
    const int c = lo::b200::omp_gicp_pcl<Point_T>(few_reg_con, max_iteration_num_s2s, FLAGS_reg_dis_thre_unit, initial_guess_tran,
                                                 false, 10.0f, &unsupported);
    if (c != -3 || (ran && !unsupported)) ++failures;
    std::printf("gicp_pcl shim compiled and linked; ran on a device: %d; failures %d\n", ran, failures);
    return failures;
}
