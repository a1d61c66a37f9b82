// test/mulls_slam.cpp:634-636 and :671-673 (CRegistration::omp_ndt, cregistration.hpp:945-1021) against the DROP-IN
// headers (include/dropin), with the reference's own header and class names and nothing edited. Include path order:
// include/dropin, include, tests/stubs/ndt_ref (a stand-in reference class that declares omp_ndt), tests/stubs.
//   ndt_caller                                  both call sites on a small scene, once with --ndt_searching_method
//                                               true (the device; without a GPU the call reports the missing device,
//                                               returns -3 and leaves Trans1_2 alone) and once false (KDTREE: the
//                                               reference member runs)
//   ndt_caller tgt.bin src.bin out.bin res      48-byte rows in (block1 / block2 ->pc_down, local_bound their bboxes);
//                                               the return value and Trans1_2 (row-major) out as 17 doubles
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
    CRegistration<Point_T> creg;
    int failures = 0;
    const bool FLAGS_reg_intersection_filter_on = true;
    Eigen::Matrix4d initial_guess_tran = Eigen::Matrix4d::Identity();
    if (argc == 5) {
        constraint_t scan2scan_reg_con;
        if (!read_rows(argv[1], scan2scan_reg_con.block1->pc_down) || !read_rows(argv[2], scan2scan_reg_con.block2->pc_down)) return 2;
        bbox(scan2scan_reg_con.block1->pc_down, scan2scan_reg_con.block1->local_bound);
        bbox(scan2scan_reg_con.block2->pc_down, scan2scan_reg_con.block2->local_bound);
        const float FLAGS_reg_voxel_size = (float)std::atof(argv[4]);
        const bool FLAGS_ndt_searching_method = true;
        const int ret = creg.omp_ndt(scan2scan_reg_con, FLAGS_reg_voxel_size, FLAGS_ndt_searching_method, initial_guess_tran,
                                     FLAGS_reg_intersection_filter_on);
        double out[17];
        out[0] = ret;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) out[1 + 4 * r + c] = scan2scan_reg_con.Trans1_2(r, c);
        FILE *f = std::fopen(argv[3], "wb");
        if (!f || std::fwrite(out, sizeof(double), 17, f) != 17) ++failures;
        if (f) std::fclose(f);
        std::printf("ndt drop-in: returned %d; failures %d\n", ret, failures);
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
    const float FLAGS_reg_voxel_size = 1.0f;
    int ran = 0;
    for (int method = 1; method >= 0; --method) {
        const bool FLAGS_ndt_searching_method = method == 1;
        // :634-636 scan to scan
        constraint_t scan2scan_reg_con;
        creg.assign_source_target_cloud(cblock_target, cblock_source, scan2scan_reg_con);
        const int a = creg.omp_ndt(scan2scan_reg_con, FLAGS_reg_voxel_size, FLAGS_ndt_searching_method, initial_guess_tran,
                                   FLAGS_reg_intersection_filter_on);
        // :671-673 scan to map
        constraint_t scan2map_reg_con;
        creg.assign_source_target_cloud(cblock_local_map, cblock_source, scan2map_reg_con);
        const int b = creg.omp_ndt(scan2map_reg_con, FLAGS_reg_voxel_size, FLAGS_ndt_searching_method, initial_guess_tran,
                                   FLAGS_reg_intersection_filter_on);
        if (!FLAGS_ndt_searching_method) { // KDTREE: the reference member
            if (a != -77 || b != -77 || scan2scan_reg_con.Trans1_2(0, 3) != 77.0 || scan2map_reg_con.Trans1_2(0, 3) != 77.0) ++failures;
        } else if (a == 1 && b == 1) { // on a device: the shift recovered to within the walk's last step
            ++ran;
            for (const constraint_t *c : {&scan2scan_reg_con, &scan2map_reg_con})
                if (std::abs(c->Trans1_2(0, 3) - 0.2) > 0.1 || std::abs(c->Trans1_2(1, 3) + 0.1) > 0.1) ++failures;
        } else if (a != -3 || b != -3 || scan2scan_reg_con.Trans1_2(0, 3) != 0.0) { // no device: -3, Trans1_2 untouched
            ++failures;
        }
    }
    std::printf("ndt drop-in compiled and linked; ran on a device: %d; failures %d\n", ran, failures);
    return failures;
}
