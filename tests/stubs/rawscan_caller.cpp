// test/mulls_slam.cpp:404-428 (a source frame's raw-scan corrections and feature extraction) and :707-711 (its motion
// compensation after the registration) against the DROP-IN headers (include/dropin), with the reference's own header and
// class names and nothing edited. Flags as a 32 / 128-beam flagfile sets them: vertical_ang_calib_on with a 0.5 degree
// correction, apply_scanner_filter, motion_compensation_method 1 (timestamps in the curvature column) or 2 (azimuth,
// begin angle 90), motion_com_while_reg_on; the other extract_semantic_pts arguments as tests/stubs/slam_frontend_caller.cpp
// passes them. Include path order as for dropin_caller.cpp: include/dropin, include, tests/stubs/ref, tests/stubs.
//   rawscan_caller                           a small synthetic scan (without a GPU every call reports the missing
//                                            device and leaves its clouds as they were)
//   rawscan_caller raw.bin method out_dir    48-byte rows in; pc_raw and the twelve feature clouds the calls leave out,
//                                            as out_dir/<name>.bin (tests/test_gpu_rawscan.py)
#include <cmath>
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
static bool write_rows(const std::string &path, const CloudPtr &c) {
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const size_t w = c->points.empty() ? 0 : std::fwrite(c->points.data(), sizeof(Point_T), c->points.size(), f);
    std::fclose(f);
    return w == c->points.size();
}

// the transform test/mulls_slam.cpp:701 computes (adjacent_pose_out), fixed here: 0.04 rad about (0.1, 0.2, 1), then
// (1.2, -0.3, 0.05) — the rotation tests/test_rawscan.py calls "small"
static Eigen::Matrix4d adjacent_pose() {
    const double ax[3] = {0.1, 0.2, 1.0}, ang = 0.04, t[3] = {1.2, -0.3, 0.05};
    const double nrm = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
    const double a[3] = {ax[0] / nrm, ax[1] / nrm, ax[2] / nrm};
    const double K[3][3] = {{0, -a[2], a[1]}, {a[2], 0, -a[0]}, {-a[1], a[0], 0}};
    Eigen::Matrix4d T = Eigen::Matrix4d::Identity();
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) {
            double kk = 0;
            for (int m = 0; m < 3; ++m) kk += K[r][m] * K[m][c];
            T(r, c) = (r == c ? 1.0 : 0.0) + std::sin(ang) * K[r][c] + (1 - std::cos(ang)) * kk;
        }
        T(r, 3) = t[r];
    }
    return T;
}

int main(int argc, char **argv) {
    CFilter<Point_T> cfilter;
    cloudblock_Ptr cblock_source(new cloudblock_t());
    int FLAGS_motion_compensation_method = 1;
    if (argc == 4) {
        if (!read_rows(argv[1], cblock_source->pc_raw)) return 2;
        FLAGS_motion_compensation_method = std::atoi(argv[2]);
    } else { // a ring of 2000 points at 10 m, timestamps 0..100 ms, plus three ego-vehicle points the scanner filter drops
        for (int i = 0; i < 2000; ++i) {
            Point_T p = {};
            const double az = 2 * M_PI * i / 2000.0;
            p.x = (float)(10 * std::cos(az)), p.y = (float)(10 * std::sin(az)), p.z = (float)(-1.5 + 0.001 * (i % 7));
            p.curvature = (float)(0.05 * i);
            cblock_source->pc_raw->points.push_back(p);
        }
        for (int i = 0; i < 3; ++i) {
            Point_T p = {};
            p.x = 0.5f * i, p.y = 0.3f, p.z = -1.0f;
            cblock_source->pc_raw->points.push_back(p);
        }
    }
    const size_t n_raw = cblock_source->pc_raw->points.size();
    const bool FLAGS_vertical_ang_calib_on = true, FLAGS_apply_scanner_filter = true, motion_com_while_reg_on = true;
    const double FLAGS_vertical_ang_correction_deg = 0.5;

    // :407-412
    if (FLAGS_vertical_ang_calib_on) //intrinsic angle correction
        cfilter.vertical_intrinsic_calibration(cblock_source->pc_raw, FLAGS_vertical_ang_correction_deg);
    if (FLAGS_motion_compensation_method == 1)                                       //calculate from time-stamp
        cfilter.get_pts_timestamp_ratio_in_frame(cblock_source->pc_raw, true);
    else if (FLAGS_motion_compensation_method == 2)                                   //calculate from azimuth
        cfilter.get_pts_timestamp_ratio_in_frame(cblock_source->pc_raw, false, 90.0); //HESAI Lidar: 90.0 (y+ axis, clockwise)
    // :418-428
    int ground_down_rate = 15, nonground_down_rate = 3;
    const bool ok = cfilter.extract_semantic_pts(cblock_source, 0.05f, 3.0f, 0.3f, 1.5f, 5.0f, ground_down_rate, nonground_down_rate, 1.0f,
                                                 50, 0.65f, 0.65f, 0.12f, 0.75f, 0.75f, true, 2, 15.0f, 3, 2.0f, false,
                                                 FLAGS_apply_scanner_filter, false, 2, 10, 0, 2, 8, 1, FLT_MAX, 0.94f, 0.17f, 0.98f, 0.34f,
                                                 true, false, 300, 200, 800, 200, 100, 10000, FLT_MAX, 0.0f, 2.0f, -7.0f, 0.3f, false,
                                                 false, 0.0f, 0.0f);
    const size_t n_filtered = cblock_source->pc_raw->points.size();
    // :705-711
    Eigen::Matrix4d adjacent_pose_out = adjacent_pose();
    if (motion_com_while_reg_on) {
        cfilter.apply_motion_compensation(cblock_source->pc_raw, adjacent_pose_out);
        cfilter.batch_apply_motion_compensation(cblock_source->pc_ground, cblock_source->pc_pillar, cblock_source->pc_facade,
                                                cblock_source->pc_beam, cblock_source->pc_roof, cblock_source->pc_vertex, adjacent_pose_out);
        cfilter.batch_apply_motion_compensation(cblock_source->pc_ground_down, cblock_source->pc_pillar_down, cblock_source->pc_facade_down,
                                                cblock_source->pc_beam_down, cblock_source->pc_roof_down, cblock_source->pc_vertex, adjacent_pose_out);
    }
    int failures = 0;
    if (cfilter.reference_body_ran) ++failures, std::printf("FAIL: a reference CFilter body ran\n");
    if (argc == 4) {
        const std::string d = argv[3];
        const std::pair<const char *, CloudPtr> outs[] = {
            {"raw", cblock_source->pc_raw},           {"ground", cblock_source->pc_ground},
            {"pillar", cblock_source->pc_pillar},     {"beam", cblock_source->pc_beam},
            {"facade", cblock_source->pc_facade},     {"roof", cblock_source->pc_roof},
            {"vertex", cblock_source->pc_vertex},     {"ground_down", cblock_source->pc_ground_down},
            {"pillar_down", cblock_source->pc_pillar_down}, {"beam_down", cblock_source->pc_beam_down},
            {"facade_down", cblock_source->pc_facade_down}, {"roof_down", cblock_source->pc_roof_down}};
        for (const auto &o : outs)
            if (!write_rows(d + "/" + o.first + ".bin", o.second)) ++failures;
        if (!ok) ++failures;
    } else if (n_filtered != n_raw - 3) { // the scanner filter runs on the host: it drops the three points in the self ring
        ++failures;
    }
    std::printf("rawscan drop-in compiled and linked; ran on a device: %d; raw %zu -> %zu after the scanner filter; failures %d\n",
                ok ? 1 : 0, n_raw, n_filtered, failures);
    return failures;
}
