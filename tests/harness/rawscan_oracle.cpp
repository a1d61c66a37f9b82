// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of the raw-scan corrections of lo::CFilter<PointT>
// (include/common/cfilter.hpp), the checker of mulls_vertical_intrinsic_calibration, mulls_timestamp_ratio and
// mulls_motion_compensation, and of the scanner filter in the drop-in extract_semantic_pts:
//   vertical_intrinsic_calibration :250-291, get_pts_timestamp_ratio_in_frame :412-467, apply_motion_compensation
//   :470-516, batch_apply_motion_compensation :519-549, scanner_filter :914-929 with the thresholds of :2334-2343.
// The members are restated line by line on 48-byte pcl::PointXYZINormal rows (x y z _ | n _ | intensity curvature _ _),
// with the reference's float / double types and std:: overloads. oracle/mulls_oracle.cpp is included, not copied or
// changed, for Eigen's matrix-to-quaternion conversion (quat_from_rotation). Per-point loops may run on several OpenMP
// threads (the reference runs the motion compensation on min(6, max) threads and the rest on one); no result depends on
// it. The reference's motion compensation shares d_quat / d_translation between its threads; here they are per point.
// Built by tests/test_rawscan.py with the flags oracle/Makefile builds the oracle with (-O3 -fopenmp -ffp-contract=off).
#include "../../oracle/mulls_oracle.cpp"

#include <cfloat>

#define max_(a, b) (((a) > (b)) ? (a) : (b)) // utility.hpp:31-32
#define min_(a, b) (((a) < (b)) ? (a) : (b))

namespace {

struct XyzinRow { // pcl::PointXYZINormal
    float x, y, z, pad0;
    float normal_x, normal_y, normal_z, pad1;
    float intensity, curvature, pad2, pad3;
};
static_assert(sizeof(XyzinRow) == 48, "48-byte rows");

#ifdef _OPENMP
int threads_of(int threads) { return threads > 0 ? threads : omp_get_max_threads(); }
#else
int threads_of(int) { return 1; }
#endif

// :250-291
bool vertical_intrinsic_calibration(XyzinRow *points, long n, double var_vertical_ang_d, bool inverse_z, int threads) {
    if (var_vertical_ang_d == 0)
        return false;
    if (var_vertical_ang_d >= 180.0)
        inverse_z = true;
    if (inverse_z) {
        for (long i = 0; i < n; i++)
            points[i].z *= (-1.0);
        return false;
    }
    double var_vertical_ang = var_vertical_ang_d / 180.0 * M_PI;
    const int nt = threads_of(threads);
#pragma omp parallel for num_threads(nt) if (nt > 1)
    for (long i = 0; i < n; i++) {
        double dist = std::sqrt(points[i].x * points[i].x + points[i].y * points[i].y + points[i].z * points[i].z);
        double v_ang = std::asin(points[i].z / dist);
        double v_ang_c = v_ang + var_vertical_ang;
        double hor_scale = std::cos(v_ang_c) / std::cos(v_ang);
        points[i].x *= hor_scale;
        points[i].y *= hor_scale;
        points[i].z = dist * std::sin(v_ang_c);
    }
    return true;
}

// :412-467
bool get_pts_timestamp_ratio_in_frame(XyzinRow *points, long n, bool timestamp_availiable, double scan_begin_ang_anticlock_x_positive_deg,
                                      float scan_duration_ms, int threads) {
    double scan_begin_ang_anticlock_x_positive_rad = scan_begin_ang_anticlock_x_positive_deg / 180.0 * M_PI;
    double last_timestamp = -DBL_MAX;
    double first_timestamp = DBL_MAX;
    double actual_scan_duration;
    const int nt = threads_of(threads);
    if (timestamp_availiable) {
        for (long i = 0; i < n; i++) {
            last_timestamp = max_(last_timestamp, points[i].curvature);
            first_timestamp = min_(first_timestamp, points[i].curvature);
        }
        actual_scan_duration = last_timestamp - first_timestamp;
        if (actual_scan_duration < scan_duration_ms * 0.75)
            scan_duration_ms = actual_scan_duration;
#pragma omp parallel for num_threads(nt) if (nt > 1)
        for (long i = 0; i < n; i++) {
            double s = (last_timestamp - points[i].curvature) / scan_duration_ms;
            points[i].curvature = min_(1.0, max_(0.0, s));
        }
        return true;
    }
#pragma omp parallel for num_threads(nt) if (nt > 1)
    for (long i = 0; i < n; i++) {
        double ang = std::atan2(points[i].y, points[i].x); // the float overload
        if (ang < 0)
            ang += 2 * M_PI;
        ang += scan_begin_ang_anticlock_x_positive_rad;
        if (ang >= 2 * M_PI)
            ang -= 2 * M_PI;
        double s = (2 * M_PI - ang) / (2 * M_PI);
        points[i].curvature = s;
    }
    return true;
}

// Eigen::Quaterniond::Identity().slerp(t, other) [3P]: (x y z w) out
void slerp_from_identity(double t, const double other[4], double out[4]) {
    const double one = 1.0 - 2.220446049250313e-16; // 1 - NumTraits<double>::epsilon()
    double d = other[3];                             // Identity().dot(other)
    double absD = std::fabs(d);
    double scale0;
    double scale1;
    if (absD >= one) {
        scale0 = 1.0 - t;
        scale1 = t;
    } else {
        double theta = std::acos(absD);
        double sinTheta = std::sin(theta);
        scale0 = std::sin((1.0 - t) * theta) / sinTheta;
        scale1 = std::sin((t * theta)) / sinTheta;
    }
    if (d < 0)
        scale1 = -scale1;
    out[0] = scale1 * other[0];
    out[1] = scale1 * other[1];
    out[2] = scale1 * other[2];
    out[3] = scale0 + scale1 * other[3];
}

// :470-491 (in place; the pc_in -> pc_out overload :493-516 computes the same on a copy)
void apply_motion_compensation(XyzinRow *points, long n, const Mat4 &Tran, float s_ambigous_thre, int threads) {
    const double estimated_translation_2_1[3] = {Tran.a[0][3], Tran.a[1][3], Tran.a[2][3]};
    double estimated_quat2_1[4];
    quat_from_rotation(Tran, estimated_quat2_1);
    const int nt = threads_of(threads);
#pragma omp parallel for num_threads(nt) if (nt > 1)
    for (long i = 0; i < n; i++) {
        if (points[i].curvature < s_ambigous_thre || points[i].curvature > 1.0 - s_ambigous_thre)
            continue;
        double d_quat[4];
        slerp_from_identity(points[i].curvature, estimated_quat2_1, d_quat);
        const double t = points[i].curvature;
        const double d_translation[3] = {t * estimated_translation_2_1[0], t * estimated_translation_2_1[1],
                                         t * estimated_translation_2_1[2]};
        const double v[3] = {points[i].x, points[i].y, points[i].z};
        // Eigen's q * v: uv = q.vec() x v; uv += uv; v + q.w() * uv + q.vec() x uv
        double uv[3] = {d_quat[1] * v[2] - d_quat[2] * v[1], d_quat[2] * v[0] - d_quat[0] * v[2], d_quat[0] * v[1] - d_quat[1] * v[0]};
        uv[0] += uv[0], uv[1] += uv[1], uv[2] += uv[2];
        const double r[3] = {v[0] + d_quat[3] * uv[0] + (d_quat[1] * uv[2] - d_quat[2] * uv[1]),
                             v[1] + d_quat[3] * uv[1] + (d_quat[2] * uv[0] - d_quat[0] * uv[2]),
                             v[2] + d_quat[3] * uv[2] + (d_quat[0] * uv[1] - d_quat[1] * uv[0])};
        points[i].x = r[0] + d_translation[0];
        points[i].y = r[1] + d_translation[1];
        points[i].z = r[2] + d_translation[2];
    }
}

// :914-929
long scanner_filter(XyzinRow *points, long n, float self_radius, float ghost_radius, float z_min_thre_ghost, float z_min_thre_global) {
    std::vector<XyzinRow> cloud_temp;
    for (long i = 0; i < n; i++) {
        float dis_square = points[i].x * points[i].x + points[i].y * points[i].y;
        if (dis_square > self_radius * self_radius && points[i].z > z_min_thre_global) {
            if (dis_square > ghost_radius * ghost_radius || points[i].z > z_min_thre_ghost)
                cloud_temp.push_back(points[i]);
        }
    }
    std::copy(cloud_temp.begin(), cloud_temp.end(), points);
    return (long)cloud_temp.size();
}

Mat4 mat4_of(const double *T) {
    Mat4 M;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) M.a[r][c] = T[4 * r + c];
    return M;
}

} // namespace

extern "C" {

// every function works in place on n 48-byte rows; threads: 0 = every core, n > 0 = n threads
int orc_vertical_intrinsic_calibration(float *rows, size_t n, double var_vertical_ang_d, int inverse_z, int threads) {
    return vertical_intrinsic_calibration(reinterpret_cast<XyzinRow *>(rows), (long)n, var_vertical_ang_d, inverse_z != 0, threads) ? 1 : 0;
}

int orc_timestamp_ratio(float *rows, size_t n, int timestamp_available, double scan_begin_ang_deg, float scan_duration_ms, int threads) {
    return get_pts_timestamp_ratio_in_frame(reinterpret_cast<XyzinRow *>(rows), (long)n, timestamp_available != 0, scan_begin_ang_deg,
                                            scan_duration_ms, threads) ? 1 : 0;
}

// T row-major
void orc_motion_compensation(float *rows, size_t n, const double *T, float s_ambiguous_thre, int threads) {
    apply_motion_compensation(reinterpret_cast<XyzinRow *>(rows), (long)n, mat4_of(T), s_ambiguous_thre, threads);
}

// :519-549: ground, pillar, beam, facade, roof (and vertex when undistort_keypoints_or_not), each with the threshold 0
void orc_batch_motion_compensation(float *const *rows, const size_t *n, const double *T, int undistort_keypoints_or_not, int threads) {
    const Mat4 M = mat4_of(T);
    for (int k = 0; k < (undistort_keypoints_or_not ? 6 : 5); ++k)
        apply_motion_compensation(reinterpret_cast<XyzinRow *>(rows[k]), (long)n[k], M, 0.0f, threads);
}

// the oracle's own motion_compensate (threshold 0), for the cross-check of the two restatements
void orc_oracle_motion_compensate(float *rows, size_t n, const double *T) {
    Cloud c(n);
    XyzinRow *r = reinterpret_cast<XyzinRow *>(rows);
    for (size_t i = 0; i < n; ++i) c[i] = Pt{r[i].x, r[i].y, r[i].z, r[i].normal_x, r[i].normal_y, r[i].normal_z, r[i].intensity, r[i].curvature};
    motion_compensate(c, mat4_of(T));
    for (size_t i = 0; i < n; ++i) r[i].x = c[i].x, r[i].y = c[i].y, r[i].z = c[i].z;
}

// extract_semantic_pts :2334-2343 with apply_scanner_filter: the thresholds as the reference computes them, then
// scanner_filter. Returns the number of rows kept (compacted to the front).
size_t orc_extract_scanner_filter(float *rows, size_t n, float approx_scanner_height, float underground_thre) {
    float self_ring_radius = 1.75;
    float ghost_radius = 20.0;
    float z_min = -approx_scanner_height - 4.0;
    float z_min_min = -approx_scanner_height + underground_thre;
    return (size_t)scanner_filter(reinterpret_cast<XyzinRow *>(rows), (long)n, self_ring_radius, ghost_radius, z_min, z_min_min);
}

} // extern "C"
