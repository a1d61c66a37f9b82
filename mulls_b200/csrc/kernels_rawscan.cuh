// Raw-scan corrections of lo::CFilter<PointT> that the SLAM driver runs on every scan (include/common/cfilter.hpp):
//   k_vertical_calib      vertical_intrinsic_calibration (:250-291), one thread per point
//   k_azimuth_ratio       get_pts_timestamp_ratio_in_frame (:412-467) without timestamps: ratio from the azimuth
//   k_ts_*                the same with timestamps (the curvature column): last / first timestamp as the reference's
//                         sequential max_ / min_ macros leave them, then the clamped ratio per point
//   k_motion_compensation apply_motion_compensation (:470-516) / batch_apply_motion_compensation (:519-549) over the
//                         concatenated clouds of one call: slerp_compensate (device_math.cuh) per point
// Every kernel reads the caller's 48-byte rows (x y z _ | n _ | intensity curvature _ _) and writes only the column it
// changes. The library is compiled with -fmad=false: no multiply-add is contracted, as in the reference's x86-64 build.
#pragma once
#include "device_math.cuh"

namespace mulls {

constexpr int kRawBlock = 256;

// vertical_intrinsic_calibration. negate_only (var >= 180 or inverse_z): z *= -1.0 and nothing else — the product is exact,
// and the x86-64 build of the reference emits it as a sign flip, which also flips the sign of a NaN. Otherwise
// dist = sqrt of the float sum of float products (std::sqrt(float)), widened; asin(z / dist), both cos and the sin in
// double; x, y scaled by the double hor_scale and stored as float; z = dist * sin(v_ang + var). A point at the origin
// gives 0 / 0: NaN, as in the reference.
__global__ void __launch_bounds__(kRawBlock) k_vertical_calib(const float *rows, uint32_t n, double var_rad, int negate_only,
                                                              float *xyz_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = rows[12 * (size_t)i], y = rows[12 * (size_t)i + 1], z = rows[12 * (size_t)i + 2];
    float *o = xyz_out + 3 * (size_t)i;
    if (negate_only) {
        o[0] = x, o[1] = y, o[2] = -z; // z *= (-1.0): exact, and compiled as a sign flip (a NaN's sign flips too)
        return;
    }
    const double dist = (double)sqrtf(x * x + y * y + z * z);
    const double v_ang = asin((double)z / dist);
    const double v_ang_c = v_ang + var_rad;
    const double hor_scale = cos(v_ang_c) / cos(v_ang);
    o[0] = (float)((double)x * hor_scale);
    o[1] = (float)((double)y * hor_scale);
    o[2] = (float)(dist * sin(v_ang_c));
}

// get_pts_timestamp_ratio_in_frame(timestamp_availiable = false). std::atan2(float, float) is the float overload; its
// value here is the double atan2 rounded to float (the correctly rounded result but for double-rounding ties). The wrap
// to [0, 2 pi), the shift by the begin angle and the ratio are double, stored as float.
__global__ void __launch_bounds__(kRawBlock) k_azimuth_ratio(const float *rows, uint32_t n, double begin_rad, float *ratio) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = rows[12 * (size_t)i], y = rows[12 * (size_t)i + 1];
    double ang = (double)(float)atan2((double)y, (double)x);
    const double two_pi = 2 * M_PI;
    if (ang < 0) ang += two_pi;
    ang += begin_rad;
    if (ang >= two_pi) ang -= two_pi;
    ratio[i] = (float)((two_pi - ang) / two_pi);
}

// ---- timestamp mode. The reference folds last = max_(last, c) and first = min_(first, c) over the points in order,
// with max_(a, b) = ((a) > (b) ? (a) : (b)). A NaN timestamp becomes the running value and the next point replaces it,
// so each result is the fold of the points after the last NaN (NaN when the last point is NaN), started from -DBL_MAX /
// DBL_MAX only when there is no NaN at all. Equal values (+0 and -0) resolve to the later point. Here: the last NaN
// index, then the extremes of the suffix as 64-bit keys (order-preserving value bits with -0 read as +0 | point index;
// the min key holds the complemented index), so that one atomicMax / atomicMin per block picks the value and, among
// equal values, the latest point. The two reductions take the column they fold as a template parameter: 9 (curvature)
// here, 8 (intensity) for the NCC intensity range of kernels_ncc.cuh, whose folds start from FLT_MAX / 0.
struct TsState {
    unsigned long long last_nan;      // index + 1 of the last NaN timestamp, 0: none
    unsigned long long max_key, min_key;
    double last, first;
    float scan_duration_ms;
    int pad;
};

__device__ __forceinline__ uint32_t ts_value_bits(float c) {
    const int o = float_to_ordered(c == 0.0f ? 0.0f : c);
    return (uint32_t)o ^ 0x80000000u;
}
__device__ __forceinline__ float ts_curvature(const float *rows, size_t i) { return rows[12 * i + 9]; }
template <int kCol>
__device__ __forceinline__ float row_column(const float *rows, size_t i) { return rows[12 * i + kCol]; }

template <int kCol>
__global__ void __launch_bounds__(kRawBlock) k_ts_last_nan(const float *rows, uint32_t n, TsState *st) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long v = (i < n && isnan(row_column<kCol>(rows, i))) ? (unsigned long long)i + 1 : 0ull;
    const unsigned long long m = __reduce_max_sync(0xffffffffu, (unsigned)v); // n < 2^32 - 1
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&st->last_nan, m);
}

template <int kCol>
__global__ void __launch_bounds__(kRawBlock) k_ts_extremes(const float *rows, uint32_t n, TsState *st) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long kmax = 0ull, kmin = ~0ull;
    if (i < n && (unsigned long long)i >= st->last_nan) { // the suffix after the last NaN: no NaN in it
        const unsigned long long vb = (unsigned long long)ts_value_bits(row_column<kCol>(rows, i)) << 32;
        kmax = vb | i;
        kmin = vb | (uint32_t)~i;
    }
    __shared__ unsigned long long s_max[kRawBlock / 32], s_min[kRawBlock / 32];
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmax, o), b = __shfl_xor_sync(0xffffffffu, kmin, o);
        kmax = a > kmax ? a : kmax;
        kmin = b < kmin ? b : kmin;
    }
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = kmax, s_min[threadIdx.x >> 5] = kmin;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kRawBlock / 32; ++w) {
            kmax = s_max[w] > kmax ? s_max[w] : kmax;
            kmin = s_min[w] < kmin ? s_min[w] : kmin;
        }
        if (kmax != 0ull) atomicMax(&st->max_key, kmax);
        if (kmin != ~0ull) atomicMin(&st->min_key, kmin);
    }
}

// one thread: last / first as the macros leave them, then :431-434 (the duration narrowed to float when shorter than
// 0.75 x scan_duration_ms)
__global__ void k_ts_setup(const float *rows, uint32_t n, float scan_duration_ms, TsState *st) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double last, first;
    if (st->last_nan == (unsigned long long)n) { // the last point is NaN: both folds end on it
        last = first = (double)ts_curvature(rows, n - 1);
    } else {
        last = (double)ts_curvature(rows, (uint32_t)st->max_key);
        first = (double)ts_curvature(rows, ~(uint32_t)st->min_key);
        if (st->last_nan == 0ull) { // no NaN: the folds start from -DBL_MAX / DBL_MAX
            last = (-DBL_MAX > last) ? -DBL_MAX : last;
            first = (DBL_MAX < first) ? DBL_MAX : first;
        }
    }
    const double actual_scan_duration = last - first;
    if (actual_scan_duration < scan_duration_ms * 0.75) scan_duration_ms = (float)actual_scan_duration;
    st->last = last;
    st->first = first;
    st->scan_duration_ms = scan_duration_ms;
}

// :436-440: s = (last - curvature) / scan_duration_ms in double, min_(1.0, max_(0.0, s)) stored as float
__global__ void __launch_bounds__(kRawBlock) k_ts_ratio(const float *rows, uint32_t n, const TsState *st, float *ratio) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double s = (st->last - (double)ts_curvature(rows, i)) / (double)st->scan_duration_ms;
    const double lo = (0.0 > s) ? 0.0 : s;
    ratio[i] = (float)((1.0 < lo) ? 1.0 : lo);
}

// ---- motion compensation over the concatenated clouds of one call: xyz_out is the point's new position, or its
// old one when its timestamp ratio falls outside [thre, 1 - thre]
struct SlerpConst {
    double q[4]; // x y z w of Eigen::Quaterniond(T.block<3,3>(0,0))
    double t[3]; // T.block<3,1>(0,3)
    double theta, sin_theta;
    int linear, neg;
};

__global__ void __launch_bounds__(kRawBlock) k_motion_compensation(const float *rows, uint32_t n, SlerpConst sc, float thre,
                                                                   float *xyz_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *r = rows + 12 * (size_t)i;
    float x = r[0], y = r[1], z = r[2];
    slerp_compensate(sc.q, sc.t, sc.linear, sc.neg, sc.theta, sc.sin_theta, thre, r[9], x, y, z);
    float *o = xyz_out + 3 * (size_t)i;
    o[0] = x, o[1] = y, o[2] = z;
}

} // namespace mulls
