// Scalar device helpers: the reference's float/double arithmetic restated for the GPU.
// The whole library is compiled with -fmad=false so that no multiply-add is contracted: the
// reference's distro build (x86-64, -O3, no -march) performs none either.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>

#include "grid_key.cuh"

namespace mulls {

__device__ __forceinline__ int float_to_ordered(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : (i ^ 0x7fffffff);
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i >= 0 ? i : (i ^ 0x7fffffff)); }

// cregistration.hpp:2686-2692 get_weight_by_dist_adaptive
__device__ __forceinline__ float weight_by_dist_adaptive(float dist, int iter_num) {
    const float unit_dist = 30.0f, b_min = 0.7f, b_max = 1.3f, b_step = 0.05f;
    float t = b_min + b_step * (float)iter_num;
    float b_current = (t < b_max) ? t : b_max;
    double tw = (double)b_current + (1.0 - (double)b_current) * (double)dist / (double)unit_dist;
    float temp_weight = (float)tw;
    temp_weight = ((double)temp_weight > 0.01) ? temp_weight : (float)0.01;
    return temp_weight;
}
// cregistration.hpp:2701-2707 get_weight_by_intensity (arguments already narrowed to float by the call)
__device__ __forceinline__ float weight_by_intensity(float i1, float i2) {
    float ratio = fabsf(i1 - i2) / 255.0f;
    return (float)exp(-1.0 * (double)ratio);
}
// cregistration.hpp:2710-2722 get_weight_by_residual, delta = 1
__device__ __forceinline__ float weight_by_residual(float res, float huber_thre) {
    if (res > huber_thre) return ((2.0f * res * huber_thre + (-1.0f) * (huber_thre * huber_thre)) / res) / res;
    return 1.0f;
}

// cfilter.hpp:470-516 apply_motion_compensation, one point: p <- slerp(Identity, q, s) * p + s * t with s = the point's
// timestamp ratio `curv` (widened) — Eigen's QuaternionBase::slerp from the identity (d = q.w: the `absD >= 1 - eps`
// linear branch and the `d < 0` sign flip, constants from the host: linear, neg, theta = acos|d|, sin theta), then
// Eigen's quaternion-vector product, in double, stored as float. A point with curv < thre or curv > 1.0 - thre is left
// as it is (false). The ingest's undistortion (thre 0) and k_motion_compensation both run this text.
// The constants are taken by reference: each is read where the reference's text reads it.
MULLS_HD bool slerp_compensate(const double *q, const double *t, const int &linear, const int &neg, const double &theta,
                               const double &sin_theta, float thre, float curv, float &x, float &y, float &z) {
    if (curv < thre || (double)curv > 1.0 - (double)thre) return false;
    const double s = (double)curv;
    double scale0, scale1;
    if (linear) {
        scale0 = 1.0 - s;
        scale1 = s;
    } else {
        scale0 = sin((1.0 - s) * theta) / sin_theta;
        scale1 = sin(s * theta) / sin_theta;
    }
    if (neg) scale1 = -scale1;
    const double qx = scale1 * q[0], qy = scale1 * q[1], qz = scale1 * q[2], qw = scale0 + scale1 * q[3];
    const double vx = x, vy = y, vz = z;
    double ux = qy * vz - qz * vy, uy = qz * vx - qx * vz, uz = qx * vy - qy * vx;
    ux += ux, uy += uy, uz += uz;
    const double rx = vx + qw * ux + (qy * uz - qz * uy);
    const double ry = vy + qw * uy + (qz * ux - qx * uz);
    const double rz = vz + qw * uz + (qx * uy - qy * ux);
    x = (float)(rx + s * t[0]);
    y = (float)(ry + s * t[1]);
    z = (float)(rz + s * t[2]);
    return true;
}

// 6x6 inverse by partial-pivot LU + identity solve (Eigen::PartialPivLU::inverse, Appendix B.9).
// Executed by ONE thread on shared-memory matrices (dynamic indexing), ~1.5k flops.
__device__ inline void inverse6(const double *A /*36 row-major*/, double *out /*36*/, double *lu /*36 scratch*/) {
    int perm[6];
    for (int i = 0; i < 36; ++i) lu[i] = A[i];
    for (int i = 0; i < 6; ++i) perm[i] = i;
    for (int k = 0; k < 6; ++k) {
        int piv = k;
        double best = fabs(lu[6 * k + k]);
        for (int r = k + 1; r < 6; ++r) {
            double v = fabs(lu[6 * r + k]);
            if (v > best) {
                best = v;
                piv = r;
            }
        }
        if (piv != k) {
            for (int c = 0; c < 6; ++c) {
                double t = lu[6 * k + c];
                lu[6 * k + c] = lu[6 * piv + c];
                lu[6 * piv + c] = t;
            }
            int t = perm[k];
            perm[k] = perm[piv];
            perm[piv] = t;
        }
        double d = lu[6 * k + k];
        for (int r = k + 1; r < 6; ++r) lu[6 * r + k] = lu[6 * r + k] / d;
        for (int r = k + 1; r < 6; ++r)
            for (int c = k + 1; c < 6; ++c) lu[6 * r + c] = lu[6 * r + c] - lu[6 * r + k] * lu[6 * k + c];
    }
    for (int col = 0; col < 6; ++col) {
        double y[6];
        for (int r = 0; r < 6; ++r) {
            double s = (perm[r] == col) ? 1.0 : 0.0;
            for (int c = 0; c < r; ++c) s = s - lu[6 * r + c] * y[c];
            y[r] = s;
        }
        for (int r = 5; r >= 0; --r) {
            double s = y[r];
            for (int c = r + 1; c < 6; ++c) s = s - lu[6 * r + c] * out[6 * c + col];
            out[6 * r + col] = s / lu[6 * r + r];
        }
    }
}

// Eigen::AngleAxisd(Matrix3d).angle(): rotation matrix -> quaternion -> 2*atan2(|v|, |w|)
__device__ inline double rotation_angle(const double *T /*row-major 4x4*/) {
    const double m00 = T[0], m01 = T[1], m02 = T[2], m10 = T[4], m11 = T[5], m12 = T[6], m20 = T[8], m21 = T[9],
                 m22 = T[10];
    double w, x, y, z;
    double t = m00 + m11 + m22;
    if (t > 0.0) {
        t = sqrt(t + 1.0);
        w = 0.5 * t;
        t = 0.5 / t;
        x = (m21 - m12) * t;
        y = (m02 - m20) * t;
        z = (m10 - m01) * t;
    } else {
        const double m[3][3] = {{m00, m01, m02}, {m10, m11, m12}, {m20, m21, m22}};
        int i = 0;
        if (m[1][1] > m[0][0]) i = 1;
        if (m[2][2] > m[i][i]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
        double q[3];
        q[i] = 0.5 * t;
        t = 0.5 / t;
        w = (m[k][j] - m[j][k]) * t;
        q[j] = (m[j][i] + m[i][j]) * t;
        q[k] = (m[k][i] + m[i][k]) * t;
        x = q[0];
        y = q[1];
        z = q[2];
    }
    double n = sqrt(x * x + y * y + z * z);
    if (n != 0.0) return 2.0 * atan2(n, fabs(w));
    return 0.0;
}

// cregistration.hpp:2740-2764 construct_trans_a -> row-major 4x4
__device__ inline void construct_trans_a(const double *x, double *T) {
    const double tx = x[0], ty = x[1], tz = x[2], alpha = x[3], beta = x[4], gamma = x[5];
    const double sa = sin(alpha), ca = cos(alpha), sb = sin(beta), cb = cos(beta), sg = sin(gamma), cg = cos(gamma);
    T[0] = cg * cb;
    T[1] = -sg * ca + cg * sb * sa;
    T[2] = sg * sa + cg * sb * ca;
    T[3] = tx;
    T[4] = sg * cb;
    T[5] = cg * ca + sg * sb * sa;
    T[6] = -cg * sa + sg * sb * ca;
    T[7] = ty;
    T[8] = -sb;
    T[9] = cb * sa;
    T[10] = cb * ca;
    T[11] = tz;
    T[12] = 0.0;
    T[13] = 0.0;
    T[14] = 0.0;
    T[15] = 1.0;
}

__device__ inline void mat4_mul(const double *A, const double *B, double *C) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = A[4 * i] * B[j];
            for (int k = 1; k < 4; ++k) s = s + A[4 * i + k] * B[4 * k + j];
            C[4 * i + j] = s;
        }
}

} // namespace mulls
