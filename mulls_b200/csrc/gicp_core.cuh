// Voxelized GICP registration: lo::CRegistration<PointT>::omp_gicp (cregistration.hpp:1024-1098) with using_voxel_gicp,
// i.e. koide_reg::FastVGICP (include/baseline_reg/fast_vgicp_impl.hpp, fast_vgicp_voxel.h, fast_vgicp_utility.h) on
// PCL 1.10 / Eigen 3.3 / Sophus, built with BUILD_WITH_SOPHUS=ON as the reference's Dockerfile does (without Sophus the
// walk compiles to nothing and the result is the identity; that build is not followed).
//
// This header holds what the device path (kernels_gicp.cuh, the host side of mulls_omp_gicp) and the CPU restatement
// under tests/harness share, so that both compute the same bits: the covariance of an ordered neighbour list, the voxel
// key, the voxel finalisation, the per-point loss_ls terms, the fixed summation order, and the Gauss-Newton walk with its
// SO3 arithmetic and its rand() draws. The prologue, the fitness transform and the epilogue are omp_ndt's
// (ndt_core.cuh): omp_gicp's :1035-1058 and :1080-1088 are the same code as omp_ndt's :955-978 and :999-1007.
// omp_gicp leaves FastVGICP at its defaults: k_correspondences 20, max_iterations 64 (max_iter_num is not applied:
// setMaximumOptimizerIterations is commented out for VGICP, :1071), rotation_epsilon 2e-3, transformation_epsilon 5e-4,
// DIRECT1 neighbours, ADDITIVE voxels, PLANE regularisation; corr_dist_threshold_ is never read (dis_thre_unit has no
// effect). No other mode is restated.
// Readings (the reference was read, not run):
//  G1 covariances (calculate_covariances): for every point of a cloud its k = 20 nearest neighbours in the same cloud,
//     the point itself included, listed in FLANN's order (ascending (squared distance, index)); data = the 4 x 20
//     matrix of (x, y, z, 1); row means by rowwise().mean() (the float sum in list order, divided by 20.0f); cov =
//     data data^T in float, the sums in list order (the fourth row and column are zero and dropped); then PLANE:
//     U diag(1, 1, 1e-2f) V^T from JacobiSVD<Matrix3f> (rc_svd<3, float>), (U(i,k) d_k) V(j,k) summed over k in
//     order. Fixed-size float products are read as index-order sums throughout.
//  G2 voxels (create_voxelmap): coord = floor(x / (float)res - 0.5f) per axis (the double resolution converted to
//     float, as Eigen 3.3 converts the scalar of a float array expression), one voxel per coord; ADDITIVE: the means
//     (x, y, z, 1) and the covariances of its points summed in input order in float from 0, then divided by the
//     point count converted to float. The voxel's fourth mean coordinate is exactly 1 and its fourth covariance row
//     and column exactly 0.
//  G3 loss_ls with DIRECT1: trans = [SO3f::exp(x.rot) | x.t] (float, host); transed = trans (a, 1) as ndt_transform;
//     the voxel of coord(transed) or none; RCR = (trans C_A) trans^T with RCR(3,3) = 1, d = mean_B - transed,
//     M = (C_B + RCR)^-1, e = (M d).head<3>, J = [(M skew(transed)).block<3,3> | -M.block<3,3>]. Every product is the
//     full 4 x 4 index-order sum, zero terms included. The inverse is not a reading of the reference: see C3.
//  G4 GaussNewton<double, 6>::delta: JJ = J^T J and J^T e in double from the float J and e (each product of two floats
//     is exact in double, so only the order of the sums matters: C1); LLT<Matrix<double, 6, 6>> is Eigen 3.3's
//     unblocked factorisation (size < 32) on the lower triangle. Its structure is followed: when a pivot x <= 0 it
//     stops there, leaving m(k, k) and everything right of column k - 1 as they were, and solve() runs on that matrix
//     anyway (Eigen 3.3 does not check info()); the forward solve L y = b goes column by column (y_i /= L_ii, then
//     y_j -= y_i L_ji), the backward solve L^T x = y row by row (x_i = (y_i - a sum) / L_ii). The order inside the
//     sums is read, not known: the squared norms, the column update A21 -= A20 A10^T (one index-order dot product per
//     entry, subtracted once) and the backward sums are read as index-order sums. Eigen computes the column update
//     with its GEMV kernel, which accumulates the columns into A21 in groups of four, and may vectorise the backward
//     .sum(), so its order most likely differs; that moves only the last bits of the step. A step with a non-finite
//     entry is replaced by Matrix<double, 6, 1>::Random() * 1e-2.
//  G5 Sophus (not pinned by the reference; restated from its published formulas, SO3<float>, epsilon 1e-5f):
//     exp(w): theta^2 = |w|^2; below epsilon^2 the Taylor factors 0.5 - theta^2 / 48 + theta^4 / 3840 and
//     1 - theta^2 / 8 + theta^4 / 384, else sin(theta / 2) / theta and cos(theta / 2); the quaternion is not
//     renormalised. log(q): n^2 = |q.vec|^2; below epsilon^2, 2 / w - (2/3) n^2 / (w w^2), else 2 atan2(n, w) / n
//     (atan2(-n, -w) for w < 0). The group product is the Hamilton product, renormalised by the constructor:
//     coeffs / sqrt(|coeffs|^2), the squared norm in Eigen 3.3's SSE2 order (x^2 + z^2) + (y^2 + w^2). matrix() is
//     Eigen's toRotationMatrix.
//  G6 the walk (computeTransformation): align() passes no guess, so x0.rot = log(SO3f(I)) = 0, below 1e-2, and x0.rot =
//     Vector3f::Random().normalized() * 1e-2f (three rand() draws); x0.t = 0. Random() draws, per coefficient in
//     index order, -1 + (2 * Scalar(rand())) / Scalar(RAND_MAX) from the process's rand(). Each of at most 64
//     iterations: loss_ls, delta (double, cast to float), x.rot = log(exp(-delta.rot) exp(x.rot)), x.t -= delta.t,
//     stop when max(500.0f |exp(delta.rot) - I|, 2000.0f |delta.t|) < 1 (1.0 / epsilon in double, converted to
//     float). iterations counts the Gauss-Newton steps taken (nr_iterations_ + 1).
//  G7 non-finite points are dropped from both clouds after the prologue (as omp_ndt's N6 leaves them out). With fewer
//     than 20 points in a cloud the reference reads uninitialised columns: such a call is refused.
//     A transformed point with a non-finite coordinate saturates (ndt_f2i) and misses every voxel.
// Choices where the reference depends on the machine (OpenMP's correspondence order, Eigen's blocked products):
//  C1 each source point contributes its 21 lower-triangle entries of J^T J, the 6 of J^T e (three-row sums in row
//     order) and its correspondence count; the points are summed in omp_ndt's order (ndt_core.cuh C1: kNdtTile-point
//     tiles with a pairwise tree, then the tiles in order). A point without a voxel contributes 0.0.
//  C2 voxel coordinates are packed into 21 bits each; a target whose coordinates do not fit is refused, a lookup
//     outside that range misses.
//  C3 Matrix4f::inverse(): on x86 Eigen 3.3 takes its SSE kernel, elsewhere its generic compute_inverse_size4 (three
//     3x3 determinant terms per cofactor, divided by the determinant). Neither is restated: gicp_inv4 is the adjugate
//     (each cofactor one 3x3 determinant) times 1 / det, with det expanded along row 0 in index order. It differs from
//     either of Eigen's kernels in the last bits of M, and so of e and J.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "ndt_core.cuh"

namespace mulls {

constexpr int kGicpK = 20;                       // k_correspondences_
constexpr int kGicpMaxIterations = 64;           // max_iterations_
constexpr double kGicpRotationEpsilon = 2e-3;    // rotation_epsilon_
constexpr double kGicpTranslationEpsilon = 5e-4; // transformation_epsilon_
constexpr int kGicpTerms = 28;                   // J^T J lower triangle (21), J^T e (6), the correspondence count
constexpr int kGicpCoordBits = 21;               // C2
constexpr int kGicpCoordBias = 1 << (kGicpCoordBits - 1);

// ---- G1: the covariance of an ordered neighbour list ---------------------------------------------------------------
// nb(t, p): the t-th neighbour's x y z into p, t = 0 .. kGicpK - 1 in list order. c: the covariance's lower triangle
// (0,0) (1,0) (1,1) (2,0) (2,1) (2,2) before the regularisation.
template <class Nb>
GF_HD void gicp_raw_covariance(Nb nb, float c[6]) {
    float m[3], p[3];
    nb(0, p);
    m[0] = p[0], m[1] = p[1], m[2] = p[2];
#ifdef __CUDA_ARCH__ // the neighbour list is in local memory: unrolled, this loop spills
#pragma unroll 1
#endif
    for (int t = 1; t < kGicpK; ++t) {
        nb(t, p);
        for (int a = 0; a < 3; ++a) m[a] = m[a] + p[a];
    }
    for (int a = 0; a < 3; ++a) m[a] = m[a] / (float)kGicpK;
    for (int a = 0; a < 6; ++a) c[a] = 0.f;
#ifdef __CUDA_ARCH__ // the neighbour list is in local memory: unrolled, this loop spills
#pragma unroll 1
#endif
    for (int t = 0; t < kGicpK; ++t) {
        nb(t, p);
        const float d[3] = {p[0] - m[0], p[1] - m[1], p[2] - m[2]};
        c[0] = c[0] + d[0] * d[0];
        c[1] = c[1] + d[1] * d[0];
        c[2] = c[2] + d[1] * d[1];
        c[3] = c[3] + d[2] * d[0];
        c[4] = c[4] + d[2] * d[1];
        c[5] = c[5] + d[2] * d[2];
    }
}
// PLANE: U diag(1, 1, 1e-2) V^T of the raw covariance c (as gicp_raw_covariance leaves it); out: 3x3 row-major
GF_HD void gicp_plane(const float c[6], float out[9]) {
    const float C[3][3] = {{c[0], c[1], c[3]}, {c[1], c[2], c[4]}, {c[3], c[4], c[5]}};
    float U[3][3], V[3][3], sv[3];
    rc_svd<3, float>(C, U, V, sv);
    const float v[3] = {1.f, 1.f, 1e-2f};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            out[3 * i + j] = ((U[i][0] * v[0]) * V[j][0] + (U[i][1] * v[1]) * V[j][1]) + (U[i][2] * v[2]) * V[j][2];
}

// ---- G2 / C2: the voxel key --------------------------------------------------------------------------------------
GF_HD int gicp_coord(float x, float res) { return ndt_f2i(floorf(x / res - 0.5f)); }
GF_HD bool gicp_key_of(float x, float y, float z, float res, uint64_t &key) {
    const int c[3] = {gicp_coord(x, res), gicp_coord(y, res), gicp_coord(z, res)};
    key = 0;
    for (int a = 0; a < 3; ++a) {
        if (c[a] < -kGicpCoordBias || c[a] >= kGicpCoordBias) return false;
        key = (key << kGicpCoordBits) | (uint64_t)(uint32_t)(c[a] + kGicpCoordBias);
    }
    return true;
}

// a target voxel: the ADDITIVE mean (x y z; w is 1) and covariance (3x3 row-major; row and column 3 are 0)
struct GicpVoxel {
    float mean[3];
    float cov[9];
};

// the sums of a voxel's points in input order: sm[3] and sc[9] start at 0 and take p(k) / cov(k) of each point
GF_HD void gicp_voxel_add(float sm[3], float sc[9], const float p[3], const float *cov) {
    for (int a = 0; a < 3; ++a) sm[a] = sm[a] + p[a];
    for (int a = 0; a < 9; ++a) sc[a] = sc[a] + cov[a];
}
GF_HD GicpVoxel gicp_voxel_finish(const float sm[3], const float sc[9], int n) {
    GicpVoxel v;
    const float fn = (float)n;
    for (int a = 0; a < 3; ++a) v.mean[a] = sm[a] / fn;
    for (int a = 0; a < 9; ++a) v.cov[a] = sc[a] / fn;
    return v;
}

// ---- G3: the per-point loss_ls terms -------------------------------------------------------------------------------
GF_HD float gicp_det3(float a, float b, float c, float d, float e, float f, float g, float h, float i) {
    return (a * (e * i - f * h) - b * (d * i - f * g)) + c * (d * h - e * g);
}
// out = m^-1 (4x4 row-major), C3: the adjugate times 1 / det, det along row 0 in index order
GF_HD void gicp_inv4(const float m[16], float out[16]) {
    float cof[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float s[9];
            int k = 0;
            for (int r = 0; r < 4; ++r) {
                if (r == i) continue;
                for (int c = 0; c < 4; ++c)
                    if (c != j) s[k++] = m[4 * r + c];
            }
            const float d = gicp_det3(s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7], s[8]);
            cof[4 * i + j] = ((i + j) & 1) ? -d : d;
        }
    const float det = ((m[0] * cof[0] + m[1] * cof[1]) + m[2] * cof[2]) + m[3] * cof[3];
    const float inv = 1.f / det;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) out[4 * j + i] = cof[4 * i + j] * inv;
}
// c = a b, 4x4 row-major, index-order sums
GF_HD void gicp_mul4(const float a[16], const float b[16], float c[16]) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            c[4 * i + j] = ((a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j]) + a[4 * i + 2] * b[8 + j]) + a[4 * i + 3] * b[12 + j];
}

// the terms of source point a (covariance ca, 3x3 row-major) against voxel v at the float transform T (rows 0..2):
// e[3] and J[3][6] as loss_ls writes losses[n] and Js[n]
GF_HD void gicp_point_loss(const float T[12], const float a[3], const float *ca, const GicpVoxel &v, float e[3], float J[3][6]) {
    const float Tm[16] = {T[0], T[1], T[2], T[3], T[4], T[5], T[6], T[7], T[8], T[9], T[10], T[11], 0.f, 0.f, 0.f, 1.f};
    float ta[3];
    ndt_transform(T, a[0], a[1], a[2], ta);
    const float tw = ((0.f * a[0] + 0.f * a[1]) + 0.f * a[2]) + 1.f * 1.f;
    const float CA[16] = {ca[0], ca[1], ca[2], 0.f, ca[3], ca[4], ca[5], 0.f, ca[6], ca[7], ca[8], 0.f, 0.f, 0.f, 0.f, 0.f};
    float TC[16], Tt[16], RCR[16];
    gicp_mul4(Tm, CA, TC);
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) Tt[4 * i + j] = Tm[4 * j + i];
    gicp_mul4(TC, Tt, RCR);
    RCR[15] = 1.f;
    const float CB[16] = {v.cov[0], v.cov[1], v.cov[2], 0.f, v.cov[3], v.cov[4], v.cov[5], 0.f,
                          v.cov[6], v.cov[7], v.cov[8], 0.f, 0.f,      0.f,      0.f,      0.f};
    float S[16], M[16];
    for (int k = 0; k < 16; ++k) S[k] = CB[k] + RCR[k];
    gicp_inv4(S, M);
    const float d[4] = {v.mean[0] - ta[0], v.mean[1] - ta[1], v.mean[2] - ta[2], 1.f - tw};
    for (int i = 0; i < 3; ++i) e[i] = ((M[4 * i] * d[0] + M[4 * i + 1] * d[1]) + M[4 * i + 2] * d[2]) + M[4 * i + 3] * d[3];
    const float K[16] = {0.f, -ta[2], ta[1], 0.f, ta[2], 0.f, -ta[0], 0.f, -ta[1], ta[0], 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float MK[16];
    gicp_mul4(M, K, MK);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            J[i][j] = MK[4 * i + j];
            J[i][3 + j] = -M[4 * i + j];
        }
}

// C1: one point's 28 terms from e and J (acc is added to, as a point has at most one DIRECT1 voxel)
GF_HD void gicp_point_terms(const float e[3], const float J[3][6], double acc[kGicpTerms]) {
    int k = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = 0; b <= a; ++b)
            acc[k++] += ((double)J[0][a] * (double)J[0][b] + (double)J[1][a] * (double)J[1][b]) + (double)J[2][a] * (double)J[2][b];
    for (int a = 0; a < 6; ++a)
        acc[21 + a] += ((double)J[0][a] * (double)e[0] + (double)J[1][a] * (double)e[1]) + (double)J[2][a] * (double)e[2];
    acc[27] += 1.0;
}

// ---- G4: GaussNewton<double, 6>::delta from the summed terms (host) -----------------------------------------------
inline void gicp_llt_solve(const double A[6][6], const double b[6], double x[6]) {
    double m[6][6];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) m[i][j] = A[i][j];
    for (int k = 0; k < 6; ++k) { // llt_inplace::unblocked
        double v = m[k][k];
        if (k > 0) {
            double s = m[k][0] * m[k][0];
            for (int j = 1; j < k; ++j) s += m[k][j] * m[k][j];
            v -= s;
        }
        if (v <= 0.0) break;
        m[k][k] = v = sqrt(v);
        for (int i = k + 1; i < 6; ++i) {
            if (k > 0) {
                double s = m[i][0] * m[k][0];
                for (int j = 1; j < k; ++j) s += m[i][j] * m[k][j];
                m[i][k] -= s;
            }
            m[i][k] /= v;
        }
    }
    double y[6];
    for (int i = 0; i < 6; ++i) y[i] = b[i];
    for (int i = 0; i < 6; ++i) { // L y = b
        y[i] /= m[i][i];
        for (int j = i + 1; j < 6; ++j) y[j] -= y[i] * m[j][i];
    }
    for (int i = 5; i >= 0; --i) { // L^T x = y
        double v = y[i];
        if (i < 5) {
            double s = m[i + 1][i] * x[i + 1];
            for (int j = i + 2; j < 6; ++j) s += m[j][i] * x[j];
            v -= s;
        }
        x[i] = v / m[i][i];
    }
}

// Eigen 3.3's Random() coefficient from the process's rand() (G6)
inline float gicp_randf() { return -1.f + (2.f * (float)std::rand()) / (float)RAND_MAX; }
inline double gicp_randd() { return -1.0 + (2.0 * (double)std::rand()) / (double)RAND_MAX; }

// ---- G5: SO3<float> --------------------------------------------------------------------------------------------------
constexpr float kGicpSo3Eps = 1e-5f;
struct GicpQuat {
    float w, x, y, z;
};
inline GicpQuat gicp_so3_exp(const float v[3]) {
    const float theta_sq = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2];
    const float theta = std::sqrt(theta_sq), half_theta = 0.5f * theta;
    float imag, real;
    if (theta_sq < kGicpSo3Eps * kGicpSo3Eps) {
        const float theta_po4 = theta_sq * theta_sq;
        imag = (0.5f - (float)(1.0 / 48.0) * theta_sq) + (float)(1.0 / 3840.0) * theta_po4;
        real = (1.f - (float)(1.0 / 8.0) * theta_sq) + (float)(1.0 / 384.0) * theta_po4;
    } else {
        imag = std::sin(half_theta) / theta;
        real = std::cos(half_theta);
    }
    return GicpQuat{real, imag * v[0], imag * v[1], imag * v[2]};
}
inline void gicp_so3_log(const GicpQuat &q, float out[3]) {
    const float squared_n = (q.x * q.x + q.y * q.y) + q.z * q.z, w = q.w;
    float f;
    if (squared_n < kGicpSo3Eps * kGicpSo3Eps) {
        const float squared_w = w * w;
        f = 2.f / w - ((float)(2.0 / 3.0) * squared_n) / (w * squared_w);
    } else {
        const float n = std::sqrt(squared_n);
        const float atan_nbyw = (w < 0.f) ? std::atan2(-n, -w) : std::atan2(n, w);
        f = (2.f * atan_nbyw) / n;
    }
    out[0] = f * q.x, out[1] = f * q.y, out[2] = f * q.z;
}
inline GicpQuat gicp_so3_mul(const GicpQuat &a, const GicpQuat &b) {
    GicpQuat r{((a.w * b.w - a.x * b.x) - a.y * b.y) - a.z * b.z, ((a.w * b.x + a.x * b.w) + a.y * b.z) - a.z * b.y,
               ((a.w * b.y + a.y * b.w) + a.z * b.x) - a.x * b.z, ((a.w * b.z + a.z * b.w) + a.x * b.y) - a.y * b.x};
    const float len = std::sqrt((r.x * r.x + r.z * r.z) + (r.y * r.y + r.w * r.w));
    r.x /= len, r.y /= len, r.z /= len, r.w /= len;
    return r;
}
inline void gicp_so3_matrix(const GicpQuat &q, float R[3][3]) {
    const float tx = 2.f * q.x, ty = 2.f * q.y, tz = 2.f * q.z;
    const float twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const float txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const float tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0][0] = 1.f - (tyy + tzz), R[0][1] = txy - twz, R[0][2] = txz + twy;
    R[1][0] = txy + twz, R[1][1] = 1.f - (txx + tzz), R[1][2] = tyz - twx;
    R[2][0] = txz - twy, R[2][1] = tyz + twx, R[2][2] = 1.f - (txx + tyy);
}
// [exp(x.rot) | x.t], rows 0..2 of the float 4x4
inline void gicp_transform_of(const float x[6], float T[12]) {
    float R[3][3];
    gicp_so3_matrix(gicp_so3_exp(x), R);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = R[i][j];
        T[4 * i + 3] = x[3 + i];
    }
}

// ---- G6: the walk (host) ---------------------------------------------------------------------------------------------
struct GicpIter {
    float x[6];     // rot (so3) then t, after the step
    float delta[6]; // the step (float)
    int n_corr;     // correspondences of the evaluation
    int random;     // the step was not finite and was replaced by Random() * 1e-2
};

// the 6x6 system of the summed terms: JJ (full, from the lower triangle) and J^T e
inline void gicp_system(const double r[kGicpTerms], double JJ[6][6], double Je[6]) {
    int k = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = 0; b <= a; ++b) JJ[a][b] = JJ[b][a] = r[k++];
    for (int a = 0; a < 6; ++a) Je[a] = r[21 + a];
}

inline bool gicp_converged(const float d[6]) {
    float R[3][3];
    gicp_so3_matrix(gicp_so3_exp(d), R);
    const float rs = (float)(1.0 / kGicpRotationEpsilon), ts = (float)(1.0 / kGicpTranslationEpsilon);
    float mr = rs * std::fabs(R[0][0] - 1.f);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const float v = rs * std::fabs(R[i][j] - (i == j ? 1.f : 0.f));
            if (v > mr) mr = v;
        }
    float mt = ts * std::fabs(d[3]);
    for (int i = 4; i < 6; ++i) {
        const float v = ts * std::fabs(d[i]);
        if (v > mt) mt = v;
    }
    return std::max(mr, mt) < 1.f;
}

// computeTransformation: `eval(T, r)` evaluates loss_ls at the float transform T and fills the kGicpTerms sums.
// Returns the Gauss-Newton steps taken; T_final the float transform; x0 the start point; trace (cap entries).
template <class Eval>
int gicp_walk(Eval eval, float T_final[12], float x0[6], int &converged, GicpIter *trace, int cap) {
    float x[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}; // log(SO3f(I)) = 0, the guess's translation 0
    const float nrm = std::sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
    if (nrm < 1e-2) { // always: prevent stacking at zero
        float v[3];
        for (int i = 0; i < 3; ++i) v[i] = gicp_randf();
        const float z = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2];
        for (int i = 0; i < 3; ++i) x[i] = (z > 0.f ? v[i] / std::sqrt(z) : v[i]) * 1e-2f;
    }
    for (int i = 0; i < 6; ++i) x0[i] = x[i];
    converged = 0;
    int it = 0;
    double r[kGicpTerms];
    while (it < kGicpMaxIterations) {
        float T[12];
        gicp_transform_of(x, T);
        eval(T, r);
        double JJ[6][6], Je[6], dd[6];
        gicp_system(r, JJ, Je);
        gicp_llt_solve(JJ, Je, dd);
        bool finite = true;
        for (int i = 0; i < 6; ++i) finite = finite && std::isfinite(dd[i]);
        if (!finite)
            for (int i = 0; i < 6; ++i) dd[i] = gicp_randd() * 1e-2;
        float d[6];
        for (int i = 0; i < 6; ++i) d[i] = (float)dd[i];
        const float nd[3] = {-d[0], -d[1], -d[2]};
        gicp_so3_log(gicp_so3_mul(gicp_so3_exp(nd), gicp_so3_exp(x)), x);
        for (int i = 3; i < 6; ++i) x[i] -= d[i];
        if (trace && it < cap) {
            for (int i = 0; i < 6; ++i) trace[it].x[i] = x[i], trace[it].delta[i] = d[i];
            trace[it].n_corr = (int)r[27];
            trace[it].random = finite ? 0 : 1;
        }
        ++it;
        if (gicp_converged(d)) {
            converged = 1;
            break;
        }
    }
    gicp_transform_of(x, T_final);
    return it;
}

// non-finite points take part in nothing (G7)
inline void gicp_keep_finite(std::vector<float4> &v) {
    size_t k = 0;
    for (const float4 &p : v)
        if (ndt_finite3(p.x, p.y, p.z)) v[k++] = p;
    v.resize(k);
}

} // namespace mulls
