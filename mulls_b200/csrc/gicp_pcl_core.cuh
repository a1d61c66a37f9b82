// Point-wise GICP registration: lo::CRegistration<PointT>::omp_gicp (cregistration.hpp:1024-1098) with
// using_voxel_gicp = false (test/mulls_slam.cpp:638, :675 with --voxel_gicp_on=false), i.e.
// koide_reg::GeneralizedIterativeClosestPoint (include/baseline_reg/gicp_omp.h, gicp_omp_impl.hpp) on PCL 1.10 /
// Eigen 3.3, whose solver is PCL's BFGS (pcl/registration/bfgs.h).
//
// This header holds what the device path (kernels_gicp_pcl.cuh, the host side of mulls_omp_gicp_pcl) and the CPU
// restatement under tests/harness share, so that both compute the same bits: the double covariance of an ordered
// neighbour list, the per-correspondence Mahalanobis matrix, the per-correspondence terms of the functor's three
// methods, applyState, computeRDerivative, the BFGS solver and the outer loop. The prologue, the fitness and the
// epilogue are omp_ndt's (ndt_core.cuh) and gicp_core.cuh's gicp_keep_finite, unchanged.
// Readings of the reference (gicp_omp.h / gicp_omp_impl.hpp were read, not run):
//  P1 prologue and epilogue: omp_gicp's :1035-1058 and :1080-1088 are omp_ndt's code (ndt_prologue, baseline_finish);
//     base_align calls align() without a guess, so the guess of computeTransformation is the identity and
//     final_transformation_ = previous_transformation_; fitness = getFitnessScore(), code -3 when
//     fitness > fitness_score_thre, Trans1_2 = final * initial_guess when the guess moved the source. Non-finite
//     points are dropped from both clouds (as gicp_core.cuh G7); align() sets every output point's data[3] to 1, and
//     PCL's point constructors set the target's to 1, so every homogeneous coordinate below is 1.
//  P2 constants (the constructor, gicp_omp.h:109-119): k_correspondences_ 20, gicp_epsilon_ 1e-3, rotation_epsilon_
//     2e-3, transformation_epsilon_ 5e-4, max_iterations_ 200, corr_dist_threshold_ 5.0, min 4 correspondences;
//     omp_gicp changes only max_inner_iterations_, to max_iter_num (cregistration.hpp:1070). dis_thre_unit and
//     voxel_size have no effect on this class.
//  P3 covariances (computeCovariances, :51-123): for every point of each cloud its 20 nearest neighbours in its own
//     cloud, the point itself included, in FLANN's order (ascending (squared distance, index), the order knn_search
//     gives k_gicp_cov); the mean summed in double from the float coordinates; each covariance entry (lower triangle)
//     adds the float product (pt.y * pt.x is float * float) into a double; then mean /= 20.0, cov(k, l) /= 20.0,
//     cov(k, l) -= mean[k] * mean[l]; U of JacobiSVD<Matrix3d> (rc_svd<3, double>); the result starts at zero and adds
//     (v_k U(i, k)) U(j, k) for k = 0, 1, 2 with v = (1, 1, 1e-3). All nine entries are kept: the result is not
//     symmetric to the bit.
//  P4 correspondences (computeTransformation, :406-473): transform_R = double(transformation_) double(guess) with the
//     identity guess, summed k = 0..3 from 0.0, R its upper 3x3; each source point moved by the float
//     transformation_ (ndt_transform's order); its nearest target under FLANN's float distance, ties to the lower
//     index; kept when (double)nn_dist < 25.0 (so a search bounded at radius 5 would be equivalent; the unbounded
//     search of the fitness is used); M = (R C_src R^T + C_tgt)^-1 in double (R C_src, then times R^T, then + C_tgt,
//     each product an index-order sum; the inverse as B7), stored as float. The list is sorted by source index (:468),
//     so the correspondence order is the source order.
//  P5 applyState (:520-530): AngleAxisf(x5, Z) * AngleAxisf(x4, Y) * AngleAxisf(x3, X) is a product of quaternions
//     (each cos(a / 2), sin(a / 2) axis in float), converted by toRotationMatrix; the quaternion product is Eigen
//     3.3's SSE kernel for float (x86 builds): x = (ax bw - az by) + (ay bz + aw bx), y = (ay bw - ax bz) + (az bx +
//     aw by), z = (az bw - ay bx) + (ax by + aw bz), w = (aw bw - ax bx) - (az bz + ay by). The top-left block becomes
//     R * I (index-order sums), the translation 0 + (float)x_i.
//  P6 the functor. operator() (:247-276): res = T p_src - p_tgt in float (res[3] = 0), maha res as index-order row
//     sums, res.dot(maha res) in Eigen's SSE order for four floats ((r0 m0 + r2 m2) + (r1 m1 + r3 m3)), widened to
//     double per point; f = sum / m. df (:280-331): res = (double)(pp - p_tgt) per axis, temp = double(maha) res
//     (index-order rows), the rotation part from the untransformed source point (base_transformation_ is the
//     identity: I p_src in float); g.head<3> = (0 + sum temp) * (2.0 / m), R = (0 + sum p_src temp^T) * (2.0 / m).
//     fdf (:335-368): the 3x3 block of maha in double, f adds res . temp ((r0 t0 + r1 t1) + r2 t2), then f /= m and
//     the same scaling. computeRDerivative (:127-178) writes g[3..5] = matricesInnerProd(dR, R) =
//     sum_i sum_j dR(j, i) R(i, j) in that loop order (gicp_omp.h:317-325), with double cos / sin of x[3..5].
//  P7 the outer loop (:406-512): transformation_ starts at the identity; each iteration matches, then
//     estimateRigidTransformationBFGS (:182-243) starts x from transformation_ (x0..2 its translation; x3 =
//     std::atan2(T(2,1), T(2,2)) and x5 = std::atan2(T(1,0), T(0,0)) on floats: the float overloads; x4 =
//     asin(-T(2,0)): cregistration.hpp:12 includes <math.h> ahead of gicp_omp.h, and libstdc++'s <math.h> brings
//     std::asin's float overload into the global namespace, so the unqualified call on a float is asinf, widened),
//     runs the do-while with gradient_tol 1e-2 and max_inner_iterations_, and on NoProgress, Success or the
//     inner cap sets transformation_ = applyState(I, x); otherwise it throws SolverDidntConvergeException. Fewer than
//     4 correspondences throw NotEnoughPointsException before the solver. A throw ends the loop without counting the
//     iteration (converged_ stays false; the result is previous_transformation_, which is transformation_). Else
//     delta = max over the 4x4 of ratio * |prev - new| (float difference, 1 / rotation_epsilon_ on the 3x3 block,
//     1 / transformation_epsilon_ elsewhere), nr_iterations_++, converged when nr_iterations_ >= 200 or delta < 1.
//  P8 with fewer than 20 points in either cloud after the prologue the reference prints an error, returns early and
//     later reads covariances it never computed: such a call is refused.
// Readings of code that is not in the reference tree, restated from what is published about it. These are readings,
// not confirmed against the header:
//  B1 PCL 1.10's bfgs.h is a port of GSL's vector_bfgs2 (multimin/vector_bfgs2.c, linesearch.c): Parameters default
//     bracket_iters = section_iters = 100, step_size = 1; the caller sets rho 0.01, sigma 0.01, tau1 9, tau2 0.05,
//     tau3 0.5, order 3. Status: NegativeGradientEpsilon -3, NotStarted -2, Running -1, Success 0, NoProgress 1.
//  B2 minimizeInit: one fdf at x; x0 = x, g0 = g, g0norm = |g0|, p = (g * -1) / g0norm, pnorm = |p|, fp0 = -g0norm,
//     and the alpha = 0 cache (x, f, g and the slope g . p) filled without a call.
//  B3 minimizeOneStep: NoProgress when pnorm, g0norm or fp0 is 0; alpha1 = min(1, 2 max(-delta_f, 10 eps |f0|) / -fp0)
//     once f decreased, else step_size; Fletcher's line search (B4) from alpha1; updatePosition (applyFDF at the
//     alpha found, so x, f and g come from the cache); then the BFGS update p = g - A dx0 - B dg0 with
//     B = dx0.g / dx0.dg0, A = -(1 + |dg0|^2 / dx0.dg0) B + dg0.g / dx0.dg0 (A = B = 0 when dx0.dg0 = 0); g0, x0,
//     g0norm updated; p scaled by (p.g >= 0 ? -1 : 1) / pnorm with the previous pnorm (as GSL), then pnorm = |p|,
//     fp0 = p.g0, and changeDirection resets the alpha = 0 cache. testGradient(eps) is Success when |g| < eps.
//  B4 the line search: applyFDF(0) from the cache; bracketing (at most bracket_iters): f(alpha) (applyF); above
//     f0 + alpha rho fp0 or not below the previous f: bracket [prev, alpha] with fpb = NaN; else df(alpha)
//     (applyDF, one df call unless cached); Success when |f'| <= -sigma fp0; f' >= 0: bracket [alpha, prev]; else
//     alpha_next = interpolate(prev, alpha, lower alpha + delta, upper alpha + tau1 delta). Sectioning (the same
//     counter, up to section_iters): alpha = interpolate(a, b, a + tau2 (b - a), b - tau3 (b - a)); f(alpha);
//     NoProgress when (a - alpha) fpa <= eps; above f0 + rho alpha fp0 or not below fa: b = alpha, fpb = NaN; else
//     df(alpha), Success on the sigma test, then the bracket moves as GSL's. Running out of iterations returns
//     Success with alpha 0. The caches are keyed on alpha: applyF calls operator(), applyDF calls df, applyFDF
//     calls fdf only when neither f nor df is cached at alpha (else applyF then applyDF).
//  B5 interpolate: the cubic branch is taken only when order > 2, !(fpb != fpa) and fpb != inf, i.e. when the two
//     slopes are equal (bfgs.h tests fpb against fpa where GSL tests it for NaN), so the quadratic is the usual
//     branch; its minimum is taken when the curvature c > a (bfgs.h compares with a where GSL compares with 0). The
//     cubic evaluates with Eigen::poly_eval and finds the derivative's roots with PolynomialSolver<double, 2>.
//  B6 Eigen 3.3's dot products and norms of 6 doubles on SSE2: (t0 + (t2 + t4)) + (t1 + (t3 + t5)).
//  B7 Matrix3d::inverse(): Eigen 3.3's compute_inverse_size3: cofactors m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1)
//     with i1 = i + 1, i2 = i + 2 (mod 3), det = (c00 m00 + c10 m10) + c20 m20, entry (r, c) = cof(c, r) * (1 / det).
// Choices where the reference depends on the machine or on code not in the tree:
//  C1 every method sums over the correspondences in omp_ndt's order (ndt_core.cuh C1: kNdtTile-point tiles with a
//     pairwise tree, then the tiles in order). operator() and df sum in OpenMP order in the reference, fdf serially:
//     for fdf this moves the last bits.
//  C2 the cubic branch of B5 takes the derivative's real roots in closed form (the linear root when 3 c3 is 0), not
//     from PolynomialSolver's companion-matrix eigenvalues; it is reached only when two slopes are exactly equal.
//  C3 a source point whose moved position is not finite has no correspondence (FLANN's answer is undefined there).
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>

#include "gicp_core.cuh"

namespace mulls {

constexpr double kGicpPclEpsilon = 1e-3;          // gicp_epsilon_
constexpr int kGicpPclMaxIterations = 200;        // max_iterations_
constexpr double kGicpPclRotationEpsilon = 2e-3;  // rotation_epsilon_
constexpr double kGicpPclTranslationEpsilon = 5e-4; // transformation_epsilon_
constexpr double kGicpPclCorrDist = 5.0;          // corr_dist_threshold_
constexpr int kGicpPclMinCorr = 4;                // estimateRigidTransformationBFGS's minimum
constexpr double kGicpPclGradientTol = 1e-2;
constexpr int kGicpPclMaxTerms = 13;
// the functor's methods and their per-correspondence term counts (C1)
enum GicpPclMethod { kGicpPclF = 0, kGicpPclDf = 1, kGicpPclFdf = 2 };
GF_HD constexpr int gicp_pcl_terms(int method) { return method == kGicpPclF ? 1 : method == kGicpPclDf ? 12 : 13; }
// BFGSSpace::Status (B1)
enum GicpPclStatus { kBfgsNegativeGradientEpsilon = -3, kBfgsNotStarted = -2, kBfgsRunning = -1, kBfgsSuccess = 0, kBfgsNoProgress = 1 };

// ---- P3: the covariance of an ordered neighbour list ----------------------------------------------------------------
// nb(t, p): the t-th neighbour's x y z into p. s: the sums of the neighbour list, s[0..2] the coordinates and s[3..8]
// the products of the lower triangle (0,0) (1,0) (1,1) (2,0) (2,1) (2,2). The reference adds into the mean and the
// covariance in one loop; every sum here takes its terms in the same order.
template <class Nb>
GF_HD void gicp_pcl_neighbour_sums(Nb nb, double s[9]) {
    for (int a = 0; a < 9; ++a) s[a] = 0.0;
#ifdef __CUDA_ARCH__ // the neighbour list is in local memory: unrolled, these loops spill
#pragma unroll 1
#endif
    for (int t = 0; t < kGicpK; ++t) {
        float p[3];
        nb(t, p);
        for (int a = 0; a < 3; ++a) s[a] += (double)p[a];
    }
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int t = 0; t < kGicpK; ++t) {
        float p[3];
        nb(t, p);
        s[3] += (double)(p[0] * p[0]);
        s[4] += (double)(p[1] * p[0]);
        s[5] += (double)(p[1] * p[1]);
        s[6] += (double)(p[2] * p[0]);
        s[7] += (double)(p[2] * p[1]);
        s[8] += (double)(p[2] * p[2]);
    }
}
// the covariance of the sums s (mean /= 20, cov /= 20, minus the mean products), then sum_k v_k U_k U_k^T with
// v = (1, 1, gicp_epsilon_); out: 3x3 row-major
GF_HD void gicp_pcl_plane(const double s[9], double out[9]) {
    double m[3], c[6];
    for (int a = 0; a < 3; ++a) m[a] = s[a] / (double)kGicpK;
    const int row[6] = {0, 1, 1, 2, 2, 2}, col[6] = {0, 0, 1, 0, 1, 2};
    for (int e = 0; e < 6; ++e) c[e] = s[3 + e] / (double)kGicpK - m[row[e]] * m[col[e]];
    const double C[3][3] = {{c[0], c[1], c[3]}, {c[1], c[2], c[4]}, {c[3], c[4], c[5]}};
    double U[3][3], V[3][3], sv[3];
    rc_svd<3, double>(C, U, V, sv);
    const double v[3] = {1.0, 1.0, kGicpPclEpsilon};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double t = 0.0;
            for (int k = 0; k < 3; ++k) t += (v[k] * U[i][k]) * U[j][k];
            out[3 * i + j] = t;
        }
}

// ---- P4 / B7: the Mahalanobis matrix of a correspondence ---------------------------------------------------------
GF_HD void gicp_pcl_inv3(const double m[9], double out[9]) {
    double cof[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            cof[i][j] = m[3 * i1 + j1] * m[3 * i2 + j2] - m[3 * i1 + j2] * m[3 * i2 + j1];
        }
    const double det = (cof[0][0] * m[0] + cof[1][0] * m[3]) + cof[2][0] * m[6];
    const double invdet = 1.0 / det;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) out[3 * r + c] = cof[c][r] * invdet;
}
// M = (R C1 R^T + C2)^-1 as float; R, C1, C2 3x3 row-major double
GF_HD void gicp_pcl_maha(const double R[9], const double *c1, const double *c2, float M[9]) {
    double RC[9], S[9], inv[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) RC[3 * i + j] = (R[3 * i] * c1[j] + R[3 * i + 1] * c1[3 + j]) + R[3 * i + 2] * c1[6 + j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) S[3 * i + j] = (RC[3 * i] * R[3 * j] + RC[3 * i + 1] * R[3 * j + 1]) + RC[3 * i + 2] * R[3 * j + 2];
    for (int k = 0; k < 9; ++k) S[k] += c2[k];
    gicp_pcl_inv3(S, inv);
    for (int k = 0; k < 9; ++k) M[k] = (float)inv[k];
}
// transform_R's upper 3x3 for the float transformation_ T (rows 0..2) and the identity guess
inline void gicp_pcl_transform_R(const float T[12], double R[9]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0.0;
            for (int k = 0; k < 4; ++k) s += (double)T[4 * i + k] * (k == j ? 1.0 : 0.0);
            R[3 * i + j] = s;
        }
}

// ---- P6: one correspondence's terms of each method (acc is added to) -------------------------------------------------
// T the float transform of the state (rows 0..2), a the source point, b its target, M its Mahalanobis matrix (3x3
// row-major; the 4x4's fourth row and column are zero)
GF_HD void gicp_pcl_terms_f(const float T[12], const float a[3], const float b[3], const float M[9], double *acc) {
    float pp[3];
    ndt_transform(T, a[0], a[1], a[2], pp);
    const float r[4] = {pp[0] - b[0], pp[1] - b[1], pp[2] - b[2], 0.f};
    float mr[4];
    for (int i = 0; i < 3; ++i) mr[i] = ((M[3 * i] * r[0] + M[3 * i + 1] * r[1]) + M[3 * i + 2] * r[2]) + 0.f * r[3];
    mr[3] = 0.f;
    acc[0] += (double)((r[0] * mr[0] + r[2] * mr[2]) + (r[1] * mr[1] + r[3] * mr[3]));
}
// I p_src in float: the untransformed source point as df and fdf read it
GF_HD void gicp_pcl_base_point(const float a[3], double p[3]) {
    for (int i = 0; i < 3; ++i)
        p[i] = (double)((((i == 0 ? 1.f : 0.f) * a[0] + (i == 1 ? 1.f : 0.f) * a[1]) + (i == 2 ? 1.f : 0.f) * a[2]) + 0.f * 1.f);
}
GF_HD void gicp_pcl_terms_df(const float T[12], const float a[3], const float b[3], const float M[9], double *acc) {
    float pp[3];
    ndt_transform(T, a[0], a[1], a[2], pp);
    const double r[3] = {(double)(pp[0] - b[0]), (double)(pp[1] - b[1]), (double)(pp[2] - b[2])};
    double t[3], p[3];
    for (int i = 0; i < 3; ++i)
        t[i] = (((double)M[3 * i] * r[0] + (double)M[3 * i + 1] * r[1]) + (double)M[3 * i + 2] * r[2]) + 0.0 * 0.0;
    gicp_pcl_base_point(a, p);
    for (int i = 0; i < 3; ++i) acc[i] += t[i];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) acc[3 + 3 * i + j] += p[i] * t[j];
}
GF_HD void gicp_pcl_terms_fdf(const float T[12], const float a[3], const float b[3], const float M[9], double *acc) {
    float pp[3];
    ndt_transform(T, a[0], a[1], a[2], pp);
    const double r[3] = {(double)(pp[0] - b[0]), (double)(pp[1] - b[1]), (double)(pp[2] - b[2])};
    double t[3], p[3];
    for (int i = 0; i < 3; ++i) t[i] = ((double)M[3 * i] * r[0] + (double)M[3 * i + 1] * r[1]) + (double)M[3 * i + 2] * r[2];
    gicp_pcl_base_point(a, p);
    acc[0] += (r[0] * t[0] + r[1] * t[1]) + r[2] * t[2];
    for (int i = 0; i < 3; ++i) acc[1 + i] += t[i];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) acc[4 + 3 * i + j] += p[i] * t[j];
}
template <int kMethod>
GF_HD void gicp_pcl_terms(const float T[12], const float a[3], const float b[3], const float M[9], double *acc) {
    if (kMethod == kGicpPclF) gicp_pcl_terms_f(T, a, b, M, acc);
    else if (kMethod == kGicpPclDf) gicp_pcl_terms_df(T, a, b, M, acc);
    else gicp_pcl_terms_fdf(T, a, b, M, acc);
}

// ---- P5: applyState(I, x) (host) ---------------------------------------------------------------------------------
inline GicpQuat gicp_pcl_quat_mul(const GicpQuat &a, const GicpQuat &b) { // Eigen 3.3's SSE kernel for float
    GicpQuat r;
    r.x = (a.x * b.w - a.z * b.y) + (a.y * b.z + a.w * b.x);
    r.y = (a.y * b.w - a.x * b.z) + (a.z * b.x + a.w * b.y);
    r.z = (a.z * b.w - a.y * b.x) + (a.x * b.y + a.w * b.z);
    r.w = (a.w * b.w - a.x * b.x) - (a.z * b.z + a.y * b.y);
    return r;
}
inline GicpQuat gicp_pcl_angle_axis(float angle, int axis) {
    const float ha = 0.5f * angle, s = std::sin(ha);
    const float u[3] = {axis == 0 ? 1.f : 0.f, axis == 1 ? 1.f : 0.f, axis == 2 ? 1.f : 0.f};
    return GicpQuat{std::cos(ha), s * u[0], s * u[1], s * u[2]};
}
// x: tx ty tz, then the X, Y, Z angles; T: rows 0..2 of the float 4x4
inline void gicp_pcl_apply_state(const double x[6], float T[12]) {
    const GicpQuat q = gicp_pcl_quat_mul(gicp_pcl_quat_mul(gicp_pcl_angle_axis((float)x[5], 2), gicp_pcl_angle_axis((float)x[4], 1)),
                                         gicp_pcl_angle_axis((float)x[3], 0));
    float R[3][3];
    gicp_so3_matrix(q, R);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            T[4 * i + j] = (R[i][0] * (j == 0 ? 1.f : 0.f) + R[i][1] * (j == 1 ? 1.f : 0.f)) + R[i][2] * (j == 2 ? 1.f : 0.f);
        T[4 * i + 3] = 0.f + (float)x[i];
    }
}

// ---- P6: computeRDerivative and the methods' host side ---------------------------------------------------------------
inline void gicp_pcl_r_derivative(const double x[6], const double R[9], double g[6]) {
    const double phi = x[3], theta = x[4], psi = x[5];
    const double cphi = std::cos(phi), sphi = std::sin(phi), ctheta = std::cos(theta), stheta = std::sin(theta);
    const double cpsi = std::cos(psi), spsi = std::sin(psi);
    double d[3][3][3]; // dR_dPhi, dR_dTheta, dR_dPsi, (row, col)
    d[0][0][0] = 0., d[0][1][0] = 0., d[0][2][0] = 0.;
    d[0][0][1] = sphi * spsi + cphi * cpsi * stheta;
    d[0][1][1] = -cpsi * sphi + cphi * spsi * stheta;
    d[0][2][1] = cphi * ctheta;
    d[0][0][2] = cphi * spsi - cpsi * sphi * stheta;
    d[0][1][2] = -cphi * cpsi - sphi * spsi * stheta;
    d[0][2][2] = -ctheta * sphi;
    d[1][0][0] = -cpsi * stheta;
    d[1][1][0] = -spsi * stheta;
    d[1][2][0] = -ctheta;
    d[1][0][1] = cpsi * ctheta * sphi;
    d[1][1][1] = ctheta * sphi * spsi;
    d[1][2][1] = -sphi * stheta;
    d[1][0][2] = cphi * cpsi * ctheta;
    d[1][1][2] = cphi * ctheta * spsi;
    d[1][2][2] = -cphi * stheta;
    d[2][0][0] = -ctheta * spsi;
    d[2][1][0] = cpsi * ctheta;
    d[2][2][0] = 0.;
    d[2][0][1] = -cphi * cpsi - sphi * spsi * stheta;
    d[2][1][1] = -cphi * spsi + cpsi * sphi * stheta;
    d[2][2][1] = 0.;
    d[2][0][2] = cpsi * sphi - cphi * spsi * stheta;
    d[2][1][2] = sphi * spsi + cphi * cpsi * stheta;
    d[2][2][2] = 0.;
    for (int k = 0; k < 3; ++k) { // matricesInnerProd
        double r = 0.;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) r += d[k][j][i] * R[3 * i + j];
        g[3 + k] = r;
    }
}
// the summed terms s of a method over m correspondences: f (operator(), fdf) and g (df, fdf)
inline double gicp_pcl_finish_f(const double *s, int m) { return s[0] / m; }
inline void gicp_pcl_finish_g(const double x[6], const double *s, int m, double g[6]) {
    double R[9];
    for (int i = 0; i < 3; ++i) g[i] = (0.0 + s[i]) * (2.0 / m);
    for (int k = 0; k < 9; ++k) R[k] = (0.0 + s[3 + k]) * (2.0 / m);
    gicp_pcl_r_derivative(x, R, g);
}

// ---- B1-B6: PCL's BFGS (host) ------------------------------------------------------------------------------------
inline double gicp_pcl_dot6(const double a[6], const double b[6]) {
    return (a[0] * b[0] + (a[2] * b[2] + a[4] * b[4])) + (a[1] * b[1] + (a[3] * b[3] + a[5] * b[5]));
}
inline double gicp_pcl_norm6(const double a[6]) { return std::sqrt(gicp_pcl_dot6(a, a)); }
// Eigen::poly_eval of c0 + c1 y + c2 y^2 + c3 y^3
inline double gicp_pcl_poly_eval(const double c[4], double y) {
    if (y * y <= 1.0) {
        double v = c[3];
        for (int i = 2; i >= 0; --i) v = v * y + c[i];
        return v;
    }
    double v = c[0];
    const double inv = 1.0 / y;
    for (int i = 1; i < 4; ++i) v = v * inv + c[i];
    return std::pow(y, 3.0) * v;
}

// Fn: double f(const double x[6]); void df(const double x[6], double g[6]); void fdf(const double x[6], double &f, double g[6])
template <class Fn>
struct GicpPclBfgs {
    static constexpr double rho = 0.01, sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, step_size = 1;
    static constexpr int order = 3, bracket_iters = 100, section_iters = 100;
    Fn &fn;
    double f = 0, gradient[6] = {};
    double delta_f = 0, fp0 = 0, x0[6] = {}, dx0[6] = {}, dg0[6] = {}, g0[6] = {}, dx[6] = {}, p[6] = {};
    double pnorm = 0, g0norm = 0;
    double f_alpha = 0, df_alpha = 0, x_alpha[6] = {}, g_alpha[6] = {};
    double f_cache_key = 0, df_cache_key = 0, x_cache_key = 0, g_cache_key = 0;
    explicit GicpPclBfgs(Fn &f_) : fn(f_) {}

    double slope() const { return gicp_pcl_dot6(g_alpha, p); }
    void move_to(double alpha) {
        for (int i = 0; i < 6; ++i) x_alpha[i] = x0[i] + alpha * p[i];
        x_cache_key = alpha;
    }
    double apply_f(double alpha) {
        if (alpha == f_cache_key) return f_alpha;
        move_to(alpha);
        f_alpha = fn.f(x_alpha);
        f_cache_key = alpha;
        return f_alpha;
    }
    double apply_df(double alpha) {
        if (alpha == df_cache_key) return df_alpha;
        move_to(alpha);
        if (alpha != g_cache_key) {
            fn.df(x_alpha, g_alpha);
            g_cache_key = alpha;
        }
        df_alpha = slope();
        df_cache_key = alpha;
        return df_alpha;
    }
    void apply_fdf(double alpha, double &fo, double &dfo) {
        if (alpha == f_cache_key && alpha == df_cache_key) {
            fo = f_alpha, dfo = df_alpha;
            return;
        }
        if (alpha == f_cache_key || alpha == df_cache_key) {
            fo = apply_f(alpha);
            dfo = apply_df(alpha);
            return;
        }
        move_to(alpha);
        fn.fdf(x_alpha, f_alpha, g_alpha);
        f_cache_key = g_cache_key = alpha;
        df_alpha = slope();
        df_cache_key = alpha;
        fo = f_alpha, dfo = df_alpha;
    }
    void change_direction() {
        for (int i = 0; i < 6; ++i) x_alpha[i] = x0[i], g_alpha[i] = g0[i];
        x_cache_key = f_cache_key = g_cache_key = 0.0;
        df_alpha = slope();
        df_cache_key = 0.0;
    }

    int minimize_init(const double x[6]) {
        delta_f = 0;
        for (int i = 0; i < 6; ++i) dx[i] = 0;
        fn.fdf(x, f, gradient);
        for (int i = 0; i < 6; ++i) x0[i] = x[i], g0[i] = gradient[i];
        g0norm = gicp_pcl_norm6(g0);
        for (int i = 0; i < 6; ++i) p[i] = gradient[i] * -1 / g0norm;
        pnorm = gicp_pcl_norm6(p);
        fp0 = -g0norm;
        for (int i = 0; i < 6; ++i) x_alpha[i] = x0[i], g_alpha[i] = g0[i];
        x_cache_key = 0, f_alpha = f, f_cache_key = 0, g_cache_key = 0;
        df_alpha = slope(), df_cache_key = 0;
        return kBfgsNotStarted;
    }

    double interpolate(double a, double fa, double fpa, double b, double fb, double fpb, double xmin, double xmax) const {
        double ymin = (xmin - a) / (b - a), ymax = (xmax - a) / (b - a), y, fmin;
        if (ymin > ymax) std::swap(ymin, ymax);
        if (order > 2 && !(fpb != fpa) && fpb != INFINITY) { // B5: the cubic
            fpa = fpa * (b - a);
            fpb = fpb * (b - a);
            const double eta = 3 * (fb - fa) - 2 * fpa - fpb, xi = fpa + fpb - 2 * (fb - fa);
            const double c[4] = {fa, fpa, eta, xi};
            auto check = [&](double yy) {
                const double v = gicp_pcl_poly_eval(c, yy);
                if (v < fmin) y = yy, fmin = v;
            };
            y = ymin;
            fmin = gicp_pcl_poly_eval(c, ymin);
            check(ymax);
            const double q0 = c[1], q1 = 2 * c[2], q2 = 3 * c[3]; // C2: the roots of q0 + q1 y + q2 y^2
            double r[2];
            int nr = 0;
            if (q2 != 0) {
                const double disc = q1 * q1 - 4 * q2 * q0;
                if (disc >= 0) {
                    const double sq = std::sqrt(disc);
                    r[0] = (-q1 - sq) / (2 * q2), r[1] = (-q1 + sq) / (2 * q2), nr = 2;
                    if (r[0] > r[1]) std::swap(r[0], r[1]);
                }
            } else if (q1 != 0) {
                r[0] = -q0 / q1, nr = 1;
            }
            for (int k = 0; k < nr; ++k)
                if (r[k] > ymin && r[k] < ymax) check(r[k]);
        } else { // the quadratic
            fpa = fpa * (b - a);
            const double fl = fa + ymin * (fpa + ymin * (fb - fa - fpa));
            const double fh = fa + ymax * (fpa + ymax * (fb - fa - fpa));
            const double c = 2 * (fb - fa - fpa);
            y = ymin, fmin = fl;
            if (fh < fmin) y = ymax, fmin = fh;
            if (c > a) {
                const double z = -fpa / c;
                if (z > ymin && z < ymax) {
                    const double fz = fa + z * (fpa + z * (fb - fa - fpa));
                    if (fz < fmin) y = z, fmin = fz;
                }
            }
        }
        return a + y * (b - a);
    }

    int line_search(double alpha1, double &alpha_new) {
        double f0, fp0l, falpha, falpha_prev, fpalpha, fpalpha_prev, delta, alpha_next;
        double alpha = alpha1, alpha_prev = 0.0;
        double a, b, fa, fb, fpa, fpb;
        int i = 0;
        apply_fdf(0.0, f0, fp0l);
        falpha_prev = f0, fpalpha_prev = fp0l;
        a = 0.0, b = alpha, fa = f0, fb = 0.0, fpa = fp0l, fpb = 0.0;
        while (i++ < bracket_iters) {
            falpha = apply_f(alpha);
            if (falpha > f0 + alpha * rho * fp0l || falpha >= falpha_prev) {
                a = alpha_prev, fa = falpha_prev, fpa = fpalpha_prev;
                b = alpha, fb = falpha, fpb = NAN;
                break;
            }
            fpalpha = apply_df(alpha);
            if (std::fabs(fpalpha) <= -sigma * fp0l) {
                alpha_new = alpha;
                return kBfgsSuccess;
            }
            if (fpalpha >= 0) {
                a = alpha, fa = falpha, fpa = fpalpha;
                b = alpha_prev, fb = falpha_prev, fpb = fpalpha_prev;
                break;
            }
            delta = alpha - alpha_prev;
            alpha_next = interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha, alpha + delta, alpha + tau1 * delta);
            alpha_prev = alpha, falpha_prev = falpha, fpalpha_prev = fpalpha;
            alpha = alpha_next;
        }
        while (i++ < section_iters) {
            delta = b - a;
            alpha = interpolate(a, fa, fpa, b, fb, fpb, a + tau2 * delta, b - tau3 * delta);
            falpha = apply_f(alpha);
            if ((a - alpha) * fpa <= DBL_EPSILON) return kBfgsNoProgress;
            if (falpha > f0 + rho * alpha * fp0l || falpha >= fa) {
                b = alpha, fb = falpha, fpb = NAN;
            } else {
                fpalpha = apply_df(alpha);
                if (std::fabs(fpalpha) <= -sigma * fp0l) {
                    alpha_new = alpha;
                    return kBfgsSuccess;
                }
                if (((b - a) >= 0 && fpalpha >= 0) || ((b - a) <= 0 && fpalpha <= 0)) {
                    b = a, fb = fa, fpb = fpa;
                    a = alpha, fa = falpha, fpa = fpalpha;
                } else {
                    a = alpha, fa = falpha, fpa = fpalpha;
                }
            }
        }
        return kBfgsSuccess;
    }

    int minimize_one_step(double x[6]) {
        double alpha = 0.0, alpha1;
        const double f0 = f;
        if (pnorm == 0.0 || g0norm == 0.0 || fp0 == 0) {
            for (int i = 0; i < 6; ++i) dx[i] = 0;
            return kBfgsNoProgress;
        }
        if (delta_f < 0) {
            const double del = std::max(-delta_f, 10 * DBL_EPSILON * std::fabs(f0));
            alpha1 = std::min(1.0, 2.0 * del / (-fp0));
        } else {
            alpha1 = std::fabs(step_size);
        }
        const int status = line_search(alpha1, alpha);
        if (status != kBfgsSuccess) return status;
        { // updatePosition
            double fo, dfo;
            apply_fdf(alpha, fo, dfo);
            f = f_alpha;
            for (int i = 0; i < 6; ++i) x[i] = x_alpha[i], gradient[i] = g_alpha[i];
        }
        delta_f = f - f0;
        for (int i = 0; i < 6; ++i) dx0[i] = x[i] - x0[i], dx[i] = dx0[i], dg0[i] = gradient[i] - g0[i];
        const double dxg = gicp_pcl_dot6(dx0, gradient), dgg = gicp_pcl_dot6(dg0, gradient), dxdg = gicp_pcl_dot6(dx0, dg0);
        const double dgnorm = gicp_pcl_norm6(dg0);
        double A = 0, B = 0;
        if (dxdg != 0) {
            B = dxg / dxdg;
            A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg;
        }
        for (int i = 0; i < 6; ++i) p[i] = gradient[i] - A * dx0[i] - B * dg0[i];
        for (int i = 0; i < 6; ++i) g0[i] = gradient[i], x0[i] = x[i];
        g0norm = gicp_pcl_norm6(g0);
        const double pg = gicp_pcl_dot6(gradient, p), dir = (pg >= 0.0) ? -1.0 : 1.0;
        for (int i = 0; i < 6; ++i) p[i] *= dir / pnorm;
        pnorm = gicp_pcl_norm6(p);
        fp0 = gicp_pcl_dot6(p, g0);
        change_direction();
        return kBfgsSuccess;
    }

    int test_gradient(double epsilon) const {
        if (epsilon < 0) return kBfgsNegativeGradientEpsilon;
        return gicp_pcl_norm6(gradient) < epsilon ? kBfgsSuccess : kBfgsRunning;
    }
};

// ---- P7: the outer loop (host) ------------------------------------------------------------------------------------
struct GicpPclIter {
    double x[6];     // the solver's state after the solve: tx ty tz, X Y Z angles
    double delta;    // the max-ratio change of the transformation
    int n_corr;      // correspondences
    int inner;       // BFGS steps taken (inner_iterations_)
    int status;      // the BFGSSpace status the do-while ended on
    int evaluations; // functor calls (operator(), df, fdf)
};

// computeTransformation. `match(T, R)` finds the correspondences of the float transformation_ T (rows 0..2) with
// transform_R's block R (double 3x3) and returns their count m; `eval(method, T, r)` sums the method's terms
// (gicp_pcl_terms) over them at the float transform T into r. Returns nr_iterations_; T_final the float transform;
// converged; trace (cap entries) one row per counted iteration.
template <class Match, class Eval>
int gicp_pcl_walk(int max_inner, Match match, Eval eval, float T_final[12], int &converged, GicpPclIter *trace, int cap) {
    float T[12] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f};
    converged = 0;
    int nr = 0;
    while (!converged) {
        double R[9];
        gicp_pcl_transform_R(T, R);
        const int m = match(T, R);
        if (m < kGicpPclMinCorr) break; // NotEnoughPointsException
        double x[6] = {(double)T[3], (double)T[7], (double)T[11], (double)std::atan2(T[9], T[10]), (double)std::asin(-T[8]),
                       (double)std::atan2(T[4], T[0])};
        struct Fn {
            Eval &eval;
            int m, calls;
            double f(const double *x) {
                float Tx[12];
                double s[kGicpPclMaxTerms];
                gicp_pcl_apply_state(x, Tx);
                eval(kGicpPclF, Tx, s);
                ++calls;
                return gicp_pcl_finish_f(s, m);
            }
            void df(const double *x, double *g) {
                float Tx[12];
                double s[kGicpPclMaxTerms];
                gicp_pcl_apply_state(x, Tx);
                eval(kGicpPclDf, Tx, s);
                ++calls;
                gicp_pcl_finish_g(x, s, m, g);
            }
            void fdf(const double *x, double &fo, double *g) {
                float Tx[12];
                double s[kGicpPclMaxTerms];
                gicp_pcl_apply_state(x, Tx);
                eval(kGicpPclFdf, Tx, s);
                ++calls;
                fo = gicp_pcl_finish_f(s, m);
                gicp_pcl_finish_g(x, s + 1, m, g);
            }
        } fn{eval, m, 0};
        GicpPclBfgs<Fn> bfgs(fn);
        int inner = 0;
        int result = bfgs.minimize_init(x);
        result = kBfgsRunning;
        do {
            ++inner;
            result = bfgs.minimize_one_step(x);
            if (result) break;
            result = bfgs.test_gradient(kGicpPclGradientTol);
        } while (result == kBfgsRunning && inner < max_inner);
        if (!(result == kBfgsNoProgress || result == kBfgsSuccess || inner == max_inner)) break; // SolverDidntConverge
        float Tn[12];
        gicp_pcl_apply_state(x, Tn);
        double delta = 0.;
        for (int k = 0; k < 4; ++k)
            for (int l = 0; l < 4; ++l) {
                const double ratio = (k < 3 && l < 3) ? 1. / kGicpPclRotationEpsilon : 1. / kGicpPclTranslationEpsilon;
                const float pv = k < 3 ? T[4 * k + l] : (l == 3 ? 1.f : 0.f), nv = k < 3 ? Tn[4 * k + l] : (l == 3 ? 1.f : 0.f);
                const double c_delta = ratio * std::fabs(pv - nv);
                if (c_delta > delta) delta = c_delta;
            }
        for (int k = 0; k < 12; ++k) T[k] = Tn[k];
        if (trace && nr < cap) {
            GicpPclIter &t = trace[nr];
            for (int i = 0; i < 6; ++i) t.x[i] = x[i];
            t.delta = delta, t.n_corr = m, t.inner = inner, t.status = result, t.evaluations = fn.calls;
        }
        ++nr;
        if (nr >= kGicpPclMaxIterations || delta < 1) converged = 1;
    }
    for (int k = 0; k < 12; ++k) T_final[k] = T[k];
    return nr;
}

} // namespace mulls
