// TEASER++ coarse registration: lo::CRegistration<PointT>::coarse_reg_teaser (cregistration.hpp:664-759), i.e.
// teaser::RobustRegistrationSolver with noise_bound, cbar2 = 1, estimate_scaling = false, GNC-TLS rotation (100
// iterations, factor 1.4, cost threshold 0.005), use_max_clique = true, kcore_heuristic_threshold = 0.5, then
// getRotationInliers().
//
// This header holds what the device path (kernels_teaser.cuh, the host side of mulls_coarse_reg_teaser) and the CPU
// restatement under tests/harness share, so that both compute the same bits. Readings of TEASER++ as published
// (master, which is what the reference's install script clones); none of them has been confirmed against a checkout:
//  T1 TIMs: v_j - v_i in double for every pair i < j, i the outer loop.
//  T2 fixed-scale pruning: a = |s_j - s_i| and b = |d_j - d_i|, each sqrt((x^2 + y^2) + z^2); the pair is an edge of
//     the consistency graph when |a - b| <= 2 * noise_bound * sqrt(cbar2) (tm_edge). A NaN compares false: no edge.
//     The scale is 1.
//  T3 maximum clique: MaxCliqueSolver in its default mode PMC_EXACT, where the k-core heuristic applies only in mode
//     KCORE_HEU: the result is a maximum clique, sorted ascending. (Older revisions applied max_core > 0.5 N without a
//     mode check and then returned the max-core vertex set; that reading is not built.) A clique of size <= 1 makes
//     the solution invalid.
//  T4 rotation TIMs: the chain graph (rotation_tim_graph's default): for clique position k, v[c_{k+1}] - v[c_k], the
//     last position wrapping to c_0.
//  T5 GNC-TLS (tm_gnc_*): the noise bound is 2 * noise_bound (solve() doubles the rotation solver's bound for TIMs;
//     the least certain reading here); noise_bound^2 < 1e-16 becomes 1e-2. Each iteration runs svdRot(src, dst, w):
//     H = X diag(w) Y^T, JacobiSVD<Matrix3d> with full U and V, V.col(2) negated when det U det V < 0, R = V U^T.
//     Residuals (dx^2 + dy^2) + dz^2. In iteration 0, mu = 1 / (2 max_r / nb^2 - 1), and mu <= 0 ends the loop. The
//     weights: 0 at r >= (mu + 1) / mu nb^2, 1 at r <= mu / (mu + 1) nb^2, else sqrt(nb^2 mu (mu + 1) / r) - mu. The
//     cost sums the previous weights times the residuals; then mu *= 1.4, and |cost - prev| < 0.005 stops. The inlier
//     mask is w >= 0.5.
//  T6 rotation inliers: the chain-TIM indices whose mask is set; MULLS compares their count with min_inlier_num.
//  T7 translation: ScalarTLSEstimator per axis over the max-clique correspondences, x = dst - R src, every range
//     noise_bound * sqrt(cbar2): 2M boundaries (x - r, +(i+1)) and (x + r, -(i+1)) sorted ascending, the running sums
//     swept with x_hat and x_cost at each boundary; the estimate is x_hat at the first index of the minimum cost.
//     (A later revision prunes the translation input by the rotation inliers; that reading is not built.)
//  T8 Eigen's product and reduction order depends on the machine. Every sum here runs in one fixed order: H and the
//     GNC cost are tm_sums order (kTmLanes strided partials in index order, then a pairwise tree, the order of
//     ransac_core.cuh C1); R src, the residuals and the norms left to right as written above; ranges.sum() and the
//     voting sweep sequentially in index order.
//  T9 where TEASER++ leaves a choice: among all maximum cliques the library returns the lexicographically smallest
//     ascending index list (PMC's multi-threaded search leaves the choice open, so this rule is the contract; where
//     the maximum clique is unique it is the reading's exact answer). Equal boundary values in the voting sort, which
//     std::sort leaves in an unspecified order, go in std::pair order: ascending signed key (tm_vote_less).
// The 3x3 SVD is ransac_core.cuh's restatement of Eigen 3.3's JacobiSVD (rc_svd3).
#pragma once
#include <cmath>
#include <cstdint>

#include "ransac_core.cuh"

namespace mulls {

constexpr int kTmLanes = kRcLanes;        // partial sums of H and the GNC cost (T8); the GNC kernel's block size
constexpr int kTmGncMaxIter = 100;
constexpr double kTmGncFactor = 1.4;
constexpr double kTmGncCostThreshold = 0.005;

// ---- T2: the pairwise consistency test of correspondences i < j; p6 holds s x y z, d x y z per correspondence -------
GF_HD double tm_tim_norm(const double *a, const double *b) {
    const double x = b[0] - a[0], y = b[1] - a[1], z = b[2] - a[2];
    return sqrt((x * x + y * y) + z * z);
}
GF_HD bool tm_edge(const double *p6, int i, int j, double beta) {
    if (i > j) {
        const int t = i;
        i = j, j = t;
    }
    const double *pi = p6 + 6 * (size_t)i, *pj = p6 + 6 * (size_t)j;
    const double a = tm_tim_norm(pi, pj), b = tm_tim_norm(pi + 3, pj + 3);
    return fabs(a - b) <= beta;
}

// ---- T8: the fixed summation order over M terms (ransac_core.cuh C1), serial form for the host -------------------------
template <int K, class Value>
inline void tm_sums_serial(int M, Value v, double out[K]) {
    rc_sums_serial<K>(M, [](int) { return true; }, v, out);
}

// ---- T5: svdRot from the 9 sums of H (row-major, H[a][b] = sum_k (x_a w_k) y_b) -------------------------------------------
GF_HD void tm_svd_rot(const double h[9], double R[9]) {
    double H[3][3], U[3][3], V[3][3];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) H[a][b] = h[3 * a + b];
    rc_svd3(H, U, V);
    if (rc_det3(U) * rc_det3(V) < 0.0)
        for (int r = 0; r < 3; ++r) V[r][2] = -V[r][2];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[3 * i + j] = (V[i][0] * U[j][0] + V[i][1] * U[j][1]) + V[i][2] * U[j][2];
}
// the 9 product terms of one TIM pair under weight w
GF_HD void tm_h_terms(const double *x, const double *y, double w, double t[9]) {
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) t[3 * a + b] = (x[a] * w) * y[b];
}
GF_HD void tm_rot_apply(const double R[9], const double *p, double out[3]) {
    for (int i = 0; i < 3; ++i) out[i] = (R[3 * i] * p[0] + R[3 * i + 1] * p[1]) + R[3 * i + 2] * p[2];
}
GF_HD double tm_residual(const double R[9], const double *x, const double *y) {
    double q[3];
    tm_rot_apply(R, x, q);
    const double dx = y[0] - q[0], dy = y[1] - q[1], dz = y[2] - q[2];
    return (dx * dx + dy * dy) + dz * dz;
}
// the squared rotation noise bound (T5); pow(x, 2) is correctly rounded, so it is x * x
GF_HD double tm_gnc_nb_sq(double noise_bound) {
    const double nb = 2.0 * noise_bound;
    const double s = nb * nb;
    return s < 1e-16 ? 1e-2 : s;
}
GF_HD double tm_gnc_mu0(double max_r, double nb_sq) { return 1.0 / (2.0 * max_r / nb_sq - 1.0); }
// the closed-form weight of one residual
GF_HD double tm_gnc_weight(double r, double mu, double nb_sq) {
    const double th1 = (mu + 1.0) / mu * nb_sq, th2 = mu / (mu + 1.0) * nb_sq;
    if (r >= th1) return 0.0;
    if (r <= th2) return 1.0;
    return sqrt(nb_sq * mu * (mu + 1.0) / r) - mu;
}

// ---- T7 / T9: the voting boundaries -------------------------------------------------------------------------------------
// a boundary: its value (-0.0 made +0.0, which `<` does not tell apart) and its signed key +-(i+1)
struct TmBound {
    double v;
    int key;
};
GF_HD bool tm_vote_less(const TmBound &a, const TmBound &b) { return a.v < b.v || (!(b.v < a.v) && a.key < b.key); }
// the sweep of ScalarTLSEstimator::estimate over the sorted boundaries: x[i] the raw measurement of correspondence i,
// every range r; m = 2M boundaries
GF_HD double tm_vote_sweep(const TmBound *h, int m, const double *x, double r) {
    const int M = m / 2;
    const double w = 1.0 / (r * r);
    double ranges_inverse_sum = 0.0;
    for (int i = 0; i < M; ++i) ranges_inverse_sum += r;
    double dot_X_weights = 0.0, dot_weights_consensus = 0.0, sum_xi = 0.0, sum_xi_square = 0.0;
    int consensus_set_cardinal = 0;
    double best_cost = 0.0, best_hat = 0.0;
    for (int i = 0; i < m; ++i) {
        const int idx = (h[i].key > 0 ? h[i].key : -h[i].key) - 1;
        const int epsilon = h[i].key > 0 ? 1 : -1;
        const double X = x[idx];
        consensus_set_cardinal += epsilon;
        dot_weights_consensus += epsilon * w;
        dot_X_weights += epsilon * w * X;
        ranges_inverse_sum -= epsilon * r;
        sum_xi += epsilon * X;
        sum_xi_square += epsilon * X * X;
        const double x_hat = dot_X_weights / dot_weights_consensus;
        const double residual = consensus_set_cardinal * x_hat * x_hat + sum_xi_square - 2 * sum_xi * x_hat;
        const double x_cost = residual + ranges_inverse_sum;
        if (i == 0 || x_cost < best_cost) best_cost = x_cost, best_hat = x_hat; // minCoeff: the first minimum
    }
    return best_hat;
}
GF_HD TmBound tm_bound(double x, double r, int i, bool upper) {
    TmBound b;
    b.v = (upper ? x + r : x - r) + 0.0;
    b.key = upper ? -(i + 1) : i + 1;
    return b;
}

} // namespace mulls
