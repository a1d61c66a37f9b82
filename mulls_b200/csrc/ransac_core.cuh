// RANSAC coarse registration: lo::CRegistration<PointT>::coarse_reg_ransac (cregistration.hpp:604-661), i.e.
// pcl::registration::CorrespondenceRejectorSampleConsensus over the correspondences i <-> i with
// pcl::SampleConsensusModelRegistration, pcl::RandomSampleConsensus and SampleConsensus::refineModel (PCL 1.10).
//
// This header holds the pieces the device path (kernels_ransac.cuh, the host side of mulls_coarse_reg_ransac) and the CPU
// restatement under tests/harness share, so that both compute the same bits: the sample stream, the
// Umeyama fit with its 3x3 Jacobi SVD, the float transform-and-compare, the fixed summation order of the fits and the
// adaptive-k walk. Readings of PCL 1.10 / Eigen 3.3 restated here (verify against a PCL checkout, as SURVEY Appendix B):
//  R1 model set-up: SampleConsensusModelRegistration(source, indices 0..N-1) computes the sample distance threshold from
//     the float mean and covariance of the N source points (computeMeanAndCovarianceMatrix, dense cloud: every point,
//     NaN included), pcl::eigen33's eigenvalues, thr = (double)((sqrt(l0) + sqrt(l1)) + sqrt(l2)) / 3.0, squared in
//     double;
//  R2 sampling: every model object seeds its boost::mt19937 with 12345u; drawIndexSample swaps shuffled_indices_[i] with
//     shuffled_indices_[i + rnd() % (N - i)], i = 0, 1, 2, rnd() = mt() >> 1, on the model's persistent shuffle;
//     isSampleGood wants all three pairwise squared source distances, summed (x^2 + y^2) + z^2 in float, > thr; a
//     selection gets up to 1000 attempts and is empty afterwards (N < 3: empty at once);
//  R3 hypothesis: estimateRigidTransformationSVD = pcl::umeyama(src, tgt, false) in double (means, sigma = (1/n) D S^T,
//     Eigen's two-sided JacobiSVD of the 3x3, S = diag(1, 1, det(U) det(V) < 0 ? -1 : 1), R = U S V^T,
//     t = mean_tgt - R mean_src), cast to a float 4x4 (bottom row 0 0 0 1);
//  R4 counting: p_tr = T [p, 1] in float, ((m_i0 x + m_i1 y) + m_i2 z) + m_i3, squared norm (dx^2 + dz^2) + dy^2 (Eigen
//     3.3's SSE2 order; the fourth component is 0 for finite points and the test fails for non-finite ones either way),
//     widened and compared with `< threshold * threshold` in double; selectWithinDistance keeps the squared errors;
//  R5 search loop: RandomSampleConsensus::computeModel, p = 0.99, a strict > replaces the best model,
//     k = log(0.01) / log(clamp(1 - w^3)), at most max_iterations + 1 hypotheses; max_skip = max_iterations * 10 as
//     unsigned (0 for max_iterations == 0: no hypothesis at all);
//  R6 refinement: SampleConsensus::refineModel(sigma 3, 1000 rounds), the loop as written (k_ransac_refine in kernels_ransac.cuh).
// Choices where the reference's result depends on the machine (Eigen's blocked dynamic-size products):
//  C1 every sum of a fit runs in the order rc_sums_serial defines: kRcLanes strided partials in index order, then a
//     pairwise tree; the 3-point hypothesis fits use it with M = 3, the refinement fits over the flagged correspondences;
//  C2 the SVD stops after kRcSvdSweeps sweeps (Eigen has no cap; a NaN ends its loop through failed comparisons);
//     Eigen's maxCoeff with a NaN entry is left open by Eigen: here a NaN does not raise the scale.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "ground_core.cuh"

namespace mulls {

constexpr int kRcLanes = 256;      // partial sums of a fit (C1); also the refinement kernel's block size
constexpr int kRcSvdSweeps = 64;   // sweep cap of the 3x3 Jacobi SVD (C2)
constexpr int kRcMaxSampleChecks = 1000;
constexpr int kRcRefineRounds = 1000;
constexpr double kRcRefineSigma = 3.0;

// ---- boost::mt19937 seeded with 12345u: the sample stream of every pcl::SampleConsensusModel object (R2) ---------------
// boost::mt19937 == std::mt19937; written out to stay free of <random> implementation questions. Host only.
struct SacMt19937 {
    uint32_t mt[624];
    int idx;
    explicit SacMt19937(uint32_t seed = 12345u) {
        mt[0] = seed;
        for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
        idx = 624;
    }
    uint32_t next() {
        if (idx >= 624) {
            for (int i = 0; i < 624; ++i) {
                const uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
                mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            idx = 0;
        }
        uint32_t y = mt[idx++];
        y ^= y >> 11;
        y ^= (y << 7) & 0x9d2c5680u;
        y ^= (y << 15) & 0xefc60000u;
        y ^= y >> 18;
        return y;
    }
};

// ---- R1: the sample distance threshold over the first n source rows (48-byte rows, x y z at floats 0..2). Host only. -----
inline double rc_sample_dist_threshold(const float *rows48, size_t n) {
    float accu[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (size_t i = 0; i < n; ++i) gf_mean_cov_add(accu, rows48[12 * i], rows48[12 * i + 1], rows48[12 * i + 2]);
    float cov[3][3], ev[3];
    gf_mean_cov_finish(accu, (float)n, cov);
    gf_eigen33_values(cov, ev);
    const double t = (double)((sqrtf(ev[0]) + sqrtf(ev[1])) + sqrtf(ev[2])) / 3.0;
    return t * t;
}

// ---- R2: getSamples on the model's persistent shuffle. Host only. -----------------------------------------------------
struct SacSampler {
    SacMt19937 rng;
    int *shuf;            // shuffled_indices_, n entries, 0..n-1 at the start
    size_t n;
    const float *rows48;  // source rows
    double thr;
    // false: the selection is empty (n < 3, or 1000 attempts without a good sample)
    bool draw(int s[3]) {
        if (n < 3) return false;
        for (int iter = 0; iter < kRcMaxSampleChecks; ++iter) {
            for (size_t i = 0; i < 3; ++i) {
                const size_t o = i + (size_t)(rng.next() >> 1) % (n - i);
                const int t = shuf[i];
                shuf[i] = shuf[o];
                shuf[o] = t;
            }
            s[0] = shuf[0], s[1] = shuf[1], s[2] = shuf[2];
            const float *p0 = rows48 + 12 * (size_t)s[0], *p1 = rows48 + 12 * (size_t)s[1], *p2 = rows48 + 12 * (size_t)s[2];
            if (sq(p1, p0) > thr && sq(p2, p0) > thr && sq(p2, p1) > thr) return true;
        }
        return false;
    }
    static double sq(const float *a, const float *b) {
        const float x = a[0] - b[0], y = a[1] - b[1], z = a[2] - b[2];
        return (double)((x * x + y * y) + z * z);
    }
};

// ---- R5: the adaptive-k walk of RandomSampleConsensus::computeModel, fed one hypothesis count at a time. Host only. ------
struct SacWalk {
    int iterations = 0, n_best = -INT_MAX, best = -1, max_iterations;
    unsigned skipped = 0, max_skip;
    double k = 1.0, log_probability, one_over_indices;
    bool stopped = false;
    SacWalk(size_t n, int max_iter)
        : max_iterations(max_iter), max_skip((unsigned)max_iter * 10u), log_probability(log(1.0 - 0.99)),
          one_over_indices(1.0 / (double)n) {}
    // the loop condition, evaluated before a sample is drawn
    bool wants() const { return !stopped && (double)iterations < k && skipped < max_skip; }
    void take(int cnt) {
        if (cnt > n_best) {
            n_best = cnt;
            best = iterations;
            const double w = (double)n_best * one_over_indices;
            double p_no_outliers = 1.0 - pow(w, 3.0);
            p_no_outliers = (DBL_EPSILON < p_no_outliers) ? p_no_outliers : DBL_EPSILON;              // std::max
            p_no_outliers = (p_no_outliers < 1.0 - DBL_EPSILON) ? p_no_outliers : 1.0 - DBL_EPSILON;  // std::min
            k = log_probability / log(p_no_outliers);
        }
        ++iterations;
        if (iterations > max_iterations) stopped = true;
    }
};

// ---- C1: the fixed summation order -------------------------------------------------------------------------------------
// sum over j in [0, M) of v(j) for the members: partial[t] = 0.0 + v(t) + v(t + L) + ... (members only, index order),
// L = kRcLanes; then for s = L/2 .. 1: partial[t] += partial[t + s] for t < s with t + s < min(M, L). Serial form
// (the refinement kernel runs the same order with one lane per partial).
// m = min(M, kRcLanes) partials in q
template <int K, class Member, class Value>
GF_HD void rc_sums_range(int M, int m, Member in, Value v, double (*q)[K], double out[K]) {
    for (int t = 0; t < m; ++t) {
        for (int c = 0; c < K; ++c) q[t][c] = 0.0;
        for (int j = t; j < M; j += kRcLanes)
            if (in(j)) {
                double x[K];
                v(j, x);
                for (int c = 0; c < K; ++c) q[t][c] += x[c];
            }
    }
    for (int s = kRcLanes / 2; s > 0; s >>= 1)
        for (int t = 0; t < s && t + s < m; ++t)
            for (int c = 0; c < K; ++c) q[t][c] += q[t + s][c];
    for (int c = 0; c < K; ++c) out[c] = m > 0 ? q[0][c] : 0.0;
}
// any M; host only (the restatement's refinement fits: the refinement kernel runs the same order with one lane per partial)
template <int K, class Member, class Value>
inline void rc_sums_serial(int M, Member in, Value v, double out[K]) {
    static thread_local double q[kRcLanes][K];
    rc_sums_range<K>(M, M < kRcLanes ? M : kRcLanes, in, v, q, out);
}

// ---- R3: Eigen 3.3's JacobiSVD of a 3x3 double (ComputeFullU | ComputeFullV) ----------------------------------------------
// the limits of JacobiSVD's scalar (R3)
template <class T> struct rc_lim;
template <> struct rc_lim<double> {
    GF_HD static double min() { return DBL_MIN; }
    GF_HD static double eps() { return DBL_EPSILON; }
};
template <> struct rc_lim<float> {
    GF_HD static float min() { return FLT_MIN; }
    GF_HD static float eps() { return FLT_EPSILON; }
};
template <int N, class T = double>
GF_HD void rc_rot_rows(T (*A)[N], int p, int q, T c, T s) { // A.applyOnTheLeft(p, q, J(c, s))
    if (c == T(1) && s == T(0)) return;
    for (int i = 0; i < N; ++i) {
        const T x = A[p][i], y = A[q][i];
        A[p][i] = c * x + s * y;
        A[q][i] = -s * x + c * y;
    }
}
template <int N, class T = double>
GF_HD void rc_rot_cols(T (*A)[N], int p, int q, T c, T s) { // apply_rotation_in_the_plane(col p, col q, J(c, s))
    if (c == T(1) && s == T(0)) return;
    for (int i = 0; i < N; ++i) {
        const T x = A[i][p], y = A[i][q];
        A[i][p] = c * x + s * y;
        A[i][q] = -s * x + c * y;
    }
}
GF_HD double rc_det3(const double m[3][3]) {
    return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}
// Eigen 3.3's two-sided JacobiSVD of a square N x N matrix of T = double or float (no QR preconditioner for a square
// matrix): JacobiSVD<Matrix<T, N, N>> is one template over the scalar, with its limits (considerAsZero = min(),
// precision = 2 epsilon()) and every operation in T. sv: the singular values, descending; the return value is
// m_nonzeroSingularValues (the sort stops at the first zero maximum).
template <int N, class T = double>
GF_HD int rc_svd(const T (*A)[N], T (*U)[N], T (*V)[N], T sv[N]) {
    T scale = T(0);
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j)
            if (fabs(A[i][j]) > scale) scale = fabs(A[i][j]);
    if (scale == T(0)) scale = T(1);
    T W[N][N];
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) {
            W[i][j] = A[i][j] / scale;
            U[i][j] = V[i][j] = (i == j) ? T(1) : T(0);
        }
    const T considerAsZero = rc_lim<T>::min(), precision = T(2) * rc_lim<T>::eps();
    T maxDiag = fabs(W[0][0]);
    for (int i = 1; i < N; ++i)
        if (maxDiag < fabs(W[i][i])) maxDiag = fabs(W[i][i]);
    bool finished = false;
    for (int sweep = 0; !finished && sweep < kRcSvdSweeps; ++sweep) {
        finished = true;
        for (int p = 1; p < N; ++p)
            for (int q = 0; q < p; ++q) {
                const T threshold = (considerAsZero < precision * maxDiag) ? precision * maxDiag : considerAsZero;
                if (!(fabs(W[p][q]) > threshold || fabs(W[q][p]) > threshold)) continue;
                finished = false;
                // real_2x2_jacobi_svd
                T m00 = W[p][p], m01 = W[p][q], m10 = W[q][p], m11 = W[q][q];
                T c1 = T(1), s1 = T(0);
                const T t = m00 + m11, d = m10 - m01;
                if (!(fabs(d) < rc_lim<T>::min())) {
                    const T u = t / d, tmp = sqrt(T(1) + u * u);
                    s1 = T(1) / tmp;
                    c1 = u / tmp;
                }
                if (!(c1 == T(1) && s1 == T(0))) {
                    const T a0 = c1 * m00 + s1 * m10, a1 = c1 * m01 + s1 * m11;
                    const T b0 = -s1 * m00 + c1 * m10, b1 = -s1 * m01 + c1 * m11;
                    m00 = a0, m01 = a1, m10 = b0, m11 = b1;
                }
                (void)m10;
                // j_right.makeJacobi(m00, m01, m11)
                T cr = T(1), sr = T(0);
                const T deno = T(2) * fabs(m01);
                if (!(deno < rc_lim<T>::min())) {
                    const T tau = (m00 - m11) / deno, w = sqrt(tau * tau + T(1));
                    const T tt = (tau > T(0)) ? T(1) / (tau + w) : T(1) / (tau - w);
                    const T sign_t = tt > T(0) ? T(1) : -T(1);
                    const T n = T(1) / sqrt(tt * tt + T(1));
                    sr = ((-sign_t * (m01 / fabs(m01))) * fabs(tt)) * n;
                    cr = n;
                }
                // j_left = rot1 * j_right.transpose(), j_right.transpose() = (cr, -sr)
                const T cl = c1 * cr - s1 * -sr, sl = c1 * -sr + s1 * cr;
                rc_rot_rows<N, T>(W, p, q, cl, sl);   // m_workMatrix.applyOnTheLeft(p, q, j_left)
                rc_rot_cols<N, T>(U, p, q, cl, sl);   // m_matrixU.applyOnTheRight(p, q, j_left.transpose())
                rc_rot_cols<N, T>(W, p, q, cr, -sr);  // m_workMatrix.applyOnTheRight(p, q, j_right)
                rc_rot_cols<N, T>(V, p, q, cr, -sr);  // m_matrixV.applyOnTheRight(p, q, j_right)
                const T dp = fabs(W[p][p]), dq = fabs(W[q][q]);
                const T dm = (dp < dq) ? dq : dp;
                if (maxDiag < dm) maxDiag = dm;
            }
    }
    for (int i = 0; i < N; ++i) {
        const T a = W[i][i];
        sv[i] = fabs(a);
        if (a < T(0))
            for (int r = 0; r < N; ++r) U[r][i] = -U[r][i];
    }
    for (int i = 0; i < N; ++i) sv[i] *= scale;
    int nonzero = N;
    for (int i = 0; i < N; ++i) { // descending, the first maximum of the tail
        int pos = i;
        for (int j = i + 1; j < N; ++j)
            if (sv[j] > sv[pos]) pos = j;
        if (sv[pos] == T(0)) {
            nonzero = i;
            break;
        }
        if (pos != i) {
            const T ts = sv[i];
            sv[i] = sv[pos], sv[pos] = ts;
            for (int r = 0; r < N; ++r) {
                T x = U[r][i];
                U[r][i] = U[r][pos], U[r][pos] = x;
                x = V[r][i];
                V[r][i] = V[r][pos], V[r][pos] = x;
            }
        }
    }
    return nonzero;
}
GF_HD void rc_svd3(const double A[3][3], double U[3][3], double V[3][3]) {
    double sv[3];
    rc_svd<3>(A, U, V, sv);
}

// the Umeyama fit from the fixed-order sums: ms[6] = sums of (sx sy sz tx ty tz), cs[9] = sums of
// (t_i - mean_t_i) (s_j - mean_s_j) row-major (i target, j source); T: rows 0..2 of the float 4x4
GF_HD void rc_umeyama_means(const double ms[6], double one_over_n, double mean[6]) {
    for (int c = 0; c < 6; ++c) mean[c] = ms[c] * one_over_n;
}
GF_HD void rc_umeyama_finish(const double mean[6], const double cs[9], double one_over_n, float T[12]) {
    double sigma[3][3], U[3][3], V[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) sigma[i][j] = one_over_n * cs[3 * i + j];
    rc_svd3(sigma, U, V);
    const double S2 = (rc_det3(U) * rc_det3(V) < 0.0) ? -1.0 : 1.0;
    double R[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = (U[i][0] * V[j][0] + U[i][1] * V[j][1]) + (U[i][2] * S2) * V[j][2];
    for (int i = 0; i < 3; ++i) {
        const double tr = mean[3 + i] - ((R[i][0] * mean[0] + R[i][1] * mean[1]) + R[i][2] * mean[2]);
        T[4 * i + 0] = (float)R[i][0], T[4 * i + 1] = (float)R[i][1], T[4 * i + 2] = (float)R[i][2], T[4 * i + 3] = (float)tr;
    }
}
// the product terms of one correspondence for the second pass
GF_HD void rc_cross_terms(const float *c6, const double mean[6], double x[9]) {
    const double s0 = (double)c6[0] - mean[0], s1 = (double)c6[1] - mean[1], s2 = (double)c6[2] - mean[2];
    const double t0 = (double)c6[3] - mean[3], t1 = (double)c6[4] - mean[4], t2 = (double)c6[5] - mean[5];
    x[0] = t0 * s0, x[1] = t0 * s1, x[2] = t0 * s2, x[3] = t1 * s0, x[4] = t1 * s1, x[5] = t1 * s2, x[6] = t2 * s0,
    x[7] = t2 * s1, x[8] = t2 * s2;
}
GF_HD void rc_point_terms(const float *c6, double x[6]) {
    for (int c = 0; c < 6; ++c) x[c] = (double)c6[c];
}

// the hypothesis of a sample (R3, C1 with M = 3): corr holds 6 floats per correspondence (sx sy sz tx ty tz)
GF_HD void rc_fit_sample(const float *corr, const int s[3], float T[12]) {
    double ms[6], mean[6], cs[9], q6[3][6], q9[3][9];
    auto in = [](int) { return true; };
    rc_sums_range<6>(3, 3, in, [&](int j, double x[6]) { rc_point_terms(corr + 6 * (size_t)s[j], x); }, q6, ms);
    const double one_over_n = 1.0 / 3.0;
    rc_umeyama_means(ms, one_over_n, mean);
    rc_sums_range<9>(3, 3, in, [&](int j, double x[9]) { rc_cross_terms(corr + 6 * (size_t)s[j], mean, x); }, q9, cs);
    rc_umeyama_finish(mean, cs, one_over_n, T);
}

// ---- R4: the squared error of one correspondence under a float transform ----------------------------------------------
GF_HD float rc_sq_error(const float T[12], const float *c6) {
    const float x = c6[0], y = c6[1], z = c6[2];
    const float px = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
    const float py = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
    const float pz = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
    const float dx = px - c6[3], dy = py - c6[4], dz = pz - c6[5];
    return (dx * dx + dz * dz) + dy * dy;
}
GF_HD bool rc_within(const float T[12], const float *c6, double thresh_sq) { return (double)rc_sq_error(T, c6) < thresh_sq; }

// the refinement's threshold update: sqrt(std::min(inlier_distance_threshold_sqr, sigma^2 * variance)),
// variance = 2.1981 * median of the squared errors
GF_HD double rc_next_threshold(double thr_sqr0, float median_err) {
    const double b = kRcRefineSigma * kRcRefineSigma * (2.1981 * (double)median_err);
    return sqrt((b < thr_sqr0) ? b : thr_sqr0);
}

} // namespace mulls
