// NDT registration: lo::CRegistration<PointT>::omp_ndt (cregistration.hpp:945-1021) with DIRECT7 neighbours, i.e.
// koide_reg::NormalDistributionsTransform and koide_reg::VoxelGridCovariance (include/baseline_reg/ndt_omp_impl.hpp,
// voxel_grid_covariance_omp_impl.hpp) on PCL 1.10 / Eigen 3.3.
//
// This header holds what the device path (kernels_ndt.cuh, the host side of mulls_omp_ndt) and the CPU restatement
// under tests/harness share, so that both compute the same bits: the leaf finalisation, the DIRECT7 cell
// arithmetic, the per-point derivatives, the fixed summation order, the Newton walk and the float step transform.
// Readings (the reference was read, not run):
//  N1 target leaves (applyFilter): min/max over the finite points in float, min_b = (int)floor(min * inv) with the float
//     inverse leaf size inv = 1.0f / resolution; a point's leaf (int)(floor(x * inv) - (float)min_b) per axis, linearised
//     with divb_mul = (1, div_x, div_x div_y). dx dy dz (int64 of (max - min) * inv, plus 1) above INT32_MAX: no leaves.
//     Each leaf sums its points in input order in double (sum, sum of p p^T). Finalise as ndt_leaf_finish. A leaf of
//     fewer than 6 points exists but is never a neighbour; nr_points = -1 (rejected) as voxel_grid_covariance_omp_impl.
//  N2 eigen-decomposition: SelfAdjointEigenSolver<Matrix3d> (tridiagonal QR) is read as any accurate symmetric
//     eigensolver; here cyclic Jacobi (ndt_eig3) on the lower triangle. The choice moves only the last bits of a double
//     covariance, before its inverse is cast to float. cov.inverse() and evecs.inverse() are Eigen's 3x3 cofactor
//     inverse (ndt_inv3).
//  N3 DIRECT7 (getNeighborhoodAtPoint7): ijk = (int)floor(x / resolution) — a float division, where the build multiplies
//     by the inverse; the two can disagree at a cell border when the resolution is not a power of two. Probes in the
//     order centre, +x, -x, +y, -y, +z, -z; each bounds-checked against min_b / max_b, used when its leaf has >= 6 points
//     and was not rejected. Coordinates beyond the int range saturate (the reference's cast is undefined there).
//  N4 derivatives (computeDerivatives / updateDerivatives): the float j_ang (8x3) and h_ang (15x3) from double cos/sin of
//     p(3..5) with the |angle| < 1e-4 shortcut (computed on the host, ndt_angle_tables); per neighbour x_trans is the
//     float-transformed point minus the double mean, then updateDerivatives in float with the exp of ndt_expf; score,
//     gradient and all 36 Hessian terms are summed per point over its neighbours in double. Eigen's float products are
//     read as index-order dot products.
//  N5 the walk (computeTransformation, computeStepLengthMT with step_max 0.1, step_min 0.05): interval_converged starts
//     true, so the More-Thuente loop and computeHessian never run (static_assert below). Each iteration: JacobiSVD<6x6>
//     solve of -g with Eigen 3.3's rank threshold (6 eps of the largest singular value), return on a zero or NaN norm,
//     normalise, reverse if -g.d > 0 (step 0 if it is exactly 0), step clamp(norm, 0.05, 0.1), float transform
//     Translation * AngleAxis(x) * AngleAxis(y) * AngleAxis(z), one evaluation, stop if nr > 35 or (nr and step < 0.1).
//     No step is shorter than 0.05 in the mixed m / rad 6-vector, so even a converged walk ends up to 0.05 off the
//     Newton point.
//  N6 non-finite coordinates: left out of the min/max, the leaves, the derivatives and the fitness count (PCL's
//     non-dense branches).
// With use_direct_search = false omp_ndt selects koide_reg::KDTREE, PCL's original neighbourhood (mulls_omp_ndt_kdtree).
// Read from the same files and PCL 1.10 / FLANN 1.9, not run, as N1-N6:
//  K1 the searchable cloud (voxel_grid_covariance_omp_impl.hpp:283-327): one centroid per leaf with nr_points >= 6, in
//     ascending leaf index (std::map order), pushed before the eigenvalue and infinite-inverse checks, so a leaf rejected
//     afterwards (nr_points = -1) stays in the kd-tree. Its xyz is the float sum of the leaf's points in input order
//     divided by (float)nr_points (:175-201, :290), not the double mean_ (ndt_kd_centroid).
//  K2 the search (voxel_grid_covariance_omp.h:472-499, pcl::KdTreeFLANN::radiusSearch over FLANN's KDTreeSingleIndex with
//     L2_Simple<float>): the query is the float moved point, xyz only; r2 = (float)((double)resolution * resolution);
//     d2 = (dx*dx + dy*dy) + dz*dz in float without contraction; a centroid is a neighbour iff d2 < r2; max_nn = 0
//     returns all neighbours, sorted by (distance, index) (RadiusResultSet's sorted copy, DistanceIndex::operator<), as
//     kernels_pca.cuh reads radiusSearch. The index is the rank among the searchable leaves, so ascending index is
//     ascending leaf index.
//  K3 the contributions (ndt_omp_impl.hpp:233-270): the KDTREE branch never checks nr_points; every neighbour goes
//     through ndt_update with the leaf's double mean and float icov as the finalisation leaves them. A leaf rejected by
//     its eigenvalues keeps icov_ = 0 (Leaf(), voxel_grid_covariance_omp.h:98-107): it adds -d1 to the score (gauss_d2
//     <= 1) and nothing to the gradient or Hessian. DIRECT7 never sees those leaves (6 or more equal points, an exactly
//     planar leaf whose smallest eigenvalue rounds below zero), so on such targets the score traces of the two modes
//     differ. The reference's infinite-inverse rejection keeps the computed inverse; ndt_leaf_finish leaves icov zero
//     there instead, because no float input reaches it: after the eigenvalue check and the inflation every eigenvalue of
//     the covariance is at least 0.01 of the largest, ev2 > 0, so an inverse entry is at most about 100 / ev2 and
//     overflows only for ev2 below about 1e-306; a covariance of float points that are not all equal (equal points
//     give exactly 0 and the eigenvalue rejection) is of the order of their spread squared or of the rounding of
//     their squares, both above 2^-300 (products of floats are multiples of 2^-298).
//  K4 no centroids (empty target, every leaf under 6 points, more than INT32_MAX cells): the reference searches an index
//     it never built (undefined); here no point has neighbours, as DIRECT7's empty-target rule says.
//  K5 everything else is the DIRECT7 path: the prologue, N1-N2, the walk and its constants (N5), C1, C2, the fitness,
//     Trans1_2 and the codes. Only the neighbourhood changes.
// The device search (kernels_ndt.cuh) keys every centroid by the cell of its own float coordinates on the leaf grid,
// clamped to [min_b, max_b] (ndt_kd_cell), and probes for a query t the cells from ndt_kd_cell(t - r') to
// ndt_kd_cell(t + r') per axis, r' = resolution (1 + 2^-16) in float. The box holds every neighbour: d2 < r2 gives
// fl(dx^2) <= d2 < r2 <= r^2 (1 + u) (sums of non-negative terms round to at least each term), so |dx| < r (1 + u) and
// |t - c| < r (1 + 3u) per axis, u = 2^-24, while r' >= r (1 + 2^-16 - 2^-24) exceeds that (r2 a normal float, i.e. a
// resolution above 1.1e-19). Then t - r' <= c <= t + r' exactly, and float rounding, the product by inv, floor, the
// saturating cast and the clamp are all monotone, so the centroid's cell lies in the box on every axis. A box spans 3
// cells per axis (4 where rounding reaches a face). Each centroid lies in its own leaf up to rounding, and a ball of
// radius r meets at most 27 cells of edge r, so a list rarely exceeds 27; it has no bound in general (a float sum of
// many points can drift), so the host grows the list capacity when a count exceeds it and repeats the evaluation.
// Choices where the reference depends on the machine (OpenMP partial sums, Eigen's vectorised products):
//  C1 the points' contributions are summed in tiles of kNdtTile points in index order: within a tile a pairwise tree
//     q[t] += q[t + s] for s = 16 .. 1 inside each group of 32, then over the kNdtTile / 32 group sums for s = 2, 1; then
//     the tiles' sums in tile order, starting from 0.0. A point without terms contributes 0.0.
//  C2 exp: ndt_expf, one exp from + - * / on doubles, rounded to float once (within 1 ulp of a correctly rounded expf).
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "ransac_core.cuh"

namespace mulls {

constexpr int kNdtTile = 128;         // points per tile of the fixed summation order (C1), the evaluation block
constexpr int kNdtTerms = 43;         // score, 6 gradient, 36 Hessian terms
constexpr int kNdtMinPoints = 6;      // min_points_per_voxel_
constexpr int kNdtMaxIterations = 35; // max_iterations_
constexpr double kNdtStepMax = 0.1;   // step_size_
constexpr double kNdtEpsilon = 0.1;   // transformation_epsilon_
constexpr double kNdtStepMin = kNdtEpsilon / 2;
constexpr double kNdtOutlierRatio = 0.55;
constexpr double kNdtMinCovarEigMult = 0.01;
// computeStepLengthMT's interval_converged = (step_max - step_min) > 0: true here, so the More-Thuente loop is dead and
// each iteration evaluates the derivatives once, at the clamped step. A change to these constants needs the line search.
static_assert(kNdtStepMax - kNdtStepMin > 0, "the NDT walk skips the More-Thuente line search only while step_max > step_min");

// ---- C2: exp of a float, from + - * / in double -----------------------------------------------------------------------
GF_HD double ndt_pow2(int k) { // 2^k, -1022 <= k <= 1023
    const uint64_t b = (uint64_t)(k + 1023) << 52;
    double d;
    memcpy(&d, &b, sizeof(d));
    return d;
}
GF_HD float ndt_expf(float v) {
    if (v != v) return v;
    if (v < -110.f) return 0.f;
    if (v > 89.f) return (float)ndt_pow2(1023) * 2.f; // +inf
    const double x = (double)v;
    const double n = floor(x * 1.4426950408889634 + 0.5);
    // Cody-Waite: ln2_hi has 32 trailing zero bits, so n * ln2_hi is exact for |n| < 2^20
    const double r = (x - n * 6.93147180369123816490e-01) - n * 1.90821492927058770002e-10;
    double p = 1.0 / 479001600.0; // Taylor to r^12 / 12!, |r| <= ln2 / 2
    const double inv[12] = {1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0, 1.0 / 40320.0, 1.0 / 5040.0, 1.0 / 720.0,
                            1.0 / 120.0,      1.0 / 24.0,      1.0 / 6.0,      0.5,           1.0,          1.0};
    for (int i = 0; i < 12; ++i) p = p * r + inv[i];
    return (float)(p * ndt_pow2((int)n));
}

// ---- float to int as the leaf arithmetic needs it: saturating, defined everywhere (N3) --------------------------------
GF_HD int ndt_f2i(float f) {
    if (!(f > -2147483648.f)) return INT_MIN; // NaN included (such points never get here)
    if (f >= 2147483648.f) return INT_MAX;
    return (int)f;
}

// the grid of the target leaves (N1)
struct NdtGrid {
    float leaf, inv;         // resolution, 1.0f / resolution
    int min_b[3], max_b[3];
    int64_t divb_mul[3];
    int ok;                  // 0: no leaves (empty target, or more than INT32_MAX cells)
};

// from the float min / max of the finite target points; n_finite = 0 gives ok = 0
inline NdtGrid ndt_grid_of(float resolution, const float mn[3], const float mx[3], size_t n_finite) {
    NdtGrid g;
    g.leaf = resolution;
    g.inv = 1.0f / resolution;
    g.ok = 0;
    for (int d = 0; d < 3; ++d) g.min_b[d] = g.max_b[d] = 0, g.divb_mul[d] = 0;
    if (n_finite == 0) return g;
    int64_t dims = 1;
    for (int d = 0; d < 3; ++d) {
        const float e = (mx[d] - mn[d]) * g.inv;
        if (!(e < 9.2e18f)) return g;
        dims *= (int64_t)e + 1;
        if (dims > INT32_MAX) return g;
    }
    for (int d = 0; d < 3; ++d) {
        g.min_b[d] = ndt_f2i(floorf(mn[d] * g.inv));
        g.max_b[d] = ndt_f2i(floorf(mx[d] * g.inv));
    }
    const int64_t div0 = (int64_t)g.max_b[0] - g.min_b[0] + 1, div1 = (int64_t)g.max_b[1] - g.min_b[1] + 1;
    g.divb_mul[0] = 1, g.divb_mul[1] = div0, g.divb_mul[2] = div0 * div1;
    g.ok = 1;
    return g;
}

// the leaf index of a finite target point (applyFilter's first pass)
GF_HD int64_t ndt_build_key(const NdtGrid &g, float x, float y, float z) {
    const int i0 = ndt_f2i(floorf(x * g.inv) - (float)g.min_b[0]);
    const int i1 = ndt_f2i(floorf(y * g.inv) - (float)g.min_b[1]);
    const int i2 = ndt_f2i(floorf(z * g.inv) - (float)g.min_b[2]);
    return (int64_t)i0 * g.divb_mul[0] + (int64_t)i1 * g.divb_mul[1] + (int64_t)i2 * g.divb_mul[2];
}

// DIRECT7 probe `k` (0..6) of a finite query point: false when the cell is outside [min_b, max_b]
GF_HD bool ndt_probe_key(const NdtGrid &g, float x, float y, float z, int k, int64_t &key) {
    const int d = (k - 1) >> 1, sgn = (k & 1) ? 1 : -1;
    int64_t c[3] = {ndt_f2i(floorf(x / g.leaf)), ndt_f2i(floorf(y / g.leaf)), ndt_f2i(floorf(z / g.leaf))};
    if (k > 0) c[d] += sgn;
    key = 0;
    for (int a = 0; a < 3; ++a) {
        if (c[a] < g.min_b[a] || c[a] > g.max_b[a]) return false;
        key += (c[a] - g.min_b[a]) * g.divb_mul[a];
    }
    return true;
}

// ---- N1/N2: the leaf finalisation ----------------------------------------------------------------------------------
// what a lookup needs of a leaf
struct NdtLeaf {
    double mean[3];
    float icov[9]; // c_inv.cast<float>(), row-major
    int ok;        // nr_points >= 6 and not rejected
    int n;         // nr_points (-1: rejected)
};

GF_HD void ndt_inv3(const double m[3][3], double out[3][3]) { // Eigen 3.3 compute_inverse_size3_helper
    double cof[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            cof[i][j] = m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
        }
    const double det = (cof[0][0] * m[0][0] + cof[1][0] * m[1][0]) + cof[2][0] * m[2][0];
    const double invdet = 1.0 / det;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) out[j][i] = cof[i][j] * invdet;
}

// cyclic Jacobi on the lower triangle of a symmetric 3x3: ascending eigenvalues, eigenvectors as the columns of V
GF_HD void ndt_eig3(const double a[3][3], double ev[3], double V[3][3]) {
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            A[i][j] = i >= j ? a[i][j] : a[j][i];
            V[i][j] = i == j ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double off = (fabs(A[1][0]) + fabs(A[2][0])) + fabs(A[2][1]);
        if (off == 0.0) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) { // A = J^T A J, columns then rows
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                A[p][q] = A[q][p] = 0.0;
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < 3; ++i) ev[i] = A[i][i];
    for (int i = 0; i < 2; ++i) { // ascending, stable
        int m = i;
        for (int j = i + 1; j < 3; ++j)
            if (ev[j] < ev[m]) m = j;
        if (m != i) {
            const double t = ev[i];
            ev[i] = ev[m], ev[m] = t;
            for (int k = 0; k < 3; ++k) {
                const double x = V[k][i];
                V[k][i] = V[k][m], V[k][m] = x;
            }
        }
    }
}

// sums: s[3] = sum of p, c[9] = sum of p p^T (row-major), n points
GF_HD NdtLeaf ndt_leaf_finish(const double s[3], const double c[9], int n) {
    NdtLeaf L;
    L.n = n;
    L.ok = 0;
    for (int i = 0; i < 3; ++i) L.mean[i] = s[i] / (double)n;
    for (int i = 0; i < 9; ++i) L.icov[i] = 0.f;
    if (n < kNdtMinPoints) return L;
    double cov[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            cov[i][j] = (c[3 * i + j] - 2.0 * (s[i] * L.mean[j])) / (double)n + L.mean[i] * L.mean[j];
    const double f = ((double)n - 1.0) / (double)n;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) cov[i][j] *= f;
    double ev[3], V[3][3];
    ndt_eig3(cov, ev, V);
    if (ev[0] < 0.0 || ev[1] < 0.0 || ev[2] <= 0.0) {
        L.n = -1;
        return L;
    }
    const double lim = kNdtMinCovarEigMult * ev[2];
    if (ev[0] < lim) {
        ev[0] = lim;
        if (ev[1] < lim) ev[1] = lim;
        double Vi[3][3];
        ndt_inv3(V, Vi);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) // (V diag) Vi
                cov[i][j] = ((V[i][0] * ev[0]) * Vi[0][j] + (V[i][1] * ev[1]) * Vi[1][j]) + (V[i][2] * ev[2]) * Vi[2][j];
    }
    double ic[3][3];
    ndt_inv3(cov, ic);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            if (ic[i][j] == (double)INFINITY || ic[i][j] == -(double)INFINITY) {
                L.n = -1;
                return L;
            }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) L.icov[3 * i + j] = (float)ic[i][j];
    L.ok = 1;
    return L;
}

// ---- K1/K2: the KDTREE neighbourhood ---------------------------------------------------------------------------------
// a leaf of n points (before the checks) is in the searchable cloud
GF_HD bool ndt_kd_searchable(int n_points) { return n_points >= kNdtMinPoints; }

// K1: the float centroid of a leaf from the float sums of its points in input order
GF_HD void ndt_kd_centroid(const float s[3], int n, float c[3]) {
    for (int a = 0; a < 3; ++a) c[a] = s[a] / (float)n;
}

// K2: the search radius squared, and radiusSearch's float distance of query q to centroid c
GF_HD float ndt_kd_r2(float resolution) { return (float)((double)resolution * (double)resolution); }
GF_HD float ndt_kd_d2(const float q[3], float cx, float cy, float cz) {
    const float dx = q[0] - cx, dy = q[1] - cy, dz = q[2] - cz;
    return (dx * dx + dy * dy) + dz * dz;
}
// (d2, index) order
GF_HD bool ndt_kd_before(float d2a, int ia, float d2b, int ib) { return d2a < d2b || (d2a == d2b && ia < ib); }

// the search cell of coordinate v on axis a: the leaf grid's cell of v itself, clamped to [min_b, max_b] (monotone in v)
GF_HD int ndt_kd_cell(const NdtGrid &g, float v, int a) {
    const int c = ndt_f2i(floorf(v * g.inv));
    return c < g.min_b[a] ? g.min_b[a] : (c > g.max_b[a] ? g.max_b[a] : c);
}
GF_HD int64_t ndt_kd_key(const NdtGrid &g, int c0, int c1, int c2) {
    return ((int64_t)c0 - g.min_b[0]) * g.divb_mul[0] + ((int64_t)c1 - g.min_b[1]) * g.divb_mul[1] +
           ((int64_t)c2 - g.min_b[2]) * g.divb_mul[2];
}
// the probe box of query t: cells lo[a] .. hi[a] per axis (the header's argument: it holds every c with d2 < r2)
GF_HD float ndt_kd_probe_radius(float resolution) { return resolution * (1.0f + 1.0f / 65536.0f); }
GF_HD void ndt_kd_box(const NdtGrid &g, float rp, const float t[3], int lo[3], int hi[3]) {
    for (int a = 0; a < 3; ++a) lo[a] = ndt_kd_cell(g, t[a] - rp, a), hi[a] = ndt_kd_cell(g, t[a] + rp, a);
}

// ---- N4: the derivatives ---------------------------------------------------------------------------------------------
// everything an evaluation needs besides the clouds: the float transform of the step (rows 0..2), the angle tables and
// the gauss constants
struct NdtEvalConst {
    float T[12];
    float j_ang[8][3];
    float h_ang[15][3];
    double gauss_d1;
    float gauss_d2;
};

// computeAngleDerivatives(p) into the float tables (host: the trig stays there)
inline void ndt_angle_tables(const double p[6], NdtEvalConst &E) {
    double cx, cy, cz, sx, sy, sz;
    if (fabs(p[3]) < 10e-5) cx = 1.0, sx = 0.0;
    else cx = cos(p[3]), sx = sin(p[3]);
    if (fabs(p[4]) < 10e-5) cy = 1.0, sy = 0.0;
    else cy = cos(p[4]), sy = sin(p[4]);
    if (fabs(p[5]) < 10e-5) cz = 1.0, sz = 0.0;
    else cz = cos(p[5]), sz = sin(p[5]);
    const double j[8][3] = {{(-sx * sz + cx * sy * cz), (-sx * cz - cx * sy * sz), (-cx * cy)},
                            {(cx * sz + sx * sy * cz), (cx * cz - sx * sy * sz), (-sx * cy)},
                            {(-sy * cz), sy * sz, cy},
                            {sx * cy * cz, (-sx * cy * sz), sx * sy},
                            {(-cx * cy * cz), cx * cy * sz, (-cx * sy)},
                            {(-cy * sz), (-cy * cz), 0},
                            {(cx * cz - sx * sy * sz), (-cx * sz - sx * sy * cz), 0},
                            {(sx * cz + cx * sy * sz), (cx * sy * cz - sx * sz), 0}};
    const double h[15][3] = {{(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), sx * cy},
                             {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), (-cx * cy)},
                             {(cx * cy * cz), (-cx * cy * sz), (cx * sy)},
                             {(sx * cy * cz), (-sx * cy * sz), (sx * sy)},
                             {(-sx * cz - cx * sy * sz), (sx * sz - cx * sy * cz), 0},
                             {(cx * cz - sx * sy * sz), (-sx * sy * cz - cx * sz), 0},
                             {(-cy * cz), (cy * sz), (sy)},
                             {(-sx * sy * cz), (sx * sy * sz), (sx * cy)},
                             {(cx * sy * cz), (-cx * sy * sz), (-cx * cy)},
                             {(sy * sz), (sy * cz), 0},
                             {(-sx * cy * sz), (-sx * cy * cz), 0},
                             {(cx * cy * sz), (cx * cy * cz), 0},
                             {(-cy * cz), (cy * sz), 0},
                             {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), 0},
                             {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), 0}};
    for (int r = 0; r < 8; ++r)
        for (int c = 0; c < 3; ++c) E.j_ang[r][c] = (float)j[r][c];
    for (int r = 0; r < 15; ++r)
        for (int c = 0; c < 3; ++c) E.h_ang[r][c] = (float)h[r][c];
}

// the gauss constants of computeTransformation (eq. 6.8), outlier ratio 0.55
inline void ndt_gauss(float resolution, double &d1, double &d2) {
    const double c1 = 10 * (1 - kNdtOutlierRatio), c2 = kNdtOutlierRatio / pow((double)resolution, 3);
    const double d3 = -log(c2);
    d1 = -log(c1 + c2) - d3;
    d2 = -2 * log((-log(c1 * exp(-0.5) + c2) - d3) / d1);
}

// the float transform of a point (R4 of ransac_core.cuh: ((m0 x + m1 y) + m2 z) + m3)
GF_HD void ndt_transform(const float T[12], float x, float y, float z, float o[3]) {
    o[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
    o[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
    o[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

GF_HD bool ndt_finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// updateDerivatives of one neighbour: adds into acc (score, gradient[6], Hessian[36] row-major) in double.
// x: the input point; xt: its transformed position minus the leaf mean (double, as the reference's x_trans).
GF_HD void ndt_update(const NdtEvalConst &E, const float x[3], const double xt_d[3], const float *ci, double acc[kNdtTerms]) {
    const float xt[3] = {(float)xt_d[0], (float)xt_d[1], (float)xt_d[2]};
    float xc[3]; // x_trans4 * c_inv4
    for (int k = 0; k < 3; ++k) xc[k] = (xt[0] * ci[k] + xt[1] * ci[3 + k]) + xt[2] * ci[6 + k];
    const float q = (xt[0] * xc[0] + xt[1] * xc[1]) + xt[2] * xc[2];
    const float gd2 = E.gauss_d2;
    float e = ndt_expf(-gd2 * q * 0.5f);
    const float score_inc = (float)(-E.gauss_d1 * (double)e);
    e = gd2 * e;
    if (e > 1.f || e < 0.f || e != e) return;
    e = (float)((double)e * E.gauss_d1);
    acc[0] += (double)score_inc;
    // point_gradient_ (3x6): identity in columns 0..2, the angle terms in 3..5
    float xj[8];
    for (int r = 0; r < 8; ++r) xj[r] = (E.j_ang[r][0] * x[0] + E.j_ang[r][1] * x[1]) + E.j_ang[r][2] * x[2];
    const float pg[3][6] = {{1.f, 0.f, 0.f, 0.f, xj[2], xj[5]}, {0.f, 1.f, 0.f, xj[0], xj[3], xj[6]}, {0.f, 0.f, 1.f, xj[1], xj[4], xj[7]}};
    float cg[3][6], g6[6];
    for (int m = 0; m < 3; ++m)
        for (int j = 0; j < 6; ++j) cg[m][j] = (ci[3 * m] * pg[0][j] + ci[3 * m + 1] * pg[1][j]) + ci[3 * m + 2] * pg[2][j];
    for (int j = 0; j < 6; ++j) {
        g6[j] = (xt[0] * cg[0][j] + xt[1] * cg[1][j]) + xt[2] * cg[2][j];
        acc[1 + j] += (double)(e * g6[j]);
    }
    float xh[15];
    for (int r = 0; r < 15; ++r) xh[r] = (E.h_ang[r][0] * x[0] + E.h_ang[r][1] * x[1]) + E.h_ang[r][2] * x[2];
    // the 3-vectors of point_hessian_ block (i, j), i, j >= 3 (eq. 6.21): a b c / b d e / c e f
    const float hv[6][3] = {{0.f, xh[0], xh[1]}, {0.f, xh[2], xh[3]}, {0.f, xh[4], xh[5]},
                            {xh[6], xh[7], xh[8]}, {xh[9], xh[10], xh[11]}, {xh[12], xh[13], xh[14]}};
    const int blk[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            const float pgc = (pg[0][j] * cg[0][i] + pg[1][j] * cg[1][i]) + pg[2][j] * cg[2][i];
            float xhij = 0.f;
            if (i >= 3 && j >= 3) {
                const float *h = hv[blk[i - 3][j - 3]];
                xhij = (xc[0] * h[0] + xc[1] * h[1]) + xc[2] * h[2];
            }
            acc[7 + 6 * i + j] += (double)(e * ((-gd2 * g6[i] * g6[j] + xhij) + pgc));
        }
}

// ---- C1: the fixed summation order over one tile, serial form (the evaluation kernel runs it with shuffles) -----------
// q[t] for t < kNdtTile (zeros past the cloud's end); returns the tile's sum
GF_HD double ndt_tile_sum(double *q) {
    for (int g = 0; g < kNdtTile; g += 32)
        for (int s = 16; s > 0; s >>= 1)
            for (int t = 0; t < s; ++t) q[g + t] += q[g + t + s];
    double w[kNdtTile / 32];
    for (int g = 0; g < kNdtTile / 32; ++g) w[g] = q[32 * g];
    for (int s = kNdtTile / 64; s > 0; s >>= 1)
        for (int t = 0; t < s; ++t) w[t] += w[t + s];
    return w[0];
}

// ---- N5: the Newton walk's pieces (host) ------------------------------------------------------------------------------
// Translation(x(0..2)) * AngleAxisf(x(3), X) * AngleAxisf(x(4), Y) * AngleAxisf(x(5), Z), rows 0..2 of the float 4x4
inline void ndt_step_transform(const double x[6], float T[12]) {
    float R[3][3][3];
    for (int a = 0; a < 3; ++a) { // AngleAxis::toRotationMatrix with the unit axis a
        const float ang = (float)x[3 + a];
        const float axis[3] = {a == 0 ? 1.f : 0.f, a == 1 ? 1.f : 0.f, a == 2 ? 1.f : 0.f};
        const float s = sinf(ang), c = cosf(ang);
        float sa[3], c1[3];
        for (int k = 0; k < 3; ++k) sa[k] = s * axis[k], c1[k] = (1.f - c) * axis[k];
        float (*M)[3] = R[a];
        float tmp = c1[0] * axis[1];
        M[0][1] = tmp - sa[2], M[1][0] = tmp + sa[2];
        tmp = c1[0] * axis[2];
        M[0][2] = tmp + sa[1], M[2][0] = tmp - sa[1];
        tmp = c1[1] * axis[2];
        M[1][2] = tmp - sa[0], M[2][1] = tmp + sa[0];
        for (int k = 0; k < 3; ++k) M[k][k] = c1[k] * axis[k] + c;
    }
    float P[3][3], Q[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) P[i][j] = (R[0][i][0] * R[1][0][j] + R[0][i][1] * R[1][1][j]) + R[0][i][2] * R[1][2][j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Q[i][j] = (P[i][0] * R[2][0][j] + P[i][1] * R[2][1][j]) + P[i][2] * R[2][2][j];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = Q[i][j];
        T[4 * i + 3] = (float)x[i];
    }
}

// JacobiSVD<Matrix<double, 6, 6>>(H, ComputeFullU | ComputeFullV).solve(b) as SVDBase::_solve_impl: rank by Eigen 3.3's
// default threshold (6 * eps times the largest singular value, at least DBL_MIN, counted over the nonzero ones);
// tmp = U^T b, tmp = diag(1 / s) tmp (a product with the reciprocal, as asDiagonal().inverse()), x = V tmp. The products
// are read as index-order dot products.
inline void ndt_svd_solve(const double H[36], const double b[6], double x[6]) {
    double A[6][6], U[6][6], V[6][6], sv[6];
    for (int i = 0; i < 36; ++i) A[i / 6][i % 6] = H[i];
    const int nz = rc_svd<6>(A, U, V, sv);
    double thr = sv[0] * (6.0 * DBL_EPSILON);
    if (thr < DBL_MIN) thr = DBL_MIN;
    int rank = nz;
    while (rank > 0 && sv[rank - 1] < thr) --rank;
    double t[6];
    for (int k = 0; k < rank; ++k) {
        double d = 0.0;
        for (int i = 0; i < 6; ++i) d += U[i][k] * b[i];
        t[k] = (1.0 / sv[k]) * d;
    }
    for (int i = 0; i < 6; ++i) {
        double d = 0.0;
        for (int k = 0; k < rank; ++k) d += V[i][k] * t[k];
        x[i] = d;
    }
}

// one iteration record of the walk
struct NdtIter {
    double p[6];  // the pose vector after the step
    double step;  // the step length (0, or in [0.05, 0.1])
    double score; // the score at p
    int reversed; // computeStepLengthMT turned the direction around (-g.d > 0)
};

// computeTransformation from the derivatives at p = 0, as a state that advances one evaluation at a time, so that one
// walk (ndt_walk) and a batch of walks in lockstep (mulls_omp_ndt_batch) run the same code. The owner evaluates score,
// gradient and Hessian at the pose vector `q` and its float transform `T` into `r`, then calls ndt_walk_advance, until
// that returns false. `T` is then the final float transform, `nr` the iteration count.
struct NdtWalk {
    double p[6], q[6], d[6], a; // pose, the pose being evaluated, the step direction and length
    double r[kNdtTerms];        // score, gradient, Hessian at q
    float T[12];                // the float transform of q
    int nr, converged, reversed;
    int in_step;                // r holds the evaluation of the current iteration's step
};

inline void ndt_walk_start(NdtWalk &W) {
    const float I[12] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f};
    for (int i = 0; i < 6; ++i) W.p[i] = W.q[i] = 0.0;
    for (int i = 0; i < 12; ++i) W.T[i] = I[i];
    W.nr = W.converged = W.reversed = W.in_step = 0;
    W.a = 0.0;
}

// consumes the evaluation of W.q: true when the next one is wanted (at W.q, W.T), false when the walk has ended. trace
// (cap entries) records every iteration.
inline bool ndt_walk_advance(NdtWalk &W, NdtIter *trace, int cap) {
    for (;;) {
        if (W.in_step) { // the end of an iteration: the step is taken
            W.in_step = 0;
            for (int i = 0; i < 6; ++i) W.p[i] = W.p[i] + W.d[i] * W.a;
            if (trace && W.nr < cap) {
                for (int i = 0; i < 6; ++i) trace[W.nr].p[i] = W.p[i];
                trace[W.nr].step = W.a, trace[W.nr].score = W.r[0], trace[W.nr].reversed = W.reversed;
            }
            const bool stop = W.nr > kNdtMaxIterations || (W.nr && fabs(W.a) < kNdtEpsilon);
            ++W.nr;
            if (stop) {
                W.converged = 1;
                return false;
            }
        }
        double b[6], *d = W.d;
        for (int i = 0; i < 6; ++i) b[i] = -W.r[1 + i];
        ndt_svd_solve(W.r + 7, b, d);
        double sq = 0.0;
        for (int i = 0; i < 6; ++i) sq += d[i] * d[i];
        const double norm = sqrt(sq);
        if (norm == 0 || norm != norm) {
            W.converged = norm == norm;
            return false;
        }
        for (int i = 0; i < 6; ++i) d[i] /= norm; // normalize(): /= sqrt(squaredNorm)
        // computeStepLengthMT
        double d_phi_0 = 0.0;
        for (int i = 0; i < 6; ++i) d_phi_0 += W.r[1 + i] * d[i];
        d_phi_0 = -d_phi_0;
        W.a = 0.0;
        W.reversed = 0;
        W.in_step = 1;
        bool step = true;
        if (d_phi_0 >= 0) {
            if (d_phi_0 == 0) step = false;
            else {
                for (int i = 0; i < 6; ++i) d[i] = -d[i];
                W.reversed = 1;
            }
        }
        if (step) {
            double a = norm < kNdtStepMax ? norm : kNdtStepMax;
            W.a = a > kNdtStepMin ? a : kNdtStepMin;
            for (int i = 0; i < 6; ++i) W.q[i] = W.p[i] + d[i] * W.a;
            ndt_step_transform(W.q, W.T);
            return true;
        }
        // no step: the iteration ends without an evaluation, on the same derivatives
    }
}

// the whole walk: `eval(q, T, out43)` evaluates at the float transform T of q and fills score, gradient, Hessian.
// Returns the iteration count; T_final the float transform; converged; trace (cap entries) records every iteration.
template <class Eval>
int ndt_walk(Eval eval, float T_final[12], int &converged, NdtIter *trace, int cap) {
    NdtWalk W;
    ndt_walk_start(W);
    do eval(W.q, W.T, W.r);
    while (ndt_walk_advance(W, trace, cap));
    for (int i = 0; i < 12; ++i) T_final[i] = W.T[i];
    converged = W.converged;
    return W.nr;
}

// ---- the prologue and epilogue (host) ----------------------------------------------------------------------------
// the prologue (cregistration.hpp:955-978) on the caller's rows: the initial guess moves the source in double with a
// float store, the intersection box is padded by 2.0 (utility.hpp:858-866) and both clouds keep the points strictly
// inside it (cfilter.hpp:950-981); the target keeps its finite points only (N6). Host only: one pass over the rows.
inline bool ndt_is_identity(const double *m) { // Matrix4d::isIdentity(1e-6)
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const double x = m[4 * i + j];
            if (i == j ? !(fabs(x - 1.0) <= 1e-6 * min(fabs(x), 1.0)) : !(fabs(x) <= 1e-6)) return false;
        }
    return true;
}
inline void ndt_prologue(const float *t48, size_t nt, const float *s48, size_t ns, const double *guess, int apply_filter,
                  const double *tbound, const double *sbound, std::vector<float4> &tgt, std::vector<float4> &src, bool &moved) {
    moved = !ndt_is_identity(guess);
    src.resize(ns);
    double sb[6] = {DBL_MAX, DBL_MAX, DBL_MAX, -DBL_MAX, -DBL_MAX, -DBL_MAX};
    for (size_t i = 0; i < ns; ++i) {
        float x = s48[12 * i], y = s48[12 * i + 1], z = s48[12 * i + 2];
        if (moved) {
            const double *t = guess;
            const double px = x, py = y, pz = z;
            x = (float)(t[0] * px + t[1] * py + t[2] * pz + t[3]);
            y = (float)(t[4] * px + t[5] * py + t[6] * pz + t[7]);
            z = (float)(t[8] * px + t[9] * py + t[10] * pz + t[11]);
            const float v[3] = {x, y, z};
            for (int d = 0; d < 3; ++d) { // get_cloud_bbx
                if (v[d] < sb[d]) sb[d] = v[d];
                if (v[d] > sb[3 + d]) sb[3 + d] = v[d];
            }
        }
        src[i] = make_float4(x, y, z, 0.f);
    }
    const double *b2 = moved ? sb : sbound;
    double ib[6];
    for (int d = 0; d < 3; ++d) {
        ib[d] = max(tbound[d], b2[d]) - 2.0;
        ib[3 + d] = min(tbound[3 + d], b2[3 + d]) + 2.0;
    }
    auto inside = [&](float x, float y, float z) {
        return !apply_filter || ((double)x > ib[0] && (double)x < ib[3] && (double)y > ib[1] && (double)y < ib[4] &&
                                 (double)z > ib[2] && (double)z < ib[5]);
    };
    size_t k = 0;
    for (size_t i = 0; i < ns; ++i)
        if (inside(src[i].x, src[i].y, src[i].z)) src[k++] = src[i];
    src.resize(k);
    tgt.clear();
    for (size_t i = 0; i < nt; ++i) {
        const float x = t48[12 * i], y = t48[12 * i + 1], z = t48[12 * i + 2];
        if (inside(x, y, z) && ndt_finite3(x, y, z)) tgt.push_back(make_float4(x, y, z, 0.f));
    }
}
// getMinMax3D over the (finite) target, then the leaf grid (N1)
inline NdtGrid ndt_grid_from(const std::vector<float4> &tgt, float resolution) {
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (const float4 &p : tgt) {
        const float v[3] = {p.x, p.y, p.z};
        for (int d = 0; d < 3; ++d) mn[d] = min(mn[d], v[d]), mx[d] = max(mx[d], v[d]);
    }
    return ndt_grid_of(resolution, mn, mx, tgt.size());
}
// Trans1_2 = (double)final * initial_guess when the guess moved the source
inline void ndt_epilogue(const float T[12], const double *guess, bool moved, double out[16]) {
    double F[16];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) F[4 * r + c] = (double)T[4 * r + c];
    F[12] = F[13] = F[14] = 0.0, F[15] = 1.0;
    if (!moved) {
        memcpy(out, F, sizeof(F));
        return;
    }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            double s = 0.0;
            for (int k = 0; k < 4; ++k) s += F[4 * r + k] * guess[4 * k + c];
            out[4 * r + c] = s;
        }
}

} // namespace mulls
