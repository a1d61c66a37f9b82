// Ground segmentation on the device: lo::CFilter<PointT>::fast_ground_filter, cfilter.hpp:1658-2036, with the per-cell
// RANSAC plane of estimate_ground_normal_by_ransac (:2038-2054) -> CProceesing::plane_seg_ransac (cprocessing.hpp:67-105)
// -> pcl::SACSegmentation (SACMODEL_PLANE, SAC_RANSAC, optimize coefficients; PCL 1.10 semantics).
//
// This header holds the per-point / per-cell work as `__host__ __device__` functions: the kernels of
// kernels_ground.cuh call them with one thread per point or one WARP per cell; compiled for the host (tests only,
// tests/harness/ground_host.cu) the same source runs with a "warp" of one lane, which lets the CPU test-suite check
// the sequential semantics (list order inside a cell, the shared random stream, the modulo-by-position sampling)
// before the code ever meets a GPU. The product path never executes the host instantiation.
//
// How the sequential reference maps onto independent work items:
//  * the reference fills grid[id].point_id by walking the cloud in index order; here the (cell, index) pairs are
//    radix-sorted (stable) so that a cell's list is a contiguous run in index order;
//  * grid[id].dist2station is "the range of the first point that arrives while the cell is still empty", re-assigned
//    by every point until the first counted one (:1737-1740): for a high point j that is range(j) if j precedes the
//    cell's first counted point and range(first counted point) otherwise; the per-cell stage always sees the latter;
//  * `j % rate` inside a cell is the position in the list (:1857, :1869, :1886), a warp-ordered slot here;
//  * every pcl::SampleConsensusModel object seeds its boost::mt19937 with 12345u, so all cells draw from the same
//    stream: its first kSacDraws outputs are tabulated once (host) and indexed per cell.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>

#include "../../include/mulls_b200/abi.h"

#if defined(__CUDACC__)
#define GF_HD __host__ __device__ __forceinline__
#else
#define GF_HD inline
#endif

namespace mulls {

constexpr int kSacDraws = 16384;      // mt19937 outputs available to one plane fit (5461 sample attempts)
constexpr uint32_t kGfNoCell = 0xffffffffu;

struct GfState {
    // k_gf_stats / k_gf_setup
    int bb[4];          // ordered-int encoded min_x, min_y, max_x, max_y
    float sum_height;
    int count_checkpoint;
    float appro_mean_height, non_ground_height_thre;
    double min_x, min_y, max_x, max_y;
    int row, col, num_grid;
    // counts
    uint32_t n_high, n_ground, n_unground, n_ground_down;
};

struct GfArgs {
    mulls_ground_params P;
    uint32_t n;
    const float4 *rows;   // cloud_in, 3 float4 per point
    GfState *st;
    // per point
    uint32_t *key, *idx;          // (cell | kGfNoCell, index) before the sort
    uint32_t *key_s, *idx_s;      // after the stable sort by cell
    int *cell_all;                // cell of every point (-1: outside the grid), for the high points
    uint32_t *high_flag, *high_pos;
    uint8_t *decision;            // per sorted position: 0 dropped, 1 ground, 2 unground
    float4 *cand;                 // per sorted position: candidate cloud of the cell (x y z, sorted position as bits)
    int *shuf;                    // per sorted position: shuffled_indices_ of the cell's SAC model
    uint8_t *inl;                 // per sorted position: refined inlier flag of the candidate
    // per cell
    uint32_t *cell_start, *cell_end;
    float *min_z, *neighbor_min_z, *outlier_thre;
    int *reliable;
    float4 *cell_normal;
    uint32_t *cell_ng, *cell_nu, *cell_og, *cell_ou;
    const uint32_t *draws;        // mt19937(12345) outputs
    float4 *out_ground, *out_ground_down, *out_unground;
};

// ---- the "warp": 32 lanes on the device, one lane on the host -------------------------------------------------------
struct Coop {
    GF_HD static int lane() {
#ifdef __CUDA_ARCH__
        return (int)(threadIdx.x & 31u);
#else
        return 0;
#endif
    }
    GF_HD static int width() {
#ifdef __CUDA_ARCH__
        return 32;
#else
        return 1;
#endif
    }
    GF_HD static int sum(int v) {
#ifdef __CUDA_ARCH__
        return (int)__reduce_add_sync(0xffffffffu, v);
#else
        return v;
#endif
    }
    GF_HD static float minf(float v) {
#ifdef __CUDA_ARCH__
        for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
#endif
        return v;
    }
    // slot of this lane among the lanes with pred (lane order); total = number of such lanes
    GF_HD static int slot(bool pred, int &total) {
#ifdef __CUDA_ARCH__
        const unsigned m = __ballot_sync(0xffffffffu, pred);
        total = __popc(m);
        return __popc(m & ((1u << (threadIdx.x & 31u)) - 1u));
#else
        total = pred ? 1 : 0;
        return 0;
#endif
    }
    GF_HD static int bcast(int v) {
#ifdef __CUDA_ARCH__
        return __shfl_sync(0xffffffffu, v, 0);
#else
        return v;
#endif
    }
    GF_HD static void sync() {
#ifdef __CUDA_ARCH__
        __syncwarp();
#endif
    }
};

GF_HD int gf_ord(float f) {
    int i;
#ifdef __CUDA_ARCH__
    i = __float_as_int(f);
#else
    union { float f; int i; } u;
    u.f = f;
    i = u.i;
#endif
    return i >= 0 ? i : (i ^ 0x7fffffff);
}
GF_HD float gf_unord(int i) {
    i = i >= 0 ? i : (i ^ 0x7fffffff);
#ifdef __CUDA_ARCH__
    return __int_as_float(i);
#else
    union { float f; int i; } u;
    u.i = i;
    return u.f;
#endif
}
GF_HD float gf_bits_to_float(uint32_t b) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    union { float f; uint32_t u; } u;
    u.u = b;
    return u.f;
#endif
}
GF_HD uint32_t gf_float_to_bits(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    union { float f; uint32_t u; } u;
    u.f = f;
    return u.u;
#endif
}

// (int)(float) as the x86 cvttss2si of the reference build: out of range -> INT_MIN (CUDA's cast would saturate)
GF_HD int gf_to_int_x86(float f) {
    if (!(f > -2147483904.0f && f < 2147483648.0f)) return INT_MIN;
    return (int)f;
}

// rate_temp of :1744-1748 / :1838-1850: method 1 linear, 2 quadratic, else the plain rate
GF_HD int gf_rate(int method, float distance_weight, int rate) {
    if (method == 1) return gf_to_int_x86(distance_weight * rate + 1);
    if (method == 2) return gf_to_int_x86(distance_weight * distance_weight * rate + 1);
    return rate;
}
GF_HD float gf_distance_weight(float standard_distance, float dist2station) {
    return (float)(1.0 * standard_distance / (dist2station + 0.0001)); // double expression stored in a float (:1743, :1836)
}
GF_HD float gf_range(const float4 a) { return sqrtf(a.x * a.x + a.y * a.y + a.z * a.z); } // :1739

// ---- per point: grid cell and role (:1728-1766) -----------------------------------------------------------------------
GF_HD void gf_assign_point(const GfArgs &A, uint32_t j) {
    const GfState &S = *A.st;
    const float4 a = A.rows[3 * (size_t)j];
    const float gr = A.P.grid_resolution;
    const int temp_col = (int)floor(((double)a.x - S.min_x) / (double)gr);
    const int temp_row = (int)floor(((double)a.y - S.min_y) / (double)gr);
    const int temp_id = temp_row * S.col + temp_col;
    uint32_t key = kGfNoCell;
    int cell = -1;
    if (temp_id >= 0 && temp_id < S.num_grid) {
        cell = temp_id;
        if (!(a.z > S.non_ground_height_thre) && a.z > -FLT_MAX) key = (uint32_t)temp_id; // counted point
    }
    A.key[j] = key;
    A.idx[j] = j;
    A.cell_all[j] = cell;
}

// ---- per sorted position: list boundaries of the cells ---------------------------------------------------------------
GF_HD void gf_mark_bounds(const GfArgs &A, uint32_t i) {
    const uint32_t k = A.key_s[i];
    if (k == kGfNoCell) return;
    if (i == 0 || A.key_s[i - 1] != k) A.cell_start[k] = i;
    if (i + 1 == A.n || A.key_s[i + 1] != k) A.cell_end[k] = i + 1;
}

// ---- per cell (cooperative): lowest point, optional grid-wise outlier filter (:1769-1788) ------------------------------
GF_HD void gf_cell_min(const GfArgs &A, int c) {
    const uint32_t start = A.cell_start[c], cnt = A.cell_end[c] - start;
    const int W = Coop::width(), lane = Coop::lane();
    float mz = FLT_MAX;
    for (uint32_t base = 0; base < cnt; base += W) {
        const uint32_t j = base + lane;
        if (j < cnt) mz = fminf(mz, A.rows[3 * (size_t)A.idx_s[start + j]].z);
    }
    mz = Coop::minf(mz);
    float othre = -FLT_MAX;
    if (A.P.apply_grid_wise_outlier_filter && (int)cnt >= A.P.min_grid_pt_num) {
        // sequential double sums in list order (every lane computes the same values)
        double sum_z = 0, sum_z2 = 0;
        for (uint32_t j = 0; j < cnt; ++j) sum_z += A.rows[3 * (size_t)A.idx_s[start + j]].z;
        const double mean_z = sum_z / (int)cnt;
        for (uint32_t j = 0; j < cnt; ++j) {
            const float z = A.rows[3 * (size_t)A.idx_s[start + j]].z;
            sum_z2 += (z - mean_z) * (z - mean_z);
        }
        const double std_z = sqrt(sum_z2 / (int)cnt);
        othre = (float)(mean_z - A.P.outlier_std_scale * std_z);
        mz = (mz > othre) ? mz : othre; // max_(min_z, min_z_outlier_thre)
    }
    if (lane == 0) {
        A.min_z[c] = mz; // FLT_MAX for an empty cell (:1722-1725)
        A.outlier_thre[c] = othre;
    }
}

// ---- per cell (one thread): 3x3 neighbourhood (:1793-1810) -------------------------------------------------------------
GF_HD void gf_cell_neighbors(const GfArgs &A, int m) {
    const GfState &S = *A.st;
    const int row = S.row, col = S.col;
    const int temp_row = m / col, temp_col = m % col;
    float nb = A.min_z[m];
    int reliable = 0;
    if (temp_row >= 1 && temp_row <= row - 2 && temp_col >= 1 && temp_col <= col - 2) {
        const int thre = A.P.min_grid_pt_num - 1;
        for (int j = -1; j <= 1; ++j)
            for (int k = -1; k <= 1; ++k) {
                const int q = m + j * col + k;
                const float z = A.min_z[q];
                nb = (nb < z) ? nb : z;
                if ((int)(A.cell_end[q] - A.cell_start[q]) > thre) ++reliable;
            }
    }
    A.neighbor_min_z[m] = nb;
    A.reliable[m] = reliable;
}

// ---- per point: the high points that go straight to cloud_unground (:1742-1755) --------------------------------------
GF_HD void gf_high_point(const GfArgs &A, uint32_t j) {
    const GfState &S = *A.st;
    uint32_t flag = 0;
    const int cell = A.cell_all[j];
    if (cell >= 0) {
        const float4 a = A.rows[3 * (size_t)j];
        if (a.z > S.non_ground_height_thre) {
            int rate = A.P.nonground_random_down_rate;
            if (A.P.distance_weight_downsampling_method > 0) {
                const uint32_t cs = A.cell_start[cell], ce = A.cell_end[cell];
                const uint32_t first = (ce > cs) ? A.idx_s[cs] : 0xffffffffu; // first counted point of the cell
                const float d2s = (j < first) ? gf_range(a) : gf_range(A.rows[3 * (size_t)first]);
                rate = gf_rate(A.P.distance_weight_downsampling_method, gf_distance_weight(A.P.standard_distance, d2s), rate);
            }
            const float intensity = A.rows[3 * (size_t)j + 2].x;
            if ((int)j % rate == 0 || intensity > A.P.intensity_thre) flag = 1;
        }
    }
    A.high_flag[j] = flag;
}
GF_HD void gf_high_emit(const GfArgs &A, uint32_t j) {
    if (!A.high_flag[j]) return;
    const float4 *r = A.rows + 3 * (size_t)j;
    float4 *o = A.out_unground + 3 * (size_t)A.high_pos[j];
    float4 a = r[0];
    a.w = (float)((double)a.z - ((double)A.st->appro_mean_height - 3.0)); // :1752
    o[0] = a, o[1] = r[1], o[2] = r[2];
}

// ---- pcl::computeMeanAndCovarianceMatrix (PCL 1.10): float accumulator xx xy xz yy yz zz x y z, in point order ----------
GF_HD void gf_mean_cov_add(float accu[9], float x, float y, float z) {
    accu[0] += x * x, accu[1] += x * y, accu[2] += x * z, accu[3] += y * y, accu[4] += y * z, accu[5] += z * z;
    accu[6] += x, accu[7] += y, accu[8] += z;
}
// accu /= count; the centroid is accu[6..8] afterwards
GF_HD void gf_mean_cov_finish(float accu[9], float count, float cov[3][3]) {
    for (int i = 0; i < 9; ++i) accu[i] /= count;
    cov[0][0] = accu[0] - accu[6] * accu[6];
    cov[0][1] = accu[1] - accu[6] * accu[7];
    cov[0][2] = accu[2] - accu[6] * accu[8];
    cov[1][1] = accu[3] - accu[7] * accu[7];
    cov[1][2] = accu[4] - accu[7] * accu[8];
    cov[2][2] = accu[5] - accu[8] * accu[8];
    cov[1][0] = cov[0][1], cov[2][0] = cov[0][2], cov[2][1] = cov[1][2];
}

// ---- pcl::SampleConsensusModelPlane pieces (PCL 1.10) ------------------------------------------------------------------
// model_coefficients.dot(Vector4f(x, y, z, 1)): Eigen's 4-wide packet reduction (a0+a2)+(a1+a3)
GF_HD float gf_plane_dot(const float c[4], float x, float y, float z) { return (c[0] * x + c[2] * z) + (c[1] * y + c[3] * 1.0f); }

GF_HD bool gf_plane_from_sample(const float4 p0, const float4 p1, const float4 p2, float c[4]) {
    const float a0 = p1.x - p0.x, a1 = p1.y - p0.y, a2 = p1.z - p0.z;
    const float b0 = p2.x - p0.x, b1 = p2.y - p0.y, b2 = p2.z - p0.z;
    const float d0 = a0 / b0, d1 = a1 / b1, d2 = a2 / b2;
    if ((d0 == d1) && (d2 == d1)) return false; // collinear
    c[0] = a1 * b2 - a2 * b1;
    c[1] = a2 * b0 - a0 * b2;
    c[2] = a0 * b1 - a1 * b0;
    c[3] = 0.0f;
    const float z = (c[0] * c[0] + c[2] * c[2]) + (c[1] * c[1] + c[3] * c[3]);
    if (z > 0.0f) {
        const float nrm = sqrtf(z);
        c[0] /= nrm, c[1] /= nrm, c[2] /= nrm, c[3] /= nrm;
    }
    // head<4>().dot(p0): the 4th product is 0 * data[3] (the row's padding; assumed finite)
    c[3] = -1.0f * ((c[0] * p0.x + c[2] * p0.z) + (c[1] * p0.y + c[3] * 0.0f));
    return true;
}

GF_HD void gf_roots2(float b, float c, float r[3]) {
    r[0] = 0.0f;
    float d = (float)((double)(b * b) - 4.0 * (double)c);
    if (d < 0.0f) d = 0.0f;
    const float sd = sqrtf(d);
    r[2] = 0.5f * (b + sd);
    r[1] = 0.5f * (b - sd);
}
GF_HD void gf_swapf(float &a, float &b) {
    const float t = a;
    a = b;
    b = t;
}
GF_HD void gf_roots(const float m[3][3], float r[3]) {
    const float c0 = m[0][0] * m[1][1] * m[2][2] + 2.0f * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                     m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
    const float c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] + m[1][1] * m[2][2] -
                     m[1][2] * m[1][2];
    const float c2 = m[0][0] + m[1][1] + m[2][2];
    if (fabsf(c0) < FLT_EPSILON) {
        gf_roots2(c2, c1, r);
        return;
    }
    const float s_inv3 = (float)(1.0 / 3.0);
    const float s_sqrt3 = sqrtf(3.0f);
    const float c2_over_3 = c2 * s_inv3;
    float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.0f) a_over_3 = 0.0f;
    const float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
    float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.0f) q = 0.0f;
    const float rho = sqrtf(-a_over_3);
    // atan2f / cosf / sinf of the reference, evaluated in double and rounded (a correctly rounded float result)
    const float theta = (float)atan2((double)sqrtf(-q), (double)half_b) * s_inv3;
    const float cos_theta = (float)cos((double)theta);
    const float sin_theta = (float)sin((double)theta);
    r[0] = c2_over_3 + 2.0f * rho * cos_theta;
    r[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    r[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    if (r[0] >= r[1]) gf_swapf(r[0], r[1]);
    if (r[1] >= r[2]) {
        gf_swapf(r[1], r[2]);
        if (r[0] >= r[1]) gf_swapf(r[0], r[1]);
    }
    if (r[0] <= 0.0f) gf_roots2(c2, c1, r);
}
GF_HD void gf_cross(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
// pcl::eigen33's scaling: mat / max|mat_ij| (1 when that is at most FLT_MIN; a NaN entry does not raise it)
GF_HD float gf_eigen33_scale(const float mat[3][3], float m[3][3]) {
    float scale = 0.0f;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) scale = fmaxf(scale, fabsf(mat[i][j]));
    if (scale <= FLT_MIN) scale = 1.0f;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[i][j] = mat[i][j] / scale;
    return scale;
}
// pcl::eigen33(mat, eigenvalues): the roots of the scaled matrix, ascending, times the scale
GF_HD void gf_eigen33_values(const float mat[3][3], float evals[3]) {
    float m[3][3];
    const float scale = gf_eigen33_scale(mat, m);
    gf_roots(m, evals);
    evals[0] *= scale, evals[1] *= scale, evals[2] *= scale;
}
// pcl::eigen33(mat, eigenvalue, eigenvector): eigenvector of the smallest eigenvalue
GF_HD void gf_eigen33_smallest(const float mat[3][3], float evec[3]) {
    float m[3][3];
    gf_eigen33_scale(mat, m);
    float r[3];
    gf_roots(m, r);
    for (int i = 0; i < 3; ++i) m[i][i] -= r[0];
    float v1[3], v2[3], v3[3];
    gf_cross(m[0], m[1], v1);
    gf_cross(m[0], m[2], v2);
    gf_cross(m[1], m[2], v3);
    const float l1 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2];
    const float l2 = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2];
    const float l3 = v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2];
    const float *v = v3;
    float len = l3;
    if (l1 >= l2 && l1 >= l3) v = v1, len = l1;
    else if (l2 >= l1 && l2 >= l3) v = v2, len = l2;
    const float s = sqrtf(len);
    evec[0] = v[0] / s, evec[1] = v[1] / s, evec[2] = v[2] / s;
}

// pcl::SACSegmentation::segment for a plane over the candidate cloud cx[0..n) of one cell. Cooperative: every lane runs
// the same control flow; the sample draws are done by lane 0, the point loops are split over the lanes. On success the
// refined inlier flags are in inl[0..n) and the refined coefficients in coeff.
GF_HD bool gf_sac_plane(const float4 *cx, int n, double threshold, int max_iterations, const uint32_t *draws, int *shuf,
                        uint8_t *inl, float coeff[4]) {
    const int W = Coop::width(), lane = Coop::lane();
    if (n < 3) return false;
    for (int i = lane; i < n; i += W) shuf[i] = i;
    Coop::sync();
    int iterations = 0, n_best = -INT_MAX, next = 0;
    double k = 1.0;
    const double log_probability = log(1.0 - 0.99);
    const double one_over_indices = 1.0 / (double)n;
    unsigned skipped = 0;
    const unsigned max_skip = (unsigned)max_iterations * 10u;
    bool have = false;
    float best[4] = {0.f, 0.f, 0.f, 0.f};
    while ((double)iterations < k && skipped < max_skip) {
        // SampleConsensusModel::getSamples / drawIndexSample / isSampleGood
        int got = 0, s0 = 0, s1 = 0, s2 = 0;
        if (lane == 0) {
            for (int iter = 0; iter < 1000 && !got; ++iter) {
                if (next + 3 > kSacDraws) break; // draw table exhausted (degenerate cell): no sample
                for (int i = 0; i < 3; ++i) {
                    const uint32_t r = draws[next++] >> 1; // boost::uniform_int<>(0, INT_MAX) on mt19937
                    const int o = i + (int)(r % (uint32_t)(n - i));
                    const int t = shuf[i];
                    shuf[i] = shuf[o];
                    shuf[o] = t;
                }
                s0 = shuf[0], s1 = shuf[1], s2 = shuf[2];
                const float4 p0 = cx[s0], p1 = cx[s1], p2 = cx[s2];
                const float d0 = (p1.x - p0.x) / (p2.x - p0.x), d1 = (p1.y - p0.y) / (p2.y - p0.y),
                            d2 = (p1.z - p0.z) / (p2.z - p0.z);
                got = ((d0 != d1) || (d2 != d1)) ? 1 : 0;
            }
        }
        got = Coop::bcast(got), s0 = Coop::bcast(s0), s1 = Coop::bcast(s1), s2 = Coop::bcast(s2), next = Coop::bcast(next);
        if (!got) break;
        float c[4];
        if (!gf_plane_from_sample(cx[s0], cx[s1], cx[s2], c)) {
            ++skipped;
            continue;
        }
        int cnt = 0;
        for (int i = lane; i < n; i += W) {
            const float4 p = cx[i];
            if ((double)fabsf(gf_plane_dot(c, p.x, p.y, p.z)) < threshold) ++cnt;
        }
        cnt = Coop::sum(cnt);
        if (cnt > n_best) {
            n_best = cnt;
            have = true;
            best[0] = c[0], best[1] = c[1], best[2] = c[2], best[3] = c[3];
            const double w = (double)n_best * one_over_indices;
            double p_no_outliers = 1.0 - pow(w, 3.0);
            p_no_outliers = (p_no_outliers > DBL_EPSILON) ? p_no_outliers : DBL_EPSILON;
            p_no_outliers = (p_no_outliers < 1.0 - DBL_EPSILON) ? p_no_outliers : 1.0 - DBL_EPSILON;
            k = log_probability / log(p_no_outliers);
        }
        ++iterations;
        if (iterations > max_iterations) break;
    }
    if (!have) return false;
    // inliers of the best model; optimizeModelCoefficients: float mean / covariance accumulated in index order
    float accu[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int n_inl = 0;
    for (int i = 0; i < n; ++i) { // every lane walks the whole list: the sums are order dependent
        const float4 p = cx[i];
        if ((double)fabsf(gf_plane_dot(best, p.x, p.y, p.z)) < threshold) {
            ++n_inl;
            gf_mean_cov_add(accu, p.x, p.y, p.z);
        }
    }
    if (n_inl == 0) return false;
    coeff[0] = best[0], coeff[1] = best[1], coeff[2] = best[2], coeff[3] = best[3];
    if (n_inl >= 4) {
        float cov[3][3];
        gf_mean_cov_finish(accu, (float)n_inl, cov);
        float ev[3];
        gf_eigen33_smallest(cov, ev);
        coeff[0] = ev[0], coeff[1] = ev[1], coeff[2] = ev[2], coeff[3] = 0.0f;
        coeff[3] = -1.0f * ((coeff[0] * accu[6] + coeff[2] * accu[8]) + (coeff[1] * accu[7] + coeff[3] * 1.0f));
    }
    for (int i = lane; i < n; i += W) {
        const float4 p = cx[i];
        inl[i] = ((double)fabsf(gf_plane_dot(coeff, p.x, p.y, p.z)) < threshold) ? 1 : 0;
    }
    Coop::sync();
    return true;
}

// ---- per cell (cooperative): the two-threshold test, the position-modulo sampling and the plane (:1830-1927) -----------
GF_HD void gf_cell_decide(const GfArgs &A, int c) {
    const mulls_ground_params &P = A.P;
    const uint32_t start = A.cell_start[c], cnt = A.cell_end[c] - start;
    const int W = Coop::width(), lane = Coop::lane();
    if (!((int)cnt >= P.min_grid_pt_num && A.reliable[c] >= P.reliable_neighbor_grid_num_thre)) {
        for (uint32_t j = lane; j < cnt; j += W) A.decision[start + j] = 0;
        if (lane == 0) A.cell_ng[c] = 0, A.cell_nu[c] = 0;
        return;
    }
    const float min_z = A.min_z[c], nb = A.neighbor_min_z[c], othre = A.outlier_thre[c];
    int ground_rate = P.ground_random_down_rate, nonground_rate = P.nonground_random_down_rate;
    if (P.distance_weight_downsampling_method > 0) {
        const float d2s = gf_range(A.rows[3 * (size_t)A.idx_s[start]]); // the cell's first counted point
        const float dw = gf_distance_weight(P.standard_distance, d2s);
        ground_rate = gf_rate(P.distance_weight_downsampling_method, dw, P.ground_random_down_rate);
        nonground_rate = gf_rate(P.distance_weight_downsampling_method, dw, P.nonground_random_down_rate);
    }
    const bool ground_cell = (min_z - nb < P.neighbor_height_diff);
    const int method = P.estimate_ground_normal_method;
    int ng = 0, nu = 0, ncand = 0;
    for (uint32_t base = 0; base < cnt; base += W) {
        const uint32_t j = base + lane;
        const bool in = j < cnt;
        int dec = 0;
        bool cand = false;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in) {
            const size_t pid = A.idx_s[start + j];
            a = A.rows[3 * pid];
            if (a.z > othre) {
                const float intensity = A.rows[3 * pid + 2].x;
                const bool take_u = ((int)j % nonground_rate == 0) || (intensity > P.intensity_thre);
                if (ground_cell) {
                    if (a.z - min_z < P.max_height_difference) {
                        if (method == 3) cand = true;
                        else if ((int)j % ground_rate == 0) dec = 1;
                    } else if (take_u) dec = 2;
                } else if (take_u) dec = 2;
            }
            A.decision[start + j] = (uint8_t)dec;
        }
        int tot;
        const int s = Coop::slot(cand, tot);
        if (cand) A.cand[start + ncand + s] = make_float4(a.x, a.y, a.z, gf_bits_to_float(start + j));
        ncand += tot;
        ng += (dec == 1), nu += (dec == 2);
    }
    ng = Coop::sum(ng), nu = Coop::sum(nu);
    Coop::sync();
    if (method == 3 && ncand >= P.min_grid_pt_num) {
        float coeff[4];
        const float dist_thre = (float)(0.3 * P.max_height_difference); // float argument of estimate_ground_normal_by_ransac
        if (gf_sac_plane(A.cand + start, ncand, (double)dist_thre, 20, A.draws, A.shuf + start, A.inl + start, coeff)) {
            const bool nz_ok = (double)fabsf(coeff[2]) > 0.8;
            int run = 0, sel = 0;
            for (int base = 0; base < ncand; base += W) {
                const int i = base + lane;
                const bool f = (i < ncand) && A.inl[start + i];
                int tot;
                const int jj = run + Coop::slot(f, tot);
                if (f && nz_ok && (jj % ground_rate == 0)) {
                    A.decision[gf_float_to_bits(A.cand[start + i].w)] = 1;
                    ++sel;
                }
                run += tot;
            }
            ng += Coop::sum(sel);
            if (lane == 0) A.cell_normal[c] = make_float4(coeff[0], coeff[1], coeff[2], 0.f);
        }
    }
    if (lane == 0) A.cell_ng[c] = (uint32_t)ng, A.cell_nu[c] = (uint32_t)nu;
}

// ---- per cell (cooperative): write the cell's ground / unground rows at their offsets (:1930-1934) -------------------
GF_HD void gf_cell_emit(const GfArgs &A, int c) {
    const uint32_t ng = A.cell_ng[c], nu = A.cell_nu[c];
    if (ng == 0 && nu == 0) return;
    const uint32_t start = A.cell_start[c], cnt = A.cell_end[c] - start;
    const int W = Coop::width(), lane = Coop::lane();
    const float min_z = A.min_z[c], nb = A.neighbor_min_z[c];
    const bool ground_cell = (min_z - nb < A.P.neighbor_height_diff);
    const int method = A.P.estimate_ground_normal_method;
    const float4 nrm = (method == 3) ? A.cell_normal[c] : make_float4(0.f, 0.f, 1.f, 0.f);
    size_t og = A.cell_og[c], ou = (size_t)A.st->n_high + A.cell_ou[c];
    for (uint32_t base = 0; base < cnt; base += W) {
        const uint32_t j = base + lane;
        const int dec = (j < cnt) ? A.decision[start + j] : 0;
        int tg, tu;
        const int sg = Coop::slot(dec == 1, tg);
        const int su = Coop::slot(dec == 2, tu);
        if (dec) {
            const float4 *r = A.rows + 3 * (size_t)A.idx_s[start + j];
            float4 a = r[0], b = r[1];
            float4 *o;
            if (dec == 1) {
                if (method == 0 || method == 3) b.x = nrm.x, b.y = nrm.y, b.z = nrm.z;
                o = A.out_ground + 3 * (og + sg);
            } else {
                a.w = ground_cell ? (a.z - min_z) : (a.z - nb); // data[3]: height above ground (:1880, :1894)
                o = A.out_unground + 3 * (ou + su);
            }
            o[0] = a, o[1] = b, o[2] = r[2];
        }
        og += tg, ou += tu;
    }
}

// ---- CFilter::voxel_downsample, cfilter.hpp:83-165 ---------------------------------------------------------------------
// one point per occupied voxel, output in voxel-index order. std::sort on idpair_t compares the voxel index only (:42)
// and is unstable: which point of a voxel leads its run is unspecified in the reference — here the lowest index
// (stable radix sort).
struct VxState {
    int bb[6];               // ordered-int encoded min xyz, max xyz (pcl::getMinMax3D)
    float mn[3];
    float inv;               // inverse_voxel_size (:99)
    unsigned long long mul_vx, mul_vy; // :117-119
    uint32_t n_out;
};
GF_HD void vx_setup(VxState &S, float voxel_size) {
    float mx[3];
    for (int d = 0; d < 3; ++d) S.mn[d] = gf_unord(S.bb[d]), mx[d] = gf_unord(S.bb[3 + d]);
    S.inv = 1.0f / voxel_size;
    const unsigned long long max_vy = (unsigned long long)(ceilf((mx[1] - S.mn[1]) * S.inv) + 1.0f);
    const unsigned long long max_vz = (unsigned long long)(ceilf((mx[2] - S.mn[2]) * S.inv) + 1.0f);
    S.mul_vx = max_vy * max_vz;
    S.mul_vy = max_vz;
}
GF_HD unsigned long long vx_key(const VxState &S, const float4 a) { // :128-132
    const unsigned long long vx = (unsigned long long)floorf((a.x - S.mn[0]) * S.inv);
    const unsigned long long vy = (unsigned long long)floorf((a.y - S.mn[1]) * S.inv);
    const unsigned long long vz = (unsigned long long)floorf((a.z - S.mn[2]) * S.inv);
    return vx * S.mul_vx + vy * S.mul_vy + vz;
}

} // namespace mulls
