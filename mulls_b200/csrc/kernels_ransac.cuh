// RANSAC coarse registration on the device (CRegistration::coarse_reg_ransac, cregistration.hpp:604-661): the readings
// and the shared arithmetic are in ransac_core.cuh. The sample stream is sequential (each attempt depends on the swaps
// before it) and is drawn on the host; these kernels fit and score the hypotheses and run the whole refinement.
//  - k_ransac_fit: one thread per hypothesis, the Umeyama fit of its three correspondences into a float 3x4;
//  - k_ransac_count: H hypotheses x N correspondences; a tile of correspondences is staged in shared memory and read as
//    broadcasts, each thread keeps kRcHypPerThread hypotheses in registers and adds integer counts (order independent);
//  - k_ransac_refine: one block of kRcLanes threads runs computeModel's final selectWithinDistance and the whole
//    SampleConsensus::refineModel loop: inlier flags and squared errors, the median by a radix select on the float
//    bits of the errors (non-negative, so the bit order is the value order), the fit in the fixed order of
//    ransac_core.cuh (C1) and the changed / oscillating tests. No host round trip per round; at most
//    kRcRefineRounds rounds.
#pragma once
#include "ransac_core.cuh"

namespace mulls {

constexpr int kRcFitBlock = 128;
constexpr int kRcCountBlock = 128;
constexpr int kRcHypPerThread = 4;
constexpr int kRcTile = 256; // correspondences staged per block

// what the refinement hands back
struct RcRefineOut {
    float T[12];     // the model the rejector reads (rows 0..2 of the float 4x4)
    int ok;          // refineModel's return value
    int n_inliers;   // inliers_.size() after it (meaningful when ok)
};

__global__ void __launch_bounds__(kRcFitBlock) k_ransac_fit(const float *__restrict__ corr, const int *__restrict__ samples, int H,
                                                            float *__restrict__ T) {
    const int h = blockIdx.x * kRcFitBlock + threadIdx.x;
    if (h >= H) return;
    const int s[3] = {samples[3 * h], samples[3 * h + 1], samples[3 * h + 2]};
    float t[12];
    rc_fit_sample(corr, s, t);
    for (int c = 0; c < 12; ++c) T[12 * (size_t)h + c] = t[c];
}

// grid (ceil(H / (kRcCountBlock * kRcHypPerThread)), ceil(n / kRcTile)); counts zeroed before
__global__ void __launch_bounds__(kRcCountBlock) k_ransac_count(const float *__restrict__ corr, int n, const float *__restrict__ T,
                                                                int H, double thresh_sq, int *__restrict__ counts) {
    __shared__ float sc[kRcTile * 6];
    const int j0 = blockIdx.y * kRcTile, m = min(kRcTile, n - j0);
    for (int i = threadIdx.x; i < m * 6; i += kRcCountBlock) sc[i] = corr[6 * (size_t)j0 + i];
    float t[kRcHypPerThread][12];
    int cnt[kRcHypPerThread];
    const int h0 = blockIdx.x * kRcCountBlock * kRcHypPerThread + threadIdx.x;
#pragma unroll
    for (int k = 0; k < kRcHypPerThread; ++k) {
        cnt[k] = 0;
        const int h = min(h0 + k * kRcCountBlock, H - 1);
#pragma unroll
        for (int c = 0; c < 12; ++c) t[k][c] = T[12 * (size_t)h + c];
    }
    __syncthreads();
    for (int j = 0; j < m; ++j) {
        const float *c6 = sc + 6 * j;
#pragma unroll
        for (int k = 0; k < kRcHypPerThread; ++k) cnt[k] += rc_within(t[k], c6, thresh_sq) ? 1 : 0;
    }
#pragma unroll
    for (int k = 0; k < kRcHypPerThread; ++k) {
        const int h = h0 + k * kRcCountBlock;
        if (h < H && cnt[k]) atomicAdd(counts + h, cnt[k]);
    }
}

struct RcRefineArgs {
    const float *corr;
    int n;
    const float *T_best;   // the best hypothesis (12 floats)
    double threshold;      // inlier_threshold_ (noise_bound)
    uint8_t *flag_a, *flag_b;
    float *err;            // squared errors of the current selection
    RcRefineOut *out;
};

namespace rc_detail {
// selectWithinDistance: flags, squared errors, the count
__device__ __forceinline__ int select(const RcRefineArgs &A, const float *T, double thresh_sq, uint8_t *flag, float *err, int *s_cnt) {
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int j = threadIdx.x; j < A.n; j += kRcLanes) {
        const float e = rc_sq_error(T, A.corr + 6 * (size_t)j);
        const bool in = (double)e < thresh_sq;
        flag[j] = in ? 1 : 0;
        if (in && err) err[j] = e;
        c += in ? 1 : 0;
    }
    if (c) atomicAdd(s_cnt, c);
    __syncthreads();
    const int r = *s_cnt;
    __syncthreads();
    return r;
}
// K fixed-order sums over the flagged correspondences (ransac_core.cuh C1): one lane per partial
template <int K, class Value>
__device__ __forceinline__ void sums(const RcRefineArgs &A, const uint8_t *flag, Value v, double (*part)[kRcLanes], double out[K]) {
    const int t = threadIdx.x, m = min(A.n, kRcLanes);
    double q[K];
    for (int c = 0; c < K; ++c) q[c] = 0.0;
    for (int j = t; j < A.n; j += kRcLanes)
        if (flag[j]) {
            double x[K];
            v(j, x);
            for (int c = 0; c < K; ++c) q[c] += x[c];
        }
    for (int c = 0; c < K; ++c) part[c][t] = q[c];
    __syncthreads();
    for (int s = kRcLanes / 2; s > 0; s >>= 1) {
        if (t < s && t + s < m)
            for (int c = 0; c < K; ++c) part[c][t] += part[c][t + s];
        __syncthreads();
    }
    for (int c = 0; c < K; ++c) out[c] = m > 0 ? part[c][0] : 0.0;
    __syncthreads();
}
// Umeyama over the flagged correspondences (count n_fit) into sT
__device__ __forceinline__ void fit(const RcRefineArgs &A, const uint8_t *flag, int n_fit, double (*part)[kRcLanes], float *sT) {
    double ms[6], mean[6], cs[9];
    sums<6>(A, flag, [&](int j, double x[6]) { rc_point_terms(A.corr + 6 * (size_t)j, x); }, part, ms);
    const double one_over_n = 1.0 / (double)n_fit;
    rc_umeyama_means(ms, one_over_n, mean);
    sums<9>(A, flag, [&](int j, double x[9]) { rc_cross_terms(A.corr + 6 * (size_t)j, mean, x); }, part, cs);
    if (threadIdx.x == 0) rc_umeyama_finish(mean, cs, one_over_n, sT);
    __syncthreads();
}
// the value of rank `rank` among the flagged errors (0-based, ascending): radix select on the float bits, 8 at a time
__device__ __forceinline__ float median(const RcRefineArgs &A, const uint8_t *flag, int rank, uint32_t *hist, uint32_t *s_pre) {
    uint32_t prefix = 0, mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += kRcLanes) hist[b] = 0;
        __syncthreads();
        for (int j = threadIdx.x; j < A.n; j += kRcLanes)
            if (flag[j]) {
                const uint32_t bits = __float_as_uint(A.err[j]);
                if ((bits & mask) == prefix) atomicAdd(hist + ((bits >> shift) & 255u), 1u);
            }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t b = 0, below = 0;
            while (b < 255 && below + hist[b] <= (uint32_t)rank) below += hist[b++];
            s_pre[0] = prefix | (b << shift);
            s_pre[1] = (uint32_t)rank - below;
        }
        __syncthreads();
        prefix = s_pre[0];
        rank = (int)s_pre[1];
        mask |= 255u << shift;
        __syncthreads();
    }
    return __uint_as_float(prefix);
}
__device__ __forceinline__ bool flags_differ(const RcRefineArgs &A, const uint8_t *a, const uint8_t *b) {
    int d = 0;
    for (int j = threadIdx.x; j < A.n; j += kRcLanes) d |= (a[j] != b[j]) ? 1 : 0;
    return __syncthreads_or(d) != 0;
}
} // namespace rc_detail

// SampleConsensus::refineModel (sigma 3, kRcRefineRounds), after computeModel's selectWithinDistance of the best model.
// Every thread runs the same control flow on block-uniform values.
__global__ void __launch_bounds__(kRcLanes) k_ransac_refine(RcRefineArgs A) {
    using namespace rc_detail;
    __shared__ double part[9][kRcLanes];
    __shared__ uint32_t hist[256], s_pre[2];
    __shared__ float sBest[12], sFit[12];
    __shared__ int s_cnt;
    if (threadIdx.x < 12) sBest[threadIdx.x] = A.T_best[threadIdx.x];
    __syncthreads();
    const double thr_sqr0 = A.threshold * A.threshold;
    int n_prev = select(A, sBest, thr_sqr0, A.flag_a, nullptr, &s_cnt);
    const int n_initial = n_prev;
    uint8_t *prev = A.flag_a, *nw = A.flag_b;
    double err_thr = A.threshold;
    int it = 0, rounds = 0, n_new_vec = 0;  // rounds: entries of inliers_sizes
    bool changed = false, osc = false;
    int sz[4] = {0, 0, 0, 0}; // the last four entries of inliers_sizes
    for (;;) {
        fit(A, prev, n_prev, part, sFit);
        sz[0] = sz[1], sz[1] = sz[2], sz[2] = sz[3], sz[3] = n_prev; // inliers_sizes.push_back(prev_inliers.size())
        ++rounds;
        const int n_new = select(A, sFit, err_thr * err_thr, nw, A.err, &s_cnt);
        n_new_vec = n_new;
        if (n_new == 0) {
            ++it;
            if (it >= kRcRefineRounds) break;
        } else {
            const float med = median(A, nw, n_new >> 1, hist, s_pre);
            err_thr = rc_next_threshold(thr_sqr0, med);
            changed = false;
            uint8_t *t = prev;
            prev = nw, nw = t; // std::swap(prev_inliers, new_inliers)
            n_new_vec = n_prev;
            n_prev = n_new;
            if (n_new_vec != n_prev) {
                if (rounds >= 4 && sz[3] == sz[1] && sz[2] == sz[0]) {
                    osc = true;
                    break;
                }
                changed = true;
            } else if (flags_differ(A, prev, nw)) {
                changed = true;
            }
        }
        if (!(changed && ++it < kRcRefineRounds)) break;
    }
    if (threadIdx.x == 0) {
        RcRefineOut o;
        const float *T = sBest;
        if (n_new_vec == 0) {
            o.ok = 0, o.n_inliers = 0;
        } else if (osc) {
            o.ok = 1, o.n_inliers = n_initial; // inliers_ and model_coefficients_ stay computeModel's
        } else if (!changed) {
            o.ok = 1, o.n_inliers = n_prev, T = sFit;
        } else {
            o.ok = 0, o.n_inliers = 0;
        }
        for (int c = 0; c < 12; ++c) o.T[c] = T[c];
        *A.out = o;
    }
}

} // namespace mulls
