// Keypoint matching of lo::CRegistration<PointT>::find_feature_correspondence_ncc (include/common/cregistration.hpp
// :409-601), the NCC ("neighborhood category context") correspondences in front of the global registration:
//   k_ts_last_nan<8> / k_ts_extremes<8> + k_ncc_range   the target's intensity range (kernels_rawscan.cuh's folds)
//   k_ncc_descriptors    the 11-float descriptor of every keypoint of both clouds, SoA [11][n_t + n_s]
//   k_ncc_pairs<kOp>     every (target, source) pair of a tile: sources staged in shared memory, kNccRows targets per
//                        thread in registers. kOp selects what the pairs feed: the row argmin (plain mode), the row
//                        argmin and the column minimum (reciprocal mode), a radix-select histogram or the gather of the
//                        selected pairs (fixed-number mode). Distances are recomputed on every pass, never stored.
//   k_ncc_select_step    one radix-select digit from the histogram
//   k_ncc_pick           plain / reciprocal: the kept (i, j) of every target row, compacted in target order afterwards
//
// The readings this library fixes, where the reference's text leaves a choice (the CPU restatement under tests/harness
// states the same list):
//  1. Fewer than 10 keypoints in either cloud: nothing is computed, the output clouds stay as they are (:421-425).
//  2. Intensity range over the target only, with the macros max_(a, b) = a > b ? a : b, min_(a, b) = a < b ? a : b
//     (utility.hpp:31-32), started from FLT_MAX and from 0 (not -FLT_MAX). A NaN intensity becomes the running value and
//     the next point replaces it; equal values (+0 and -0) resolve to the later point. The source uses the target's range.
//  3. Descriptor: components 0-3 / 4-7 are the decimal digit pairs of (int)normal[0] / (int)normal[1] (/1000000,
//     %1000000/10000, %10000/100, %100, C++ integer semantics) converted to float; 8 is (i - min) / (max - min) in float,
//     times the double 255.0, rounded to float; 9 is normal[3] * 100 and 10 is data[3] * 30, in float. (int) of a NaN or
//     out-of-range float is the x86 result INT_MIN (x86_cvtt below: CUDA's conversion saturates instead). A constant
//     target intensity gives 0 / 0 and x / 0; the NaN and infinities that follow flow on unchanged.
//  4. Distance: d = 0.0f, d += fabsf(t[k] - s[k]) for k = 0..10, in float, in that order (-fmad=false: no contraction).
//     d is never negative: +0 or more, +inf or NaN.
//  5. Plain mode: per target i, the first j with d < best from (FLT_MAX, 0). NaN never wins; a row with no finite value
//     below FLT_MAX pairs with source 0. The first minimum is the lowest j among equal minima: the 64-bit key
//     (d bits << 32 | j) and an atomicMin give it whatever order the tiles finish in.
//  6. Reciprocal mode: target i is dropped iff best_i > d[r][j_i] + 0.0f for some target r, i.e. iff best_i exceeds the
//     minimum over the non-NaN values of column j_i (an empty minimum is +inf), so one pass decides both.
//  7. Fixed-number mode (reciprocal ignored): K = min_(corr_num, M) with M = n_t * n_s compared as size_t, so a negative
//     corr_num means M and 0 stays 0. The first K pairs in the total order (distance, pair index i * n_s + j), NaN after
//     every number, which is std::sort's output when ties keep push order. Pair indices are int in the reference:
//     M > INT_MAX is refused. Then the pairs are walked in order and one is skipped when its target or its source already
//     holds more than 6 kept pairs (at most 7 each); that walk is O(K) integer work and runs on the host.
//  8. The output clouds receive whole input rows, target and source in step, appended.
#pragma once
#include <cfloat>
#include <climits>

#include "kernels_rawscan.cuh"

namespace mulls {

constexpr int kNccDim = 11;
constexpr int kNccBlock = 128; // threads of a pair kernel block
constexpr int kNccRows = 4;    // target rows per thread
constexpr int kNccTileS = 256; // sources per block, staged in shared memory
constexpr int kNccBins = 256;  // radix-select digit: 8 bits
constexpr int kNccTileT = kNccBlock * kNccRows;
static_assert(kNccBins == kNccTileS, "the histogram reuses the column-minimum buffer");

// x86's cvttss2si: truncation inside [-2^31, 2^31), INT_MIN for everything else and for NaN
__device__ __forceinline__ int x86_cvtt(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN; }

// the order-preserving 32-bit key of a distance (d >= +0, +inf or NaN): its bits, NaN after +inf
__device__ __forceinline__ uint32_t ncc_key(float d) { return isnan(d) ? 0xffffffffu : __float_as_uint(d); }

// one thread: min / max as the macros leave them over the target's intensities (reading 2), from the state of
// k_ts_last_nan<8> / k_ts_extremes<8>
__global__ void k_ncc_range(const float *rows, uint32_t n_t, const TsState *st, float *range) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float mn, mx;
    if (st->last_nan == (unsigned long long)n_t) { // the last intensity is NaN: both folds end on it
        mn = mx = row_column<8>(rows, n_t - 1);
    } else {
        mx = row_column<8>(rows, (uint32_t)st->max_key);
        mn = row_column<8>(rows, ~(uint32_t)st->min_key);
        if (st->last_nan == 0ull) { // no NaN: the folds start from FLT_MAX / 0, earlier than every point
            mx = (0.0f > mx) ? 0.0f : mx;
            mn = (FLT_MAX < mn) ? FLT_MAX : mn;
        }
    }
    range[0] = mn;
    range[1] = mx;
}

// reading 3, one thread per keypoint of both clouds (the target's rows first)
__global__ void __launch_bounds__(kRawBlock) k_ncc_descriptors(const float *rows, uint32_t n, const float *range, float *desc) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *r = rows + 12 * (size_t)i;
    const int c = x86_cvtt(r[4]), f = x86_cvtt(r[5]); // normal[0], normal[1]
    desc[0 * (size_t)n + i] = (float)(c / 1000000);
    desc[1 * (size_t)n + i] = (float)((c % 1000000) / 10000);
    desc[2 * (size_t)n + i] = (float)((c % 10000) / 100);
    desc[3 * (size_t)n + i] = (float)(c % 100);
    desc[4 * (size_t)n + i] = (float)(f / 1000000);
    desc[5 * (size_t)n + i] = (float)((f % 1000000) / 10000);
    desc[6 * (size_t)n + i] = (float)((f % 10000) / 100);
    desc[7 * (size_t)n + i] = (float)(f % 100);
    const float mn = range[0], mx = range[1];
    desc[8 * (size_t)n + i] = (float)((double)((r[8] - mn) / (mx - mn)) * 255.0);
    desc[9 * (size_t)n + i] = r[7] * 100.0f;  // normal[3]
    desc[10 * (size_t)n + i] = r[3] * 30.0f;  // data[3]
}

// the radix select of the fixed-number mode. Mode 0 selects the K-th smallest distance key T, mode 1 (only when fewer
// pairs equal to T are taken than exist) the rank-th smallest pair index E among the pairs whose key is T
struct NccSelect {
    uint32_t prefix_key, prefix_idx; // the digits chosen so far
    uint32_t rank;                   // 0-based rank still to find below the prefix
    uint32_t T, E;                   // threshold key; last pair index taken at the threshold (~0u: all)
    uint32_t need_eq, count_eq;      // pairs at the threshold taken / present
    uint32_t pad;
    unsigned long long count; // pairs gathered
    uint32_t hist[kNccBins];
};

struct NccPairs {
    const float *desc; // [11][n_all]: targets in columns 0..n_t-1, sources in n_t..n_all-1
    uint32_t n_all, n_t, n_s;
};

enum NccOp { kNccRow = 0, kNccRowCol = 1, kNccHistKey = 2, kNccHistIdx = 3, kNccGather = 4 };

__device__ __forceinline__ float ncc_l1(const float (&t)[kNccDim], const float (&s)[12]) {
    float d = 0.0f;
#pragma unroll
    for (int k = 0; k < kNccDim; ++k) d += fabsf(t[k] - s[k]);
    return d;
}

// blockIdx.x: kNccTileT targets, blockIdx.y: kNccTileS sources. shift: the digit of a histogram pass; K: gather bound
template <int kOp>
__global__ void __launch_bounds__(kNccBlock) k_ncc_pairs(NccPairs P, unsigned long long *row_key, uint32_t *col_min,
                                                         NccSelect *sel, int shift, unsigned long long *gathered,
                                                         unsigned long long K) {
    __shared__ float4 s_src[kNccTileS][3];
    __shared__ uint32_t s_aux[kNccTileS]; // column minima (kNccRowCol) or the histogram
    const uint32_t j0 = blockIdx.y * kNccTileS;
    const uint32_t nj = min((uint32_t)kNccTileS, P.n_s - j0);
    for (uint32_t t = threadIdx.x; t < (uint32_t)kNccTileS; t += kNccBlock) {
        float v[12];
#pragma unroll
        for (int k = 0; k < kNccDim; ++k) v[k] = t < nj ? P.desc[(size_t)k * P.n_all + P.n_t + j0 + t] : 0.0f;
        v[11] = 0.0f;
        s_src[t][0] = make_float4(v[0], v[1], v[2], v[3]);
        s_src[t][1] = make_float4(v[4], v[5], v[6], v[7]);
        s_src[t][2] = make_float4(v[8], v[9], v[10], v[11]);
        s_aux[t] = kOp == kNccRowCol ? 0xffffffffu : 0u;
    }
    float td[kNccRows][kNccDim];
    uint32_t ti[kNccRows];
    bool tv[kNccRows];
#pragma unroll
    for (int r = 0; r < kNccRows; ++r) {
        ti[r] = blockIdx.x * kNccTileT + r * kNccBlock + threadIdx.x;
        tv[r] = ti[r] < P.n_t;
#pragma unroll
        for (int k = 0; k < kNccDim; ++k) td[r][k] = tv[r] ? P.desc[(size_t)k * P.n_all + ti[r]] : 0.0f;
    }
    uint32_t pre = 0, T = 0, E = 0;
    if (kOp == kNccHistKey) pre = sel->prefix_key;
    if (kOp == kNccHistIdx) pre = sel->prefix_idx, T = sel->T;
    if (kOp == kNccGather) T = sel->T, E = sel->E;
    float best[kNccRows];
    uint32_t bj[kNccRows];
#pragma unroll
    for (int r = 0; r < kNccRows; ++r) best[r] = FLT_MAX, bj[r] = 0;
    __syncthreads();

    for (uint32_t jj = 0; jj < nj; ++jj) {
        float s[12];
        const float4 a = s_src[jj][0], b = s_src[jj][1], c = s_src[jj][2];
        s[0] = a.x, s[1] = a.y, s[2] = a.z, s[3] = a.w, s[4] = b.x, s[5] = b.y, s[6] = b.z, s[7] = b.w;
        s[8] = c.x, s[9] = c.y, s[10] = c.z, s[11] = c.w;
        const uint32_t j = j0 + jj;
        uint32_t cm = 0xffffffffu;
#pragma unroll
        for (int r = 0; r < kNccRows; ++r) {
            const float d = ncc_l1(td[r], s);
            if (!tv[r]) continue;
            if (kOp == kNccRow || kOp == kNccRowCol) {
                if (d < best[r]) best[r] = d, bj[r] = j;
                if (kOp == kNccRowCol) cm = min(cm, ncc_key(d));
            } else {
                const uint32_t key = ncc_key(d), idx = ti[r] * P.n_s + j;
                if (kOp == kNccHistKey) {
                    if (((unsigned long long)(key ^ pre) >> (shift + 8)) == 0ull) atomicAdd(&s_aux[(key >> shift) & 0xffu], 1u);
                } else if (kOp == kNccHistIdx) {
                    if (key == T && ((unsigned long long)(idx ^ pre) >> (shift + 8)) == 0ull) atomicAdd(&s_aux[(idx >> shift) & 0xffu], 1u);
                } else if (key < T || (key == T && idx <= E)) {
                    const unsigned long long pos = atomicAdd(&sel->count, 1ull);
                    if (pos < K) gathered[pos] = ((unsigned long long)key << 32) | idx;
                }
            }
        }
        if (kOp == kNccRowCol) { // the column's minimum over this warp's rows; the block's in shared memory
            cm = __reduce_min_sync(0xffffffffu, cm);
            if ((threadIdx.x & 31) == 0 && cm != 0xffffffffu) atomicMin(&s_aux[jj], cm);
        }
    }

    if (kOp == kNccRow || kOp == kNccRowCol) {
#pragma unroll
        for (int r = 0; r < kNccRows; ++r)
            if (tv[r] && best[r] < FLT_MAX) atomicMin(&row_key[ti[r]], ((unsigned long long)__float_as_uint(best[r]) << 32) | bj[r]);
    }
    if (kOp == kNccRowCol || kOp == kNccHistKey || kOp == kNccHistIdx) {
        __syncthreads();
        for (uint32_t t = threadIdx.x; t < (uint32_t)kNccTileS; t += kNccBlock) {
            const uint32_t v = s_aux[t];
            if (kOp == kNccRowCol && t < nj && v != 0xffffffffu) atomicMin(&col_min[j0 + t], v);
            if (kOp != kNccRowCol && v) atomicAdd(&sel->hist[t], v);
        }
    }
}

// plain / reciprocal: every row starts at (FLT_MAX, source 0), every column minimum empty
__global__ void __launch_bounds__(kRawBlock) k_ncc_init(unsigned long long *row_key, uint32_t n_t, uint32_t *col_min, uint32_t n_s) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_t) row_key[i] = (unsigned long long)__float_as_uint(FLT_MAX) << 32;
    if (i < n_s) col_min[i] = 0xffffffffu;
}

// one thread: the digit at `shift` whose bin holds the remaining rank; the histogram is cleared for the next pass
__global__ void k_ncc_select_step(NccSelect *sel, int shift, int mode) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t cum = 0, b = 0, h = 0;
    for (; b < (uint32_t)kNccBins; ++b) {
        h = sel->hist[b];
        if (sel->rank < cum + h) break;
        cum += h;
    }
    sel->rank -= cum;
    if (mode == 0) {
        sel->prefix_key |= b << shift;
        if (shift == 0) sel->T = sel->prefix_key, sel->need_eq = sel->rank + 1, sel->count_eq = h;
    } else {
        sel->prefix_idx |= b << shift;
        if (shift == 0) sel->E = sel->prefix_idx;
    }
    for (int k = 0; k < kNccBins; ++k) sel->hist[k] = 0;
}

// plain / reciprocal: candidate (i << 32 | j) of every target row and whether it is kept (readings 5 and 6)
__global__ void __launch_bounds__(kRawBlock) k_ncc_pick(const unsigned long long *row_key, const uint32_t *col_min, uint32_t n_t,
                                                        int reciprocal, unsigned long long *cand, uint8_t *keep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_t) return;
    const unsigned long long rk = row_key[i];
    const uint32_t j = (uint32_t)rk;
    const float best = __uint_as_float((uint32_t)(rk >> 32));
    const uint32_t cmk = reciprocal ? col_min[j] : 0xffffffffu;
    cand[i] = ((unsigned long long)i << 32) | j;
    keep[i] = (cmk != 0xffffffffu && best > __uint_as_float(cmk)) ? 0 : 1;
}

} // namespace mulls
