// Statistical outlier removal: lo::CFilter<PointT>::sor_filter (include/common/cfilter.hpp:203-247), i.e.
// pcl::StatisticalOutlierRemoval<PointT>::applyFilterIndices (PCL 1.10, restated in SURVEY Appendix B item 10), over
// the grid the ingest built for a one-pair batch whose only target class is the cloud (full level pyramid, non-finite
// points left out: mulls_sor_filter). Three kernels:
//   k_sor_dist   one thread per finite point, in the grid's Morton order (neighbouring threads share cells): exact
//                mean_k + 1 nearest neighbours (knn_search, search_core.cuh), drop one zero (the query itself), sum the
//                square roots of the others in ascending order in double, store (float)(sum / mean_k) at the point's
//                input index (.w of its normal)
//   k_sor_stats  PCL's two sums in input order, sequentially: one warp, lanes load coalesced, every lane adds the same
//                values in index order (lane 0 writes). A parallel reduction would round differently and move the
//                threshold in its last bits, flipping points that sit on it. Then mean, stddev and threshold.
//   k_sor_mark   keep bit i (bit i % 8 of byte i / 8) iff NOT (distances[i] > threshold), and the kept count
// The mean distance depends only on the sorted multiset of the mean_k + 1 smallest squared distances: whichever of
// several tied neighbours the search lists, the values summed and their order are the same.
#pragma once
#include "device_math.cuh"
#include "device_types.cuh"
#include "kernels_ingest.cuh"
#include "kernels_iterate.cuh" // grid_of

namespace mulls {

// mean_k <= kSorMaxMeanK: the largest list instance holds mean_k + 1 = 64 neighbours (the reference uses 20)
constexpr int kSorMaxMeanK = 63;
constexpr int kSorBlock = 128;
// the level k_sor_dist's search starts from: the smallest block, since most points of a map have their neighbours
// within a cell or two; a sparse neighbourhood climbs the pyramid from there
constexpr int kSorStartLevel = 1;

// PCL sums sqrt(nn_dists[k]) into a double. Which sqrt overload that binds to cannot be settled without PCL's source;
// this reads it as the double one. The one place of that choice on the device.
MULLS_HD double sor_sqrt(float d2) { return sqrt((double)d2); }

template <int kCap>
__global__ void __launch_bounds__(kSorBlock) k_sor_dist(DeviceArrays A, int mean_k, float *dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const PairConst &pc = A.pc[0];
    const PairState &ps = A.ps[0];
    if (i >= (uint32_t)ps.n_tgt[0] || A.hash_used[1]) return;
    const GridView g = grid_of(A, pc, ps, 0);
    const float4 p = g.pos[i];
    KnnList<kCap> kl;
    knn_search(g, p.x, p.y, p.z, kSorStartLevel, mean_k + 1, kl);
    double sum = 0.0;
    for (int t = 1; t <= mean_k; ++t) sum += sor_sqrt(kl.d2[t]); // position 0: the query itself (or a duplicate), d2 = 0
    dist[__float_as_int(g.nrm[i].w)] = (float)(sum / mean_k);
}

// one warp. out->n_valid / n_kept: the finite points / 0 (k_sor_mark counts).
__global__ void __launch_bounds__(32) k_sor_stats(DeviceArrays A, const float *dist, uint32_t n, double n_std,
                                                  mulls_sor_stats *out) {
    const unsigned lane = threadIdx.x;
    constexpr uint32_t kTile = 4 * 32;
    double sum = 0.0, sq_sum = 0.0;
    float v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = (r * 32 + lane < n) ? dist[r * 32 + lane] : 0.0f;
    for (uint32_t base = 0; base < n; base += kTile) {
        float nx[4]; // the next tile is loaded while this one is summed
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const uint32_t idx = base + kTile + r * 32 + lane;
            nx[r] = idx < n ? dist[idx] : 0.0f;
        }
        // padding past n adds +0.0 to both sums: exact
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll 8
            for (int t = 0; t < 32; ++t) {
                const float x = __shfl_sync(0xffffffffu, v[r], t);
                sum += (double)x;
                sq_sum += (double)(x * x); // PCL: the float product, widened
            }
#pragma unroll
        for (int r = 0; r < 4; ++r) v[r] = nx[r];
    }
    if (lane == 0) {
        const double valid = (double)A.ps[0].n_tgt[0];
        const double mean = sum / valid;
        const double variance = (sq_sum - sum * sum / valid) / (valid - 1);
        const double stddev = sqrt(variance);
        out->mean = mean;
        out->stddev = stddev;
        out->threshold = mean + n_std * stddev;
        out->n_valid = (uint64_t)A.ps[0].n_tgt[0];
        out->n_kept = 0;
    }
}

// keep[w] bit b = point 32 w + b (little-endian words: bit i % 8 of byte i / 8)
__global__ void __launch_bounds__(256) k_sor_mark(const float *dist, uint32_t n, mulls_sor_stats *st, uint32_t *keep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool kept = i < n && !((double)dist[i] > st->threshold);
    const unsigned b = __ballot_sync(0xffffffffu, kept);
    if ((threadIdx.x & 31) == 0 && i < n) {
        keep[i >> 5] = b;
        if (b) atomicAdd(reinterpret_cast<unsigned long long *>(&st->n_kept), (unsigned long long)__popc(b));
    }
}

} // namespace mulls
