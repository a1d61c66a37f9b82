// NDT registration on the device (CRegistration::omp_ndt, cregistration.hpp:945-1021): the readings and the shared
// arithmetic are in ndt_core.cuh. The Newton walk (SVD solve, trig, the float step transform) runs on the host, one
// evaluation per iteration on the device:
//  - k_ndt_keys: the leaf index of every target point (N1), sorted with its point index by a stable radix sort, so the
//    points of a leaf are consecutive and in input order;
//  - k_ndt_leaves: one thread per leaf (a run of equal keys): the sums in input order and ndt_leaf_finish; the run keys
//    are the sorted leaf table that DIRECT7 probes by binary search;
//  - k_ndt_eval: one thread per source point in tiles of kNdtTile: transform, 7 probes, ndt_update per neighbour, then
//    the tile's sums of the 43 terms in the order of C1 (shuffles inside a warp, then the warps);
//  - k_ndt_tiles: one thread per term, the tiles' sums in tile order;
//  - k_ndt_fitness: getFitnessScore's exact unbounded 1-NN squared distance of the moved source (knn_search over the
//    full-pyramid grid of the target the ingest built), -1 for a point that is not counted.
#pragma once
#include "device_types.cuh"
#include "kernels_iterate.cuh" // grid_of
#include "ndt_core.cuh"

namespace mulls {

constexpr int kNdtKeyBlock = 256;

__global__ void __launch_bounds__(kNdtKeyBlock) k_ndt_keys(const float4 *__restrict__ tgt, int n, NdtGrid g,
                                                           uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int i = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (i >= n) return;
    const float4 p = tgt[i];
    keys[i] = (uint64_t)ndt_build_key(g, p.x, p.y, p.z);
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(kNdtKeyBlock) k_ndt_leaves(const float4 *__restrict__ tgt, const uint32_t *__restrict__ order,
                                                             const int *__restrict__ offs, const int *__restrict__ counts,
                                                             const int *__restrict__ n_runs, NdtLeaf *__restrict__ leaves) {
    const int r = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (r >= *n_runs) return;
    double s[3] = {0.0, 0.0, 0.0}, c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const int o = offs[r], n = counts[r];
    for (int k = 0; k < n; ++k) {
        const float4 p = tgt[order[o + k]];
        const double v[3] = {(double)p.x, (double)p.y, (double)p.z};
        for (int a = 0; a < 3; ++a) {
            s[a] += v[a];
            for (int b = 0; b < 3; ++b) c[3 * a + b] += v[a] * v[b];
        }
    }
    leaves[r] = ndt_leaf_finish(s, c, n);
}

struct NdtEvalArgs {
    const float4 *src; // x y z, the input source after the intersection filter
    int n_src;
    NdtGrid g;
    const uint64_t *leaf_keys; // ascending
    const NdtLeaf *leaves;
    const int *n_leaves;
    double *tile_sums; // [tiles][kNdtTerms]
};

__device__ __forceinline__ int ndt_find_leaf(const uint64_t *keys, int n, uint64_t key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == key) ? lo : -1;
}

__global__ void __launch_bounds__(kNdtTile) k_ndt_eval(NdtEvalArgs A, NdtEvalConst E) {
    const int i = blockIdx.x * kNdtTile + threadIdx.x;
    double acc[kNdtTerms];
#pragma unroll
    for (int c = 0; c < kNdtTerms; ++c) acc[c] = 0.0;
    if (i < A.n_src && A.g.ok) {
        const float4 p = A.src[i];
        if (ndt_finite3(p.x, p.y, p.z)) {
            const float x[3] = {p.x, p.y, p.z};
            float t[3];
            ndt_transform(E.T, p.x, p.y, p.z, t);
            const int nl = *A.n_leaves;
            if (ndt_finite3(t[0], t[1], t[2]))
                for (int k = 0; k < 7; ++k) {
                    int64_t key;
                    if (!ndt_probe_key(A.g, t[0], t[1], t[2], k, key)) continue;
                    const int l = ndt_find_leaf(A.leaf_keys, nl, (uint64_t)key);
                    if (l < 0 || !A.leaves[l].ok) continue;
                    const NdtLeaf &L = A.leaves[l];
                    const double xt[3] = {(double)t[0] - L.mean[0], (double)t[1] - L.mean[1], (double)t[2] - L.mean[2]};
                    ndt_update(E, x, xt, L.icov, acc);
                }
        }
    }
    // C1: the pairwise tree inside the warp, then over the warps
    __shared__ double s_w[kNdtTile / 32][kNdtTerms];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < kNdtTerms; ++c) {
        double v = acc[c];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_down_sync(0xffffffffu, v, s);
        if (lane == 0) s_w[w][c] = v;
    }
    __syncthreads();
    if (threadIdx.x < kNdtTerms) {
        double q[kNdtTile / 32];
#pragma unroll
        for (int g = 0; g < kNdtTile / 32; ++g) q[g] = s_w[g][threadIdx.x];
#pragma unroll
        for (int s = kNdtTile / 64; s > 0; s >>= 1)
#pragma unroll
            for (int t = 0; t < s; ++t) q[t] += q[t + s];
        A.tile_sums[(size_t)blockIdx.x * kNdtTerms + threadIdx.x] = q[0];
    }
}

__global__ void __launch_bounds__(64) k_ndt_tiles(const double *__restrict__ tile_sums, int tiles, double *__restrict__ out) {
    const int c = threadIdx.x;
    if (c >= kNdtTerms) return;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += tile_sums[(size_t)t * kNdtTerms + c];
    out[c] = s;
}

// d2[i]: the squared distance of moved source point i to its nearest target, -1 when the point is not counted
__global__ void __launch_bounds__(128) k_ndt_fitness(DeviceArrays A, const float4 *__restrict__ src, int n, NdtEvalConst E,
                                                     float *__restrict__ d2) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    const float4 p = src[i];
    float t[3];
    ndt_transform(E.T, p.x, p.y, p.z, t);
    float r = -1.f;
    if (ndt_finite3(p.x, p.y, p.z) && ndt_finite3(t[0], t[1], t[2]) && A.ps[0].n_tgt[0] > 0 && !A.hash_used[1]) {
        const GridView g = grid_of(A, A.pc[0], A.ps[0], 0);
        KnnList<1> kl;
        knn_search(g, t[0], t[1], t[2], 1, 1, kl);
        if (kl.n > 0) r = kl.d2[0];
    }
    d2[i] = r;
}

} // namespace mulls
