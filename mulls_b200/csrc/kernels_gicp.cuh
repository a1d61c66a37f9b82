// Voxelized GICP registration on the device (CRegistration::omp_gicp, cregistration.hpp:1024-1098): the readings and the
// shared arithmetic are in gicp_core.cuh. The Gauss-Newton walk (LLT solve, SO3 exp / log, the rand() draws) runs on
// the host, one evaluation per iteration on the device:
//  - k_gicp_cov: one thread per point of a cloud the ingest built a full-pyramid grid of, in the grid's order: its 20
//    nearest neighbours (knn_search, FLANN's order) and their covariance, stored at the point's input index;
//  - k_gicp_plane: one thread per point, the PLANE regularisation of its covariance (G1) in place;
//  - k_gicp_keys: the voxel key of every target point (G2), sorted with its point index by the stable radix sort omp_ndt
//    uses (sort_runs in mulls_b200.cu), so the points of a voxel are consecutive and in input order;
//  - k_gicp_voxels: one thread per voxel (a run of equal keys): the ADDITIVE sums in input order and the division;
//  - k_gicp_eval: one thread per source point in tiles of kNdtTile: transform, DIRECT1 lookup by binary search in the
//    sorted voxel keys, the loss terms, then the tile's sums of the 28 terms in C1's order (tile_tree_store);
//  - k_gicp_tiles: one thread per term, the tiles' sums in tile order.
// The fitness is omp_ndt's k_ndt_fitness over the target's grid.
#pragma once
#include "device_types.cuh"
#include "gicp_core.cuh"
#include "kernels_ndt.cuh"
#include "kernels_sor.cuh" // kSorStartLevel

namespace mulls {

constexpr int kGicpCovBlock = 128;

// point i of the ingested cloud (in the grid's order): its kGicpK nearest neighbours (knn_search, FLANN's order), handed
// to fin(input index, nb) with nb(t, p) the t-th neighbour's x y z. Shared by the covariances of both GICP variants.
template <class Fin>
__device__ __forceinline__ void gicp_cov_neighbours(const DeviceArrays &A, int i, Fin fin) {
    const PairConst &pc = A.pc[0];
    const PairState &ps = A.ps[0];
    if (i >= ps.n_tgt[0] || A.hash_used[1]) return;
    const GridView g = grid_of(A, pc, ps, 0);
    const float4 p = g.pos[i];
    KnnList<kGicpK> kl;
    knn_search(g, p.x, p.y, p.z, kSorStartLevel, kGicpK, kl);
    fin(knn_orig(g, i), [&](int t, float q[3]) {
        const float4 v = g.pos[kl.j[t]];
        q[0] = v.x, q[1] = v.y, q[2] = v.z;
    });
}

// the raw covariance (6 floats) into cov[9 * input index]; k_gicp_plane regularises it in place
__global__ void __launch_bounds__(kGicpCovBlock) k_gicp_cov(DeviceArrays A, float *__restrict__ cov) {
    gicp_cov_neighbours(A, blockIdx.x * kGicpCovBlock + threadIdx.x, [&](int orig, auto nb) {
        float c[6];
        gicp_raw_covariance(nb, c);
        float *o = cov + 9 * (size_t)orig;
#pragma unroll
        for (int a = 0; a < 6; ++a) o[a] = c[a];
    });
}

__global__ void __launch_bounds__(kGicpCovBlock) k_gicp_plane(float *__restrict__ cov, int n) {
    const int i = blockIdx.x * kGicpCovBlock + threadIdx.x;
    if (i >= n) return;
    float *o = cov + 9 * (size_t)i, c[6], r[9];
#pragma unroll
    for (int a = 0; a < 6; ++a) c[a] = o[a];
    gicp_plane(c, r);
#pragma unroll
    for (int a = 0; a < 9; ++a) o[a] = r[a];
}

__global__ void __launch_bounds__(kNdtKeyBlock) k_gicp_keys(const float4 *__restrict__ tgt, int n, float res,
                                                            uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int i = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (i >= n) return;
    const float4 p = tgt[i];
    uint64_t k = 0;
    gicp_key_of(p.x, p.y, p.z, res, k); // in range: the host checked the target's bounds (C2)
    keys[i] = k;
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(kNdtKeyBlock) k_gicp_voxels(const float4 *__restrict__ tgt, const float *__restrict__ cov,
                                                              const uint32_t *__restrict__ order, const int *__restrict__ offs,
                                                              const int *__restrict__ counts, const int *__restrict__ n_runs,
                                                              GicpVoxel *__restrict__ vox) {
    const int r = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (r >= *n_runs) return;
    float sm[3] = {0.f, 0.f, 0.f}, sc[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const int o = offs[r], n = counts[r];
    for (int k = 0; k < n; ++k) {
        const uint32_t j = order[o + k];
        const float4 p = tgt[j];
        const float v[3] = {p.x, p.y, p.z};
        gicp_voxel_add(sm, sc, v, cov + 9 * (size_t)j);
    }
    vox[r] = gicp_voxel_finish(sm, sc, n);
}

struct GicpEvalArgs {
    const float4 *src;     // x y z, the source after the prologue (finite)
    const float *src_cov;  // [n_src][9]
    int n_src;
    float res;             // voxel resolution (float)
    const uint64_t *keys;  // voxel keys, ascending
    const GicpVoxel *vox;
    const int *n_vox;
    double *tile_sums;     // [tiles][kGicpTerms]
};

__global__ void __launch_bounds__(kNdtTile) k_gicp_eval(GicpEvalArgs A, NdtEvalConst E) {
    const int i = blockIdx.x * kNdtTile + threadIdx.x;
    double acc[kGicpTerms];
#pragma unroll
    for (int c = 0; c < kGicpTerms; ++c) acc[c] = 0.0;
    if (i < A.n_src) {
        const float4 p = A.src[i];
        float t[3];
        ndt_transform(E.T, p.x, p.y, p.z, t);
        uint64_t key;
        if (gicp_key_of(t[0], t[1], t[2], A.res, key)) {
            const int l = ndt_find_leaf(A.keys, *A.n_vox, key);
            if (l >= 0) {
                const float a[3] = {p.x, p.y, p.z};
                float e[3], J[3][6];
                gicp_point_loss(E.T, a, A.src_cov + 9 * (size_t)i, A.vox[l], e, J);
                gicp_point_terms(e, J, acc);
            }
        }
    }
    tile_tree_store<kGicpTerms>(acc, A.tile_sums);
}

__global__ void __launch_bounds__(32) k_gicp_tiles(const double *__restrict__ tile_sums, int tiles, double *__restrict__ out) {
    const int c = threadIdx.x;
    if (c >= kGicpTerms) return;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += tile_sums[(size_t)t * kGicpTerms + c];
    out[c] = s;
}

} // namespace mulls
