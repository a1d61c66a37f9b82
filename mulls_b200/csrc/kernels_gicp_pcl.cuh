// Point-wise GICP registration on the device (CRegistration::omp_gicp with using_voxel_gicp = false,
// koide_reg::GeneralizedIterativeClosestPoint): the readings and the shared arithmetic are in gicp_pcl_core.cuh. The
// outer loop and PCL's BFGS run on the host; the device does every pass over the points:
//  - k_gicp_pcl_cov: one thread per point of an ingested cloud: its 20 nearest neighbours (gicp_cov_neighbours, the
//    search k_gicp_cov runs) and their double sums (P3), stored at the point's input index;
//  - k_gicp_pcl_plane: one thread per point, the covariance of the sums, its SVD and the reconstruction with
//    (1, 1, 1e-3) in place (P3);
//  - k_gicp_pcl_match: once per outer iteration, one thread per source point: the move by transformation_, the exact
//    nearest target (the search of k_ndt_fitness), the 25.0 test and M (P4); a flag per point, which
//    cub::DeviceSelect::Flagged compacts in source order;
//  - k_gicp_pcl_eval<method>: once per functor call, one thread per correspondence in tiles of kNdtTile: the method's
//    1 (operator()), 12 (df) or 13 (fdf) terms, then the tile's sums in C1's order (tile_tree_store);
//  - k_gicp_pcl_tiles: one thread per term, the tiles' sums in tile order.
// The fitness is omp_ndt's k_ndt_fitness over the target's grid.
#pragma once
#include "gicp_pcl_core.cuh"
#include "kernels_gicp.cuh"

namespace mulls {

// the neighbour list's 9 sums into cov[9 * input index]; k_gicp_pcl_plane turns them into the covariance in place
__global__ void __launch_bounds__(kGicpCovBlock) k_gicp_pcl_cov(DeviceArrays A, double *__restrict__ cov) {
    gicp_cov_neighbours(A, blockIdx.x * kGicpCovBlock + threadIdx.x, [&](int orig, auto nb) {
        double s[9];
        gicp_pcl_neighbour_sums(nb, s);
        double *o = cov + 9 * (size_t)orig;
#pragma unroll
        for (int a = 0; a < 9; ++a) o[a] = s[a];
    });
}

__global__ void __launch_bounds__(kGicpCovBlock) k_gicp_pcl_plane(double *__restrict__ cov, int n) {
    const int i = blockIdx.x * kGicpCovBlock + threadIdx.x;
    if (i >= n) return;
    double *o = cov + 9 * (size_t)i, c[9], r[9];
#pragma unroll
    for (int a = 0; a < 9; ++a) c[a] = o[a];
    gicp_pcl_plane(c, r);
#pragma unroll
    for (int a = 0; a < 9; ++a) o[a] = r[a];
}

// transformation_ (float, rows 0..2) and transform_R's 3x3 block (double, row-major)
struct GicpPclMatchConst {
    float T[12];
    double R[9];
};

// flag[i] = 1 when source point i has a correspondence; then tix[i] is its target's input index and
// maha[9 i ..] its M (3x3 row-major float)
__global__ void __launch_bounds__(128) k_gicp_pcl_match(DeviceArrays A, const float4 *__restrict__ src, int n,
                                                        const double *__restrict__ src_cov, const double *__restrict__ tgt_cov,
                                                        GicpPclMatchConst C, int *__restrict__ flag, int *__restrict__ tix,
                                                        float *__restrict__ maha) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    const float4 p = src[i];
    float t[3];
    ndt_transform(C.T, p.x, p.y, p.z, t);
    int keep = 0;
    if (ndt_finite3(t[0], t[1], t[2]) && A.ps[0].n_tgt[0] > 0 && !A.hash_used[1]) { // C3
        const GridView g = grid_of(A, A.pc[0], A.ps[0], 0);
        KnnList<1> kl;
        knn_search(g, t[0], t[1], t[2], 1, 1, kl);
        if (kl.n > 0 && (double)kl.d2[0] < kGicpPclCorrDist * kGicpPclCorrDist) {
            const int j = knn_orig(g, kl.j[0]);
            float M[9];
            gicp_pcl_maha(C.R, src_cov + 9 * (size_t)i, tgt_cov + 9 * (size_t)j, M);
            tix[i] = j;
#pragma unroll
            for (int k = 0; k < 9; ++k) maha[9 * (size_t)i + k] = M[k];
            keep = 1;
        }
    }
    flag[i] = keep;
}

struct GicpPclEvalArgs {
    const float4 *src;  // the source after the prologue (finite)
    const float4 *tgt;  // the target after the prologue, input order
    const int *list;    // the correspondences' source indices, ascending
    const int *tix;     // [n_src] the target of each source point with a correspondence
    const float *maha;  // [n_src][9]
    int m;              // correspondences
    double *tile_sums;  // [tiles][terms]
};

template <int kMethod>
__global__ void __launch_bounds__(kNdtTile) k_gicp_pcl_eval(GicpPclEvalArgs A, NdtEvalConst E) {
    constexpr int kTerms = gicp_pcl_terms(kMethod);
    const int c = blockIdx.x * kNdtTile + threadIdx.x;
    double acc[kTerms];
#pragma unroll
    for (int k = 0; k < kTerms; ++k) acc[k] = 0.0;
    if (c < A.m) {
        const int s = A.list[c];
        const float4 p = A.src[s], q = A.tgt[A.tix[s]];
        const float a[3] = {p.x, p.y, p.z}, b[3] = {q.x, q.y, q.z};
        float M[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) M[k] = A.maha[9 * (size_t)s + k];
        gicp_pcl_terms<kMethod>(E.T, a, b, M, acc);
    }
    tile_tree_store<kTerms>(acc, A.tile_sums);
}

__global__ void __launch_bounds__(32) k_gicp_pcl_tiles(const double *__restrict__ tile_sums, int tiles, int terms,
                                                       double *__restrict__ out) {
    const int c = threadIdx.x;
    if (c >= terms) return;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += tile_sums[(size_t)t * terms + c];
    out[c] = s;
}

} // namespace mulls
