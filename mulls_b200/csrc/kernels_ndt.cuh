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
//  - KDTREE (K1-K5): k_ndt_kd_centroids, k_ndt_kd_pack and per evaluation k_ndt_kd_search, k_ndt_eval_kd (below);
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

// the leaf of `key` among keys[lo, hi) (ascending), -1 when there is none
__device__ __forceinline__ int ndt_find_leaf(const uint64_t *keys, int lo, int hi, uint64_t key) {
    const int n = hi;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == key) ? lo : -1;
}
__device__ __forceinline__ int ndt_find_leaf(const uint64_t *keys, int n, uint64_t key) { return ndt_find_leaf(keys, 0, n, key); }
// the first of keys[0, n) (ascending) that is not below key
__device__ __forceinline__ int ndt_lower_bound(const uint64_t *keys, int n, uint64_t key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// N4 for source point p: transform, the 7 probes among the leaves keys[lo, hi) (each key carries `key_hi` above the
// leaf index: the pair in a batch, 0 for one pair), ndt_update per neighbour into acc
__device__ __forceinline__ void ndt_point_terms(float4 p, const NdtGrid &g, const uint64_t *keys, uint64_t key_hi, int lo, int hi,
                                                const NdtLeaf *leaves, const NdtEvalConst &E, double (&acc)[kNdtTerms]) {
    if (!ndt_finite3(p.x, p.y, p.z)) return;
    const float x[3] = {p.x, p.y, p.z};
    float t[3];
    ndt_transform(E.T, p.x, p.y, p.z, t);
    if (!ndt_finite3(t[0], t[1], t[2])) return;
    for (int k = 0; k < 7; ++k) {
        int64_t key;
        if (!ndt_probe_key(g, t[0], t[1], t[2], k, key)) continue;
        const int l = ndt_find_leaf(keys, lo, hi, key_hi | (uint64_t)key);
        if (l < 0 || !leaves[l].ok) continue;
        const NdtLeaf &L = leaves[l];
        const double xt[3] = {(double)t[0] - L.mean[0], (double)t[1] - L.mean[1], (double)t[2] - L.mean[2]};
        ndt_update(E, x, xt, L.icov, acc);
    }
}

// C1 of ndt_core.cuh over one block of kNdtTile threads, each holding its point's kTerms sums in acc: the pairwise tree
// inside each warp (shuffles), then over the warps; thread c < kTerms stores the tile's sum of term c at
// tile_sums[blockIdx.x * kTerms + c]. Shared by every evaluation that sums in that order (NDT, GICP).
template <int kTerms>
__device__ __forceinline__ void tile_tree_store(const double (&acc)[kTerms], double *tile_sums) {
    __shared__ double s_w[kNdtTile / 32][kTerms];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < kTerms; ++c) {
        double v = acc[c];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_down_sync(0xffffffffu, v, s);
        if (lane == 0) s_w[w][c] = v;
    }
    __syncthreads();
    if (threadIdx.x < kTerms) {
        double q[kNdtTile / 32];
#pragma unroll
        for (int g = 0; g < kNdtTile / 32; ++g) q[g] = s_w[g][threadIdx.x];
#pragma unroll
        for (int s = kNdtTile / 64; s > 0; s >>= 1)
#pragma unroll
            for (int t = 0; t < s; ++t) q[t] += q[t + s];
        tile_sums[(size_t)blockIdx.x * kTerms + threadIdx.x] = q[0];
    }
}

__global__ void __launch_bounds__(kNdtTile) k_ndt_eval(NdtEvalArgs A, NdtEvalConst E) {
    const int i = blockIdx.x * kNdtTile + threadIdx.x;
    double acc[kNdtTerms];
#pragma unroll
    for (int c = 0; c < kNdtTerms; ++c) acc[c] = 0.0;
    if (i < A.n_src && A.g.ok) ndt_point_terms(A.src[i], A.g, A.leaf_keys, 0, 0, *A.n_leaves, A.leaves, E, acc);
    tile_tree_store<kNdtTerms>(acc, A.tile_sums);
}

// ---- KDTREE (mulls_omp_ndt_kdtree, K1-K5 of ndt_core.cuh) --------------------------------------------------------------
//  - k_ndt_kd_centroids: one thread per leaf (run r, ascending leaf index): the float centroid of a searchable leaf and
//    the key of its own search cell; other runs and the slots past the last run get the key ~0, which sorts last;
//  - the (key, run) pairs sorted once per call, k_ndt_kd_pack: the centroids in key order, the run in .w;
//  - k_ndt_kd_search: one thread per source point per evaluation: the probe box, one contiguous key range per (y, z)
//    row of it, the exact float test, and the neighbour list in (d2, run) order written to list[k * n_src + i];
//  - k_ndt_eval_kd: k_ndt_eval's tiles, ndt_update over the point's list in that order.
constexpr uint64_t kNdtKdNoKey = ~0ull;

__global__ void __launch_bounds__(kNdtKeyBlock) k_ndt_kd_centroids(const float4 *__restrict__ tgt, const uint32_t *__restrict__ order,
                                                                   const int *__restrict__ offs, const int *__restrict__ counts,
                                                                   const int *__restrict__ n_runs, int n, NdtGrid g,
                                                                   float4 *__restrict__ cent, uint64_t *__restrict__ keys,
                                                                   uint32_t *__restrict__ vals) {
    const int r = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (r >= n) return;
    uint64_t key = kNdtKdNoKey;
    if (r < *n_runs && ndt_kd_searchable(counts[r])) {
        const int o = offs[r], m = counts[r];
        float s[3] = {0.f, 0.f, 0.f}, c[3];
        for (int k = 0; k < m; ++k) {
            const float4 p = tgt[order[o + k]];
            s[0] += p.x, s[1] += p.y, s[2] += p.z;
        }
        ndt_kd_centroid(s, m, c);
        cent[r] = make_float4(c[0], c[1], c[2], 0.f);
        key = (uint64_t)ndt_kd_key(g, ndt_kd_cell(g, c[0], 0), ndt_kd_cell(g, c[1], 1), ndt_kd_cell(g, c[2], 2));
    }
    keys[r] = key;
    vals[r] = (uint32_t)r;
}

__global__ void __launch_bounds__(kNdtKeyBlock) k_ndt_kd_pack(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ runs,
                                                              const float4 *__restrict__ cent, int n, float4 *__restrict__ pts) {
    const int j = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (j >= n || keys[j] == kNdtKdNoKey) return;
    const float4 c = cent[runs[j]];
    pts[j] = make_float4(c.x, c.y, c.z, __int_as_float((int)runs[j]));
}

struct NdtKdArgs {
    const float4 *src;
    int n_src;
    NdtGrid g;
    float r2, rp;            // K2's r2 and the probe radius r'
    const uint64_t *keys;    // the sorted centroid keys, kNdtKdNoKey past the searchable ones
    const float4 *pts;       // the centroids in key order, run index in .w
    int n_keys;
    int cap;                 // list entries per point
    int2 *list;              // [cap][n_src]: (d2 bits, run)
    int *count;              // [n_src]: the neighbour count, cap or not
    int *max_count;          // the largest count above cap (0 when every list fits)
};

__global__ void __launch_bounds__(kNdtTile) k_ndt_kd_search(NdtKdArgs A, NdtEvalConst E) {
    const int i = blockIdx.x * kNdtTile + threadIdx.x;
    if (i >= A.n_src) return;
    int cnt = 0;
    const float4 p = A.src[i];
    float t[3];
    ndt_transform(E.T, p.x, p.y, p.z, t);
    if (A.g.ok && ndt_finite3(p.x, p.y, p.z) && ndt_finite3(t[0], t[1], t[2])) {
        int lo[3], hi[3];
        ndt_kd_box(A.g, A.rp, t, lo, hi);
        for (int z = lo[2]; z <= hi[2]; ++z)
            for (int y = lo[1]; y <= hi[1]; ++y) {
                const uint64_t k0 = (uint64_t)ndt_kd_key(A.g, lo[0], y, z), k1 = (uint64_t)ndt_kd_key(A.g, hi[0], y, z);
                for (int j = ndt_lower_bound(A.keys, A.n_keys, k0); j < A.n_keys && A.keys[j] <= k1; ++j) {
                    const float4 c = A.pts[j];
                    const float d2 = ndt_kd_d2(t, c.x, c.y, c.z);
                    if (!(d2 < A.r2)) continue;
                    if (cnt < A.cap) { // insertion in (d2, run) order
                        const int run = __float_as_int(c.w);
                        int k = cnt;
                        for (; k > 0; --k) {
                            const int2 e = A.list[(size_t)(k - 1) * A.n_src + i];
                            if (!ndt_kd_before(d2, run, __int_as_float(e.x), e.y)) break;
                            A.list[(size_t)k * A.n_src + i] = e;
                        }
                        A.list[(size_t)k * A.n_src + i] = make_int2(__float_as_int(d2), run);
                    }
                    ++cnt;
                }
            }
    }
    A.count[i] = cnt;
    if (cnt > A.cap) atomicMax(A.max_count, cnt);
}

struct NdtKdEvalArgs {
    const float4 *src;
    int n_src, cap;
    const int2 *list;
    const int *count;
    const NdtLeaf *leaves;
    double *tile_sums; // [tiles][kNdtTerms]
};

__global__ void __launch_bounds__(kNdtTile) k_ndt_eval_kd(NdtKdEvalArgs A, NdtEvalConst E) {
    const int i = blockIdx.x * kNdtTile + threadIdx.x;
    double acc[kNdtTerms];
#pragma unroll
    for (int c = 0; c < kNdtTerms; ++c) acc[c] = 0.0;
    if (i < A.n_src) {
        const int m = min(A.count[i], A.cap);
        const float4 p = A.src[i];
        const float x[3] = {p.x, p.y, p.z};
        float t[3];
        ndt_transform(E.T, p.x, p.y, p.z, t);
        for (int k = 0; k < m; ++k) {
            const NdtLeaf &L = A.leaves[A.list[(size_t)k * A.n_src + i].y];
            const double xt[3] = {(double)t[0] - L.mean[0], (double)t[1] - L.mean[1], (double)t[2] - L.mean[2]};
            ndt_update(E, x, xt, L.icov, acc);
        }
    }
    tile_tree_store<kNdtTerms>(acc, A.tile_sums);
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

// ---- a batch of pairs (mulls_omp_ndt_batch) -------------------------------------------------------------------------
// The leaves of all targets come from one sort: a pair's leaf index (below 2^31, N1) goes in the low 32 bits of the key
// and the pair above it, so the stable sort keeps each leaf's points in input order and each pair's leaves are the one
// pair's leaves, consecutive. The evaluation runs over the tiles of every live pair at once; a tile never spans two
// pairs, so each pair's tile sums and their order are the one pair's (C1).
struct NdtPairDev {
    NdtGrid g;
    int src_off, n_src;       // the pair's sources in the batch's source array
    int tgt_off, n_tgt;       // its target points in the leaf build (n_tgt = 0 when the grid is not ok)
    int leaf_begin, leaf_end; // its leaves among the sorted runs (k_ndt_leaf_ranges)
};

// a live pair of one evaluation launch: its constants and its tiles [tile_begin, tile_end) of the launch
struct NdtLiveSlot {
    NdtEvalConst E;
    int pair, tile_begin, tile_end;
};

// the last of pairs[0, n) whose offset (member `off`) is <= i: the pair of element i (empty pairs share the offset of
// the next one and are skipped)
template <int NdtPairDev::*off>
__device__ __forceinline__ int ndt_pair_of(const NdtPairDev *pairs, int n, int i) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pairs[mid].*off <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kNdtKeyBlock) k_ndt_keys_batch(const float4 *__restrict__ tgt, int n, const NdtPairDev *__restrict__ pairs,
                                                                 int n_pairs, uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int i = blockIdx.x * kNdtKeyBlock + threadIdx.x;
    if (i >= n) return;
    const int p = ndt_pair_of<&NdtPairDev::tgt_off>(pairs, n_pairs, i);
    const float4 q = tgt[i];
    // a finite point inside its pair's min / max: the leaf index is in [0, 2^31) (N1)
    keys[i] = ((uint64_t)p << 32) | (uint64_t)ndt_build_key(pairs[p].g, q.x, q.y, q.z);
    vals[i] = (uint32_t)i;
}

// one thread per pair: its leaves among the n_runs sorted run keys
__global__ void __launch_bounds__(64) k_ndt_leaf_ranges(const uint64_t *__restrict__ run_keys, const int *__restrict__ n_runs,
                                                        NdtPairDev *__restrict__ pairs, int n_pairs) {
    const int p = blockIdx.x * 64 + threadIdx.x;
    if (p >= n_pairs) return;
    const int n = *n_runs;
    int b[2];
    for (int e = 0; e < 2; ++e) {
        const uint64_t key = (uint64_t)(p + e) << 32;
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (run_keys[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        b[e] = lo;
    }
    pairs[p].leaf_begin = b[0], pairs[p].leaf_end = b[1];
}

struct NdtBatchEvalArgs {
    const float4 *src;
    const NdtPairDev *pairs;
    const uint64_t *leaf_keys;
    const NdtLeaf *leaves;
    const NdtLiveSlot *slots;
    int n_slots;
    double *tile_sums; // [launch tiles][kNdtTerms]
};

__global__ void __launch_bounds__(kNdtTile) k_ndt_eval_batch(NdtBatchEvalArgs A) {
    __shared__ NdtEvalConst s_E;
    __shared__ int s_slot;
    if (threadIdx.x == 0) {
        int lo = 0, hi = A.n_slots - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (A.slots[mid].tile_begin <= (int)blockIdx.x) lo = mid;
            else hi = mid - 1;
        }
        s_slot = lo;
    }
    __syncthreads();
    const NdtLiveSlot *S = A.slots + s_slot;
    static_assert(sizeof(NdtEvalConst) % 4 == 0, "copied as words");
    for (int w = threadIdx.x; w < (int)(sizeof(NdtEvalConst) / 4); w += kNdtTile)
        reinterpret_cast<int *>(&s_E)[w] = reinterpret_cast<const int *>(&S->E)[w];
    __syncthreads();
    const int pair = S->pair;
    const NdtPairDev &P = A.pairs[pair];
    const int i = ((int)blockIdx.x - S->tile_begin) * kNdtTile + threadIdx.x;
    double acc[kNdtTerms];
#pragma unroll
    for (int c = 0; c < kNdtTerms; ++c) acc[c] = 0.0;
    if (i < P.n_src && P.g.ok)
        ndt_point_terms(A.src[P.src_off + i], P.g, A.leaf_keys, (uint64_t)pair << 32, P.leaf_begin, P.leaf_end, A.leaves, s_E, acc);
    tile_tree_store<kNdtTerms>(acc, A.tile_sums);
}

// block s, thread c: live slot s's tiles summed in tile order (k_ndt_tiles per pair) into out[s][c]
__global__ void __launch_bounds__(64) k_ndt_tiles_batch(const double *__restrict__ tile_sums, const NdtLiveSlot *__restrict__ slots,
                                                        double *__restrict__ out) {
    const int c = threadIdx.x;
    if (c >= kNdtTerms) return;
    const int b = slots[blockIdx.x].tile_begin, e = slots[blockIdx.x].tile_end;
    double s = 0.0;
    for (int t = b; t < e; ++t) s += tile_sums[(size_t)t * kNdtTerms + c];
    out[(size_t)blockIdx.x * kNdtTerms + c] = s;
}

// k_ndt_fitness over the sources of all pairs, each moved by its pair's final transform T[pair] and searched in its
// pair's grid (pair p of the ingest's batch)
__global__ void __launch_bounds__(128) k_ndt_fitness_batch(DeviceArrays A, const float4 *__restrict__ src, int n,
                                                           const NdtPairDev *__restrict__ pairs, int n_pairs,
                                                           const float *__restrict__ T, float *__restrict__ d2) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    const int p = ndt_pair_of<&NdtPairDev::src_off>(pairs, n_pairs, i);
    const float4 q = src[i];
    float t[3];
    ndt_transform(T + 12 * p, q.x, q.y, q.z, t);
    float r = -1.f;
    if (ndt_finite3(q.x, q.y, q.z) && ndt_finite3(t[0], t[1], t[2]) && A.ps[p].n_tgt[0] > 0 && !A.hash_used[1]) {
        const GridView g = grid_of(A, A.pc[p], A.ps[p], 0);
        KnnList<1> kl;
        knn_search(g, t[0], t[1], t[2], 1, 1, kl);
        if (kl.n > 0) r = kl.d2[0];
    }
    d2[i] = r;
}

} // namespace mulls
