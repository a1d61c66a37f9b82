// PCA neighbourhood features: lo::PrincipleComponentAnalysis<PointT>::get_pc_pca_feature
// (include/common/pca.hpp:294-354) with get_pca_feature (:390-434) — for every stride-th point the at most
// k nearest neighbours within `radius` (pcl::KdTreeFLANN::radiusSearch: sorted by distance, truncated to
// max_nn, the query point itself included), their covariance / (n-1), eigen-pairs in descending order
// (pcl::PCA), principal direction = first eigenvector, normal = col0 x col1.
//
// One WARP per query on the same Morton-sorted cloud + hashed grid the registration path builds: lanes
// probe the 27 cells of the level whose cell size covers the radius in parallel, stream the candidates
// into a shared-memory list, radix-select the k-th smallest distance when more than k are in range, and
// reduce mean and covariance with shuffles. k_pca<true> gives every query its distance-adaptive radius (one warp per
// query keeps it warp-uniform); k_pca<false> is the fixed radius. fp64 accumulation; the 3x3 symmetric eigen problem is solved
// by cyclic Jacobi in fp64 (the reference's float SelfAdjointEigenSolver agrees to float rounding, which
// is the tolerance the parity tests state).
#pragma once
#include <type_traits>

#include "device_math.cuh"
#include "device_types.cuh"
#include "kernels_ingest.cuh"

namespace mulls {

constexpr int kPcaWarps = 4;
constexpr int kPcaCap = 1024; // candidates kept in shared memory per query

struct PcaArgs {
    float radius;
    float r2;       // (float)((double)radius * radius): the value FLANN's radius search compares against
    int k;          // max_nn (<= 0: unlimited)
    int stride;     // pca_down_rate
    float *eigenvalues, *principal, *normal; // [n][3], indexed by ORIGINAL point index
    int *pt_num;                             // [n]
    // optional (classification, needs 1 <= k <= kPcaListCap): the neighbour list of every query as radiusSearch returns
    // it — ORIGINAL indices sorted by (distance, index), bit 31 = close_to_query_point (pca.hpp:337) — and, with it,
    // pcl::PCA's float mean / covariance accumulated in exactly that order (bit-reproducible against the CPU path)
    uint32_t *nbr; // [n][k]
};
constexpr int kPcaListCap = 64;

// Distance-adaptive neighbourhoods (get_pc_pca_feature with distance_adaptive_on, pca.hpp:310-326): a query farther than
// unit_dist from the origin searches the radius sqrt(dist / unit_dist) * radius. `radius` / `r2` stay the base radius,
// which the close / far split of the neighbour lists keeps reading (pca.hpp:337).
struct PcaAdaptiveArgs : PcaArgs {
    float unit_dist; // > 0
};
template <bool kAdaptive> using PcaKernelArgs = std::conditional_t<kAdaptive, PcaAdaptiveArgs, PcaArgs>;

// dist = std::sqrt(float x*x + y*y + z*z) (the float overload, widened); strict `dist > unit_dist`; the radius is the
// double product narrowed to float
__device__ __forceinline__ float pca_adaptive_radius(float x, float y, float z, float radius, float unit_dist) {
    const double dist = (double)__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    return dist > (double)unit_dist ? (float)(__dsqrt_rn(__ddiv_rn(dist, (double)unit_dist)) * (double)radius) : radius;
}

__device__ inline void jacobi_eig3(double A[3][3], double w[3], double V[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (A[p][q] == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                const double t = ((theta >= 0) ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < 3; ++i) w[i] = A[i][i];
}

// eigen-pairs of the 3x3 covariance in descending order -> eigenvalues, principal direction, normal = col0 x col1
__device__ inline void pca_finish(double Am[3][3], const PcaArgs &P, int orig) {
    double w[3], V[3][3];
    jacobi_eig3(Am, w, V);
    int o0 = 0, o1 = 1, o2 = 2; // descending eigenvalues
    if (w[o0] < w[o1]) { int t = o0; o0 = o1; o1 = t; }
    if (w[o0] < w[o2]) { int t = o0; o0 = o2; o2 = t; }
    if (w[o1] < w[o2]) { int t = o1; o1 = o2; o2 = t; }
    const double e0[3] = {V[0][o0], V[1][o0], V[2][o0]}, e1[3] = {V[0][o1], V[1][o1], V[2][o1]};
    const double e2[3] = {e0[1] * e1[2] - e0[2] * e1[1], e0[2] * e1[0] - e0[0] * e1[2], e0[0] * e1[1] - e0[1] * e1[0]};
    const double n0 = sqrt(e0[0] * e0[0] + e0[1] * e0[1] + e0[2] * e0[2]);
    const double n2 = sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    const double ww[3] = {w[o0], w[o1], w[o2]};
    for (int d = 0; d < 3; ++d) {
        P.eigenvalues[3 * orig + d] = (float)ww[d];
        P.principal[3 * orig + d] = (float)(e0[d] / n0);
        P.normal[3 * orig + d] = (float)(e2[d] / n2);
    }
}

// warp-wide: number of list entries with key < v (keys are the uint bit patterns of non-negative floats)
__device__ __forceinline__ int count_less(const uint32_t *keys, int m, uint32_t v, int lane) {
    int c = 0;
    for (int i = lane; i < m; i += 32) c += (keys[i] < v) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    return c;
}

template <bool kAdaptive>
__global__ void __launch_bounds__(kPcaWarps * 32) k_pca(DeviceArrays A, PcaKernelArgs<kAdaptive> P) {
    __shared__ uint32_t s_key[kPcaWarps][kPcaCap]; // d2 bits
    __shared__ int s_idx[kPcaWarps][kPcaCap];      // sorted-position of the neighbour
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const PairConst &pc = A.pc[0];
    const PairState &ps = A.ps[0];
    const int n = ps.n_tgt[0];
    const int qi = blockIdx.x * kPcaWarps + warp; // query = sorted position
    if (qi >= n || A.hash_used[1]) return;
    const float4 *pos = A.tgt_pos + pc.tgt_base[0];
    const float4 *nrm = A.tgt_nrm + pc.tgt_base[0];
    const int orig = __float_as_int(nrm[qi].w);
    if (orig % P.stride != 0) return; // pca.hpp:304: for (i = 0; i < n; i += pca_down_rate)
    const float4 p = pos[qi];
    uint32_t *keys = s_key[warp];
    int *idxs = s_idx[warp];
    // this query's search radius (warp-uniform: one warp serves one query)
    float radius = P.radius, r2 = P.r2;
    if constexpr (kAdaptive) {
        radius = pca_adaptive_radius(p.x, p.y, p.z, P.radius, P.unit_dist);
        r2 = (float)((double)radius * (double)radius);
    }

    // level whose cells are at least as wide as the radius: its 3x3x3 block around p covers the sphere (the adaptive
    // ingest builds the full pyramid, whose top block spans the grid whatever the radius)
    int lq = 0;
    while (lq < ps.n_levels - 1 && 0.999f * ps.h0 * (float)(1 << lq) < radius) ++lq;
    // Progressive radius: a 3x3x3 block of level-l cells contains every point within 0.999*h_l of p. Where the cloud is
    // dense the k nearest neighbours lie well inside the radius, so start two levels finer and accept the first level
    // whose guaranteed sphere already holds k points — same neighbours, a fraction of the candidates.
    float rb2 = r2; // squared acceptance bound of the candidate stream
    uint32_t my_start = 0, my_count = 0;
    int m = 0;       // entries in the list (capped)
    int m_total = 0; // neighbours within the bound
    for (int l = (P.k > 0) ? max(0, lq - 2) : lq;; ++l) {
        const bool last = l >= lq;
        if (!last) {
            const float cover = 0.999f * ps.h0 * (float)(1 << l);
            rb2 = fminf(cover * cover, r2);
        } else {
            rb2 = r2;
        }
        const int ncell = (1 << kCoordBits) >> l;
        const int cx = ((int)floorf((p.x - ps.origin[0]) * ps.inv_h0)) >> l;
        const int cy = ((int)floorf((p.y - ps.origin[1]) * ps.inv_h0)) >> l;
        const int cz = ((int)floorf((p.z - ps.origin[2]) * ps.inv_h0)) >> l;
        my_start = 0, my_count = 0;
        if (lane < 27) {
            const int x = cx + lane % 3 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane / 9 - 1;
            if (x >= 0 && y >= 0 && z >= 0 && x < ncell && y < ncell && z < ncell) {
                const HashEntry *table = A.hash + ps.hash_base[0];
                const uint32_t klo = cell_key_lo((uint32_t)x, (uint32_t)y, (uint32_t)z), khi = cell_key_hi((uint32_t)z, l);
                uint32_t slot = cell_hash(klo, khi) & ps.hash_mask[0];
                while (true) {
                    const uint4 e = __ldg(reinterpret_cast<const uint4 *>(&table[slot]));
                    if (e.x == klo && (e.y & kKeyHiMask) == khi) {
                        my_start = e.z;
                        my_count = e.w;
                        break;
                    }
                    if (e.x == 0u && e.y == 0u) break;
                    slot = (slot + 1) & ps.hash_mask[0];
                }
            }
        }
        // stream the candidates within the bound into the list (FLANN's radius result set keeps dist < r2)
        m_total = 0;
        for (int c = 0; c < 27; ++c) {
            const uint32_t start = __shfl_sync(0xffffffffu, my_start, c), count = __shfl_sync(0xffffffffu, my_count, c);
            for (uint32_t base = 0; base < count; base += 32) {
                const uint32_t j = start + base + lane;
                bool in = false;
                float d2 = 0.f;
                if (base + lane < count) {
                    const float4 q = __ldg(&pos[j]);
                    d2 = flann_l2(p.x, p.y, p.z, q.x, q.y, q.z);
                    in = d2 < rb2;
                }
                const unsigned b = __ballot_sync(0xffffffffu, in);
                const int off = m_total + __popc(b & ((1u << lane) - 1u));
                if (in && off < kPcaCap) {
                    keys[off] = __float_as_uint(d2);
                    idxs[off] = (int)j;
                }
                m_total += __popc(b);
            }
        }
        if (last || m_total >= P.k) break; // the k nearest are all inside this level's sphere
        __syncwarp();
    }
    __syncwarp();
    m = min(m_total, kPcaCap);
    int kk = (P.k > 0) ? P.k : m_total;
    if (kk > kPcaCap) kk = kPcaCap; // documented limit of this kernel (the reference uses k = 25..50)
    int n_sel = min(m_total, kk);
    // threshold T (as float bits) = the n_sel-th smallest distance; selected = {key < T} + ties in index order
    uint32_t T = 0xffffffffu;
    int n_less = m;
    if (m_total > kk) {
        if (m_total <= kPcaCap) {
            // bisection on the bit pattern over the shared-memory list: the largest v with count(key < v) < kk
            uint32_t v = 0;
            for (int bit = 30; bit >= 0; --bit) {
                const uint32_t trial = v | (1u << bit);
                if (count_less(keys, m, trial, lane) < kk) v = trial;
            }
            T = v; // exactly the kk-th smallest key
            n_less = count_less(keys, m, T, lane);
        } else {
            // more candidates than the list holds: bisect by re-scanning the cells (rare; dense raw scans)
            uint32_t v = 0;
            for (int bit = 30; bit >= 0; --bit) {
                const uint32_t trial = v | (1u << bit);
                int cl = 0;
                for (int c = 0; c < 27; ++c) {
                    const uint32_t start = __shfl_sync(0xffffffffu, my_start, c), count = __shfl_sync(0xffffffffu, my_count, c);
                    for (uint32_t t = lane; t < count; t += 32) {
                        const float4 q = __ldg(&pos[start + t]);
                        const float d2 = flann_l2(p.x, p.y, p.z, q.x, q.y, q.z);
                        cl += (d2 < rb2 && __float_as_uint(d2) < trial) ? 1 : 0;
                    }
                }
                for (int o = 16; o > 0; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
                if (cl < kk) v = trial;
            }
            T = v;
            // Everything below T and every tie at T fit the list: the tie rule below picks among all the ties. Else the
            // list keeps the ties to take only — those with the lowest ORIGINAL indices among ALL the ties in the cells,
            // not among the ones a capped list would happen to hold: lim = the need-th smallest index of a tie, by
            // bisection on the original index.
            int n_below = 0, n_at = 0;
            for (int c = 0; c < 27; ++c) {
                const uint32_t start = __shfl_sync(0xffffffffu, my_start, c), count = __shfl_sync(0xffffffffu, my_count, c);
                for (uint32_t t = lane; t < count; t += 32) {
                    const float4 q = __ldg(&pos[start + t]);
                    const float d2 = flann_l2(p.x, p.y, p.z, q.x, q.y, q.z);
                    n_below += (d2 < rb2 && __float_as_uint(d2) < T) ? 1 : 0;
                    n_at += (d2 < rb2 && __float_as_uint(d2) == T) ? 1 : 0;
                }
            }
            for (int o = 16; o > 0; o >>= 1) {
                n_below += __shfl_xor_sync(0xffffffffu, n_below, o);
                n_at += __shfl_xor_sync(0xffffffffu, n_at, o);
            }
            const int need = kk - n_below; // >= 1: count(key < T) < kk <= count(key <= T)
            uint32_t lim = 0xffffffffu;    // all ties
            if (n_below + n_at > kPcaCap) {
                lim = 0;
                for (int bit = 30; bit >= 0; --bit) {
                    const uint32_t trial = lim | (1u << bit);
                    int cl = 0;
                    for (int c = 0; c < 27; ++c) {
                        const uint32_t start = __shfl_sync(0xffffffffu, my_start, c), count = __shfl_sync(0xffffffffu, my_count, c);
                        for (uint32_t t = lane; t < count; t += 32) {
                            const float4 q = __ldg(&pos[start + t]);
                            const float d2 = flann_l2(p.x, p.y, p.z, q.x, q.y, q.z);
                            cl += (d2 < rb2 && __float_as_uint(d2) == T &&
                                   (uint32_t)__float_as_int(__ldg(&nrm[start + t]).w) < trial) ? 1 : 0;
                        }
                    }
                    for (int o = 16; o > 0; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
                    if (cl < need) lim = trial;
                }
            }
            // rebuild the list: the n_below entries below T and the ties up to lim (all of them, or the `need` to take)
            int mt = 0;
            for (int c = 0; c < 27; ++c) {
                const uint32_t start = __shfl_sync(0xffffffffu, my_start, c), count = __shfl_sync(0xffffffffu, my_count, c);
                for (uint32_t base = 0; base < count; base += 32) {
                    const uint32_t j = start + base + lane;
                    bool in = false;
                    float d2 = 0.f;
                    if (base + lane < count) {
                        const float4 q = __ldg(&pos[j]);
                        d2 = flann_l2(p.x, p.y, p.z, q.x, q.y, q.z);
                        in = d2 < rb2 && (__float_as_uint(d2) < T || (__float_as_uint(d2) == T &&
                                                                      (uint32_t)__float_as_int(__ldg(&nrm[j]).w) <= lim));
                    }
                    const unsigned b = __ballot_sync(0xffffffffu, in);
                    const int off = mt + __popc(b & ((1u << lane) - 1u));
                    if (in && off < kPcaCap) {
                        keys[off] = __float_as_uint(d2);
                        idxs[off] = (int)j;
                    }
                    mt += __popc(b);
                }
            }
            __syncwarp();
            m = min(mt, kPcaCap);
            n_less = count_less(keys, m, T, lane);
        }
    }
    // ties at T: take them in ascending ORIGINAL index until n_sel is reached (the sorted-by-(d2,index)
    // order the radius search truncates)
    int need_ties = (m_total > kk) ? (n_sel - n_less) : 0x7fffffff;
    int tie_limit = 0x7fffffff; // ties with original index <= tie_limit are selected
    if (m_total > kk) {
        int n_ties = 0;
        for (int i = lane; i < m; i += 32) n_ties += (keys[i] == T) ? 1 : 0;
        for (int o = 16; o > 0; o >>= 1) n_ties += __shfl_xor_sync(0xffffffffu, n_ties, o);
        if (n_ties > need_ties) {
            int last = -1;
            for (int r = 0; r < need_ties; ++r) { // need_ties-th smallest original index among the ties
                int best = 0x7fffffff;
                for (int i = lane; i < m; i += 32)
                    if (keys[i] == T) {
                        const int oi = __float_as_int(__ldg(&nrm[idxs[i]]).w);
                        if (oi > last && oi < best) best = oi;
                    }
                for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
                last = best;
            }
            tie_limit = last;
        }
    }
    auto selected = [&](int i) -> bool {
        const uint32_t key = keys[i];
        if (m_total <= kk) return true;
        if (key < T) return true;
        if (key > T) return false;
        if (tie_limit == 0x7fffffff) return true;
        return __float_as_int(__ldg(&nrm[idxs[i]]).w) <= tie_limit;
    };
    if (lane == 0) P.pt_num[orig] = n_sel;
    __shared__ uint32_t s_lkey[kPcaWarps][kPcaListCap];
    __shared__ int s_lorig[kPcaWarps][kPcaListCap];
    __shared__ float s_lxyz[kPcaWarps][kPcaListCap][3];
    __shared__ uint8_t s_lrank[kPcaWarps][kPcaListCap];
    const bool lists = P.nbr != nullptr && n_sel <= kPcaListCap;
    if (lists) {
        // compact the selected entries, rank them by (distance, original index), store them in that order
        int cnt = 0;
        for (int base = 0; base < m; base += 32) {
            const int i = base + lane;
            const bool sel = i < m && selected(i);
            const unsigned b = __ballot_sync(0xffffffffu, sel);
            const int off = cnt + __popc(b & ((1u << lane) - 1u));
            if (sel && off < kPcaListCap) {
                const float4 q = __ldg(&pos[idxs[i]]);
                s_lkey[warp][off] = keys[i];
                s_lorig[warp][off] = __float_as_int(__ldg(&nrm[idxs[i]]).w);
                s_lxyz[warp][off][0] = q.x, s_lxyz[warp][off][1] = q.y, s_lxyz[warp][off][2] = q.z;
            }
            cnt += __popc(b);
        }
        __syncwarp();
        for (int i = lane; i < n_sel; i += 32) {
            const uint32_t ki = s_lkey[warp][i];
            const int oi = s_lorig[warp][i];
            int rank = 0;
            for (int t = 0; t < n_sel; ++t) {
                const uint32_t kt = s_lkey[warp][t];
                rank += (kt < ki || (kt == ki && s_lorig[warp][t] < oi)) ? 1 : 0;
            }
            s_lrank[warp][rank] = (uint8_t)i;
            const bool close = (double)__uint_as_float(ki) < 0.64 * (double)P.radius * (double)P.radius;
            P.nbr[(size_t)orig * P.k + rank] = (uint32_t)oi | (close ? 0x80000000u : 0u);
        }
        __syncwarp();
    }
    if (n_sel <= 3) { // pca.hpp:396-397: no feature for tiny neighbourhoods
        if (lane < 3) P.eigenvalues[3 * orig + lane] = P.principal[3 * orig + lane] = P.normal[3 * orig + lane] = 0.f;
        return;
    }
    if (lists) {
        if (lane == 0) { // pcl::PCA: float centroid, float covariance / (n-1), neighbours in radiusSearch order
            float mu[3] = {0.f, 0.f, 0.f};
            for (int t = 0; t < n_sel; ++t) {
                const float *q = s_lxyz[warp][s_lrank[warp][t]];
                mu[0] += q[0], mu[1] += q[1], mu[2] += q[2];
            }
            mu[0] /= (float)n_sel, mu[1] /= (float)n_sel, mu[2] /= (float)n_sel;
            float c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
            for (int t = 0; t < n_sel; ++t) {
                const float *q = s_lxyz[warp][s_lrank[warp][t]];
                const float dx = q[0] - mu[0], dy = q[1] - mu[1], dz = q[2] - mu[2];
                c00 += dx * dx, c01 += dx * dy, c02 += dx * dz, c11 += dy * dy, c12 += dy * dz, c22 += dz * dz;
            }
            const float dn = (float)(n_sel - 1);
            double Am[3][3] = {{(double)(c00 / dn), (double)(c01 / dn), (double)(c02 / dn)},
                               {(double)(c01 / dn), (double)(c11 / dn), (double)(c12 / dn)},
                               {(double)(c02 / dn), (double)(c12 / dn), (double)(c22 / dn)}};
            pca_finish(Am, P, orig);
        }
        return;
    }
    // mean, then covariance / (n-1)
    double sx = 0, sy = 0, sz = 0;
    for (int i = lane; i < m; i += 32)
        if (selected(i)) {
            const float4 q = __ldg(&pos[idxs[i]]);
            sx += q.x, sy += q.y, sz += q.z;
        }
    for (int o = 16; o > 0; o >>= 1) {
        sx += __shfl_xor_sync(0xffffffffu, sx, o);
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        sz += __shfl_xor_sync(0xffffffffu, sz, o);
    }
    const double mx = sx / n_sel, my = sy / n_sel, mz = sz / n_sel;
    double c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
    for (int i = lane; i < m; i += 32)
        if (selected(i)) {
            const float4 q = __ldg(&pos[idxs[i]]);
            const double dx = q.x - mx, dy = q.y - my, dz = q.z - mz;
            c00 += dx * dx, c01 += dx * dy, c02 += dx * dz, c11 += dy * dy, c12 += dy * dz, c22 += dz * dz;
        }
    for (int o = 16; o > 0; o >>= 1) {
        c00 += __shfl_xor_sync(0xffffffffu, c00, o);
        c01 += __shfl_xor_sync(0xffffffffu, c01, o);
        c02 += __shfl_xor_sync(0xffffffffu, c02, o);
        c11 += __shfl_xor_sync(0xffffffffu, c11, o);
        c12 += __shfl_xor_sync(0xffffffffu, c12, o);
        c22 += __shfl_xor_sync(0xffffffffu, c22, o);
    }
    if (lane == 0) {
        const double inv = 1.0 / (double)(n_sel - 1);
        double Am[3][3] = {{c00 * inv, c01 * inv, c02 * inv}, {c01 * inv, c11 * inv, c12 * inv}, {c02 * inv, c12 * inv, c22 * inv}};
        pca_finish(Am, P, orig);
    }
}

} // namespace mulls
