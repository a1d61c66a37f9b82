// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::omp_ndt with KDTREE
// (use_direct_search = false, include/common/cregistration.hpp:945-1021; K1-K5 of mulls_b200/csrc/ndt_core.cuh), the
// checker of mulls_omp_ndt_kdtree. Everything but the neighbourhood (prologue, leaf grid and finalisation, derivatives,
// the summation order C1, the Newton walk) comes from ndt_core.cuh, as in tests/harness/ndt_oracle.cpp (DIRECT7): the
// leaves by a stable sort of the leaf keys, the fitness by brute force over the target. The KDTREE candidates are chosen
// independently of the device's search cells: every searchable leaf whose leaf cell is within 2 cells of the query's
// cell on each axis, the margin widened by the largest distance, in cells, between a centroid's own cell and its
// leaf's; then the float test and the (d2, index) sort of K2. The tiles are evaluated in parallel (OpenMP) and their
// sums added in tile order, so the thread count does not change a bit.
// Built by tests/test_ndt_kdtree.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "../../include/mulls_b200/abi.h"
#include "../../mulls_b200/csrc/ndt_core.cuh"

using namespace mulls;

namespace {

struct Leaves {
    std::vector<int64_t> keys; // ascending
    std::vector<NdtLeaf> leaf;
    std::vector<int> count;         // points per leaf
    std::vector<float> cent;        // K1: the float centroid of every leaf (3 per leaf)
    std::vector<int> rank;          // K1: the index in the searchable cloud, -1 when not searchable
    int dev = 0;                    // the largest |own cell of a centroid - its leaf's cell| over the axes
};

Leaves build_leaves(const std::vector<float4> &tgt, const NdtGrid &g) {
    Leaves L;
    if (!g.ok) return L;
    const size_t n = tgt.size();
    std::vector<int64_t> key(n);
    for (size_t i = 0; i < n; ++i) key[i] = ndt_build_key(g, tgt[i].x, tgt[i].y, tgt[i].z);
    std::vector<size_t> ord(n);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return (uint64_t)key[a] < (uint64_t)key[b]; });
    for (size_t a = 0; a < n;) {
        size_t b = a;
        double s[3] = {0, 0, 0}, c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        float fs[3] = {0.f, 0.f, 0.f};
        while (b < n && key[ord[b]] == key[ord[a]]) {
            const float4 p = tgt[ord[b]];
            fs[0] += p.x, fs[1] += p.y, fs[2] += p.z;
            const double v[3] = {(double)p.x, (double)p.y, (double)p.z};
            for (int i = 0; i < 3; ++i) {
                s[i] += v[i];
                for (int j = 0; j < 3; ++j) c[3 * i + j] += v[i] * v[j];
            }
            ++b;
        }
        const int m = (int)(b - a);
        L.keys.push_back(key[ord[a]]);
        L.leaf.push_back(ndt_leaf_finish(s, c, m));
        L.count.push_back(m);
        float ce[3];
        ndt_kd_centroid(fs, m, ce);
        L.cent.insert(L.cent.end(), ce, ce + 3);
        a = b;
    }
    int nk = 0;
    for (size_t l = 0; l < L.keys.size(); ++l) {
        const bool sr = ndt_kd_searchable(L.count[l]);
        L.rank.push_back(sr ? nk++ : -1);
        if (!sr) continue;
        const int64_t i[3] = {L.keys[l] % g.divb_mul[1], (L.keys[l] / g.divb_mul[1]) % (g.divb_mul[2] / g.divb_mul[1]),
                              L.keys[l] / g.divb_mul[2]};
        for (int d = 0; d < 3; ++d) {
            const int64_t own = (int64_t)ndt_f2i(floorf(L.cent[3 * l + d] * g.inv)) - g.min_b[d];
            L.dev = std::max(L.dev, (int)std::min<int64_t>(std::llabs(own - i[d]), 1 << 20));
        }
    }
    return L;
}

// K2: the neighbours of the moved point t, as (d2, leaf) in (d2, index) order
void kd_neighbours(const NdtGrid &g, const Leaves &L, float resolution, const float t[3], std::vector<std::pair<float, int>> &nb) {
    nb.clear();
    if (!g.ok) return;
    const float r2 = ndt_kd_r2(resolution);
    const int64_t M = 2 + L.dev, div[3] = {g.divb_mul[1], g.divb_mul[2] / g.divb_mul[1], 0};
    const int64_t dims[3] = {div[0], div[1], (int64_t)g.max_b[2] - g.min_b[2] + 1};
    int64_t q[3];
    for (int d = 0; d < 3; ++d) q[d] = (int64_t)ndt_f2i(floorf(t[d] * g.inv)) - g.min_b[d];
    const int64_t x0 = std::max<int64_t>(q[0] - M, 0), x1 = std::min<int64_t>(q[0] + M, dims[0] - 1);
    for (int64_t k = std::max<int64_t>(q[2] - M, 0); k <= std::min<int64_t>(q[2] + M, dims[2] - 1); ++k)
        for (int64_t j = std::max<int64_t>(q[1] - M, 0); j <= std::min<int64_t>(q[1] + M, dims[1] - 1); ++j) {
            if (x0 > x1) continue;
            const int64_t k0 = x0 + j * g.divb_mul[1] + k * g.divb_mul[2], k1 = x1 + j * g.divb_mul[1] + k * g.divb_mul[2];
            for (auto it = std::lower_bound(L.keys.begin(), L.keys.end(), k0); it != L.keys.end() && *it <= k1; ++it) {
                const int l = (int)(it - L.keys.begin());
                if (L.rank[l] < 0) continue;
                const float d2 = ndt_kd_d2(t, L.cent[3 * l], L.cent[3 * l + 1], L.cent[3 * l + 2]);
                if (d2 < r2) nb.push_back({d2, l});
            }
        }
    std::sort(nb.begin(), nb.end(), [&](const std::pair<float, int> &a, const std::pair<float, int> &b) {
        return ndt_kd_before(a.first, L.rank[a.second], b.first, L.rank[b.second]);
    });
}

// score, gradient and Hessian with the KDTREE neighbourhood; the tiles in parallel, their sums in tile order (C1)
void evaluate_kd(const std::vector<float4> &src, const NdtGrid &g, const Leaves &L, float resolution, const NdtEvalConst &E,
                 double r[kNdtTerms]) {
    const long n = (long)src.size(), tiles = (n + kNdtTile - 1) / kNdtTile;
    std::vector<double> ts((size_t)tiles * kNdtTerms);
#pragma omp parallel for schedule(dynamic, 4)
    for (long tl = 0; tl < tiles; ++tl) {
        std::vector<double> acc((size_t)kNdtTile * kNdtTerms, 0.0), q(kNdtTile);
        std::vector<std::pair<float, int>> nb;
        for (int t = 0; t < kNdtTile && tl * kNdtTile + t < n; ++t) {
            const float4 p = src[tl * kNdtTile + t];
            if (!ndt_finite3(p.x, p.y, p.z)) continue;
            const float x[3] = {p.x, p.y, p.z};
            float tr[3];
            ndt_transform(E.T, p.x, p.y, p.z, tr);
            if (!ndt_finite3(tr[0], tr[1], tr[2])) continue;
            kd_neighbours(g, L, resolution, tr, nb);
            for (const auto &e : nb) {
                const NdtLeaf &lf = L.leaf[e.second];
                const double xt[3] = {(double)tr[0] - lf.mean[0], (double)tr[1] - lf.mean[1], (double)tr[2] - lf.mean[2]};
                ndt_update(E, x, xt, lf.icov, &acc[(size_t)t * kNdtTerms]);
            }
        }
        for (int c = 0; c < kNdtTerms; ++c) {
            for (int t = 0; t < kNdtTile; ++t) q[t] = acc[(size_t)t * kNdtTerms + c];
            ts[(size_t)tl * kNdtTerms + c] = ndt_tile_sum(q.data());
        }
    }
    for (int c = 0; c < kNdtTerms; ++c) {
        r[c] = 0.0;
        for (long tl = 0; tl < tiles; ++tl) r[c] += ts[(size_t)tl * kNdtTerms + c];
    }
}

void consts_at(const double p[6], const float T[12], float resolution, NdtEvalConst &E) {
    std::memcpy(E.T, T, sizeof(E.T));
    ndt_angle_tables(p, E);
    double d1, d2;
    ndt_gauss(resolution, d1, d2);
    E.gauss_d1 = d1, E.gauss_d2 = (float)d2;
}

std::vector<float4> rows_of(const float *r48, long n) {
    std::vector<float4> v(n);
    for (long i = 0; i < n; ++i) v[i] = make_float4(r48[12 * i], r48[12 * i + 1], r48[12 * i + 2], 0.f);
    return v;
}

} // namespace

extern "C" {

// omp_ndt with KDTREE (mulls_omp_ndt_kdtree's arguments)
int orc_ndt_kdtree(const float *t48, long nt, const float *s48, long ns, float resolution, const double *guess,
                   int apply_filter, float thre, const double *tb, const double *sb, mulls_ndt_result *out, mulls_ndt_iter *trace,
                   int cap) {
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(t48, (size_t)nt, s48, (size_t)ns, guess, apply_filter, tb, sb, tgt, src, moved);
    const NdtGrid g = ndt_grid_from(tgt, resolution);
    const Leaves L = build_leaves(tgt, g);
    NdtEvalConst E;
    auto eval = [&](const double p[6], const float T[12], double r[kNdtTerms]) {
        consts_at(p, T, resolution, E);
        evaluate_kd(src, g, L, resolution, E, r);
    };
    std::vector<NdtIter> tr(cap > 0 ? cap : 0);
    float T[12];
    int converged = 0;
    const int iters = ndt_walk(eval, T, converged, tr.data(), (int)tr.size());
    double fitness = DBL_MAX, sum = 0.0;
    int cnt = 0;
    if (!tgt.empty()) {
        std::vector<float> d2(src.size(), -1.f);
#pragma omp parallel for schedule(dynamic, 64)
        for (long i = 0; i < (long)src.size(); ++i) {
            const float4 p = src[i];
            float m[3];
            ndt_transform(T, p.x, p.y, p.z, m);
            if (!ndt_finite3(p.x, p.y, p.z) || !ndt_finite3(m[0], m[1], m[2])) continue;
            float best = INFINITY;
            for (const float4 &q : tgt) {
                const float dx = m[0] - q.x, dy = m[1] - q.y, dz = m[2] - q.z;
                const float d = (dx * dx + dy * dy) + dz * dz;
                best = d < best ? d : best;
            }
            d2[i] = best;
        }
        for (float d : d2)
            if (d >= 0.f) sum += (double)d, ++cnt;
        if (cnt) fitness = sum / cnt;
    }
    ndt_epilogue(T, guess, moved, out->trans);
    out->code = fitness > (double)thre ? -3 : 1;
    out->iterations = iters;
    out->converged = converged;
    out->fitness = fitness;
    out->n_target = (int)tgt.size();
    out->n_source = (int)src.size();
    for (int i = 0; i < std::min(iters, cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].p[c] = tr[i].p[c];
        trace[i].step = tr[i].step, trace[i].score = tr[i].score, trace[i].reversed = tr[i].reversed;
    }
    return 0;
}

static void finite_target(const float *t48, long nt, float resolution, std::vector<float4> &tgt, NdtGrid &g) {
    std::vector<float4> all = rows_of(t48, nt);
    tgt.clear();
    for (const float4 &q : all)
        if (ndt_finite3(q.x, q.y, q.z)) tgt.push_back(q);
    g = ndt_grid_from(tgt, resolution);
}

// K1 of a target cloud (no filter), in ascending leaf index (orc_ndt_leaves' order in ndt_oracle.cpp): up to cap leaves' float centroids (3 each), point
// counts and searchable ranks (-1: not searchable); returns the leaf count
long orc_ndt_centroids(const float *t48, long nt, float resolution, long cap, float *cent, int *count, int *rank) {
    std::vector<float4> tgt;
    NdtGrid g;
    finite_target(t48, nt, resolution, tgt, g);
    const Leaves L = build_leaves(tgt, g);
    for (long i = 0; i < (long)L.keys.size() && i < cap; ++i) {
        for (int c = 0; c < 3; ++c) cent[3 * i + c] = L.cent[3 * i + c];
        count[i] = L.count[i], rank[i] = L.rank[i];
    }
    return (long)L.keys.size();
}

// K2 at the pose vector p (no filter): per source point the neighbour count and up to cap neighbours (the leaf in
// ascending leaf index, d2) in their order, row i of leaf[ns][cap] / d2[ns][cap]
void orc_ndt_kdtree_neighbours(const float *t48, long nt, const float *s48, long ns, float resolution, const double *p, int cap,
                               int *count, int *leaf, float *d2) {
    std::vector<float4> tgt, src = rows_of(s48, ns);
    NdtGrid g;
    finite_target(t48, nt, resolution, tgt, g);
    const Leaves L = build_leaves(tgt, g);
    float T[12];
    ndt_step_transform(p, T);
    std::vector<std::pair<float, int>> nb;
    for (long i = 0; i < ns; ++i) {
        count[i] = 0;
        const float4 q = src[i];
        float t[3];
        ndt_transform(T, q.x, q.y, q.z, t);
        if (!ndt_finite3(q.x, q.y, q.z) || !ndt_finite3(t[0], t[1], t[2])) continue;
        kd_neighbours(g, L, resolution, t, nb);
        count[i] = (int)nb.size();
        for (int k = 0; k < (int)nb.size() && k < cap; ++k) leaf[(size_t)i * cap + k] = nb[k].second, d2[(size_t)i * cap + k] = nb[k].first;
    }
}

// score, gradient and Hessian with KDTREE at the pose vector p (no filter)
void orc_ndt_kdtree_eval(const float *t48, long nt, const float *s48, long ns, float resolution, const double *p, double *out) {
    std::vector<float4> tgt, src = rows_of(s48, ns);
    NdtGrid g;
    finite_target(t48, nt, resolution, tgt, g);
    const Leaves L = build_leaves(tgt, g);
    float T[12];
    ndt_step_transform(p, T);
    NdtEvalConst E;
    consts_at(p, T, resolution, E);
    evaluate_kd(src, g, L, resolution, E, out);
}

} // extern "C"
