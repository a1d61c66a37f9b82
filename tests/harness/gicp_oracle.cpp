// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::omp_gicp with using_voxel_gicp
// (include/common/cregistration.hpp:1024-1098, koide_reg::FastVGICP), the checker of mulls_omp_gicp. The readings and
// every piece both sides must compute alike (prologue, covariance of a neighbour list, voxel key and finalisation, loss
// terms, the summation order C1, the walk with its rand() draws, the epilogue) come from mulls_b200/csrc/gicp_core.cuh
// and run here on the host, sequentially: the exact k nearest neighbours in FLANN's order (squared distance, index) on
// a hash grid, the voxels by a stable sort of the keys, the DIRECT1 lookup by binary search, the fitness by the same
// exact nearest search. Built by tests/test_gicp.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <unordered_map>
#include <vector>

#include "../../include/mulls_b200/abi.h"
#include "../../mulls_b200/csrc/gicp_core.cuh"

using namespace mulls;

namespace {

// exact k nearest neighbours, ascending under (squared distance as FLANN computes it, index)
struct HashGrid {
    const std::vector<float4> *pts = nullptr;
    float h = 1.f;
    int64_t lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    std::unordered_map<uint64_t, std::vector<int>> cells;
    static uint64_t pack(int64_t x, int64_t y, int64_t z) {
        return ((uint64_t)(x + (1 << 20)) << 42) | ((uint64_t)(y + (1 << 20)) << 21) | (uint64_t)(z + (1 << 20));
    }
    int64_t cell(float v, int a) const {
        const double c = std::floor((double)v / h);
        return (int64_t)std::max(std::min(c, 1e15), -1e15);
    }
    void build(const std::vector<float4> &p) {
        pts = &p;
        float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
        for (const float4 &q : p) {
            const float v[3] = {q.x, q.y, q.z};
            for (int a = 0; a < 3; ++a) mn[a] = std::min(mn[a], v[a]), mx[a] = std::max(mx[a], v[a]);
        }
        double vol = 1.0, ext_max = 0.0;
        for (int a = 0; a < 3; ++a) ext_max = std::max(ext_max, (double)mx[a] - mn[a]);
        for (int a = 0; a < 3; ++a) vol *= std::max((double)mx[a] - mn[a], 1e-3 * std::max(ext_max, 1e-3));
        h = (float)std::max(std::cbrt(vol * 16.0 / std::max<size_t>(p.size(), 1)), 1e-4 * std::max(ext_max, 1e-3));
        for (int a = 0; a < 3; ++a) lo[a] = (int64_t)std::floor((double)mn[a] / h), hi[a] = (int64_t)std::floor((double)mx[a] / h);
        for (size_t i = 0; i < p.size(); ++i) cells[pack(cell(p[i].x, 0), cell(p[i].y, 1), cell(p[i].z, 2))].push_back((int)i);
    }
    void knn(float px, float py, float pz, int k, std::vector<std::pair<float, int>> &best) const {
        best.clear();
        const int64_t c[3] = {cell(px, 0), cell(py, 1), cell(pz, 2)};
        auto less = [](const std::pair<float, int> &a, const std::pair<float, int> &b) {
            return a.first < b.first || (a.first == b.first && a.second < b.second);
        };
        auto visit = [&](int64_t x, int64_t y, int64_t z) {
            auto it = cells.find(pack(x, y, z));
            if (it == cells.end()) return;
            for (int j : it->second) {
                const float4 q = (*pts)[j];
                const float dx = px - q.x, dy = py - q.y, dz = pz - q.z;
                const std::pair<float, int> e((dx * dx + dy * dy) + dz * dz, j);
                if ((int)best.size() == k && !less(e, best.back())) continue;
                best.insert(std::upper_bound(best.begin(), best.end(), e, less), e);
                if ((int)best.size() > k) best.pop_back();
            }
        };
        int64_t r0 = 0; // the shells before r0 hold no cell
        for (int a = 0; a < 3; ++a) r0 = std::max(r0, std::max(lo[a] - c[a], c[a] - hi[a]));
        for (int64_t r = r0;; ++r) {
            int64_t a0[3], a1[3];
            bool any = true, all = true;
            for (int a = 0; a < 3; ++a) {
                a0[a] = std::max(c[a] - r, lo[a]), a1[a] = std::min(c[a] + r, hi[a]);
                any = any && a0[a] <= a1[a];
                all = all && c[a] - r <= lo[a] && c[a] + r >= hi[a];
            }
            if (any)
                for (int64_t x = a0[0]; x <= a1[0]; ++x)
                    for (int64_t y = a0[1]; y <= a1[1]; ++y) {
                        if (std::llabs(x - c[0]) == r || std::llabs(y - c[1]) == r) {
                            for (int64_t z = a0[2]; z <= a1[2]; ++z) visit(x, y, z);
                        } else {
                            if (c[2] - r >= lo[2] && c[2] - r <= hi[2]) visit(x, y, c[2] - r);
                            if (r > 0 && c[2] + r >= lo[2] && c[2] + r <= hi[2]) visit(x, y, c[2] + r);
                        }
                    }
            if (all) break;
            const double cover = (double)r * h;
            if ((int)best.size() == k && (double)best.back().first < cover * cover * 0.999) break;
        }
    }
};

// G1 for every point of a cloud (at least kGicpK points)
std::vector<float> covariances(const std::vector<float4> &p) {
    HashGrid G;
    G.build(p);
    std::vector<float> cov(p.size() * 9);
#pragma omp parallel for schedule(dynamic, 256)
    for (long i = 0; i < (long)p.size(); ++i) {
        std::vector<std::pair<float, int>> nb;
        G.knn(p[i].x, p[i].y, p[i].z, kGicpK, nb);
        float c[6];
        gicp_raw_covariance([&](int t, float q[3]) {
            const float4 v = p[nb[t].second];
            q[0] = v.x, q[1] = v.y, q[2] = v.z;
        }, c);
        gicp_plane(c, &cov[9 * i]);
    }
    return cov;
}

struct Voxels {
    std::vector<uint64_t> keys; // ascending
    std::vector<GicpVoxel> vox;
    std::vector<int> n;
};
Voxels build_voxels(const std::vector<float4> &tgt, const std::vector<float> &cov, float res) {
    Voxels V;
    const size_t n = tgt.size();
    std::vector<uint64_t> key(n);
    for (size_t i = 0; i < n; ++i) gicp_key_of(tgt[i].x, tgt[i].y, tgt[i].z, res, key[i]);
    std::vector<size_t> ord(n);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return key[a] < key[b]; });
    for (size_t a = 0; a < n;) {
        size_t b = a;
        float sm[3] = {0.f, 0.f, 0.f}, sc[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        while (b < n && key[ord[b]] == key[ord[a]]) {
            const float4 q = tgt[ord[b]];
            const float v[3] = {q.x, q.y, q.z};
            gicp_voxel_add(sm, sc, v, &cov[9 * ord[b]]);
            ++b;
        }
        V.keys.push_back(key[ord[a]]);
        V.vox.push_back(gicp_voxel_finish(sm, sc, (int)(b - a)));
        V.n.push_back((int)(b - a));
        a = b;
    }
    return V;
}

void evaluate(const std::vector<float4> &src, const std::vector<float> &scov, const Voxels &V, float res, const float T[12],
              double r[kGicpTerms]) {
    const size_t n = src.size();
    for (int c = 0; c < kGicpTerms; ++c) r[c] = 0.0;
    std::vector<double> acc((size_t)kNdtTile * kGicpTerms), q(kNdtTile);
    for (size_t t0 = 0; t0 < n; t0 += kNdtTile) {
        std::fill(acc.begin(), acc.end(), 0.0);
        for (int t = 0; t < kNdtTile && t0 + t < n; ++t) {
            const float4 p = src[t0 + t];
            float tr[3];
            ndt_transform(T, p.x, p.y, p.z, tr);
            uint64_t key;
            if (!gicp_key_of(tr[0], tr[1], tr[2], res, key)) continue;
            auto it = std::lower_bound(V.keys.begin(), V.keys.end(), key);
            if (it == V.keys.end() || *it != key) continue;
            const float a[3] = {p.x, p.y, p.z};
            float e[3], J[3][6];
            gicp_point_loss(T, a, &scov[9 * (t0 + t)], V.vox[it - V.keys.begin()], e, J);
            gicp_point_terms(e, J, &acc[(size_t)t * kGicpTerms]);
        }
        for (int c = 0; c < kGicpTerms; ++c) {
            for (int t = 0; t < kNdtTile; ++t) q[t] = acc[(size_t)t * kGicpTerms + c];
            r[c] += ndt_tile_sum(q.data());
        }
    }
}

std::vector<float4> xyz_of(const float *xyz, long n) {
    std::vector<float4> v(n);
    for (long i = 0; i < n; ++i) v[i] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 0.f);
    return v;
}

} // namespace

extern "C" {

int orc_gicp(const float *t48, long nt, const float *s48, long ns, float res, const double *guess, int apply_filter, float thre,
             const double *tb, const double *sb, mulls_gicp_result *out, mulls_gicp_iter *trace, int cap) {
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(t48, (size_t)nt, s48, (size_t)ns, guess, apply_filter, tb, sb, tgt, src, moved);
    gicp_keep_finite(src);
    if ((long)tgt.size() < kGicpK || (long)src.size() < kGicpK) return MULLS_E_UNSUPPORTED;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (const float4 &p : tgt) {
        const float v[3] = {p.x, p.y, p.z};
        for (int d = 0; d < 3; ++d) mn[d] = std::min(mn[d], v[d]), mx[d] = std::max(mx[d], v[d]);
    }
    uint64_t k;
    if (!gicp_key_of(mn[0], mn[1], mn[2], res, k) || !gicp_key_of(mx[0], mx[1], mx[2], res, k)) return MULLS_E_UNSUPPORTED;
    const std::vector<float> scov = covariances(src), tcov = covariances(tgt);
    const Voxels V = build_voxels(tgt, tcov, res);
    auto eval = [&](const float T[12], double r[kGicpTerms]) { evaluate(src, scov, V, res, T, r); };
    std::vector<GicpIter> tr(cap > 0 ? cap : 0);
    float T[12];
    int converged = 0;
    const int iters = gicp_walk(eval, T, out->x0, converged, tr.data(), (int)tr.size());
    // getFitnessScore over the same exact nearest search
    HashGrid G;
    G.build(tgt);
    std::vector<float> d2(src.size(), -1.f);
#pragma omp parallel for schedule(dynamic, 256)
    for (long i = 0; i < (long)src.size(); ++i) {
        float m[3];
        ndt_transform(T, src[i].x, src[i].y, src[i].z, m);
        if (!ndt_finite3(m[0], m[1], m[2])) continue;
        std::vector<std::pair<float, int>> nb;
        G.knn(m[0], m[1], m[2], 1, nb);
        d2[i] = nb[0].first;
    }
    double fitness = DBL_MAX, sum = 0.0;
    int cnt = 0;
    for (float d : d2)
        if (d >= 0.f) sum += (double)d, ++cnt;
    if (cnt) fitness = sum / cnt;
    ndt_epilogue(T, guess, moved, out->trans);
    out->code = fitness > (double)thre ? -3 : 1;
    out->iterations = iters;
    out->converged = converged;
    out->fitness = fitness;
    out->n_target = (int)tgt.size();
    out->n_source = (int)src.size();
    for (int i = 0; i < std::min(iters, cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].x[c] = tr[i].x[c], trace[i].delta[c] = tr[i].delta[c];
        trace[i].n_corr = tr[i].n_corr, trace[i].random_step = tr[i].random;
    }
    return MULLS_OK;
}

// the regularised covariances (n x 9, row-major 3x3) of a finite cloud of at least 20 points
void orc_gicp_covariances(const float *xyz, long n, float *out) {
    const std::vector<float> c = covariances(xyz_of(xyz, n));
    std::memcpy(out, c.data(), c.size() * sizeof(float));
}
// the 20 neighbour indices of every point, in list order
void orc_gicp_neighbours(const float *xyz, long n, int *out) {
    const std::vector<float4> p = xyz_of(xyz, n);
    HashGrid G;
    G.build(p);
    for (long i = 0; i < n; ++i) {
        std::vector<std::pair<float, int>> nb;
        G.knn(p[i].x, p[i].y, p[i].z, kGicpK, nb);
        for (int t = 0; t < kGicpK; ++t) out[kGicpK * i + t] = nb[t].second;
    }
}
// the voxels of a finite target: count, and up to cap of them (key, point count, mean, covariance)
long orc_gicp_voxels(const float *xyz, long n, float res, long cap, uint64_t *keys, int *cnt, float *mean, float *cov) {
    const std::vector<float4> p = xyz_of(xyz, n);
    const Voxels V = build_voxels(p, covariances(p), res);
    for (long i = 0; i < (long)V.keys.size() && i < cap; ++i) {
        keys[i] = V.keys[i], cnt[i] = V.n[i];
        std::memcpy(mean + 3 * i, V.vox[i].mean, 3 * sizeof(float));
        std::memcpy(cov + 9 * i, V.vox[i].cov, 9 * sizeof(float));
    }
    return (long)V.keys.size();
}
// the 28 summed terms at the point x (so3, translation) of the walk
void orc_gicp_eval(const float *txyz, long nt, const float *sxyz, long ns, float res, const float *x, double *out) {
    const std::vector<float4> t = xyz_of(txyz, nt), s = xyz_of(sxyz, ns);
    const Voxels V = build_voxels(t, covariances(t), res);
    float T[12];
    gicp_transform_of(x, T);
    evaluate(s, covariances(s), V, res, T, out);
}
void orc_gicp_voxel_coord(const float *xyz, long n, float res, int *out) {
    for (long i = 0; i < 3 * n; ++i) out[i] = gicp_coord(xyz[i], res);
}
void orc_gicp_so3_exp(const float *v, float *q) {
    const GicpQuat r = gicp_so3_exp(v);
    q[0] = r.w, q[1] = r.x, q[2] = r.y, q[3] = r.z;
}
void orc_gicp_so3_log(const float *q, float *v) { gicp_so3_log(GicpQuat{q[0], q[1], q[2], q[3]}, v); }
void orc_gicp_so3_mul(const float *a, const float *b, float *q) {
    const GicpQuat r = gicp_so3_mul(GicpQuat{a[0], a[1], a[2], a[3]}, GicpQuat{b[0], b[1], b[2], b[3]});
    q[0] = r.w, q[1] = r.x, q[2] = r.y, q[3] = r.z;
}
void orc_gicp_transform(const float *x, float *T) { gicp_transform_of(x, T); }
void orc_gicp_llt_solve(const double *A, const double *b, double *x) {
    double M[6][6];
    for (int i = 0; i < 36; ++i) M[i / 6][i % 6] = A[i];
    gicp_llt_solve(M, b, x);
}

} // extern "C"
