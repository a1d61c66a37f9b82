// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::omp_ndt with DIRECT7
// (include/common/cregistration.hpp:945-1021), the checker of mulls_omp_ndt. The readings and every piece both sides
// must compute alike (prologue, leaf grid and finalisation, DIRECT7 probes, derivatives, the summation order C1, the
// Newton walk) come from mulls_b200/csrc/ndt_core.cuh and run here on the host, sequentially: the leaves by a stable
// sort of the leaf keys, the DIRECT7 lookup by binary search, the fitness by brute force over the target.
// Built by tests/test_ndt.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include <algorithm>
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
        while (b < n && key[ord[b]] == key[ord[a]]) {
            const float4 p = tgt[ord[b]];
            const double v[3] = {(double)p.x, (double)p.y, (double)p.z};
            for (int i = 0; i < 3; ++i) {
                s[i] += v[i];
                for (int j = 0; j < 3; ++j) c[3 * i + j] += v[i] * v[j];
            }
            ++b;
        }
        L.keys.push_back(key[ord[a]]);
        L.leaf.push_back(ndt_leaf_finish(s, c, (int)(b - a)));
        a = b;
    }
    return L;
}

void evaluate(const std::vector<float4> &src, const NdtGrid &g, const Leaves &L, const NdtEvalConst &E, double r[kNdtTerms]) {
    const size_t n = src.size();
    for (int c = 0; c < kNdtTerms; ++c) r[c] = 0.0;
    std::vector<double> acc((size_t)kNdtTile * kNdtTerms), q(kNdtTile);
    for (size_t t0 = 0; t0 < n; t0 += kNdtTile) {
        std::fill(acc.begin(), acc.end(), 0.0);
        for (int t = 0; t < kNdtTile && t0 + t < n; ++t) {
            const float4 p = src[t0 + t];
            if (!g.ok || !ndt_finite3(p.x, p.y, p.z)) continue;
            const float x[3] = {p.x, p.y, p.z};
            float tr[3];
            ndt_transform(E.T, p.x, p.y, p.z, tr);
            if (!ndt_finite3(tr[0], tr[1], tr[2])) continue;
            for (int k = 0; k < 7; ++k) {
                int64_t key;
                if (!ndt_probe_key(g, tr[0], tr[1], tr[2], k, key)) continue;
                auto it = std::lower_bound(L.keys.begin(), L.keys.end(), key,
                                           [](int64_t a, int64_t b) { return (uint64_t)a < (uint64_t)b; });
                if (it == L.keys.end() || *it != key) continue;
                const NdtLeaf &lf = L.leaf[it - L.keys.begin()];
                if (!lf.ok) continue;
                const double xt[3] = {(double)tr[0] - lf.mean[0], (double)tr[1] - lf.mean[1], (double)tr[2] - lf.mean[2]};
                ndt_update(E, x, xt, lf.icov, &acc[(size_t)t * kNdtTerms]);
            }
        }
        for (int c = 0; c < kNdtTerms; ++c) {
            for (int t = 0; t < kNdtTile; ++t) q[t] = acc[(size_t)t * kNdtTerms + c];
            r[c] += ndt_tile_sum(q.data());
        }
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

int orc_ndt(const float *t48, long nt, const float *s48, long ns, float resolution, const double *guess, int apply_filter,
            float thre, const double *tb, const double *sb, mulls_ndt_result *out, mulls_ndt_iter *trace, int cap) {
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(t48, (size_t)nt, s48, (size_t)ns, guess, apply_filter, tb, sb, tgt, src, moved);
    const NdtGrid g = ndt_grid_from(tgt, resolution);
    const Leaves L = build_leaves(tgt, g);
    NdtEvalConst E;
    auto eval = [&](const double p[6], const float T[12], double r[kNdtTerms]) {
        consts_at(p, T, resolution, E);
        evaluate(src, g, L, E, r);
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

// the leaves of a target cloud (no filter): count, and up to cap of them (key, point count, mean, float icov, ok)
long orc_ndt_leaves(const float *t48, long nt, float resolution, long cap, int64_t *keys, int *n, double *mean, float *icov, int *ok) {
    std::vector<float4> all = rows_of(t48, nt), tgt;
    for (const float4 &p : all)
        if (ndt_finite3(p.x, p.y, p.z)) tgt.push_back(p);
    const NdtGrid g = ndt_grid_from(tgt, resolution);
    const Leaves L = build_leaves(tgt, g);
    for (long i = 0; i < (long)L.keys.size() && i < cap; ++i) {
        keys[i] = L.keys[i];
        n[i] = L.leaf[i].n;
        ok[i] = L.leaf[i].ok;
        for (int c = 0; c < 3; ++c) mean[3 * i + c] = L.leaf[i].mean[c];
        for (int c = 0; c < 9; ++c) icov[9 * i + c] = L.leaf[i].icov[c];
    }
    return (long)L.keys.size();
}

// score, gradient and Hessian at the pose vector p (no filter)
void orc_ndt_eval(const float *t48, long nt, const float *s48, long ns, float resolution, const double *p, double *out) {
    std::vector<float4> all = rows_of(t48, nt), tgt, src = rows_of(s48, ns);
    for (const float4 &q : all)
        if (ndt_finite3(q.x, q.y, q.z)) tgt.push_back(q);
    const NdtGrid g = ndt_grid_from(tgt, resolution);
    const Leaves L = build_leaves(tgt, g);
    float T[12];
    ndt_step_transform(p, T);
    NdtEvalConst E;
    consts_at(p, T, resolution, E);
    evaluate(src, g, L, E, out);
}

// ndt_svd_solve on one 6x6 system (row-major H)
void orc_ndt_solve(const double *H, const double *b, double *x) { ndt_svd_solve(H, b, x); }

void orc_ndt_expf(const float *in, float *out, long n) {
    for (long i = 0; i < n; ++i) out[i] = ndt_expf(in[i]);
}

void orc_ndt_gauss(float resolution, double *d1, double *d2) { ndt_gauss(resolution, *d1, *d2); }

} // extern "C"
