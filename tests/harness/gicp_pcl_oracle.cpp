// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::omp_gicp with
// using_voxel_gicp = false (include/common/cregistration.hpp:1024-1098, koide_reg::GeneralizedIterativeClosestPoint with
// PCL's BFGS), the checker of mulls_omp_gicp_pcl. The readings and every piece both sides must compute alike
// (prologue, neighbour sums and covariances, the Mahalanobis matrices, the functor's terms, the summation order C1,
// applyState, BFGS, the outer loop, the epilogue) come from mulls_b200/csrc/gicp_pcl_core.cuh and run here on the host,
// sequentially, on the exact nearest-neighbour search of gicp_oracle.cpp (FLANN's order on a hash grid). Built by
// tests/test_gicp_pcl.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include "gicp_oracle.cpp"

#include "../../mulls_b200/csrc/gicp_pcl_core.cuh"

namespace {

// P3 for every point of a cloud (at least kGicpK points): 9 doubles per point
std::vector<double> pcl_covariances(const std::vector<float4> &p) {
    HashGrid G;
    G.build(p);
    std::vector<double> cov(p.size() * 9);
#pragma omp parallel for schedule(dynamic, 256)
    for (long i = 0; i < (long)p.size(); ++i) {
        std::vector<std::pair<float, int>> nb;
        G.knn(p[i].x, p[i].y, p[i].z, kGicpK, nb);
        double s[9];
        gicp_pcl_neighbour_sums([&](int t, float q[3]) {
            const float4 v = p[nb[t].second];
            q[0] = v.x, q[1] = v.y, q[2] = v.z;
        }, s);
        gicp_pcl_plane(s, &cov[9 * i]);
    }
    return cov;
}

struct Scene {
    std::vector<float4> tgt, src;
    std::vector<double> tcov, scov;
    HashGrid G; // over tgt
    std::vector<int> list, tix;
    std::vector<float> maha;
    void init() {
        tcov = pcl_covariances(tgt);
        scov = pcl_covariances(src);
        G.build(tgt);
        tix.assign(src.size(), 0);
        maha.assign(src.size() * 9, 0.f);
    }
    // P4: the correspondences of the float transformation_ T, in source order
    int match(const float T[12], const double R[9]) {
        const long n = (long)src.size();
        std::vector<char> keep(n, 0);
#pragma omp parallel for schedule(dynamic, 256)
        for (long i = 0; i < n; ++i) {
            float t[3];
            ndt_transform(T, src[i].x, src[i].y, src[i].z, t);
            if (!ndt_finite3(t[0], t[1], t[2])) continue; // C3
            std::vector<std::pair<float, int>> nb;
            G.knn(t[0], t[1], t[2], 1, nb);
            if (nb.empty() || !((double)nb[0].first < kGicpPclCorrDist * kGicpPclCorrDist)) continue;
            const int j = nb[0].second;
            gicp_pcl_maha(R, &scov[9 * i], &tcov[9 * (size_t)j], &maha[9 * i]);
            tix[i] = j;
            keep[i] = 1;
        }
        list.clear();
        for (long i = 0; i < n; ++i)
            if (keep[i]) list.push_back((int)i);
        return (int)list.size();
    }
    // the method's terms summed over the correspondences in C1's order
    void eval(int method, const float T[12], double *r) {
        const int terms = gicp_pcl_terms(method), m = (int)list.size();
        for (int c = 0; c < terms; ++c) r[c] = 0.0;
        std::vector<double> acc((size_t)kNdtTile * kGicpPclMaxTerms), q(kNdtTile);
        for (int t0 = 0; t0 < m; t0 += kNdtTile) {
            std::fill(acc.begin(), acc.end(), 0.0);
            for (int t = 0; t < kNdtTile && t0 + t < m; ++t) {
                const int s = list[t0 + t];
                const float4 p = src[s], qq = tgt[tix[s]];
                const float a[3] = {p.x, p.y, p.z}, b[3] = {qq.x, qq.y, qq.z};
                double *o = &acc[(size_t)t * kGicpPclMaxTerms];
                if (method == kGicpPclF) gicp_pcl_terms<kGicpPclF>(T, a, b, &maha[9 * (size_t)s], o);
                else if (method == kGicpPclDf) gicp_pcl_terms<kGicpPclDf>(T, a, b, &maha[9 * (size_t)s], o);
                else gicp_pcl_terms<kGicpPclFdf>(T, a, b, &maha[9 * (size_t)s], o);
            }
            for (int c = 0; c < terms; ++c) {
                for (int t = 0; t < kNdtTile; ++t) q[t] = acc[(size_t)t * kGicpPclMaxTerms + c];
                r[c] += ndt_tile_sum(q.data());
            }
        }
    }
};

// the BFGS functor over a caller's fdf (tests of the solver alone)
typedef void (*FdfFn)(const double *x, double *f, double *g);
struct CbFn {
    FdfFn cb;
    int calls;
    double f(const double *x) {
        double fo, g[6];
        cb(x, &fo, g);
        ++calls;
        return fo;
    }
    void df(const double *x, double *g) {
        double fo;
        cb(x, &fo, g);
        ++calls;
    }
    void fdf(const double *x, double &fo, double *g) {
        cb(x, &fo, g);
        ++calls;
    }
};

} // namespace

extern "C" {

int orc_gicp_pcl(const float *t48, long nt, const float *s48, long ns, int max_iter, const double *guess, int apply_filter,
                 float thre, const double *tb, const double *sb, mulls_gicp_pcl_result *out, mulls_gicp_pcl_iter *trace, int cap) {
    Scene S;
    bool moved = false;
    ndt_prologue(t48, (size_t)nt, s48, (size_t)ns, guess, apply_filter, tb, sb, S.tgt, S.src, moved);
    gicp_keep_finite(S.src);
    if ((long)S.tgt.size() < kGicpK || (long)S.src.size() < kGicpK) return MULLS_E_UNSUPPORTED;
    S.init();
    auto match = [&](const float T[12], const double R[9]) { return S.match(T, R); };
    auto eval = [&](int method, const float T[12], double *r) { S.eval(method, T, r); };
    std::vector<GicpPclIter> tr(cap > 0 ? cap : 0);
    float T[12];
    int converged = 0;
    const int iters = gicp_pcl_walk(max_iter, match, eval, T, converged, tr.data(), (int)tr.size());
    // getFitnessScore over the same exact nearest search
    std::vector<float> d2(S.src.size(), -1.f);
#pragma omp parallel for schedule(dynamic, 256)
    for (long i = 0; i < (long)S.src.size(); ++i) {
        float m[3];
        ndt_transform(T, S.src[i].x, S.src[i].y, S.src[i].z, m);
        if (!ndt_finite3(m[0], m[1], m[2])) continue;
        std::vector<std::pair<float, int>> nb;
        S.G.knn(m[0], m[1], m[2], 1, nb);
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
    out->n_target = (int)S.tgt.size();
    out->n_source = (int)S.src.size();
    for (int i = 0; i < std::min(iters, cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].x[c] = tr[i].x[c];
        trace[i].delta = tr[i].delta, trace[i].n_corr = tr[i].n_corr, trace[i].inner_iterations = tr[i].inner;
        trace[i].status = tr[i].status, trace[i].evaluations = tr[i].evaluations;
    }
    return MULLS_OK;
}

// the covariances (n x 9, row-major 3x3, double) of a finite cloud of at least 20 points
void orc_gicp_pcl_covariances(const float *xyz, long n, double *out) {
    const std::vector<double> c = pcl_covariances(xyz_of(xyz, n));
    std::memcpy(out, c.data(), c.size() * sizeof(double));
}
void orc_gicp_pcl_maha(const double *R, const double *c1, const double *c2, float *M) { gicp_pcl_maha(R, c1, c2, M); }
void orc_gicp_pcl_inv3(const double *m, double *out) { gicp_pcl_inv3(m, out); }
void orc_gicp_pcl_apply_state(const double *x, float *T) { gicp_pcl_apply_state(x, T); }
// the correspondences of transformation_ = T0 (rows 0..2, float) and the three methods at x: f of operator(), g of df,
// f and g of fdf; returns the correspondence count. src_idx / tgt_idx (may be NULL) receive the pairs.
int orc_gicp_pcl_functor(const float *txyz, long nt, const float *sxyz, long ns, const float *T0, const double *x, double *f,
                         double *g_df, double *f_fdf, double *g_fdf, int *src_idx, int *tgt_idx) {
    Scene S;
    S.tgt = xyz_of(txyz, nt), S.src = xyz_of(sxyz, ns);
    S.init();
    double R[9];
    gicp_pcl_transform_R(T0, R);
    const int m = S.match(T0, R);
    for (int c = 0; c < m; ++c) {
        if (src_idx) src_idx[c] = S.list[c];
        if (tgt_idx) tgt_idx[c] = S.tix[S.list[c]];
    }
    float T[12];
    gicp_pcl_apply_state(x, T);
    double s[kGicpPclMaxTerms];
    S.eval(kGicpPclF, T, s);
    *f = gicp_pcl_finish_f(s, m);
    S.eval(kGicpPclDf, T, s);
    gicp_pcl_finish_g(x, s, m, g_df);
    S.eval(kGicpPclFdf, T, s);
    *f_fdf = gicp_pcl_finish_f(s, m);
    gicp_pcl_finish_g(x, s + 1, m, g_fdf);
    return m;
}
// estimateRigidTransformationBFGS's solve on a caller's function: x (in: start, out: result), the do-while with
// gradient tolerance tol and max_inner steps; returns the status, steps and functor calls in info[0..2]
void orc_gicp_pcl_bfgs(FdfFn cb, double *x, int max_inner, double tol, int *info) {
    CbFn fn{cb, 0};
    GicpPclBfgs<CbFn> bfgs(fn);
    int inner = 0;
    int result = bfgs.minimize_init(x);
    result = kBfgsRunning;
    do {
        ++inner;
        result = bfgs.minimize_one_step(x);
        if (result) break;
        result = bfgs.test_gradient(tol);
    } while (result == kBfgsRunning && inner < max_inner);
    info[0] = result, info[1] = inner, info[2] = fn.calls;
}

} // extern "C"
