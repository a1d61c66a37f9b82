// TEST INFRASTRUCTURE, NOT PRODUCT CODE. CPU restatement of lo::CRegistration<PointT>::coarse_reg_teaser
// (include/common/cregistration.hpp:664-759), the checker of mulls_coarse_reg_teaser, over the readings T1-T9 of
// mulls_b200/csrc/teaser_core.cuh, sequentially: the consistency graph (T1-T2), its core numbers by bucket peeling
// (Matula-Beck, not the device's h-index iteration), the clique number by a recursive colour-bounded branch and bound
// over the whole graph (no core pruning, no greedy bound), the lexicographically smallest clique of that size by a
// depth-first search in index order (T3, T9), GNC-TLS over the chain TIMs (T4-T6) and the voted translation with
// std::sort (T7). The arithmetic the device must match bit for bit (the edge test, svdRot, the weights, the fixed-order
// sums, the sweep) comes from teaser_core.cuh. orc_tm_clique exposes the clique step on a given graph.
// Built by tests/test_teaser.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/mulls_b200/abi.h"
#include "../../mulls_b200/csrc/teaser_core.cuh"

using namespace mulls;

namespace {

struct Graph {
    int n, W;
    std::vector<uint64_t> adj;
    const uint64_t *row(int v) const { return adj.data() + (size_t)v * W; }
};
using Set = std::vector<uint64_t>;

bool has(const Set &s, int v) { return (s[v >> 6] >> (v & 63)) & 1ull; }
void clear_bit(Set &s, int v) { s[v >> 6] &= ~(1ull << (v & 63)); }
int lowest(const Set &s) {
    for (size_t w = 0; w < s.size(); ++w)
        if (s[w]) return (int)(64 * w) + __builtin_ctzll(s[w]);
    return -1;
}
bool empty(const Set &s) { return lowest(s) < 0; }

// greedy colouring in index order: the vertices by class, and the class number of each
void colour(const Graph &g, Set Q, std::vector<int> &order, std::vector<int> &col) {
    order.clear(), col.clear();
    int k = 0;
    while (!empty(Q)) {
        ++k;
        Set U = Q;
        for (int v = lowest(U); v >= 0; v = lowest(U)) {
            clear_bit(U, v), clear_bit(Q, v);
            for (int w = 0; w < g.W; ++w) U[w] &= ~g.row(v)[w];
            order.push_back(v), col.push_back(k);
        }
    }
}
int colours(const Graph &g, const Set &P) {
    std::vector<int> o, c;
    colour(g, P, o, c);
    return c.empty() ? 0 : c.back();
}

// the clique number: MCQ-style expansion, branching on the highest colour class first
void expand_max(const Graph &g, int size, Set P, int &best) {
    std::vector<int> order, col;
    colour(g, P, order, col);
    for (int k = (int)order.size() - 1; k >= 0; --k) {
        if (size + col[k] <= best) return;
        const int v = order[k];
        Set C(g.W);
        for (int w = 0; w < g.W; ++w) C[w] = P[w] & g.row(v)[w];
        if (empty(C)) best = std::max(best, size + 1);
        else expand_max(g, size + 1, C, best);
        clear_bit(P, v);
    }
}
// the lexicographically smallest clique of `target` vertices within P, extending `path`
bool expand_lex(const Graph &g, int target, Set P, std::vector<int> &path) {
    if ((int)path.size() == target) return true;
    for (int v = lowest(P); v >= 0; v = lowest(P)) {
        if ((int)path.size() + colours(g, P) < target) return false;
        Set C(g.W);
        clear_bit(P, v);
        for (int w = 0; w < g.W; ++w) C[w] = P[w] & g.row(v)[w];
        path.push_back(v);
        if (expand_lex(g, target, C, path)) return true;
        path.pop_back();
    }
    return false;
}
// T3 + T9: the maximum clique, lexicographically smallest; the clique number in *omega (1 for a graph without edges)
std::vector<int> max_clique(const Graph &g) {
    Set all(g.W, 0);
    for (int v = 0; v < g.n; ++v) all[v >> 6] |= 1ull << (v & 63);
    int best = g.n > 0 ? 1 : 0;
    expand_max(g, 0, all, best);
    std::vector<int> path;
    if (best > 0) expand_lex(g, best, all, path);
    return path;
}
// core numbers by peeling: repeatedly remove a vertex of least remaining degree
std::vector<int> core_numbers(const Graph &g) {
    std::vector<int> deg(g.n), core(g.n, 0);
    int maxd = 0;
    for (int v = 0; v < g.n; ++v) {
        int d = 0;
        for (int w = 0; w < g.W; ++w) d += __builtin_popcountll(g.row(v)[w]);
        deg[v] = d, maxd = std::max(maxd, d);
    }
    std::vector<std::vector<int>> bucket(maxd + 1);
    for (int v = 0; v < g.n; ++v) bucket[deg[v]].push_back(v);
    std::vector<char> gone(g.n, 0);
    int k = 0;
    for (int done = 0; done < g.n;) {
        int d = 0;
        while (d <= maxd) {
            while (!bucket[d].empty() && (gone[bucket[d].back()] || deg[bucket[d].back()] != d)) bucket[d].pop_back();
            if (!bucket[d].empty()) break;
            ++d;
        }
        const int v = bucket[d].back();
        bucket[d].pop_back();
        k = std::max(k, d);
        core[v] = k, gone[v] = 1, ++done;
        for (int w = 0; w < g.W; ++w)
            for (uint64_t b = g.row(v)[w]; b; b &= b - 1) {
                const int u = 64 * w + __builtin_ctzll(b);
                if (!gone[u]) bucket[--deg[u]].push_back(u);
            }
    }
    return core;
}

} // namespace

extern "C" {

// the clique step on a given graph (n vertices, W = ceil(n / 64) words a row, symmetric): writes the clique to out
// (room for n) and returns its size
int orc_tm_clique(int n, const uint64_t *adj, int *out) {
    Graph g{n, (n + 63) / 64, std::vector<uint64_t>(adj, adj + (size_t)n * ((n + 63) / 64))};
    const std::vector<int> c = max_clique(g);
    std::copy(c.begin(), c.end(), out);
    return (int)c.size();
}
void orc_tm_core(int n, const uint64_t *adj, int *core_out) {
    Graph g{n, (n + 63) / 64, std::vector<uint64_t>(adj, adj + (size_t)n * ((n + 63) / 64))};
    const std::vector<int> c = core_numbers(g);
    std::copy(c.begin(), c.end(), core_out);
}
// the graph of T1-T2 (n x W words)
void orc_tm_graph(const float *t48, const float *s48, long N, float noise_bound, uint64_t *adj) {
    std::vector<double> p6(6 * N);
    for (long i = 0; i < N; ++i)
        for (int c = 0; c < 3; ++c) p6[6 * i + c] = (double)s48[12 * i + c], p6[6 * i + 3 + c] = (double)t48[12 * i + c];
    const int W = (int)((N + 63) / 64);
    std::memset(adj, 0, (size_t)N * W * 8);
    for (long i = 0; i < N; ++i)
        for (long j = i + 1; j < N; ++j)
            if (tm_edge(p6.data(), (int)i, (int)j, 2.0 * (double)noise_bound)) {
                adj[(size_t)i * W + (j >> 6)] |= 1ull << (j & 63);
                adj[(size_t)j * W + (i >> 6)] |= 1ull << (i & 63);
            }
}

// returns 0; status and info as mulls_coarse_reg_teaser (search_launches 0); tran written when status >= 0; clique_out
// (room for N) and mask_out (room for N) receive the clique and the rotation-inlier mask
int orc_teaser(const float *t48, long nt, const float *s48, long ns, float noise_bound, int min_inlier_num, double *tran_mat,
               int *status, mulls_teaser_info *info, int *clique_out, uint8_t *mask_out) {
    *info = mulls_teaser_info{};
    *status = -1;
    if (nt != ns || nt <= 3) return 0;
    const long N = nt;
    const double nb = (double)noise_bound;
    std::vector<double> p6(6 * N); // src = source, dst = target
    for (long i = 0; i < N; ++i)
        for (int c = 0; c < 3; ++c) p6[6 * i + c] = (double)s48[12 * i + c], p6[6 * i + 3 + c] = (double)t48[12 * i + c];
    Graph g{(int)N, (int)((N + 63) / 64), {}};
    g.adj.assign((size_t)N * g.W, 0);
    orc_tm_graph(t48, s48, N, noise_bound, g.adj.data());
    for (long i = 0; i < N; ++i)
        for (int w = 0; w < g.W; ++w) info->n_edges += __builtin_popcountll(g.row((int)i)[w]);
    info->n_edges /= 2;
    for (int c : core_numbers(g)) info->max_core = std::max(info->max_core, c);
    const std::vector<int> clique = max_clique(g);
    const int M = (int)clique.size();
    info->clique_size = M;
    std::copy(clique.begin(), clique.end(), clique_out);
    if (M <= 1) return 0; // solution.valid = false
    // ---- T4-T6: GNC-TLS over the chain TIMs ----
    std::vector<double> tims(6 * (size_t)M), w(M, 1.0), r(M);
    for (int k = 0; k < M; ++k) {
        const double *a = &p6[6 * (size_t)clique[k]], *b = &p6[6 * (size_t)clique[k + 1 < M ? k + 1 : 0]];
        for (int c = 0; c < 6; ++c) tims[6 * (size_t)k + c] = b[c] - a[c];
    }
    const double nb_sq = tm_gnc_nb_sq(nb);
    double mu = 1.0, prev_cost = INFINITY, R[9];
    int it = 0;
    for (int i = 0; i < kTmGncMaxIter; ++i) {
        it = i + 1;
        double h[9];
        tm_sums_serial<9>(M, [&](int k, double x[9]) { tm_h_terms(&tims[6 * (size_t)k], &tims[6 * (size_t)k + 3], w[k], x); }, h);
        tm_svd_rot(h, R);
        for (int k = 0; k < M; ++k) r[k] = tm_residual(R, &tims[6 * (size_t)k], &tims[6 * (size_t)k + 3]);
        if (i == 0) {
            const double max_residual = *std::max_element(r.begin(), r.end());
            mu = tm_gnc_mu0(max_residual, nb_sq);
            if (mu <= 0) break;
        }
        double cost;
        tm_sums_serial<1>(M, [&](int k, double x[1]) { x[0] = w[k] * r[k]; }, &cost);
        for (int k = 0; k < M; ++k) w[k] = tm_gnc_weight(r[k], mu, nb_sq);
        const double cost_diff = std::abs(cost - prev_cost);
        mu = mu * kTmGncFactor;
        prev_cost = cost;
        if (cost_diff < kTmGncCostThreshold) break;
    }
    int inl = 0;
    for (int k = 0; k < M; ++k) {
        mask_out[k] = w[k] >= 0.5 ? 1 : 0;
        inl += mask_out[k];
    }
    info->gnc_iterations = it;
    info->rotation_inliers = inl;
    // ---- T7: TLS voting per axis over the clique's correspondences ----
    double t[3];
    for (int a = 0; a < 3; ++a) {
        std::vector<double> x(M);
        std::vector<TmBound> hb;
        for (int i = 0; i < M; ++i) {
            const double *p = &p6[6 * (size_t)clique[i]];
            x[i] = p[3 + a] - ((R[3 * a] * p[0] + R[3 * a + 1] * p[1]) + R[3 * a + 2] * p[2]);
            hb.push_back(tm_bound(x[i], nb, i, false));
            hb.push_back(tm_bound(x[i], nb, i, true));
        }
        std::sort(hb.begin(), hb.end(), tm_vote_less);
        t[a] = tm_vote_sweep(hb.data(), 2 * M, x.data(), nb);
    }
    const size_t cnt = (size_t)inl;
    if (cnt >= (size_t)(int64_t)min_inlier_num) {
        for (int rr = 0; rr < 3; ++rr) {
            for (int c = 0; c < 3; ++c) tran_mat[4 * rr + c] = R[3 * rr + c];
            tran_mat[4 * rr + 3] = t[rr];
        }
        tran_mat[12] = tran_mat[13] = tran_mat[14] = 0.0;
        tran_mat[15] = 1.0;
        *status = cnt >= (size_t)(int64_t)(int32_t)((uint32_t)min_inlier_num * 2u) ? 1 : 0;
    }
    return 0;
}

} // extern "C"
