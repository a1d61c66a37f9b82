// TEST INFRASTRUCTURE, NOT PRODUCT CODE. The walks of several NDT registrations advanced in lockstep, one evaluation of
// every live walk per round, as mulls_omp_ndt_batch advances them (ndt_walk_start / ndt_walk_advance of
// mulls_b200/csrc/ndt_core.cuh), over the CPU restatement's leaves and evaluation (tests/harness/ndt_oracle.cpp, included
// here). tests/test_ndt_batch.py checks that each walk ends as ndt_walk (orc_ndt) ends it for that pair alone.
// Built by tests/test_ndt_batch.py with nvcc as host code (-x cu), host flags -O2 -ffp-contract=off.
#include "ndt_oracle.cpp"

extern "C" {

// n pairs: rows t48[i] / s48[i] with nt[i] / ns[i] points, resolution res[i], guesses[16 i], apply_filter[i], bounds
// tb[6 i], sb[6 i];
// out[i] receives the walk's iterations, converged, n_target, n_source and trans (Trans1_2; code and fitness are left
// out), trace[i * cap ..] its rows. Returns the number of rounds (the longest walk's evaluations).
int orc_ndt_lockstep(int n, const float *const *t48, const long *nt, const float *const *s48, const long *ns, const float *res,
                     const double *guesses, const int *apply_filter, const double *tb, const double *sb, mulls_ndt_result *out,
                     mulls_ndt_iter *trace, int cap) {
    struct Pair {
        std::vector<float4> tgt, src;
        bool moved = false;
        NdtGrid g;
        Leaves L;
        NdtWalk W;
        std::vector<NdtIter> tr;
    };
    std::vector<Pair> P(n);
    for (int i = 0; i < n; ++i) {
        Pair &p = P[i];
        ndt_prologue(t48[i], (size_t)nt[i], s48[i], (size_t)ns[i], guesses + 16 * i, apply_filter[i], tb + 6 * i, sb + 6 * i, p.tgt,
                     p.src, p.moved);
        p.g = ndt_grid_from(p.tgt, res[i]);
        p.L = build_leaves(p.tgt, p.g);
        p.tr.resize(cap > 0 ? cap : 0);
        ndt_walk_start(p.W);
    }
    std::vector<int> live(n), next;
    for (int i = 0; i < n; ++i) live[i] = i;
    int rounds = 0;
    while (!live.empty()) {
        ++rounds;
        for (int i : live) { // every live walk is evaluated before any advances
            NdtEvalConst E;
            consts_at(P[i].W.q, P[i].W.T, res[i], E);
            evaluate(P[i].src, P[i].g, P[i].L, E, P[i].W.r);
        }
        next.clear();
        for (int i : live)
            if (ndt_walk_advance(P[i].W, P[i].tr.data(), (int)P[i].tr.size())) next.push_back(i);
        live.swap(next);
    }
    for (int i = 0; i < n; ++i) {
        const Pair &p = P[i];
        mulls_ndt_result &o = out[i];
        ndt_epilogue(p.W.T, guesses + 16 * i, p.moved, o.trans);
        o.iterations = p.W.nr;
        o.converged = p.W.converged;
        o.n_target = (int)p.tgt.size();
        o.n_source = (int)p.src.size();
        for (int k = 0; k < std::min(p.W.nr, cap); ++k) {
            mulls_ndt_iter &d = trace[(size_t)i * cap + k];
            for (int c = 0; c < 6; ++c) d.p[c] = p.tr[k].p[c];
            d.step = p.tr[k].step, d.score = p.tr[k].score, d.reversed = p.tr[k].reversed;
        }
    }
    return rounds;
}

} // extern "C"
