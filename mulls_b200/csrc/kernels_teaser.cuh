// TEASER++ coarse registration on the device (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759): the
// readings and the shared arithmetic are in teaser_core.cuh.
//  - k_tm_graph: the consistency graph as an N x W bitset (W = ceil(N / 64) words a row), one thread per word, i.e.
//    64 pair tests (T2) in double; the degrees and the edge count in the same pass;
//  - k_tm_hindex: one h-index step per vertex (one warp each); from the degrees, repeated until nothing changes, it
//    gives the core numbers (they are unique, so any exact method agrees);
//  - k_tm_greedy: one block, a greedy clique (highest core number first, ties to the lower index): the lower bound;
//  - k_tm_compact: the graph induced by the vertices whose core number can reach the bound, indices in ascending order;
//  - k_tm_search: the exact search, one warp per root vertex r over the neighbours above r, candidate sets as bitsets
//    (the node being expanded in registers, the stack in global memory), pruned by a greedy colouring. kTmMax finds
//    the clique number (a global best raised with atomicMax) on the graph relabelled in ascending core number, so that
//    each root's candidates are about its core number; as MCQ does, it colours a node once and branches on the
//    candidates of the highest colours in that order (kTmOrder of them kept per level). kTmLex decides
//    for each r whether an omega-clique has r as its smallest vertex, branching on the lowest candidate first, so its
//    first success is the lexicographically smallest omega-clique from r; the smallest successful r wins (T9). Each
//    launch runs a bounded amount of work per warp and leaves its stack in global memory; the host relaunches.
//  - k_tm_gnc: one block, the whole GNC-TLS loop (T4-T6);
//  - k_tm_vote: one block per axis, a bitonic sort of the 2M boundaries and the sweep (T7).
#pragma once
#include "teaser_core.cuh"

namespace mulls {

constexpr int kTmGraphBlock = 256;
constexpr int kTmWarpsPerBlock = 4;  // k_tm_hindex and k_tm_search
constexpr int kTmVoteBlock = 1024;
constexpr int kTmGreedyBlock = 1024;

// ---- the graph ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTmGraphBlock) k_tm_graph(const double *__restrict__ p6, int n, int W, double beta,
                                                            uint64_t *__restrict__ adj, int *__restrict__ deg,
                                                            unsigned long long *__restrict__ n_edges) {
    const size_t t = (size_t)blockIdx.x * kTmGraphBlock + threadIdx.x;
    if (t >= (size_t)n * W) return;
    const int i = (int)(t / W), w = (int)(t % W);
    uint64_t bits = 0;
    const int j0 = 64 * w, j1 = min(n, j0 + 64);
    for (int j = j0; j < j1; ++j)
        if (j != i && tm_edge(p6, i, j, beta)) bits |= 1ull << (j - j0);
    adj[t] = bits;
    const int c = __popcll(bits);
    if (c) {
        atomicAdd(deg + i, c);
        atomicAdd(n_edges, (unsigned long long)c);
    }
}

// ---- core numbers: h(v) <- max k <= h(v) with |{u in N(v) : h(u) >= k}| >= k ----------------------------------------------
__device__ __forceinline__ int tm_count_at_least(const uint64_t *row, int W, const int *h, int k, int lane) {
    int c = 0;
    for (int w = lane; w < W; w += 32) {
        uint64_t b = row[w];
        while (b) {
            const int u = 64 * w + __ffsll((long long)b) - 1;
            b &= b - 1;
            c += (h[u] >= k) ? 1 : 0;
        }
    }
    return __reduce_add_sync(0xffffffffu, c);
}
__global__ void __launch_bounds__(32 * kTmWarpsPerBlock) k_tm_hindex(const uint64_t *__restrict__ adj, int n, int W, int *h,
                                                                     int *changed) {
    const int v = blockIdx.x * kTmWarpsPerBlock + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (v >= n) return;
    const uint64_t *row = adj + (size_t)v * W;
    const int hv = *(volatile int *)(h + v);
    if (hv == 0 || tm_count_at_least(row, W, h, hv, lane) >= hv) return;
    int lo = 0, hi = hv - 1; // count(lo) >= lo holds; the answer is in [lo, hi]
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (tm_count_at_least(row, W, h, mid, lane) >= mid) lo = mid;
        else hi = mid - 1;
    }
    if (lane == 0) {
        *(volatile int *)(h + v) = lo;
        *changed = 1;
    }
}

// ---- the greedy lower bound: one block; cand is W words of scratch; out[0] the clique size --------------------------------------
__device__ __forceinline__ unsigned long long tm_max_u64(unsigned long long x) {
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, o);
        x = y > x ? y : x;
    }
    return x;
}
__global__ void __launch_bounds__(kTmGreedyBlock) k_tm_greedy(const uint64_t *__restrict__ adj, int n, int W,
                                                              const int *__restrict__ core, uint64_t *cand, int *out) {
    __shared__ unsigned long long s_key[kTmGreedyBlock / 32], s_best;
    const int tid = threadIdx.x, lane = tid & 31;
    for (int w = tid; w < W; w += kTmGreedyBlock) cand[w] = (64 * w + 64 <= n) ? ~0ull : (n > 64 * w ? (1ull << (n - 64 * w)) - 1 : 0ull);
    __syncthreads();
    int size = 0;
    for (;;) {
        unsigned long long key = 0; // (core + 1) << 32 | ~index: the highest core number, then the lowest index
        for (int w = tid; w < W; w += kTmGreedyBlock)
            for (uint64_t b = cand[w]; b; b &= b - 1) {
                const int u = 64 * w + __ffsll((long long)b) - 1;
                const unsigned long long k = ((unsigned long long)(core[u] + 1) << 32) | (0xffffffffu - (unsigned)u);
                key = k > key ? k : key;
            }
        key = tm_max_u64(key);
        if (lane == 0) s_key[tid / 32] = key;
        __syncthreads();
        if (tid < 32) {
            const unsigned long long k = tm_max_u64(s_key[lane]);
            if (lane == 0) s_best = k;
        }
        __syncthreads();
        key = s_best;
        if (!key) break;
        const int v = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
        ++size;
        for (int w = tid; w < W; w += kTmGreedyBlock) cand[w] &= adj[(size_t)v * W + w];
        __syncthreads();
    }
    if (tid == 0) out[0] = size;
}

// ---- the pruned graph: row i' is old row map[i'], bit j' is old bit map[j'] ---------------------------------------------------
__global__ void __launch_bounds__(kTmGraphBlock) k_tm_compact(const uint64_t *__restrict__ adj, int W, const int *__restrict__ map,
                                                              int n2, int W2, uint64_t *__restrict__ adj2) {
    const size_t t = (size_t)blockIdx.x * kTmGraphBlock + threadIdx.x;
    if (t >= (size_t)n2 * W2) return;
    const int i = (int)(t / W2), w = (int)(t % W2);
    const uint64_t *row = adj + (size_t)map[i] * W;
    uint64_t bits = 0;
    const int j0 = 64 * w, j1 = min(n2, j0 + 64);
    for (int j = j0; j < j1; ++j) {
        const int u = map[j];
        if ((row[u >> 6] >> (u & 63)) & 1ull) bits |= 1ull << (j - j0);
    }
    adj2[t] = bits;
}

// ---- the exact search ------------------------------------------------------------------------------------------------------
enum TmMode { kTmMax = 0, kTmLex = 1 };
constexpr int kTmOrder = 32; // kTmMax: branch candidates a level keeps from its colouring
struct TmSlot {
    int task;   // the root vertex, -1: none
    int level;  // the clique size of the node on top of the stack
};
// kTmMax, per level: the branch candidates of the level's last colouring (colour > best - level at that time), kept as
// a ring of the last kTmOrder taken, highest colour last
struct TmLevel {
    int m;       // candidates left; -1: colour the level (fresh, or the ring ran out with candidates left over)
    int pos;     // the next candidate is ring[(pos - 1) mod kTmOrder]
    int partial; // the colouring had more candidates than the ring holds
    int pad;
};
struct TmCtl {
    int next_task;                  // the next root to hand out
    int best;                       // kTmMax: the largest clique size found
    int active;                     // slots holding a task at the end of the last launch
    int pad;
    unsigned long long found;       // kTmLex: (root << 32) | slot of the smallest successful root, ~0 while none
    unsigned long long work;        // words of the pruned graph processed so far
    unsigned long long nodes;       // search nodes expanded so far
};
struct TmSearchArgs {
    const uint64_t *adj; // pruned graph, n x W
    const int *core;     // kTmMax: the core number of each vertex of the pruned graph
    int n, W;
    int levels;          // stack levels per slot: the clique bound + 1
    int mode;
    int target;          // kTmLex: omega
    int ub;              // kTmMax: the clique bound, reaching it ends the search
    unsigned long long launch_words; // work per warp and launch
    uint64_t *stack;     // slots x levels x W
    int *path;           // slots x levels: the vertex chosen at each level
    TmLevel *lvl;        // slots x levels
    int2 *ring;          // slots x levels x kTmOrder: (vertex, colour)
    TmSlot *slots;
    TmCtl *ctl;
};

// a warp's bitset of W <= 32 * WPL words in registers: lane l holds words l, l + 32, ...
template <int WPL> struct TmBits {
    uint64_t x[WPL];
    __device__ __forceinline__ void load(const uint64_t *p, int W, int lane) {
#pragma unroll
        for (int i = 0; i < WPL; ++i) x[i] = (lane + 32 * i < W) ? p[lane + 32 * i] : 0ull;
    }
    // the lowest set bit, or INT_MAX
    __device__ __forceinline__ int first() const {
#pragma unroll
        for (int i = 0; i < WPL; ++i) {
            const unsigned m = __ballot_sync(0xffffffffu, x[i] != 0ull);
            if (m) {
                const int l = __ffs(m) - 1;
                const uint64_t w = __shfl_sync(0xffffffffu, x[i], l);
                return 64 * (32 * i + l) + __ffsll((long long)w) - 1;
            }
        }
        return INT_MAX;
    }
    __device__ __forceinline__ void clear(int v, int lane) {
        const int w = v >> 6;
#pragma unroll
        for (int i = 0; i < WPL; ++i)
            if (lane + 32 * i == w) x[i] &= ~(1ull << (v & 63));
    }
    __device__ __forceinline__ void andnot_row(const uint64_t *row, int W, int lane) {
#pragma unroll
        for (int i = 0; i < WPL; ++i)
            if (lane + 32 * i < W) x[i] &= ~row[lane + 32 * i];
    }
    __device__ __forceinline__ int count() const {
        int c = 0;
#pragma unroll
        for (int i = 0; i < WPL; ++i) c += __popcll(x[i]);
        return __reduce_add_sync(0xffffffffu, c);
    }
};

template <int WPL>
__global__ void __launch_bounds__(32 * kTmWarpsPerBlock, 1) k_tm_search(TmSearchArgs A) {
    const int lane = threadIdx.x & 31;
    const int slot = blockIdx.x * kTmWarpsPerBlock + threadIdx.x / 32;
    const int W = A.W;
    uint64_t *stk = A.stack + (size_t)slot * A.levels * W;
    int *path = A.path + (size_t)slot * A.levels;
    TmLevel *lvl = A.lvl + (size_t)slot * A.levels;
    int2 *ring = A.ring + (size_t)slot * A.levels * kTmOrder;
    volatile TmCtl *ctl = A.ctl;
    int task = A.slots[slot].task, level = A.slots[slot].level;
    unsigned long long work = 0, nodes = 0;
    while (work < A.launch_words) {
        if (task < 0) { // take the next root
            int t = 0;
            if (lane == 0) t = atomicAdd(&A.ctl->next_task, 1);
            t = __shfl_sync(0xffffffffu, t, 0);
            if (t >= A.n) break;
            if (A.mode == kTmLex && (unsigned long long)t > (ctl->found >> 32)) break; // roots are handed out ascending
            if (A.mode == kTmMax && ctl->best >= A.ub) break;
            if (A.mode == kTmMax && A.core[t] + 1 <= ctl->best) continue; // no clique through t beats the best
            task = t, level = 1;
            const uint64_t *row = A.adj + (size_t)t * W;
            for (int w = lane; w < W; w += 32) { // the neighbours above t
                uint64_t m = 0;
                if (64 * w + 63 <= t) m = 0;
                else if (64 * w > t) m = ~0ull;
                else m = ~0ull << (t - 64 * w) << 1;
                stk[(size_t)1 * W + w] = row[w] & m;
            }
            if (lane == 0) {
                path[0] = t;
                lvl[1].m = -1;
            }
            work += W;
            __syncwarp();
        }
        // the node on top of the stack: clique size `level`, candidates P = stk[level]
        if ((A.mode == kTmLex && (unsigned long long)task > (ctl->found >> 32)) || (A.mode == kTmMax && ctl->best >= A.ub)) {
            task = -1;
            continue;
        }
        ++nodes;
        uint64_t *P = stk + (size_t)level * W;
        int branch = -1;
        if (A.mode == kTmMax) {
            // MCQ: colour P once, keep the candidates whose colour can beat the best, branch on them from the highest
            // colour down; recolour only when the ring ran out with candidates left over
            const int best = ctl->best;
            TmLevel L = lvl[level];
            if (L.m < 0) {
                const int t = best - level; // colours up to t cannot beat the best
                TmBits<WPL> Q, U;
                Q.load(P, W, lane);
                int c = 0, total = 0;
                for (int v = Q.first(); v != INT_MAX; v = Q.first()) {
                    ++c;
                    U = Q;
                    for (int u = v; u != INT_MAX; u = U.first()) { // one colour class: an independent set taken greedily
                        U.clear(u, lane), Q.clear(u, lane);
                        U.andnot_row(A.adj + (size_t)u * W, W, lane);
                        if (c > t) {
                            if (lane == 0) ring[level * kTmOrder + total % kTmOrder] = make_int2(u, c);
                            ++total;
                        }
                        work += 2 * W;
                    }
                }
                L.m = min(total, kTmOrder), L.pos = total, L.partial = total > kTmOrder ? 1 : 0;
                __syncwarp();
            }
            int2 cand = make_int2(-1, 0);
            if (L.m > 0) cand = ring[level * kTmOrder + (L.pos - 1) % kTmOrder];
            if (L.m == 0 || cand.y + level <= best) { // every candidate left has a colour that cannot beat the best
                if (--level == 0) task = -1;
                continue;
            }
            --L.m, --L.pos;
            if (L.m == 0 && L.partial) L.m = -1;
            if (lane == 0) lvl[level] = L;
            branch = cand.x;
        } else {
            // lex: branch on the lowest candidate while the colouring still reaches the target
            const int need = max(1, A.target - level);
            TmBits<WPL> Q, U;
            Q.load(P, W, lane);
            const int pc = Q.count();
            work += W;
            if (pc < need) { // fewer candidates than colours wanted
                if (--level == 0) task = -1;
                continue;
            }
            if (pc == need) { // every candidate must join: a success exactly when they form a clique
                bool ok = true;
                TmBits<WPL> R = Q;
                for (int u = R.first(); u != INT_MAX && ok; u = R.first()) {
                    R.clear(u, lane);
                    TmBits<WPL> X = Q;
                    X.clear(u, lane);
                    X.andnot_row(A.adj + (size_t)u * W, W, lane);
                    ok = X.first() == INT_MAX;
                    work += 2 * W;
                }
                if (ok && lane == 0) {
                    int k = level;
                    for (int w = 0; w < W; ++w)
                        for (uint64_t b = P[w]; b; b &= b - 1) path[k++] = 64 * w + __ffsll((long long)b) - 1;
                    __threadfence();
                    atomicMin((unsigned long long *)&A.ctl->found, ((unsigned long long)task << 32) | (unsigned)slot);
                }
                __syncwarp();
                if (ok) task = -1;
                else if (--level == 0) task = -1;
                continue;
            }
            const int lowest = Q.first();
            int ncol = 0;
            for (int v = lowest; v != INT_MAX && ncol < need; v = Q.first()) {
                ++ncol;
                U = Q;
                for (int u = v; u != INT_MAX; u = U.first()) {
                    U.clear(u, lane), Q.clear(u, lane);
                    U.andnot_row(A.adj + (size_t)u * W, W, lane);
                    work += 2 * W;
                }
            }
            if (ncol < need) { // no clique here can reach the target: back up
                if (--level == 0) task = -1;
                continue;
            }
            branch = lowest; // candidates in ascending order: the first success is the smallest
        }
        // branch on `branch`: drop it from P, push P & N(branch)
        const uint64_t *row = A.adj + (size_t)branch * W;
        uint64_t *C = P + W;
        for (int w = lane; w < W; w += 32) {
            uint64_t p = P[w];
            if (w == (branch >> 6)) p &= ~(1ull << (branch & 63));
            P[w] = p;
            C[w] = p & row[w];
        }
        work += W;
        if (lane == 0) {
            path[level] = branch;
            if (level + 1 < A.levels) lvl[level + 1].m = -1;
        }
        __syncwarp();
        ++level;
        if (A.mode == kTmMax) {
            if (level > ctl->best && lane == 0) atomicMax(&A.ctl->best, level);
        } else if (level == A.target) {
            if (lane == 0) {
                __threadfence();
                atomicMin((unsigned long long *)&A.ctl->found, ((unsigned long long)task << 32) | (unsigned)slot);
            }
            task = -1;
        }
        __syncwarp();
    }
    if (lane == 0) {
        A.slots[slot].task = task, A.slots[slot].level = level;
        if (task >= 0) atomicAdd(&A.ctl->active, 1);
        atomicAdd(&A.ctl->work, work);
        atomicAdd(&A.ctl->nodes, nodes);
    }
}

// ---- GNC-TLS rotation (T4-T6): one block of kTmLanes threads -------------------------------------------------------------
struct TmGncArgs {
    const double *p6;   // all N correspondences
    const int *clique;  // M ascending indices
    int M;
    double noise_bound;
    double *tims;       // M x 6: source TIM, target TIM
    double *w, *r;      // weights, residuals
    uint8_t *mask;      // rotation inlier mask
    double *R;          // 9, row-major
    int *out;           // [0] iterations (svdRot calls), [1] inlier count
};
template <int K, class Value>
__device__ __forceinline__ void tm_block_sums(int M, Value v, double (*part)[kTmLanes], double out[K]) {
    const int t = threadIdx.x, m = min(M, kTmLanes);
    double q[K];
    for (int c = 0; c < K; ++c) q[c] = 0.0;
    for (int j = t; j < M; j += kTmLanes) {
        double x[K];
        v(j, x);
        for (int c = 0; c < K; ++c) q[c] += x[c];
    }
    for (int c = 0; c < K; ++c) part[c][t] = q[c];
    __syncthreads();
    for (int s = kTmLanes / 2; s > 0; s >>= 1) {
        if (t < s && t + s < m)
            for (int c = 0; c < K; ++c) part[c][t] += part[c][t + s];
        __syncthreads();
    }
    for (int c = 0; c < K; ++c) out[c] = m > 0 ? part[c][0] : 0.0;
    __syncthreads();
}
__global__ void __launch_bounds__(kTmLanes) k_tm_gnc(TmGncArgs A) {
    __shared__ double part[9][kTmLanes];
    __shared__ double sR[9];
    __shared__ double s_max;
    const int M = A.M;
    for (int k = threadIdx.x; k < M; k += kTmLanes) { // T4: the chain TIMs
        const double *a = A.p6 + 6 * (size_t)A.clique[k], *b = A.p6 + 6 * (size_t)A.clique[k + 1 < M ? k + 1 : 0];
        for (int c = 0; c < 6; ++c) A.tims[6 * (size_t)k + c] = b[c] - a[c];
        A.w[k] = 1.0;
    }
    __syncthreads();
    const double nb_sq = tm_gnc_nb_sq(A.noise_bound);
    double mu = 1.0, prev_cost = INFINITY;
    int it = 0;
    for (int i = 0; i < kTmGncMaxIter; ++i) {
        it = i + 1;
        double h[9];
        tm_block_sums<9>(M, [&](int k, double x[9]) { tm_h_terms(A.tims + 6 * (size_t)k, A.tims + 6 * (size_t)k + 3, A.w[k], x); }, part, h);
        if (threadIdx.x == 0) tm_svd_rot(h, sR);
        __syncthreads();
        double R[9];
        for (int c = 0; c < 9; ++c) R[c] = sR[c];
        double mx = -INFINITY;
        for (int k = threadIdx.x; k < M; k += kTmLanes) {
            const double r = tm_residual(R, A.tims + 6 * (size_t)k, A.tims + 6 * (size_t)k + 3);
            A.r[k] = r;
            mx = r > mx ? r : mx;
        }
        if (i == 0) { // the largest residual (a maximum is the same in any order)
            part[0][threadIdx.x] = mx;
            __syncthreads();
            for (int s = kTmLanes / 2; s > 0; s >>= 1) {
                if (threadIdx.x < s && part[0][threadIdx.x + s] > part[0][threadIdx.x]) part[0][threadIdx.x] = part[0][threadIdx.x + s];
                __syncthreads();
            }
            if (threadIdx.x == 0) s_max = part[0][0];
            __syncthreads();
            mu = tm_gnc_mu0(s_max, nb_sq);
            if (mu <= 0.0) break;
        }
        double cost;
        tm_block_sums<1>(M, [&](int k, double x[1]) { x[0] = A.w[k] * A.r[k]; }, part, &cost);
        for (int k = threadIdx.x; k < M; k += kTmLanes) A.w[k] = tm_gnc_weight(A.r[k], mu, nb_sq);
        __syncthreads();
        const double cost_diff = fabs(cost - prev_cost);
        mu = mu * kTmGncFactor;
        prev_cost = cost;
        if (cost_diff < kTmGncCostThreshold) break;
    }
    int c = 0;
    for (int k = threadIdx.x; k < M; k += kTmLanes) {
        const bool in = A.w[k] >= 0.5;
        A.mask[k] = in ? 1 : 0;
        c += in ? 1 : 0;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) atomicAdd(A.out + 1, c);
    if (threadIdx.x < 9) A.R[threadIdx.x] = sR[threadIdx.x];
    if (threadIdx.x == 0) A.out[0] = it;
}

// ---- TLS translation voting (T7): block a = axis a; bnd holds `padded` boundaries per axis ---------------------------------
__global__ void __launch_bounds__(kTmVoteBlock) k_tm_vote(const double *__restrict__ p6, const int *__restrict__ clique, int M,
                                                          const double *__restrict__ R, double range, double *x3, TmBound *bnd,
                                                          int padded, double *t_out) {
    const int a = blockIdx.x;
    double *x = x3 + (size_t)a * M;
    TmBound *h = bnd + (size_t)a * padded;
    double Ra[3] = {R[3 * a], R[3 * a + 1], R[3 * a + 2]};
    for (int i = threadIdx.x; i < M; i += kTmVoteBlock) {
        const double *p = p6 + 6 * (size_t)clique[i];
        const double xi = p[3 + a] - ((Ra[0] * p[0] + Ra[1] * p[1]) + Ra[2] * p[2]);
        x[i] = xi;
        h[2 * i] = tm_bound(xi, range, i, false);
        h[2 * i + 1] = tm_bound(xi, range, i, true);
    }
    for (int i = 2 * M + threadIdx.x; i < padded; i += kTmVoteBlock) h[i] = TmBound{INFINITY, INT_MAX}; // after every boundary
    __syncthreads();
    for (int k = 2; k <= padded; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < padded; i += kTmVoteBlock) {
                const int l = i ^ j;
                if (l > i) {
                    const TmBound p = h[i], q = h[l];
                    const bool up = (i & k) == 0;
                    if (up ? tm_vote_less(q, p) : tm_vote_less(p, q)) h[i] = q, h[l] = p;
                }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0) t_out[a] = tm_vote_sweep(h, 2 * M, x, range);
}

} // namespace mulls
