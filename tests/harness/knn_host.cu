// TEST INFRASTRUCTURE. Instantiates the templated k-nearest search of mulls_b200/csrc/search_core.cuh (knn_search,
// KnnList<kCap>) on the CPU over the grid search_host.cu builds (same keys, hash and entry layout as k_hash_build; the
// file is included, not copied), with every list capacity the device instantiates: 10 (k_search_shoot) and 16 / 32 / 64
// (k_sor_dist). Built by tests/test_sor.py with nvcc (host code only; no CUDA call is made). The product never executes
// this instantiation.
#include "search_host.cu"

namespace {

template <int kCap>
void knn_all(const HostGrid &G, const float *q, uint32_t m, int k, int start_level, int *out_idx, float *out_d2, int *out_n) {
    for (uint32_t i = 0; i < m; ++i) {
        KnnList<kCap> kl;
        knn_search(G.g, q[3 * i], q[3 * i + 1], q[3 * i + 2], start_level, k, kl);
        out_n[i] = kl.n;
        for (int t = 0; t < k; ++t) {
            int oi = -1;
            float d = INFINITY;
            if (t < kl.n) {
                std::memcpy(&oi, &G.g.nrm[kl.j[t]].w, 4);
                d = kl.d2[t];
            }
            out_idx[(size_t)i * k + t] = oi;
            out_d2[(size_t)i * k + t] = d;
        }
    }
}

} // namespace

extern "C" {

// q: m x 3 floats. Results [m][k] as ORIGINAL target indices (-1 / +inf past the n[i] found), ascending under the total
// order (FLANN float distance, original index). cap: the list instance (10, 16, 32, 64), k <= cap. -1: no such instance.
int kh_knn(void *h, const float *q, uint32_t m, int cap, int k, int start_level, int *out_idx, float *out_d2, int *out_n) {
    const HostGrid &G = *(const HostGrid *)h;
    if (k < 1 || k > cap) return -1;
    switch (cap) {
    case 10: knn_all<10>(G, q, m, k, start_level, out_idx, out_d2, out_n); return 0;
    case 16: knn_all<16>(G, q, m, k, start_level, out_idx, out_d2, out_n); return 0;
    case 32: knn_all<32>(G, q, m, k, start_level, out_idx, out_d2, out_n); return 0;
    case 64: knn_all<64>(G, q, m, k, start_level, out_idx, out_d2, out_n); return 0;
    default: return -1;
    }
}

} // extern "C"
