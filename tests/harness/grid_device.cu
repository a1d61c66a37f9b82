// Device check of the multi-level hashed grid: runs the library's own k_hash_layout, k_hash_clear and k_hash_build
// (mulls_b200/csrc/kernels_ingest.cuh) on sorted 64-bit keys given by the caller, and returns the table they built.
// tests/test_gpu_spatial_index.py compares it with the cells it enumerates from the same keys.
#include <cuda_runtime.h>
#include <cstring>
#include <vector>

#include "../../mulls_b200/csrc/kernels_ingest.cuh"

using namespace mulls;

extern "C" {

// keys[n]: [pair*12+seg | morton36] sorted, filtered-out points (~0) at the tail. Per pair p:
//   seg_start[12p+s], seg_count[12p+s], hash_entries[6p+c] (cells of all levels below n_levels[p]), n_levels[p].
// pool: entries of the hash pool. Out: used[3] = hash_used, hash_base / hash_mask[6 * n_pairs],
// table[pool * 4] (uint32 words of the HashEntry array). Returns 0, or 1 + the CUDA error.
int gd_build(const uint64_t *keys, uint32_t n, int n_pairs, const uint32_t *seg_start, const uint32_t *seg_count,
             const uint32_t *hash_entries, const int *n_levels, uint32_t pool, uint32_t *used, uint32_t *hash_base,
             uint32_t *hash_mask, uint32_t *table) {
    std::vector<PairState> hps(n_pairs);
    std::memset(hps.data(), 0, hps.size() * sizeof(PairState));
    for (int p = 0; p < n_pairs; ++p) {
        hps[p].n_levels = n_levels[p];
        for (int s = 0; s < kNumSegs; ++s) {
            hps[p].seg_start[s] = seg_start[kNumSegs * p + s];
            hps[p].seg_count[s] = seg_count[kNumSegs * p + s];
        }
        for (int c = 0; c < kNumClasses; ++c) hps[p].hash_entries[c] = hash_entries[kNumClasses * p + c];
    }
    DeviceArrays A;
    std::memset(&A, 0, sizeof(A));
    uint64_t *d_keys = nullptr;
    cudaError_t e = cudaSuccess;
    auto ok = [&](cudaError_t r) { return (e = (e == cudaSuccess ? r : e)) == cudaSuccess; };
    ok(cudaMalloc(&d_keys, std::max<size_t>(n, 1) * sizeof(uint64_t)));
    ok(cudaMalloc(&A.ps, n_pairs * sizeof(PairState)));
    ok(cudaMalloc(&A.hash, (size_t)pool * sizeof(HashEntry)));
    ok(cudaMalloc(&A.hash_used, 3 * sizeof(uint32_t)));
    int *d_running = nullptr; // the pairs' running counter and its mirror (an overflowing layout stops every pair)
    ok(cudaMalloc(&d_running, 2 * sizeof(int)));
    A.running = d_running;
    A.h_running = d_running + 1;
    A.hash_pool_entries = pool;
    if (ok(cudaMemcpy(d_keys, keys, n * sizeof(uint64_t), cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(A.ps, hps.data(), n_pairs * sizeof(PairState), cudaMemcpyHostToDevice)) &&
        ok(cudaMemset(A.hash_used, 0, 3 * sizeof(uint32_t))) &&
        ok(cudaMemcpy(d_running, std::vector<int>(2, n_pairs).data(), 2 * sizeof(int), cudaMemcpyHostToDevice)) &&
        // a pool of garbage: k_hash_clear must zero every slot the layout hands out
        ok(cudaMemset(A.hash, 0xa5, (size_t)pool * sizeof(HashEntry)))) {
        k_hash_layout<<<1, 32>>>(A, n_pairs);
        k_hash_clear<<<1184, 256>>>(A);
        if (n) k_hash_build<<<(n + 255) / 256, 256>>>(A, d_keys, n);
        ok(cudaGetLastError());
        ok(cudaDeviceSynchronize());
        ok(cudaMemcpy(used, A.hash_used, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        ok(cudaMemcpy(table, A.hash, (size_t)pool * sizeof(HashEntry), cudaMemcpyDeviceToHost));
        ok(cudaMemcpy(hps.data(), A.ps, n_pairs * sizeof(PairState), cudaMemcpyDeviceToHost));
        for (int p = 0; p < n_pairs; ++p)
            for (int c = 0; c < kNumClasses; ++c) {
                hash_base[kNumClasses * p + c] = hps[p].hash_base[c];
                hash_mask[kNumClasses * p + c] = hps[p].hash_mask[c];
            }
    }
    cudaFree(d_keys);
    cudaFree(A.ps);
    cudaFree(A.hash);
    cudaFree(A.hash_used);
    cudaFree(d_running);
    return e == cudaSuccess ? 0 : 1 + (int)e;
}

} // extern "C"
