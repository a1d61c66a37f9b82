// Device check of the ingest's Morton sort: runs the library's own ingest kernels (mulls_b200/csrc/kernels_ingest.cuh)
// in launch_ingest's order, from the bounding boxes to the cell counts, on clouds given by the caller, and returns the
// sorted keys, the SoA slices' input indices and the pair state. tests/test_gpu_ingest_sort.py compares the order with
// a stable sort of the Morton codes in numpy.
#include <cuda_runtime.h>
#include <cstring>
#include <vector>

#include "../../mulls_b200/csrc/kernels_ingest.cuh"

using namespace mulls;

extern "C" {

// rows[n_in * 12]: the clouds as 48-byte rows, in (pair, segment) order; in_n[12 * n_pairs]: their sizes.
// tbound[6 * n_pairs]: each pair's target bound (the intersection filter is on). Out: keys[n_in] (sorted),
// tgt_idx / src_idx[n_in]: normal .w of the target and source slices (the point's index in its input cloud),
// seg_start / seg_count[12 * n_pairs], h0_origin[4 * n_pairs] = h0 and the grid origin, ibb[6 * n_pairs] = the
// intersection box, hash_entries[6 * n_pairs]. Returns 0, or 1 + the CUDA error.
int is_run(const float *rows, const uint32_t *in_n, int n_pairs, const double *tbound, uint64_t *keys, int32_t *tgt_idx,
           int32_t *src_idx, uint32_t *seg_start, uint32_t *seg_count, float *h0_origin, double *ibb,
           uint32_t *hash_entries) {
    std::vector<PairConst> hpc(n_pairs);
    std::vector<ChunkDesc> chunks, tiles;
    size_t n_in = 0, n_tgt = 0, n_src = 0;
    for (int p = 0; p < n_pairs; ++p) {
        PairConst &pc = hpc[p];
        std::memset(&pc, 0, sizeof(pc));
        pc.max_iter = 1;
        pc.apply_filter = 1;
        pc.thre_unit = 1.5f;
        for (int i = 0; i < 16; ++i) pc.init[i] = (i % 5 == 0) ? 1.0 : 0.0;
        for (int i = 0; i < 6; ++i) pc.tbound[i] = tbound[6 * p + i];
        for (int s = 0; s < kNumSegs; ++s) {
            const uint32_t n = in_n[kNumSegs * p + s];
            pc.in_off[s] = (uint32_t)n_in;
            pc.in_n[s] = n;
            pc.in_fmt[s] = 0;
            for (uint32_t f = 0; f < n; f += kIngestBlock) chunks.push_back(ChunkDesc{(uint32_t)p, (uint32_t)s, f});
            for (uint32_t f = 0; f < n; f += kSortTile) tiles.push_back(ChunkDesc{(uint32_t)p, (uint32_t)s, f});
            if (s < kNumClasses) pc.tgt_base[s] = (uint32_t)n_tgt, n_tgt += n;
            else pc.src_base[s - kNumClasses] = (uint32_t)n_src, n_src += n;
            n_in += n;
        }
    }
    DeviceArrays A;
    std::memset(&A, 0, sizeof(A));
    cudaError_t e = cudaSuccess;
    auto ok = [&](cudaError_t r) { return (e = (e == cudaSuccess ? r : e)) == cudaSuccess; };
    float4 *d_in = nullptr, *d_src_pos = nullptr, *d_src_nrm = nullptr;
    int *d_running = nullptr;
    const size_t nin1 = n_in ? n_in : 1;
    ok(cudaMalloc(&d_in, 3 * nin1 * sizeof(float4)));
    ok(cudaMalloc(&A.keys_a, nin1 * sizeof(uint64_t)));
    ok(cudaMalloc(&A.keys_b, nin1 * sizeof(uint64_t)));
    ok(cudaMalloc(&A.tgt_pos, (n_tgt + 1) * sizeof(float4)));
    ok(cudaMalloc(&A.tgt_nrm, (n_tgt + 1) * sizeof(float4)));
    ok(cudaMalloc(&d_src_pos, (n_src + 1) * sizeof(float4)));
    ok(cudaMalloc(&d_src_nrm, (n_src + 1) * sizeof(float4)));
    ok(cudaMalloc(&A.pc, n_pairs * sizeof(PairConst)));
    ok(cudaMalloc(&A.ps, n_pairs * sizeof(PairState)));
    ok(cudaMalloc(&A.in_chunks, (chunks.size() + 1) * sizeof(ChunkDesc)));
    ok(cudaMalloc(&A.sort_tiles, (tiles.size() + 1) * sizeof(ChunkDesc)));
    ok(cudaMalloc(&A.digit_hist, (size_t)n_pairs * kNumSegs * kSortPasses * kSortBins * sizeof(uint32_t)));
    ok(cudaMalloc(&A.sort_status, (tiles.size() + 1) * kSortBins * sizeof(uint64_t)));
    ok(cudaMalloc(&A.sort_ctr, kSortPasses * sizeof(uint32_t)));
    ok(cudaMalloc(&d_running, 2 * sizeof(int)));
    A.in_aos = d_in;
    A.src_pos[0] = d_src_pos;
    A.src_nrm[0] = d_src_nrm;
    A.running = d_running;
    A.h_running = d_running + 1;
    for (int p = 0; p < n_pairs; ++p)
        for (int s = 0; s < kNumSegs; ++s) hpc[p].in_ptr[s] = d_in + 3 * (size_t)hpc[p].in_off[s];
    std::vector<PairState> hps(n_pairs); // as k_state_init leaves it
    std::memset(hps.data(), 0, hps.size() * sizeof(PairState));
    for (PairState &ps : hps)
        for (int d = 0; d < 3; ++d) {
            ps.bb_src[d] = ps.bb_tgt[d] = 0x7fffffff;
            ps.bb_src[3 + d] = ps.bb_tgt[3 + d] = (int)0x80000000;
        }
    const unsigned n_inc = (unsigned)chunks.size(), n_tiles = (unsigned)tiles.size();
    uint32_t epoch = 0;
    if (ok(cudaMemcpy(d_in, rows, n_in * 48, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(A.pc, hpc.data(), n_pairs * sizeof(PairConst), cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(A.in_chunks, chunks.data(), chunks.size() * sizeof(ChunkDesc), cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(A.sort_tiles, tiles.data(), tiles.size() * sizeof(ChunkDesc), cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(A.ps, hps.data(), n_pairs * sizeof(PairState), cudaMemcpyHostToDevice)) &&
        ok(cudaMemset(A.sort_status, 0, (tiles.size() + 1) * kSortBins * sizeof(uint64_t))) &&
        ok(cudaMemset(A.digit_hist, 0, (size_t)n_pairs * kNumSegs * kSortPasses * kSortBins * sizeof(uint32_t))) &&
        ok(cudaMemset(A.sort_ctr, 0, kSortPasses * sizeof(uint32_t)))) {
        if (n_inc) k_ingest_bbox<false><<<n_inc, kIngestBlock>>>(A);
        k_pair_setup<<<1, 128>>>(A, n_pairs);
        if (n_tiles) {
            k_make_keys<false><<<n_tiles, kIngestBlock>>>(A);
            k_digit_scan<<<n_pairs * kNumSegs, kSortBins>>>(A);
            for (int pass = 0; pass < kSortPasses - 1; ++pass) enqueue_sort_pass(A, 0, pass, n_tiles, n_pairs, false, epoch);
        }
        k_seg_offsets<<<1, 256>>>(A, n_pairs);
        if (n_tiles) {
            enqueue_sort_pass(A, 0, kSortPasses - 1, n_tiles, n_pairs, false, epoch);
            k_cell_count<<<(unsigned)((n_in + 255) / 256), 256>>>(A, A.keys_a, (uint32_t)n_in);
        }
        ok(cudaGetLastError());
        ok(cudaDeviceSynchronize());
        ok(cudaMemcpy(keys, A.keys_a, n_in * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        std::vector<float4> nrm(std::max(n_tgt, n_src) + 1);
        ok(cudaMemcpy(nrm.data(), A.tgt_nrm, n_tgt * sizeof(float4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_tgt; ++i) std::memcpy(&tgt_idx[i], &nrm[i].w, 4);
        ok(cudaMemcpy(nrm.data(), d_src_nrm, n_src * sizeof(float4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_src; ++i) std::memcpy(&src_idx[i], &nrm[i].w, 4);
        ok(cudaMemcpy(hps.data(), A.ps, n_pairs * sizeof(PairState), cudaMemcpyDeviceToHost));
        for (int p = 0; p < n_pairs; ++p) {
            for (int s = 0; s < kNumSegs; ++s) {
                seg_start[kNumSegs * p + s] = hps[p].seg_start[s];
                seg_count[kNumSegs * p + s] = hps[p].seg_count[s];
            }
            h0_origin[4 * p] = hps[p].h0;
            for (int d = 0; d < 3; ++d) h0_origin[4 * p + 1 + d] = hps[p].origin[d];
            for (int d = 0; d < 6; ++d) ibb[6 * p + d] = hps[p].ibb[d];
            for (int c = 0; c < kNumClasses; ++c) hash_entries[kNumClasses * p + c] = hps[p].hash_entries[c];
        }
    }
    cudaFree(d_in);
    cudaFree(A.keys_a);
    cudaFree(A.keys_b);
    cudaFree(A.tgt_pos);
    cudaFree(A.tgt_nrm);
    cudaFree(d_src_pos);
    cudaFree(d_src_nrm);
    cudaFree(A.pc);
    cudaFree(A.ps);
    cudaFree(A.in_chunks);
    cudaFree(A.sort_tiles);
    cudaFree(A.digit_hist);
    cudaFree(A.sort_status);
    cudaFree(A.sort_ctr);
    cudaFree(d_running);
    return e == cudaSuccess ? 0 : 1 + (int)e;
}

} // extern "C"
