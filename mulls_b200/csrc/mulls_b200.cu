// libmulls_b200.so — host side of the C-ABI (include/mulls_b200/abi.h) and kernel launch sequence.
// CUDA runtime only: no torch, no PCL/Eigen. One context = one device, one stream.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <memory>
#include <cmath>
#include <cstdio>
#include <chrono>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <dlfcn.h>
#include <mutex>

#include "device_types.cuh"
#include "host_pack.h"
#include "scan_io.h"
#include "kernels_ingest.cuh"
#include "kernels_iterate.cuh"
#include "kernels_pca.cuh"
#include "kernels_map.cuh"
#include "kernels_classify.cuh"
#include "kernels_ground.cuh"
#include "kernels_sor.cuh"
#include "kernels_rawscan.cuh"
#include "kernels_ncc.cuh"
#include "kernels_ransac.cuh"
#include "kernels_teaser.cuh"
#include "kernels_ndt.cuh"
#include "kernels_gicp.cuh"
#include "kernels_gicp_pcl.cuh"

using namespace mulls;

namespace {
std::string g_create_error;
}

// ---- NCCL without a link-time dependency: the five entry points used, resolved from libnccl.so.2 on first use ----
namespace {
struct ncclUniqueIdBytes {
    char internal[128]; // nccl.h: ncclUniqueId
};
struct NcclApi {
    typedef int (*get_id_t)(void *);
    typedef int (*init_rank_t)(void **, int, ncclUniqueIdBytes, int);
    typedef int (*all_reduce_t)(const void *, void *, size_t, int, int, void *, cudaStream_t);
    typedef int (*destroy_t)(void *);
    typedef const char *(*err_t)(int);
    get_id_t get_id = nullptr;
    init_rank_t init_rank = nullptr;
    all_reduce_t all_reduce = nullptr;
    destroy_t destroy = nullptr;
    err_t err = nullptr;
    bool ok = false;
};
NcclApi &nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        api.get_id = (NcclApi::get_id_t)dlsym(h, "ncclGetUniqueId");
        api.init_rank = (NcclApi::init_rank_t)dlsym(h, "ncclCommInitRank");
        api.all_reduce = (NcclApi::all_reduce_t)dlsym(h, "ncclAllReduce");
        api.destroy = (NcclApi::destroy_t)dlsym(h, "ncclCommDestroy");
        api.err = (NcclApi::err_t)dlsym(h, "ncclGetErrorString");
        api.ok = api.get_id && api.init_rank && api.all_reduce && api.destroy;
    });
    return api;
}
// the all-reduce hook of run_impl over NCCL: user = the communicator (nccl.h: ncclInt32 = 2, ncclFloat64 = 8; ncclSum = 0, ncclMin = 3)
int nccl_allreduce_hook(void *user, void *buf, size_t count, int dtype, int op, void *stream) {
    if (count == 0) return 0;
    return nccl_api().all_reduce(buf, buf, count, dtype == 0 ? 8 : 2, op == 0 ? 0 : 3, user, (cudaStream_t)stream);
}
} // namespace


struct mulls_map;

// a device buffer of the context that only grows (grow_scratch); freed with the context
struct Scratch {
    void *p = nullptr;
    size_t bytes = 0;
    Scratch() = default;
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    ~Scratch() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr, bytes = 0;
    }
};

struct mulls_ctx {
    int device = 0;
    size_t max_pairs = 0, max_src = 0, max_tgt = 0;
    size_t cap_src = 0, cap_tgt = 0, cap_in = 0, cap_it_chunks = 0, cap_in_chunks = 0, cap_sort_tiles = 0;
    cudaStream_t stream = nullptr;
    DeviceArrays A{};
    void *cub_temp = nullptr;
    size_t cub_temp_bytes = 0;
    mulls_icp_result *d_results = nullptr;
    mulls_icp_result *h_results = nullptr; // pinned
    uint32_t *h_flags = nullptr;           // pinned copy of hash_used (3 words), then the target count of ingest_cloud
    int *h_running = nullptr;              // mapped pinned: pairs still iterating
    std::vector<cudaEvent_t> ev_done;      // one per iteration (launch-loop flow control)
    mulls_icp_trace *d_trace = nullptr;
    std::vector<PairConst> h_pc;
    std::vector<ChunkDesc> h_in_chunks, h_it_chunks, h_sort_tiles;
    uint32_t sort_epoch = 0; // sort passes run on the context (k_sort_pass look-back words)
    size_t n_pairs = 0, n_in = 0, n_src_total = 0, n_tgt_total = 0;
    int max_iter_max = 0;
    bool uploaded = false;
    void *nccl_comm = nullptr; // ncclComm_t created by mulls_nccl_init (destroyed with the context)
    bool any_keep_less = false;
    bool grid_valid = false; // pair 0's sorted target slices and grid are those of the last registration (mulls_nn_query)
    // tunables
    // iteration loop as a CUDA graph: WHILE(pairs running) { search, resolve, accumulate, solve } + posterior, finalize,
    // collect — one launch, the loop condition is set on the device (no host polling). Built on first use, rebuilt when
    // the batch shape baked into its kernel nodes changes. 0: the host launch loop (per-kernel events for the bench's
    // roofline).
    int use_graph = 1;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    int graph_key[2] = {-1, -1}; // the batch shape baked into the kernel nodes
    uint64_t graph_body_launches = 0, graph_tail_launches = 0; // kernels recorded per loop iteration and after the loop
    LoopCtl *h_ctl = nullptr;            // pinned staging of the control block
    int num_sms = 132;
    bool any_normal_shooting = false;
    bool any_undistort = false;
    // repack host clouds to the 28 B/point wire format on the host cores before the DMA (host_pack.h):
    // 0 never, 1 always, 2 when a call ships at least kPackMinPoints points (small calls are latency-bound: raw rows)
    int host_pack = 2;
    float4 *h_stage = nullptr; // pinned staging of the packed clouds (allocated on first use)
    size_t h_stage_slots = 0;
    // timing
    cudaEvent_t ev_begin = nullptr, ev_ingest = nullptr, ev_iter = nullptr, ev_end = nullptr, ev_h2d0 = nullptr;
    bool h2d_timed = false;                 // ev_h2d0 was recorded by the upload of the current one-shot call
    float up_ms_pack = 0.f, up_ms_host = 0.f; // host-side times of that upload
    std::vector<cudaEvent_t> ev_search; // 2 per iteration
    mulls_run_stats stats{};
    std::vector<void *> allocs;
    std::string err;
    // one-shot batch calls with host buffers (mulls_icp_run_batch) are double-buffered: the second half of the batch is
    // packed and copied on the twin's stream while the first half is being registered on this one
    mulls_ctx *twin = nullptr;
    // small batches run the whole iteration loop as one cooperative kernel (k_icp_loop) when every chunk and pair has a
    // co-resident block: their count on this device (0: not yet queried, -1: unavailable)
    int loop_kernel_blocks = 0;
    struct Pending {                 // a run that has been enqueued and not yet finished (run_finish)
        uint64_t launches = 0;
        int n_search_ev = 0;
        bool graphed = false, hooked = false, active = false;
        mulls_icp_trace *trace = nullptr; // what run_finish needs to run the call again after growing the hash pool
        mulls_allreduce_fn hook = nullptr;
        void *user = nullptr;
    } pend;
    // device scratch, grown on demand (grow_scratch)
    Scratch pca_buf;             // PCA
    Scratch cls_buf;             // classification (mulls_classify_nground)
    Scratch gf_buf, gf_cell_buf; // ground filter (mulls_fast_ground_filter): per-point part and per-cell part
    Scratch vx_buf, ext_buf;     // voxel filter; clouds handed between the stages of extract_semantic_pts
    Scratch sor_buf;             // statistical outlier filter: mean distances, keep mask, statistics
    Scratch raw_buf;             // raw-scan corrections: the rows of the call, the column it returns, timestamp state
    Scratch ncc_buf;             // NCC keypoint matching: rows, descriptors, row / column minima or select state, sort
    Scratch rc_buf;              // RANSAC coarse registration: correspondences, hypotheses, counts, refinement state
    Scratch nms_buf;             // keypoint NMS: rows, sorted rows, keys, sort scratch, cell hash, kept indices
    Scratch ndt_buf;             // NDT: clouds, leaf keys and sort scratch, leaves, tile sums, fitness distances
    Scratch ndt_kd_buf;          // NDT with KDTREE: the per-point neighbour lists, grown to the longest list seen
    Scratch gicp_buf;            // GICP: clouds, covariances, voxel keys and sort scratch, voxels, tile sums, distances
    Scratch gicp_pcl_buf;        // point-wise GICP: clouds, covariances, correspondences, tile sums, distances
    Scratch tm_buf;              // TEASER++: correspondences, graph, core numbers, GNC and voting state
    Scratch tm_srch_buf;         // TEASER++: the pruned graph and the clique search's stacks
    void *rc_host = nullptr;     // pinned: two chunks of sample triples and their counts
    // the local map whose clouds the target slices of pair 0 currently index (set by mulls_icp_run_to_map, cleared
    // by any other upload): what block1->tree_* are to MapManager::map_based_dynamic_close_removal
    const mulls_map *tree_map = nullptr;
    uint64_t tree_epoch = 0;
};

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) {                                                                      \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                            \
            return MULLS_E_CUDA;                                                                      \
        }                                                                                             \
    } while (0)

// makes s at least `bytes` long (16 at least). The old buffer goes through cudaFree, which waits for the device: no
// kernel still reads it when it is released.
static int grow_scratch(mulls_ctx *ctx, Scratch &s, size_t bytes) {
    bytes = std::max<size_t>(bytes, 16);
    if (bytes <= s.bytes) return MULLS_OK;
    s.release();
    CK(cudaMalloc(&s.p, bytes));
    s.bytes = bytes;
    return MULLS_OK;
}

template <typename T>
static cudaError_t dev_alloc(mulls_ctx *ctx, T **p, size_t n) {
    void *v = nullptr;
    cudaError_t e = cudaMalloc(&v, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) {
        ctx->allocs.push_back(v);
        *p = (T *)v;
    }
    return e;
}

static inline size_t ceil_div(size_t a, size_t b) { return (a + b - 1) / b; }
static inline double wall_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

static void drop_iteration_graph(mulls_ctx *ctx) {
    if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec), ctx->graph_exec = nullptr;
    if (ctx->graph) cudaGraphDestroy(ctx->graph), ctx->graph = nullptr;
}

// The device arrays of one call in one Scratch: take(p, count) reserves `count` elements of *p's type at the next
// 256-byte boundary and remembers p; grow() makes the Scratch hold them all and points each p at its array.
struct ScratchLayout {
    size_t bytes = 0; // the arrays taken so far
    template <typename T> void take(T *&p, size_t count) { add(&p, count * sizeof(T), &bind<T>); }
    void take_bytes(void *&p, size_t n) { add(&p, n, &bind<void>); }
    int grow(mulls_ctx *ctx, Scratch &s) const {
        const int rc = grow_scratch(ctx, s, bytes);
        if (rc == MULLS_OK)
            for (int i = 0; i < n_slots; ++i) slots[i].bind(slots[i].p, (char *)s.p + slots[i].off);
        return rc;
    }

  private:
    template <typename T> static void bind(void *p, char *at) { *(T **)p = (T *)at; }
    struct Slot {
        void *p; // the T * to set
        void (*bind)(void *, char *);
        size_t off;
    };
    static constexpr int kMaxSlots = 40;
    Slot slots[kMaxSlots];
    int n_slots = 0;
    void add(void *p, size_t n, void (*b)(void *, char *)) {
        assert(n_slots < kMaxSlots);
        slots[n_slots++] = Slot{p, b, bytes};
        bytes += ceil_div(std::max<size_t>(n, 1), 256) * 256;
    }
};

extern "C" {

void mulls_icp_default_params(mulls_icp_params *p) {
    std::memset(p, 0, sizeof(*p));
    p->max_iter_num = 20;
    p->dis_thre_unit = 1.5f;
    p->converge_translation = 0.002f;
    p->converge_rotation_d = 0.01f;
    p->dis_thre_min = 0.4f;
    p->dis_thre_update_rate = 1.1f;
    std::strcpy(p->used_feature_type, "111110");
    std::strcpy(p->weight_strategy, "1101");
    p->z_xy_balanced_ratio = 1.0f;
    p->pt2pt_residual_window = 0.1f;
    p->pt2pl_residual_window = 0.1f;
    p->pt2li_residual_window = 0.1f;
    p->apply_intersection_filter = 1;
    p->normal_bearing = 45.0f;
    p->sigma_thre = 0.5f;
    p->min_neccessary_corr_ratio = 0.03f;
    p->max_bearable_rotation_d = 45.0f;
    const double big = 1.7976931348623157e308;
    for (int d = 0; d < 3; ++d) {
        p->target_bound[d] = -big;
        p->target_bound[3 + d] = big;
    }
}

const char *mulls_last_error(const mulls_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

void mulls_destroy(mulls_ctx *ctx) {
    if (!ctx) return;
    if (ctx->twin) mulls_destroy(ctx->twin), ctx->twin = nullptr;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (void *p : ctx->allocs) cudaFree(p);
    if (ctx->cub_temp) cudaFree(ctx->cub_temp);
    if (ctx->rc_host) cudaFreeHost(ctx->rc_host);
    if (ctx->h_results) cudaFreeHost(ctx->h_results);
    if (ctx->h_flags) cudaFreeHost(ctx->h_flags);
    if (ctx->h_running) cudaFreeHost(ctx->h_running);
    if (ctx->nccl_comm && nccl_api().ok) nccl_api().destroy(ctx->nccl_comm);
    if (ctx->h_ctl) cudaFreeHost(ctx->h_ctl);
    drop_iteration_graph(ctx);
    if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
    for (cudaEvent_t e : ctx->ev_done) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->ev_search) cudaEventDestroy(e);
    if (ctx->ev_begin) cudaEventDestroy(ctx->ev_begin);
    if (ctx->ev_ingest) cudaEventDestroy(ctx->ev_ingest);
    if (ctx->ev_iter) cudaEventDestroy(ctx->ev_iter);
    if (ctx->ev_end) cudaEventDestroy(ctx->ev_end);
    if (ctx->ev_h2d0) cudaEventDestroy(ctx->ev_h2d0);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx; // frees the Scratch buffers, with ctx->device current
}

mulls_ctx *mulls_create(int device, size_t max_pairs, size_t max_src_pts, size_t max_tgt_pts) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        g_create_error = std::string("mulls_create: no CUDA device (") + cudaGetErrorString(e) +
                         "); mulls_b200 has no CPU fallback";
        return nullptr;
    }
    if (device < 0 || device >= ndev || max_pairs == 0) {
        g_create_error = "mulls_create: bad device index or max_pairs";
        return nullptr;
    }
    mulls_ctx *ctx = new mulls_ctx();
    ctx->device = device;
    ctx->max_pairs = max_pairs;
    ctx->max_src = max_src_pts;
    ctx->max_tgt = max_tgt_pts;
    auto fail = [&](const char *what, cudaError_t err) -> mulls_ctx * {
        g_create_error = std::string("mulls_create: ") + what + ": " + cudaGetErrorString(err);
        mulls_destroy(ctx);
        return nullptr;
    };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("stream", e);
    const size_t cs = ctx->cap_src = max_pairs * max_src_pts;
    const size_t ct = ctx->cap_tgt = max_pairs * max_tgt_pts;
    const size_t cin = ctx->cap_in = cs + ct;
    if (cin >= (1ull << 31)) {
        g_create_error = "mulls_create: more than 2^31 points per context";
        mulls_destroy(ctx);
        return nullptr;
    }
    // every cloud adds at most one partial chunk
    ctx->cap_it_chunks = ceil_div(cs, kIterBlock) + max_pairs * (kNumClasses + 1);
    ctx->cap_in_chunks = ceil_div(cin, kIngestBlock) + max_pairs * kNumSegs;
    ctx->cap_sort_tiles = ceil_div(cin, kSortTile) + max_pairs * kNumSegs;
    DeviceArrays &A = ctx->A;
    float4 *in = nullptr;
#define ALLOC(ptr, n)                                                   \
    if ((e = dev_alloc(ctx, &(ptr), (n))) != cudaSuccess) return fail(#ptr, e)
    ALLOC(in, 3 * cin);
    A.in_aos = in;
    ALLOC(A.keys_a, cin);
    ALLOC(A.keys_b, cin);
    ALLOC(A.sort_tiles, ctx->cap_sort_tiles);
    ALLOC(A.digit_hist, max_pairs * kNumSegs * kSortPasses * kSortBins);
    ALLOC(A.sort_status, ctx->cap_sort_tiles * kSortBins);
    ALLOC(A.sort_ctr, kSortPasses);
    ALLOC(A.tgt_pos, ct + kScanOverrun); // (walk_scan_leaf's last group reads past a cell)
    ALLOC(A.tgt_nrm, ct);
    for (int b = 0; b < 2; ++b) {
        ALLOC(A.src_pos[b], cs);
        ALLOC(A.src_nrm[b], cs);
        ALLOC(A.src_prevj[b], cs);
        ALLOC(A.src_cert[b], cs);
    }
    ALLOC(A.nn_idx, cs);
    ALLOC(A.nn_d2, cs);
    ALLOC(A.flags, cs);
    ALLOC(A.corr_j, cs);
    ALLOC(A.corr_w, cs);
    ALLOC(A.claim, ct);
    // hash pool: every class table has a power-of-two capacity of 1.25x to 8x its cells (k_hash_layout). On a 64-beam
    // scan pair the cells of all levels are about 0.55 per target point, so 12 entries per point (192 B) leave room for
    // kHashSlack and the rounding. That is a first size, not a bound: a point opens up to one cell per level (12), and
    // sparse clouds come close to it (about 7 cells per point for 20 000 points spread over a 500 m cube). When the
    // target clouds of a call need more, the pool grows to what they need and the call runs again (grow_hash_pool).
    {
        size_t pool = 12 * ct + 64 * max_pairs * kNumClasses;
        if (pool >= (1ull << 32)) pool = (1ull << 32) - 1;
        A.hash_pool_entries = (uint32_t)pool;
        ALLOC(A.hash, pool);
    }
    ALLOC(A.hash_used, 3);
    ALLOC(A.ctl, 1);
    ALLOC(A.blk_kept, ctx->cap_it_chunks);
    ALLOC(A.partials, ctx->cap_it_chunks * kTerms);
    ALLOC(A.post_partials, ctx->cap_it_chunks * 2);
    ALLOC(A.pc, max_pairs);
    ALLOC(A.ps, max_pairs);
    ALLOC(A.in_chunks, ctx->cap_in_chunks);
    ALLOC(A.it_chunks, ctx->cap_it_chunks);
    ALLOC(A.live_chunks, 2 * ctx->cap_it_chunks);
    A.live_stride = (uint32_t)ctx->cap_it_chunks;
    {
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
        ctx->num_sms = sms;
    }
    ALLOC(ctx->d_results, max_pairs + ceil_div(max_pairs * sizeof(uint64_t), sizeof(mulls_icp_result)) + 1);
    ALLOC(ctx->d_trace, max_pairs);
    ALLOC(A.running, 1);
    ALLOC(A.xch_i32, 32);
    ALLOC(A.xch_f64, kNumClasses * kTerms + 8);
#undef ALLOC
    if ((e = cudaHostAlloc((void **)&ctx->h_running, (1 + kIterFlags) * sizeof(int), cudaHostAllocMapped)) != cudaSuccess)
        return fail("mapped flag", e);
    {
        int *dptr = nullptr;
        if ((e = cudaHostGetDevicePointer((void **)&dptr, ctx->h_running, 0)) != cudaSuccess) return fail("mapped flag", e);
        A.h_running = dptr;
        A.h_running_iter = dptr + 1;
    }
    ctx->ev_done.resize(MULLS_MAX_TRACE_ITERS);
    for (auto &ev : ctx->ev_done) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    A.trace = ctx->d_trace; // written only when LoopCtl::trace_on is set for the run
    if ((e = cudaMallocHost((void **)&ctx->h_results, max_pairs * (sizeof(mulls_icp_result) + sizeof(uint64_t)))) != cudaSuccess)
        return fail("pinned results", e);
    if ((e = cudaMallocHost((void **)&ctx->h_flags, 4 * sizeof(uint32_t))) != cudaSuccess) return fail("pinned flags", e);
    if ((e = cudaMallocHost((void **)&ctx->h_ctl, sizeof(LoopCtl))) != cudaSuccess) return fail("pinned control block", e);
    // radix-sort temp storage of the keypoint suppression (launch_nms), whose keys live in keys_a / keys_b
    {
        size_t bytes = 0;
        cub::DeviceRadixSort::SortKeys(nullptr, bytes, A.keys_a, A.keys_b, (int)cin, 0, 64, ctx->stream);
        ctx->cub_temp_bytes = bytes;
        if ((e = cudaMalloc(&ctx->cub_temp, std::max<size_t>(bytes, 16))) != cudaSuccess) return fail("cub temp", e);
    }
    cudaEventCreate(&ctx->ev_begin);
    cudaEventCreate(&ctx->ev_ingest);
    cudaEventCreate(&ctx->ev_iter);
    cudaEventCreate(&ctx->ev_end);
    cudaEventCreate(&ctx->ev_h2d0);
    ctx->ev_search.resize(2 * MULLS_MAX_TRACE_ITERS);
    for (auto &ev : ctx->ev_search) cudaEventCreate(&ev);
    if ((e = cudaMemsetAsync(A.ps, 0, max_pairs * sizeof(PairState), ctx->stream)) != cudaSuccess) return fail("memset", e);
    // look-back words of epoch 0: older than any pass
    if ((e = cudaMemsetAsync(A.sort_status, 0, ctx->cap_sort_tiles * kSortBins * sizeof(uint64_t), ctx->stream)) != cudaSuccess)
        return fail("memset", e);
    if ((e = cudaStreamSynchronize(ctx->stream)) != cudaSuccess) return fail("sync", e);
    return ctx;
}

int mulls_set_tunable(mulls_ctx *ctx, const char *name, int value) {
    if (!ctx || !name) return MULLS_E_ARG;
    if (ctx->twin) {
        const int rc = mulls_set_tunable(ctx->twin, name, value);
        if (rc != MULLS_OK) return rc;
    }
    std::string n(name);
    if (n == "use_graph") ctx->use_graph = value;
    else if (n == "host_pack") ctx->host_pack = value;
    else if (n == "pack_threads") PackPool::get().ensure_workers(value);
    else return MULLS_E_ARG;
    return MULLS_OK;
}

int mulls_pack_rows(const float *aos48, size_t n, int format, float *out) {
    if ((n > 0 && (!aos48 || !out)) || (format != kFmtPacked28 && format != kFmtPacked32) || ((uintptr_t)out % 16) != 0)
        return MULLS_E_ARG;
    pack_rows(aos48, 0, n, format, out, out + 4 * n);
    _mm_sfence();
    return MULLS_OK;
}

// ---- scans in, poses out (csrc/scan_io.h: host code, no device involved) -------------------------------------
static int io_code(int rc) {
    switch (rc) {
    case mulls_io::kOk: return MULLS_OK;
    case mulls_io::kArg: return MULLS_E_ARG;
    case mulls_io::kCapacity: return MULLS_E_CAPACITY;
    case mulls_io::kUnsupported: return MULLS_E_UNSUPPORTED;
    default: return MULLS_E_IO;
    }
}
int mulls_scan_probe(const char *path, size_t *n_points) { return io_code(mulls_io::probe_scan(path, n_points)); }
int mulls_scan_read(const char *path, float *rows48, size_t capacity_points, size_t *n_points, double local_bound[6],
                    int normalize_intensity) {
    return io_code(mulls_io::read_scan(path, rows48, capacity_points, n_points, local_bound, normalize_intensity));
}
int mulls_pose_write(const char *path, const double pose[16], int overwrite) {
    return io_code(mulls_io::append_pose(path, pose, overwrite));
}
void *mulls_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void mulls_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

int mulls_get_stats(const mulls_ctx *ctx, mulls_run_stats *out) {
    if (!ctx || !out) return MULLS_E_ARG;
    *out = ctx->stats;
    return MULLS_OK;
}

// Eigen::Quaterniond(T.block<3,3>(0,0)) of a row-major 4x4, its translation and the constants of Eigen's
// slerp(Identity -> q): d = q.w, linear when |d| >= 1 - eps, neg when d < 0, theta = acos|d| (cfilter.hpp:472-475)
static SlerpConst slerp_const_of(const double *T) {
    SlerpConst sc;
    double *q = sc.q; // x y z w
    double t = T[0] + T[5] + T[10];
    if (t > 0.0) {
        t = std::sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (T[9] - T[6]) * t;
        q[1] = (T[2] - T[8]) * t;
        q[2] = (T[4] - T[1]) * t;
    } else {
        int i = 0;
        if (T[5] > T[0]) i = 1;
        if (T[10] > T[5 * i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(T[5 * i] - T[5 * j] - T[5 * k] + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (T[4 * k + j] - T[4 * j + k]) * t;
        q[j] = (T[4 * j + i] + T[4 * i + j]) * t;
        q[k] = (T[4 * k + i] + T[4 * i + k]) * t;
    }
    sc.t[0] = T[3], sc.t[1] = T[7], sc.t[2] = T[11];
    const double one = 1.0 - 2.220446049250313e-16;
    const double d = q[3], absD = std::fabs(d);
    sc.linear = (absD >= one) ? 1 : 0;
    sc.neg = (d < 0) ? 1 : 0;
    sc.theta = sc.linear ? 0.0 : std::acos(absD);
    sc.sin_theta = sc.linear ? 1.0 : std::sin(sc.theta);
    return sc;
}

// Inverse of the initial guess (Eigen Matrix4d::inverse: cofactors / determinant) and the slerp constants of its
// rotation (cregistration.hpp:1248, cfilter.hpp:499-502).
static void setup_undistortion(const double *m, PairConst &pc) {
    double inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    double T[16];
    for (int i = 0; i < 16; ++i) T[i] = inv[i] * (1.0 / det);
    const SlerpConst sc = slerp_const_of(T);
    for (int i = 0; i < 4; ++i) pc.ud_q[i] = sc.q[i];
    for (int i = 0; i < 3; ++i) pc.ud_t[i] = sc.t[i];
    pc.ud_linear = sc.linear;
    pc.ud_neg = sc.neg;
    pc.ud_theta = sc.theta;
    pc.ud_sin_theta = sc.sin_theta;
}

// ------------------------------------------------------------------------------------------------
static int build_pair_const(mulls_ctx *ctx, const mulls_icp_params &P, const double *init, PairConst &pc) {
    if (P.max_iter_num > MULLS_MAX_TRACE_ITERS) {
        ctx->err = "max_iter_num > 64";
        return MULLS_E_ARG;
    }
    std::memset(&pc, 0, sizeof(pc));
    pc.max_iter = P.max_iter_num;
    const size_t nu = strnlen(P.used_feature_type, 8), nw = strnlen(P.weight_strategy, 8);
    for (int c = 0; c < kNumClasses; ++c) pc.used[c] = (c < (int)nu && P.used_feature_type[c] == '1') ? 1 : 0;
    pc.w_balance = (nw > 0 && P.weight_strategy[0] == '1');
    pc.w_residual = (nw > 1 && P.weight_strategy[1] == '1');
    pc.w_dist = (nw > 2 && P.weight_strategy[2] == '1');
    pc.w_intensity = (nw > 3 && P.weight_strategy[3] == '1');
    pc.z_xy_ratio = P.z_xy_balanced_ratio;
    pc.win_pt2pt = P.pt2pt_residual_window;
    pc.win_pt2pl = P.pt2pl_residual_window;
    pc.win_pt2li = P.pt2li_residual_window;
    pc.thre_unit = P.dis_thre_unit;
    pc.thre_min = P.dis_thre_min;
    pc.thre_rate = P.dis_thre_update_rate;
    pc.conv_t = P.converge_translation;
    // the float/double mix of cregistration.hpp:1162-1164
    pc.conv_r = (float)(P.converge_rotation_d / 180.0 * M_PI);
    pc.max_t = (float)(2.0 * P.dis_thre_unit);
    pc.max_r = (float)(P.max_bearable_rotation_d / 180.0 * M_PI);
    pc.min_ratio = P.min_neccessary_corr_ratio;
    // the intersection filter is skipped in the undistortion variant (cregistration.hpp:1186)
    pc.undistort = P.apply_motion_undistortion_while_registration ? 1 : 0;
    pc.apply_filter = (P.apply_intersection_filter && !pc.undistort) ? 1 : 0;
    if (pc.undistort) setup_undistortion(init, pc);
    // :1191 keep_less_source_pts is skipped in the undistortion variant
    pc.keep_less = (P.keep_less_source_points && !pc.undistort) ? 1 : 0;
    pc.random_seed = P.random_seed;
    pc.normal_shooting = P.normal_shooting_on ? 1 : 0;
    pc.cos_thre = std::cos(P.normal_bearing / 180.0 * M_PI);
    pc.sigma_thre = (double)P.sigma_thre;
    for (int i = 0; i < 16; ++i) pc.init[i] = init[i];
    for (int i = 0; i < 6; ++i) pc.tbound[i] = P.target_bound[i];
    return MULLS_OK;
}

// Copies the clouds into HBM on the context's stream: repacked on the host cores first when the call ships enough
// points (host_pack), as caller rows otherwise. resident = true (mulls_batch_upload): the copies are waited for, since
// the clouds must survive the caller's buffers. resident = false (one-shot calls): the copies stay in flight and the
// registration that follows waits for them. tgt_on_device: the target views already point into HBM and are read there.
static int upload_impl(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt, const mulls_cloud_view *src,
                       const mulls_icp_params *params, const double *init_guess, const uint32_t *src_index_base,
                       const uint32_t *src_global_n, bool resident = true, bool tgt_on_device = false) {
    if (!ctx || !tgt || !src || !params || !init_guess || n_pairs == 0) return MULLS_E_ARG;
    ctx->tree_map = nullptr;
    ctx->grid_valid = false;
    if (n_pairs > ctx->max_pairs) {
        ctx->err = "more pairs than the context was created for";
        return MULLS_E_CAPACITY;
    }
    CK(cudaSetDevice(ctx->device));
    ctx->uploaded = false;
    const double t_up0 = wall_ms();
    ctx->h2d_timed = false;
    ctx->up_ms_pack = 0.f;
    ctx->h_pc.assign(n_pairs, PairConst());
    ctx->h_in_chunks.clear();
    ctx->h_it_chunks.clear();
    ctx->h_sort_tiles.clear();
    size_t in_off = 0, s_off = 0, t_off = 0;
    int max_iter_max = 0;
    bool any_keep_less = false, any_shoot = false, any_undistort = false;
    for (size_t p = 0; p < n_pairs; ++p) {
        PairConst &pc = ctx->h_pc[p];
        int rc = build_pair_const(ctx, params[p], init_guess + 16 * p, pc);
        if (rc != MULLS_OK) return rc;
        max_iter_max = std::max(max_iter_max, pc.max_iter);
        any_keep_less = any_keep_less || pc.keep_less;
        any_shoot = any_shoot || pc.normal_shooting;
        any_undistort = any_undistort || pc.undistort;
        size_t ns = 0, nt = 0;
        for (int c = 0; c < kNumClasses; ++c) {
            nt += tgt[p * kNumClasses + c].n;
            ns += src[p * kNumClasses + c].n;
        }
        if (ns > ctx->max_src || nt > ctx->max_tgt) {
            ctx->err = "pair exceeds max_src_pts / max_tgt_pts of the context";
            return MULLS_E_CAPACITY;
        }
        for (int s = 0; s < kNumSegs; ++s) {
            const mulls_cloud_view &v = (s < kNumClasses) ? tgt[p * kNumClasses + s] : src[p * kNumClasses + (s - kNumClasses)];
            if (v.n > 0 && !v.aos48) return MULLS_E_ARG;
            pc.in_off[s] = (uint32_t)in_off;
            pc.in_n[s] = (uint32_t)v.n;
            for (size_t f = 0; f < v.n; f += kIngestBlock)
                ctx->h_in_chunks.push_back(ChunkDesc{(uint32_t)p, (uint32_t)s, (uint32_t)f});
            for (size_t f = 0; f < v.n; f += kSortTile)
                ctx->h_sort_tiles.push_back(ChunkDesc{(uint32_t)p, (uint32_t)s, (uint32_t)f});
            in_off += v.n;
        }
        pc.chunk_begin = (uint32_t)ctx->h_it_chunks.size();
        for (int c = 0; c < kNumClasses; ++c) {
            pc.tgt_base[c] = (uint32_t)t_off;
            pc.src_base[c] = (uint32_t)s_off;
            t_off += tgt[p * kNumClasses + c].n;
            const size_t n = src[p * kNumClasses + c].n;
            s_off += n;
            pc.class_chunk_begin[c] = (uint32_t)ctx->h_it_chunks.size();
            // class 0 always owns at least one chunk so that the per-pair "last block" logic (status
            // codes, iteration counter) also runs for pairs without any source point
            const size_t n_eff = (c == 0 && n == 0) ? 1 : n;
            for (size_t f = 0; f < n_eff; f += kIterBlock) ctx->h_it_chunks.push_back(ChunkDesc{(uint32_t)p, (uint32_t)c, (uint32_t)f});
            pc.src_index_base[c] = src_index_base ? src_index_base[c] : 0;
            pc.src_global_n[c] = src_global_n ? src_global_n[c] : (uint32_t)n;
        }
        pc.class_chunk_begin[kNumClasses] = (uint32_t)ctx->h_it_chunks.size();
        pc.chunk_end = (uint32_t)ctx->h_it_chunks.size();
        pc.sharded = src_index_base ? 1 : 0;
    }
    if (ctx->h_in_chunks.size() > ctx->cap_in_chunks || ctx->h_it_chunks.size() > ctx->cap_it_chunks ||
        ctx->h_sort_tiles.size() > ctx->cap_sort_tiles) {
        ctx->err = "internal: chunk table capacity";
        return MULLS_E_CAPACITY;
    }
    // the clouds: repacked on the host cores and copied pair by pair (host_pack), or copied as they are; a device-resident
    // target (the local map) is read in place
    size_t host_points = 0;
    for (size_t p = 0; p < n_pairs; ++p)
        for (int s = 0; s < kNumSegs; ++s)
            if (!(tgt_on_device && s < kNumClasses)) host_points += ctx->h_pc[p].in_n[s];
    const size_t kPackMinPoints = 1u << 18;
    bool tables_sent = false;
    const bool pack = ctx->host_pack == 1 || (ctx->host_pack == 2 && host_points >= kPackMinPoints);
    if (pack) {
        if (!ctx->h_stage) {
            const size_t slots = 2 * ctx->cap_in + 4 * kNumSegs * ctx->max_pairs;
            CK(cudaHostAlloc((void **)&ctx->h_stage, slots * sizeof(float4), cudaHostAllocDefault));
            ctx->h_stage_slots = slots;
        }
        CK(cudaStreamSynchronize(ctx->stream)); // the staging may still be read by a copy of a call that failed half-way
        PackPool &pool = PackPool::get();
        pool.ensure_workers(0);
        std::unique_ptr<std::atomic<int>[]> pending(new std::atomic<int>[n_pairs]);
        std::vector<size_t> slot_begin(n_pairs + 1, 0);
        std::vector<PackJob> jobs;
        const size_t kJobPts = 16384; // multiple of 4 (pack_rows)
        size_t slot = 0;
        for (size_t p = 0; p < n_pairs; ++p) {
            PairConst &pc = ctx->h_pc[p];
            const int fmt = pc.undistort ? kFmtPacked32 : kFmtPacked28;
            slot_begin[p] = slot;
            int n_jobs = 0;
            for (int s = 0; s < kNumSegs; ++s) {
                const mulls_cloud_view &v = (s < kNumClasses) ? tgt[p * kNumClasses + s] : src[p * kNumClasses + (s - kNumClasses)];
                pc.in_ptr[s] = ctx->A.in_aos + slot;
                pc.in_fmt[s] = (uint32_t)fmt;
                if (tgt_on_device && s < kNumClasses) { // the view already points into HBM (device-resident local map)
                    pc.in_ptr[s] = (const float4 *)v.aos48;
                    pc.in_fmt[s] = kFmtRows48;
                    continue;
                }
                if (v.n == 0) continue;
                float *pos = reinterpret_cast<float *>(ctx->h_stage + slot);
                float *nrm = reinterpret_cast<float *>(ctx->h_stage + slot + v.n);
                for (size_t f = 0; f < v.n; f += kJobPts) {
                    jobs.push_back(PackJob{v.aos48, pos, nrm, f, std::min(kJobPts, v.n - f), fmt, &pending[p]});
                    ++n_jobs;
                }
                slot += packed_slots(v.n, fmt);
            }
            pending[p].store(n_jobs, std::memory_order_relaxed);
        }
        slot_begin[n_pairs] = slot;
        if (slot > ctx->h_stage_slots || slot > 3 * ctx->cap_in) {
            ctx->err = "internal: packed staging capacity";
            return MULLS_E_CAPACITY;
        }
        pool.submit(jobs); // FIFO: pair 0 is packed first, and its DMA runs while the next pairs are being packed
        // the (pageable, hence synchronously staged) tables go first: queued behind the clouds they would wait for them
        cudaError_t ce = cudaMemcpyAsync(ctx->A.pc, ctx->h_pc.data(), n_pairs * sizeof(PairConst), cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess && !ctx->h_in_chunks.empty())
            ce = cudaMemcpyAsync(ctx->A.in_chunks, ctx->h_in_chunks.data(), ctx->h_in_chunks.size() * sizeof(ChunkDesc),
                                 cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess && !ctx->h_it_chunks.empty())
            ce = cudaMemcpyAsync(ctx->A.it_chunks, ctx->h_it_chunks.data(), ctx->h_it_chunks.size() * sizeof(ChunkDesc),
                                 cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess && !ctx->h_sort_tiles.empty())
            ce = cudaMemcpyAsync(ctx->A.sort_tiles, ctx->h_sort_tiles.data(), ctx->h_sort_tiles.size() * sizeof(ChunkDesc),
                                 cudaMemcpyHostToDevice, ctx->stream);
        tables_sent = true; // (every job is waited for even after an error: the jobs point at `pending`)
        if (ce == cudaSuccess && cudaEventRecord(ctx->ev_h2d0, ctx->stream) == cudaSuccess) ctx->h2d_timed = true;
        const double t_pack0 = wall_ms();
        for (size_t p = 0; p < n_pairs; ++p) {
            pool.help_until_done(pending[p]);
            if (p + 1 == n_pairs) ctx->up_ms_pack = (float)(wall_ms() - t_pack0);
            const size_t b = slot_begin[p], e = slot_begin[p + 1];
            if (e > b && ce == cudaSuccess)
                ce = cudaMemcpyAsync((void *)(ctx->A.in_aos + b), ctx->h_stage + b, (e - b) * sizeof(float4), cudaMemcpyHostToDevice,
                                     ctx->stream);
        }
        CK(ce);
    } else {
    if (cudaEventRecord(ctx->ev_h2d0, ctx->stream) == cudaSuccess) ctx->h2d_timed = true;
    for (size_t p = 0; p < n_pairs; ++p) {
        PairConst &pc = ctx->h_pc[p];
        for (int s = 0; s < kNumSegs; ++s) {
            const mulls_cloud_view &v = (s < kNumClasses) ? tgt[p * kNumClasses + s] : src[p * kNumClasses + (s - kNumClasses)];
            pc.in_ptr[s] = ctx->A.in_aos + 3 * (size_t)pc.in_off[s];
            pc.in_fmt[s] = kFmtRows48;
            if (v.n == 0) continue;
            if (tgt_on_device && s < kNumClasses) { // the view already points into HBM (device-resident local map)
                pc.in_ptr[s] = (const float4 *)v.aos48;
                continue;
            }
            CK(cudaMemcpyAsync((void *)(ctx->A.in_aos + 3 * (size_t)pc.in_off[s]), v.aos48, v.n * 48, cudaMemcpyHostToDevice,
                               ctx->stream));
        }
    }
    }
    if (!tables_sent) {
        CK(cudaMemcpyAsync(ctx->A.pc, ctx->h_pc.data(), n_pairs * sizeof(PairConst), cudaMemcpyHostToDevice, ctx->stream));
        if (!ctx->h_in_chunks.empty())
            CK(cudaMemcpyAsync(ctx->A.in_chunks, ctx->h_in_chunks.data(), ctx->h_in_chunks.size() * sizeof(ChunkDesc),
                               cudaMemcpyHostToDevice, ctx->stream));
        if (!ctx->h_it_chunks.empty())
            CK(cudaMemcpyAsync(ctx->A.it_chunks, ctx->h_it_chunks.data(), ctx->h_it_chunks.size() * sizeof(ChunkDesc),
                               cudaMemcpyHostToDevice, ctx->stream));
        if (!ctx->h_sort_tiles.empty())
            CK(cudaMemcpyAsync(ctx->A.sort_tiles, ctx->h_sort_tiles.data(), ctx->h_sort_tiles.size() * sizeof(ChunkDesc),
                               cudaMemcpyHostToDevice, ctx->stream));
    }
    // The tables above live in pageable vectors: cudaMemcpyAsync has already staged them when it returns. The clouds,
    // however, may be the caller's pinned buffers (truly asynchronous copies): a resident upload returns to the caller
    // before anything else runs, so it waits here; a one-shot call goes straight on to run_impl, which synchronises
    // before it returns — the kernels are queued while the clouds are still crossing PCIe.
    if (resident) CK(cudaStreamSynchronize(ctx->stream));
    ctx->n_pairs = n_pairs;
    ctx->n_in = in_off;
    ctx->n_src_total = s_off;
    ctx->n_tgt_total = t_off;
    ctx->max_iter_max = max_iter_max;
    ctx->any_keep_less = any_keep_less;
    ctx->any_normal_shooting = any_shoot;
    ctx->any_undistort = any_undistort;
    ctx->uploaded = true;
    ctx->up_ms_host = (float)(wall_ms() - t_up0);
    return MULLS_OK;
}

// One cross-rank all-reduce of a sharded run: the caller's callback enqueues it on the context's stream.
static int exchange(mulls_ctx *ctx, mulls_allreduce_fn hook, void *user, void *buf, size_t count, int dtype, int op) {
    if (hook(user, buf, count, dtype, op, (void *)ctx->stream) == 0) return MULLS_OK;
    ctx->err = "all-reduce callback failed";
    return MULLS_E_COMM;
}

// Ingest phase on the resident inputs: state reset, initial guess, intersection filter, Morton sort,
// hashed multi-level grid. Shared by the registration path and mulls_pca_features. finite_only (mulls_sor_filter, no
// source, no motion undistortion): points with a non-finite coordinate stay out of the bbox and of the grid.
static int launch_ingest(mulls_ctx *ctx, DeviceArrays &A, bool trace, uint64_t &launches, mulls_allreduce_fn hook = nullptr,
                         void *user = nullptr, bool finite_only = false) {
    cudaStream_t st = ctx->stream;
    const int np = (int)ctx->n_pairs;
    const uint32_t n_in = (uint32_t)ctx->n_in;
    if (trace) CK(cudaMemsetAsync(ctx->d_trace, 0, np * sizeof(mulls_icp_trace), st));
    CK(cudaMemsetAsync(A.claim, 0x7f, std::max<size_t>(ctx->n_tgt_total, 1) * sizeof(unsigned), st));
    k_state_init<<<(unsigned)ceil_div(np, 128), 128, 0, st>>>(A, np);
    ++launches;
    const unsigned n_inc = (unsigned)ctx->h_in_chunks.size();
    if (n_inc) {
        if (ctx->any_undistort) k_ingest_bbox<true><<<n_inc, kIngestBlock, 0, st>>>(A);
        else if (finite_only) k_ingest_bbox<false, true><<<n_inc, kIngestBlock, 0, st>>>(A);
        else k_ingest_bbox<false><<<n_inc, kIngestBlock, 0, st>>>(A);
        ++launches;
    }
    if (hook) { // sharded source: the intersection filter needs the bbox over all shards
        k_shard_pack_setup<<<1, 1, 0, st>>>(A, 0);
        if (const int rc = exchange(ctx, hook, user, A.xch_i32, 6, 1, 1); rc != MULLS_OK) return rc;
        k_shard_pack_setup<<<1, 1, 0, st>>>(A, 1);
        launches += 2;
    }
    k_pair_setup<<<(unsigned)ceil_div(np, 128), 128, 0, st>>>(A, np);
    ++launches;
    const unsigned n_tiles = (unsigned)ctx->h_sort_tiles.size();
    if (n_inc) {
        CK(cudaMemsetAsync(A.digit_hist, 0, (size_t)np * kNumSegs * kSortPasses * kSortBins * sizeof(uint32_t), st));
        CK(cudaMemsetAsync(A.sort_ctr, 0, kSortPasses * sizeof(uint32_t), st));
        if (ctx->any_undistort) k_make_keys<true><<<n_tiles, kIngestBlock, 0, st>>>(A);
        else if (finite_only) k_make_keys<false, true><<<n_tiles, kIngestBlock, 0, st>>>(A);
        else k_make_keys<false><<<n_tiles, kIngestBlock, 0, st>>>(A);
        ++launches;
        if (ctx->any_keep_less) { // random down-sampling of :2866-2892: radix select of the k-th sampling key
            const unsigned pb = (unsigned)ceil_div(np, 64);
            k_keepless_plan<<<pb, 64, 0, st>>>(A, np);
            for (int pass = 0; pass < 8; ++pass) {
                k_keepless_hist<<<n_inc, kIngestBlock, 0, st>>>(A, pass);
                k_keepless_step<<<pb, 64, 0, st>>>(A, np, pass);
            }
            k_keepless_mark<<<n_inc, kIngestBlock, 0, st>>>(A);
            launches += 18;
        }
        // the Morton order inside every segment: digit offsets, then sort passes 0-2 (pass 3 needs the segment starts)
        k_digit_scan<<<(unsigned)(np * kNumSegs), kSortBins, 0, st>>>(A);
        for (int pass = 0; pass < kSortPasses - 1; ++pass)
            enqueue_sort_pass(A, st, pass, n_tiles, np, ctx->any_undistort, ctx->sort_epoch);
        launches += kSortPasses;
    }
    k_seg_offsets<<<1, 256, 0, st>>>(A, np);
    ++launches;
    if (hook) { // global class sizes (:1195-1201 counts, K_filter_distant_point test)
        k_shard_pack_setup<<<1, 1, 0, st>>>(A, 2);
        if (const int rc = exchange(ctx, hook, user, A.xch_i32, kNumClasses, 1, 0); rc != MULLS_OK) return rc;
        k_shard_pack_setup<<<1, 1, 0, st>>>(A, 3);
        launches += 2;
    }
    if (n_in) {
        const unsigned nb = (unsigned)ceil_div(n_in, 256);
        enqueue_sort_pass(A, st, kSortPasses - 1, n_tiles, np, ctx->any_undistort, ctx->sort_epoch);
        k_cell_count<<<nb, 256, 0, st>>>(A, A.keys_a, n_in);
        k_hash_layout<<<1, 32, 0, st>>>(A, np);
        k_hash_clear<<<1184, 256, 0, st>>>(A);
        k_hash_build<<<nb, 256, 0, st>>>(A, A.keys_a, n_in);
        launches += 5;
    } else {
        k_hash_layout<<<1, 32, 0, st>>>(A, np);
        ++launches;
    }
    return MULLS_OK;
}

// The iteration kernels run a fixed number of resident blocks that fetch live chunks (for_each_live_chunk): grids are
// sized by the SM count and the blocks an SM holds, never by the batch.
// ... and, for small batches, by the chunks there are (rounded up to a power of two: the grids are part of the graph)
static unsigned chunk_bucket(const mulls_ctx *ctx) {
    unsigned b = 1;
    while (b < (unsigned)ctx->h_it_chunks.size()) b <<= 1;
    return b;
}
static unsigned resident_grid(const mulls_ctx *ctx, int blocks_per_sm, unsigned chunks_per_block = 1) {
    return std::min((unsigned)(ctx->num_sms * blocks_per_sm), (chunk_bucket(ctx) + chunks_per_block - 1) / chunks_per_block);
}
constexpr int kShootBlocksPerSm = 8;
constexpr int kPollPause = 64; // _mm_pause() count between two cudaEventQuery calls of the launch loop's flow control

// One ICP iteration: k_search [, k_search_shoot], k_resolve, k_accumulate, k_solve, and a sharded run's three exchanges.
// it < 0 records the graph's loop body: all three k_search modes (each checks the device-side iteration counter) and
// k_solve over every pair slot, setting the loop condition `handle`. it >= 0 is iteration `it` of the host launch loop:
// its one search mode, exact grids, the search timed by ev_search[2it], ev_search[2it+1]. Counts its kernels in `launches`.
static int enqueue_iteration(mulls_ctx *ctx, int it, mulls_allreduce_fn hook, void *user, unsigned long long handle,
                             uint64_t &launches) {
    cudaStream_t st = ctx->stream;
    const DeviceArrays &A = ctx->A;
    const bool recording = it < 0;
    const int buf = recording ? -1 : it & 1;
    if (hook) // other ranks' claims of the previous iteration must not survive in this rank's table
        CK(cudaMemsetAsync(A.claim, 0x7f, std::max<size_t>(ctx->n_tgt_total, 1) * sizeof(unsigned), st));
    if (!recording) CK(cudaEventRecord(ctx->ev_search[2 * it], st));
    const unsigned search_grid = resident_grid(ctx, kSearchBlocksPerSm);
    const int mode = recording ? -1 : search_mode_of(it);
    if (mode < 0 || mode == 0) k_search<0><<<search_grid, kIterBlock, 0, st>>>(A, buf, it);
    if (mode < 0 || mode == 1) k_search<1><<<search_grid, kIterBlock, 0, st>>>(A, buf, it);
    if (mode < 0 || mode == 2) k_search<2><<<search_grid, kIterBlock, 0, st>>>(A, buf, it);
    launches += recording ? 3 : 1;
    if (ctx->any_normal_shooting) {
        k_search_shoot<<<resident_grid(ctx, kShootBlocksPerSm), kIterBlock, 0, st>>>(A, buf);
        ++launches;
    }
    if (!recording) CK(cudaEventRecord(ctx->ev_search[2 * it + 1], st));
    if (hook) { // exchange 1: the duplicate-check claims of all shards (min of source indices)
        if (const int rc = exchange(ctx, hook, user, A.claim, ctx->n_tgt_total, 1, 1); rc != MULLS_OK) return rc;
    }
    k_resolve<<<resident_grid(ctx, kResolveBlocksPerSm), kIterBlock, 0, st>>>(A, buf);
    if (hook) { // exchange 2: correspondence counts (w_ground, -2 test) and surviving source counts
        k_shard_counts<<<1, kIterBlock, 0, st>>>(A, 0);
        if (const int rc = exchange(ctx, hook, user, A.xch_i32, 2 * kNumClasses, 1, 0); rc != MULLS_OK) return rc;
        k_shard_counts<<<1, kIterBlock, 0, st>>>(A, 1);
        launches += 2;
    }
    k_accumulate<<<resident_grid(ctx, kAccumulateBlocksPerSm, kIterBlock / 32), kIterBlock, 0, st>>>(A, buf); // a chunk per warp
    k_solve<<<recording ? (unsigned)std::max<size_t>(ctx->max_pairs, 1) : (unsigned)ctx->n_pairs, kSolveThreads, 0, st>>>(A, buf, handle);
    launches += 3;
    if (hook) { // exchange 3: per-class normal-equation sums; then every rank solves the same system
        if (const int rc = exchange(ctx, hook, user, A.xch_f64, kNumClasses * kTerms, 0, 0); rc != MULLS_OK) return rc;
        k_shard_solve<<<1, 32, 0, st>>>(A, buf, it);
        ++launches;
    }
    return MULLS_OK;
}

// What follows the loop: k_posterior, k_finalize (sharded: k_shard_post, exchange, k_shard_post), k_collect. recording
// (the iteration graph): grids for the context's capacity. Otherwise exact grids, and ev_iter before k_collect.
static int enqueue_tail(mulls_ctx *ctx, bool recording, mulls_allreduce_fn hook, void *user, uint64_t &launches) {
    cudaStream_t st = ctx->stream;
    const DeviceArrays &A = ctx->A;
    const unsigned pairs = recording ? (unsigned)std::max<size_t>(ctx->max_pairs, 1) : (unsigned)ctx->n_pairs;
    const int np = recording ? -1 : (int)ctx->n_pairs;
    k_posterior<<<recording ? std::min((unsigned)std::max<size_t>(ctx->cap_it_chunks, 1), chunk_bucket(ctx))
                            : (unsigned)ctx->h_it_chunks.size(), kIterBlock, 0, st>>>(A);
    if (hook) {
        k_shard_post<<<1, 32, 0, st>>>(A, 0);
        if (const int rc = exchange(ctx, hook, user, A.xch_f64, 2, 0, 0); rc != MULLS_OK) return rc;
        k_shard_post<<<1, 32, 0, st>>>(A, 1);
    } else {
        k_finalize<<<(unsigned)ceil_div(pairs, 64), 64, 0, st>>>(A, np);
    }
    if (!recording) CK(cudaEventRecord(ctx->ev_iter, st));
    k_collect<<<(unsigned)ceil_div(pairs, 128), 128, 0, st>>>(A, np, ctx->d_results);
    launches += hook ? 4 : 3;
    return MULLS_OK;
}

// The iteration loop as a CUDA graph (CUDA 12.4+ conditional nodes): WHILE(handle) { enqueue_iteration } followed by
// enqueue_tail. Kernel nodes are recorded once per context with grids sized for its capacity; what a run needs to know
// (chunk / pair counts, trace switch, loop counter) is read from LoopCtl in device memory. k_solve's last block sets the
// loop condition: no host polling, one launch. A failed recording ends its capture and leaves no graph behind.
static int build_iteration_graph(mulls_ctx *ctx) {
    const int key[2] = {(int)chunk_bucket(ctx), ctx->any_normal_shooting ? 1 : 0};
    if (ctx->graph_exec && std::memcmp(key, ctx->graph_key, sizeof(key)) == 0) return MULLS_OK;
    drop_iteration_graph(ctx);
    cudaStream_t st = ctx->stream;
    const int rc = [&]() -> int {
        CK(cudaGraphCreate(&ctx->graph, 0));
        cudaGraphConditionalHandle handle;
        CK(cudaGraphConditionalHandleCreate(&handle, ctx->graph, 1, cudaGraphCondAssignDefault));
        cudaGraphNodeParams wp = {cudaGraphNodeTypeConditional};
        wp.conditional.handle = handle;
        wp.conditional.type = cudaGraphCondTypeWhile;
        wp.conditional.size = 1;
        cudaGraphNode_t while_node;
        CK(cudaGraphAddNode(&while_node, ctx->graph, nullptr, 0, &wp));
        uint64_t body = 0, tail = 0;
        CK(cudaStreamBeginCaptureToGraph(st, wp.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
        int rc = enqueue_iteration(ctx, -1, nullptr, nullptr, (unsigned long long)handle, body);
        CK(cudaStreamEndCapture(st, nullptr)); // (before rc is tested: the stream leaves capture mode in any case)
        if (rc != MULLS_OK) return rc;
        CK(cudaStreamBeginCaptureToGraph(st, ctx->graph, &while_node, nullptr, 1, cudaStreamCaptureModeThreadLocal));
        rc = enqueue_tail(ctx, true, nullptr, nullptr, tail);
        CK(cudaStreamEndCapture(st, nullptr));
        if (rc != MULLS_OK) return rc;
        CK(cudaGraphInstantiate(&ctx->graph_exec, ctx->graph, 0));
        ctx->graph_body_launches = body, ctx->graph_tail_launches = tail;
        return MULLS_OK;
    }();
    if (rc != MULLS_OK) return drop_iteration_graph(ctx), rc;
    std::memcpy(ctx->graph_key, key, sizeof(key));
    return MULLS_OK;
}

// After a run whose grid did not fit the hash pool (h_flags copied back, stream synchronised): grows the pool to the
// entries k_hash_layout found the target clouds need, so that the same inputs fit when they run again. The iteration
// graph has the old pool's address baked into its kernel nodes: it is dropped, and recorded anew by its next use.
static int grow_hash_pool(mulls_ctx *ctx) {
    const uint32_t need = ctx->h_flags[2];
    DeviceArrays &A = ctx->A;
    if (need <= A.hash_pool_entries || need == 0xffffffffu) {
        ctx->err = "hash pool exhausted (the target clouds need " + std::to_string(need) + " grid entries)";
        return MULLS_E_CAPACITY;
    }
    HashEntry *fresh = nullptr;
    if (cudaMalloc(&fresh, (size_t)need * sizeof(HashEntry)) != cudaSuccess) {
        cudaGetLastError();
        ctx->err = "hash pool exhausted, and no device memory to grow it to " + std::to_string(need) + " entries";
        return MULLS_E_CAPACITY;
    }
    std::replace(ctx->allocs.begin(), ctx->allocs.end(), (void *)A.hash, (void *)fresh);
    CK(cudaFree(A.hash));
    A.hash = fresh;
    A.hash_pool_entries = need;
    drop_iteration_graph(ctx);
    return MULLS_OK;
}

// run_impl and run_finish return through here: an error exit may leave async copies from / into the caller's buffers
// (clouds, trace, results) in flight, so nothing is handed back before the stream has drained.
static int drain_on_error(mulls_ctx *ctx, int rc) {
    if (rc != MULLS_OK && ctx && ctx->stream) cudaStreamSynchronize(ctx->stream);
    return rc;
}

static int run_finish(mulls_ctx *ctx, mulls_icp_result *out);
// Launch the whole path on the resident inputs. If `hook` is given (sharded mode) it is called between
// the phases that need a cross-rank exchange.
// finish_now = false: everything is enqueued on the context's stream and the call returns; run_finish waits for it
static int run_impl(mulls_ctx *ctx, mulls_icp_result *out, mulls_icp_trace *trace, mulls_allreduce_fn hook, void *user,
                    bool finish_now = true) {
    return drain_on_error(ctx, [&]() -> int {
        if (!ctx || !ctx->uploaded) return MULLS_E_ARG;
        ctx->pend.active = false;
        CK(cudaSetDevice(ctx->device));
        cudaStream_t st = ctx->stream;
        DeviceArrays A = ctx->A;
        const int np = (int)ctx->n_pairs;
        uint64_t launches = 0;
        CK(cudaEventRecord(ctx->ev_begin, st));
        if (const int rc = launch_ingest(ctx, A, trace != nullptr, launches, hook, user); rc != MULLS_OK) return rc;
        const unsigned n_itc = (unsigned)ctx->h_it_chunks.size(); // (>= 1: upload_impl gives class 0 of every pair a chunk)
        {
            LoopCtl &c = *ctx->h_ctl; // (the previous run has been synchronised: the staging copy is free)
            c = LoopCtl();
            c.n_it_chunks = (int)n_itc, c.n_pairs = np, c.trace_on = trace ? 1 : 0, c.max_iter = ctx->max_iter_max;
            CK(cudaMemcpyAsync(A.ctl, ctx->h_ctl, sizeof(LoopCtl), cudaMemcpyHostToDevice, st));
            // the chunks that own source points after the intersection filter: work list of iteration 0
            k_live_init<<<(unsigned)ceil_div(n_itc, 256), 256, 0, st>>>(A);
            ++launches;
        }
        // small batches: one cooperative kernel runs the whole loop (every chunk and every pair must find a co-resident block)
        bool looped = false;
        if (!hook && ctx->use_graph && !ctx->any_normal_shooting) {
            if (ctx->loop_kernel_blocks == 0) {
                int per_sm = 0, coop = 0;
                cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device);
                if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_icp_loop, kIterBlock, 0) == cudaSuccess && per_sm > 0)
                    ctx->loop_kernel_blocks = per_sm * ctx->num_sms;
                else
                    ctx->loop_kernel_blocks = -1, cudaGetLastError();
            }
            looped = ctx->loop_kernel_blocks > 0 && n_itc <= (unsigned)ctx->loop_kernel_blocks && np <= ctx->loop_kernel_blocks;
        }
        const bool graphed = !hook && ctx->use_graph && !looped;
        if (const int rc = graphed ? build_iteration_graph(ctx) : MULLS_OK; rc != MULLS_OK) return rc;
        CK(cudaEventRecord(ctx->ev_ingest, st));
        int n_search_ev = 0;
        if (graphed) {
            CK(cudaGraphLaunch(ctx->graph_exec, st));
            CK(cudaMemcpyAsync(ctx->h_ctl, A.ctl, sizeof(LoopCtl), cudaMemcpyDeviceToHost, st)); // iterations executed
            CK(cudaEventRecord(ctx->ev_iter, st));
        } else {
            if (looped) {
                DeviceArrays Aarg = A;
                void *args[] = {&Aarg};
                const unsigned grid = std::max(1u, std::min((unsigned)ctx->loop_kernel_blocks, std::max(n_itc, (unsigned)np)));
                CK(cudaLaunchCooperativeKernel((const void *)k_icp_loop, dim3(grid), dim3(kIterBlock), args, 0, st));
                ++launches;
            } else {
                for (int it = 0; it < ctx->max_iter_max; ++it) {
                    // flow control: stay at most two iterations ahead of the device and stop launching as soon
                    // as every pair has converged or failed (the device mirrors its counter into mapped memory)
                    if (it >= 2) {
                        // (poll with pauses: several contexts spinning inside the driver slow each other's launches down)
                        while (cudaEventQuery(ctx->ev_done[it - 2]) == cudaErrorNotReady)
                            for (int k = 0; k < kPollPause; ++k) _mm_pause();
                        // Sharded runs must take this decision identically on every rank (the ranks issue matching collectives):
                        // they read the count the device recorded at the END of iteration it-2 — written once, before
                        // ev_done[it-2] — never the live flag, whose value at this instant depends on each rank's timing.
                        if (hook ? ((volatile int *)ctx->h_running)[1 + (it - 2)] <= 0 : *(volatile int *)ctx->h_running <= 0) break;
                    }
                    if (const int rc = enqueue_iteration(ctx, it, hook, user, 0ull, launches); rc != MULLS_OK) return rc;
                    CK(cudaEventRecord(ctx->ev_done[it], st));
                    n_search_ev = it + 1;
                }
            }
            if (const int rc = enqueue_tail(ctx, false, hook, user, launches); rc != MULLS_OK) return rc;
        }
        CK(cudaMemcpyAsync(ctx->h_results, ctx->d_results, np * (sizeof(mulls_icp_result) + sizeof(uint64_t)), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(ctx->h_flags, A.hash_used, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        if (trace) CK(cudaMemcpyAsync(trace, ctx->d_trace, np * sizeof(mulls_icp_trace), cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(ctx->ev_end, st));
        ctx->pend.launches = launches, ctx->pend.n_search_ev = n_search_ev, ctx->pend.graphed = graphed, ctx->pend.hooked = hook != nullptr;
        ctx->pend.trace = trace, ctx->pend.hook = hook, ctx->pend.user = user;
        ctx->pend.active = true;
        if (!finish_now) return MULLS_OK;
        return run_finish(ctx, out);
    }());
}

static int run_finish(mulls_ctx *ctx, mulls_icp_result *out) {
    return drain_on_error(ctx, [&]() -> int {
        if (!ctx || !ctx->pend.active) return MULLS_E_ARG;
        ctx->pend.active = false;
        cudaStream_t st = ctx->stream;
        const int np = (int)ctx->n_pairs;
        uint64_t launches = ctx->pend.launches;
        const int n_search_ev = ctx->pend.n_search_ev;
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        if (ctx->pend.graphed) launches += (uint64_t)ctx->h_ctl->it * ctx->graph_body_launches + ctx->graph_tail_launches;
        if (ctx->h_flags[1]) {
            // the grid did not fit (k_hash_layout stopped every pair): grow the pool and run the call again on the inputs
            // still in HBM. The grown pool holds the layout's last attempt by construction, so this happens at most once. A
            // sharded run grows on every rank alike: the target clouds, and so their grids, are the same on all of them.
            const int rc = grow_hash_pool(ctx);
            if (rc != MULLS_OK) return rc;
            return run_impl(ctx, out, ctx->pend.trace, ctx->pend.hook, ctx->pend.user);
        }
        if (out) std::memcpy(out, ctx->h_results, np * sizeof(mulls_icp_result));
        // statistics
        mulls_run_stats &S = ctx->stats;
        S = mulls_run_stats();
        S.kernel_launches = launches;
        cudaEventElapsedTime(&S.ms_ingest, ctx->ev_begin, ctx->ev_ingest);
        cudaEventElapsedTime(&S.ms_iterate, ctx->ev_ingest, ctx->ev_iter);
        cudaEventElapsedTime(&S.ms_total, ctx->ev_begin, ctx->ev_end);
        if (ctx->h2d_timed) cudaEventElapsedTime(&S.ms_h2d, ctx->ev_h2d0, ctx->ev_begin);
        S.ms_host_pack = ctx->up_ms_pack, S.ms_host_upload = ctx->up_ms_host;
        ctx->h2d_timed = false;
        float ms = 0.f;
        for (int it = 0; it < n_search_ev; ++it) {
            float t = 0.f;
            cudaEventElapsedTime(&t, ctx->ev_search[2 * it], ctx->ev_search[2 * it + 1]);
            S.ms_search_iter[it] = t;
            ms += t;
        }
        S.ms_search = ms;
        S.search_launches = (uint64_t)n_search_ev;
        for (int p = 0; p < np; ++p) S.iterations += (uint64_t)ctx->h_results[p].iters;
        // algorithmic bytes are accumulated on the device per executed iteration (k_collect puts them behind the results)
        {
            const uint64_t *ab = reinterpret_cast<const uint64_t *>(ctx->h_results + np);
            for (int p = 0; p < np; ++p) S.algorithmic_bytes += ab[p];
        }
        ctx->grid_valid = !ctx->pend.hooked;
        return MULLS_OK;
    }());
}

int mulls_batch_upload(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt, const mulls_cloud_view *src,
                       const mulls_icp_params *params, const double *init_guess) {
    return upload_impl(ctx, n_pairs, tgt, src, params, init_guess, nullptr, nullptr);
}

int mulls_batch_run_resident(mulls_ctx *ctx, mulls_icp_result *out, mulls_icp_trace *trace) {
    return run_impl(ctx, out, trace, nullptr, nullptr);
}

// One-shot batch on ONE context (host buffers in, results out). With >= 2 pairs and the iteration graph the batch is
// double-buffered over the context and its twin (own stream and buffers, created on first use): the second half is
// packed and copied while the first half is being registered; both halves are collected at the end.
static int one_shot_batch(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt, const mulls_cloud_view *src,
                          const mulls_icp_params *params, const double *init_guess, mulls_icp_result *out, mulls_icp_trace *trace) {
    const double t0 = wall_ms();
    const bool split = ctx->use_graph && n_pairs >= 2 && n_pairs <= ctx->max_pairs;
    if (split && !ctx->twin) {
        mulls_ctx *t = mulls_create(ctx->device, (ctx->max_pairs + 1) / 2, ctx->max_src, ctx->max_tgt);
        if (t) { // (no memory for it: the call simply runs on one context)
            t->use_graph = ctx->use_graph, t->host_pack = ctx->host_pack;
            ctx->twin = t;
        }
    }
    if (!split || !ctx->twin) {
        int rc = upload_impl(ctx, n_pairs, tgt, src, params, init_guess, nullptr, nullptr, /*resident=*/false);
        if (rc != MULLS_OK) return rc;
        rc = run_impl(ctx, out, trace, nullptr, nullptr);
        ctx->uploaded = false; // nothing stays resident after a one-shot call
        ctx->stats.ms_host_call = (float)(wall_ms() - t0);
        return rc;
    }
    mulls_ctx *a = ctx, *b = ctx->twin;
    const size_t n0 = (n_pairs + 1) / 2, n1 = n_pairs - n0;
    int rc = upload_impl(a, n0, tgt, src, params, init_guess, nullptr, nullptr, /*resident=*/false);
    if (rc == MULLS_OK) rc = run_impl(a, nullptr, trace, nullptr, nullptr, /*finish_now=*/false);
    int rcb = MULLS_OK;
    if (rc == MULLS_OK) {
        rcb = upload_impl(b, n1, tgt + n0 * kNumClasses, src + n0 * kNumClasses, params + n0, init_guess + 16 * n0, nullptr, nullptr,
                          /*resident=*/false);
        if (rcb == MULLS_OK) rcb = run_impl(b, nullptr, trace ? trace + n0 : nullptr, nullptr, nullptr, /*finish_now=*/false);
    }
    // whatever happened, nothing is handed back while one of the two streams still works on the caller's buffers
    if (rc == MULLS_OK) rc = run_finish(a, out);
    else cudaStreamSynchronize(a->stream);
    if (rc == MULLS_OK && rcb == MULLS_OK) rcb = run_finish(b, out ? out + n0 : nullptr);
    else if (b->stream) cudaStreamSynchronize(b->stream), b->pend.active = false;
    a->uploaded = b->uploaded = false;
    if (rc == MULLS_OK && rcb != MULLS_OK) {
        ctx->err = b->err;
        rc = rcb;
    }
    if (rc == MULLS_OK) { // the call's statistics: both halves (device times overlap: the longer one is reported)
        mulls_run_stats &S = a->stats;
        const mulls_run_stats &T = b->stats;
        S.kernel_launches += T.kernel_launches, S.algorithmic_bytes += T.algorithmic_bytes, S.iterations += T.iterations;
        S.ms_ingest = std::max(S.ms_ingest, T.ms_ingest), S.ms_iterate = std::max(S.ms_iterate, T.ms_iterate);
        S.ms_total = std::max(S.ms_total, T.ms_total);
        S.ms_h2d += T.ms_h2d, S.ms_host_pack += T.ms_host_pack, S.ms_host_upload += T.ms_host_upload;
    }
    ctx->stats.ms_host_call = (float)(wall_ms() - t0);
    return rc;
}

int mulls_icp_run_batch(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tgt, const mulls_cloud_view *src,
                        const mulls_icp_params *params, const double *init_guess, mulls_icp_result *out,
                        mulls_icp_trace *trace) {
    if (!ctx || !tgt || !src || !params || !init_guess || n_pairs == 0) return MULLS_E_ARG;
    return one_shot_batch(ctx, n_pairs, tgt, src, params, init_guess, out, trace);
}

int mulls_icp_run(mulls_ctx *ctx, const mulls_cloud_view tgt[MULLS_NUM_CLASSES], const mulls_cloud_view src[MULLS_NUM_CLASSES],
                  const mulls_icp_params *params, const double init_guess[16], mulls_icp_result *out,
                  mulls_icp_trace *trace) {
    return mulls_icp_run_batch(ctx, 1, tgt, src, params, init_guess, out, trace);
}

} // extern "C"

extern "C" {

int mulls_nccl_unique_id(char id[MULLS_NCCL_ID_BYTES]) {
    if (!id) return MULLS_E_ARG;
    NcclApi &api = nccl_api();
    if (!api.ok) return MULLS_E_COMM;
    ncclUniqueIdBytes u;
    if (api.get_id(&u) != 0) return MULLS_E_COMM;
    std::memcpy(id, u.internal, MULLS_NCCL_ID_BYTES);
    return MULLS_OK;
}

int mulls_nccl_init(mulls_ctx *ctx, int rank, int world, const char id[MULLS_NCCL_ID_BYTES]) {
    if (!ctx || !id || world < 1 || rank < 0 || rank >= world) return MULLS_E_ARG;
    NcclApi &api = nccl_api();
    if (!api.ok) {
        ctx->err = "libnccl.so.2 not found (or too old)";
        return MULLS_E_COMM;
    }
    CK(cudaSetDevice(ctx->device));
    if (ctx->nccl_comm) api.destroy(ctx->nccl_comm), ctx->nccl_comm = nullptr;
    ncclUniqueIdBytes u;
    std::memcpy(u.internal, id, MULLS_NCCL_ID_BYTES);
    const int rc = api.init_rank(&ctx->nccl_comm, world, u, rank);
    if (rc != 0) {
        ctx->err = std::string("ncclCommInitRank: ") + (api.err ? api.err(rc) : "failed");
        ctx->nccl_comm = nullptr;
        return MULLS_E_COMM;
    }
    return MULLS_OK;
}

int mulls_icp_run_sharded_nccl(mulls_ctx *ctx, void *comm, const mulls_cloud_view tgt[MULLS_NUM_CLASSES],
                               const mulls_cloud_view src_shard[MULLS_NUM_CLASSES], const uint32_t src_index_base[MULLS_NUM_CLASSES],
                               const uint32_t src_global_n[MULLS_NUM_CLASSES], const mulls_icp_params *params,
                               const double init_guess[16], mulls_icp_result *out, mulls_icp_trace *trace) {
    if (!ctx) return MULLS_E_ARG;
    if (!comm) comm = ctx->nccl_comm;
    if (!comm || !nccl_api().ok) {
        ctx->err = "no NCCL communicator: call mulls_nccl_init first (or pass an ncclComm_t)";
        return MULLS_E_COMM;
    }
    return mulls_icp_run_sharded(ctx, tgt, src_shard, src_index_base, src_global_n, params, init_guess, nccl_allreduce_hook, comm, out,
                                 trace);
}

int mulls_nn_query(mulls_ctx *ctx, int cls, const float *xyz, size_t n, int32_t *idx, float *d2) {
    if (!ctx || cls < 0 || cls >= kNumClasses || (n > 0 && (!xyz || !idx || !d2))) return MULLS_E_ARG;
    if (!ctx->grid_valid) {
        ctx->err = "mulls_nn_query: no registration has run on this context since its last upload";
        return MULLS_E_ARG;
    }
    if (n == 0) return MULLS_OK;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    float *d_q = nullptr;
    int *d_i = nullptr;
    float *d_d = nullptr;
    CK(cudaMallocAsync((void **)&d_q, 3 * n * sizeof(float), st));
    CK(cudaMallocAsync((void **)&d_i, n * sizeof(int), st));
    CK(cudaMallocAsync((void **)&d_d, n * sizeof(float), st));
    CK(cudaMemcpyAsync(d_q, xyz, 3 * n * sizeof(float), cudaMemcpyHostToDevice, st));
    k_nn_query<<<(unsigned)ceil_div(n, kIterBlock), kIterBlock, 0, st>>>(ctx->A, cls, d_q, (uint32_t)n, d_i, d_d);
    CK(cudaMemcpyAsync(idx, d_i, n * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(d2, d_d, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    cudaFreeAsync(d_q, st);
    cudaFreeAsync(d_i, st);
    cudaFreeAsync(d_d, st);
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    return MULLS_OK;
}

int mulls_icp_run_sharded(mulls_ctx *ctx, const mulls_cloud_view tgt[MULLS_NUM_CLASSES],
                          const mulls_cloud_view src_shard[MULLS_NUM_CLASSES],
                          const uint32_t src_index_base[MULLS_NUM_CLASSES], const uint32_t src_global_n[MULLS_NUM_CLASSES],
                          const mulls_icp_params *params, const double init_guess[16], mulls_allreduce_fn allreduce,
                          void *user, mulls_icp_result *out, mulls_icp_trace *trace) {
    if (!ctx || !allreduce || !params) return MULLS_E_ARG;
    if (params->keep_less_source_points && !params->apply_motion_undistortion_while_registration) {
        // the down-sampling quota and its sampling keys are defined over the WHOLE source cloud (:2866-2892); a
        // shard-local plan would keep ~world times too many points and a different subset than the unsharded run
        ctx->err = "keep_less_source_points is not supported for a source-sharded registration";
        return MULLS_E_UNSUPPORTED;
    }
    int rc = upload_impl(ctx, 1, tgt, src_shard, params, init_guess, src_index_base, src_global_n, /*resident=*/false);
    if (rc != MULLS_OK) return rc;
    rc = run_impl(ctx, out, trace, allreduce, user);
    ctx->uploaded = false;
    return rc;
}

} // extern "C"

// ================================================================================================
// Stateless front-end calls: PCA, statistical outlier removal, raw-scan corrections, NCC matching, RANSAC, and the
// chain of extract_semantic_pts (voxel filter, ground filter, non-ground classification)
// ================================================================================================
// The call frame of every public front-end entry point. The body enqueues the call on ctx->stream and counts the kernels
// of this library it launches. An error exit may leave a copy from or into a caller's buffer in flight: nothing is
// handed back before the stream drains. A call that succeeds leaves its launches and device span in ctx->stats.
template <typename Body>
static int front_call(mulls_ctx *ctx, Body &&body) {
    if (!ctx) return MULLS_E_ARG;
    ctx->stats = mulls_run_stats();
    uint64_t launches = 0;
    const int rc = [&]() -> int {
        CK(cudaSetDevice(ctx->device));
        CK(cudaEventRecord(ctx->ev_begin, ctx->stream));
        if (const int rc = body(launches); rc != MULLS_OK) return rc;
        CK(cudaEventRecord(ctx->ev_end, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaGetLastError());
        return MULLS_OK;
    }();
    if (rc != MULLS_OK) {
        cudaStreamSynchronize(ctx->stream);
        return rc;
    }
    ctx->stats.kernel_launches = launches;
    cudaEventElapsedTime(&ctx->stats.ms_total, ctx->ev_begin, ctx->ev_end);
    return MULLS_OK;
}

// a front-end call takes no more points than the targets of a registration
static int check_capacity(mulls_ctx *ctx, size_t n, const char *fn) {
    if (n <= ctx->max_tgt) return MULLS_OK;
    ctx->err = std::string(fn) + ": " + std::to_string(n) + " points exceed max_tgt_pts of the context";
    return MULLS_E_CAPACITY;
}

// Uploads one cloud (host rows, or rows already in HBM) as the only target class of a one-pair batch and builds its
// grid with the filter-less ingest of a registration; the resident batch is gone afterwards. radius > 0 becomes
// dis_thre_unit (the grid's top level then covers 2.5 x radius), 0 keeps the default. full_pyramid sets
// normal_shooting_on, which asks k_pair_setup for the full level pyramid, whose top block spans the whole grid.
// finite_only keeps points with a non-finite coordinate out of the bbox and the grid. The grid must fit the hash pool
// before a kernel reads it: else the pool grows and the grid is built again from the cloud already in HBM (it fits by
// construction). `A` receives the device arrays, n_tgt the count of target points in the grid.
// ingest_clouds: the same for n host clouds at once, cloud i as the target of pair i (n_tgt is pair 0's count).
static int ingest_clouds(mulls_ctx *ctx, size_t n, const mulls_cloud_view *clouds, bool on_device, float radius,
                         bool full_pyramid, bool finite_only, DeviceArrays &A, int &n_tgt, uint64_t &launches) {
    mulls_icp_params P;
    mulls_icp_default_params(&P);
    std::strcpy(P.used_feature_type, "100000");
    P.apply_intersection_filter = 0;
    if (radius > 0.f) P.dis_thre_unit = radius;
    if (full_pyramid) P.normal_shooting_on = 1;
    P.max_iter_num = 0;
    std::vector<mulls_icp_params> params(n, P);
    std::vector<mulls_cloud_view> tgt(n * MULLS_NUM_CLASSES, mulls_cloud_view{nullptr, 0}), src(tgt);
    std::vector<double> ident(16 * n, 0.0);
    for (size_t i = 0; i < n; ++i) {
        tgt[i * MULLS_NUM_CLASSES] = clouds[i];
        for (int d = 0; d < 4; ++d) ident[16 * i + 5 * d] = 1.0;
    }
    int rc = upload_impl(ctx, n, tgt.data(), src.data(), params.data(), ident.data(), nullptr, nullptr, /*resident=*/false, on_device);
    ctx->uploaded = false;
    if (rc != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    A = ctx->A;
    A.trace = nullptr;
    if ((rc = launch_ingest(ctx, A, false, launches, nullptr, nullptr, finite_only)) != MULLS_OK) return rc;
    CK(cudaMemcpyAsync(ctx->h_flags, A.hash_used, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ctx->h_flags + 3, (const char *)A.ps + offsetof(PairState, n_tgt), sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    n_tgt = (int)ctx->h_flags[3];
    if (ctx->h_flags[1]) {
        if ((rc = grow_hash_pool(ctx)) != MULLS_OK) return rc;
        A.hash = ctx->A.hash, A.hash_pool_entries = ctx->A.hash_pool_entries;
        if ((rc = launch_ingest(ctx, A, false, launches, nullptr, nullptr, finite_only)) != MULLS_OK) return rc;
    }
    return MULLS_OK;
}
static int ingest_cloud(mulls_ctx *ctx, mulls_cloud_view cloud, bool on_device, float radius, bool full_pyramid,
                        bool finite_only, DeviceArrays &A, int &n_tgt, uint64_t &launches) {
    return ingest_clouds(ctx, 1, &cloud, on_device, radius, full_pyramid, finite_only, A, n_tgt, launches);
}

// PCA features of one cloud (host rows, or rows already in HBM) into ctx->pca_buf; `args` receives the device arrays.
// unit_dist > 0: distance-adaptive neighbourhoods (k_pca<true>). The PCA is not waited for: the caller consumes the
// arrays on ctx->stream.
static int pca_on_device(mulls_ctx *ctx, mulls_cloud_view cloud, bool cloud_on_device, float radius, int k, int stride,
                         PcaArgs &args, uint64_t &launches, float unit_dist = 0.f) {
    const bool adaptive = unit_dist > 0.f;
    // an adaptive radius grows without bound with the range: it needs the full level pyramid
    DeviceArrays A;
    int n_tgt = 0;
    int rc = ingest_cloud(ctx, cloud, cloud_on_device, radius, adaptive, false, A, n_tgt, launches);
    if (rc != MULLS_OK) return rc;
    const size_t n = cloud.n;
    ScratchLayout L;
    L.take(args.eigenvalues, 3 * n), L.take(args.principal, 3 * n), L.take(args.normal, 3 * n), L.take(args.pt_num, n);
    const size_t outputs = L.bytes;
    // k within the list capacity (the reference uses 20..50): the neighbour lists, and with them pcl::PCA's float mean /
    // covariance accumulated in radiusSearch order — bit-reproducible against the CPU path; larger or unlimited k: fp64
    // warp reduction
    args.nbr = nullptr;
    if (k >= 1 && k <= kPcaListCap) L.take(args.nbr, n * (size_t)k);
    if ((rc = L.grow(ctx, ctx->pca_buf)) != MULLS_OK) return rc;
    args.radius = radius;
    args.r2 = (float)((double)radius * (double)radius);
    args.k = k;
    args.stride = stride;
    cudaStream_t st = ctx->stream;
    CK(cudaMemsetAsync(args.eigenvalues, 0, outputs, st)); // the four outputs, from the layout's start
    if (n && adaptive) {
        PcaAdaptiveArgs aa;
        static_cast<PcaArgs &>(aa) = args;
        aa.unit_dist = unit_dist;
        k_pca<true><<<(unsigned)ceil_div(n, kPcaWarps), kPcaWarps * 32, 0, st>>>(A, aa);
        ++launches;
    } else if (n) {
        k_pca<false><<<(unsigned)ceil_div(n, kPcaWarps), kPcaWarps * 32, 0, st>>>(A, args);
        ++launches;
    }
    return MULLS_OK;
}

// mulls_pca_features / mulls_pca_features_adaptive (unit_dist > 0)
static int pca_features_impl(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int k, int stride, float unit_dist,
                             mulls_pca_out *out, uint64_t &launches) {
    if (!out || !out->eigenvalues || !out->principal || !out->normal || !out->pt_num || stride < 1 || !(radius > 0.f))
        return MULLS_E_ARG;
    PcaArgs args;
    const size_t n = cloud.n;
    int rc = pca_on_device(ctx, cloud, false, radius, k, stride, args, launches, unit_dist);
    if (rc != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    if (n) {
        CK(cudaMemcpyAsync(out->eigenvalues, args.eigenvalues, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out->principal, args.principal, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out->normal, args.normal, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out->pt_num, args.pt_num, n * sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    return MULLS_OK;
}

extern "C" {

int mulls_pca_features(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int k, int stride, mulls_pca_out *out) {
    return front_call(ctx, [&](uint64_t &launches) { return pca_features_impl(ctx, cloud, radius, k, stride, 0.f, out, launches); });
}

int mulls_pca_features_adaptive(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int k, int stride, float unit_dist,
                                mulls_pca_out *out) {
    return front_call(ctx, [&](uint64_t &launches) {
        return unit_dist > 0.f ? pca_features_impl(ctx, cloud, radius, k, stride, unit_dist, out, launches) : MULLS_E_ARG;
    });
}

// ================================================================================================
// Statistical outlier removal (CFilter::sor_filter, cfilter.hpp:203-247): kernels_sor.cuh
// ================================================================================================
static int sor_filter_impl(mulls_ctx *ctx, mulls_cloud_view cloud, int mean_k, double n_std, uint8_t *keep_bits, float *mean_dist,
                           mulls_sor_stats *stats, uint64_t &launches) {
    if (mean_k < 1 || mean_k > kSorMaxMeanK || (cloud.n > 0 && (!cloud.aos48 || !keep_bits))) return MULLS_E_ARG;
    const size_t n = cloud.n;
    int rc = check_capacity(ctx, n, "mulls_sor_filter");
    if (rc != MULLS_OK) return rc;
    if (n <= (size_t)mean_k) { // (checked again on the finite points after the ingest)
        ctx->err = "mulls_sor_filter: the cloud needs more than mean_k finite points";
        return MULLS_E_ARG;
    }
    // the search has no radius: the full level pyramid; the finite points must be more than mean_k
    DeviceArrays A;
    int n_valid = 0;
    if ((rc = ingest_cloud(ctx, cloud, false, 0.f, true, /*finite_only=*/true, A, n_valid, launches)) != MULLS_OK) return rc;
    if (n_valid <= mean_k) {
        ctx->err = "mulls_sor_filter: " + std::to_string(n_valid) + " finite points, mean_k + 1 = " + std::to_string(mean_k + 1) +
                   " neighbours wanted per point";
        return MULLS_E_ARG;
    }
    float *d_dist;
    uint32_t *d_keep;
    mulls_sor_stats *d_stats;
    ScratchLayout L;
    L.take(d_dist, n), L.take(d_keep, ceil_div(n, 32)), L.take(d_stats, 1);
    if ((rc = L.grow(ctx, ctx->sor_buf)) != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    CK(cudaMemsetAsync(d_dist, 0, n * sizeof(float), st)); // non-finite points: distance 0, as PCL
    const unsigned nb = (unsigned)ceil_div((size_t)n_valid, kSorBlock);
    if (mean_k + 1 <= 16) k_sor_dist<16><<<nb, kSorBlock, 0, st>>>(A, mean_k, d_dist);
    else if (mean_k + 1 <= 32) k_sor_dist<32><<<nb, kSorBlock, 0, st>>>(A, mean_k, d_dist);
    else k_sor_dist<64><<<nb, kSorBlock, 0, st>>>(A, mean_k, d_dist);
    k_sor_stats<<<1, 32, 0, st>>>(A, d_dist, (uint32_t)n, n_std, d_stats);
    k_sor_mark<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(d_dist, (uint32_t)n, d_stats, d_keep);
    launches += 3;
    CK(cudaMemcpyAsync(keep_bits, d_keep, (n + 7) / 8, cudaMemcpyDeviceToHost, st));
    if (mean_dist) CK(cudaMemcpyAsync(mean_dist, d_dist, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (stats) CK(cudaMemcpyAsync(stats, d_stats, sizeof(*stats), cudaMemcpyDeviceToHost, st));
    return MULLS_OK;
}
int mulls_sor_filter(mulls_ctx *ctx, mulls_cloud_view cloud, int mean_k, double n_std, uint8_t *keep_bits, float *mean_dist,
                     mulls_sor_stats *stats) {
    return front_call(ctx, [&](uint64_t &launches) {
        return sor_filter_impl(ctx, cloud, mean_k, n_std, keep_bits, mean_dist, stats, launches);
    });
}

// ================================================================================================
// Raw-scan corrections (CFilter::vertical_intrinsic_calibration, get_pts_timestamp_ratio_in_frame,
// apply_motion_compensation, cfilter.hpp:250-291, :412-549): kernels_rawscan.cuh. Stateless: the rows go up, the changed
// column comes back, nothing stays resident.
// ================================================================================================
// raw_buf = [rows of the call, 48 B each][out_floats per point][TsState]; the rows of the n_clouds clouds are copied
// one after the other
static int raw_upload(mulls_ctx *ctx, const mulls_cloud_view *clouds, int n_clouds, size_t n_total, int out_floats,
                      float **d_rows, float **d_out, TsState **d_st) {
    ScratchLayout L;
    L.take(*d_rows, n_total * 12), L.take(*d_out, n_total * out_floats), L.take(*d_st, 1);
    int rc = L.grow(ctx, ctx->raw_buf);
    if (rc != MULLS_OK) return rc;
    size_t at = 0;
    for (int c = 0; c < n_clouds; ++c) {
        if (clouds[c].n)
            CK(cudaMemcpyAsync(*d_rows + at * 12, clouds[c].aos48, clouds[c].n * 48, cudaMemcpyHostToDevice, ctx->stream));
        at += clouds[c].n;
    }
    return MULLS_OK;
}

static int vertical_calib_impl(mulls_ctx *ctx, mulls_cloud_view cloud, double var_vertical_ang_d, int inverse_z, float *xyz_out,
                               int *applied, uint64_t &launches) {
    if (!applied || (cloud.n > 0 && (!cloud.aos48 || !xyz_out))) return MULLS_E_ARG;
    int rc = check_capacity(ctx, cloud.n, "mulls_vertical_intrinsic_calibration");
    if (rc != MULLS_OK) return rc;
    *applied = 0;
    if (var_vertical_ang_d == 0) { // :252-253: the cloud is left as it is
        for (size_t i = 0; i < cloud.n; ++i)
            for (int d = 0; d < 3; ++d) xyz_out[3 * i + d] = cloud.aos48[12 * i + d];
        return MULLS_OK;
    }
    const int negate_only = (var_vertical_ang_d >= 180.0 || inverse_z) ? 1 : 0; // :255-263
    if (cloud.n > 0) {
        float *d_rows, *d_out;
        TsState *d_st;
        if ((rc = raw_upload(ctx, &cloud, 1, cloud.n, 3, &d_rows, &d_out, &d_st)) != MULLS_OK) return rc;
        const double var_rad = var_vertical_ang_d / 180.0 * M_PI;
        k_vertical_calib<<<(unsigned)ceil_div(cloud.n, kRawBlock), kRawBlock, 0, ctx->stream>>>(d_rows, (uint32_t)cloud.n, var_rad,
                                                                                                negate_only, d_out);
        ++launches;
        CK(cudaMemcpyAsync(xyz_out, d_out, cloud.n * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
    *applied = negate_only ? 0 : 1;
    return MULLS_OK;
}

static int timestamp_ratio_impl(mulls_ctx *ctx, mulls_cloud_view cloud, int timestamp_available, double scan_begin_ang_deg,
                                float scan_duration_ms, float *ratio_out, uint64_t &launches) {
    if (cloud.n > 0 && (!cloud.aos48 || !ratio_out)) return MULLS_E_ARG;
    int rc = check_capacity(ctx, cloud.n, "mulls_timestamp_ratio");
    if (rc != MULLS_OK) return rc;
    const size_t n = cloud.n;
    if (n == 0) return MULLS_OK;
    float *d_rows, *d_out;
    TsState *d_st;
    if ((rc = raw_upload(ctx, &cloud, 1, n, 1, &d_rows, &d_out, &d_st)) != MULLS_OK) return rc;
    const unsigned nb = (unsigned)ceil_div(n, kRawBlock);
    cudaStream_t st = ctx->stream;
    if (timestamp_available) {
        TsState init{};
        init.min_key = ~0ull;
        CK(cudaMemcpyAsync(d_st, &init, sizeof(init), cudaMemcpyHostToDevice, st));
        k_ts_last_nan<9><<<nb, kRawBlock, 0, st>>>(d_rows, (uint32_t)n, d_st);
        k_ts_extremes<9><<<nb, kRawBlock, 0, st>>>(d_rows, (uint32_t)n, d_st);
        k_ts_setup<<<1, 32, 0, st>>>(d_rows, (uint32_t)n, scan_duration_ms, d_st);
        k_ts_ratio<<<nb, kRawBlock, 0, st>>>(d_rows, (uint32_t)n, d_st, d_out);
        launches += 4;
    } else {
        k_azimuth_ratio<<<nb, kRawBlock, 0, st>>>(d_rows, (uint32_t)n, scan_begin_ang_deg / 180.0 * M_PI, d_out);
        launches += 1;
    }
    CK(cudaMemcpyAsync(ratio_out, d_out, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    return MULLS_OK;
}

static int motion_compensation_impl(mulls_ctx *ctx, const mulls_cloud_view *clouds, int n_clouds, const double *T,
                                    float s_ambiguous_thre, float *const *xyz_out, uint64_t &launches) {
    if (!clouds || !T || !xyz_out || n_clouds < 1 || n_clouds > MULLS_NUM_CLASSES) return MULLS_E_ARG;
    size_t n = 0;
    for (int c = 0; c < n_clouds; ++c) {
        if (clouds[c].n > 0 && (!clouds[c].aos48 || !xyz_out[c])) return MULLS_E_ARG;
        n += clouds[c].n;
    }
    int rc = check_capacity(ctx, n, "mulls_motion_compensation");
    if (rc != MULLS_OK || n == 0) return rc;
    float *d_rows, *d_out;
    TsState *d_st;
    if ((rc = raw_upload(ctx, clouds, n_clouds, n, 3, &d_rows, &d_out, &d_st)) != MULLS_OK) return rc;
    const SlerpConst sc = slerp_const_of(T);
    k_motion_compensation<<<(unsigned)ceil_div(n, kRawBlock), kRawBlock, 0, ctx->stream>>>(d_rows, (uint32_t)n, sc, s_ambiguous_thre,
                                                                                           d_out);
    ++launches;
    size_t at = 0;
    for (int c = 0; c < n_clouds; ++c) {
        if (clouds[c].n)
            CK(cudaMemcpyAsync(xyz_out[c], d_out + 3 * at, clouds[c].n * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        at += clouds[c].n;
    }
    return MULLS_OK;
}

int mulls_vertical_intrinsic_calibration(mulls_ctx *ctx, mulls_cloud_view cloud, double var_vertical_ang_d, int inverse_z,
                                         float *xyz_out, int *applied) {
    return front_call(ctx, [&](uint64_t &launches) {
        return vertical_calib_impl(ctx, cloud, var_vertical_ang_d, inverse_z, xyz_out, applied, launches);
    });
}
int mulls_timestamp_ratio(mulls_ctx *ctx, mulls_cloud_view cloud, int timestamp_available, double scan_begin_ang_deg,
                          float scan_duration_ms, float *ratio_out) {
    return front_call(ctx, [&](uint64_t &launches) {
        return timestamp_ratio_impl(ctx, cloud, timestamp_available, scan_begin_ang_deg, scan_duration_ms, ratio_out, launches);
    });
}
int mulls_motion_compensation(mulls_ctx *ctx, const mulls_cloud_view *clouds, int n_clouds, const double T[16],
                              float s_ambiguous_thre, float *const *xyz_out) {
    return front_call(ctx, [&](uint64_t &launches) {
        return motion_compensation_impl(ctx, clouds, n_clouds, T, s_ambiguous_thre, xyz_out, launches);
    });
}

// ================================================================================================
// NCC keypoint matching (CRegistration::find_feature_correspondence_ncc, cregistration.hpp:409-601): kernels_ncc.cuh.
// Stateless like the raw-scan corrections: the resident batch and its grid are left alone.
// ================================================================================================
static int ncc_impl(mulls_ctx *ctx, mulls_cloud_view tk, mulls_cloud_view sk, int fixed_num_corr, int corr_num, int reciprocal_on,
                    int32_t *tgt_idx, int32_t *src_idx, size_t cap, size_t *n_out, int *performed, uint64_t &launches) {
    if (!n_out || !performed || (tk.n && !tk.aos48) || (sk.n && !sk.aos48) || (cap && (!tgt_idx || !src_idx)))
        return MULLS_E_ARG;
    *n_out = 0;
    *performed = 0;
    const char *fn = "mulls_ncc_correspondences";
    int rc;
    if ((rc = check_capacity(ctx, tk.n, fn)) != MULLS_OK || (rc = check_capacity(ctx, sk.n, fn)) != MULLS_OK) return rc;
    const size_t nt = tk.n, ns = sk.n, n_all = nt + ns;
    if (nt < 10 || ns < 10) return MULLS_OK; // :421-425
    const size_t M = nt * ns;
    size_t K = 0;
    if (fixed_num_corr) {
        if (M > (size_t)INT_MAX) { // :559 forms the pair index in int
            ctx->err = std::string(fn) + ": " + std::to_string(nt) + " x " + std::to_string(ns) +
                       " pairs exceed INT_MAX in the fixed-number mode";
            return MULLS_E_ARG;
        }
        K = ((size_t)corr_num < M) ? (size_t)corr_num : M; // :565 min_(corr_num, dist_array.size()): int vs size_t
    }
    const size_t gy = ceil_div(ns, kNccTileS);
    if (gy > 65535) {
        ctx->err = std::string(fn) + ": too many source keypoints for one grid";
        return MULLS_E_CAPACITY;
    }
    cudaStream_t st = ctx->stream;
    float *d_rows, *d_desc, *d_range;
    TsState *d_ts;
    ScratchLayout L;
    L.take(d_rows, n_all * 12), L.take(d_desc, n_all * kNccDim), L.take(d_ts, 1), L.take(d_range, 2);
    unsigned long long *d_rowkey = nullptr, *d_cand = nullptr, *d_out = nullptr, *d_gath = nullptr, *d_sorted = nullptr;
    uint32_t *d_colmin = nullptr;
    uint8_t *d_keep = nullptr;
    int *d_num = nullptr;
    NccSelect *d_sel = nullptr;
    void *d_tmp;
    size_t tmp_bytes = 0;
    if (!fixed_num_corr) {
        L.take(d_rowkey, nt), L.take(d_colmin, ns), L.take(d_cand, nt), L.take(d_keep, nt), L.take(d_out, nt), L.take(d_num, 1);
        CK(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, (unsigned long long *)nullptr, (uint8_t *)nullptr,
                                      (unsigned long long *)nullptr, (int *)nullptr, (int)nt, st));
    } else {
        L.take(d_sel, 1), L.take(d_gath, K), L.take(d_sorted, K);
        CK(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                          (int)std::max<size_t>(K, 1), 0, 64, st));
    }
    L.take_bytes(d_tmp, tmp_bytes);
    if ((rc = L.grow(ctx, ctx->ncc_buf)) != MULLS_OK) return rc;
    CK(cudaMemcpyAsync(d_rows, tk.aos48, nt * 48, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync((char *)d_rows + nt * 48, sk.aos48, ns * 48, cudaMemcpyHostToDevice, st));
    TsState ts0{};
    ts0.min_key = ~0ull;
    CK(cudaMemcpyAsync(d_ts, &ts0, sizeof(ts0), cudaMemcpyHostToDevice, st));
    const unsigned nbt = (unsigned)ceil_div(nt, kRawBlock);
    k_ts_last_nan<8><<<nbt, kRawBlock, 0, st>>>(d_rows, (uint32_t)nt, d_ts);
    k_ts_extremes<8><<<nbt, kRawBlock, 0, st>>>(d_rows, (uint32_t)nt, d_ts);
    k_ncc_range<<<1, 32, 0, st>>>(d_rows, (uint32_t)nt, d_ts, d_range);
    k_ncc_descriptors<<<(unsigned)ceil_div(n_all, kRawBlock), kRawBlock, 0, st>>>(d_rows, (uint32_t)n_all, d_range, d_desc);
    launches += 4;
    const NccPairs P{d_desc, (uint32_t)n_all, (uint32_t)nt, (uint32_t)ns};
    const dim3 grid((unsigned)ceil_div(nt, kNccTileT), (unsigned)gy);
    std::vector<std::pair<int32_t, int32_t>> res;
    if (!fixed_num_corr) {
        k_ncc_init<<<(unsigned)ceil_div(std::max(nt, ns), kRawBlock), kRawBlock, 0, st>>>(d_rowkey, (uint32_t)nt, d_colmin, (uint32_t)ns);
        if (reciprocal_on)
            k_ncc_pairs<kNccRowCol><<<grid, kNccBlock, 0, st>>>(P, d_rowkey, d_colmin, nullptr, 0, nullptr, 0);
        else
            k_ncc_pairs<kNccRow><<<grid, kNccBlock, 0, st>>>(P, d_rowkey, nullptr, nullptr, 0, nullptr, 0);
        k_ncc_pick<<<nbt, kRawBlock, 0, st>>>(d_rowkey, d_colmin, (uint32_t)nt, reciprocal_on ? 1 : 0, d_cand, d_keep);
        launches += 3;
        size_t tb = tmp_bytes;
        CK(cub::DeviceSelect::Flagged(d_tmp, tb, d_cand, d_keep, d_out, d_num, (int)nt, st));
        std::vector<unsigned long long> h(nt);
        int n_kept = 0;
        CK(cudaMemcpyAsync(&n_kept, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h.data(), d_out, nt * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(st));
        res.reserve(n_kept);
        for (int k = 0; k < n_kept; ++k) res.emplace_back((int32_t)(h[k] >> 32), (int32_t)(uint32_t)h[k]);
    } else if (K > 0) {
        NccSelect s0{};
        s0.rank = (uint32_t)(K - 1);
        s0.E = 0xffffffffu;
        if (K == M) s0.T = 0xffffffffu; // every pair: nothing to select
        CK(cudaMemcpyAsync(d_sel, &s0, offsetof(NccSelect, hist), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_sel->hist, 0, sizeof(s0.hist), st));
        if (K < M) {
            for (int shift = 24; shift >= 0; shift -= 8) { // the K-th smallest distance key T
                k_ncc_pairs<kNccHistKey><<<grid, kNccBlock, 0, st>>>(P, nullptr, nullptr, d_sel, shift, nullptr, 0);
                k_ncc_select_step<<<1, 32, 0, st>>>(d_sel, shift, 0);
                launches += 2;
            }
            NccSelect h_sel;
            CK(cudaMemcpyAsync(&h_sel, d_sel, offsetof(NccSelect, hist), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (h_sel.need_eq < h_sel.count_eq) { // ties at T: the need_eq lowest pair indices among them
                for (int shift = 24; shift >= 0; shift -= 8) {
                    k_ncc_pairs<kNccHistIdx><<<grid, kNccBlock, 0, st>>>(P, nullptr, nullptr, d_sel, shift, nullptr, 0);
                    k_ncc_select_step<<<1, 32, 0, st>>>(d_sel, shift, 1);
                    launches += 2;
                }
            }
        }
        k_ncc_pairs<kNccGather><<<grid, kNccBlock, 0, st>>>(P, nullptr, nullptr, d_sel, 0, d_gath, K);
        size_t tb = tmp_bytes;
        CK(cub::DeviceRadixSort::SortKeys(d_tmp, tb, d_gath, d_sorted, (int)K, 0, 64, st));
        launches += 1;
        std::vector<unsigned long long> h(K);
        unsigned long long gathered = 0;
        CK(cudaMemcpyAsync(&gathered, &d_sel->count, sizeof(gathered), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h.data(), d_sorted, K * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(st));
        if (gathered != K) {
            ctx->err = std::string(fn) + ": the select gathered " + std::to_string(gathered) + " pairs for K = " + std::to_string(K);
            return MULLS_E_CUDA;
        }
        // :567-586, the walk over the first K pairs in order: at most 7 pairs per target and per source
        std::vector<int> count_target_kpt(nt, 0), count_source_kpt(ns, 0);
        const int max_corr_num = 6;
        for (size_t k = 0; k < K; ++k) {
            const uint32_t index = (uint32_t)h[k];
            const int i = (int)(index / ns), j = (int)(index % ns);
            if (count_target_kpt[i] > max_corr_num || count_source_kpt[j] > max_corr_num) continue;
            count_target_kpt[i]++;
            count_source_kpt[j]++;
            res.emplace_back(i, j);
        }
    }
    if (res.size() > cap) {
        ctx->err = std::string(fn) + ": " + std::to_string(res.size()) + " correspondences, room for " + std::to_string(cap);
        return MULLS_E_ARG;
    }
    for (size_t k = 0; k < res.size(); ++k) tgt_idx[k] = res[k].first, src_idx[k] = res[k].second;
    *n_out = res.size();
    *performed = 1;
    return MULLS_OK;
}
int mulls_ncc_correspondences(mulls_ctx *ctx, mulls_cloud_view target_kpts, mulls_cloud_view source_kpts, int fixed_num_corr,
                              int corr_num, int reciprocal_on, int32_t *tgt_idx, int32_t *src_idx, size_t cap, size_t *n_out,
                              int *performed) {
    return front_call(ctx, [&](uint64_t &launches) {
        return ncc_impl(ctx, target_kpts, source_kpts, fixed_num_corr, corr_num, reciprocal_on, tgt_idx, src_idx, cap, n_out,
                        performed, launches);
    });
}

// ================================================================================================
// RANSAC coarse registration (CRegistration::coarse_reg_ransac, cregistration.hpp:604-661): ransac_core.cuh,
// kernels_ransac.cuh. Stateless like the NCC matching: the resident batch and its grid are left alone.
// The sample stream is drawn here in chunks: kRcFirstChunk hypotheses, then up to kRcChunk. After each chunk the counts
// come down and the adaptive-k walk is replayed over them. Once a k is known, the next chunk is drawn while the device
// fits and scores the current one, never past ceil(k) hypotheses: a search that ends early draws little more than it uses.
// ================================================================================================
static constexpr int kRcFirstChunk = 64;
static constexpr int kRcChunk = 4096;

static int ransac_impl(mulls_ctx *ctx, mulls_cloud_view tv, mulls_cloud_view sv, float noise_bound, int min_inlier_num,
                       int max_iter_num, double *tran_mat, int *status, int *n_inliers, int *n_hypotheses, uint64_t &launches) {
    if (!tran_mat || !status || !n_inliers || !n_hypotheses || (tv.n && !tv.aos48) || (sv.n && !sv.aos48))
        return MULLS_E_ARG;
    const char *fn = "mulls_coarse_reg_ransac";
    const size_t N = tv.n;
    if (sv.n < N) { // the reference would read source rows past the end
        ctx->err = std::string(fn) + ": " + std::to_string(sv.n) + " source points for " + std::to_string(N) + " target points";
        return MULLS_E_ARG;
    }
    int rc;
    if ((rc = check_capacity(ctx, N, fn)) != MULLS_OK) return rc;
    if (N > (size_t)INT_MAX) {
        ctx->err = std::string(fn) + ": more than INT_MAX correspondences";
        return MULLS_E_ARG;
    }
    if (ceil_div(N, kRcTile) > 65535) { // k_ransac_count's grid.y
        ctx->err = std::string(fn) + ": " + std::to_string(N) + " correspondences exceed one count grid (" +
                   std::to_string((size_t)65535 * kRcTile) + ")";
        return MULLS_E_CAPACITY;
    }
    float T[12] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f}; // identity
    size_t n_final = 0;
    int hyps = 0;
    if (N > 0) { // an empty correspondence list returns before the rejector runs (getCorrespondences)
        cudaStream_t st = ctx->stream;
        float *d_corr, *d_best, *d_T[2];
        int *d_samp[2], *d_cnt[2];
        RcRefineArgs A{};
        ScratchLayout L;
        L.take(d_corr, N * 6), L.take(d_samp[0], 3 * kRcChunk), L.take(d_samp[1], 3 * kRcChunk);
        L.take(d_T[0], 12 * kRcChunk), L.take(d_T[1], 12 * kRcChunk), L.take(d_cnt[0], kRcChunk), L.take(d_cnt[1], kRcChunk);
        L.take(d_best, 12), L.take(A.flag_a, N), L.take(A.flag_b, N), L.take(A.err, N), L.take(A.out, 1);
        if ((rc = L.grow(ctx, ctx->rc_buf)) != MULLS_OK) return rc;
        if (!ctx->rc_host) CK(cudaMallocHost(&ctx->rc_host, 2 * kRcChunk * 4 * sizeof(int)));
        int *h_samp[2] = {(int *)ctx->rc_host, (int *)ctx->rc_host + 3 * kRcChunk};
        int *h_cnt[2] = {(int *)ctx->rc_host + 6 * kRcChunk, (int *)ctx->rc_host + 7 * kRcChunk};
        // the correspondences i <-> i: source x y z, target x y z
        std::vector<float> c6(N * 6);
        for (size_t i = 0; i < N; ++i)
            for (int c = 0; c < 3; ++c) c6[6 * i + c] = sv.aos48[12 * i + c], c6[6 * i + 3 + c] = tv.aos48[12 * i + c];
        CK(cudaMemcpyAsync(d_corr, c6.data(), N * 6 * sizeof(float), cudaMemcpyHostToDevice, st));
        std::vector<int> shuf(N);
        for (size_t i = 0; i < N; ++i) shuf[i] = (int)i;
        SacSampler S{SacMt19937(), shuf.data(), N, sv.aos48, rc_sample_dist_threshold(sv.aos48, N)};
        SacWalk W(N, max_iter_num);
        // no more hypotheses than the walk can take: max_iterations + 1, or none when max_skip is 0
        const int64_t cap_hyp = W.max_skip == 0 ? 0 : (max_iter_num < 0 ? 1 : (int64_t)max_iter_num + 1);
        int64_t produced = 0;
        bool exhausted = false;
        // draws up to `want` samples, and never more hypotheses than the walk can take: cap_hyp, and once a count is in,
        // ceil(k) (k only falls as the best count rises, so the k known now bounds the walk's end)
        auto draw_chunk = [&](int *dst, int want) {
            const int64_t lim = (W.best >= 0 && W.k < (double)cap_hyp) ? (int64_t)ceil(W.k) : cap_hyp;
            int c = 0;
            while (c < want && produced < lim && !exhausted) {
                if (!S.draw(dst + 3 * c)) {
                    exhausted = true;
                    break;
                }
                ++c, ++produced;
            }
            return c;
        };
        const double thresh_sq = (double)noise_bound * (double)noise_bound;
        int cnt[2] = {draw_chunk(h_samp[0], kRcFirstChunk), 0}, cur = 0;
        bool done = !W.wants();
        while (!done && cnt[cur] > 0) {
            const int H = cnt[cur];
            CK(cudaMemcpyAsync(d_samp[cur], h_samp[cur], (size_t)H * 3 * sizeof(int), cudaMemcpyHostToDevice, st));
            CK(cudaMemsetAsync(d_cnt[cur], 0, (size_t)H * sizeof(int), st));
            k_ransac_fit<<<(unsigned)ceil_div(H, kRcFitBlock), kRcFitBlock, 0, st>>>(d_corr, d_samp[cur], H, d_T[cur]);
            const dim3 grid((unsigned)ceil_div(H, kRcCountBlock * kRcHypPerThread), (unsigned)ceil_div(N, kRcTile));
            k_ransac_count<<<grid, kRcCountBlock, 0, st>>>(d_corr, (int)N, d_T[cur], H, thresh_sq, d_cnt[cur]);
            CK(cudaMemcpyAsync(h_cnt[cur], d_cnt[cur], (size_t)H * sizeof(int), cudaMemcpyDeviceToHost, st));
            launches += 2;
            const int nxt = cur ^ 1;
            // the next chunk is drawn while this one is scored, once a k is known to bound it
            cnt[nxt] = W.best >= 0 ? draw_chunk(h_samp[nxt], kRcChunk) : 0;
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(st));
            const int best_before = W.best;
            for (int h = 0; h < H && !done; ++h) {
                if (!W.wants()) done = true;
                else W.take(h_cnt[cur][h]);
            }
            if (W.best != best_before) // keep the best model before its chunk buffer is reused
                CK(cudaMemcpyAsync(d_best, d_T[cur] + 12 * (size_t)(W.best - hyps), 12 * sizeof(float), cudaMemcpyDeviceToDevice, st));
            hyps += H;
            if (!W.wants()) done = true;
            else if (cnt[nxt] == 0) cnt[nxt] = draw_chunk(h_samp[nxt], kRcChunk); // after the first chunk
            cur = nxt;
        }
        hyps = W.iterations;
        if (W.best < 0) { // computeModel failed: every correspondence, identity
            n_final = N;
        } else {
            A.corr = d_corr, A.n = (int)N, A.T_best = d_best, A.threshold = (double)noise_bound;
            k_ransac_refine<<<1, kRcLanes, 0, st>>>(A);
            launches += 1;
            RcRefineOut o;
            CK(cudaMemcpyAsync(&o, A.out, sizeof(o), cudaMemcpyDeviceToHost, st));
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(st));
            if (!o.ok) {
                n_final = 0; // refinement failed: no correspondences; T stays the identity (PCL's is uninitialised)
            } else if (o.n_inliers < 3) {
                n_final = N;
            } else {
                n_final = (size_t)o.n_inliers;
                std::memcpy(T, o.T, sizeof(T));
            }
        }
    }
    // final_corres->size() >= min_inlier_num: int against size_t, so a negative minimum is never reached
    const size_t lo = (size_t)(int64_t)min_inlier_num, hi = (size_t)(int64_t)(int32_t)((uint32_t)min_inlier_num * 2u);
    int stat = -1;
    if (n_final >= lo) {
        stat = n_final >= hi ? 1 : 0;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c) tran_mat[4 * r + c] = (double)T[4 * r + c];
        tran_mat[12] = tran_mat[13] = tran_mat[14] = 0.0;
        tran_mat[15] = 1.0;
    }
    *status = stat;
    *n_inliers = (int)n_final;
    *n_hypotheses = hyps;
    return MULLS_OK;
}
int mulls_coarse_reg_ransac(mulls_ctx *ctx, mulls_cloud_view target_pts, mulls_cloud_view source_pts, float noise_bound,
                            int min_inlier_num, int max_iter_num, double tran_mat[16], int *status, int *n_inliers,
                            int *n_hypotheses) {
    return front_call(ctx, [&](uint64_t &launches) {
        return ransac_impl(ctx, target_pts, source_pts, noise_bound, min_inlier_num, max_iter_num, tran_mat, status, n_inliers,
                           n_hypotheses, launches);
    });
}

// ================================================================================================
// TEASER++ coarse registration (CRegistration::coarse_reg_teaser, cregistration.hpp:664-759): teaser_core.cuh,
// kernels_teaser.cuh. Stateless like the RANSAC: the resident batch and its grid are left alone.
// The graph, its core numbers and a greedy clique come first. Vertices whose core number is below the greedy size
// minus one cannot be in a maximum clique and are dropped. Unless the greedy clique already meets the core bound, a
// kTmMax search finds the clique number; a kTmLex search then finds the lexicographically smallest clique of that
// size. Both run in launches of at most kTmLaunchWords words per warp, the host relaunching until the search is done.
// ================================================================================================
static constexpr int kTmHindexBatch = 4;                           // h-index steps between two looks at the flag
static constexpr unsigned long long kTmLaunchWords = 1ull << 18;   // search work per warp and launch
static constexpr int kTmMaxSlots = 2048;                           // warps of one search launch, at most
static constexpr size_t kTmStackBytes = (size_t)256 << 20;         // the stacks of all slots together, at most
static constexpr size_t kTmKeepBytes = (size_t)64 << 20;           // search scratch a context keeps after a call, at most

static int teaser_impl(mulls_ctx *ctx, mulls_cloud_view tv, mulls_cloud_view sv, float noise_bound, int min_inlier_num,
                       double *tran_mat, int *status, mulls_teaser_info *info_out, uint64_t &launches) {
    if (!tran_mat || !status || (tv.n && !tv.aos48) || (sv.n && !sv.aos48)) return MULLS_E_ARG;
    const char *fn = "mulls_coarse_reg_teaser";
    mulls_teaser_info info{};
    const size_t N = tv.n;
    if (sv.n != N || N <= 3) { // cregistration.hpp:675-685
        *status = -1;
        if (info_out) *info_out = info;
        return MULLS_OK;
    }
    if (N > (size_t)MULLS_TEASER_MAX_CORR) {
        ctx->err = std::string(fn) + ": " + std::to_string(N) + " correspondences exceed MULLS_TEASER_MAX_CORR (" +
                   std::to_string(MULLS_TEASER_MAX_CORR) + ")";
        return MULLS_E_CAPACITY;
    }
    int rc;
    if ((rc = check_capacity(ctx, N, fn)) != MULLS_OK) return rc;
    const int n = (int)N, W = (int)ceil_div(N, 64);
    const double nb = (double)noise_bound;
    int padded = 1;
    while (padded < 2 * n) padded <<= 1;
    cudaStream_t st = ctx->stream;
    // ---- the graph, the core numbers, the greedy clique ----
    double *d_p6, *d_tims, *d_w, *d_r, *d_R, *d_x3, *d_t;
    uint64_t *d_adj, *d_cand;
    int *d_core, *d_small, *d_clique, *d_gout;
    unsigned long long *d_edges;
    uint8_t *d_mask;
    TmBound *d_bnd;
    ScratchLayout L;
    L.take(d_p6, 6 * N), L.take(d_adj, N * W), L.take(d_core, N), L.take(d_small, 2), L.take(d_edges, 1), L.take(d_cand, W);
    L.take(d_clique, N), L.take(d_tims, 6 * N), L.take(d_w, N), L.take(d_r, N), L.take(d_mask, N), L.take(d_R, 9);
    L.take(d_gout, 2), L.take(d_x3, 3 * N), L.take(d_bnd, 3 * (size_t)padded), L.take(d_t, 3);
    if ((rc = L.grow(ctx, ctx->tm_buf)) != MULLS_OK) return rc;
    std::vector<double> p6(6 * N); // solve(src, dst): source x y z, target x y z, widened
    for (size_t i = 0; i < N; ++i)
        for (int c = 0; c < 3; ++c) p6[6 * i + c] = (double)sv.aos48[12 * i + c], p6[6 * i + 3 + c] = (double)tv.aos48[12 * i + c];
    CK(cudaMemcpyAsync(d_p6, p6.data(), 6 * N * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_core, 0, N * sizeof(int), st));
    CK(cudaMemsetAsync(d_edges, 0, sizeof(unsigned long long), st));
    k_tm_graph<<<(unsigned)ceil_div(N * W, kTmGraphBlock), kTmGraphBlock, 0, st>>>(d_p6, n, W, 2.0 * nb, d_adj, d_core, d_edges);
    ++launches;
    const unsigned hb = (unsigned)ceil_div(N, kTmWarpsPerBlock);
    for (;;) { // h-index steps from the degrees until one changes nothing
        for (int b = 0; b < kTmHindexBatch; ++b) {
            if (b == kTmHindexBatch - 1) CK(cudaMemsetAsync(d_small, 0, sizeof(int), st));
            k_tm_hindex<<<hb, 32 * kTmWarpsPerBlock, 0, st>>>(d_adj, n, W, d_core, d_small);
            ++launches;
        }
        int changed = 0;
        CK(cudaMemcpyAsync(&changed, d_small, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (!changed) break;
    }
    k_tm_greedy<<<1, kTmGreedyBlock, 0, st>>>(d_adj, n, W, d_core, d_cand, d_small + 1);
    ++launches;
    std::vector<int> core(N);
    int lb = 0;
    unsigned long long edges2 = 0;
    CK(cudaMemcpyAsync(core.data(), d_core, N * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&lb, d_small + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&edges2, d_edges, sizeof(edges2), cudaMemcpyDeviceToHost, st));
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    info.n_edges = (int64_t)(edges2 / 2);
    for (int c : core) info.max_core = std::max(info.max_core, c);
    const int ub = info.max_core + 1;
    int omega = lb;
    std::vector<int> clique;
    if (lb >= 2) { // an edge exists
        // ---- the pruned graph and the search ----
        std::vector<int> map, map_core, rcore;
        for (int i = 0; i < n; ++i)
            if (core[i] >= lb - 1) map.push_back(i);
        map_core = map; // kTmMax: ascending core number, then index
        std::stable_sort(map_core.begin(), map_core.end(), [&](int a, int b) { return core[a] < core[b]; });
        for (int v : map_core) rcore.push_back(core[v]);
        const int n2 = (int)map.size(), W2 = (int)ceil_div((size_t)n2, 64), levels = ub + 1;
        const size_t per_slot = (size_t)levels * (W2 * sizeof(uint64_t) + sizeof(int) + sizeof(TmLevel) + kTmOrder * sizeof(int2));
        size_t slots = std::min<size_t>({(size_t)kTmMaxSlots, ceil_div((size_t)n2, kTmWarpsPerBlock) * kTmWarpsPerBlock,
                                         std::max<size_t>(kTmStackBytes / per_slot, 1)});
        slots = ceil_div(slots, kTmWarpsPerBlock) * kTmWarpsPerBlock;
        int *d_map, *d_rcore;
        TmSearchArgs S{};
        ScratchLayout L2;
        L2.take(d_map, n2), L2.take(d_rcore, n2), L2.take(S.stack, slots * levels * W2), L2.take(S.path, slots * levels), L2.take(S.slots, slots);
        L2.take(S.lvl, slots * levels), L2.take(S.ring, slots * levels * kTmOrder);
        L2.take(S.ctl, 1);
        uint64_t *d_adj2;
        L2.take(d_adj2, (size_t)n2 * W2);
        if ((rc = L2.grow(ctx, ctx->tm_srch_buf)) != MULLS_OK) return rc;
        // the pruned graph with its vertices in the order `m`
        auto compact = [&](const std::vector<int> &m) -> int {
            CK(cudaMemcpyAsync(d_map, m.data(), n2 * sizeof(int), cudaMemcpyHostToDevice, st));
            k_tm_compact<<<(unsigned)ceil_div((size_t)n2 * W2, kTmGraphBlock), kTmGraphBlock, 0, st>>>(d_adj, W, d_map, n2, W2, d_adj2);
            ++launches;
            return MULLS_OK;
        };
        CK(cudaMemcpyAsync(d_rcore, rcore.data(), n2 * sizeof(int), cudaMemcpyHostToDevice, st));
        S.adj = d_adj2, S.core = d_rcore, S.n = n2, S.W = W2, S.levels = levels, S.ub = ub, S.launch_words = kTmLaunchWords;
        TmCtl h{};
        auto search = [&](int mode, int target, int best0) -> int {
            TmCtl c0{};
            c0.best = best0;
            c0.found = ~0ull;
            CK(cudaMemcpyAsync(S.ctl, &c0, sizeof(c0), cudaMemcpyHostToDevice, st));
            CK(cudaMemsetAsync(S.slots, 0xff, slots * sizeof(TmSlot), st)); // task -1: none
            S.mode = mode, S.target = target;
            unsigned long long work_seen = 0;
            for (;;) {
                CK(cudaMemsetAsync(&S.ctl->active, 0, sizeof(int), st));
                const unsigned nb = (unsigned)(slots / kTmWarpsPerBlock), nt = 32 * kTmWarpsPerBlock;
                if (W2 <= 32) k_tm_search<1><<<nb, nt, 0, st>>>(S);
                else if (W2 <= 64) k_tm_search<2><<<nb, nt, 0, st>>>(S);
                else if (W2 <= 128) k_tm_search<4><<<nb, nt, 0, st>>>(S);
                else if (W2 <= 256) k_tm_search<8><<<nb, nt, 0, st>>>(S);
                else k_tm_search<16><<<nb, nt, 0, st>>>(S);
                ++launches, ++info.search_launches;
                CK(cudaMemcpyAsync(&h, S.ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
                CK(cudaGetLastError());
                CK(cudaStreamSynchronize(st));
                const bool stop = mode == kTmLex ? h.found != ~0ull : h.best >= ub;
                if (h.active == 0 && (stop || h.next_task >= n2)) break;
                if (info.search_launches >= MULLS_TEASER_SEARCH_LAUNCHES) {
                    ctx->err = std::string(fn) + ": the maximum-clique search used MULLS_TEASER_SEARCH_LAUNCHES launches (" +
                               std::to_string(n2) + " vertices after pruning, clique bound " + std::to_string(ub) +
                               (mode == kTmMax ? ", proving the clique number; best so far " + std::to_string(h.best)
                                               : ", finding the smallest clique of " + std::to_string(target)) + ")";
                    return MULLS_E_CAPACITY;
                }
                if (h.work == work_seen) { // every launch takes a root or expands a node
                    ctx->err = std::string(fn) + ": a search launch made no progress";
                    return MULLS_E_CUDA;
                }
                work_seen = h.work;
            }
            return MULLS_OK;
        };
        if (lb < ub) {
            if ((rc = compact(map_core)) != MULLS_OK || (rc = search(kTmMax, 0, lb)) != MULLS_OK) return rc;
            omega = h.best;
        }
        if ((rc = compact(map)) != MULLS_OK || (rc = search(kTmLex, omega, 0)) != MULLS_OK) return rc;
        if (h.found == ~0ull) {
            ctx->err = std::string(fn) + ": no clique of the size the search found";
            return MULLS_E_CUDA;
        }
        std::vector<int> path(omega);
        CK(cudaMemcpyAsync(path.data(), S.path + (size_t)(h.found & 0xffffffffu) * levels, omega * sizeof(int),
                           cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (int v : path) clique.push_back(map[v]);
    }
    info.clique_size = omega;
    const bool valid = omega >= 2; // T3: a clique of at most one vertex
    double R[9], t[3];
    if (valid) {
        // ---- GNC-TLS and the voting ----
        const int M = omega;
        CK(cudaMemcpyAsync(d_clique, clique.data(), M * sizeof(int), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_gout, 0, 2 * sizeof(int), st));
        TmGncArgs G{d_p6, d_clique, M, nb, d_tims, d_w, d_r, d_mask, d_R, d_gout};
        k_tm_gnc<<<1, kTmLanes, 0, st>>>(G);
        int pm = 1;
        while (pm < 2 * M) pm <<= 1;
        k_tm_vote<<<3, kTmVoteBlock, 0, st>>>(d_p6, d_clique, M, d_R, nb, d_x3, d_bnd, pm, d_t);
        launches += 2;
        int gout[2];
        CK(cudaMemcpyAsync(gout, d_gout, sizeof(gout), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(R, d_R, sizeof(R), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(t, d_t, sizeof(t), cudaMemcpyDeviceToHost, st));
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(st));
        info.gnc_iterations = gout[0];
        info.rotation_inliers = gout[1];
    }
    // inliers.size() >= min_inlier_num: int against size_t, so a negative minimum is never reached
    const size_t cnt = (size_t)info.rotation_inliers;
    const size_t lo = (size_t)(int64_t)min_inlier_num, hi = (size_t)(int64_t)(int32_t)((uint32_t)min_inlier_num * 2u);
    int stat = -1;
    if (valid && cnt >= lo) {
        stat = cnt >= hi ? 1 : 0;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) tran_mat[4 * r + c] = R[3 * r + c];
            tran_mat[4 * r + 3] = t[r];
        }
        tran_mat[12] = tran_mat[13] = tran_mat[14] = 0.0;
        tran_mat[15] = 1.0;
    }
    *status = stat;
    if (info_out) *info_out = info;
    return MULLS_OK;
}
int mulls_coarse_reg_teaser(mulls_ctx *ctx, mulls_cloud_view target_pts, mulls_cloud_view source_pts, float noise_bound,
                            int min_inlier_num, double tran_mat[16], int *status, mulls_teaser_info *info) {
    const int rc = front_call(ctx, [&](uint64_t &launches) {
        return teaser_impl(ctx, target_pts, source_pts, noise_bound, min_inlier_num, tran_mat, status, info, launches);
    });
    // a hard graph can take hundreds of MiB of search stacks: do not keep them on the context (the stream has drained)
    if (ctx && ctx->tm_srch_buf.bytes > kTmKeepBytes) ctx->tm_srch_buf.release();
    return rc;
}

// ================================================================================================
// The baseline registrations (CRegistration::omp_ndt, omp_gicp): what both share on the host
// ================================================================================================
// the temporary bytes of sort_runs over n keys
static int sort_runs_bytes(mulls_ctx *ctx, int n, size_t &bytes) {
    size_t cub_sort = 0, cub_rle = 0, cub_scan = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint32_t *)nullptr,
                                       (uint32_t *)nullptr, std::max(n, 1)));
    CK(cub::DeviceRunLengthEncode::Encode(nullptr, cub_rle, (uint64_t *)nullptr, (uint64_t *)nullptr, (int *)nullptr,
                                          (int *)nullptr, std::max(n, 1)));
    CK(cub::DeviceScan::ExclusiveSum(nullptr, cub_scan, (int *)nullptr, (int *)nullptr, std::max(n, 1)));
    bytes = std::max(cub_sort, std::max(cub_rle, cub_scan));
    return MULLS_OK;
}
// keys ka with values va (the point indices) sorted stably into kb / vb, then the runs of equal keys: uk the run keys
// (ascending), cnt the run lengths, off their exclusive prefix sum, *nr the run count
static int sort_runs(mulls_ctx *ctx, void *d_cub, size_t cub_bytes, int n, uint64_t *ka, uint64_t *kb, uint32_t *va,
                     uint32_t *vb, uint64_t *uk, int *cnt, int *off, int *nr, cudaStream_t st) {
    size_t b = cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(d_cub, b, ka, kb, va, vb, n, 0, 64, st));
    CK(cudaMemsetAsync(cnt, 0, n * 4ull, st));
    b = cub_bytes;
    CK(cub::DeviceRunLengthEncode::Encode(d_cub, b, kb, uk, cnt, nr, n, st));
    b = cub_bytes;
    CK(cub::DeviceScan::ExclusiveSum(d_cub, b, cnt, off, n, st));
    return MULLS_OK;
}
// the full-pyramid grid of finite points (the rows the ingest takes): what getFitnessScore and the k-nearest
// covariances search
static int ingest_points(mulls_ctx *ctx, const std::vector<float4> &pts, DeviceArrays &A, uint64_t &launches) {
    std::vector<float> rows(pts.size() * 12, 0.f);
    for (size_t i = 0; i < pts.size(); ++i) rows[12 * i] = pts[i].x, rows[12 * i + 1] = pts[i].y, rows[12 * i + 2] = pts[i].z;
    int n_in = 0;
    mulls_cloud_view cv{rows.data(), pts.size()};
    return ingest_cloud(ctx, cv, false, 0.f, true, true, A, n_in, launches);
}
// the host's share of the epilogue: the mean of the n distances d2 that count (DBL_MAX when none does), Trans1_2 and the code
static void baseline_score(const float *d2, int n, const float T[12], const double *guess, bool moved, float fitness_thre,
                           double trans[16], int &code, double &fitness) {
    fitness = DBL_MAX;
    double sum = 0.0;
    int cnt = 0;
    for (int i = 0; i < n; ++i)
        if (d2[i] >= 0.f) sum += (double)d2[i], ++cnt;
    if (cnt) fitness = sum / cnt;
    ndt_epilogue(T, guess, moved, trans);
    code = fitness > (double)fitness_thre ? -3 : 1;
}
// the epilogue: getFitnessScore (the exact unbounded nearest target of every moved source point, summed in index
// order; DBL_MAX when nothing counts) over the target's grid A (NULL: no target), Trans1_2 and the code
static int baseline_finish(mulls_ctx *ctx, const DeviceArrays *A, const float4 *d_s, int ns, float *d_d2, const float T[12],
                           const double *guess, bool moved, float fitness_thre, double trans[16], int &code, double &fitness,
                           uint64_t &launches) {
    cudaStream_t st = ctx->stream;
    std::vector<float> d2;
    if (A && ns > 0) {
        NdtEvalConst E;
        std::memcpy(E.T, T, sizeof(E.T));
        k_ndt_fitness<<<(unsigned)ceil_div(ns, 128), 128, 0, st>>>(*A, d_s, ns, E, d_d2);
        launches += 1;
        d2.resize(ns);
        CK(cudaMemcpyAsync(d2.data(), d_d2, ns * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    baseline_score(d2.data(), (int)d2.size(), T, guess, moved, fitness_thre, trans, code, fitness);
    return MULLS_OK;
}

// ================================================================================================
// NDT registration (CRegistration::omp_ndt, cregistration.hpp:945-1021, DIRECT7 or KDTREE): ndt_core.cuh, kernels_ndt.cuh
// ================================================================================================
enum class NdtSearch { direct7, kdtree };
// the neighbour list entries a KDTREE call starts with: most points have fewer; a call whose longest list is longer
// grows them once, in its first evaluation (tests/test_ndt_kdtree.py's dense_cube scene goes through that path)
constexpr int kNdtKdListCap = 8;

static bool ndt_args_ok(mulls_cloud_view tv, mulls_cloud_view sv, float resolution, const double *guess, const double *tbound,
                        const double *sbound, const mulls_ndt_result *out, const mulls_ndt_iter *trace, int trace_cap) {
    return out && guess && tbound && sbound && (!tv.n || tv.aos48) && (!sv.n || sv.aos48) && resolution > 0.f &&
           (trace_cap <= 0 || trace);
}

// the arguments are checked (ndt_args_ok)
static int ndt_impl(mulls_ctx *ctx, const char *fn, mulls_cloud_view tv, mulls_cloud_view sv, float resolution, NdtSearch search,
                    const double *guess, int apply_filter, float fitness_thre, const double *tbound, const double *sbound,
                    mulls_ndt_result *out, mulls_ndt_iter *trace, int trace_cap, uint64_t &launches) {
    int rc;
    if ((rc = check_capacity(ctx, tv.n, fn)) != MULLS_OK) return rc;
    if (sv.n > ctx->max_src) {
        ctx->err = std::string(fn) + ": " + std::to_string(sv.n) + " source points exceed max_src_pts of the context";
        return MULLS_E_CAPACITY;
    }
    const bool kd = search == NdtSearch::kdtree;
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(tv.aos48, tv.n, sv.aos48, sv.n, guess, apply_filter, tbound, sbound, tgt, src, moved);
    const NdtGrid g = ndt_grid_from(tgt, resolution);
    const int nt = (int)tgt.size(), ns = (int)src.size(), tiles = (int)ceil_div((size_t)ns, kNdtTile);
    cudaStream_t st = ctx->stream;
    size_t cub_bytes = 0;
    if ((rc = sort_runs_bytes(ctx, nt, cub_bytes)) != MULLS_OK) return rc;
    float4 *d_t, *d_s, *d_cent, *d_kpts;
    uint64_t *d_ka, *d_kb, *d_uk;
    uint32_t *d_va, *d_vb;
    int *d_cnt, *d_off, *d_nr, *d_ncnt;
    NdtLeaf *d_lv;
    double *d_ts, *d_out;
    float *d_d2;
    void *d_cub;
    ScratchLayout L;
    L.take(d_t, nt), L.take(d_s, ns), L.take(d_ka, nt), L.take(d_kb, nt), L.take(d_va, nt), L.take(d_vb, nt), L.take(d_uk, nt);
    L.take(d_cnt, nt), L.take(d_off, nt), L.take(d_nr, 1), L.take(d_lv, nt), L.take(d_ts, (size_t)tiles * kNdtTerms);
    L.take(d_out, kNdtTerms), L.take(d_d2, ns), L.take_bytes(d_cub, cub_bytes);
    if (kd) L.take(d_cent, nt), L.take(d_kpts, nt), L.take(d_ncnt, (size_t)ns + 1);
    if ((rc = L.grow(ctx, ctx->ndt_buf)) != MULLS_OK) return rc;
    if (nt) CK(cudaMemcpyAsync(d_t, tgt.data(), nt * sizeof(float4), cudaMemcpyHostToDevice, st));
    if (ns) CK(cudaMemcpyAsync(d_s, src.data(), ns * sizeof(float4), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_nr, 0, sizeof(int), st));
    if (g.ok) { // the leaves (N1)
        k_ndt_keys<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, nt, g, d_ka, d_va);
        if ((rc = sort_runs(ctx, d_cub, cub_bytes, nt, d_ka, d_kb, d_va, d_vb, d_uk, d_cnt, d_off, d_nr, st)) != MULLS_OK) return rc;
        k_ndt_leaves<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, d_vb, d_off, d_cnt, d_nr, d_lv);
        launches += 2;
        if (kd) { // the searchable centroids in the order of their own cells (K1)
            k_ndt_kd_centroids<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, d_vb, d_off, d_cnt, d_nr, nt,
                                                                                                g, d_cent, d_ka, d_va);
            size_t b = cub_bytes;
            CK(cub::DeviceRadixSort::SortPairs(d_cub, b, d_ka, d_kb, d_va, d_vb, nt, 0, 64, st));
            k_ndt_kd_pack<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_kb, d_vb, d_cent, nt, d_kpts);
            launches += 2;
        }
    }
    NdtEvalConst E;
    {
        double d1, d2;
        ndt_gauss(resolution, d1, d2);
        E.gauss_d1 = d1, E.gauss_d2 = (float)d2;
    }
    NdtEvalArgs EA{d_s, ns, g, d_uk, d_lv, d_nr, d_ts};
    // KDTREE: the lists live in their own buffer, so that growing it leaves the leaf tables in place
    NdtKdArgs KA{d_s, ns, g, ndt_kd_r2(resolution), ndt_kd_probe_radius(resolution), d_kb, d_kpts, nt, 0, nullptr,
                 d_ncnt, d_ncnt + ns};
    auto kd_lists = [&](int cap) {
        const int r = grow_scratch(ctx, ctx->ndt_kd_buf, (size_t)cap * std::max(ns, 1) * sizeof(int2));
        if (r == MULLS_OK) KA.cap = cap, KA.list = (int2 *)ctx->ndt_kd_buf.p;
        return r;
    };
    if (kd && g.ok && ns > 0 && (rc = kd_lists(kNdtKdListCap)) != MULLS_OK) return rc;
    int err = MULLS_OK;
    auto eval = [&](const double p[6], const float T[12], double r[kNdtTerms]) {
        for (int c = 0; c < kNdtTerms; ++c) r[c] = 0.0;
        if (err != MULLS_OK || ns == 0 || (kd && !g.ok)) return; // K4: no centroids, no neighbours
        std::memcpy(E.T, T, sizeof(E.T));
        ndt_angle_tables(p, E);
        // KDTREE: a point with more neighbours than the lists hold makes the host grow them to the longest list and
        // evaluate again; the result does not depend on the capacity
        for (;;) {
            int longest = 0;
            cudaError_t e = cudaSuccess;
            if (!kd) {
                k_ndt_eval<<<(unsigned)tiles, kNdtTile, 0, st>>>(EA, E);
                launches += 1;
            } else {
                e = cudaMemsetAsync(KA.max_count, 0, sizeof(int), st);
                k_ndt_kd_search<<<(unsigned)tiles, kNdtTile, 0, st>>>(KA, E);
                const NdtKdEvalArgs KE{d_s, ns, KA.cap, KA.list, KA.count, d_lv, d_ts};
                k_ndt_eval_kd<<<(unsigned)tiles, kNdtTile, 0, st>>>(KE, E);
                launches += 2;
            }
            k_ndt_tiles<<<1, 64, 0, st>>>(d_ts, tiles, d_out);
            launches += 1;
            if (e == cudaSuccess) e = cudaMemcpyAsync(r, d_out, kNdtTerms * sizeof(double), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess && kd) e = cudaMemcpyAsync(&longest, KA.max_count, sizeof(int), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) {
                ctx->err = std::string(fn) + ": " + cudaGetErrorString(e);
                err = MULLS_E_CUDA;
                return;
            }
            if (longest <= KA.cap) return;
            if ((err = kd_lists(longest)) != MULLS_OK) return;
        }
    };
    std::vector<NdtIter> tr(trace_cap > 0 ? trace_cap : 0);
    float T[12];
    int converged = 0;
    const int iters = ndt_walk(eval, T, converged, tr.data(), (int)tr.size());
    if (err != MULLS_OK) return err;
    DeviceArrays A;
    const bool fit = nt > 0 && ns > 0;
    if (fit && (rc = ingest_points(ctx, tgt, A, launches)) != MULLS_OK) return rc;
    if ((rc = baseline_finish(ctx, fit ? &A : nullptr, d_s, ns, d_d2, T, guess, moved, fitness_thre, out->trans, out->code,
                              out->fitness, launches)) != MULLS_OK)
        return rc;
    out->iterations = iters;
    out->converged = converged;
    out->n_target = nt;
    out->n_source = ns;
    for (int i = 0; i < std::min(iters, trace_cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].p[c] = tr[i].p[c];
        trace[i].step = tr[i].step, trace[i].score = tr[i].score, trace[i].reversed = tr[i].reversed;
    }
    return MULLS_OK;
}
int mulls_omp_ndt(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, float ndt_resolution, int use_direct_search,
                  const double initial_guess[16], int apply_intersection_filter, float fitness_score_thre,
                  const double target_bound[6], const double source_bound[6], mulls_ndt_result *out, mulls_ndt_iter *trace,
                  int trace_cap) {
    return front_call(ctx, [&](uint64_t &launches) {
        if (!ndt_args_ok(target, source, ndt_resolution, initial_guess, target_bound, source_bound, out, trace, trace_cap))
            return (int)MULLS_E_ARG;
        if (!use_direct_search) {
            ctx->err = "mulls_omp_ndt: only the DIRECT7 neighbour search runs on the device (KDTREE: mulls_omp_ndt_kdtree)";
            return (int)MULLS_E_UNSUPPORTED;
        }
        return ndt_impl(ctx, "mulls_omp_ndt", target, source, ndt_resolution, NdtSearch::direct7, initial_guess,
                        apply_intersection_filter, fitness_score_thre, target_bound, source_bound, out, trace, trace_cap, launches);
    });
}
int mulls_omp_ndt_kdtree(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, float ndt_resolution,
                         const double initial_guess[16], int apply_intersection_filter, float fitness_score_thre,
                         const double target_bound[6], const double source_bound[6], mulls_ndt_result *out,
                         mulls_ndt_iter *trace, int trace_cap) {
    return front_call(ctx, [&](uint64_t &launches) {
        if (!ndt_args_ok(target, source, ndt_resolution, initial_guess, target_bound, source_bound, out, trace, trace_cap))
            return (int)MULLS_E_ARG;
        return ndt_impl(ctx, "mulls_omp_ndt_kdtree", target, source, ndt_resolution, NdtSearch::kdtree, initial_guess,
                        apply_intersection_filter, fitness_score_thre, target_bound, source_bound, out, trace, trace_cap, launches);
    });
}

// A batch of NDT registrations with shared parameters (mulls_omp_ndt_batch): pair i computes what ndt_impl computes for
// it alone. The prologues run on the host's worker pool; the leaves of all targets come from one sort
// (k_ndt_keys_batch); every iteration evaluates all live pairs in one launch and downloads their 43 terms at once;
// one ingest of all filtered targets and one fitness launch end the batch.
struct NdtBatchPair {
    mulls_cloud_view tv, sv;
    const double *guess, *tbound, *sbound;
    int apply_filter;
    float resolution;
    std::vector<float4> tgt, src;
    bool moved = false;
    NdtGrid g;
    static void prologue(void *arg) {
        NdtBatchPair &b = *(NdtBatchPair *)arg;
        ndt_prologue(b.tv.aos48, b.tv.n, b.sv.aos48, b.sv.n, b.guess, b.apply_filter, b.tbound, b.sbound, b.tgt, b.src, b.moved);
        b.g = ndt_grid_from(b.tgt, b.resolution);
    }
};
static int ndt_batch_impl(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *tv, const mulls_cloud_view *sv,
                          float resolution, int use_direct_search, const double *guesses, int apply_filter, float fitness_thre,
                          const double *tbounds, const double *sbounds, mulls_ndt_result *out, mulls_ndt_iter *trace,
                          int trace_cap, uint64_t &launches) {
    if (!out || !tv || !sv || !guesses || !tbounds || !sbounds || n_pairs == 0 || !(resolution > 0.f) || (trace_cap > 0 && !trace))
        return MULLS_E_ARG;
    const std::string fn = "mulls_omp_ndt_batch";
    for (size_t p = 0; p < n_pairs; ++p)
        if ((tv[p].n && !tv[p].aos48) || (sv[p].n && !sv[p].aos48)) {
            ctx->err = fn + ": pair " + std::to_string(p) + ": NULL rows with n > 0";
            return MULLS_E_ARG;
        }
    if (!use_direct_search) {
        ctx->err = fn + ": only the DIRECT7 neighbour search runs on the device";
        return MULLS_E_UNSUPPORTED;
    }
    if (n_pairs > ctx->max_pairs) {
        ctx->err = fn + ": " + std::to_string(n_pairs) + " pairs exceed max_pairs of the context";
        return MULLS_E_CAPACITY;
    }
    for (size_t p = 0; p < n_pairs; ++p)
        if (tv[p].n > ctx->max_tgt || sv[p].n > ctx->max_src) {
            ctx->err = fn + ": pair " + std::to_string(p) + ": " + std::to_string(tv[p].n) + " target / " +
                       std::to_string(sv[p].n) + " source points exceed max_tgt_pts / max_src_pts of the context";
            return MULLS_E_CAPACITY;
        }
    const int P = (int)n_pairs;
    std::vector<NdtBatchPair> B(P);
    { // the prologues on the worker pool
        PackPool &pool = PackPool::get();
        pool.ensure_workers(0);
        std::atomic<int> pending(P);
        std::vector<PackJob> jobs(P);
        for (int p = 0; p < P; ++p) {
            NdtBatchPair &b = B[p];
            b.tv = tv[p], b.sv = sv[p], b.guess = guesses + 16 * p, b.tbound = tbounds + 6 * p, b.sbound = sbounds + 6 * p;
            b.apply_filter = apply_filter, b.resolution = resolution;
            jobs[p].pending = &pending;
            jobs[p].task = &NdtBatchPair::prologue;
            jobs[p].arg = &b;
        }
        pool.submit(jobs);
        pool.help_until_done(pending);
    }
    // the pair table: sources of every pair, targets of the pairs with leaves, tiles of the evaluation
    std::vector<NdtPairDev> pd(P);
    std::vector<int> tile_off(P + 1, 0);
    int nt_leaf = 0, ns_all = 0;
    for (int p = 0; p < P; ++p) {
        NdtPairDev &d = pd[p];
        d.g = B[p].g;
        d.src_off = ns_all, d.n_src = (int)B[p].src.size();
        d.tgt_off = nt_leaf, d.n_tgt = d.g.ok ? (int)B[p].tgt.size() : 0;
        d.leaf_begin = d.leaf_end = 0;
        ns_all += d.n_src, nt_leaf += d.n_tgt;
        tile_off[p + 1] = tile_off[p] + (int)ceil_div((size_t)d.n_src, kNdtTile);
    }
    const int tiles_all = tile_off[P];
    cudaStream_t st = ctx->stream;
    size_t cub_bytes = 0;
    int rc;
    if ((rc = sort_runs_bytes(ctx, nt_leaf, cub_bytes)) != MULLS_OK) return rc;
    NdtPairDev *d_pd;
    NdtLiveSlot *d_sl;
    float *d_T, *d_d2;
    float4 *d_t, *d_s;
    uint64_t *d_ka, *d_kb, *d_uk;
    uint32_t *d_va, *d_vb;
    int *d_cnt, *d_off, *d_nr;
    NdtLeaf *d_lv;
    double *d_ts, *d_out;
    void *d_cub;
    ScratchLayout L;
    L.take(d_pd, P), L.take(d_sl, P), L.take(d_T, P * 12), L.take(d_t, nt_leaf), L.take(d_s, ns_all), L.take(d_ka, nt_leaf);
    L.take(d_kb, nt_leaf), L.take(d_va, nt_leaf), L.take(d_vb, nt_leaf), L.take(d_uk, nt_leaf), L.take(d_cnt, nt_leaf);
    L.take(d_off, nt_leaf), L.take(d_nr, 1), L.take(d_lv, nt_leaf), L.take(d_ts, (size_t)tiles_all * kNdtTerms);
    L.take(d_out, (size_t)P * kNdtTerms), L.take(d_d2, ns_all), L.take_bytes(d_cub, cub_bytes);
    if ((rc = L.grow(ctx, ctx->ndt_buf)) != MULLS_OK) return rc;
    for (int p = 0; p < P; ++p) {
        if (pd[p].n_tgt)
            CK(cudaMemcpyAsync(d_t + pd[p].tgt_off, B[p].tgt.data(), pd[p].n_tgt * sizeof(float4), cudaMemcpyHostToDevice, st));
        if (pd[p].n_src)
            CK(cudaMemcpyAsync(d_s + pd[p].src_off, B[p].src.data(), pd[p].n_src * sizeof(float4), cudaMemcpyHostToDevice, st));
    }
    CK(cudaMemcpyAsync(d_pd, pd.data(), P * sizeof(NdtPairDev), cudaMemcpyHostToDevice, st));
    if (nt_leaf) { // the leaves of every pair whose grid is ok (N1)
        k_ndt_keys_batch<<<(unsigned)ceil_div(nt_leaf, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, nt_leaf, d_pd, P, d_ka, d_va);
        if ((rc = sort_runs(ctx, d_cub, cub_bytes, nt_leaf, d_ka, d_kb, d_va, d_vb, d_uk, d_cnt, d_off, d_nr, st)) != MULLS_OK)
            return rc;
        k_ndt_leaves<<<(unsigned)ceil_div(nt_leaf, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, d_vb, d_off, d_cnt, d_nr, d_lv);
        k_ndt_leaf_ranges<<<(unsigned)ceil_div(P, 64), 64, 0, st>>>(d_uk, d_nr, d_pd, P);
        launches += 3;
    }
    // the walks in lockstep: each round evaluates every live pair with sources in one launch
    double gd1, gd2;
    ndt_gauss(resolution, gd1, gd2);
    std::vector<NdtWalk> W(P);
    std::vector<NdtIter> tr((size_t)P * (trace_cap > 0 ? trace_cap : 0));
    const int cap = trace_cap > 0 ? trace_cap : 0;
    std::vector<int> live(P), next;
    for (int p = 0; p < P; ++p) ndt_walk_start(W[p]), live[p] = p;
    std::vector<NdtLiveSlot> slots;
    std::vector<double> r;
    while (!live.empty()) {
        slots.clear();
        for (int p : live) {
            for (int c = 0; c < kNdtTerms; ++c) W[p].r[c] = 0.0;
            if (pd[p].n_src == 0) continue;
            NdtLiveSlot s;
            std::memcpy(s.E.T, W[p].T, sizeof(s.E.T));
            ndt_angle_tables(W[p].q, s.E);
            s.E.gauss_d1 = gd1, s.E.gauss_d2 = (float)gd2;
            s.pair = p;
            s.tile_begin = slots.empty() ? 0 : slots.back().tile_end;
            s.tile_end = s.tile_begin + (tile_off[p + 1] - tile_off[p]);
            slots.push_back(s);
        }
        if (!slots.empty()) {
            const int ns = (int)slots.size();
            CK(cudaMemcpyAsync(d_sl, slots.data(), ns * sizeof(NdtLiveSlot), cudaMemcpyHostToDevice, st));
            NdtBatchEvalArgs EA{d_s, d_pd, d_uk, d_lv, d_sl, ns, d_ts};
            k_ndt_eval_batch<<<(unsigned)slots.back().tile_end, kNdtTile, 0, st>>>(EA);
            k_ndt_tiles_batch<<<(unsigned)ns, 64, 0, st>>>(d_ts, d_sl, d_out);
            launches += 2;
            r.resize((size_t)ns * kNdtTerms);
            CK(cudaMemcpyAsync(r.data(), d_out, r.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (int k = 0; k < ns; ++k) std::memcpy(W[slots[k].pair].r, &r[(size_t)k * kNdtTerms], kNdtTerms * sizeof(double));
        }
        next.clear();
        for (int p : live)
            if (ndt_walk_advance(W[p], tr.data() + (size_t)p * cap, cap)) next.push_back(p);
        live.swap(next);
    }
    // the fitness: one ingest of the filtered targets that need it, one search over all sources
    std::vector<float> d2(ns_all, -1.f);
    std::vector<std::vector<float>> rows(P);
    std::vector<mulls_cloud_view> views(P, mulls_cloud_view{nullptr, 0});
    bool any_fit = false;
    for (int p = 0; p < P; ++p) {
        if (B[p].tgt.empty() || B[p].src.empty()) continue;
        const std::vector<float4> &t = B[p].tgt;
        rows[p].assign(t.size() * 12, 0.f);
        for (size_t i = 0; i < t.size(); ++i) rows[p][12 * i] = t[i].x, rows[p][12 * i + 1] = t[i].y, rows[p][12 * i + 2] = t[i].z;
        views[p] = mulls_cloud_view{rows[p].data(), t.size()};
        any_fit = true;
    }
    if (any_fit) {
        DeviceArrays A;
        int n_in = 0;
        if ((rc = ingest_clouds(ctx, P, views.data(), false, 0.f, true, true, A, n_in, launches)) != MULLS_OK) return rc;
        std::vector<float> T(12 * P);
        for (int p = 0; p < P; ++p) std::memcpy(&T[12 * p], W[p].T, 12 * sizeof(float));
        CK(cudaMemcpyAsync(d_T, T.data(), T.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        k_ndt_fitness_batch<<<(unsigned)ceil_div(ns_all, 128), 128, 0, st>>>(A, d_s, ns_all, d_pd, P, d_T, d_d2);
        launches += 1;
        CK(cudaMemcpyAsync(d2.data(), d_d2, ns_all * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    for (int p = 0; p < P; ++p) {
        mulls_ndt_result &o = out[p];
        const bool fit = views[p].n > 0;
        baseline_score(d2.data() + pd[p].src_off, fit ? pd[p].n_src : 0, W[p].T, B[p].guess, B[p].moved, fitness_thre, o.trans,
                       o.code, o.fitness);
        o.iterations = W[p].nr;
        o.converged = W[p].converged;
        o.n_target = (int)B[p].tgt.size();
        o.n_source = pd[p].n_src;
        for (int i = 0; i < std::min(W[p].nr, cap); ++i) {
            const NdtIter &t = tr[(size_t)p * cap + i];
            mulls_ndt_iter &d = trace[(size_t)p * cap + i];
            for (int c = 0; c < 6; ++c) d.p[c] = t.p[c];
            d.step = t.step, d.score = t.score, d.reversed = t.reversed;
        }
    }
    return MULLS_OK;
}
int mulls_omp_ndt_batch(mulls_ctx *ctx, size_t n_pairs, const mulls_cloud_view *targets, const mulls_cloud_view *sources,
                        float ndt_resolution, int use_direct_search, const double *initial_guesses, int apply_intersection_filter,
                        float fitness_score_thre, const double *target_bounds, const double *source_bounds, mulls_ndt_result *out,
                        mulls_ndt_iter *trace, int trace_cap) {
    return front_call(ctx, [&](uint64_t &launches) {
        return ndt_batch_impl(ctx, n_pairs, targets, sources, ndt_resolution, use_direct_search, initial_guesses,
                              apply_intersection_filter, fitness_score_thre, target_bounds, source_bounds, out, trace, trace_cap,
                              launches);
    });
}

// ================================================================================================
// Voxelized GICP registration (CRegistration::omp_gicp, cregistration.hpp:1024-1098, FastVGICP): gicp_core.cuh,
// kernels_gicp.cuh
// ================================================================================================
static int gicp_impl(mulls_ctx *ctx, mulls_cloud_view tv, mulls_cloud_view sv, int using_voxel_gicp, float voxel_size,
                     const double *guess, int apply_filter, float fitness_thre, const double *tbound, const double *sbound,
                     mulls_gicp_result *out, mulls_gicp_iter *trace, int trace_cap, uint64_t &launches) {
    if (!out || !guess || !tbound || !sbound || (tv.n && !tv.aos48) || (sv.n && !sv.aos48) || !(voxel_size > 0.f) ||
        (trace_cap > 0 && !trace))
        return MULLS_E_ARG;
    const char *fn = "mulls_omp_gicp";
    if (!using_voxel_gicp) {
        ctx->err = std::string(fn) + ": only the voxelized GICP (FastVGICP) runs on the device";
        return MULLS_E_UNSUPPORTED;
    }
    int rc;
    // both clouds go through the ingest (their k-nearest covariances)
    if ((rc = check_capacity(ctx, tv.n, fn)) != MULLS_OK || (rc = check_capacity(ctx, sv.n, fn)) != MULLS_OK) return rc;
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(tv.aos48, tv.n, sv.aos48, sv.n, guess, apply_filter, tbound, sbound, tgt, src, moved);
    gicp_keep_finite(src); // (the prologue keeps the target's finite points only)
    const int nt = (int)tgt.size(), ns = (int)src.size(), tiles = (int)ceil_div((size_t)ns, kNdtTile);
    if (nt < kGicpK || ns < kGicpK) {
        ctx->err = std::string(fn) + ": " + std::to_string(nt) + " target and " + std::to_string(ns) +
                   " source points after the prologue; the covariances need " + std::to_string(kGicpK) + " in each";
        return MULLS_E_UNSUPPORTED;
    }
    { // C2: the voxel coordinate is monotonic in each axis, so the target's bounds bound every key
        float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
        for (const float4 &p : tgt) {
            const float v[3] = {p.x, p.y, p.z};
            for (int d = 0; d < 3; ++d) mn[d] = std::min(mn[d], v[d]), mx[d] = std::max(mx[d], v[d]);
        }
        uint64_t k;
        if (!gicp_key_of(mn[0], mn[1], mn[2], voxel_size, k) || !gicp_key_of(mx[0], mx[1], mx[2], voxel_size, k)) {
            ctx->err = std::string(fn) + ": the target's voxel coordinates exceed " + std::to_string(kGicpCoordBits) + " bits";
            return MULLS_E_UNSUPPORTED;
        }
    }
    cudaStream_t st = ctx->stream;
    size_t cub_bytes = 0;
    if ((rc = sort_runs_bytes(ctx, nt, cub_bytes)) != MULLS_OK) return rc;
    float4 *d_t, *d_s;
    float *d_ct, *d_cs, *d_d2; // covariances: 9 floats per point
    uint64_t *d_ka, *d_kb, *d_uk;
    uint32_t *d_va, *d_vb;
    int *d_cnt, *d_off, *d_nr;
    GicpVoxel *d_vx;
    double *d_ts, *d_out;
    void *d_cub;
    ScratchLayout L;
    L.take(d_t, nt), L.take(d_s, ns), L.take(d_ct, nt * 9ull), L.take(d_cs, ns * 9ull), L.take(d_ka, nt), L.take(d_kb, nt);
    L.take(d_va, nt), L.take(d_vb, nt), L.take(d_uk, nt), L.take(d_cnt, nt), L.take(d_off, nt), L.take(d_nr, 1), L.take(d_vx, nt);
    L.take(d_ts, (size_t)tiles * kGicpTerms), L.take(d_out, kGicpTerms), L.take(d_d2, ns), L.take_bytes(d_cub, cub_bytes);
    if ((rc = L.grow(ctx, ctx->gicp_buf)) != MULLS_OK) return rc;
    CK(cudaMemcpyAsync(d_t, tgt.data(), nt * sizeof(float4), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_s, src.data(), ns * sizeof(float4), cudaMemcpyHostToDevice, st));
    // G1: the source's covariances, then the target's (its grid stays for the fitness)
    DeviceArrays A;
    if ((rc = ingest_points(ctx, src, A, launches)) != MULLS_OK) return rc;
    k_gicp_cov<<<(unsigned)ceil_div(ns, kGicpCovBlock), kGicpCovBlock, 0, st>>>(A, d_cs);
    k_gicp_plane<<<(unsigned)ceil_div(ns, kGicpCovBlock), kGicpCovBlock, 0, st>>>(d_cs, ns);
    if ((rc = ingest_points(ctx, tgt, A, launches)) != MULLS_OK) return rc;
    k_gicp_cov<<<(unsigned)ceil_div(nt, kGicpCovBlock), kGicpCovBlock, 0, st>>>(A, d_ct);
    k_gicp_plane<<<(unsigned)ceil_div(nt, kGicpCovBlock), kGicpCovBlock, 0, st>>>(d_ct, nt);
    // G2: the voxels
    k_gicp_keys<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, nt, voxel_size, d_ka, d_va);
    if ((rc = sort_runs(ctx, d_cub, cub_bytes, nt, d_ka, d_kb, d_va, d_vb, d_uk, d_cnt, d_off, d_nr, st)) != MULLS_OK) return rc;
    k_gicp_voxels<<<(unsigned)ceil_div(nt, kNdtKeyBlock), kNdtKeyBlock, 0, st>>>(d_t, d_ct, d_vb, d_off, d_cnt, d_nr, d_vx);
    launches += 6;
    GicpEvalArgs EA{d_s, d_cs, ns, voxel_size, d_uk, d_vx, d_nr, d_ts};
    NdtEvalConst E;
    int err = MULLS_OK;
    auto eval = [&](const float T[12], double r[kGicpTerms]) {
        for (int c = 0; c < kGicpTerms; ++c) r[c] = 0.0;
        if (err != MULLS_OK) return;
        std::memcpy(E.T, T, sizeof(E.T));
        k_gicp_eval<<<(unsigned)tiles, kNdtTile, 0, st>>>(EA, E);
        k_gicp_tiles<<<1, 32, 0, st>>>(d_ts, tiles, d_out);
        launches += 2;
        cudaError_t e = cudaMemcpyAsync(r, d_out, kGicpTerms * sizeof(double), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            ctx->err = std::string(fn) + ": " + cudaGetErrorString(e);
            err = MULLS_E_CUDA;
        }
    };
    std::vector<GicpIter> tr(trace_cap > 0 ? trace_cap : 0);
    float T[12];
    int converged = 0;
    const int iters = gicp_walk(eval, T, out->x0, converged, tr.data(), (int)tr.size());
    if (err != MULLS_OK) return err;
    if ((rc = baseline_finish(ctx, &A, d_s, ns, d_d2, T, guess, moved, fitness_thre, out->trans, out->code, out->fitness,
                              launches)) != MULLS_OK)
        return rc;
    out->iterations = iters;
    out->converged = converged;
    out->n_target = nt;
    out->n_source = ns;
    for (int i = 0; i < std::min(iters, trace_cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].x[c] = tr[i].x[c], trace[i].delta[c] = tr[i].delta[c];
        trace[i].n_corr = tr[i].n_corr, trace[i].random_step = tr[i].random;
    }
    return MULLS_OK;
}
int mulls_omp_gicp(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, int using_voxel_gicp, float voxel_size,
                   const double initial_guess[16], int apply_intersection_filter, float fitness_score_thre,
                   const double target_bound[6], const double source_bound[6], mulls_gicp_result *out, mulls_gicp_iter *trace,
                   int trace_cap) {
    return front_call(ctx, [&](uint64_t &launches) {
        return gicp_impl(ctx, target, source, using_voxel_gicp, voxel_size, initial_guess, apply_intersection_filter,
                         fitness_score_thre, target_bound, source_bound, out, trace, trace_cap, launches);
    });
}

// ================================================================================================
// Point-wise GICP registration (CRegistration::omp_gicp without using_voxel_gicp, GeneralizedIterativeClosestPoint with
// PCL's BFGS): gicp_pcl_core.cuh, kernels_gicp_pcl.cuh
// ================================================================================================
static int gicp_pcl_impl(mulls_ctx *ctx, mulls_cloud_view tv, mulls_cloud_view sv, int max_iter_num, const double *guess,
                         int apply_filter, float fitness_thre, const double *tbound, const double *sbound,
                         mulls_gicp_pcl_result *out, mulls_gicp_pcl_iter *trace, int trace_cap, uint64_t &launches) {
    if (!out || !guess || !tbound || !sbound || (tv.n && !tv.aos48) || (sv.n && !sv.aos48) || (trace_cap > 0 && !trace))
        return MULLS_E_ARG;
    const char *fn = "mulls_omp_gicp_pcl";
    int rc;
    // both clouds go through the ingest (their k-nearest covariances)
    if ((rc = check_capacity(ctx, tv.n, fn)) != MULLS_OK || (rc = check_capacity(ctx, sv.n, fn)) != MULLS_OK) return rc;
    std::vector<float4> tgt, src;
    bool moved = false;
    ndt_prologue(tv.aos48, tv.n, sv.aos48, sv.n, guess, apply_filter, tbound, sbound, tgt, src, moved);
    gicp_keep_finite(src); // (the prologue keeps the target's finite points only)
    const int nt = (int)tgt.size(), ns = (int)src.size();
    if (nt < kGicpK || ns < kGicpK) { // P8
        ctx->err = std::string(fn) + ": " + std::to_string(nt) + " target and " + std::to_string(ns) +
                   " source points after the prologue; the covariances need " + std::to_string(kGicpK) + " in each";
        return MULLS_E_UNSUPPORTED;
    }
    cudaStream_t st = ctx->stream;
    const thrust::counting_iterator<int> iota(0);
    size_t cub_bytes = 0;
    CK(cub::DeviceSelect::Flagged(nullptr, cub_bytes, iota, (const int *)nullptr, (int *)nullptr, (int *)nullptr, ns));
    const int max_tiles = (int)ceil_div((size_t)ns, kNdtTile);
    float4 *d_t, *d_s;
    double *d_ct, *d_cs, *d_ts, *d_out; // covariances: 9 doubles per point
    int *d_flag, *d_tix, *d_list, *d_m;
    float *d_maha, *d_d2;
    void *d_cub;
    ScratchLayout L;
    L.take(d_t, nt), L.take(d_s, ns), L.take(d_ct, nt * 9ull), L.take(d_cs, ns * 9ull), L.take(d_flag, ns), L.take(d_tix, ns);
    L.take(d_list, ns), L.take(d_m, 1), L.take(d_maha, ns * 9ull), L.take(d_ts, (size_t)max_tiles * kGicpPclMaxTerms);
    L.take(d_out, kGicpPclMaxTerms), L.take(d_d2, ns), L.take_bytes(d_cub, cub_bytes);
    if ((rc = L.grow(ctx, ctx->gicp_pcl_buf)) != MULLS_OK) return rc;
    CK(cudaMemcpyAsync(d_t, tgt.data(), nt * sizeof(float4), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_s, src.data(), ns * sizeof(float4), cudaMemcpyHostToDevice, st));
    // P3: the source's covariances, then the target's (its grid stays for the matches and the fitness)
    DeviceArrays A;
    if ((rc = ingest_points(ctx, src, A, launches)) != MULLS_OK) return rc;
    k_gicp_pcl_cov<<<(unsigned)ceil_div(ns, kGicpCovBlock), kGicpCovBlock, 0, st>>>(A, d_cs);
    k_gicp_pcl_plane<<<(unsigned)ceil_div(ns, kGicpCovBlock), kGicpCovBlock, 0, st>>>(d_cs, ns);
    if ((rc = ingest_points(ctx, tgt, A, launches)) != MULLS_OK) return rc;
    k_gicp_pcl_cov<<<(unsigned)ceil_div(nt, kGicpCovBlock), kGicpCovBlock, 0, st>>>(A, d_ct);
    k_gicp_pcl_plane<<<(unsigned)ceil_div(nt, kGicpCovBlock), kGicpCovBlock, 0, st>>>(d_ct, nt);
    launches += 4;
    int err = MULLS_OK;
    auto fail = [&](cudaError_t e) {
        if (e == cudaSuccess || err != MULLS_OK) return;
        ctx->err = std::string(fn) + ": " + cudaGetErrorString(e);
        err = MULLS_E_CUDA;
    };
    int m = 0; // the current correspondences
    auto match = [&](const float T[12], const double R[9]) {
        if (err != MULLS_OK) return 0;
        GicpPclMatchConst MC;
        std::memcpy(MC.T, T, sizeof(MC.T));
        std::memcpy(MC.R, R, sizeof(MC.R));
        k_gicp_pcl_match<<<(unsigned)ceil_div(ns, 128), 128, 0, st>>>(A, d_s, ns, d_cs, d_ct, MC, d_flag, d_tix, d_maha);
        size_t b = cub_bytes;
        cudaError_t e = cub::DeviceSelect::Flagged(d_cub, b, iota, (const int *)d_flag, d_list, d_m, ns, st);
        launches += 2;
        if (e == cudaSuccess) e = cudaMemcpyAsync(&m, d_m, sizeof(int), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        fail(e);
        return err == MULLS_OK ? m : 0;
    };
    NdtEvalConst E;
    auto eval = [&](int method, const float T[12], double *r) {
        const int terms = gicp_pcl_terms(method);
        for (int c = 0; c < terms; ++c) r[c] = 0.0;
        if (err != MULLS_OK) return;
        std::memcpy(E.T, T, sizeof(E.T));
        const int tiles = (int)ceil_div((size_t)m, kNdtTile);
        const GicpPclEvalArgs EA{d_s, d_t, d_list, d_tix, d_maha, m, d_ts};
        if (method == kGicpPclF) k_gicp_pcl_eval<kGicpPclF><<<(unsigned)tiles, kNdtTile, 0, st>>>(EA, E);
        else if (method == kGicpPclDf) k_gicp_pcl_eval<kGicpPclDf><<<(unsigned)tiles, kNdtTile, 0, st>>>(EA, E);
        else k_gicp_pcl_eval<kGicpPclFdf><<<(unsigned)tiles, kNdtTile, 0, st>>>(EA, E);
        k_gicp_pcl_tiles<<<1, 32, 0, st>>>(d_ts, tiles, terms, d_out);
        launches += 2;
        cudaError_t e = cudaMemcpyAsync(r, d_out, terms * sizeof(double), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        fail(e);
    };
    std::vector<GicpPclIter> tr(trace_cap > 0 ? trace_cap : 0);
    float T[12];
    int converged = 0;
    const int iters = gicp_pcl_walk(max_iter_num, match, eval, T, converged, tr.data(), (int)tr.size());
    if (err != MULLS_OK) return err;
    if ((rc = baseline_finish(ctx, &A, d_s, ns, d_d2, T, guess, moved, fitness_thre, out->trans, out->code, out->fitness,
                              launches)) != MULLS_OK)
        return rc;
    out->iterations = iters;
    out->converged = converged;
    out->n_target = nt;
    out->n_source = ns;
    for (int i = 0; i < std::min(iters, trace_cap); ++i) {
        for (int c = 0; c < 6; ++c) trace[i].x[c] = tr[i].x[c];
        trace[i].delta = tr[i].delta, trace[i].n_corr = tr[i].n_corr, trace[i].inner_iterations = tr[i].inner;
        trace[i].status = tr[i].status, trace[i].evaluations = tr[i].evaluations;
    }
    return MULLS_OK;
}
int mulls_omp_gicp_pcl(mulls_ctx *ctx, mulls_cloud_view target, mulls_cloud_view source, int max_iter_num,
                       const double initial_guess[16], int apply_intersection_filter, float fitness_score_thre,
                       const double target_bound[6], const double source_bound[6], mulls_gicp_pcl_result *out,
                       mulls_gicp_pcl_iter *trace, int trace_cap) {
    return front_call(ctx, [&](uint64_t &launches) {
        return gicp_pcl_impl(ctx, target, source, max_iter_num, initial_guess, apply_intersection_filter, fitness_score_thre,
                             target_bound, source_bound, out, trace, trace_cap, launches);
    });
}

// ================================================================================================
// Device-resident local map (MapManager::update_local_map, src/map_manager.cpp:17-145)
// ================================================================================================
} // extern "C"

struct mulls_map {
    mulls_ctx *ctx = nullptr;
    size_t cap = 0;                      // rows per class buffer
    float4 *buf[2][kNumClasses] = {};    // the map, ping-pong
    float4 *mid[kNumClasses] = {};       // after append + transform + radius crop
    float4 *scan[kNumClasses] = {};      // the scan's down clouds of the running update
    uint8_t *drop[kNumClasses] = {};     // per scan point: removed by the dynamic filter
    int cur = 0;
    uint32_t n[kNumClasses] = {};
    double pose[16];
    double local_bound[6], bound[6];
    MapState *d_state = nullptr, *h_state = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    mulls_map_info last{};
    uint64_t epoch = 0; // bumped by every change of the content
};

namespace {
// Eigen::Matrix4d::inverse(): adjugate / determinant
void host_inverse4(const double *m, double *out) {
    double inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    for (int i = 0; i < 16; ++i) out[i] = inv[i] * (1.0 / det);
}
void host_mul4(const double *a, const double *b, double *out) { // sequential over k
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += a[4 * i + k] * b[4 * k + j];
            out[4 * i + j] = acc;
        }
}
void map_fill_info(const mulls_map *m, mulls_map_info *info) {
    *info = m->last;
    for (int i = 0; i < 16; ++i) info->pose_lo[i] = m->pose[i];
    for (int i = 0; i < 6; ++i) info->local_bound[i] = m->local_bound[i], info->bound[i] = m->bound[i];
    for (int c = 0; c < kNumClasses; ++c) info->n[c] = m->n[c];
    info->feature_point_num = (int)(m->n[0] + m->n[1] + m->n[2] + m->n[3] + m->n[4]);
}
} // namespace

extern "C" {

void mulls_map_default_params(mulls_map_params *p) { // include/pgo/map_manager.h:22-32
    std::memset(p, 0, sizeof(*p));
    p->local_map_radius = 80.f;
    p->max_num_pts = 20000;
    p->kept_vertex_num = 800;
    p->last_frame_reliable_radius = 60.f;
    p->map_based_dynamic_removal_on = 0;
    std::strcpy(p->used_feature_type, "111110");
    p->dynamic_removal_center_radius = 30.0f;
    p->dynamic_dist_thre_min = 0.3f;
    p->dynamic_dist_thre_max = 3.0f;
    p->near_dist_thre = 0.03f;
    p->recalculate_feature_on = 0;
    p->random_seed = 0;
}

void mulls_map_destroy(mulls_map *m) {
    if (!m) return;
    mulls_ctx *ctx = m->ctx;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->tree_map == m) ctx->tree_map = nullptr;
    for (int c = 0; c < kNumClasses; ++c) {
        cudaFree(m->buf[0][c]);
        cudaFree(m->buf[1][c]);
        cudaFree(m->mid[c]);
        cudaFree(m->scan[c]);
        cudaFree(m->drop[c]);
    }
    cudaFree(m->d_state);
    if (m->h_state) cudaFreeHost(m->h_state);
    if (m->ev0) cudaEventDestroy(m->ev0);
    if (m->ev1) cudaEventDestroy(m->ev1);
    delete m;
}

mulls_map *mulls_map_create(mulls_ctx *ctx, size_t max_pts_per_class) {
    if (!ctx || max_pts_per_class == 0 || max_pts_per_class >= (1ull << 31)) return nullptr;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return nullptr;
    mulls_map *m = new mulls_map();
    m->ctx = ctx;
    m->cap = max_pts_per_class;
    bool ok = true;
    const size_t bytes = max_pts_per_class * 48;
    for (int c = 0; c < kNumClasses && ok; ++c) {
        ok = ok && cudaMalloc((void **)&m->buf[0][c], bytes) == cudaSuccess;
        ok = ok && cudaMalloc((void **)&m->buf[1][c], bytes) == cudaSuccess;
        ok = ok && cudaMalloc((void **)&m->mid[c], bytes) == cudaSuccess;
        ok = ok && cudaMalloc((void **)&m->scan[c], bytes) == cudaSuccess;
        ok = ok && cudaMalloc((void **)&m->drop[c], max_pts_per_class) == cudaSuccess;
    }
    ok = ok && cudaMalloc((void **)&m->d_state, sizeof(MapState)) == cudaSuccess;
    ok = ok && cudaMallocHost((void **)&m->h_state, sizeof(MapState)) == cudaSuccess;
    ok = ok && cudaEventCreate(&m->ev0) == cudaSuccess && cudaEventCreate(&m->ev1) == cudaSuccess;
    if (!ok) {
        ctx->err = std::string("mulls_map_create: ") + cudaGetErrorString(cudaGetLastError());
        mulls_map_destroy(m);
        return nullptr;
    }
    const double big = 1.7976931348623157e308;
    for (int i = 0; i < 16; ++i) m->pose[i] = (i % 5 == 0) ? 1.0 : 0.0; // cloudblock_t starts at the identity pose
    for (int d = 0; d < 3; ++d) {
        m->local_bound[d] = m->bound[d] = big;
        m->local_bound[3 + d] = m->bound[3 + d] = -big;
    }
    return m;
}

int mulls_map_set(mulls_map *m, const mulls_cloud_view cls[MULLS_NUM_CLASSES], const double pose_lo[16]) {
    if (!m || !cls || !pose_lo) return MULLS_E_ARG;
    mulls_ctx *ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    for (int c = 0; c < kNumClasses; ++c) {
        if (cls[c].n > m->cap) {
            ctx->err = "mulls_map_set: class cloud larger than the map's capacity";
            return MULLS_E_CAPACITY;
        }
        if (cls[c].n > 0 && !cls[c].aos48) return MULLS_E_ARG;
    }
    const double big = 1.7976931348623157e308;
    double lb[6] = {big, big, big, -big, -big, -big};
    for (int c = 0; c < kNumClasses; ++c) {
        if (cls[c].n)
            CK(cudaMemcpyAsync(m->buf[m->cur][c], cls[c].aos48, cls[c].n * 48, cudaMemcpyHostToDevice, ctx->stream));
        m->n[c] = (uint32_t)cls[c].n;
        for (size_t i = 0; i < cls[c].n; ++i) // get_cloud_bbx, utility.hpp:817-847
            for (int d = 0; d < 3; ++d) {
                const double v = cls[c].aos48[12 * i + d];
                if (lb[d] > v) lb[d] = v;
                if (lb[3 + d] < v) lb[3 + d] = v;
            }
    }
    CK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 16; ++i) m->pose[i] = pose_lo[i];
    for (int i = 0; i < 6; ++i) m->local_bound[i] = lb[i];
    // the world-frame box is refreshed by the next update; until then report the local one moved by the pose's translation
    for (int d = 0; d < 3; ++d) {
        m->bound[d] = lb[d] + pose_lo[4 * d + 3];
        m->bound[3 + d] = lb[3 + d] + pose_lo[4 * d + 3];
    }
    m->last = mulls_map_info();
    ++m->epoch;
    if (ctx->tree_map == m) ctx->tree_map = nullptr;
    return MULLS_OK;
}

int mulls_map_get_info(const mulls_map *m, mulls_map_info *info) {
    if (!m || !info) return MULLS_E_ARG;
    map_fill_info(m, info);
    return MULLS_OK;
}

int mulls_map_download(mulls_map *m, int cls, float *out_aos48, size_t cap, size_t *n) {
    if (!m || cls < 0 || cls >= kNumClasses || !n) return MULLS_E_ARG;
    mulls_ctx *ctx = m->ctx;
    *n = m->n[cls];
    if (!out_aos48) return MULLS_OK;
    if (cap < m->n[cls]) {
        ctx->err = "mulls_map_download: buffer too small";
        return MULLS_E_CAPACITY;
    }
    CK(cudaSetDevice(ctx->device));
    if (m->n[cls]) CK(cudaMemcpy(out_aos48, m->buf[m->cur][cls], (size_t)m->n[cls] * 48, cudaMemcpyDeviceToHost));
    return MULLS_OK;
}

int mulls_map_update(mulls_map *m, const mulls_cloud_view scan_down[MULLS_NUM_CLASSES], const double scan_pose_lo[16],
                     const mulls_map_params *params, mulls_map_info *info) {
    if (!m || !scan_down || !scan_pose_lo || !params) return MULLS_E_ARG;
    mulls_ctx *ctx = m->ctx;
    const mulls_map_params &P = *params;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    MapArgs M;
    std::memset(&M, 0, sizeof(M));
    const size_t nu = strnlen(P.used_feature_type, 8);
    for (int c = 0; c < kNumClasses; ++c) {
        M.used[c] = (c < (int)nu && P.used_feature_type[c] == '1') ? 1 : 0;
        if (scan_down[c].n > 0 && !scan_down[c].aos48) return MULLS_E_ARG;
        if (scan_down[c].n > m->cap || (size_t)m->n[c] + scan_down[c].n > m->cap) {
            ctx->err = "mulls_map_update: map + scan exceed max_pts_per_class";
            return MULLS_E_CAPACITY;
        }
    }
    // :28, :32 tran_target_map = pose_scan^-1 * pose_map and its inverse
    double inv_scan[16];
    host_inverse4(scan_pose_lo, inv_scan);
    host_mul4(inv_scan, m->pose, M.T);
    host_inverse4(M.T, M.Tinv);
    for (int i = 0; i < 16; ++i) M.pose[i] = scan_pose_lo[i];
    M.radius = (double)P.local_map_radius;
    M.max_num_pts = P.max_num_pts;
    M.kept_vertex_num = P.kept_vertex_num;
    M.seed = P.random_seed;
    M.state = m->d_state;
    const int nxt = m->cur ^ 1;
    for (int c = 0; c < kNumClasses; ++c) {
        M.old_pts[c] = m->buf[m->cur][c];
        M.scan_pts[c] = m->scan[c];
        M.scan_drop[c] = nullptr;
        M.mid[c] = m->mid[c];
        M.out[c] = m->buf[nxt][c];
        M.n_old[c] = m->n[c];
        M.n_scan[c] = (uint32_t)scan_down[c].n;
    }
    CK(cudaEventRecord(m->ev0, st));
    for (int c = 0; c < kNumClasses; ++c)
        if (scan_down[c].n)
            CK(cudaMemcpyAsync(m->scan[c], scan_down[c].aos48, scan_down[c].n * 48, cudaMemcpyHostToDevice, st));
    // :37-48 map-based dynamic object removal on the scan's pillar / beam / facade points
    const int feature_point_num = (int)(m->n[0] + m->n[1] + m->n[2] + m->n[3] + m->n[4]);
    if (P.map_based_dynamic_removal_on && feature_point_num > P.max_num_pts / 5) {
        if (ctx->tree_map != m || ctx->tree_epoch != m->epoch) {
            ctx->err = "mulls_map_update: map_based_dynamic_removal_on needs the target trees of the preceding "
                       "mulls_icp_run_to_map on this map";
            return MULLS_E_ARG;
        }
        MapDynArgs D;
        std::memset(&D, 0, sizeof(D));
        const int order[3] = {MULLS_PILLAR, MULLS_BEAM, MULLS_FACADE};
        size_t nq = 0;
        for (int k = 0; k < 3; ++k) {
            const int c = order[k];
            D.cls[k] = c;
            D.scan_pts[k] = m->scan[c];
            D.drop[k] = m->drop[c];
            D.n_scan[k] = M.used[c] ? (uint32_t)scan_down[c].n : 0u;
            if (D.n_scan[k]) {
                CK(cudaMemsetAsync(m->drop[c], 0, D.n_scan[k], st));
                M.scan_drop[c] = m->drop[c];
            }
            nq += D.n_scan[k];
        }
        for (int i = 0; i < 16; ++i) D.Tinv[i] = M.Tinv[i];
        D.center_radius = P.dynamic_removal_center_radius;
        D.dist_min = P.dynamic_dist_thre_min;
        // :34 max_(dynamic_dist_thre_max, dynamic_dist_thre_min + 0.1)
        D.dist_max = ((double)P.dynamic_dist_thre_max > (double)P.dynamic_dist_thre_min + 0.1)
                         ? P.dynamic_dist_thre_max
                         : (float)((double)P.dynamic_dist_thre_min + 0.1);
        D.near_thre = P.near_dist_thre;
        if (nq) k_map_dynamic<<<(unsigned)ceil_div(nq * 32, 256), 256, 0, st>>>(ctx->A, D);
    }
    k_map_merge<<<kNumClasses, kMapBlock, 0, st>>>(M);
    k_map_sample<<<kNumClasses, kMapBlock, 0, st>>>(M);
    CK(cudaMemcpyAsync(m->h_state, m->d_state, sizeof(MapState), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(m->ev1, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    // the map now lives in the other buffer, in the scan's frame
    m->cur = nxt;
    const MapState &S = *m->h_state;
    const double big = 1.7976931348623157e308;
    double lb[6] = {big, big, big, -big, -big, -big}, gb[6] = {big, big, big, -big, -big, -big};
    for (int c = 0; c < kNumClasses; ++c) {
        m->n[c] = S.n_out[c];
        m->last.n_appended[c] = S.n_appended[c];
        if (S.n_out[c] == 0) continue;
        for (int d = 0; d < 3; ++d) {
            lb[d] = std::min(lb[d], (double)S.lb[c][d]);
            lb[3 + d] = std::max(lb[3 + d], (double)S.lb[c][3 + d]);
            gb[d] = std::min(gb[d], (double)S.gb[c][d]);
            gb[3 + d] = std::max(gb[3 + d], (double)S.gb[c][3 + d]);
        }
    }
    for (int i = 0; i < 6; ++i) m->local_bound[i] = lb[i], m->bound[i] = gb[i];
    for (int i = 0; i < 16; ++i) m->pose[i] = scan_pose_lo[i];
    cudaEventElapsedTime(&m->last.ms_update, m->ev0, m->ev1);
    ++m->epoch;
    ctx->tree_map = nullptr; // :134 free_tree()
    // :95-115 update_cloud_vectors: re-estimate the direction of the map's pillar and beam points from the map itself
    // (PCA over at most 20 neighbours within 1.8 m) and keep the ones that still look like a pillar / a beam. The
    // bounding boxes above are not refreshed (the reference computes them before this step).
    if (P.recalculate_feature_on) {
        const float pca_radius = 1.8f, sin_high_pillar = 0.80f, sin_low_beam = 0.25f, min_linearity = 0.65f;
        const int pca_max_k = 20, pca_min_k = 6;
        const int cls[2] = {MULLS_PILLAR, MULLS_BEAM};
        const float lo[2] = {0.0f, sin_low_beam}, hi[2] = {sin_high_pillar, 1.0f};
        bool any = false;
        for (int k = 0; k < 2; ++k) {
            const int c = cls[k];
            if (!M.used[c] || m->n[c] == 0) continue;
            mulls_cloud_view v{(const float *)m->buf[m->cur][c], m->n[c]};
            PcaArgs args;
            uint64_t launches = 0;
            const int rc = pca_on_device(ctx, v, true, pca_radius, pca_max_k, 1, args, launches);
            if (rc != MULLS_OK) return rc;
            k_map_revector<<<1, kMapBlock, 0, st>>>(m->buf[m->cur][c], m->n[c], args, pca_min_k, lo[k], hi[k], min_linearity,
                                                   m->mid[c], &m->d_state->n_out[c]);
            std::swap(m->buf[m->cur][c], m->mid[c]);
            any = true;
        }
        if (any) {
            CK(cudaMemcpyAsync(m->h_state, m->d_state, sizeof(MapState), cudaMemcpyDeviceToHost, st));
            CK(cudaEventRecord(m->ev1, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaGetLastError());
            for (int k = 0; k < 2; ++k) m->n[cls[k]] = m->h_state->n_out[cls[k]];
            cudaEventElapsedTime(&m->last.ms_update, m->ev0, m->ev1);
        }
    }
    if (info) map_fill_info(m, info);
    return MULLS_OK;
}

int mulls_icp_run_to_map(mulls_ctx *ctx, mulls_map *m, const mulls_cloud_view src[MULLS_NUM_CLASSES],
                         const mulls_icp_params *params, const double init_guess[16], mulls_icp_result *out,
                         mulls_icp_trace *trace) {
    if (!ctx || !m || !src || !params || !init_guess) return MULLS_E_ARG;
    if (ctx != m->ctx) {
        ctx->err = "mulls_icp_run_to_map: the map belongs to another context";
        return MULLS_E_ARG;
    }
    mulls_cloud_view tgt[MULLS_NUM_CLASSES];
    for (int c = 0; c < kNumClasses; ++c) {
        tgt[c].aos48 = (const float *)m->buf[m->cur][c];
        tgt[c].n = m->n[c];
    }
    mulls_icp_params P = *params;
    for (int i = 0; i < 6; ++i) P.target_bound[i] = m->local_bound[i]; // block1->local_bound, cregistration.hpp:2916
    int rc = upload_impl(ctx, 1, tgt, src, &P, init_guess, nullptr, nullptr, /*resident=*/false, /*tgt_on_device=*/true);
    if (rc != MULLS_OK) return rc;
    rc = run_impl(ctx, out, trace, nullptr, nullptr);
    ctx->uploaded = false;
    if (rc == MULLS_OK) { // the sorted target slices of this run stand in for block1->tree_*
        ctx->tree_map = m;
        ctx->tree_epoch = m->epoch;
    }
    return rc;
}

// ================================================================================================
// Keypoint non-maximum suppression (CFilter::non_max_suppress, cfilter.hpp:1183-1312): kernels_nms.cuh. One device NMS
// for classify_nground_pts' four class clouds and for mulls_non_max_suppress' one cloud.
// ================================================================================================
// Slots of the cell hash of k_nms_select for clouds of at most `cap` points, 0 for none: a cloud of at most one chunk
// never looks back at earlier chunks, and a radius whose square is not > 0 suppresses nothing. Load factor <= 1/2.
static uint32_t nms_hash_slots(size_t cap, float r2) {
    if (cap <= (size_t)kNmsBlock || !(r2 > 0.f)) return 0;
    uint32_t h = 1;
    while (h < 2 * cap) h <<= 1;
    return h;
}
// 1 / the cell edge. The edge exceeds every per-axis |dx| of a pair whose float flann_l2 is < r2: such a |dx| is below
// sqrt(r2) (1 + 2^-22), the margin here is 2^-10 and also covers the double rounding of x * (1 / edge). The floor keeps the edge
// above the distances a flushed product could hide. DESIGN §16.
static double nms_inv_cell(float r2) { return 1.0 / std::max(std::sqrt((double)r2) * (1.0 + 1.0 / 1024), 1e-18); }

// sorts the active clouds of N by score and runs the greedy walk: 3 kernels of this library and one radix sort. N's hash
// slots, when it has them, are contiguous from hash[0].
static int launch_nms(mulls_ctx *ctx, const NmsArgs &N, void *cub_temp, size_t cub_bytes, uint64_t &launches) {
    cudaStream_t st = ctx->stream;
    const unsigned gb = (unsigned)ceil_div(N.total, 256);
    CK(cudaMemsetAsync(N.keys_a, 0xff, N.total * sizeof(uint64_t), st));
    if (N.hash[0]) CK(cudaMemsetAsync(N.hash[0], 0xff, (size_t)N.n_clouds * (N.hash_mask + 1ull) * sizeof(NmsSlot), st));
    k_nms_keys<<<dim3(gb, N.n_clouds), 256, 0, st>>>(N);
    CK(cub::DeviceRadixSort::SortKeys(cub_temp, cub_bytes, N.keys_a, N.keys_b, (int)N.total, 0, 64, st));
    k_nms_gather<<<gb, 256, 0, st>>>(N);
    k_nms_select<<<N.n_clouds, kNmsBlock, 0, st>>>(N);
    launches += 3;
    return MULLS_OK;
}

struct NmsCounts { // device-side n / n_kept / ran of the one cloud of mulls_non_max_suppress, and its host copy
    uint32_t n, n_kept, ran, pad;
};

static int nms_impl(mulls_ctx *ctx, mulls_cloud_view cloud, float radius, int32_t *kept_idx, size_t *n_kept, int *performed,
                    NmsCounts &hc, uint64_t &launches) {
    if (!kept_idx || !n_kept || !performed || (cloud.n > 0 && !cloud.aos48)) {
        ctx->err = "mulls_non_max_suppress: NULL cloud rows or output";
        return MULLS_E_ARG;
    }
    const size_t n = cloud.n;
    int rc = check_capacity(ctx, n, "mulls_non_max_suppress");
    if (rc != MULLS_OK) return rc;
    if (n < 10) return MULLS_OK; // cfilter.hpp:1189-1191: no sort, no device work
    if (n >= kNmsMaxPoints) {
        ctx->err = "mulls_non_max_suppress: at most 2^29 - 1 points";
        return MULLS_E_CAPACITY;
    }
    cudaStream_t st = ctx->stream;
    const float r2 = (float)((double)radius * (double)radius);
    const uint32_t slots = nms_hash_slots(n, r2);
    size_t cub_bytes = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)n, 0, 64, st));
    NmsArgs N;
    std::memset(&N, 0, sizeof(N));
    float4 *d_in;
    NmsSlot *d_hash;
    int32_t *d_next;
    NmsCounts *d_cnt;
    void *d_cub;
    ScratchLayout L;
    L.take(d_in, 3 * n), L.take(N.sorted[0], 3 * n), L.take(N.sel[0], n), L.take(N.kept_idx[0], n), L.take(N.order, n);
    L.take(N.keys_a, n), L.take(N.keys_b, n), L.take(d_hash, slots), L.take(d_next, slots ? n : 0), L.take(d_cnt, 1);
    L.take_bytes(d_cub, cub_bytes);
    if ((rc = L.grow(ctx, ctx->nms_buf)) != MULLS_OK) return rc;
    hc = NmsCounts{(uint32_t)n, 0, 0, 0};
    CK(cudaMemcpyAsync(d_cnt, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_in, cloud.aos48, n * 48, cudaMemcpyDefault, st));
    N.n_clouds = 1;
    N.on_mask = 1;
    N.n = &d_cnt->n;
    N.n_kept = &d_cnt->n_kept;
    N.ran = &d_cnt->ran;
    N.r2 = r2;
    N.inv_cell = nms_inv_cell(r2);
    N.in[0] = d_in;
    if (slots) N.hash[0] = d_hash, N.next[0] = d_next;
    N.hash_mask = slots - 1;
    N.total = (uint32_t)n;
    if ((rc = launch_nms(ctx, N, d_cub, cub_bytes, launches)) != MULLS_OK) return rc;
    // all n entries: one copy instead of a count read-back first; the ones past the kept count are unspecified
    CK(cudaMemcpyAsync(kept_idx, N.kept_idx[0], n * sizeof(int32_t), cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(&hc, d_cnt, sizeof(hc), cudaMemcpyDeviceToHost, st));
    return MULLS_OK;
}

int mulls_non_max_suppress(mulls_ctx *ctx, mulls_cloud_view cloud, float non_max_radius, int32_t *kept_idx, size_t *n_kept,
                           int *performed) {
    NmsCounts hc{0, 0, 0, 0};
    const int rc = front_call(ctx, [&](uint64_t &launches) {
        return nms_impl(ctx, cloud, non_max_radius, kept_idx, n_kept, performed, hc, launches);
    });
    if (rc != MULLS_OK) return rc;
    *n_kept = hc.n_kept;
    *performed = hc.ran ? 1 : 0;
    return MULLS_OK;
}

// ================================================================================================
// Non-ground feature classification (CFilter::classify_nground_pts, cfilter.hpp:2058-2290)
// ================================================================================================
void mulls_classify_default_params(mulls_classify_params *p) {
    std::memset(p, 0, sizeof(*p));
    p->neighbor_searching_radius = 1.0f;
    p->neighbor_k = 50;
    p->neigh_k_min = 8;
    p->pca_down_rate = 1;
    p->edge_thre = 0.65f;
    p->planar_thre = 0.65f;
    p->edge_thre_down = 0.75f;
    p->planar_thre_down = 0.75f;
    p->extract_vertex_points_method = 2;
    p->curvature_thre = 0.12f;
    p->vertex_curvature_non_max_radius = 1.5f;
    p->linear_vertical_sin_high_thre = 0.94f;
    p->linear_vertical_sin_low_thre = 0.17f;
    p->planar_vertical_sin_high_thre = 0.98f;
    p->planar_vertical_sin_low_thre = 0.34f;
    p->fixed_num_downsampling = 0;
    p->pillar_down_fixed_num = 200;
    p->facade_down_fixed_num = 800;
    p->beam_down_fixed_num = 200;
    p->roof_down_fixed_num = 100;
    p->unground_down_fixed_num = 20000;
    p->beam_height_max = FLT_MAX;
    p->roof_height_min = -FLT_MAX;
    p->feature_pts_ratio_guess = 0.3f;
    p->sharpen_with_nms = 1;
    p->use_distance_adaptive_pca = 0;
    p->random_seed = 0;
    p->pca_unit_distance = 0.f;
}

static int classify_impl(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_classify_params *params, mulls_classify_out *out,
                         uint64_t &launches) {
    if (!params || !out || (cloud_in.n > 0 && !cloud_in.aos48)) return MULLS_E_ARG;
    const mulls_classify_params &P = *params;
    // the reference names two units (30 at cfilter.hpp:2093, 35 as get_pc_pca_feature's default): the caller picks one
    if (P.use_distance_adaptive_pca && !(P.pca_unit_distance > 0.f)) {
        ctx->err = "mulls_classify_nground: use_distance_adaptive_pca needs pca_unit_distance > 0";
        return MULLS_E_UNSUPPORTED;
    }
    const float unit_dist = P.use_distance_adaptive_pca ? P.pca_unit_distance : 0.f;
    if (P.neighbor_k < 1 || P.neighbor_k > kPcaListCap || !(P.neighbor_searching_radius > 0.f)) {
        ctx->err = "mulls_classify_nground: neighbor_k must be 1..64 and the radius positive";
        return MULLS_E_ARG;
    }
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) out->n[k] = 0;
    const size_t n0 = cloud_in.n;
    if (n0 == 0) return MULLS_OK;
    if (const int rc = check_capacity(ctx, n0, "mulls_classify_nground"); rc != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    // :2086-2087 random_downsample_pcl(cloud_in, unground_down_fixed_num): the size it leaves is known up front
    size_t n = n0;
    const bool sample_in = P.fixed_num_downsampling && P.unground_down_fixed_num >= 0 && n0 > (size_t)P.unground_down_fixed_num;
    if (sample_in) n = (size_t)P.unground_down_fixed_num;
    const int stride = P.pca_down_rate > 0 ? P.pca_down_rate : 1;
    const size_t row_b = 48;
    ClsArgs C;
    std::memset(&C, 0, sizeof(C));
    float4 *d_in, *d_sel;
    uint32_t *d_ord;
    NmsSlot *d_hash;
    int32_t *d_next;
    ScratchLayout L;
    L.take(d_in, 3 * n0), L.take(C.rows, 3 * n0);
    for (int c = 0; c < 4; ++c)
        L.take(C.cls[c], 3 * n0), L.take(C.cls_sorted[c], 3 * n0), L.take(C.down[c], 3 * n0), L.take(C.down2[c], 3 * n0);
    L.take(C.sect, 6 * n0), L.take(C.vrows, 3 * n0), L.take(C.vertex, 3 * n0), L.take(d_sel, 4 * n0), L.take(d_ord, n0);
    // non_max_suppress(cloud, cloud_down, 0.25 * neighbor_searching_radius) (:2236-2255) on the four class clouds
    const float nms_radius = (float)(0.25 * (double)P.neighbor_searching_radius);
    const float nms_r2 = (float)((double)nms_radius * (double)nms_radius);
    const uint32_t nms_slots = nms_hash_slots(n, nms_r2);
    L.take(d_hash, 4 * (size_t)nms_slots), L.take(d_next, nms_slots ? 4 * n0 : 0);
    L.take(C.label0, n0), L.take(C.label, n0), L.take(C.downflag, n0), L.take(C.st4, n0), L.take(C.vflag, n0), L.take(C.st, 1);
    if (const int rc = L.grow(ctx, ctx->cls_buf); rc != MULLS_OK) return rc;
    C.P = P;
    C.n = (uint32_t)n;
    C.stride = stride;
    CK(cudaMemsetAsync(C.st, 0, sizeof(ClsState), st));
    if (sample_in) {
        CK(cudaMemcpyAsync(d_in, cloud_in.aos48, n0 * row_b, cudaMemcpyDefault, st)); // host or device rows
        k_rows_sample<<<1, kClsBlock, 0, st>>>(d_in, (uint32_t)n0, P.unground_down_fixed_num, P.random_seed,
                                               18u, C.rows);
        ++launches;
    } else {
        CK(cudaMemcpyAsync(C.rows, cloud_in.aos48, n0 * row_b, cudaMemcpyDefault, st));
    }
    ClsState hs;
    std::memset(&hs, 0, sizeof(hs));
    if (n > 0) {
        // :2089-2097 PCA of every pca_down_rate-th point, with the neighbour lists
        mulls_cloud_view v{(const float *)C.rows, n};
        const int rc = pca_on_device(ctx, v, true, P.neighbor_searching_radius, P.neighbor_k, stride, C.F, launches, unit_dist);
        if (rc != MULLS_OK) return rc;
        const unsigned gb = (unsigned)ceil_div(n, 256);
        k_cls_label<<<gb, 256, 0, st>>>(C);
        k_cls_compact<<<8, kClsBlock, 0, st>>>(C);
        k_cls_promote_pre<<<gb, 256, 0, st>>>(C);
        k_cls_promote<<<1, kClsBlock, 0, st>>>(C);
        k_cls_promote_apply<<<gb, 256, 0, st>>>(C);
        k_cls_compact2<<<4, kClsBlock, 0, st>>>(C);
        k_cls_encode<<<gb, 256, 0, st>>>(C);
        k_cls_compact_vertex<<<1, kClsBlock, 0, st>>>(C);
        launches += 8;
        if (P.sharpen_with_nms) {
            const int fixed[4] = {P.pillar_down_fixed_num, P.beam_down_fixed_num, P.facade_down_fixed_num, P.roof_down_fixed_num};
            NmsArgs N;
            std::memset(&N, 0, sizeof(N));
            N.n_clouds = 4;
            N.n = C.st->n_cls2;
            N.n_kept = C.st->n_down; // n_down stays what the threshold loop left (0 when sharpening) where NMS does not run
            N.ran = C.st->nms_ran;
            N.r2 = nms_r2;
            N.inv_cell = nms_inv_cell(nms_r2);
            N.hash_mask = nms_slots - 1;
            N.total = (uint32_t)n;
            N.keys_a = ctx->A.keys_a;
            N.keys_b = ctx->A.keys_b;
            N.order = d_ord;
            for (int c = 0; c < 4; ++c) {
                if (fixed[c] > 0) N.on_mask |= 1u << c;
                N.in[c] = C.cls[c];
                N.sorted[c] = C.cls_sorted[c];
                N.kept_rows[c] = C.down[c];
                N.sel[c] = d_sel + (size_t)c * n0;
                if (nms_slots) {
                    N.hash[c] = d_hash + (size_t)c * nms_slots;
                    N.next[c] = d_next + (size_t)c * n0;
                }
            }
            if (const int rc = launch_nms(ctx, N, ctx->cub_temp, ctx->cub_temp_bytes, launches); rc != MULLS_OK) return rc;
        }
        if (P.fixed_num_downsampling) {
            k_cls_fixed<<<4, kClsBlock, 0, st>>>(C);
            ++launches;
        }
        CK(cudaMemcpyAsync(&hs, C.st, sizeof(ClsState), cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    // results
    const float4 *src[MULLS_OUT_COUNT];
    size_t cnt[MULLS_OUT_COUNT];
    for (int c = 0; c < 4; ++c) {
        src[c] = hs.nms_ran[c] ? C.cls_sorted[c] : C.cls[c];
        cnt[c] = hs.n_cls2[c];
        src[4 + c] = P.fixed_num_downsampling ? C.down2[c] : C.down[c];
        cnt[4 + c] = P.fixed_num_downsampling ? hs.n_down2[c] : hs.n_down[c];
    }
    src[MULLS_OUT_VERTEX] = C.vertex, cnt[MULLS_OUT_VERTEX] = hs.n_vertex;
    src[MULLS_OUT_UNGROUND] = C.rows, cnt[MULLS_OUT_UNGROUND] = n;
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) {
        out->n[k] = cnt[k];
        if (!out->rows[k] || cnt[k] == 0) continue;
        if (cnt[k] > out->cap) {
            ctx->err = "mulls_classify_nground: output buffer too small";
            return MULLS_E_CAPACITY;
        }
        CK(cudaMemcpyAsync(out->rows[k], src[k], cnt[k] * row_b, cudaMemcpyDefault, st));
    }
    return MULLS_OK;
}

int mulls_classify_nground(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_classify_params *params,
                           mulls_classify_out *out) {
    return front_call(ctx, [&](uint64_t &launches) { return classify_impl(ctx, cloud_in, params, out, launches); });
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// Ground segmentation (CFilter::fast_ground_filter, cfilter.hpp:1658-2036)
// ------------------------------------------------------------------------------------------------
namespace {
// first kSacDraws outputs of boost::mt19937 seeded with 12345u (every pcl::SampleConsensusModel object starts there)
const uint32_t *sac_draw_table() {
    static std::vector<uint32_t> tab;
    if (tab.empty()) {
        std::vector<uint32_t> t(kSacDraws);
        SacMt19937 mt;
        for (int k = 0; k < kSacDraws; ++k) t[k] = mt.next();
        tab.swap(t);
    }
    return tab.data();
}
int host_ord(float f) {
    int i;
    std::memcpy(&i, &f, 4);
    return i >= 0 ? i : (i ^ 0x7fffffff);
}
} // namespace

extern "C" {

void mulls_ground_default_params(mulls_ground_params *p) { // extract_semantic_pts as test/mulls_slam.cpp calls it (gflags :78-104)
    if (!p) return;
    std::memset(p, 0, sizeof(*p));
    p->min_grid_pt_num = 10;
    p->grid_resolution = 3.0f;
    p->max_height_difference = 0.3f;
    p->neighbor_height_diff = 1.5f;
    p->max_ground_height = 5.0f;
    p->ground_random_down_rate = 15;
    p->ground_random_down_down_rate = 2;
    p->nonground_random_down_rate = 3;
    p->reliable_neighbor_grid_num_thre = 0;
    p->estimate_ground_normal_method = 3;
    p->normal_estimation_radius = 2.0f;
    p->distance_weight_downsampling_method = 2;
    p->standard_distance = 15.0f;
    p->fixed_num_downsampling = 0;
    p->down_ground_fixed_num = 300;
    p->intensity_thre = FLT_MAX;
    p->apply_grid_wise_outlier_filter = 0;
    p->outlier_std_scale = 3.0f;
    p->random_seed = 0;
}

static int ground_impl(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_ground_params *params, mulls_ground_out *out,
                       uint64_t &launches) {
    if (!params || !out || (cloud_in.n > 0 && !cloud_in.aos48)) return MULLS_E_ARG;
    const mulls_ground_params &P = *params;
    if (P.estimate_ground_normal_method != 0 && P.estimate_ground_normal_method != 3) {
        ctx->err = "mulls_fast_ground_filter: estimate_ground_normal_method 1 / 2 (pcl::NormalEstimation) are not implemented";
        return MULLS_E_UNSUPPORTED;
    }
    if (P.ground_random_down_rate < 1 || P.nonground_random_down_rate < 1 || P.ground_random_down_down_rate < 1 ||
        !(P.grid_resolution > 0.f)) {
        ctx->err = "mulls_fast_ground_filter: the down-sampling rates must be >= 1 and grid_resolution positive";
        return MULLS_E_ARG;
    }
    out->n_ground = out->n_ground_down = out->n_unground = 0;
    const size_t n = cloud_in.n;
    if (n == 0) return MULLS_OK;
    if (const int rc = check_capacity(ctx, n, "mulls_fast_ground_filter"); rc != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    // temporary storage of the library sort / scans
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (uint32_t *)nullptr, (int)n, 0, 32, st);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, st);
    // per-point scratch
    const size_t row_b = 48;
    const size_t tmp_bytes = std::max(sort_bytes, scan_bytes);
    GfArgs A;
    std::memset(&A, 0, sizeof(A));
    void *tmp;
    ScratchLayout L;
    L.take(A.rows, 3 * n), L.take(A.out_ground, 3 * n), L.take(A.out_ground_down, 3 * n);
    L.take(A.out_unground, 3 * n), L.take(A.key, n), L.take(A.idx, n), L.take(A.key_s, n), L.take(A.idx_s, n);
    L.take(A.cell_all, n), L.take(A.high_flag, n), L.take(A.high_pos, n), L.take(A.decision, n), L.take(A.cand, n);
    L.take(A.shuf, n), L.take(A.inl, n), L.take(A.st, 1), L.take(A.draws, kSacDraws), L.take_bytes(tmp, tmp_bytes);
    if (const int rc = L.grow(ctx, ctx->gf_buf); rc != MULLS_OK) return rc;
    A.P = P;
    A.n = (uint32_t)n;
    CK(cudaMemcpyAsync((void *)A.rows, cloud_in.aos48, n * row_b, cudaMemcpyDefault, st)); // host or device rows
    CK(cudaMemcpyAsync((void *)A.draws, sac_draw_table(), kSacDraws * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    GfState hs;
    std::memset(&hs, 0, sizeof(hs));
    hs.bb[0] = hs.bb[1] = host_ord(FLT_MAX);
    hs.bb[2] = hs.bb[3] = host_ord(-FLT_MAX);
    CK(cudaMemcpyAsync(A.st, &hs, sizeof(GfState), cudaMemcpyHostToDevice, st));
    const unsigned pb = (unsigned)ceil_div(n, kGfBlock);
    k_gf_bbox<<<pb, kGfBlock, 0, st>>>(A);
    k_gf_setup<<<1, 32, 0, st>>>(A);
    launches += 2;
    CK(cudaMemcpyAsync(&hs, A.st, sizeof(GfState), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    if (hs.num_grid < 0 || hs.num_grid > (1 << 26)) {
        ctx->err = "mulls_fast_ground_filter: the cloud spans more than 2^26 grid cells (outliers far from the scan?)";
        return MULLS_E_CAPACITY;
    }
    const int num_grid = hs.num_grid;
    if (num_grid > 0) { // (a degenerate cloud with zero extent along x or y has no cell: every point fails the id test)
        const size_t g = (size_t)num_grid;
        size_t cscan = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, cscan, (uint32_t *)nullptr, (uint32_t *)nullptr, num_grid, st);
        void *ctmp;
        ScratchLayout CL;
        CL.take(A.cell_start, g), CL.take(A.cell_end, g), CL.take(A.min_z, g), CL.take(A.neighbor_min_z, g);
        CL.take(A.outlier_thre, g), CL.take(A.reliable, g), CL.take(A.cell_normal, g), CL.take(A.cell_ng, g);
        CL.take(A.cell_nu, g), CL.take(A.cell_og, g), CL.take(A.cell_ou, g), CL.take_bytes(ctmp, cscan);
        if (const int rc = CL.grow(ctx, ctx->gf_cell_buf); rc != MULLS_OK) return rc;
        CK(cudaMemsetAsync(A.cell_start, 0, 4 * g, st));
        CK(cudaMemsetAsync(A.cell_end, 0, 4 * g, st));
        const unsigned wb = (unsigned)ceil_div(g * 32, kGfBlock), cbk = (unsigned)ceil_div(g, kGfBlock);
        k_gf_assign<<<pb, kGfBlock, 0, st>>>(A);
        size_t b1 = tmp_bytes;
        CK(cub::DeviceRadixSort::SortPairs(tmp, b1, A.key, A.key_s, A.idx, A.idx_s, (int)n, 0, 32, st));
        k_gf_bounds<<<pb, kGfBlock, 0, st>>>(A);
        k_gf_cell_min<<<wb, kGfBlock, 0, st>>>(A, num_grid);
        k_gf_neighbors<<<cbk, kGfBlock, 0, st>>>(A, num_grid);
        k_gf_high<<<pb, kGfBlock, 0, st>>>(A);
        size_t b2 = tmp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(tmp, b2, A.high_flag, A.high_pos, (int)n, st));
        k_gf_high_emit<<<pb, kGfBlock, 0, st>>>(A);
        k_gf_cell_decide<<<wb, kGfBlock, 0, st>>>(A, num_grid);
        size_t b3 = cscan;
        CK(cub::DeviceScan::ExclusiveSum(ctmp, b3, A.cell_ng, A.cell_og, num_grid, st));
        b3 = cscan;
        CK(cub::DeviceScan::ExclusiveSum(ctmp, b3, A.cell_nu, A.cell_ou, num_grid, st));
        k_gf_totals<<<1, 1, 0, st>>>(A, num_grid);
        k_gf_cell_emit<<<wb, kGfBlock, 0, st>>>(A, num_grid);
        k_gf_down<<<1, kClsBlock, 0, st>>>(A);
        launches += 10;
        CK(cudaMemcpyAsync(&hs, A.st, sizeof(GfState), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        out->n_ground = hs.n_ground, out->n_ground_down = hs.n_ground_down, out->n_unground = hs.n_unground;
        if (hs.n_ground > out->cap || hs.n_unground > out->cap) {
            ctx->err = "mulls_fast_ground_filter: output buffer too small";
            return MULLS_E_CAPACITY;
        }
        if (out->ground && hs.n_ground)
            CK(cudaMemcpyAsync(out->ground, A.out_ground, hs.n_ground * row_b, cudaMemcpyDefault, st));
        if (out->ground_down && hs.n_ground_down)
            CK(cudaMemcpyAsync(out->ground_down, A.out_ground_down, hs.n_ground_down * row_b, cudaMemcpyDefault, st));
        if (out->unground && hs.n_unground)
            CK(cudaMemcpyAsync(out->unground, A.out_unground, hs.n_unground * row_b, cudaMemcpyDefault, st));
    }
    return MULLS_OK;
}

int mulls_fast_ground_filter(mulls_ctx *ctx, mulls_cloud_view cloud_in, const mulls_ground_params *params,
                             mulls_ground_out *out) {
    return front_call(ctx, [&](uint64_t &launches) { return ground_impl(ctx, cloud_in, params, out, launches); });
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// CFilter::voxel_downsample (cfilter.hpp:83-165) and the chain of CFilter::extract_semantic_pts (:2295-2413)
// ------------------------------------------------------------------------------------------------
extern "C" {

static int voxel_impl(mulls_ctx *ctx, mulls_cloud_view cloud_in, float voxel_size, float *out, size_t cap, size_t *n_out,
                      uint64_t &launches) {
    if (!n_out || (cloud_in.n > 0 && (!cloud_in.aos48 || !out))) return MULLS_E_ARG;
    *n_out = 0;
    const size_t n = cloud_in.n;
    if (n == 0) return MULLS_OK;
    if (const int rc = check_capacity(ctx, n, "mulls_voxel_downsample"); rc != MULLS_OK) return rc;
    cudaStream_t st = ctx->stream;
    const size_t row_b = 48;
    if (voxel_size < 0.001) { // :89-97 disabled: cloud_out = cloud_in
        if (n > cap) {
            ctx->err = "mulls_voxel_downsample: output buffer too small";
            return MULLS_E_CAPACITY;
        }
        CK(cudaMemcpyAsync(out, cloud_in.aos48, n * row_b, cudaMemcpyDefault, st));
        *n_out = n;
        return MULLS_OK;
    }
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                    (uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, 0, 64, st);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, st);
    const size_t tmp_bytes = std::max(sort_bytes, scan_bytes);
    VxArgs V;
    V.n = (uint32_t)n;
    V.voxel_size = voxel_size;
    void *tmp;
    ScratchLayout L;
    L.take(V.rows, 3 * n), L.take(V.out, 3 * n), L.take(V.key, n), L.take(V.key_s, n), L.take(V.idx, n), L.take(V.idx_s, n);
    L.take(V.head, n), L.take(V.pos, n), L.take(V.st, 1), L.take_bytes(tmp, tmp_bytes);
    if (const int rc = L.grow(ctx, ctx->vx_buf); rc != MULLS_OK) return rc;
    VxState hs;
    std::memset(&hs, 0, sizeof(hs));
    for (int d = 0; d < 3; ++d) hs.bb[d] = host_ord(FLT_MAX), hs.bb[3 + d] = host_ord(-FLT_MAX);
    CK(cudaMemcpyAsync((void *)V.rows, cloud_in.aos48, n * row_b, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(V.st, &hs, sizeof(VxState), cudaMemcpyHostToDevice, st));
    const unsigned pb = (unsigned)ceil_div(n, kGfBlock);
    k_vx_bbox<<<pb, kGfBlock, 0, st>>>(V);
    k_vx_setup<<<1, 1, 0, st>>>(V);
    k_vx_keys<<<pb, kGfBlock, 0, st>>>(V);
    size_t b1 = tmp_bytes;
    CK(cub::DeviceRadixSort::SortPairs(tmp, b1, V.key, V.key_s, V.idx, V.idx_s, (int)n, 0, 64, st));
    k_vx_heads<<<pb, kGfBlock, 0, st>>>(V);
    size_t b2 = tmp_bytes;
    CK(cub::DeviceScan::ExclusiveSum(tmp, b2, V.head, V.pos, (int)n, st));
    k_vx_gather<<<pb, kGfBlock, 0, st>>>(V);
    launches += 5;
    CK(cudaMemcpyAsync(&hs, V.st, sizeof(VxState), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    *n_out = hs.n_out;
    if (hs.n_out > cap) {
        ctx->err = "mulls_voxel_downsample: output buffer too small";
        return MULLS_E_CAPACITY;
    }
    CK(cudaMemcpyAsync(out, V.out, (size_t)hs.n_out * row_b, cudaMemcpyDefault, st));
    return MULLS_OK;
}

int mulls_voxel_downsample(mulls_ctx *ctx, mulls_cloud_view cloud_in, float voxel_size, float *out, size_t cap, size_t *n_out) {
    return front_call(ctx, [&](uint64_t &launches) { return voxel_impl(ctx, cloud_in, voxel_size, out, cap, n_out, launches); });
}

// the three stages in one call frame: one launch count, one device span
static int extract_impl(mulls_ctx *ctx, mulls_cloud_view pc_raw, const mulls_extract_params *params, mulls_extract_out *out,
                        uint64_t &launches) {
    if (!params || !out || (pc_raw.n > 0 && !pc_raw.aos48)) return MULLS_E_ARG;
    out->n_down = out->n_ground = out->n_ground_down = 0;
    for (int k = 0; k < MULLS_OUT_COUNT; ++k) out->cls.n[k] = 0;
    const size_t n = pc_raw.n;
    if (n == 0) return MULLS_OK;
    if ((out->pc_down || out->pc_ground || out->pc_ground_down) && out->cap < n) {
        ctx->err = "mulls_extract_semantic_pts: the output buffers must hold pc_raw.n rows";
        return MULLS_E_ARG;
    }
    // the clouds handed from stage to stage stay in HBM: pc_down and the ground filter's cloud_unground
    const size_t row_b = 48;
    float *d_down, *d_ung;
    ScratchLayout L;
    L.take(d_down, 12 * n), L.take(d_ung, 12 * n);
    int rc = L.grow(ctx, ctx->ext_buf);
    if (rc != MULLS_OK) return rc;
    // :2346 voxel_downsample(pc_raw, pc_down) (pc_sketch, :2348, is not a feature cloud and is not produced)
    size_t n_down = 0;
    rc = voxel_impl(ctx, pc_raw, params->vf_downsample_resolution, d_down, n, &n_down, launches);
    if (rc != MULLS_OK) return rc;
    out->n_down = n_down;
    if (out->pc_down && n_down) CK(cudaMemcpyAsync(out->pc_down, d_down, n_down * row_b, cudaMemcpyDefault, ctx->stream));
    // :2355-2361 fast_ground_filter(pc_down -> pc_ground, pc_ground_down, pc_unground)
    mulls_ground_out g;
    std::memset(&g, 0, sizeof(g));
    g.ground = out->pc_ground, g.ground_down = out->pc_ground_down, g.unground = d_ung;
    g.cap = n;
    rc = ground_impl(ctx, mulls_cloud_view{d_down, n_down}, &params->ground, &g, launches);
    if (rc != MULLS_OK) return rc;
    out->n_ground = g.n_ground, out->n_ground_down = g.n_ground_down;
    // :2378-2391 classify_nground_pts(pc_unground -> pillar, beam, facade, roof, their down clouds, vertex)
    return classify_impl(ctx, mulls_cloud_view{d_ung, g.n_unground}, &params->classify, &out->cls, launches);
}

int mulls_extract_semantic_pts(mulls_ctx *ctx, mulls_cloud_view pc_raw, const mulls_extract_params *params,
                               mulls_extract_out *out) {
    return front_call(ctx, [&](uint64_t &launches) { return extract_impl(ctx, pc_raw, params, out, launches); });
}

} // extern "C"
