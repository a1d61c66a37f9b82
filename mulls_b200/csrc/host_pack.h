// Host-side wire format of a cloud + the worker pool that produces it.
//
// The boundary hands the library pcl::PointXYZINormal rows (48 B/point, utility.hpp:40) of which the path reads
// 28 B: x y z, intensity, normal / principal direction (SURVEY §8d) — plus `curvature` (the timestamp ratio) when
// motion undistortion is on (cregistration.hpp:1248-1258). PCIe, not HBM, bounds the end-to-end rate of batched
// registrations (11.5 MB of rows per 120k/120k pair), so the rows are repacked on the host cores into pinned staging
// before the DMA:
//   format 1 (28 B/point):  [n x float4 (x y z intensity)] [n x 3 floats (nx ny nz)]   (padded to a float4 boundary)
//   format 2 (32 B/point):  [n x float4 (x y z intensity)] [n x float4 (nx ny nz curvature)]
// The ingest (load_input_point, kernels_ingest.cuh) reads either format or the raw rows (format 0: device-resident clouds of the local map, PCA).
// The pool is a process-wide set of detached worker threads fed by every context / lane; the submitting thread
// helps until its own jobs are done.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>
#include <xmmintrin.h>

namespace mulls {

enum : int { kFmtRows48 = 0, kFmtPacked28 = 1, kFmtPacked32 = 2 };

// float4 slots a segment of n points occupies in the given format
static inline size_t packed_slots(size_t n, int fmt) {
    if (fmt == kFmtPacked28) return n + (3 * n + 3) / 4;
    if (fmt == kFmtPacked32) return 2 * n;
    return 3 * n;
}

// Pack rows [first, first+count) of `rows` (48 B each) into `pos` (float4 per point, 16 B aligned) and `nrm`
// (format 1: 3 floats per point; format 2: float4 per point; the array base is 16 B aligned). `first` must be a
// multiple of 4 so that the 3-float groups of four points stay 16 B aligned.
static inline void pack_rows(const float *rows, size_t first, size_t count, int fmt, float *pos, float *nrm) {
    const float *p = rows + 12 * first;
    float *po = pos + 4 * first;
    size_t i = 0;
    if (fmt == kFmtPacked28) {
        float *no = nrm + 3 * first;
        for (; i + 4 <= count; i += 4, p += 48, po += 16, no += 12) {
            __m128 a[4], b[4];
            for (int k = 0; k < 4; ++k) {
                const __m128 xyz = _mm_loadu_ps(p + 12 * k);
                b[k] = _mm_loadu_ps(p + 12 * k + 4);
                const __m128 c = _mm_load_ss(p + 12 * k + 8);
                const __m128 t = _mm_shuffle_ps(xyz, c, _MM_SHUFFLE(0, 0, 2, 2)); // z z i i
                a[k] = _mm_shuffle_ps(xyz, t, _MM_SHUFFLE(2, 0, 1, 0));           // x y z i
            }
            _mm_stream_ps(po, a[0]);
            _mm_stream_ps(po + 4, a[1]);
            _mm_stream_ps(po + 8, a[2]);
            _mm_stream_ps(po + 12, a[3]);
            const __m128 t0 = _mm_shuffle_ps(b[0], b[1], _MM_SHUFFLE(0, 0, 2, 2)); // b0z b0z b1x b1x
            const __m128 t2 = _mm_shuffle_ps(b[2], b[3], _MM_SHUFFLE(0, 0, 2, 2)); // b2z b2z b3x b3x
            _mm_stream_ps(no, _mm_shuffle_ps(b[0], t0, _MM_SHUFFLE(2, 0, 1, 0)));     // b0x b0y b0z b1x
            _mm_stream_ps(no + 4, _mm_shuffle_ps(b[1], b[2], _MM_SHUFFLE(1, 0, 2, 1))); // b1y b1z b2x b2y
            _mm_stream_ps(no + 8, _mm_shuffle_ps(t2, b[3], _MM_SHUFFLE(2, 1, 2, 0)));   // b2z b3x b3y b3z
        }
        for (; i < count; ++i, p += 12, po += 4, no += 3) {
            po[0] = p[0], po[1] = p[1], po[2] = p[2], po[3] = p[8];
            no[0] = p[4], no[1] = p[5], no[2] = p[6];
        }
    } else { // kFmtPacked32
        float *no = nrm + 4 * first;
        for (; i < count; ++i, p += 12, po += 4, no += 4) {
            const __m128 xyz = _mm_loadu_ps(p);
            const __m128 b = _mm_loadu_ps(p + 4);
            const __m128 c = _mm_loadu_ps(p + 8);                              // i curv _ _
            const __m128 t = _mm_shuffle_ps(xyz, c, _MM_SHUFFLE(0, 0, 2, 2));  // z z i i
            const __m128 u = _mm_shuffle_ps(b, c, _MM_SHUFFLE(1, 1, 2, 2));    // nz nz curv curv
            _mm_stream_ps(po, _mm_shuffle_ps(xyz, t, _MM_SHUFFLE(2, 0, 1, 0))); // x y z i
            _mm_stream_ps(no, _mm_shuffle_ps(b, u, _MM_SHUFFLE(2, 0, 1, 0)));   // nx ny nz curv
        }
    }
}

struct PackJob {
    const float *rows;
    float *pos, *nrm;
    size_t first, count;
    int fmt;
    std::atomic<int> *pending; // decremented when the job is done
    void (*task)(void *) = nullptr; // set: the job runs task(arg) instead of packing rows
    void *arg = nullptr;
};

class PackPool {
  public:
    static PackPool &get() {
        static PackPool *pool = new PackPool(); // never destroyed: the workers are detached and outlive static teardown
        return *pool;
    }
    // make sure at least `n` workers exist (n <= 0: the default, MULLS_PACK_THREADS or hw/16 clamped to 2..8)
    void ensure_workers(int n) {
        if (n <= 0) {
            const char *env = std::getenv("MULLS_PACK_THREADS");
            n = env ? std::atoi(env) : 0;
            if (n <= 0) {
                const int hw = (int)std::thread::hardware_concurrency();
                n = hw / 16; // a few streaming workers saturate a PCIe link; more only contend for host memory bandwidth
                if (n < 2) n = 2;
                if (n > 8) n = 8;
            }
        }
        std::lock_guard<std::mutex> lk(m_);
        while (n_workers_ < n) {
            std::thread([this]() { worker(); }).detach();
            ++n_workers_;
        }
    }
    int workers() {
        std::lock_guard<std::mutex> lk(m_);
        return n_workers_;
    }
    void submit(const std::vector<PackJob> &jobs) {
        {
            std::lock_guard<std::mutex> lk(m_);
            for (const PackJob &j : jobs) q_.push_back(j);
        }
        cv_.notify_all();
    }
    // the submitting thread helps (any job, not only its own) until `pending` reaches zero
    void help_until_done(std::atomic<int> &pending) {
        while (pending.load(std::memory_order_acquire) > 0) {
            PackJob j;
            bool have = false;
            {
                std::lock_guard<std::mutex> lk(m_);
                if (!q_.empty()) {
                    j = q_.front();
                    q_.pop_front();
                    have = true;
                }
            }
            if (have) run(j);
            else std::this_thread::yield();
        }
    }

  private:
    static void run(const PackJob &j) {
        if (j.task) j.task(j.arg);
        else {
            pack_rows(j.rows, j.first, j.count, j.fmt, j.pos, j.nrm);
            _mm_sfence(); // the streaming stores must be visible before the DMA is queued
        }
        j.pending->fetch_sub(1, std::memory_order_release);
    }
    void worker() {
        for (;;) {
            PackJob j;
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [this]() { return !q_.empty(); });
                j = q_.front();
                q_.pop_front();
            }
            run(j);
        }
    }
    std::mutex m_;
    std::condition_variable cv_;
    std::deque<PackJob> q_;
    int n_workers_ = 0;
};

} // namespace mulls
