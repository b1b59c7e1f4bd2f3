// host_stage.h -- parallel staging copies of pageable frames into the engine's page-locked buffer.
//
// A 1280x720 BGR frame is 2.76 MB; one host thread needs a noticeable share of an end-to-end BotSort.update(dets, img) at
// 256 detections to copy it.  StagePool splits the copy into cache-line
// aligned pieces over a few persistent worker threads plus the caller; the caller is told when each piece lands (in
// order) so that it can queue that piece's host-to-device DMA while the rest is still being copied.
//
// Helpers make the isolated copy faster (scripts/microbench/stage_pool_test.cpp) but can make the whole update() slower:
// they are woken from a condition variable once per frame and the frame goes as several small DMAs instead of one
// (scripts/sweep_stage.sh compares the settings).  Helpers are therefore opt-in: BOXMOT_B200_STAGE_THREADS=N (caller
// included), default 1.
//
// Host-only C++ (no CUDA types).  The pool is created lazily, re-created after a fork (worker threads do not survive
// one), and joined when the process-wide instance is destroyed.
#pragma once
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <mutex>
#include <thread>
#include <vector>

namespace bmb {

class StagePool {
   public:
    static constexpr int MAX_PIECES = 16;
    static constexpr size_t MIN_PIECE = 256 * 1024;   // below this a second thread costs more than it saves

    // process-wide pool; BOXMOT_B200_STAGE_THREADS = copying threads including the caller (default 1: no helpers)
    static StagePool& instance() {
        static StagePool* pool = nullptr;
        static pid_t owner = 0;
        static std::mutex guard;
        std::lock_guard<std::mutex> lk(guard);
        if (!pool || owner != getpid()) {   // first use, or a forked child (the parent's threads are not here)
            int w = 0;
            if (const char* e = std::getenv("BOXMOT_B200_STAGE_THREADS")) w = std::atoi(e) - 1;
            if (w < 0) w = 0;
            if (w > MAX_PIECES - 1) w = MAX_PIECES - 1;
            const unsigned hc = std::thread::hardware_concurrency();
            if (hc && (unsigned)w > hc - 1) w = (int)hc - 1;
            pool = new StagePool(w);        // a forked child abandons the parent's object (its threads never existed here)
            owner = getpid();
        }
        return *pool;
    }

    explicit StagePool(int workers) : n_workers_(workers) {
        for (int i = 0; i < workers; ++i) threads_.emplace_back([this, i] { run(i); });
    }
    ~StagePool() {
        {
            std::lock_guard<std::mutex> lk(m_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }
    StagePool(const StagePool&) = delete;
    StagePool& operator=(const StagePool&) = delete;

    int workers() const { return n_workers_; }

    // dst[0, n) = src[0, n).  `landed(offset, bytes)` is called on the calling thread, piece by piece in address
    // order, as soon as that piece is complete (the caller's own piece is the first one).
    template <typename Landed>
    void copy(void* dst, const void* src, size_t n, Landed landed) {
        int pieces = n_workers_ + 1;
        while (pieces > 1 && n / pieces < MIN_PIECE) --pieces;
        if (pieces <= 1) {
            std::memcpy(dst, src, n);
            landed((size_t)0, n);
            return;
        }
        const size_t step = ((n / pieces) + 63) & ~(size_t)63;
        {
            std::lock_guard<std::mutex> lk(m_);
            n_jobs_ = pieces - 1;
            for (int j = 0; j < n_jobs_; ++j) {
                const size_t o = step * (size_t)(j + 1);
                const size_t len = (j + 1 == pieces - 1) ? n - o : step;
                jobs_[j] = {static_cast<char*>(dst) + o, static_cast<const char*>(src) + o, len};
                done_[j].store(0, std::memory_order_relaxed);
                claimed_[j].store(0, std::memory_order_relaxed);
            }
            next_job_ = 0;
            ++generation_;
        }
        cv_.notify_all();
        std::exception_ptr failed;
        auto tell = [&](size_t off, size_t len) {
            if (failed) return;
            try { landed(off, len); } catch (...) { failed = std::current_exception(); }
        };
        std::memcpy(dst, src, step);
        tell((size_t)0, step);
        const int nj = pieces - 1;
        for (int j = 0; j < nj; ++j) {
            // a helper that has not picked its piece up yet (still waking) loses it to the caller
            if (!done_[j].load(std::memory_order_acquire) && claim(j)) {
                std::memcpy(jobs_[j].dst, jobs_[j].src, jobs_[j].n);
                done_[j].store(1, std::memory_order_release);
            }
            while (!done_[j].load(std::memory_order_acquire)) cpu_relax();
            tell(step * (size_t)(j + 1), jobs_[j].n);
        }
        {   // no helper may still hold a job index when the next call rewrites the table
            std::lock_guard<std::mutex> lk(m_);
            n_jobs_ = 0;
        }
        while (active_.load(std::memory_order_acquire) != 0) cpu_relax();
        if (failed) std::rethrow_exception(failed);
    }

    void copy(void* dst, const void* src, size_t n) {
        copy(dst, src, n, [](size_t, size_t) {});
    }

   private:
    struct Job { char* dst; const char* src; size_t n; };

    static void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();
#else
        std::this_thread::yield();
#endif
    }
    // pieces are claimed through one flag each: whoever flips it from 0 to 1 copies the piece
    bool claim(int j) {
        int expected = 0;
        return claimed_[j].compare_exchange_strong(expected, 1, std::memory_order_acq_rel);
    }
    void run(int /*index*/) {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return stop_ || generation_ != seen; });
                if (stop_) return;
                seen = generation_;
            }
            for (;;) {
                int j;
                {
                    std::lock_guard<std::mutex> lk(m_);
                    if (generation_ != seen || next_job_ >= n_jobs_) break;
                    j = next_job_++;
                    active_.fetch_add(1, std::memory_order_acq_rel);     // counted in under the lock that hands the index out
                }
                if (claim(j)) {
                    std::memcpy(jobs_[j].dst, jobs_[j].src, jobs_[j].n);
                    done_[j].store(1, std::memory_order_release);
                }
                active_.fetch_sub(1, std::memory_order_acq_rel);
            }
        }
    }

    int n_workers_;
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_;
    bool stop_ = false;
    uint64_t generation_ = 0;
    int n_jobs_ = 0, next_job_ = 0;
    Job jobs_[MAX_PIECES]{};
    std::atomic<int> done_[MAX_PIECES]{};
    std::atomic<int> claimed_[MAX_PIECES]{};
    std::atomic<int> active_{0};
};

}  // namespace bmb
