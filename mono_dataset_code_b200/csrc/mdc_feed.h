// The decode-ahead pool of the sequence feeds (mdc_sequence.cpp, mdc_jpeg_gpu.cu).  Host-only C++, so that g++ and nvcc's host pass
// both compile it and the feeds' test harnesses need no source file of their own for it.
//
// `count` frames are read in chunks of `chunk`, chunk k into slot k & 1 of the caller's buffers, one chunk ahead of the caller.
// min(threads, count, chunk) workers live for the whole call and take the frames of a chunk one by one from an atomic counter, so a
// slow frame or a descheduled thread does not hold the chunk up.  read(worker, k, i) reads frame i of chunk k; `worker` indexes the
// caller's per-thread scratch.  It returns false to take no further frames of chunk k on that worker.
//
//   start()     MDC_OK, or MDC_ERR_IO with "<who>: cannot start decode threads (<what>)"
//   wait(k)     returns once every worker is done with chunk k; what read wrote for chunk k is visible to the caller then
//   release(k)  the caller is done with chunk k's slot: the workers may read chunk k + 2 into it
//
// The destructor stops the workers and joins them, whatever chunk the caller stopped at.
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <exception>
#include <functional>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

#include "mdc_internal.h"

class mdc_feed_pool {
public:
    using read_fn = std::function<bool(int worker, int k, int i)>;

    mdc_feed_pool(int count, int chunk, int threads, read_fn read)
        : count_(count), chunk_(chunk), chunks_((count + chunk - 1) / chunk), workers_(std::min(threads, std::min(count, chunk))),
          read_(std::move(read)), done_(static_cast<size_t>(chunks_), 0), next_(static_cast<size_t>(chunks_)) {
        for (auto& a : next_) a.store(0, std::memory_order_relaxed);
    }
    ~mdc_feed_pool() { stop(); }

    int workers() const { return workers_; }
    int chunks() const { return chunks_; }

    int start(const char* who) {
        try {
            for (int t = 0; t < workers_; ++t) pool_.emplace_back(&mdc_feed_pool::work, this, t);
        } catch (const std::exception& e) {
            stop();
            mdc_set_error("%s: cannot start decode threads (%s)", who, e.what());
            return MDC_ERR_IO;
        }
        return MDC_OK;
    }
    void wait(int k) {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return done_[static_cast<size_t>(k)] == workers_; });
    }
    void release(int k) {
        {
            std::lock_guard<std::mutex> lk(mu_);
            released_ = k + 2;
        }
        cv_.notify_all();
    }

private:
    void work(int t) {
        for (int k = 0; k < chunks_; ++k) {
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return abort_ || k <= released_; });
                if (abort_) return;
            }
            const int n = std::min(chunk_, count_ - k * chunk_);
            for (int i; (i = next_[static_cast<size_t>(k)].fetch_add(1, std::memory_order_relaxed)) < n;)
                if (!read_(t, k, i)) break;
            std::lock_guard<std::mutex> lk(mu_);
            ++done_[static_cast<size_t>(k)];
            cv_.notify_all();
        }
    }
    // wakes the workers that wait for a slot the caller will not release, and joins every worker
    void stop() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            abort_ = true;
        }
        cv_.notify_all();
        for (auto& th : pool_) th.join();
        pool_.clear();
    }

    const int count_, chunk_, chunks_, workers_;
    const read_fn read_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::vector<int> done_;                    // workers finished with chunk k
    std::vector<std::atomic<int>> next_;       // next frame of chunk k nobody has taken yet
    int released_ = 1;                         // chunks whose slot may be written: 0 .. released_ (both slots are free at the start)
    bool abort_ = false;
    std::vector<std::thread> pool_;
};
