// The decode-ahead pool of the sequence feeds (csrc/mdc_feed.h) under ThreadSanitizer, with a read function that writes a tag per
// frame into the slot of its chunk.  For every thread count, chunk size and frame count of the sweep, three consumers:
//   all      waits for every chunk, checks it, and releases it;
//   fail     as all, but one frame's read returns false: its worker takes no further frame of that chunk, the others finish it;
//   stop     waits for chunk j and returns without releasing it: the pool's destructor must still join every worker.
// Checked: every frame is read exactly once; no chunk k + 2 is read before release(k); a chunk's slot holds the tags of its own
// frames at wait(k) and has the same checksum just before release(k), after a sleep.  Data races are ThreadSanitizer's to report.
// Built and run by tests/test_feed_pool.py.  usage: feed_pool_harness
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "mdc_feed.h"

static char g_err[512];
void mdc_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

namespace {

enum Mode { kAll, kFail, kStop };
const char* const kModeName[] = {"all", "fail", "stop"};

uint64_t tag(int k, int i) { return (static_cast<uint64_t>(k) << 32) ^ static_cast<uint64_t>(i) ^ 0x5a5a000000005a5aull; }

[[noreturn]] void fail(const char* what, int threads, int chunk, int count, Mode mode, int k, int i) {
    printf("FAIL %s: threads %d chunk %d count %d mode %s, chunk %d frame %d\n", what, threads, chunk, count, kModeName[mode], k, i);
    fflush(stdout);
    std::_Exit(1);
}

void run(int threads, int chunk, int count, Mode mode) {
    const int chunks = (count + chunk - 1) / chunk;
    const int fail_k = chunks > 1 ? 1 : 0;                                   // kFail: the frame whose read returns false
    const int fail_i = (std::min(chunk, count - fail_k * chunk)) / 2;
    const int stop_at = chunks > 1 ? 1 : 0;                                  // kStop: the chunk the consumer stops at
    std::vector<uint64_t> slot[2] = {std::vector<uint64_t>(static_cast<size_t>(chunk)), std::vector<uint64_t>(static_cast<size_t>(chunk))};
    std::vector<std::atomic<int>> reads(static_cast<size_t>(count));
    std::vector<std::atomic<int>> stopped(static_cast<size_t>(chunks));     // the worker whose read returned false in chunk k, or -1
    for (auto& a : reads) a.store(0);
    for (auto& a : stopped) a.store(-1);
    std::atomic<int> released{1};             // the consumer's own record of release(k): k + 2, stored before the call
    {
        mdc_feed_pool pool(count, chunk, threads, [&](int t, int k, int i) {
            if (k > released.load(std::memory_order_acquire)) fail("chunk read before its slot was released", threads, chunk, count, mode, k, i);
            if (stopped[static_cast<size_t>(k)].load() == t) fail("frame taken after read returned false", threads, chunk, count, mode, k, i);
            reads[static_cast<size_t>(k * chunk + i)].fetch_add(1);
            slot[k & 1][static_cast<size_t>(i)] = tag(k, i);
            if ((k + i) % 7 == 0) std::this_thread::yield();
            if (mode == kFail && k == fail_k && i == fail_i) { stopped[static_cast<size_t>(k)].store(t); return false; }
            return true;
        });
        if (pool.chunks() != chunks || pool.workers() != std::min(threads, std::min(count, chunk)))
            fail("chunk or worker count", threads, chunk, count, mode, -1, -1);
        if (pool.start("feed_pool_harness") != MDC_OK) fail(g_err, threads, chunk, count, mode, -1, -1);
        const int workers = pool.workers();
        for (int k = 0; k < chunks; ++k) {
            pool.wait(k);
            if (mode == kStop && k == stop_at) break;
            const int n = std::min(chunk, count - k * chunk);
            uint64_t sum = 0;
            for (int i = 0; i < n; ++i) {
                // with one worker, the frames after the failing one are left unread
                const bool unread = mode == kFail && k == fail_k && i > fail_i && workers == 1;
                if (reads[static_cast<size_t>(k * chunk + i)].load() != (unread ? 0 : 1)) fail("frame not read exactly once", threads, chunk, count, mode, k, i);
                if (!unread && slot[k & 1][static_cast<size_t>(i)] != tag(k, i)) fail("slot holds another frame", threads, chunk, count, mode, k, i);
                sum += slot[k & 1][static_cast<size_t>(i)] * static_cast<uint64_t>(2 * i + 1);
            }
            if (k % 3 == 0) std::this_thread::sleep_for(std::chrono::microseconds(200));
            else std::this_thread::yield();
            uint64_t again = 0;
            for (int i = 0; i < n; ++i) again += slot[k & 1][static_cast<size_t>(i)] * static_cast<uint64_t>(2 * i + 1);
            if (again != sum) fail("slot changed between wait and release", threads, chunk, count, mode, k, -1);
            released.store(k + 2, std::memory_order_release);
            pool.release(k);
        }
    }      // the pool joins its workers here
    if (mode == kStop)
        for (int f = (stop_at + 2) * chunk; f < count; ++f)
            if (reads[static_cast<size_t>(f)].load() != 0) fail("chunk read after the consumer stopped", threads, chunk, count, mode, f / chunk, f % chunk);
}

}  // namespace

int main() {
    int runs = 0;
    for (int threads : {1, 2, 3, 8, 64})
        for (int chunk : {1, 2, 16, 256}) {
            std::vector<int> counts;
            for (int c : {0, 1, chunk - 1, chunk, chunk + 1, 3 * chunk + 1})
                if (c >= 0 && std::find(counts.begin(), counts.end(), c) == counts.end()) counts.push_back(c);
            for (int count : counts)
                for (Mode mode : {kAll, kFail, kStop}) {
                    if (mode != kAll && count == 0) continue;
                    run(threads, chunk, count, mode);
                    ++runs;
                }
        }
    printf("feed pool: %d runs passed\n", runs);
    return 0;
}
