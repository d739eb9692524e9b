// The sequence reader's decode-ahead host feed (mdc_seq_prepare, csrc/mdc_sequence.cpp) without a GPU, under the sanitizers: the
// context is a stub whose input size is the sequence's, and the per-chunk prepare call is a fake that copies the staged 8-bit frames
// into level 0 as floats.  So level 0 of frame k must equal mdc_seq_read_gray8 of frame first + k, whatever chunk and slot it
// went through.  Built and run by tests/test_sequence_feed_host.py.
// usage:
//   seq_feed_harness range <seq dir> <threads>...       first 0 and 1, counts C-1, C, C+1 and 3C+1 for each thread count's chunk C
//   seq_feed_harness bad <seq dir> <bad id> <threads>    the bad frame at the start of the third chunk of a call of 4C frames
//   seq_feed_harness args <seq dir>                      the argument checks: codes and messages, nothing written or prepared
#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mdc_b200.h"
#include "mdc_internal.h"

// the GPU side of the library is not linked here
struct mdc_ctx { int in_w, in_h, out_w, out_h; };
static thread_local char g_err[512];
void mdc_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}
extern "C" const char* mdc_last_error(void) { return g_err; }
extern "C" int mdc_host_alloc(void** p, size_t n) { *p = malloc(n); return *p ? 0 : 1; }
extern "C" void mdc_host_free(void* p) { free(p); }
void mdc_ctx_geometry(const mdc_ctx* c, int* in_w, int* in_h, int* out_w, int* out_h) {
    *in_w = c->in_w; *in_h = c->in_h; *out_w = c->out_w; *out_h = c->out_h;
}
static int g_prepared = 0;      // frames the fake prepare call has taken
extern "C" int mdc_prepare_batch_host(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned, float* const* out_levels, int) {
    const size_t n = static_cast<size_t>(n_frames) * c->in_w * c->in_h;
    for (size_t p = 0; p < n; ++p) out_levels[0][p] = frames[p];
    g_prepared += n_frames;
    return MDC_OK;
}

namespace {

constexpr uint32_t kSentinel = 0xdeadbeefu;

[[noreturn]] void fail(const std::string& what) {
    printf("FAIL %s\n", what.c_str());
    fflush(stdout);
    std::_Exit(1);
}

int chunk_of(int threads) { return std::min(256, std::max(16, 2 * threads)); }

struct Seq {
    mdc_seq* s = nullptr;
    int n = 0, w = 0, h = 0;
    std::vector<std::vector<uint8_t>> raw;      // mdc_seq_read_gray8 of every frame (empty if it fails)
    explicit Seq(const char* dir) {
        if (mdc_seq_open(dir, &s) != MDC_OK) fail(std::string("cannot open ") + dir);
        n = mdc_seq_num_images(s);
        raw.resize(static_cast<size_t>(n));
        for (int id = 0; id < n; ++id) {
            int fw = 0, fh = 0;
            if (mdc_seq_read_gray8(s, id, nullptr, 0, &fw, &fh) != MDC_OK) continue;
            if (w == 0) { w = fw; h = fh; }
            if (fw != w || fh != h) continue;
            raw[static_cast<size_t>(id)].resize(static_cast<size_t>(fw) * fh);
            if (mdc_seq_read_gray8(s, id, raw[static_cast<size_t>(id)].data(), raw[static_cast<size_t>(id)].size(), &fw, &fh) != MDC_OK)
                fail("frame " + std::to_string(id) + " reads once and not twice");
        }
    }
    ~Seq() { mdc_seq_close(s); }
};

// level-0 rows for `count` frames with a guard row before and after, every word set to kSentinel
struct Out {
    size_t n_px;
    int count;
    std::vector<float> rows;
    Out(size_t n_px_, int count_) : n_px(n_px_), count(count_), rows((static_cast<size_t>(count_) + 2) * n_px_) {
        for (float& v : rows) memcpy(&v, &kSentinel, 4);
    }
    float* level0() { return rows.data() + n_px; }
    bool row_untouched(int r) const {
        for (size_t p = 0; p < n_px; ++p) {
            uint32_t u;
            memcpy(&u, &rows[static_cast<size_t>(r) * n_px + p], 4);
            if (u != kSentinel) return false;
        }
        return true;
    }
    // rows 1 .. written hold frames first .. first + written - 1; the others are untouched
    void check(const Seq& q, int first, int written, const std::string& what) const {
        for (int r = 0; r < count + 2; ++r) {
            const int k = r - 1;
            if (k < 0 || k >= written) {
                if (!row_untouched(r)) fail(what + ": row of frame " + std::to_string(k) + " was written");
                continue;
            }
            const std::vector<uint8_t>& exp = q.raw[static_cast<size_t>(first + k)];
            if (exp.size() != n_px) fail(what + ": frame " + std::to_string(first + k) + " has no expectation");
            for (size_t p = 0; p < n_px; ++p)
                if (rows[static_cast<size_t>(r) * n_px + p] != static_cast<float>(exp[p]))
                    fail(what + ": frame " + std::to_string(k) + " (entry " + std::to_string(first + k) + ") differs at pixel " + std::to_string(p));
        }
    }
};

int run_range(const char* dir, const std::vector<int>& threads) {
    Seq q(dir);
    mdc_ctx ctx{q.w, q.h, q.w, q.h};
    const size_t n_px = static_cast<size_t>(q.w) * q.h;
    int calls = 0;
    for (int t : threads) {
        const int c = chunk_of(t);
        for (int first : {0, 1})
            for (int count : {c - 1, c, c + 1, 3 * c + 1}) {
                const std::string what = "threads " + std::to_string(t) + " (chunk " + std::to_string(c) + ") first " + std::to_string(first) +
                                         " count " + std::to_string(count);
                if (first + count > q.n) fail(what + ": the sequence has only " + std::to_string(q.n) + " frames");
                Out out(n_px, count);
                float* lv = out.level0();
                const int before = g_prepared;
                const int rc = mdc_seq_prepare(&ctx, q.s, first, count, 0, &lv, 1, t);
                if (rc != MDC_OK) fail(what + ": rc " + std::to_string(rc) + ": " + mdc_last_error());
                if (g_prepared - before != count) fail(what + ": " + std::to_string(g_prepared - before) + " frames prepared");
                out.check(q, first, count, what);
                ++calls;
            }
    }
    printf("range: %d calls passed\n", calls);
    return 0;
}

int run_bad(const char* dir, int bad, int threads) {
    Seq q(dir);
    mdc_ctx ctx{q.w, q.h, q.w, q.h};
    const int c = chunk_of(threads), first = bad - 2 * c, count = 4 * c;
    if (first < 0 || first + count > q.n) fail("the bad frame is not at the start of a third chunk inside the sequence");
    Out out(static_cast<size_t>(q.w) * q.h, count);
    float* lv = out.level0();
    const int rc = mdc_seq_prepare(&ctx, q.s, first, count, 0, &lv, 1, threads);
    const std::string err = mdc_last_error();
    if (rc != MDC_ERR_FORMAT) fail("rc " + std::to_string(rc) + " instead of MDC_ERR_FORMAT: " + err);
    if (err.rfind("mdc_seq_prepare: ", 0) != 0 || err.find(mdc_seq_name(q.s, bad)) == std::string::npos)
        fail("the message does not name the bad entry: " + err);
    if (g_prepared != 2 * c) fail(std::to_string(g_prepared) + " frames prepared");
    out.check(q, first, 2 * c, "bad frame " + std::to_string(bad));
    printf("bad: %s\n", err.c_str());
    return 0;
}

int run_args(const char* dir) {
    Seq q(dir);
    mdc_ctx ctx{q.w, q.h, q.w, q.h}, none{0, 0, 0, 0}, rect{q.w, q.h, 1, 1};
    const int n = q.n;
    Out out(static_cast<size_t>(q.w) * q.h, 4);
    std::vector<float> level1(static_cast<size_t>(4 * (q.w / 2) * (q.h / 2)));
    float* two[2] = {out.level0(), level1.data()};
    float* null1[2] = {out.level0(), nullptr};
    const std::string N = std::to_string(n);
    struct Case { mdc_ctx* c; const mdc_seq* s; int first, count; unsigned flags; float* const* lv; int levels; int rc; std::string msg; };
    const Case cases[] = {
        {&ctx, nullptr, 0, 4, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: bad argument"},
        {&ctx, q.s, 0, 4, 0, nullptr, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: bad argument"},
        {nullptr, nullptr, 0, 4, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: bad argument"},
        {&ctx, q.s, -1, 4, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: frames first = -1, count = 4 outside the sequence's " + N},
        {&ctx, q.s, 0, -1, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: frames first = 0, count = -1 outside the sequence's " + N},
        {&ctx, q.s, n - 3, 4, 0, two, 2, MDC_ERR_INVALID_ARG,
         "mdc_seq_prepare: frames first = " + std::to_string(n - 3) + ", count = 4 outside the sequence's " + N},
        {&ctx, q.s, 1, INT_MAX, 0, two, 2, MDC_ERR_INVALID_ARG,
         "mdc_seq_prepare: frames first = 1, count = " + std::to_string(INT_MAX) + " outside the sequence's " + N},
        {&ctx, q.s, INT_MAX, 1, 0, two, 2, MDC_ERR_INVALID_ARG,
         "mdc_seq_prepare: frames first = " + std::to_string(INT_MAX) + ", count = 1 outside the sequence's " + N},
        {&ctx, q.s, n + 1, 0, 0, two, 2, MDC_ERR_INVALID_ARG,
         "mdc_seq_prepare: frames first = " + std::to_string(n + 1) + ", count = 0 outside the sequence's " + N},
        {&ctx, q.s, 0, 4, 0, two, 0, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: 0 pyramid levels (1..8)"},
        {&ctx, q.s, 0, 4, 0, two, 9, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: 9 pyramid levels (1..8)"},
        // the checks that need no context come first
        {nullptr, q.s, -1, 4, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: frames first = -1, count = 4 outside the sequence's " + N},
        {nullptr, q.s, 0, 4, 0, two, 0, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: 0 pyramid levels (1..8)"},
        {&none, q.s, 0, 4, 0, two, 9, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: 9 pyramid levels (1..8)"},
        {nullptr, q.s, 0, 4, 0, two, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: bad argument"},
        {&none, q.s, 0, 4, 0, two, 2, MDC_ERR_INVALID_OBJECT, "mdc_seq_prepare: context has no image geometry"},
        {&none, q.s, 0, 0, 0, two, 2, MDC_ERR_INVALID_OBJECT, "mdc_seq_prepare: context has no image geometry"},
        {&ctx, q.s, 0, 4, 0, null1, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: output level 1 is NULL"},
        {&ctx, q.s, 0, 0, 0, null1, 2, MDC_ERR_INVALID_ARG, "mdc_seq_prepare: output level 1 is NULL"},
        // rectifying to 1 x 1: level 1 has no pixels and may be NULL; count = 0 prepares nothing
        {&rect, q.s, 2, 0, MDC_RECTIFY, null1, 2, MDC_OK, ""},
        {&ctx, q.s, n, 0, 0, two, 2, MDC_OK, ""},
    };
    int k = 0;
    for (const Case& t : cases) {
        mdc_set_error("%s", "");
        const int rc = mdc_seq_prepare(t.c, t.s, t.first, t.count, t.flags, t.lv, t.levels, 4);
        if (rc != t.rc || (t.rc != MDC_OK && t.msg != mdc_last_error()))
            fail("case " + std::to_string(k) + ": rc " + std::to_string(rc) + " \"" + mdc_last_error() + "\", expected rc " + std::to_string(t.rc) +
                 " \"" + t.msg + "\"");
        ++k;
    }
    if (g_prepared != 0) fail("an argument error prepared frames");
    for (int r = 0; r < out.count + 2; ++r)
        if (!out.row_untouched(r)) fail("an argument error wrote the output");
    printf("args: %d cases passed\n", k);
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    const std::string mode = argc > 2 ? argv[1] : "";
    if (mode == "range" && argc > 3) {
        std::vector<int> threads;
        for (int i = 3; i < argc; ++i) threads.push_back(atoi(argv[i]));
        return run_range(argv[2], threads);
    }
    if (mode == "bad" && argc == 5) return run_bad(argv[2], atoi(argv[3]), atoi(argv[4]));
    if (mode == "args" && argc == 3) return run_args(argv[2]);
    fprintf(stderr, "usage: seq_feed_harness range <dir> <threads>... | bad <dir> <bad id> <threads> | args <dir>\n");
    return 2;
}
