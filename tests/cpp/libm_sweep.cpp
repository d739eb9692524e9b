// The restated exp and log (csrc/mdc_libm.h, host build) against this process's libm, bit for bit.  Prints the glibc version and
// whether the CPU has FMA and AVX2 (which select glibc's FMA build of exp and log), then one line per sweep:
//   <name> <points> <mismatches> [first mismatching input as hex bits]
// Sweeps run on all hardware threads.  NaN results match when both are NaN.
#include <gnu/libc-version.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#include "mdc_b200.h"
#include "mdc_libm.h"

namespace {

uint64_t mix(uint64_t z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

bool same(double a, double b) { return (std::isnan(a) && std::isnan(b)) || mdc_lm_bits(a) == mdc_lm_bits(b); }

// point(i) for i in [0, n): compares op on every point
void sweep(const char* name, int op, uint64_t n, const std::function<double(uint64_t)>& point) {
    const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
    std::atomic<uint64_t> bad{0}, first{~0ull};
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; ++t)
        th.emplace_back([&, t] {
            uint64_t b = 0;
            for (uint64_t i = t; i < n; i += nt) {
                const double x = point(i);
                const double r = op == MDC_LIBM_EXP ? mdc_exp(x) : mdc_log(x);
                const double l = op == MDC_LIBM_EXP ? exp(x) : log(x);
                if (!same(r, l)) {
                    if (b++ == 0) {
                        uint64_t f = first.load();
                        while (f == ~0ull && !first.compare_exchange_weak(f, mdc_lm_bits(x))) {}
                    }
                }
            }
            bad += b;
        });
    for (auto& t : th) t.join();
    printf("%s %llu %llu", name, (unsigned long long)n, (unsigned long long)bad.load());
    if (bad) printf(" %016llx", (unsigned long long)first.load());
    printf("\n");
    fflush(stdout);
}

}  // namespace

int main(int argc, char** argv) {
    const uint64_t dense = argc > 1 ? strtoull(argv[1], nullptr, 10) : (1ull << 30);
    printf("glibc %s fma %d avx2 %d\n", gnu_get_libc_version(), __builtin_cpu_supports("fma") ? 1 : 0, __builtin_cpu_supports("avx2") ? 1 : 0);
    // exp on [0, 1]: `dense` points spread evenly, each with random low mantissa bits, then 1 itself
    sweep("exp_dense_0_1", MDC_LIBM_EXP, dense + 1, [dense](uint64_t i) {
        if (i == dense) return 1.0;
        const double step = 1.0 / static_cast<double>(dense);
        return std::nextafter(static_cast<double>(i) * step, 0.0) + step * static_cast<double>(mix(i) >> 11) * 0x1p-53;
    });
    // exp: the points where the reduction x * 128 / ln 2 crosses k + 1/2 (the table index changes), +-4096 ulps around each
    sweep("exp_table_boundaries", MDC_LIBM_EXP, 200ull * 8193, [](uint64_t i) {
        const double c = (static_cast<double>(i / 8193) + 0.5) * 0.0054152123481245725;      // ln 2 / 128
        return mdc_lm_dbl(mdc_lm_bits(c) + (i % 8193) - 4096);
    });
    // exp over its whole finite range, including the over- and underflow paths and the subnormal results
    sweep("exp_wide", MDC_LIBM_EXP, 1ull << 26, [](uint64_t i) { return -760.0 + 1480.0 * static_cast<double>(mix(i) >> 11) * 0x1p-53; });
    sweep("exp_tiny", MDC_LIBM_EXP, 1ull << 22, [](uint64_t i) {
        return mdc_lm_dbl((mix(i) & 0x800fffffffffffffull) | (static_cast<uint64_t>(0x380 + (i % 0x80)) << 52));
    });
    // log on [20, DBL_MAX]: every binade from 16 up, random mantissas, and +-64 ulps around each of the 128 table subintervals' edges
    sweep("log_20_max", MDC_LIBM_LOG, 1021ull << 18, [](uint64_t i) {
        const uint64_t e = 0x403 + (i >> 18);
        double x = mdc_lm_dbl((e << 52) | (mix(i) & 0xfffffffffffffull));
        return x < 20.0 ? x + 4.0 : x;
    });
    sweep("log_table_edges", MDC_LIBM_LOG, 1021ull * 128 * 129, [](uint64_t i) {
        const uint64_t e = 0x403 + i / (128 * 129), j = (i / 129) % 128;
        const uint64_t edge = ((e << 52) | 0x6000000000000ull) + (j << 45);    // ix - OFF crosses a multiple of 2^45
        const double x = mdc_lm_dbl(edge + (i % 129) - 64);
        return x < 20.0 ? 20.0 : x;
    });
    // log's other paths: near 1, below 20, subnormals, negatives
    sweep("log_near_1", MDC_LIBM_LOG, 1ull << 24, [](uint64_t i) { return 0.9375 + 0.1272 * static_cast<double>(mix(i) >> 11) * 0x1p-53; });
    sweep("log_all_binades", MDC_LIBM_LOG, 1ull << 24, [](uint64_t i) { return mdc_lm_dbl(mix(i) & 0x7fffffffffffffffull); });
    sweep("log_subnormal", MDC_LIBM_LOG, 1ull << 20, [](uint64_t i) { return mdc_lm_dbl(mix(i) & 0x000fffffffffffffull); });
    static const double special[] = {0.0, -0.0, INFINITY, -INFINITY, NAN, -NAN, 1.0, -1.0, 20.0, 5e-324, 2.2250738585072014e-308,
                                     1.7976931348623157e308, -1e-300, 0.9375, 1.0 + 0x1.09p-4, 709.782712893384, -745.1332191019412, 1e-300};
    const size_t ns = sizeof special / sizeof special[0];
    sweep("exp_special", MDC_LIBM_EXP, ns, [](uint64_t i) { return special[i]; });
    sweep("log_special", MDC_LIBM_LOG, ns, [](uint64_t i) { return special[i]; });
    return 0;
}
