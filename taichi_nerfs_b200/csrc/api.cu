// api.cu — library-level entry points: version, per-thread error string, launch counter.
#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "common.cuh"

namespace {
thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};
}  // namespace

namespace ngp {

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;  // H100 SXM
    }
    return cached;
}

}  // namespace ngp

extern "C" {

int ngp_version(void) { return 100; }  // 0.1.0

const char* ngp_last_error(void) { return g_err; }

int64_t ngp_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
