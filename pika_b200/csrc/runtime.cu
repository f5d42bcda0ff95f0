// Library-wide runtime helpers: last-error string, launch counter, SM count.
#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;           // the H100 SXM's count, should the query fail
    }
    return n;
}
}  // namespace pk

extern "C" const char* pk_last_error(void) { return pk::g_err; }
extern "C" int pk_version(void) { return 104; }
extern "C" long long pk_launch_count(void) { return pk::g_launches.load(); }
