// Library-level entry points: version, thread-local error text, launch counter.
#include "common.cuh"
#include <atomic>

namespace effdet {

static thread_local char g_err[768] = "";
static std::atomic<unsigned long long> g_launches{0};

char* err_buf() { return g_err; }

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

}  // namespace effdet

extern "C" int effdet_version(void) { return 101; }
extern "C" const char* effdet_last_error(void) { return effdet::err_buf(); }
extern "C" uint64_t effdet_launch_count(void) { return effdet::g_launches.load(std::memory_order_relaxed); }
extern "C" void effdet_reset_launch_count(void) { effdet::g_launches.store(0, std::memory_order_relaxed); }
