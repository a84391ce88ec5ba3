// api.cu -- ABI version and the thread-local error message of libo3dml_b200.
#include "../../include/o3dml_b200.h"
#include "common.cuh"
#include <stdarg.h>
#include <atomic>

static thread_local char g_err[512] = "";

extern "C" void o3dml_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* o3dml_last_error(void) { return g_err; }
extern "C" int o3dml_abi_version(void) { return O3DML_ABI_VERSION; }

static std::atomic<unsigned long long> g_launches{0};
void o3dml::count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" void o3dml_launch_count_add(unsigned long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" unsigned long long o3dml_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
