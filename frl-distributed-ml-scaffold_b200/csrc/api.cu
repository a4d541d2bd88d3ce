// Library-level entry points: version, error string, launch counter, device queries.
#include <atomic>
#include <stdarg.h>
#include <string.h>

#include "frl_common.cuh"

namespace frl {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int after_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
        return static_cast<int>(e);
    }
    return 0;
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

}  // namespace frl

extern "C" int frl_abi_version(void) { return FRL_ABI_VERSION; }
extern "C" const char* frl_last_error(void) { return frl::g_err; }
extern "C" uint64_t frl_launch_count(void) { return frl::g_launches.load(std::memory_order_relaxed); }
extern "C" void frl_launch_count_reset(void) { frl::g_launches.store(0, std::memory_order_relaxed); }

extern "C" int frl_device_sm_count(void) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    return n;
}

extern "C" int frl_device_arch(void) {
    int dev = 0, major = 0, minor = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return -1;
    return major * 10 + minor;
}
