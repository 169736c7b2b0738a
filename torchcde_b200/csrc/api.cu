// Error plumbing and device queries behind the C ABI (include/torchcde_b200.h).
#include <stdarg.h>

#include "common.cuh"

namespace tcde {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

int cuda_failed(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return TCDE_ERR_CUDA;
}

// SMs of the current device; 132 (an H100 SXM) only if the runtime cannot say, which the launches that follow report
int sm_count() {
    constexpr int kFallback = 132;
    static thread_local int cached_dev = -1;
    static thread_local int cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return kFallback;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = kFallback;
        cached = n;
        cached_dev = dev;
    }
    return cached;
}

}  // namespace tcde

extern "C" int tcde_abi_version(void) { return TCDE_ABI_VERSION; }

extern "C" const char* tcde_last_error(void) { return tcde::g_error; }

extern "C" int tcde_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    TCDE_CHECK_CUDA(cudaGetDevice(&dev));
    int n = 0, major = 0, minor = 0;
    TCDE_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    TCDE_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    TCDE_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (sm_count) *sm_count = n;
    if (cc_major) *cc_major = major;
    if (cc_minor) *cc_minor = minor;
    return TCDE_OK;
}
