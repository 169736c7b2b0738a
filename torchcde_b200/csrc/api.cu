// Error plumbing, device queries and the solve-variant switch behind the C ABI (include/torchcde_b200.h).
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

static int g_solve_variant = kVariantAuto;
int current_solve_variant() { return g_solve_variant; }

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

extern "C" int tcde_set_solve_variant(int variant) {
    using namespace tcde;
    TCDE_CHECK_ARG(variant >= 0 && (variant & 15) <= 6,
                   "variant=%d (0 auto, 1 CUDA-core kernel, 3 / 4 tensor-core kernel with the 3xTF32 / 2xFP16 operand split; "
                   "2, 6 / 5 are aliases of 3 / 4)", variant);
    // bits above 15 (profiling switches of earlier kernels) are accepted and ignored; 2, 6 and 5 are aliases from the
    // development history
    static const SolveVariant canonical[7] = {kVariantAuto, kVariantSimt, kVariantTf32, kVariantTf32,
                                              kVariantFp16, kVariantFp16, kVariantTf32};
    g_solve_variant = canonical[variant & 15];
    return TCDE_OK;
}
