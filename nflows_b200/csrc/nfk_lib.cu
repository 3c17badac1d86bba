// Library-level entry points of the C ABI (include/nfk.h).
#include <stdarg.h>

#include "nfk_common.cuh"

namespace nfk {
thread_local char g_last_error[512] = "";
std::atomic<int64_t> g_launch_count{0};

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
    return code;
}
}  // namespace nfk

extern "C" {

int nfk_version(void) { return NFK_ABI_VERSION; }

const char* nfk_last_error(void) { return nfk::g_last_error; }

int64_t nfk_launch_count(void) { return nfk::g_launch_count.load(); }

int nfk_check_device(void) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return nfk::fail(NFK_E_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
    int major = 0;
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e != cudaSuccess) return nfk::fail(NFK_E_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
    if (major != 9) return nfk::fail(NFK_E_UNSUPPORTED, "libnfk_sm90 needs compute capability 9.x (sm_90a), found %d.x", major);
    return NFK_OK;
}

}  // extern "C"
