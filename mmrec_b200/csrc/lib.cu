// Library-wide plumbing: error string, device check, SM count.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace mmrec {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

long long g_launches = 0;

}  // namespace mmrec

extern "C" int mmrec_abi_version(void) { return MMREC_ABI_VERSION; }

extern "C" int64_t mmrec_launch_count(void) { return (int64_t)mmrec::g_launches; }

extern "C" const char* mmrec_last_error(void) { return mmrec::g_err; }

extern "C" int mmrec_device_check(void) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
        mmrec::set_error("device_check: no CUDA device: %s", cudaGetErrorString(cudaGetLastError()));
        return MMREC_ECUDA;
    }
    if (major != 9) {
        mmrec::set_error("device_check: compute capability %d.x, this library carries sm_90a code only", major);
        return MMREC_EUNSUPPORTED;
    }
    return MMREC_OK;
}
