// Library-level entry points: version, last error, device info.
#include <cstdarg>
#include <cstdio>
#include "dc_common.cuh"

static thread_local char g_err[512] = "";

void dc_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int dc_sm_count() {
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

extern "C" {

int dc_version(void) { return 116; }

const char *dc_last_error(void) { return g_err; }

int dc_device_info(int *sm_count, int *cc_major, int *cc_minor) {
    int dev = 0;
    DC_CUDA(cudaGetDevice(&dev));
    int v = 0;
    if (sm_count) { DC_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev)); *sm_count = v; }
    if (cc_major) { DC_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev)); *cc_major = v; }
    if (cc_minor) { DC_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev)); *cc_minor = v; }
    return DC_OK;
}

}  // extern "C"
