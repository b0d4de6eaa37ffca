// Library-level entry points: version, thread-local error string, device query,
// workspace initialisation.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

void slb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int slb_sms() {
    static thread_local int cached_dev = -1;
    static thread_local int cached_sms = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached_dev = dev;
        cached_sms = n;
    }
    return cached_sms;
}

extern "C" {

int slb_version(void) { return SLB_VERSION; }

const char* slb_last_error(void) { return g_err; }

int slb_sm_count(void) { return slb_sms(); }

int slb_workspace_init(void* workspace, size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(workspace != nullptr || workspace_bytes == 0, "workspace_init: null workspace");
    if (workspace_bytes == 0) return SLB_OK;
    cudaError_t e = cudaMemsetAsync(workspace, 0, workspace_bytes, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) {
        slb_set_error("workspace_init: %s", cudaGetErrorString(e));
        return SLB_ECUDA;
    }
    return SLB_OK;
}

}  // extern "C"
