// Library-level entry points: version, thread-local error string, device check.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include <stdarg.h>

static thread_local char g_err[1024] = "";

void br_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" {

int br_version(void) { return 100; }

int br_last_error(char* buf, size_t n) {
    if (!buf || !n) return (int)strlen(g_err);
    strncpy(buf, g_err, n - 1);
    buf[n - 1] = 0;
    return (int)strlen(buf);
}

int br_device_ok(void) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { br_set_error("no CUDA device"); return 0; }
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (major != 9) { br_set_error("libbioreason_b200 targets sm_90a only (found sm_%d)", major * 10); return 0; }
    return 1;
}

}  // extern "C"
