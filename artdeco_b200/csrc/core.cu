// Library-wide state for the C ABI: last-error string, version, device probe.
#include "common.cuh"
#include <stdio.h>
#include <string.h>

static thread_local char g_err[512] = "";

void adb_set_error(const char* where, cudaError_t e) {
    snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}
void adb_set_error_msg(const char* msg) {
    strncpy(g_err, msg, sizeof(g_err) - 1);
    g_err[sizeof(g_err) - 1] = 0;
}

ADB_API const char* adb_last_error(void) { return g_err; }

ADB_API int adb_version(void) { return 100; }

// Returns ADB_OK iff the current device is compute capability 9.0 (the library holds sm_90a code only).
ADB_API int adb_check_device(void) {
    int dev = 0;
    ADB_CUDA(cudaGetDevice(&dev));
    int major = 0, minor = 0;
    ADB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    ADB_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) {
        snprintf(g_err, sizeof(g_err), "artdeco_b200 is built for sm_90a only; device is sm_%d%d", major, minor);
        return ADB_ERR_INVALID;
    }
    return ADB_OK;
}
