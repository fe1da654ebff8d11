// Shared device/host helpers for the artdeco_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define ADB_OK 0
#define ADB_ERR_INVALID 1   // bad argument (null pointer, negative size, unsupported shape)
#define ADB_ERR_CUDA 2      // a CUDA runtime call or launch failed
#define ADB_ERR_WORKSPACE 3 // caller-provided workspace too small

#define ADB_API extern "C" __attribute__((visibility("default")))

// Records the last CUDA error string for adb_last_error().
void adb_set_error(const char* where, cudaError_t e);
void adb_set_error_msg(const char* msg);

#define ADB_CHECK_LAUNCH(where)                                  \
    do {                                                         \
        cudaError_t _e = cudaGetLastError();                     \
        if (_e != cudaSuccess) { adb_set_error(where, _e); return ADB_ERR_CUDA; } \
    } while (0)

#define ADB_CUDA(call)                                           \
    do {                                                         \
        cudaError_t _e = (call);                                 \
        if (_e != cudaSuccess) { adb_set_error(#call, _e); return ADB_ERR_CUDA; } \
    } while (0)

#define ADB_REQUIRE(cond, msg)                                   \
    do { if (!(cond)) { adb_set_error_msg(msg); return ADB_ERR_INVALID; } } while (0)

static inline int adb_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

#ifdef __cplusplus
#include <mutex>
// One-time, PER-DEVICE launch setup (cudaFuncSetAttribute is a per-device property and the SM count differs between
// devices: a process may drive several GPUs, as the reference allows with --device_mapper / device_backend).
// Keyed by the current device ordinal; the mutex makes the first call on each device thread-safe.
struct AdbDeviceOnce {
    static constexpr int MAX_DEV = 64;
    std::mutex mu;
    bool done[MAX_DEV] = {};
    int sms[MAX_DEV] = {};
    // Runs `setup()` (returns an ADB status) the first time the CURRENT device is seen; *num_sms = its SM count.
    template <class F>
    int ensure(F&& setup, int* num_sms = nullptr) {
        int dev = 0;
        ADB_CUDA(cudaGetDevice(&dev));
        ADB_REQUIRE(dev >= 0 && dev < MAX_DEV, "device ordinal out of range");
        std::lock_guard<std::mutex> lk(mu);
        if (!done[dev]) {
            ADB_CUDA(cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev));
            const int rc = setup();
            if (rc != ADB_OK) return rc;
            done[dev] = true;
        }
        if (num_sms) *num_sms = sms[dev];
        return ADB_OK;
    }
};
#endif

__device__ __forceinline__ float adb_warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// Streaming (read-once) 128-bit load that does not pollute L1.
__device__ __forceinline__ float4 adb_ldg_stream4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
