// Shared host-side helpers of libb200e2tts.so: error reporting, launch accounting, launch checks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <mutex>

#include "../../include/b200_e2tts.h"

namespace b200 {

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

#define B200_FAIL(...)                                   \
    do {                                                 \
        snprintf(b200::g_err, sizeof(b200::g_err), __VA_ARGS__); \
        return -1;                                       \
    } while (0)

#define B200_REQUIRE(cond, ...) \
    do {                        \
        if (!(cond)) B200_FAIL(__VA_ARGS__); \
    } while (0)

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

constexpr int kMaxDevices = 64;
inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
// SM count of the CURRENT device (cached per device: a process may drive several GPUs)
inline int num_sms() {
    static std::atomic<int> cache[kMaxDevices];
    const int dev = current_device();
    int n = cache[dev].load(std::memory_order_relaxed);
    if (!n) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;   // H100 SXM
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
// One-time, per-device kernel attribute (cudaFuncSetAttribute applies to the current device's context): SURVEY §8b asks for
// std::once_flag-guarded initialisation because autograd / DDP call the library from several threads.
struct DeviceOnce {
    std::once_flag flag[kMaxDevices];
    cudaError_t err[kMaxDevices] = {};
};
template <typename K>
inline cudaError_t set_max_smem_once(DeviceOnce& once, K kern, int bytes) {
    const int dev = current_device();
    std::call_once(once.flag[dev], [&] { once.err[dev] = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); });
    return once.err[dev];
}

}  // namespace b200
