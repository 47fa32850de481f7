// Shared host-side helpers of libb200e2tts.so: error reporting, launch accounting, launch checks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

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

// Programmatic dependent launch needs a `make PDL=1` build AND B200_PDL=1 at run time: with it every library kernel is launched through
// cudaLaunchKernelEx with cudaLaunchAttributeProgrammaticStreamSerialization, without it through the plain <<< >>> launch.
#ifndef B200_PDL_BUILD
#define B200_PDL_BUILD 0
#endif
inline bool pdl_enabled() {
#if B200_PDL_BUILD
    static const bool on = getenv("B200_PDL") && atoi(getenv("B200_PDL")) != 0;
    return on;
#else
    return false;   // the kernels of this build do not execute griddepcontrol.wait: never launch them as programmatic dependents
#endif
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// B200_LAUNCH((kernel<...>), grid, block, smem, stream, args...) — errors surface through check_launch() as before
#define B200_LAUNCH(kern, grid, block, smem, st, ...)                                  \
    do {                                                                               \
        if (b200::pdl_enabled()) (void)b200::launch_pdl(kern, grid, block, smem, st, __VA_ARGS__); \
        else kern<<<grid, block, smem, st>>>(__VA_ARGS__);                             \
    } while (0)

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
