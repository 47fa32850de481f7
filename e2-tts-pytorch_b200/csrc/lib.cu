// Library-wide state of libb200e2tts.so (error string, launch counter, version).
#include "common.cuh"

namespace b200 {
thread_local char g_err[512] = {0};
std::atomic<uint64_t> g_launches{0};
}  // namespace b200

namespace b200 {
__global__ void seed_advance_kernel(unsigned long long* w) {
    unsigned long long z = *w + 0x9E3779B97F4A7C15ull;   // splitmix64 step: successive replays of a graph see unrelated seeds
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    *w = z ^ (z >> 31);
}
}  // namespace b200

extern "C" int b200_seed_advance(uint64_t* seed_dev, b200_stream_t stream) {
    B200_REQUIRE(seed_dev, "seed_advance: null pointer");
    b200::seed_advance_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<unsigned long long*>(seed_dev));
    return b200::check_launch("seed_advance_kernel");
}

extern "C" const char* b200_last_error(void) { return b200::g_err; }
extern "C" int b200_version(void) { return 90; }   // the compute capability the library is built for (sm_90a)
extern "C" uint64_t b200_launch_count(void) { return b200::g_launches.load(); }
