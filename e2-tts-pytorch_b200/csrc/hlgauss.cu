// HL-Gauss classification head of DurationPredictor(hl_gauss_loss=..., use_regression=False) (e2_tts.py:966-967, 1035-1040, 1107,
// 1111; hl-gauss-pytorch HLGaussLoss, SURVEY A.6) on the fp32 logits b200_small_linear writes. One CTA per item: the Gaussian
// histogram of the target, a max-shifted log-softmax, the soft-target cross-entropy and the saved softmax - p in one pass; the batch
// mean is taken by the last CTA in item order, so the loss has the same bits on every launch.
#include "common.cuh"

namespace b200 {

constexpr int HG_THREADS = 256;
constexpr int HG_MAX_BINS = 4096;   // one item's exp(l - max) is held in shared memory (16 KB)
constexpr int HG_MAX_B = 64;        // the row limit of b200_small_linear, which computes the logits

// warp xor trees, then warp 0 combines the 8 warp results in a fixed tree: the same bits for the same inputs on every launch
__device__ __forceinline__ float hg_block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();   // the previous reduction's result has been read
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float s = lane < HG_THREADS / 32 ? red[lane] : 0.f;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[HG_THREADS / 32] = s;
    }
    __syncthreads();
    return red[HG_THREADS / 32];
}
__device__ __forceinline__ float hg_block_max(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float s = lane < HG_THREADS / 32 ? red[lane] : -INFINITY;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) s = fmaxf(s, __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) red[HG_THREADS / 32] = s;
    }
    __syncthreads();
    return red[HG_THREADS / 32];
}

// erf(b) - erf(a) for a <= b. Where both lie on one side of 0 it is taken as a difference of erfc values, which keeps the relative
// accuracy of a bin far in a tail (there erf(b) - erf(a) cancels to a few ulps of 1).
__device__ __forceinline__ float hg_erf_diff(float a, float b) {
    if (a >= 0.f) return erfcf(a) - erfcf(b);
    if (b <= 0.f) return erfcf(-b) - erfcf(-a);
    return erff(b) - erff(a);
}
// bin edge j of linspace(min, max, num_bins + 1): min + j * bin_size rounded once, the last edge max itself
__device__ __forceinline__ float hg_edge(const b200_hl_gauss_args& a, float bin, int j) {
    return j == a.num_bins ? a.max_value : fmaf((float)j, bin, a.min_value);
}

__global__ void __launch_bounds__(HG_THREADS) hl_gauss_fwd_kernel(const b200_hl_gauss_args a) {
    __shared__ float se[HG_MAX_BINS];   // exp(l - max)
    __shared__ float red[HG_THREADS / 32 + 1];
    const int b = blockIdx.x, nb = a.num_bins, tid = threadIdx.x;
    const float* l = a.logits + (size_t)b * nb;
    const float bin = (a.max_value - a.min_value) / (float)nb;
    float m = -INFINITY;
    for (int i = tid; i < nb; i += HG_THREADS) m = fmaxf(m, l[i]);
    m = hg_block_max(m, red);
    float s = 0.f;
    for (int i = tid; i < nb; i += HG_THREADS) {
        const float e = expf(l[i] - m);
        se[i] = e;
        s += e;
    }
    const float S = hg_block_sum(s, red);   // its barriers also publish se
    if (!a.target) {   // prediction: sum_i softmax_i * centre_i (e2_tts.py:1107)
        float acc = 0.f;
        for (int i = tid; i < nb; i += HG_THREADS) acc += (se[i] / S) * ((hg_edge(a, bin, i) + hg_edge(a, bin, i + 1)) * 0.5f);
        acc = hg_block_sum(acc, red);
        if (tid == 0) a.pred[b] = acc;
        return;
    }
    float y = a.target[b];
    if (a.clamp_to_range) y = fminf(fmaxf(y, a.min_value), a.max_value);
    const float s2 = a.sigma * 1.41421356f;   // sqrt(2) sigma
    const float x0 = (a.min_value - y) / s2, xn = (a.max_value - y) / s2;
    // the reference normalises by z = erf(x_N) - erf(x_0) in fp32, which is 0 (its loss NaN) for a target so far outside the support
    // that both erf values round to the same +-1; the masses themselves are taken through erfc
    const float z = (erff(xn) - erff(x0) == 0.f) ? __int_as_float(0x7fc00000) : hg_erf_diff(x0, xn);
    const float logS = logf(S);
    float ce = 0.f;
    float* diff = a.diff + (size_t)b * nb;
    for (int i = tid; i < nb; i += HG_THREADS) {
        const float xa = (hg_edge(a, bin, i) - y) / s2, xb = (hg_edge(a, bin, i + 1) - y) / s2;
        const float p = hg_erf_diff(xa, xb) / z;
        ce += p * ((l[i] - m) - logS);
        diff[i] = se[i] / S - p;
    }
    ce = hg_block_sum(ce, red);
    if (tid == 0) {
        a.ce[b] = -ce;
        __threadfence();
        // atomicInc wraps to 0 after B - 1: the CTA that sees B - 1 is the last one and the counter is ready for the next launch
        if (atomicInc(a.ws_count, (unsigned)(a.B - 1)) == (unsigned)(a.B - 1)) {
            __threadfence();
            float t = 0.f;
            for (int j = 0; j < a.B; ++j) t += __ldcg(a.ce + j);
            *a.loss = t / (float)a.B;
        }
    }
}

__global__ void __launch_bounds__(256) hl_gauss_bwd_kernel(const b200_hl_gauss_args a) {
    const float g = __ldg(a.dloss) / (float)a.B;
    const int n = a.B * a.num_bins;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) a.dlogits[i] = g * a.diff[i];
}

}  // namespace b200

using namespace b200;

static int check_hl_gauss(const b200_hl_gauss_args* a) {
    B200_REQUIRE(a, "hl_gauss: null pointer");
    B200_REQUIRE(a->B >= 1 && a->B <= HG_MAX_B, "hl_gauss: batch must be 1..%d (got %d)", HG_MAX_B, a->B);
    B200_REQUIRE(a->num_bins >= 2 && a->num_bins <= HG_MAX_BINS, "hl_gauss: num_bins must be 2..%d (got %d)", HG_MAX_BINS, a->num_bins);
    B200_REQUIRE(isfinite(a->min_value) && isfinite(a->max_value) && a->min_value < a->max_value,
                 "hl_gauss: min_value < max_value, both finite, is required");
    B200_REQUIRE(isfinite(a->sigma) && a->sigma > 0.f, "hl_gauss: sigma must be positive and finite");
    B200_REQUIRE(a->clamp_to_range == 0 || a->clamp_to_range == 1, "hl_gauss: clamp_to_range must be 0 or 1");
    return 0;
}
extern "C" int b200_hl_gauss_fwd(const b200_hl_gauss_args* a, b200_stream_t stream) {
    if (check_hl_gauss(a)) return -1;
    B200_REQUIRE(a->logits, "hl_gauss_fwd: null logits");
    if (a->target) B200_REQUIRE(a->ce && a->loss && a->diff && a->ws_count, "hl_gauss_fwd: training mode needs ce, loss, diff and ws_count");
    else B200_REQUIRE(a->pred, "hl_gauss_fwd: prediction mode needs pred");
    hl_gauss_fwd_kernel<<<a->B, HG_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("hl_gauss_fwd_kernel");
}
extern "C" int b200_hl_gauss_bwd(const b200_hl_gauss_args* a, b200_stream_t stream) {
    if (check_hl_gauss(a)) return -1;
    B200_REQUIRE(a->diff && a->dloss && a->dlogits, "hl_gauss_bwd: null pointer");
    const int n = a->B * a->num_bins;
    hl_gauss_bwd_kernel<<<(n + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("hl_gauss_bwd_kernel");
}
