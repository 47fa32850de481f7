// Multi-tensor kernels for the step AROUND the forward/backward hot path (SURVEY §8f row 1, §8e):
//   flat_gather  : every parameter gradient -> one contiguous fp32 buffer (x 1/world), ONE launch, so the data-parallel exchange is a
//                  single ncclAllReduce over one buffer instead of DDP's bucket copies + hooks (trainer.py:155-162, :270)
//   flat_accumulate : the same walk, adding (x scale) into the buffer instead of overwriting it: gradient accumulation over micro-batches
//   sumsq        : global gradient norm^2 of that buffer (clip_grad_norm_, trainer.py:272-273)
//   adopt_step   : gradient clip + Adopt update (adam-atan2-pytorch `Adopt`, trainer.py:183, :275) + EMA of the parameters
//                  (ema-pytorch `EMA.update`, trainer.py:279) in ONE pass: 5 reads + 4 writes of fp32 per parameter
// All HBM-bound, one 16-byte vector per thread per tensor; parameters stay separate nn.Parameter storages (a chunk table
// maps pieces of <= 64 Ki elements onto CTAs), optimizer / EMA state and gradients are flat buffers owned by the caller.
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

__global__ void __launch_bounds__(256) flat_gather_kernel(const b200_chunk* __restrict__ chunks, float* __restrict__ flat, float scale,
                                                          float* __restrict__ used) {
    const b200_chunk c = chunks[blockIdx.x];
    const float* __restrict__ src = reinterpret_cast<const float*>(c.ptr);
    float* __restrict__ dst = flat + c.flat_offset;
    if (used && threadIdx.x == 0) used[c.pidx] = src ? 1.f : 0.f;   // every piece of a parameter writes the same value
    if (src == nullptr) {   // parameter without a gradient this step (text stream when the text is dropped): its slot is zero
        for (int i = threadIdx.x; i < c.n; i += 256) dst[i] = 0.f;
        return;
    }
    const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    const int n4 = vec ? c.n >> 2 : 0;
    for (int i = threadIdx.x; i < n4; i += 256) {
        float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
        v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
        reinterpret_cast<float4*>(dst)[i] = v;
    }
    for (int i = n4 * 4 + threadIdx.x; i < c.n; i += 256) dst[i] = __ldg(src + i) * scale;
}

// accumulate: flat[flat_offset + i] = fmaf(scale, ptr[i], flat[flat_offset + i]) — the gather's twin for gradient accumulation over
// micro-batches. A NULL ptr leaves its slot as it is, and `used` is only ever set (the OR of the presence flags over the calls).
__global__ void __launch_bounds__(256) flat_accumulate_kernel(const b200_chunk* __restrict__ chunks, float* __restrict__ flat, float scale,
                                                              float* __restrict__ used) {
    const b200_chunk c = chunks[blockIdx.x];
    const float* __restrict__ src = reinterpret_cast<const float*>(c.ptr);
    if (src == nullptr) return;
    float* __restrict__ dst = flat + c.flat_offset;
    if (used && threadIdx.x == 0) used[c.pidx] = 1.f;
    const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    const int n4 = vec ? c.n >> 2 : 0;
    for (int i = threadIdx.x; i < n4; i += 256) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(src) + i);
        float4 a = reinterpret_cast<const float4*>(dst)[i];
        a.x = fmaf(scale, g.x, a.x); a.y = fmaf(scale, g.y, a.y); a.z = fmaf(scale, g.z, a.z); a.w = fmaf(scale, g.w, a.w);
        reinterpret_cast<float4*>(dst)[i] = a;
    }
    for (int i = n4 * 4 + threadIdx.x; i < c.n; i += 256) dst[i] = fmaf(scale, __ldg(src + i), dst[i]);
}

// sumsq: the block partials go to a static device array and the last block to finish adds them in block order, so the norm is
// the same bit for bit on every call with the same input (no float atomics whose order depends on the schedule): a resumed run
// clips exactly as the uninterrupted one. One call at a time per device (stream order), like every other user of the buffer.
constexpr int kSumsqMaxGrid = 4096;
__device__ float g_sumsq_part[kSumsqMaxGrid];
__device__ unsigned int g_sumsq_ticket;   // blocks of the current call that have written their partial; reset by the last one

__device__ __forceinline__ float block_sum_256(float acc, float* part) {   // fixed order; the result is valid in thread 0
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int i = 0; i < 8; ++i) s += part[i];
    return s;
}

__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
    float acc = 0.f;
    const long long n4 = ((reinterpret_cast<uintptr_t>(x) & 15) == 0) ? (n >> 2) : 0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    for (long long i = n4 * 4 + (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) acc += x[i] * x[i];
    __shared__ float part[8];
    __shared__ bool last;
    const float s = block_sum_256(acc, part);
    if (threadIdx.x == 0) {
        g_sumsq_part[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(&g_sumsq_ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    float a = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += 256) a += __ldcg(g_sumsq_part + i);
    __syncthreads();   // part[] is reused
    const float total = block_sum_256(a, part);
    if (threadIdx.x == 0) {
        *out = total;
        g_sumsq_ticket = 0u;
    }
}

struct AdoptP {
    const b200_chunk* chunks;
    const float* grad;
    float *m, *v, *ema;
    const float* gradnorm_sq;
    const float* used;
    float max_grad_norm, lr, one_minus_beta1, one_minus_beta2, eps, weight_decay, ema_weight;
    int* chunk_state;
    int ema_mode;
};

__device__ __forceinline__ void adopt_elem(const AdoptP& p, float g, float& w, float& m, float& v, float& e, float clip, bool live, bool first) {
    g *= clip;
    if (!live) {                 // no rank produced a gradient for this parameter: torch optimisers skip it (grad is None)
    } else if (first) {          // Adopt's first sight of a parameter only initialises v = g^2 (m = 0) and leaves the parameter alone
        if (p.weight_decay > 0.f) w *= (1.f - p.lr * p.weight_decay);
        v = g * g;
        m = 0.f;
    } else {
        if (p.weight_decay > 0.f) w *= (1.f - p.lr * p.weight_decay);
        const float u = g / fmaxf(sqrtf(v), p.eps);
        m += p.one_minus_beta1 * (u - m);
        w -= p.lr * m;
        v += p.one_minus_beta2 * (g * g - v);
    }
    if (p.ema_mode == 1) e += p.ema_weight * (w - e);
    else if (p.ema_mode == 2) e = w;
}

__global__ void __launch_bounds__(256) adopt_step_kernel(const AdoptP p) {
    const b200_chunk c = p.chunks[blockIdx.x];
    float* __restrict__ w = reinterpret_cast<float*>(c.ptr);
    const long long off = c.flat_offset;
    const bool live = !p.used || __ldg(p.used + c.pidx) > 0.f;
    if (!live && !p.ema_mode) return;
    const bool first = p.chunk_state[blockIdx.x] == 0;   // read by every thread before thread 0 flips it below (barrier in between)
    __syncthreads();
    if (live && first && threadIdx.x == 0) p.chunk_state[blockIdx.x] = 1;
    float clip = 1.f;
    if (p.gradnorm_sq && p.max_grad_norm > 0.f) {   // clip_grad_norm_: clamp(max_norm / (norm + 1e-6), max=1), so a NaN norm gives a NaN
        const float q = p.max_grad_norm / (sqrtf(__ldg(p.gradnorm_sq)) + 1e-6f);   // coefficient (every weight), not fminf's 1
        clip = q > 1.f ? 1.f : q;
    }
    const bool vec = ((reinterpret_cast<uintptr_t>(w) & 15) == 0) && ((off & 3) == 0);
    const int n4 = vec ? c.n >> 2 : 0;
    for (int i = threadIdx.x; i < n4; i += 256) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.grad + off) + i);
        float4 wv = reinterpret_cast<float4*>(w)[i];
        float4 mv = reinterpret_cast<float4*>(p.m + off)[i];
        float4 vv = reinterpret_cast<float4*>(p.v + off)[i];
        float4 ev = p.ema_mode ? reinterpret_cast<float4*>(p.ema + off)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        adopt_elem(p, g.x, wv.x, mv.x, vv.x, ev.x, clip, live, first);
        adopt_elem(p, g.y, wv.y, mv.y, vv.y, ev.y, clip, live, first);
        adopt_elem(p, g.z, wv.z, mv.z, vv.z, ev.z, clip, live, first);
        adopt_elem(p, g.w, wv.w, mv.w, vv.w, ev.w, clip, live, first);
        reinterpret_cast<float4*>(w)[i] = wv;
        reinterpret_cast<float4*>(p.m + off)[i] = mv;
        reinterpret_cast<float4*>(p.v + off)[i] = vv;
        if (p.ema_mode) reinterpret_cast<float4*>(p.ema + off)[i] = ev;
    }
    for (int i = n4 * 4 + threadIdx.x; i < c.n; i += 256) {
        float wv = w[i], mv = p.m[off + i], vv = p.v[off + i], ev = p.ema_mode ? p.ema[off + i] : 0.f;
        adopt_elem(p, p.grad[off + i], wv, mv, vv, ev, clip, live, first);
        w[i] = wv; p.m[off + i] = mv; p.v[off + i] = vv;
        if (p.ema_mode) p.ema[off + i] = ev;
    }
}

// scatter: param_ptr[i] = flat[flat_offset + i] (EMA weights back into a module's parameters, e.g. for sampling with the EMA model)
__global__ void __launch_bounds__(256) flat_scatter_kernel(const b200_chunk* __restrict__ chunks, const float* __restrict__ flat) {
    const b200_chunk c = chunks[blockIdx.x];
    float* __restrict__ dst = reinterpret_cast<float*>(c.ptr);
    const float* __restrict__ src = flat + c.flat_offset;
    for (int i = threadIdx.x; i < c.n; i += 256) dst[i] = src[i];
}

}  // namespace b200

using namespace b200;

extern "C" int b200_flat_gather(const b200_chunk* chunks_dev, int32_t n_chunks, float* flat, float scale, float* used, b200_stream_t stream) {
    B200_REQUIRE(chunks_dev && flat && n_chunks > 0, "flat_gather: null pointer / empty table");
    flat_gather_kernel<<<n_chunks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(chunks_dev, flat, scale, used);
    return check_launch("flat_gather_kernel");
}

extern "C" int b200_flat_accumulate(const b200_chunk* chunks_dev, int32_t n_chunks, float* flat, float scale, float* used, b200_stream_t stream) {
    B200_REQUIRE(chunks_dev && flat && n_chunks > 0, "flat_accumulate: null pointer / empty table");
    flat_accumulate_kernel<<<n_chunks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(chunks_dev, flat, scale, used);
    return check_launch("flat_accumulate_kernel");
}

extern "C" int b200_flat_scatter(const b200_chunk* chunks_dev, int32_t n_chunks, const float* flat, b200_stream_t stream) {
    B200_REQUIRE(chunks_dev && flat && n_chunks > 0, "flat_scatter: null pointer / empty table");
    flat_scatter_kernel<<<n_chunks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(chunks_dev, flat);
    return check_launch("flat_scatter_kernel");
}

extern "C" int b200_sumsq(const float* x, int64_t n, float* out, b200_stream_t stream) {
    B200_REQUIRE(x && out && n > 0, "sumsq: null pointer / empty buffer");
    const long long blocks = (n / 4 + 255) / 256;
    const long long cap = (long long)num_sms() * 8 < kSumsqMaxGrid ? (long long)num_sms() * 8 : kSumsqMaxGrid;
    const int grid = (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
    sumsq_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, (long long)n, out);
    return check_launch("sumsq_kernel");
}

extern "C" int b200_adopt_step(const b200_adopt_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->chunks_dev && a->n_chunks > 0 && a->grad_flat && a->m_flat && a->v_flat && a->chunk_state, "adopt_step: null pointer");
    B200_REQUIRE(a->ema_mode == 0 || a->ema_flat, "adopt_step: ema_mode %d needs ema_flat", a->ema_mode);
    B200_REQUIRE(a->ema_mode >= 0 && a->ema_mode <= 2, "adopt_step: ema_mode must be 0 (off), 1 (lerp) or 2 (copy)");
    AdoptP p{};
    p.chunks = a->chunks_dev; p.grad = a->grad_flat; p.m = a->m_flat; p.v = a->v_flat; p.ema = a->ema_flat;
    p.gradnorm_sq = a->gradnorm_sq; p.max_grad_norm = a->max_grad_norm; p.used = a->used;
    p.lr = a->lr;
    // the lerp weights 1 - beta: formed in double by the caller (as torch's lerp_(x, 1. - beta) does) when given, else from the fp32 betas
    p.one_minus_beta1 = a->one_minus_beta1 != 0.f ? a->one_minus_beta1 : 1.f - a->beta1;
    p.one_minus_beta2 = a->one_minus_beta2 != 0.f ? a->one_minus_beta2 : 1.f - a->beta2;
    p.eps = a->eps; p.weight_decay = a->weight_decay;
    p.chunk_state = a->chunk_state; p.ema_mode = a->ema_mode; p.ema_weight = a->ema_weight;
    adopt_step_kernel<<<a->n_chunks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("adopt_step_kernel");
}
