// Runge–Kutta solver passes of E2TTS.sample (torchdiffeq rk4 / dopri5 / bosh3 / fehlberg2 / adaptive_heun, SURVEY A.7): stage
// inputs, the step's error norm, the initial-step norms and the dense output. Memory-bound fp32 passes over the ODE state; the
// tableau weights arrive as fp32 scalars formed on the host (include/b200_e2tts.h).
#include "common.cuh"

namespace b200 {
namespace {

constexpr int kOdeThreads = 256;
constexpr int kOdeMaxSources = 7;

struct Sources {
    const float* k[kOdeMaxSources];
    float w[kOdeMaxSources];
};

// W = 4: one float4 per pointer (every pointer 16-byte aligned); W = 1: one element
template <int W>
__device__ __forceinline__ void ld(const float* p, long long i, float (&v)[W]) {
    if constexpr (W == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        v[0] = __ldg(p + i);
    }
}
template <int W>
__device__ __forceinline__ void st(float* p, long long i, const float (&v)[W]) {
    if constexpr (W == 4) *reinterpret_cast<float4*>(p + i) = make_float4(v[0], v[1], v[2], v[3]);
    else p[i] = v[0];
}
// acc = sum_j w_j k_j, in source order (torchdiffeq's k.matmul(weights))
template <int S, int W>
__device__ __forceinline__ void weighted_sum(const Sources& s, long long i, float (&acc)[W]) {
#pragma unroll
    for (int l = 0; l < W; ++l) acc[l] = 0.f;
#pragma unroll
    for (int j = 0; j < S; ++j) {
        float v[W];
        ld<W>(s.k[j], i, v);
#pragma unroll
        for (int l = 0; l < W; ++l) acc[l] = fmaf(s.w[j], v[l], acc[l]);
    }
}

// Visits every element once: float4 units [0, n/4) when vec, then the scalar rest, each by a grid-stride loop.
template <typename Body>
__device__ __forceinline__ void visit(long long n, bool vec, Body& body) {
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    const long long nv = vec ? n / 4 : 0;
    for (long long u = tid; u < nv; u += stride) body.template run<4>(4 * u);
    for (long long i = 4 * nv + tid; i < n; i += stride) body.template run<1>(i);
}

// fixed-order block sum of a double (8 warps); the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double part[kOdeThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();   // part[] may still be read by a previous call
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kOdeThreads / 32; ++w) t += part[w];
    return t;
}

template <int S>
struct CombineBody {
    const float* y0; Sources s; float* out;
    template <int W>
    __device__ __forceinline__ void run(long long i) {
        float acc[W], y[W];
        weighted_sum<S, W>(s, i, acc);
        ld<W>(y0, i, y);
#pragma unroll
        for (int l = 0; l < W; ++l) acc[l] = y[l] + acc[l];
        st<W>(out, i, acc);
    }
};

template <int S>
__global__ void __launch_bounds__(kOdeThreads) ode_combine_kernel(const float* y0, Sources s, float* out, long long n, bool vec) {
    CombineBody<S> b{y0, s, out};
    visit(n, vec, b);
}

template <int S>
struct ErrorBody {
    const float* y0; Sources err, sol; float* y1; bool write_y1; float atol, rtol; double acc;
    template <int W>
    __device__ __forceinline__ void run(long long i) {
        float y[W], y1v[W], e[W];
        ld<W>(y0, i, y);
        if (write_y1) {
            weighted_sum<S, W>(sol, i, y1v);
#pragma unroll
            for (int l = 0; l < W; ++l) y1v[l] = y[l] + y1v[l];
            st<W>(y1, i, y1v);
        } else {
            ld<W>(y1, i, y1v);
        }
        weighted_sum<S, W>(err, i, e);
#pragma unroll
        for (int l = 0; l < W; ++l) {
            const float tol = atol + rtol * fmaxf(fabsf(y[l]), fabsf(y1v[l]));
            const double q = (double)(e[l] / tol);
            acc = fma(q, q, acc);
        }
    }
};

template <int S>
__global__ void __launch_bounds__(kOdeThreads) ode_step_error_kernel(const float* y0, Sources err, Sources sol, float* y1, bool write_y1,
                                                                     float atol, float rtol, double* ws, long long n, bool vec) {
    ErrorBody<S> b{y0, err, sol, y1, write_y1, atol, rtol, 0.0};
    visit(n, vec, b);
    const double t = block_sum(b.acc);
    if (threadIdx.x == 0) ws[blockIdx.x] = t;
}

struct NormsBody {
    const float *y0, *a, *b, *c; float atol, rtol; double acc0, acc1;
    template <int W>
    __device__ __forceinline__ void run(long long i) {
        float y[W], u[W], v[W], w[W];
        ld<W>(y0, i, y);
        if (a) ld<W>(a, i, u);
        ld<W>(b, i, v);
        if (c) ld<W>(c, i, w);
#pragma unroll
        for (int l = 0; l < W; ++l) {
            const float scale = atol + fabsf(y[l]) * rtol;
            if (a) { const double q = (double)(u[l] / scale); acc0 = fma(q, q, acc0); }
            const double q = (double)((c ? v[l] - w[l] : v[l]) / scale);
            acc1 = fma(q, q, acc1);
        }
    }
};

__global__ void __launch_bounds__(kOdeThreads) ode_norms_kernel(const float* y0, const float* a, const float* b, const float* c, float atol,
                                                                float rtol, double* ws, int ws_len, long long n, bool vec) {
    NormsBody body{y0, a, b, c, atol, rtol, 0.0, 0.0};
    visit(n, vec, body);
    const double t0 = block_sum(body.acc0), t1 = block_sum(body.acc1);
    if (threadIdx.x == 0) { ws[blockIdx.x] = t0; ws[ws_len + blockIdx.x] = t1; }
}

// out[ch] = sqrt(sum of the channel's partials / n), partials added in a fixed order
__global__ void __launch_bounds__(kOdeThreads) ode_rms_finalize_kernel(const double* ws, int ws_len, int parts, int nch, float* out, long long n) {
    for (int ch = 0; ch < nch; ++ch) {
        double v = 0.0;
        for (int j = threadIdx.x; j < parts; j += kOdeThreads) v += ws[(size_t)ch * ws_len + j];
        const double t = block_sum(v);
        if (threadIdx.x == 0) out[ch] = (float)sqrt(t / (double)n);
    }
}

template <int S>
struct DenseBody {
    const float *y0, *y1; Sources mid; float dt, x; float* out;
    template <int W>
    __device__ __forceinline__ void run(long long i) {
        float ym[W], a0[W], a1[W], f0[W], f1[W], r[W];
        weighted_sum<S, W>(mid, i, ym);
        ld<W>(y0, i, a0);
        ld<W>(y1, i, a1);
        ld<W>(mid.k[0], i, f0);
        ld<W>(mid.k[S - 1], i, f1);
        const float x2 = x * x, x3 = x2 * x, x4 = x3 * x, dt2 = 2.f * dt;
#pragma unroll
        for (int l = 0; l < W; ++l) {
            const float y_mid = a0[l] + ym[l];
            const float ca = dt2 * (f1[l] - f0[l]) - 8.f * (a1[l] + a0[l]) + 16.f * y_mid;
            const float cb = dt * (5.f * f0[l] - 3.f * f1[l]) + 18.f * a0[l] + 14.f * a1[l] - 32.f * y_mid;
            const float cc = dt * (f1[l] - 4.f * f0[l]) - 11.f * a0[l] - 5.f * a1[l] + 16.f * y_mid;
            const float cd = dt * f0[l];
            float t = a0[l] + x * cd;
            t = t + x2 * cc;
            t = t + x3 * cb;
            r[l] = t + x4 * ca;
        }
        st<W>(out, i, r);
    }
};

template <int S>
__global__ void __launch_bounds__(kOdeThreads) ode_dense_kernel(const float* y0, const float* y1, Sources mid, float dt, float x, float* out,
                                                                long long n, bool vec) {
    DenseBody<S> b{y0, y1, mid, dt, x, out};
    visit(n, vec, b);
}

bool aligned16(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int sources(Sources& s, const float* const (&k)[kOdeMaxSources], const float (&w)[kOdeMaxSources], int S, const char* what, bool& vec) {
    B200_REQUIRE(S >= 1 && S <= kOdeMaxSources, "%s: S=%d sources, want 1..%d", what, S, kOdeMaxSources);
    for (int j = 0; j < kOdeMaxSources; ++j) {
        B200_REQUIRE(j >= S || k[j], "%s: source k%d is null", what, j);
        s.k[j] = j < S ? k[j] : nullptr;
        s.w[j] = j < S ? w[j] : 0.f;
        vec = vec && aligned16(s.k[j]);
    }
    return 0;
}

unsigned elementwise_grid(long long n) {
    const long long g = (n + 4 * kOdeThreads - 1) / (4 * kOdeThreads), cap = (long long)num_sms() * 16;
    return (unsigned)(g < cap ? g : cap);
}
unsigned reduction_grid(long long n, int ws_len) {
    const long long g = (n + 4 * kOdeThreads - 1) / (4 * kOdeThreads);
    return (unsigned)(g < ws_len ? g : ws_len);
}

bool tol_ok(float atol, float rtol) { return isfinite(atol) && isfinite(rtol) && atol >= 0.f && rtol >= 0.f; }

// dispatch a kernel template on the number of sources
#define B200_ODE_DISPATCH(S, KERNEL, ...)                         \
    switch (S) {                                                  \
        case 1: KERNEL<1><<<__VA_ARGS__; break;                   \
        case 2: KERNEL<2><<<__VA_ARGS__; break;                   \
        case 3: KERNEL<3><<<__VA_ARGS__; break;                   \
        case 4: KERNEL<4><<<__VA_ARGS__; break;                   \
        case 5: KERNEL<5><<<__VA_ARGS__; break;                   \
        case 6: KERNEL<6><<<__VA_ARGS__; break;                   \
        default: KERNEL<7><<<__VA_ARGS__; break;                  \
    }

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_ode_combine(const b200_ode_combine_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->y0 && a->out && a->n > 0, "ode_combine: bad arguments");
    bool vec = aligned16(a->y0) && aligned16(a->out);
    Sources s;
    const float* const k[] = {a->k0, a->k1, a->k2, a->k3, a->k4, a->k5, a->k6};
    const float w[] = {a->w0, a->w1, a->w2, a->w3, a->w4, a->w5, a->w6};
    if (sources(s, k, w, a->S, "ode_combine", vec)) return -1;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_ODE_DISPATCH(a->S, ode_combine_kernel, elementwise_grid(a->n), kOdeThreads, 0, st>>>(a->y0, s, a->out, a->n, vec))
    return check_launch("ode_combine_kernel");
}

extern "C" int b200_ode_step_error(const b200_ode_step_error_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->y0 && a->y1 && a->ws && a->ratio && a->n > 0, "ode_step_error: bad arguments");
    B200_REQUIRE(a->ws_len >= 1 && a->ws_len <= 65535, "ode_step_error: ws_len=%d, want 1..65535", a->ws_len);
    B200_REQUIRE(tol_ok(a->atol, a->rtol), "ode_step_error: atol=%g rtol=%g, want finite and >= 0", a->atol, a->rtol);
    bool vec = aligned16(a->y0) && aligned16(a->y1);
    Sources err, sol;
    const float* const k[] = {a->k0, a->k1, a->k2, a->k3, a->k4, a->k5, a->k6};
    const float e[] = {a->e0, a->e1, a->e2, a->e3, a->e4, a->e5, a->e6};
    const float s[] = {a->s0, a->s1, a->s2, a->s3, a->s4, a->s5, a->s6};
    if (sources(err, k, e, a->S, "ode_step_error", vec) || sources(sol, k, s, a->S, "ode_step_error", vec)) return -1;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const unsigned grid = reduction_grid(a->n, a->ws_len);
    B200_ODE_DISPATCH(a->S, ode_step_error_kernel, grid, kOdeThreads, 0, st>>>(a->y0, err, sol, a->y1, a->write_y1 != 0, a->atol, a->rtol,
                                                                                   a->ws, a->n, vec))
    if (int rc = check_launch("ode_step_error_kernel")) return rc;
    ode_rms_finalize_kernel<<<1, kOdeThreads, 0, st>>>(a->ws, a->ws_len, (int)grid, 1, a->ratio, a->n);
    return check_launch("ode_rms_finalize_kernel");
}

extern "C" int b200_ode_scaled_norms(const b200_ode_norms_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->y0 && a->b && a->ws && a->out && a->n > 0, "ode_scaled_norms: bad arguments");
    B200_REQUIRE(a->ws_len >= 1 && a->ws_len <= 65535, "ode_scaled_norms: ws_len=%d, want 1..65535", a->ws_len);
    B200_REQUIRE(tol_ok(a->atol, a->rtol), "ode_scaled_norms: atol=%g rtol=%g, want finite and >= 0", a->atol, a->rtol);
    const bool vec = aligned16(a->y0) && aligned16(a->a) && aligned16(a->b) && aligned16(a->c);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const unsigned grid = reduction_grid(a->n, a->ws_len);
    ode_norms_kernel<<<grid, kOdeThreads, 0, st>>>(a->y0, a->a, a->b, a->c, a->atol, a->rtol, a->ws, a->ws_len, a->n, vec);
    if (int rc = check_launch("ode_norms_kernel")) return rc;
    ode_rms_finalize_kernel<<<1, kOdeThreads, 0, st>>>(a->ws, a->ws_len, (int)grid, 2, a->out, a->n);
    return check_launch("ode_rms_finalize_kernel");
}

extern "C" int b200_ode_dense_output(const b200_ode_dense_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->y0 && a->y1 && a->out && a->n > 0, "ode_dense_output: bad arguments");
    B200_REQUIRE(isfinite(a->dt) && isfinite(a->x), "ode_dense_output: dt=%g x=%g, want finite", a->dt, a->x);
    bool vec = aligned16(a->y0) && aligned16(a->y1) && aligned16(a->out);
    Sources s;
    const float* const k[] = {a->k0, a->k1, a->k2, a->k3, a->k4, a->k5, a->k6};
    const float m[] = {a->m0, a->m1, a->m2, a->m3, a->m4, a->m5, a->m6};
    if (sources(s, k, m, a->S, "ode_dense_output", vec)) return -1;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_ODE_DISPATCH(a->S, ode_dense_kernel, elementwise_grid(a->n), kOdeThreads, 0, st>>>(a->y0, a->y1, s, a->dt, a->x, a->out, a->n, vec))
    return check_launch("ode_dense_kernel");
}
