// Shared-memory FFT building blocks (complex helpers, register DFTs of radix 2/3/4/5, one Stockham autosort stage), used by the
// MelSpec STFT (small.cu) and the Vocos inverse STFT (vocos.cu). Every stage loops over its butterflies with a 256-thread stride.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// forward DFT of R points in registers, e^{-2 pi i q r / R}
__device__ __forceinline__ float2 c_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 c_sub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 c_mul(float2 a, float2 w) { return make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x); }
__device__ __forceinline__ float2 c_mul_mi(float2 a) { return make_float2(a.y, -a.x); }   // -i a, exact
template <int R> __device__ __forceinline__ void dft_small(float2* v);
template <> __device__ __forceinline__ void dft_small<2>(float2* v) {
    const float2 a = v[0], b = v[1];
    v[0] = c_add(a, b); v[1] = c_sub(a, b);
}
template <> __device__ __forceinline__ void dft_small<4>(float2* v) {
    const float2 t0 = c_add(v[0], v[2]), t1 = c_sub(v[0], v[2]), t2 = c_add(v[1], v[3]), t3 = c_mul_mi(c_sub(v[1], v[3]));
    v[0] = c_add(t0, t2); v[2] = c_sub(t0, t2); v[1] = c_add(t1, t3); v[3] = c_sub(t1, t3);
}
template <> __device__ __forceinline__ void dft_small<3>(float2* v) {
    constexpr float S1 = 0.866025403784438647f;   // sin(2 pi / 3)
    const float2 s = c_add(v[1], v[2]), d = c_sub(v[1], v[2]);
    const float2 t = make_float2(v[0].x - 0.5f * s.x, v[0].y - 0.5f * s.y);
    const float2 u = make_float2(S1 * d.y, -S1 * d.x);   // -i sin(2 pi / 3) (v1 - v2)
    v[0] = c_add(v[0], s); v[1] = c_add(t, u); v[2] = c_sub(t, u);
}
template <> __device__ __forceinline__ void dft_small<5>(float2* v) {
    constexpr float C1 = 0.309016994374947424f, C2 = -0.809016994374947424f;   // cos(2 pi / 5), cos(4 pi / 5)
    constexpr float S1 = 0.951056516295153572f, S2 = 0.587785252292473129f;    // sin(2 pi / 5), sin(4 pi / 5)
    const float2 b1 = c_add(v[1], v[4]), b2 = c_add(v[2], v[3]), d1 = c_sub(v[1], v[4]), d2 = c_sub(v[2], v[3]);
    const float2 t1 = make_float2(v[0].x + C1 * b1.x + C2 * b2.x, v[0].y + C1 * b1.y + C2 * b2.y);
    const float2 t2 = make_float2(v[0].x + C2 * b1.x + C1 * b2.x, v[0].y + C2 * b1.y + C1 * b2.y);
    const float2 u1 = c_mul_mi(make_float2(S1 * d1.x + S2 * d2.x, S1 * d1.y + S2 * d2.y));
    const float2 u2 = c_mul_mi(make_float2(S2 * d1.x - S1 * d2.x, S2 * d1.y - S1 * d2.y));
    v[0] = c_add(v[0], c_add(b1, b2));
    v[1] = c_add(t1, u1); v[4] = c_sub(t1, u1); v[2] = c_add(t2, u2); v[3] = c_sub(t2, u2);
}

// one Stockham stage of radix R after Ns points of every sub-transform are done: butterfly j reads in[j + q n/R] (q < R), turns
// input q by e^{-2 pi i q k / (Ns R)} (k = j mod Ns) and writes out[(j - k) R + k + r Ns]
template <int R>
__device__ __forceinline__ void stockham_stage(const float2* __restrict__ in, float2* __restrict__ out, const float2* __restrict__ tw, int n, int Ns) {
    const int m = n / R, tstep = n / (Ns * R);
    for (int j = threadIdx.x; j < m; j += 256) {
        const int k = j % Ns;
        float2 v[R];
#pragma unroll
        for (int q = 0; q < R; ++q) v[q] = in[j + q * m];
#pragma unroll
        for (int q = 1; q < R; ++q) v[q] = c_mul(v[q], tw[q * k * tstep]);
        dft_small<R>(v);
        const int o = (j - k) * R + k;
#pragma unroll
        for (int r = 0; r < R; ++r) out[o + r * Ns] = v[r];
    }
}

}  // namespace b200
