// Standalone bring-up harness for the wgmma GEMM (not part of the library): compares b200_gemm against
// a naive fp32 kernel on the same bf16 inputs, over operand-major / tail / epilogue / split-K cases, then
// times the cfg2 shapes.  Build: make test_gemm ; run on an H100: timeout 120 ./test_gemm [wide]
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../include/b200_e2tts.h"

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(2); } } while (0)

__global__ void ref_gemm(const __nv_bfloat16* A, long lda, int a_mn, const __nv_bfloat16* A2, long lda2, int K1,
                         const __nv_bfloat16* B, long ldb, int b_mn, float* C, int M, int N, int K) {
    int n = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (n >= N) return;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
        float a;
        if (A2 && k >= K1) a = __bfloat162float(A2[(long)m * lda2 + (k - K1)]);
        else a = __bfloat162float(a_mn ? A[(long)k * lda + m] : A[(long)m * lda + k]);
        float b = __bfloat162float(b_mn ? B[(long)k * ldb + n] : B[(long)n * ldb + k]);
        acc += a * b;
    }
    C[(long)m * N + n] = acc;
}

__global__ void tiny_kernel(float* p) { if (threadIdx.x == 0 && blockIdx.x == 0) p[0] += 1.f; }
__global__ void tiny_smem_kernel(float* p) { extern __shared__ float sm[]; sm[threadIdx.x] = p[threadIdx.x]; __syncthreads(); if (threadIdx.x == 0) p[0] = sm[1]; }

static float frand() { return (float)rand() / RAND_MAX * 2.f - 1.f; }
static __nv_bfloat16* dev_bf16(size_t n, float scale = 1.f) {
    std::vector<__nv_bfloat16> h(n);
    for (size_t i = 0; i < n; ++i) h[i] = __float2bfloat16(frand() * scale);
    __nv_bfloat16* d; CK(cudaMalloc(&d, n * 2)); CK(cudaMemcpy(d, h.data(), n * 2, cudaMemcpyHostToDevice)); return d;
}
static float* dev_f32(size_t n, float scale = 1.f, float off = 0.f) {
    std::vector<float> h(n);
    for (size_t i = 0; i < n; ++i) h[i] = frand() * scale + off;
    float* d; CK(cudaMalloc(&d, n * 4)); CK(cudaMemcpy(d, h.data(), n * 4, cudaMemcpyHostToDevice)); return d;
}
static double gelu(double x) { return 0.5 * x * (1.0 + erf(x * 0.70710678118654752440)); }

struct Case { const char* name; int M, N, K; int a_mn, b_mn; int K1; int bias, colscale, rowmask, resid, geglu, split, fp32; int tile = 0; };

static int run_case(const Case& c) {
    const int M = c.M, N = c.N, K = c.K;
    long lda = c.a_mn ? ((M + 7) / 8 * 8) : (((c.K1 ? c.K1 : K) + 7) / 8 * 8);
    long ldb = c.b_mn ? ((N + 7) / 8 * 8) : ((K + 7) / 8 * 8);
    long lda2 = c.K1 ? ((K - c.K1 + 7) / 8 * 8) : 0;
    __nv_bfloat16* A = dev_bf16(c.a_mn ? (size_t)K * lda : (size_t)M * lda);
    __nv_bfloat16* A2 = c.K1 ? dev_bf16((size_t)M * lda2) : nullptr;
    __nv_bfloat16* B = dev_bf16(c.b_mn ? (size_t)K * ldb : (size_t)N * ldb);
    float* Cref; CK(cudaMalloc(&Cref, (size_t)M * N * 4));
    ref_gemm<<<dim3((N + 127) / 128, M), 128>>>(A, lda, c.a_mn, A2, lda2, c.K1, B, ldb, c.b_mn, Cref, M, N, K);
    CK(cudaDeviceSynchronize());
    std::vector<float> ref((size_t)M * N);
    CK(cudaMemcpy(ref.data(), Cref, ref.size() * 4, cudaMemcpyDeviceToHost));

    float* bias = c.bias ? dev_f32(N) : nullptr;
    const int rpb = 48;
    int nb = (M + rpb - 1) / rpb;
    float* cs = c.colscale ? dev_f32((size_t)nb * N, 0.5f, 1.f) : nullptr;
    std::vector<unsigned char> hmask(M);
    for (int i = 0; i < M; ++i) hmask[i] = (i % 5) != 0;
    unsigned char* mask = nullptr;
    if (c.rowmask) { CK(cudaMalloc(&mask, M)); CK(cudaMemcpy(mask, hmask.data(), M, cudaMemcpyHostToDevice)); }
    long ldr = (N + 7) / 8 * 8;
    __nv_bfloat16* resid = c.resid ? dev_bf16((size_t)M * ldr) : nullptr;
    std::vector<float> hb(N), hcs((size_t)nb * N);
    std::vector<__nv_bfloat16> hres((size_t)M * ldr);
    if (bias) CK(cudaMemcpy(hb.data(), bias, N * 4, cudaMemcpyDeviceToHost));
    if (cs) CK(cudaMemcpy(hcs.data(), cs, hcs.size() * 4, cudaMemcpyDeviceToHost));
    if (resid) CK(cudaMemcpy(hres.data(), resid, hres.size() * 2, cudaMemcpyDeviceToHost));

    const int Nout = c.geglu ? N / 2 : N;
    long ldd = (Nout + 7) / 8 * 8;
    void* D; CK(cudaMalloc(&D, (size_t)M * ldd * 4)); CK(cudaMemset(D, 0xff, (size_t)M * ldd * 4));
    void* D2 = nullptr; long ldd2 = N;
    if (c.geglu) { CK(cudaMalloc(&D2, (size_t)M * N * 2)); }

    b200_gemm_args g = {};
    g.A = A; g.lda = lda; g.A2 = A2; g.lda2 = lda2; g.K1 = c.K1; g.B = B; g.ldb = ldb;
    g.M = M; g.N = N; g.K = K; g.a_mn_major = c.a_mn; g.b_mn_major = c.b_mn;
    g.D = D; g.ldd = ldd; g.d_fp32 = c.fp32; g.D2 = D2; g.ldd2 = ldd2;
    g.bias = bias; g.colscale = cs; g.rows_per_batch = rpb; g.rowmask = mask; g.resid = resid; g.ldr = ldr;
    g.geglu = c.geglu; g.dropout_p = 0.f; g.seed = 0; g.split_k = c.split; g.force_tile = c.tile;
    int rc = b200_gemm(&g, 0);
    if (rc) { printf("[%s] b200_gemm rc=%d: %s\n", c.name, rc, b200_last_error()); return 1; }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("[%s] kernel failed: %s\n", c.name, cudaGetErrorString(e)); exit(3); }

    std::vector<float> out((size_t)M * Nout);
    if (c.fp32) {
        std::vector<float> h((size_t)M * ldd);
        CK(cudaMemcpy(h.data(), D, h.size() * 4, cudaMemcpyDeviceToHost));
        for (int m = 0; m < M; ++m) for (int n = 0; n < Nout; ++n) out[(size_t)m * Nout + n] = h[(size_t)m * ldd + n];
    } else {
        std::vector<__nv_bfloat16> h((size_t)M * ldd);
        CK(cudaMemcpy(h.data(), D, h.size() * 2, cudaMemcpyDeviceToHost));
        for (int m = 0; m < M; ++m) for (int n = 0; n < Nout; ++n) out[(size_t)m * Nout + n] = __bfloat162float(h[(size_t)m * ldd + n]);
    }
    double max_err = 0, max_ref = 0;
    for (int m = 0; m < M; ++m)
        for (int n = 0; n < Nout; ++n) {
            double want;
            if (c.geglu) {
                int t = n / 64, j = n % 64;
                double u = ref[(size_t)m * N + t * 128 + j] + (bias ? hb[t * 128 + j] : 0.f);
                double gg = ref[(size_t)m * N + t * 128 + 64 + j] + (bias ? hb[t * 128 + 64 + j] : 0.f);
                want = u * gelu(gg);
            } else {
                want = ref[(size_t)m * N + n];
                if (bias) want += hb[n];
                if (cs) want *= hcs[(size_t)(m / rpb) * N + n];
                if (mask && !hmask[m]) want = 0;
                if (resid) want += __bfloat162float(hres[(size_t)m * ldr + n]);
            }
            double err = fabs(want - out[(size_t)m * Nout + n]);
            if (err > max_err) max_err = err;
            if (fabs(want) > max_ref) max_ref = fabs(want);
        }
    double tol = (c.fp32 ? 2e-3 : 1.2e-2) * (max_ref + 1e-6);
    int bad = !(max_err <= tol);
    printf("[%-28s] M=%d N=%d K=%d  max_err=%.4g (max_ref=%.4g) %s\n", c.name, M, N, K, max_err, max_ref, bad ? "FAIL" : "ok");
    cudaFree(A); cudaFree(A2); cudaFree(B); cudaFree(Cref); cudaFree(bias); cudaFree(cs); cudaFree(mask); cudaFree(resid); cudaFree(D); cudaFree(D2);
    return bad;
}

static void bench(const char* name, int M, int N, int K, int a_mn, int b_mn, int split, int fp32, int geglu, int tile = 0, int epi = 0) {
    long lda = a_mn ? M : K, ldb = b_mn ? N : K;
    __nv_bfloat16* A = dev_bf16((size_t)M * K, 0.1f); __nv_bfloat16* B = dev_bf16((size_t)N * K, 0.1f);
    void* D; CK(cudaMalloc(&D, (size_t)M * N * 4)); void* D2; CK(cudaMalloc(&D2, (size_t)M * N * 2));
    b200_gemm_args g = {};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.M = M; g.N = N; g.K = K; g.a_mn_major = a_mn; g.b_mn_major = b_mn;
    g.D = D; g.ldd = geglu ? N / 2 : N; g.d_fp32 = fp32; g.split_k = split; g.geglu = geglu; g.D2 = geglu ? D2 : nullptr; g.ldd2 = N; g.force_tile = tile;
    if (epi & 1) g.bias = dev_f32(N);
    if (epi & 2) { g.colscale = dev_f32((size_t)(M / 1056 + 1) * N, 0.5f, 1.f); g.rows_per_batch = 1056; }
    if (epi & 4) { unsigned char* mk; CK(cudaMalloc(&mk, M)); CK(cudaMemset(mk, 1, M)); g.rowmask = mk; }
    if (epi & 8) { g.resid = dev_bf16((size_t)M * N); g.ldr = N; }
    for (int i = 0; i < 3; ++i) if (b200_gemm(&g, 0)) { printf("bench %s: %s\n", name, b200_last_error()); return; }
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int it = 20;
    cudaEventRecord(e0);
    for (int i = 0; i < it; ++i) b200_gemm(&g, 0);
    cudaEventRecord(e1);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("bench %s failed: %s\n", name, cudaGetErrorString(e)); exit(3); }
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= it;
    printf("bench %-24s epi=%d tile=%d M=%d N=%d K=%d split=%d: %.3f ms  %.1f TFLOP/s\n", name, epi, tile, M, N, K, split, ms, 2.0 * M * N * K / ms * 1e-9);
    cudaFree(A); cudaFree(B); cudaFree(D); cudaFree(D2);
}

int main(int argc, char** argv) {
    srand(1);
    std::vector<Case> cases = {
        {"kmajor 128x128x64", 128, 128, 64, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1},
        {"kmajor 256x256x512", 256, 256, 512, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1},
        {"kmajor tails", 300, 200, 104, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0},
        {"kmajor many tiles", 1024 + 32, 640, 256, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0},
        {"b mn-major (dX)", 384, 256, 192, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0},
        {"a mn-major", 256, 128, 320, 1, 0, 0, 0, 0, 0, 0, 0, 1, 1},
        {"both mn-major (dW)", 256, 192, 1000, 1, 1, 0, 0, 0, 0, 0, 0, 1, 1},
        {"both mn-major split-k", 256, 192, 2000, 1, 1, 0, 0, 0, 0, 0, 0, 4, 1},
        {"two-source A", 320, 128, 192, 0, 0, 128, 0, 0, 0, 0, 0, 1, 0},
        {"bias+gate+mask+resid", 300, 264, 128, 0, 0, 0, 1, 1, 1, 1, 0, 1, 0},
        {"bias fp32 N=100", 200, 100, 128, 0, 0, 0, 1, 0, 0, 0, 0, 1, 1},
        {"geglu", 260, 512, 128, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0},
    };
    int bad = 0;
    if (argc > 1 && !strcmp(argv[1], "wide")) {   // 128 x 256 tiles (force_tile 3)
        cases.push_back({"kmajor multi-wave", 2048 + 32, 768, 512, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0});
        cases.push_back({"dW-like split", 512, 512, 4096, 1, 1, 0, 0, 0, 0, 0, 0, 4, 1});
        cases.push_back({"two-source wide", 1000, 512, 768, 0, 0, 512, 1, 0, 0, 1, 0, 1, 0});
        cases.push_back({"geglu wide", 1100, 1408, 256, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0});
        for (auto c : cases) { c.tile = 3; bad += run_case(c); }
        printf("wide-tile correctness: %d failing case(s)\n", bad);
        if (bad) return 1;
        for (int tile = 2; tile <= 3; ++tile) {
            bench("ff-in (geglu)", 16896, 4096, 512, 0, 0, 1, 0, 1, tile, 1);
            bench("ff-out", 16896, 512, 2048, 0, 0, 1, 0, 0, tile);
            bench("attn-out", 16896, 512, 512, 0, 0, 1, 0, 0, tile, 6);
            bench("qkv", 16896, 1552, 512, 0, 0, 1, 0, 0, tile);
            bench("cross (S streams)", 67584, 512, 768, 0, 0, 1, 0, 0, tile);
            bench("dX ff-in", 16896, 512, 4096, 0, 1, 1, 0, 0, tile);
            bench("dX qkv", 16896, 512, 1552, 0, 1, 1, 0, 0, tile);
            bench("dW ff-in", 4096, 512, 16896, 1, 1, 4, 1, 0, tile);
            bench("dW ff-out", 512, 2048, 16896, 1, 1, 4, 1, 0, tile);
            bench("dW attn-out split16", 512, 512, 16896, 1, 1, 16, 1, 0, tile);
            bench("square 8192", 8192, 8192, 8192, 0, 0, 1, 0, 0, tile);
        }
        return 0;
    }
    for (auto& c : cases) bad += run_case(c);
    for (auto c : cases) { c.tile = 2; bad += run_case(c); }   // same cases on the 256 x 128 CTA tile
    printf("correctness: %d failing case(s)\n", bad);
    if (argc > 4) {   // fixed-cost probe: per-launch time of a one-tile GEMM, alone and interleaved with other kernels
        const int M = 128, N = 128, K = 64;
        __nv_bfloat16* A = dev_bf16((size_t)M * K); __nv_bfloat16* B = dev_bf16((size_t)N * K);
        void* D; CK(cudaMalloc(&D, (size_t)M * N * 2)); float* scratch; CK(cudaMalloc(&scratch, 4096));
        b200_gemm_args g = {}; g.A = A; g.lda = K; g.B = B; g.ldb = K; g.M = M; g.N = N; g.K = K; g.D = D; g.ldd = N; g.split_k = 1;
        cudaFuncSetAttribute(tiny_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int mode = 0; mode < 4; ++mode) {
            for (int w = 0; w < 5; ++w) b200_gemm(&g, 0);
            cudaDeviceSynchronize();
            const int it = 200;
            cudaEventRecord(e0);
            for (int i = 0; i < it; ++i) {
                b200_gemm(&g, 0);
                if (mode == 1) tiny_kernel<<<132, 256>>>(scratch);
                if (mode == 2) tiny_smem_kernel<<<132, 256, 100 * 1024>>>(scratch);
                if (mode == 3) { tiny_kernel<<<132, 256>>>(scratch); tiny_kernel<<<132, 256>>>(scratch); }
            }
            cudaEventRecord(e1);
            CK(cudaDeviceSynchronize());
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            printf("latency mode %d (0 gemm only, 1 gemm+tiny, 2 gemm+tiny(100KB smem), 3 gemm+2 tiny): %.2f us per iteration\n", mode, ms * 1e3 / it);
        }
        cudaEventRecord(e0);
        for (int i = 0; i < 200; ++i) tiny_kernel<<<132, 256>>>(scratch);
        cudaEventRecord(e1); CK(cudaDeviceSynchronize());
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        printf("tiny kernel alone: %.2f us per launch\n", ms * 1e3 / 200);
        return 0;
    }
    if (argc > 3) {   // ncu targets: one shape per run
        const int which = atoi(argv[3]);
        if (which == 0) bench("attn-out", 16896, 512, 512, 0, 0, 1, 0, 0, 0, 6);
        if (which == 1) bench("ff-in (geglu)", 16896, 4096, 512, 0, 0, 1, 0, 1, 0, 1);
        if (which == 2) bench("dW small", 512, 512, 67584, 1, 1, 10, 1, 0, 0, 0);
        return 0;
    }
    if (argc > 2) {
        for (int epi : {0, 1, 2, 4, 8, 7}) bench("ff-out", 16896, 512, 2048, 0, 0, 1, 0, 0, 0, epi);
        for (int epi : {0, 2, 4, 6}) bench("attn-out", 16896, 512, 512, 0, 0, 1, 0, 0, 0, epi);
        bench("attn-out bmn", 16896, 512, 512, 0, 1, 1, 0, 0, 0, 0);
        return 0;
    }
    if (argc > 1) {
        bench("ff-in (geglu)", 16896, 4096, 512, 0, 0, 1, 0, 1);
        bench("ff-out", 16896, 512, 2048, 0, 0, 1, 0, 0);
        bench("qkv", 16896, 1552, 512, 0, 0, 1, 0, 0);
        bench("cross (S streams)", 67584, 512, 768, 0, 0, 1, 0, 0);
        bench("dX ff-in", 16896, 512, 4096, 0, 1, 1, 0, 0);
        bench("dW ff-in", 4096, 512, 16896, 1, 1, 4, 1, 0);
        bench("dW attn-out split16", 512, 512, 16896, 1, 1, 16, 1, 0);
        bench("square 8192", 8192, 8192, 8192, 0, 0, 1, 0, 0);
        for (int tile = 1; tile <= 2; ++tile) {
            bench("ff-in (geglu)", 16896, 4096, 512, 0, 0, 1, 0, 1, tile);
            bench("ff-out", 16896, 512, 2048, 0, 0, 1, 0, 0, tile);
            bench("qkv", 16896, 1552, 512, 0, 0, 1, 0, 0, tile);
            bench("cross (S streams)", 67584, 512, 768, 0, 0, 1, 0, 0, tile);
            bench("dX ff-in", 16896, 512, 4096, 0, 1, 1, 0, 0, tile);
            bench("dW ff-in", 4096, 512, 16896, 1, 1, 4, 1, 0, tile);
            bench("square 8192", 8192, 8192, 8192, 0, 0, 1, 0, 0, tile);
        }
    }
    return bad ? 1 : 0;
}
