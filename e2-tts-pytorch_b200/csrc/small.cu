// Conditioning-path and convolution kernels: small-batch fp32 linears (time MLP, every AdaptiveRMSNorm /
// AdaLNZero gamma projection batched into one launch, duration head), Fourier time features, the masked
// depthwise conv + SiLU positional module, and the masked mean pool of the duration predictor.
#include "common.cuh"
#include "ptx.cuh"
#include "fft.cuh"

namespace b200 {

__device__ __forceinline__ float sl_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float sl_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ size_t yidx(const b200_small_linear_args& a, int b, int n) {
    return a.seg_major ? ((size_t)(n / a.seg) * a.B + b) * a.seg + (n % a.seg) : (size_t)b * a.N + n;
}
__device__ __forceinline__ int act_of(int act, int seg, int n) { return act == 5 ? (((n / seg) & 1) ? 2 : 3) : act; }
__device__ __forceinline__ float act_fwd(int a, float z) {
    switch (a) {
        case 1: return z * sl_sigmoid(z);
        case 2: return sl_sigmoid(z);
        case 3: return 1.f + z;
        case 4: return z > 20.f ? z : log1pf(expf(z));
        default: return z;
    }
}
__device__ __forceinline__ float act_bwd(int a, float z) {
    switch (a) {
        case 1: { const float s = sl_sigmoid(z); return s * (1.f + z * (1.f - s)); }
        case 2: { const float s = sl_sigmoid(z); return s * (1.f - s); }
        case 4: return sl_sigmoid(z);
        default: return 1.f;
    }
}

constexpr int SL_MAXB = 64;

// One warp per output feature n, all batch rows at once: the weight row streams through once (the first version looped
// over 8-row batch chunks and re-read it), X is staged in shared memory when it fits. 16 partial sums per lane are combined
// by recursive halving so that lane b ends up owning batch row b.
constexpr int SL_XS_MAX = 12 * 1024;   // floats of X staged in smem (48 KB)

__device__ __forceinline__ void sl_halve16(float (&v)[16], int lane) {   // on return lane l (mod 16) holds the 32-lane sum of v[l % 16] in v[0]
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
        const bool hi = lane & o;
#pragma unroll
        for (int i = 0; i < o; ++i) {
            const float send = hi ? v[i] : v[i + o];
            const float keep = hi ? v[i + o] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 16);
}

__global__ void __launch_bounds__(256) small_linear_fwd_kernel(const b200_small_linear_args a, int n_per_warp, int x_in_smem) {
    extern __shared__ __align__(16) float xs[];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    if (x_in_smem) {
        for (int i = threadIdx.x; i < a.B * a.K; i += 256) xs[i] = a.X[i];
        __syncthreads();
    }
    const float* X = x_in_smem ? xs : a.X;
    const int nbeg = (blockIdx.x * 8 + wl) * n_per_warp;
    for (int n = nbeg; n < min(a.N, nbeg + n_per_warp); ++n) {
        const float* w = a.W + (size_t)n * a.K;
        const float bias = a.bias ? a.bias[n] : 0.f;
        const int ac = act_of(a.act, a.seg, n);
        for (int b0 = 0; b0 < a.B; b0 += 16) {
            float acc[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = 0.f;
            const int nb = min(16, a.B - b0);
            if ((a.K & 3) == 0) {
                for (int k = lane * 4; k < a.K; k += 128) {
                    const float4 wv = __ldg(reinterpret_cast<const float4*>(w + k));
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (j < nb) {
                            const float4 xv = *reinterpret_cast<const float4*>(X + (size_t)(b0 + j) * a.K + k);
                            acc[j] += wv.x * xv.x + wv.y * xv.y + wv.z * xv.z + wv.w * xv.w;
                        }
                    }
                }
            } else {
                for (int k = lane; k < a.K; k += 32) {
                    const float wv = __ldg(w + k);
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (j < nb) acc[j] += wv * X[(size_t)(b0 + j) * a.K + k];
                }
            }
            sl_halve16(acc, lane);
            const int b = b0 + (lane & 15);
            if (lane < 16 && b < a.B) {
                const float z = acc[0] + bias;
                if (a.Z) a.Z[yidx(a, b, n)] = z;
                a.Y[yidx(a, b, n)] = act_fwd(ac, z);
            }
        }
    }
}
// one warp per output feature n: dZ[:,n], dbias[n], dW[n,:]
__global__ void __launch_bounds__(256) small_linear_bwd_w_kernel(const b200_small_linear_args a) {
    __shared__ float sdz[8][SL_MAXB];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int n = blockIdx.x * 8 + wl;
    if (n >= a.N) return;
    const int ac = act_of(a.act, a.seg, n);
    float db = 0.f;
    for (int b = lane; b < a.B; b += 32) {
        const float dz = a.dY[yidx(a, b, n)] * act_bwd(ac, a.Z[yidx(a, b, n)]);
        sdz[wl][b] = dz;
        a.dZ[yidx(a, b, n)] = dz;
        db += dz;
    }
    db = sl_warp_sum(db);
    if (lane == 0 && a.dbias) a.dbias[n] = db;
    __syncwarp();
    for (int k = lane; k < a.K; k += 32) {
        float acc = 0.f;
        for (int b = 0; b < a.B; ++b) acc += sdz[wl][b] * __ldg(a.X + (size_t)b * a.K + k);
        a.dW[(size_t)n * a.K + k] = acc;
    }
}
// dX[b,k] += sum_{n in block slab} dZ[b,n] W[n,k]   (dX zeroed by the host wrapper)
// The block's dZ slab [B][256] is staged in shared memory once (the first version re-derived the strided dZ index with an integer
// division for every (n, b), walked W twice and finished with 16x more scalar atomics). Fast path: a thread owns four
// consecutive k (16-byte W loads, 16-byte vector reductions into dX) and one of two 128-row halves of the slab.
constexpr int SL_SLAB = 256;   // largest slab of output features per block (a multiple of 8; smaller slabs when N is small)
__global__ void __launch_bounds__(256) small_linear_bwd_x_kernel(const b200_small_linear_args a, int slab) {
    extern __shared__ __align__(16) float sdz[];   // [B][slab]
    const int n0 = blockIdx.x * slab, n1 = min(a.N, n0 + slab);
    for (int i = threadIdx.x; i < a.B * slab; i += 256) {
        const int b = i / slab, nn = i % slab;
        sdz[i] = (n0 + nn < n1) ? a.dZ[yidx(a, b, n0 + nn)] : 0.f;
    }
    __syncthreads();
    if ((a.K & 3) == 0 && a.K <= 512 && ((reinterpret_cast<uintptr_t>(a.dX) | reinterpret_cast<uintptr_t>(a.W)) & 15) == 0) {
        const int kq = threadIdx.x & 127, grp = threadIdx.x >> 7, half = slab >> 1;
        if (kq * 4 >= a.K) return;
        for (int b0 = 0; b0 < a.B; b0 += 16) {
            const int nb = min(16, a.B - b0);
            float4 acc[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int nn = grp * half; nn < grp * half + half; nn += 4) {
                float4 w[4];
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    w[u] = (n0 + nn + u < n1) ? __ldg(reinterpret_cast<const float4*>(a.W + (size_t)(n0 + nn + u) * a.K + kq * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (j < nb) {
                        const float4 z = *reinterpret_cast<const float4*>(&sdz[(b0 + j) * slab + nn]);   // broadcast read
                        acc[j].x += w[0].x * z.x + w[1].x * z.y + w[2].x * z.z + w[3].x * z.w;
                        acc[j].y += w[0].y * z.x + w[1].y * z.y + w[2].y * z.z + w[3].y * z.w;
                        acc[j].z += w[0].z * z.x + w[1].z * z.y + w[2].z * z.z + w[3].z * z.w;
                        acc[j].w += w[0].w * z.x + w[1].w * z.y + w[2].w * z.z + w[3].w * z.w;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < nb) red_add_v4(a.dX + (size_t)(b0 + j) * a.K + kq * 4, acc[j].x, acc[j].y, acc[j].z, acc[j].w);
        }
        return;
    }
    // generic shapes (e.g. the K = dim + 1 input of the time MLP): a thread owns one k column, 16 batch rows in registers
    for (int k = threadIdx.x; k < a.K; k += 256) {
        for (int b0 = 0; b0 < a.B; b0 += 16) {
            const int nb = min(16, a.B - b0);
            float acc[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = 0.f;
            for (int nn = 0; nn < slab; nn += 4) {
                float w[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) w[u] = (n0 + nn + u < n1) ? __ldg(a.W + (size_t)(n0 + nn + u) * a.K + k) : 0.f;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (j < nb) {
                        const float4 z = *reinterpret_cast<const float4*>(&sdz[(b0 + j) * slab + nn]);
                        acc[j] += w[0] * z.x + w[1] * z.y + w[2] * z.z + w[3] * z.w;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < nb) atomicAdd(a.dX + (size_t)(b0 + j) * a.K + k, acc[j]);
        }
    }
}

__global__ void fourier_embed_kernel(const float* times, const float* w, float* out, int B, int half) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, j = i % half;
    const float t = times[b];
    const float f = t * w[j] * 2.f * 3.14159265358979323846f;
    float s, c;
    sincosf(f, &s, &c);
    float* o = out + (size_t)b * (2 * half + 1);
    if (j == 0) o[0] = t;
    o[1 + j] = s;
    o[1 + half + j] = c;
}

// ------------------------------------------------------------------------------------------------ depthwise conv
// y = m * silu(conv1d_depthwise(m * x) + bias)  on bf16 [B, Np, D]  (DepthwiseConv, e2_tts.py:295-328).
// Tile = 64 tokens x 64 channels staged in shared memory as fp32 (+ 15 halo rows each side). A thread owns a channel PAIR and a
// run of consecutive tokens: its 31 taps sit in registers as fp32x2 and every window element is read once (one LDS.64) and fed to
// all the outputs it touches, so the inner loop is pure FMA on fp32 pairs. (The scalar version of round 1
// issued one FMA per slot: 110 FFMA per element in backward, 94 us per call, FMA-pipe bound at half the fp32 peak.)
// Forward also stores the bf16 pre-activation; backward reads it back instead of recomputing the convolution over tile + halo
// (the same trade as the GEGLU pre-activations: +2 B per element of HBM traffic for 42 % fewer FMAs).
constexpr int CV_TN = 64, CV_TC = 64, CV_HALO = 15;
constexpr int CV_R = CV_TN + 2 * CV_HALO;   // staged rows of a tile: token n0 - 15 + r

typedef float2 cf2;
__device__ __forceinline__ cf2 cv_ffma2(cf2 a, cf2 b, cf2 c) { return ffma2(a, b, c); }

__device__ __forceinline__ bool tok_ok(const unsigned char* mask, int b, int n, int Np) {
    return n >= 0 && n < Np && (!mask || mask[(size_t)b * Np + n]);
}
__device__ __forceinline__ void cv_unpack8(const uint4& u, float (&v)[8]) {
    v[0] = bf16_lo(u.x); v[1] = bf16_hi(u.x); v[2] = bf16_lo(u.y); v[3] = bf16_hi(u.y);
    v[4] = bf16_lo(u.z); v[5] = bf16_hi(u.z); v[6] = bf16_lo(u.w); v[7] = bf16_hi(u.w);
}
// the tile's taps, staged once per block as [31][CV_TC] so that channel pairs are adjacent (one conflict-free LDS.64 per tap and thread);
// centred inside a 31-wide window (kernel sizes < 31 are zero-padded); flip = reversed taps. (Per-thread global loads of the 62 taps
// cost more address arithmetic and load latency than the convolution itself.)
__device__ __forceinline__ void cv_stage_taps(const b200_dwconv_args& a, int c0, bool flip, float (*sw)[CV_TC]) {
    const int shift = CV_HALO - a.ksize / 2;
    const int c = threadIdx.x & (CV_TC - 1);          // 256 threads = 64 channels x 4 tap phases (no integer division in the loop)
    const float* wrow = a.weight + (size_t)(c0 + c) * a.ksize - shift;
    const bool cin = c0 + c < a.D;
    for (int k = threadIdx.x / CV_TC; k < 31; k += 256 / CV_TC) {
        const bool in = cin && k >= shift && k - shift < a.ksize;
        sw[flip ? 30 - k : k][c] = in ? __ldg(wrow + k) : 0.f;
    }
}
__device__ __forceinline__ void cv_load_taps(const float (*sw)[CV_TC], int cp, cf2 (&w)[31]) {
#pragma unroll
    for (int k = 0; k < 31; ++k) w[k] = *reinterpret_cast<const cf2*>(&sw[k][2 * cp]);
}
// out[j] (+)= sum_k w[k] * src[row0 + j + k][2cp .. 2cp+1],  j < ROWS: one pass over the ROWS + 30 window rows
template <int ROWS>
__device__ __forceinline__ void conv_rows2(const cf2 (&w)[31], const float (*src)[CV_TC], int row0, int cp, cf2 (&out)[ROWS]) {
#pragma unroll
    for (int m = 0; m < ROWS + 30; ++m) {
        const cf2 v = *reinterpret_cast<const cf2*>(&src[row0 + m][2 * cp]);
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            const int k = m - j;
            if (k >= 0 && k < 31) out[j] = cv_ffma2(w[k], v, out[j]);
        }
    }
}

// 256 threads = 32 channel pairs x 8 groups of 8 tokens. A block marches CV_FWD_TILES consecutive token tiles: the taps are staged once,
// and the global loads of tile t+1 (three 16-byte pieces + their validity per thread) are issued before the convolution of tile t, so
// their latency hides behind the FMA loop instead of stalling every warp of the block.
constexpr int CV_FWD_TILES = 2;
// RESID: y = x + (the masked SiLU output), the add unmasked (b200_dwconv_args.residual)
template <bool RESID = false>
__global__ void __launch_bounds__(256, 3) dwconv_fwd_kernel(const b200_dwconv_args a) {
    __shared__ __align__(16) float xs[CV_R][CV_TC];
    __shared__ __align__(16) float sw[31][CV_TC];
    __shared__ unsigned char sok[CV_R];
    const int c0 = blockIdx.y * CV_TC, b = blockIdx.z;
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(a.x);
    const int ntiles = (a.Np + CV_TN - 1) / CV_TN;
    const int t0 = blockIdx.x * CV_FWD_TILES, t1 = min(ntiles, t0 + CV_FWD_TILES);
    cv_stage_taps(a, c0, false, sw);
    constexpr int NIT = (CV_R * (CV_TC / 8) + 255) / 256;
    uint4 u[NIT];
    bool okrow = false;       // threads < CV_R: validity (inside the sequence and not masked) of staged row threadIdx.x
    auto issue = [&](int n0) {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int i = threadIdx.x + it * 256, r = i >> 3, cc = (i & 7) * 8, n = n0 - CV_HALO + r;
            u[it] = make_uint4(0u, 0u, 0u, 0u);
            // bounds only: masked rows are read and zeroed at staging time (their validity arrives through sok)
            if (i < CV_R * (CV_TC / 8) && n >= 0 && n < a.Np && c0 + cc < a.D)
                u[it] = *reinterpret_cast<const uint4*>(x + ((size_t)b * a.Np + n) * a.D + c0 + cc);
        }
        okrow = threadIdx.x < CV_R && tok_ok(a.mask, b, n0 - CV_HALO + (int)threadIdx.x, a.Np);
    };
    issue(t0 * CV_TN);
    const int cp = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int ch = c0 + 2 * cp;
    const bool cok = ch < a.D;
    const cf2 bias2 = cok ? make_float2(__ldg(a.bias + ch), __ldg(a.bias + ch + 1)) : make_float2(0.f, 0.f);
    __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y);
    __nv_bfloat16* pre = reinterpret_cast<__nv_bfloat16*>(a.pre);
    for (int t = t0; t < t1; ++t) {
        const int n0 = t * CV_TN;
        __syncthreads();      // the previous tile's convolution is done with xs / sok (first pass: the taps are staged)
        if (threadIdx.x < CV_R) sok[threadIdx.x] = okrow;
        __syncthreads();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int i = threadIdx.x + it * 256, r = i >> 3, cc = (i & 7) * 8;
            if (i < CV_R * (CV_TC / 8)) {
                float v[8];
                cv_unpack8(sok[r] ? u[it] : make_uint4(0u, 0u, 0u, 0u), v);
                *reinterpret_cast<float4*>(&xs[r][cc]) = make_float4(v[0], v[1], v[2], v[3]);
                *reinterpret_cast<float4*>(&xs[r][cc + 4]) = make_float4(v[4], v[5], v[6], v[7]);
            }
        }
        __syncthreads();
        if (t + 1 < t1) issue(n0 + CV_TN);   // in flight during the convolution below
        if (!cok) continue;
        cf2 w[31];
        cv_load_taps(sw, cp, w);
        cf2 out[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = bias2;
        conv_rows2<8>(w, xs, rg * 8, cp, out);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = rg * 8 + j, n = n0 + r;
            if (n < a.Np) {
                const size_t off = ((size_t)b * a.Np + n) * a.D + ch;
                const bool ok = sok[r + CV_HALO];
                float o0 = ok ? __fdividef(out[j].x, 1.f + __expf(-out[j].x)) : 0.f, o1 = ok ? __fdividef(out[j].y, 1.f + __expf(-out[j].y)) : 0.f;
                if constexpr (RESID) {
                    const uint32_t ux = *reinterpret_cast<const uint32_t*>(x + off);
                    o0 += bf16_lo(ux); o1 += bf16_hi(ux);
                }
                *reinterpret_cast<uint32_t*>(y + off) = pack_bf16(o0, o1);
                if (pre) *reinterpret_cast<uint32_t*>(pre + off) = pack_bf16(out[j].x, out[j].y);
            }
        }
    }
}

constexpr int CV_TILES_PER_BLOCK = 4;   // n-tiles marched by one block: weight/bias partial sums stay in registers across them

// Backward. Staging turns dy into d(pre-activation) = dy * silu'(pre) on the fly (rows outside the sequence or masked: 0). Then the
// block splits by warp: warps 0-3 compute dx = flipped conv of d_pre (taps in registers), warps 4-7 accumulate the tap gradients
// dW[k] += d_pre[n] * x[n + k - 15] and d(bias) in registers across the block's tiles — both halves run 31 paired FMAs per element pair.
// RESID: dx = dy + the convolution's dx (b200_dwconv_args.residual)
template <bool RESID = false>
__global__ void __launch_bounds__(256, 2) dwconv_bwd_kernel(const b200_dwconv_args a) {
    extern __shared__ __align__(16) float sm[];
    float (*xs)[CV_TC] = reinterpret_cast<float (*)[CV_TC]>(sm);                          // [CV_R] masked x
    float (*dps)[CV_TC] = reinterpret_cast<float (*)[CV_TC]>(sm + CV_R * CV_TC);           // [CV_R] d_pre
    float (*sdw)[CV_TC] = reinterpret_cast<float (*)[CV_TC]>(sm + 2 * CV_R * CV_TC);       // [32] flipped taps, then (31 tap grads + bias grad)
    unsigned char* sok = reinterpret_cast<unsigned char*>(sm + (2 * CV_R + 32) * CV_TC);   // [CV_R] row validity
    const int c0 = blockIdx.y * CV_TC, b = blockIdx.z;
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(a.x);
    const __nv_bfloat16* dy = reinterpret_cast<const __nv_bfloat16*>(a.dy);
    const __nv_bfloat16* pre = reinterpret_cast<const __nv_bfloat16*>(a.pre);
    __nv_bfloat16* dx = reinterpret_cast<__nv_bfloat16*>(a.dx);
    const int cp = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int role = wrp >> 2, rg = wrp & 3;   // role 0: dx, role 1: dW / d(bias); 16 tokens per thread
    const int ch = c0 + 2 * cp;
    const bool cok = ch < a.D;
    cf2 wv[31];                                // role 0: flipped taps; role 1: tap-gradient partial sums
    cv_stage_taps(a, c0, true, sdw);
    __syncthreads();
    if (role == 0) {
        cv_load_taps(sdw, cp, wv);
    } else {
#pragma unroll
        for (int k = 0; k < 31; ++k) wv[k] = make_float2(0.f, 0.f);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * CV_TC; i += 256) sdw[i / CV_TC][i % CV_TC] = 0.f;   // ordered before its use by the tile loop's barriers
    cf2 db2 = make_float2(0.f, 0.f);
    const int ntiles = (a.Np + CV_TN - 1) / CV_TN;
    for (int tile = blockIdx.x * CV_TILES_PER_BLOCK; tile < min(ntiles, (int)(blockIdx.x + 1) * CV_TILES_PER_BLOCK); ++tile) {
        const int n0 = tile * CV_TN;
        __syncthreads();
        if (threadIdx.x < CV_R) sok[threadIdx.x] = tok_ok(a.mask, b, n0 - CV_HALO + (int)threadIdx.x, a.Np);
        __syncthreads();
        for (int i = threadIdx.x; i < CV_R * (CV_TC / 8); i += 256) {
            const int r = i / (CV_TC / 8), cc = (i % (CV_TC / 8)) * 8;
            float xv[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (sok[r] && c0 + cc < a.D) {
                const size_t off = ((size_t)b * a.Np + (n0 - CV_HALO + r)) * a.D + c0 + cc;
                const uint4 ux = *reinterpret_cast<const uint4*>(x + off), ud = *reinterpret_cast<const uint4*>(dy + off),
                            up = *reinterpret_cast<const uint4*>(pre + off);
                float pv[8];
                cv_unpack8(ux, xv); cv_unpack8(ud, dv); cv_unpack8(up, pv);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float sg = __fdividef(1.f, 1.f + __expf(-pv[j]));
                    dv[j] *= sg * (1.f + pv[j] * (1.f - sg));
                }
            }
            *reinterpret_cast<float4*>(&xs[r][cc]) = make_float4(xv[0], xv[1], xv[2], xv[3]);
            *reinterpret_cast<float4*>(&xs[r][cc + 4]) = make_float4(xv[4], xv[5], xv[6], xv[7]);
            *reinterpret_cast<float4*>(&dps[r][cc]) = make_float4(dv[0], dv[1], dv[2], dv[3]);
            *reinterpret_cast<float4*>(&dps[r][cc + 4]) = make_float4(dv[4], dv[5], dv[6], dv[7]);
        }
        __syncthreads();
        if (!cok) continue;
        if (role == 0) {
            cf2 dxo[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) dxo[j] = make_float2(0.f, 0.f);
            conv_rows2<16>(wv, dps, rg * 16, cp, dxo);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int r = rg * 16 + j, n = n0 + r;
                if (n < a.Np) {
                    const bool ok = sok[r + CV_HALO];
                    const size_t off = ((size_t)b * a.Np + n) * a.D + ch;
                    float v0 = ok ? dxo[j].x : 0.f, v1 = ok ? dxo[j].y : 0.f;
                    if constexpr (RESID) {
                        const uint32_t ud = *reinterpret_cast<const uint32_t*>(dy + off);
                        v0 += bf16_lo(ud); v1 += bf16_hi(ud);
                    }
                    *reinterpret_cast<uint32_t*>(dx + off) = pack_bf16(v0, v1);
                }
            }
        } else {
            cf2 dpr[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                dpr[j] = *reinterpret_cast<const cf2*>(&dps[rg * 16 + CV_HALO + j][2 * cp]);   // 0 for rows outside the sequence / masked
                db2.x += dpr[j].x; db2.y += dpr[j].y;
            }
#pragma unroll
            for (int m = 0; m < 46; ++m) {
                const cf2 v = *reinterpret_cast<const cf2*>(&xs[rg * 16 + m][2 * cp]);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int k = m - j;
                    if (k >= 0 && k < 31) wv[k] = cv_ffma2(dpr[j], v, wv[k]);
                }
            }
        }
    }
    if (cok && role == 1) {
#pragma unroll
        for (int k = 0; k < 31; ++k) {
            atomicAdd(&sdw[k][2 * cp], wv[k].x);
            atomicAdd(&sdw[k][2 * cp + 1], wv[k].y);
        }
        atomicAdd(&sdw[31][2 * cp], db2.x);
        atomicAdd(&sdw[31][2 * cp + 1], db2.y);
    }
    __syncthreads();
    if (threadIdx.x < CV_TC && c0 + (int)threadIdx.x < a.D) {
        const int cl = threadIdx.x, shift = CV_HALO - a.ksize / 2;
        for (int k = 0; k < a.ksize; ++k) atomicAdd(a.dweight + (size_t)(c0 + cl) * a.ksize + k, sdw[k + shift][cl]);
        atomicAdd(a.dbias + c0 + cl, sdw[31][cl]);
    }
}

// ------------------------------------------------------------------------------------------------ masked mean
__global__ void __launch_bounds__(256) masked_mean_fwd_kernel(const __nv_bfloat16* x, const unsigned char* mask, float* out, int N, int D) {
    const int b = blockIdx.y, d = blockIdx.x * 256 + threadIdx.x;
    if (d >= D) return;
    float acc = 0.f, den = 0.f;
    for (int n = 0; n < N; ++n) {
        const bool m = !mask || mask[(size_t)b * N + n];
        if (m) { acc += __bfloat162float(x[((size_t)b * N + n) * D + d]); den += 1.f; }
    }
    out[(size_t)b * D + d] = acc / fmaxf(den, 1.f);
}
__global__ void __launch_bounds__(256) masked_mean_bwd_kernel(const float* dout, const unsigned char* mask, __nv_bfloat16* dx, int N, int D) {
    __shared__ float sden;
    const int b = blockIdx.y;
    if (threadIdx.x == 0) {
        float den = 0.f;
        for (int n = 0; n < N; ++n) den += (!mask || mask[(size_t)b * N + n]) ? 1.f : 0.f;
        sden = fmaxf(den, 1.f);
    }
    __syncthreads();
    const long long total = (long long)N * D;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int n = (int)(i / D), d = (int)(i % D);
        const bool m = !mask || mask[(size_t)b * N + n];
        dx[(size_t)b * N * D + i] = __float2bfloat16(m ? dout[(size_t)b * D + d] / sden : 0.f);
    }
}


// ------------------------------------------------------------------------------------------------ ODE / CFG helpers
// out = y + a * f  (fixed-grid midpoint / Euler update, torchdiffeq semantics A.7)
__global__ void __launch_bounds__(256) axpy_kernel(const float* y, const float* f, float a, float* out, long long n) {
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) out[i] = y[i] + a * f[i];
}
// per-sample fp64 reductions for the APG projection (e2_tts.py:113-124): red[b] = (<pred - null, pred>, <pred, pred>)
__global__ void __launch_bounds__(256) cfg_reduce_kernel(const float* pred, const float* null_pred, double* red, long long per) {
    const int b = blockIdx.y;
    const float* p = pred + (size_t)b * per;
    const float* q = null_pred + (size_t)b * per;
    double d0 = 0.0, d1 = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < per; i += (long long)gridDim.x * 256) {
        const double pv = p[i], uv = (double)p[i] - (double)q[i];
        d0 += uv * pv; d1 += pv * pv;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 += __shfl_xor_sync(0xffffffffu, d1, o); }
    __shared__ double s0[8], s1[8];
    if ((threadIdx.x & 31) == 0) { s0[threadIdx.x >> 5] = d0; s1[threadIdx.x >> 5] = d1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, c = 0;
        for (int k = 0; k < 8; ++k) { a += s0[k]; c += s1[k]; }
        atomicAdd(red + 2 * b, a);
        atomicAdd(red + 2 * b + 1, c);
    }
}
// out = pred + (orth + par * keep) * strength, par = (<upd, unit>) unit, unit = pred / max(||pred||, 1e-12)
__global__ void __launch_bounds__(256) cfg_apply_kernel(const float* pred, const float* null_pred, const double* red, float* out, long long per,
                                                         float strength, int remove_parallel, float keep) {
    const int b = blockIdx.y;
    const double nrm = fmax(sqrt(red[2 * b + 1]), 1e-12);
    const double coef = red[2 * b] / (nrm * nrm);   // <upd, unit> / ||pred||
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < per; i += (long long)gridDim.x * 256) {
        const size_t j = (size_t)b * per + i;
        const double pv = pred[j], uv = pv - (double)null_pred[j];
        double upd = uv;
        if (remove_parallel) {
            const float par = (float)(coef * pv);            // reference casts parallel/orthogonal back to fp32 (:124)
            const float orth = (float)(uv - coef * pv);
            upd = (double)(orth + par * keep);
        }
        out[j] = (float)(pv + upd * strength);
    }
}

// ------------------------------------------------------------------------------------------------ MelSpec
// torchaudio MelSpectrogram -> log(clamp(., 1e-5)) (e2_tts.py:248-290), with the reference's mel_spec_kwargs: a periodic Hann window of
// win_length <= n_fft taps placed at (n_fft - win_length) / 2 (torch.stft), reflect-padded (center) or valid-only framing, |X| times
// a normalisation scale, raised to `power`. One block per (frame, batch item): the windowed frame goes through a shared-memory FFT,
// the n_fft/2+1 bins become |X|^power, then the mel filterbank restricted to each filter's non-zero band (HTK triangles: 1 008 of
// the 51 300 entries of the reference's 513 x 100 matrix are non-zero; the bands are found once per call by mel_bands_kernel), log.
// Output [B, n_mels, frames] like the reference, or [B, frames, n_mels].
// Two FFTs: power-of-two n_fft keeps the in-place radix-2 kernel (bit-reversed load, log2(n_fft) butterfly stages, an n_fft/2
// twiddle table); any other 5-smooth n_fft runs a Stockham autosort FFT of radix-4/2/3/5 stages, ping-ponging between two
// shared-memory buffers so that no digit-reversal permutation is needed (twiddle table of n_fft entries).
// (Round 1 used a direct O(n^2) DFT and the dense filterbank: ~1 M serial FMAs per frame.)
constexpr int MEL_MAX_STAGES = 12;   // 4096 = 4^6; the longest 5-smooth factorisation below 4096 is 3^7 (2187)

struct MelParams {
    const float* wave; const float* window; const float* fb; const int2* bands; float* out; const int* wave_lens;
    int nw_max, n_fft, hop, n_mels, frames, out_bnd;
    int win_off, win_len, center;
    float power, scale;
    int log2n;                                          // radix-2 kernel
    int nstages; int radix[MEL_MAX_STAGES];             // Stockham kernel, in stage order
};

__global__ void mel_bands_kernel(const float* __restrict__ fb, int nbins, int n_mels, int2* __restrict__ bands) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_mels) return;
    int lo = nbins, hi = 0;
    for (int k = 0; k < nbins; ++k)
        if (fb[(size_t)k * n_mels + m] != 0.f) { lo = min(lo, k); hi = k + 1; }
    bands[m] = make_int2(lo, hi);   // empty filter: lo >= hi
}

__device__ __forceinline__ size_t mel_out_index(const MelParams& p, int b, int f, int m) {
    return p.out_bnd ? ((size_t)b * p.frames + f) * p.n_mels + m : ((size_t)b * p.n_mels + m) * p.frames + f;
}

// ragged batch (on-device collate, trainer.py:61-82): sample b has wave_lens[b] samples and its own frame count (centred: reflect-
// padded at ITS end, valid framing: 1 + (len - n_fft) / hop); the frames behind them are the collate's zero padding, and an item
// too short for any frame (len <= n_fft/2 centred, len < n_fft otherwise) is all zeros. Returns the item's length, or -1 after
// writing frame f's zero row.
__device__ __forceinline__ int mel_frame_len(const MelParams& p, int f, int b) {
    const int nw = p.wave_lens ? min(__ldg(p.wave_lens + b), p.nw_max) : p.nw_max;
    if (p.wave_lens) {
        const int pad = p.center ? p.n_fft / 2 : 0;
        if (nw <= pad || nw + 2 * pad < p.n_fft || f >= 1 + (nw + 2 * pad - p.n_fft) / p.hop) {
            if (p.out_bnd) {           // one contiguous row
                float* row = p.out + ((size_t)b * p.frames + f) * p.n_mels;
                for (int m = threadIdx.x; m < p.n_mels; m += 256) row[m] = 0.f;
            } else {
                for (int m = threadIdx.x; m < p.n_mels; m += 256) p.out[((size_t)b * p.n_mels + m) * p.frames + f] = 0.f;
            }
            return -1;
        }
    }
    return nw;
}

// sample n of frame f times its window tap (0 outside the window's win_len taps at win_off). PLAIN: the defaults (win_len = n_fft,
// center, power 1, scale 1) compiled without the switches, so the default path runs the instructions it always ran.
template <bool PLAIN>
__device__ __forceinline__ float mel_sample(const MelParams& p, int b, int nw, int f, int n) {
    const unsigned t = (unsigned)(n - p.win_off);
    if (!PLAIN && t >= (unsigned)p.win_len) return 0.f;
    int j = f * p.hop + n;
    if (PLAIN || p.center) {                   // reflect padding by n_fft/2
        j -= p.n_fft / 2;
        if (j < 0) j = -j;
        if (j >= nw) j = 2 * (nw - 1) - j;
    }
    return __ldg(p.wave + (size_t)b * p.nw_max + j) * __ldg(p.window + t);   // read-only path: the struct carries no __restrict__
}

// |X_k| * scale raised to the power, then the band-limited filterbank and the log
template <bool PLAIN>
__device__ __forceinline__ void mel_finish(const MelParams& p, const float2* z, float* mag, int b, int f) {
    const int nbins = p.n_fft / 2 + 1;
    for (int k = threadIdx.x; k < nbins; k += 256) {
        const float a = sqrtf(z[k].x * z[k].x + z[k].y * z[k].y);
        if (PLAIN) { mag[k] = a; continue; }
        const float m = a * p.scale;
        mag[k] = p.power == 1.f ? m : (p.power == 2.f ? m * m : powf(m, p.power));
    }
    __syncthreads();
    for (int m = threadIdx.x; m < p.n_mels; m += 256) {
        const int2 bd = __ldg(p.bands + m);
        float acc = 0.f;
        for (int k = bd.x; k < bd.y; ++k) acc += mag[k] * __ldg(p.fb + (size_t)k * p.n_mels + m);
        p.out[mel_out_index(p, b, f, m)] = logf(fmaxf(acc, 1e-5f));
    }
}

template <bool PLAIN>
__global__ void __launch_bounds__(256) melspec_kernel(const MelParams p) {
    extern __shared__ float2 zsm[];
    const int n_fft = p.n_fft, log2n = p.log2n;
    float2* z = zsm;                 // [n_fft] in-place FFT buffer
    float2* tw = z + n_fft;          // [n_fft/2] twiddles e^{-2 pi i k / n_fft}
    float* mag = reinterpret_cast<float*>(tw + n_fft / 2);   // [n_fft/2 + 1]
    const int f = blockIdx.x, b = blockIdx.y;
    const int nw = mel_frame_len(p, f, b);
    if (nw < 0) return;
    for (int n = threadIdx.x; n < n_fft; n += 256) {
        const int r = (int)(__brev((unsigned)n) >> (32 - log2n));
        z[r] = make_float2(mel_sample<PLAIN>(p, b, nw, f, n), 0.f);
        if (n < n_fft / 2) {
            float sn, cs;
            sincospif(-2.f * (float)n / (float)n_fft, &sn, &cs);
            tw[n] = make_float2(cs, sn);
        }
    }
    __syncthreads();
    for (int s = 1; s <= log2n; ++s) {
        const int half = 1 << (s - 1), tstride = n_fft >> s;
        for (int t = threadIdx.x; t < n_fft / 2; t += 256) {
            const int pos = t & (half - 1);
            const int i = ((t >> (s - 1)) << s) + pos, j = i + half;
            const float2 w = tw[pos * tstride], u = z[i], x = z[j];
            const float2 v = make_float2(x.x * w.x - x.y * w.y, x.x * w.y + x.y * w.x);
            z[i] = make_float2(u.x + v.x, u.y + v.y);
            z[j] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
    mel_finish<PLAIN>(p, z, mag, b, f);
}

template <bool PLAIN>
__global__ void __launch_bounds__(256) melspec_mixed_kernel(const MelParams p) {
    extern __shared__ float2 zsm[];
    const int n_fft = p.n_fft;
    float2* z0 = zsm;                      // [2 n_fft]: Stockham ping-pong, stage s reads z0 + (s & 1) n_fft
    float2* tw = zsm + 2 * n_fft;          // [n_fft] twiddles e^{-2 pi i k / n_fft}
    const int f = blockIdx.x, b = blockIdx.y;
    const int nw = mel_frame_len(p, f, b);
    if (nw < 0) return;
    for (int n = threadIdx.x; n < n_fft; n += 256) {
        z0[n] = make_float2(mel_sample<PLAIN>(p, b, nw, f, n), 0.f);
        float sn, cs;
        sincospif(-2.f * (float)n / (float)n_fft, &sn, &cs);
        tw[n] = make_float2(cs, sn);
    }
    __syncthreads();
    int Ns = 1;
    for (int s = 0; s < p.nstages; ++s) {
        const float2* in = z0 + (s & 1) * n_fft;
        float2* out = z0 + ((s & 1) ^ 1) * n_fft;
        switch (p.radix[s]) {
            case 4: stockham_stage<4>(in, out, tw, n_fft, Ns); break;
            case 2: stockham_stage<2>(in, out, tw, n_fft, Ns); break;
            case 3: stockham_stage<3>(in, out, tw, n_fft, Ns); break;
            default: stockham_stage<5>(in, out, tw, n_fft, Ns); break;
        }
        Ns *= p.radix[s];
        __syncthreads();
    }
    const int last = p.nstages & 1;
    mel_finish<PLAIN>(p, z0 + last * n_fft, reinterpret_cast<float*>(z0 + (last ^ 1) * n_fft), b, f);   // |X|^p in the free buffer
}

}  // namespace b200

using namespace b200;

extern "C" int b200_small_linear_fwd(const b200_small_linear_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->X && a->W && a->Y, "small_linear_fwd: null pointer");
    B200_REQUIRE(a->B > 0 && a->B <= SL_MAXB && a->N > 0 && a->K > 0, "small_linear: batch must be 1..%d", SL_MAXB);
    B200_REQUIRE(a->act >= 0 && a->act <= 5 && (a->act != 5 || a->seg > 0), "small_linear: bad activation");
    B200_REQUIRE(!a->seg_major || (a->seg > 0 && a->N % a->seg == 0), "small_linear: seg_major needs N %% seg == 0");
    {
        const int x_in_smem = ((long long)a->B * a->K <= SL_XS_MAX) ? 1 : 0;
        const size_t smem = x_in_smem ? (size_t)a->B * a->K * sizeof(float) : 0;
        static DeviceOnce once;
        cudaError_t e = set_max_smem_once(once, small_linear_fwd_kernel, SL_XS_MAX * (int)sizeof(float));
        B200_REQUIRE(e == cudaSuccess, "small_linear_fwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        // enough outputs per warp to amortise the X staging, but at least ~2 blocks per SM when N is large
        int npw = 1;
        while (npw < 8 && (a->N + 8 * (npw * 2) - 1) / (8 * (npw * 2)) >= 2 * num_sms()) npw *= 2;
        const int per_block = 8 * npw;
        small_linear_fwd_kernel<<<(a->N + per_block - 1) / per_block, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*a, npw, x_in_smem);
    }
    return check_launch("small_linear_fwd_kernel");
}
extern "C" int b200_small_linear_bwd(const b200_small_linear_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->X && a->W && a->Z && a->dY && a->dZ && a->dW, "small_linear_bwd: null pointer");
    B200_REQUIRE(a->B > 0 && a->B <= SL_MAXB && a->N > 0 && a->K > 0, "small_linear: batch must be 1..%d", SL_MAXB);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    small_linear_bwd_w_kernel<<<(a->N + 7) / 8, 256, 0, st>>>(*a);
    if (int rc = check_launch("small_linear_bwd_w_kernel")) return rc;
    if (a->dX) {
        cudaError_t e = cudaMemsetAsync(a->dX, 0, (size_t)a->B * a->K * sizeof(float), st);
        B200_REQUIRE(e == cudaSuccess, "small_linear_bwd: memset: %s", cudaGetErrorString(e));
        int slab = SL_SLAB;   // fewer features per block when N is small, so that the slabs still cover the GPU
        while (slab > 32 && (a->N + slab - 1) / slab < num_sms()) slab >>= 1;
        const size_t smem = (size_t)a->B * slab * sizeof(float);   // <= 64 KB
        static DeviceOnce once;
        cudaError_t e2 = set_max_smem_once(once, small_linear_bwd_x_kernel, SL_MAXB * SL_SLAB * (int)sizeof(float));
        B200_REQUIRE(e2 == cudaSuccess, "small_linear_bwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e2));
        small_linear_bwd_x_kernel<<<(a->N + slab - 1) / slab, 256, smem, st>>>(*a, slab);
        return check_launch("small_linear_bwd_x_kernel");
    }
    return 0;
}
extern "C" int b200_fourier_embed(const float* times, const float* weights, float* out, int32_t B, int32_t half, b200_stream_t stream) {
    B200_REQUIRE(times && weights && out && B > 0 && half > 0, "fourier_embed: bad arguments");
    fourier_embed_kernel<<<(B * half + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(times, weights, out, B, half);
    return check_launch("fourier_embed_kernel");
}

static int check_conv(const b200_dwconv_args* a) {
    B200_REQUIRE(a && a->x && a->weight && a->bias, "dwconv: null pointer");
    B200_REQUIRE((a->ksize & 1) && a->ksize >= 1 && a->ksize <= 31, "dwconv: kernel_size must be odd and <= 31 (got %d)", a->ksize);
    B200_REQUIRE(a->D % 8 == 0 && a->B > 0 && a->B <= 65535 && a->Np > 0, "dwconv: unsupported shape");
    B200_REQUIRE(a->residual == 0 || a->residual == 1, "dwconv: residual must be 0 or 1 (got %d)", a->residual);
    return 0;
}
extern "C" int b200_dwconv_fwd(const b200_dwconv_args* a, b200_stream_t stream) {
    if (check_conv(a)) return -1;
    B200_REQUIRE(a->y, "dwconv_fwd: null output");
    B200_REQUIRE(!a->residual || a->y != a->x, "dwconv_fwd: with residual, y must not alias x (neighbouring tiles read x)");
    const int ntiles = (a->Np + CV_TN - 1) / CV_TN;
    dim3 grid((ntiles + CV_FWD_TILES - 1) / CV_FWD_TILES, (a->D + CV_TC - 1) / CV_TC, a->B);
    if (a->residual) dwconv_fwd_kernel<true><<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    else dwconv_fwd_kernel<false><<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("dwconv_fwd_kernel");
}
extern "C" int b200_dwconv_bwd(const b200_dwconv_args* a, b200_stream_t stream) {
    if (check_conv(a)) return -1;
    B200_REQUIRE(a->dy && a->dx && a->dweight && a->dbias, "dwconv_bwd: null pointer");
    B200_REQUIRE(a->pre, "dwconv_bwd: the pre-activation saved by b200_dwconv_fwd (args.pre) is required");
    const size_t smem = (size_t)(2 * CV_R + 32) * CV_TC * sizeof(float) + 128;
    const int ntiles = (a->Np + CV_TN - 1) / CV_TN;
    dim3 grid((ntiles + CV_TILES_PER_BLOCK - 1) / CV_TILES_PER_BLOCK, (a->D + CV_TC - 1) / CV_TC, a->B);
    if (a->residual) {
        static DeviceOnce once_r;
        B200_REQUIRE(set_max_smem_once(once_r, dwconv_bwd_kernel<true>, (int)smem) == cudaSuccess, "dwconv_bwd: cudaFuncSetAttribute failed");
        dwconv_bwd_kernel<true><<<grid, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    } else {
        static DeviceOnce once;
        B200_REQUIRE(set_max_smem_once(once, dwconv_bwd_kernel<false>, (int)smem) == cudaSuccess, "dwconv_bwd: cudaFuncSetAttribute failed");
        dwconv_bwd_kernel<false><<<grid, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    }
    return check_launch("dwconv_bwd_kernel");
}

extern "C" int b200_masked_mean_fwd(const void* x, const uint8_t* mask, float* out, int32_t B, int32_t N, int32_t D, b200_stream_t stream) {
    B200_REQUIRE(x && out && B > 0 && N > 0 && D > 0, "masked_mean_fwd: bad arguments");
    masked_mean_fwd_kernel<<<dim3((D + 255) / 256, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>((const __nv_bfloat16*)x, mask, out, N, D);
    return check_launch("masked_mean_fwd_kernel");
}
extern "C" int b200_masked_mean_bwd(const float* dout, const uint8_t* mask, void* dx, int32_t B, int32_t N, int32_t D, b200_stream_t stream) {
    B200_REQUIRE(dout && dx && B > 0 && N > 0 && D > 0, "masked_mean_bwd: bad arguments");
    masked_mean_bwd_kernel<<<dim3(64, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(dout, mask, (__nv_bfloat16*)dx, N, D);
    return check_launch("masked_mean_bwd_kernel");
}

extern "C" int b200_axpy(const float* y, const float* f, float a, float* out, int64_t n, b200_stream_t stream) {
    B200_REQUIRE(y && f && out && n > 0, "axpy: bad arguments");
    const long long g = (n + 255) / 256;
    axpy_kernel<<<(unsigned)(g > num_sms() * 16 ? num_sms() * 16 : g), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(y, f, a, out, n);
    return check_launch("axpy_kernel");
}
extern "C" int b200_cfg_combine(const float* pred, const float* null_pred, double* ws_red, float* out, int32_t B, int64_t per_sample,
                                float cfg_strength, int32_t remove_parallel, float keep_parallel_frac, b200_stream_t stream) {
    B200_REQUIRE(pred && null_pred && ws_red && out && B > 0 && B <= 65535 && per_sample > 0, "cfg_combine: bad arguments");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(ws_red, 0, (size_t)B * 2 * sizeof(double), st);
    B200_REQUIRE(e == cudaSuccess, "cfg_combine: memset: %s", cudaGetErrorString(e));
    const int gx = (int)((per_sample + 256 * 8 - 1) / (256 * 8));
    cfg_reduce_kernel<<<dim3(gx < 1 ? 1 : gx, B), 256, 0, st>>>(pred, null_pred, ws_red, per_sample);
    if (int rc = check_launch("cfg_reduce_kernel")) return rc;
    cfg_apply_kernel<<<dim3(gx < 1 ? 1 : gx, B), 256, 0, st>>>(pred, null_pred, ws_red, out, per_sample, cfg_strength, remove_parallel, keep_parallel_frac);
    return check_launch("cfg_apply_kernel");
}
// n_fft = 2^a 3^b 5^c -> radices in stage order (4s first, then a leftover 2, 3s, 5s); 0 stages when n_fft is not 5-smooth
static int mel_factor(int n, int* radix) {
    int s = 0;
    while (n % 4 == 0 && s < MEL_MAX_STAGES) { radix[s++] = 4; n /= 4; }
    for (int r : {2, 3, 5})
        while (n % r == 0 && s < MEL_MAX_STAGES) { radix[s++] = r; n /= r; }
    return n == 1 ? s : 0;
}
extern "C" int b200_melspec_ex(const b200_melspec_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->wave && a->window && a->fb && a->out && a->ws_bands && a->B > 0 && a->B <= 65535, "melspec: bad arguments");
    const int n_fft = a->n_fft;
    MelParams p{};
    p.nstages = n_fft >= 64 && n_fft <= 4096 ? mel_factor(n_fft, p.radix) : 0;
    B200_REQUIRE(p.nstages > 0, "melspec: n_fft must be in [64, 4096] with no prime factor other than 2, 3 and 5 (got %d)", n_fft);
    B200_REQUIRE(a->hop > 0 && a->n_mels > 0, "melspec: hop and n_mels must be positive");
    B200_REQUIRE(a->win_length >= 1 && a->win_length <= n_fft, "melspec: win_length must be in [1, n_fft] (got %d)", a->win_length);
    B200_REQUIRE(a->power > 0.f && a->norm_scale > 0.f, "melspec: power and norm_scale must be positive");
    B200_REQUIRE(a->center ? a->nw > n_fft / 2 : a->nw >= n_fft,
                 "melspec: the wave must be longer than n_fft/2 with center (reflect padding), at least n_fft long without");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(a->ws_bands) & 7) == 0, "melspec: ws_bands must be 8-byte aligned");
    const int pad = a->center ? n_fft / 2 : 0;
    p.wave = a->wave; p.window = a->window; p.fb = a->fb; p.bands = reinterpret_cast<const int2*>(a->ws_bands); p.out = a->out;
    p.wave_lens = a->wave_lens;
    p.nw_max = a->nw; p.n_fft = n_fft; p.hop = a->hop; p.n_mels = a->n_mels; p.out_bnd = a->out_bnd;
    p.frames = 1 + (a->nw + 2 * pad - n_fft) / a->hop;
    p.win_off = (n_fft - a->win_length) / 2; p.win_len = a->win_length; p.center = a->center ? 1 : 0;
    p.power = a->power; p.scale = a->norm_scale;
    while ((1 << p.log2n) < n_fft) ++p.log2n;
    mel_bands_kernel<<<(a->n_mels + 127) / 128, 128, 0, st>>>(a->fb, n_fft / 2 + 1, a->n_mels, reinterpret_cast<int2*>(a->ws_bands));
    if (int rc = check_launch("mel_bands_kernel")) return rc;
    const bool plain = p.win_len == n_fft && p.center && p.power == 1.f && p.scale == 1.f;
    const dim3 grid(p.frames, a->B);
    if ((n_fft & (n_fft - 1)) == 0) {
        const size_t smem = (size_t)n_fft * 8 + (size_t)(n_fft / 2) * 8 + (size_t)(n_fft / 2 + 1) * 4;   // <= 52 KB at 4096
        static DeviceOnce once, once_p;
        if (plain) {
            B200_REQUIRE(set_max_smem_once(once_p, melspec_kernel<true>, 64 * 1024) == cudaSuccess, "melspec: cudaFuncSetAttribute failed");
            melspec_kernel<true><<<grid, 256, smem, st>>>(p);
        } else {
            B200_REQUIRE(set_max_smem_once(once, melspec_kernel<false>, 64 * 1024) == cudaSuccess, "melspec: cudaFuncSetAttribute failed");
            melspec_kernel<false><<<grid, 256, smem, st>>>(p);
        }
        return check_launch("melspec_kernel");
    }
    // two buffers and the twiddles: <= 97 200 B at 4050, the largest 5-smooth size, so the opt-in above 48 KB is needed (H100: 227 KB)
    const size_t smem = (size_t)n_fft * 3 * 8;
    static DeviceOnce once, once_p;
    if (plain) {
        B200_REQUIRE(set_max_smem_once(once_p, melspec_mixed_kernel<true>, 3 * 8 * 4096) == cudaSuccess, "melspec: cudaFuncSetAttribute failed");
        melspec_mixed_kernel<true><<<grid, 256, smem, st>>>(p);
    } else {
        B200_REQUIRE(set_max_smem_once(once, melspec_mixed_kernel<false>, 3 * 8 * 4096) == cudaSuccess, "melspec: cudaFuncSetAttribute failed");
        melspec_mixed_kernel<false><<<grid, 256, smem, st>>>(p);
    }
    return check_launch("melspec_mixed_kernel");
}
extern "C" int b200_melspec(const float* wave, const float* window, const float* fb, float* out, int32_t B, int32_t nw, int32_t n_fft,
                            int32_t hop, int32_t n_mels, int32_t* ws_bands, const int32_t* wave_lens, int32_t out_bnd, b200_stream_t stream) {
    b200_melspec_args a{};
    a.wave = wave; a.window = window; a.fb = fb; a.out = out; a.B = B; a.nw = nw; a.n_fft = n_fft; a.hop = hop; a.n_mels = n_mels;
    a.ws_bands = ws_bands; a.wave_lens = wave_lens; a.out_bnd = out_bnd;
    a.win_length = n_fft; a.center = 1; a.power = 1.f; a.norm_scale = 1.f;
    return b200_melspec_ex(&a, stream);
}
