// Vocos mel decoder (the reference's E2TTS(use_vocos=True), e2_tts.py:1244, :1440-1451): the non-GEMM stages of the published
// vocos-mel-24khz network. The backbone's embed Conv1d runs as im2col + b200_gemm, each ConvNeXt block as dwconv+LayerNorm here, then
// b200_gemm with the GELU epilogue (pwconv1) and b200_gemm with the (z + bias) * gamma + x epilogue (pwconv2); the head's Linear is an
// fp32-output b200_gemm, and its inverse STFT is the two kernels at the end of this file.
// A ragged batch is a [B * T] row layout with per-item frame counts lens[b]; every kernel keeps the items apart (zero padding at each
// item's own ends, padded rows neither read nor left non-zero), so an item decodes bit for bit as it would alone.
#include <cuda_bf16.h>

#include "common.cuh"
#include "fft.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int VOCOS_TAPS = 7;             // ConvNeXt dwconv and embed kernel size (padding 3)
constexpr int VOCOS_MAX_PAIRS = 16;       // LayerNorm width: D / 64 column pairs per lane, D <= 1024
constexpr int ISTFT_MAX_STAGES = 6;       // 4096 = 4^6

__device__ __forceinline__ int item_len(const int32_t* lens, int b, int T) { return min(max(__ldg(lens + b), 0), T); }

__device__ __forceinline__ float vocos_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// one block per row (b, t); column c * 7 + j of the row = mel[b, t + j - 3, c]
__global__ void __launch_bounds__(256) vocos_im2col_kernel(const float* __restrict__ mel, const int32_t* __restrict__ lens,
                                                           __nv_bfloat16* __restrict__ A, int T, int C, int lda, int db_to_amp) {
    const int row = blockIdx.x, b = row / T, t = row - b * T;
    const int len = item_len(lens, b, T);
    __nv_bfloat16* out = A + (size_t)row * lda;
    for (int col = threadIdx.x; col < lda; col += 256) {
        const int c = col / VOCOS_TAPS, s = t + (col - c * VOCOS_TAPS) - VOCOS_TAPS / 2;
        float v = 0.f;
        if (t < len && c < C && s >= 0 && s < len) {
            v = __ldg(mel + ((size_t)b * T + s) * C + c);
            if (db_to_amp) v = (float)exp10((double)v * 0.05);   // 10^(x/20) rounded once to fp32
        }
        out[col] = __float2bfloat16_rn(v);
    }
}

// One warp per row; lane l holds the column pairs 64 i + 2 l. CONV: depthwise k-7 conv + bias over the item's rows first.
// The statistics are two-pass over the fp32 values held in registers: mean, then the mean squared deviation (biased, as nn.LayerNorm).
template <bool CONV>
__global__ void __launch_bounds__(256) vocos_ln_kernel(const b200_vocos_ln_args a) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= a.B * a.T) return;
    const int b = row / a.T, t = row - b * a.T, D = a.D, np = D >> 6;
    const int len = item_len(a.lens, b, a.T);
    __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y) + (size_t)row * D;
    if (t >= len) {
        for (int i = 0; i < np; ++i) *reinterpret_cast<uint32_t*>(y + 64 * i + 2 * lane) = 0u;
        return;
    }
    const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(a.x) + (size_t)b * a.T * D;
    float v[2 * VOCOS_MAX_PAIRS];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < VOCOS_MAX_PAIRS; ++i) {
        if (i >= np) break;
        const int c = 64 * i + 2 * lane;
        float v0, v1;
        if constexpr (CONV) {
            v0 = __ldg(a.conv_b + c); v1 = __ldg(a.conv_b + c + 1);
#pragma unroll
            for (int j = 0; j < VOCOS_TAPS; ++j) {
                const int s = t + j - VOCOS_TAPS / 2;
                if (s < 0 || s >= len) continue;
                const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(xb + (size_t)s * D + c));
                v0 = fmaf(__ldg(a.conv_w + c * VOCOS_TAPS + j), bf16_lo(u), v0);
                v1 = fmaf(__ldg(a.conv_w + (c + 1) * VOCOS_TAPS + j), bf16_hi(u), v1);
            }
        } else {
            const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(xb + (size_t)t * D + c));
            v0 = bf16_lo(u); v1 = bf16_hi(u);
        }
        v[2 * i] = v0; v[2 * i + 1] = v1;
        sum += v0 + v1;
    }
    const float mean = vocos_warp_sum(sum) / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < VOCOS_MAX_PAIRS; ++i) {
        if (i >= np) break;
        const float d0 = v[2 * i] - mean, d1 = v[2 * i + 1] - mean;
        sq = fmaf(d0, d0, fmaf(d1, d1, sq));
    }
    const float rstd = 1.f / sqrtf(vocos_warp_sum(sq) / (float)D + a.eps);
#pragma unroll
    for (int i = 0; i < VOCOS_MAX_PAIRS; ++i) {
        if (i >= np) break;
        const int c = 64 * i + 2 * lane;
        const float o0 = fmaf((v[2 * i] - mean) * rstd, __ldg(a.ln_w + c), __ldg(a.ln_b + c));
        const float o1 = fmaf((v[2 * i + 1] - mean) * rstd, __ldg(a.ln_w + c + 1), __ldg(a.ln_b + c + 1));
        *reinterpret_cast<uint32_t*>(y + c) = pack_bf16(o0, o1);
    }
}

struct IstftParams {
    const float* spec; const float* window; const int32_t* lens; float* frames; float* audio;
    int T, n_fft, hop, pad, nstages;
    int radix[ISTFT_MAX_STAGES];
};

// One block per frame (t, b) of the item: spectrum -> inverse real FFT -> window, into the frame workspace. The inverse real FFT is the
// forward complex FFT of conj(X) over the Hermitian extension of the n_fft/2 + 1 bins: irfft(X)[n] = Re(FFT(conj X)[n]) / n_fft.
__global__ void __launch_bounds__(256) vocos_istft_frames_kernel(const IstftParams p) {
    extern __shared__ float2 zsm[];
    const int N = p.n_fft, t = blockIdx.x, b = blockIdx.y;
    if (t >= item_len(p.lens, b, p.T)) return;
    float2* z0 = zsm;            // [2 N]: Stockham ping-pong, stage s reads z0 + (s & 1) N
    float2* tw = zsm + 2 * N;    // [N] twiddles e^{-2 pi i k / N}
    const float* row = p.spec + ((size_t)b * p.T + t) * (N + 2);
    const int K = N / 2 + 1;
    for (int k = threadIdx.x; k < K; k += 256) {
        const float m = fminf(expf(__ldg(row + k)), 100.f);
        float sn, cs;
        sincosf(__ldg(row + K + k), &sn, &cs);   // full range reduction: the phases are unbounded
        const float re = m * cs, im = (k == 0 || k == N / 2) ? 0.f : m * sn;
        z0[k] = make_float2(re, -im);
        if (k > 0 && k < N / 2) z0[N - k] = make_float2(re, im);
    }
    for (int n = threadIdx.x; n < N; n += 256) {
        float sn, cs;
        sincospif(-2.f * (float)n / (float)N, &sn, &cs);
        tw[n] = make_float2(cs, sn);
    }
    __syncthreads();
    int Ns = 1;
    for (int s = 0; s < p.nstages; ++s) {
        const float2* in = z0 + (s & 1) * N;
        float2* out = z0 + ((s & 1) ^ 1) * N;
        if (p.radix[s] == 4) stockham_stage<4>(in, out, tw, N, Ns);
        else stockham_stage<2>(in, out, tw, N, Ns);
        Ns *= p.radix[s];
        __syncthreads();
    }
    const float2* z = z0 + (p.nstages & 1) * N;
    float* out = p.frames + ((size_t)b * p.T + t) * N;
    const float scale = 1.f / (float)N;   // exact: N is a power of two
    for (int n = threadIdx.x; n < N; n += 256) out[n] = z[n].x * scale * __ldg(p.window + n);
}

// One thread per output sample n of item b: position m = n + pad of the overlap-added signal takes frames t with t hop <= m <
// t hop + n_fft and t < lens[b], summed in increasing t together with the window^2 envelope of the same frames.
__global__ void __launch_bounds__(256) vocos_istft_ola_kernel(const IstftParams p) {
    const int b = blockIdx.y, n = blockIdx.x * 256 + threadIdx.x, total = p.T * p.hop;
    if (n >= total) return;
    const int len = item_len(p.lens, b, p.T);
    float* out = p.audio + (size_t)b * total;
    if (n >= len * p.hop) { out[n] = 0.f; return; }
    const int m = n + p.pad;
    const int first = m - p.n_fft + 1;
    const int t0 = first <= 0 ? 0 : (first + p.hop - 1) / p.hop, t1 = min(len - 1, m / p.hop);
    float acc = 0.f, env = 0.f;
    for (int t = t0; t <= t1; ++t) {
        const int k = m - t * p.hop;
        const float w = __ldg(p.window + k);
        acc += __ldg(p.frames + ((size_t)b * p.T + t) * p.n_fft + k);
        env = fmaf(w, w, env);
    }
    out[n] = acc / env;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_vocos_im2col(const float* mel, const int32_t* lens, void* A, int32_t B, int32_t T, int32_t C, int32_t lda, int32_t db_to_amp,
                                 b200_stream_t stream) {
    B200_REQUIRE(mel && lens && A, "vocos_im2col: null pointer");
    B200_REQUIRE(B > 0 && T > 0 && C > 0 && (long long)B * T < (1ll << 31), "vocos_im2col: bad shape B=%d T=%d C=%d", B, T, C);
    B200_REQUIRE(lda >= VOCOS_TAPS * C && (lda % 8) == 0, "vocos_im2col: lda=%d must be a multiple of 8 and >= 7 C", lda);
    vocos_im2col_kernel<<<B * T, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(mel, lens, reinterpret_cast<__nv_bfloat16*>(A), T, C,
                                                                                     lda, db_to_amp);
    return check_launch("vocos_im2col_kernel");
}

static int check_ln(const b200_vocos_ln_args* a, bool conv) {
    B200_REQUIRE(a && a->x && a->y && a->lens && a->ln_w && a->ln_b && (!conv || (a->conv_w && a->conv_b)), "vocos_ln: null pointer");
    B200_REQUIRE(a->x != a->y, "vocos_ln: y must not alias x");
    B200_REQUIRE(a->B > 0 && a->T > 0 && (long long)a->B * a->T < (1ll << 31), "vocos_ln: bad shape B=%d T=%d", a->B, a->T);
    B200_REQUIRE(a->D > 0 && (a->D % 64) == 0 && a->D <= 64 * VOCOS_MAX_PAIRS, "vocos_ln: D=%d must be a multiple of 64 up to 1024", a->D);
    return 0;
}

extern "C" int b200_vocos_dwconv_ln(const b200_vocos_ln_args* a, b200_stream_t stream) {
    if (int rc = check_ln(a, true)) return rc;
    vocos_ln_kernel<true><<<(a->B * a->T + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("vocos_dwconv_ln_kernel");
}

extern "C" int b200_vocos_ln(const b200_vocos_ln_args* a, b200_stream_t stream) {
    if (int rc = check_ln(a, false)) return rc;
    vocos_ln_kernel<false><<<(a->B * a->T + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("vocos_ln_kernel");
}

extern "C" int b200_vocos_istft(const b200_vocos_istft_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->spec && a->window && a->lens && a->frames && a->audio, "vocos_istft: null pointer");
    const int N = a->n_fft;
    B200_REQUIRE(N >= 64 && N <= 4096 && (N & (N - 1)) == 0, "vocos_istft: n_fft=%d must be a power of two in [64, 4096]", N);
    B200_REQUIRE(a->hop >= 1 && a->hop <= N && ((N - a->hop) % 2) == 0, "vocos_istft: hop=%d must be in [1, n_fft] with n_fft - hop even",
                 a->hop);
    B200_REQUIRE(a->B > 0 && a->B <= 65535 && a->T > 0 && (long long)a->T * a->hop < (1ll << 31), "vocos_istft: bad shape B=%d T=%d",
                 a->B, a->T);
    IstftParams p{};
    p.spec = a->spec; p.window = a->window; p.lens = a->lens; p.frames = a->frames; p.audio = a->audio;
    p.T = a->T; p.n_fft = N; p.hop = a->hop; p.pad = (N - a->hop) / 2;
    for (int n = N; n > 1; n /= (n >= 4 ? 4 : 2)) p.radix[p.nstages++] = n >= 4 ? 4 : 2;
    static DeviceOnce once;
    B200_REQUIRE(set_max_smem_once(once, vocos_istft_frames_kernel, 3 * 8 * 4096) == cudaSuccess, "vocos_istft: cudaFuncSetAttribute failed");
    vocos_istft_frames_kernel<<<dim3(a->T, a->B), 256, (size_t)N * 3 * 8, st>>>(p);
    if (int rc = check_launch("vocos_istft_frames_kernel")) return rc;
    vocos_istft_ola_kernel<<<dim3((a->T * a->hop + 255) / 256, a->B), 256, 0, st>>>(p);
    return check_launch("vocos_istft_ola_kernel");
}
