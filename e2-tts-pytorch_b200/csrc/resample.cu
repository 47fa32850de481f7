// Resampling of a ragged, mixed-rate batch ahead of the mel (trainer.py:116-118: torchaudio.transforms.Resample per item in the
// reference's dataset). One block covers RS_OUT_PER_BLOCK outputs of one item; each output is one fma chain over its phase's band of
// non-zero taps, read from shared memory when the item's rate pair fits there. HBM traffic: 4 B per input sample read (the band
// overlap of neighbouring outputs is served by L1), 4 B per output sample written.
#include "common.cuh"

namespace b200 {

constexpr int RS_THREADS = 256;
constexpr int RS_OUT_PER_THREAD = 8;
constexpr int RS_OUT_PER_BLOCK = RS_THREADS * RS_OUT_PER_THREAD;
constexpr int RS_PAIR_WORDS = 6;
constexpr int RS_SMEM_MAX = 48 * 1024;

struct RsPair {
    int orig, nw, width, phase0, tap0, ntaps;
};

// torchaudio's length: ceil(torch.as_tensor(new' * L / orig')) — the quotient rounded to double, then to float, then a float ceil —
// capped at the new' (L div orig' + 1) samples its strided convolution produces
__device__ __forceinline__ int rs_out_len(const RsPair& p, int L) {
    const long long num = (long long)p.nw * L;
    const float q = __double2float_rn((double)num / (double)p.orig);
    const long long n = min((long long)ceilf(q), (long long)p.nw * (L / p.orig + 1));
    return (int)n;
}

template <bool STAGE>
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const b200_resample_args a) {
    extern __shared__ int32_t rs_smem[];
    const int b = blockIdx.y;
    const int len = min(max(__ldg(a.wave_lens + b), 0), a.nw);
    const int pi = __ldg(a.pair_idx + b);
    const float* x = a.wave + (size_t)b * a.nw;
    float* y = a.out + (size_t)b * a.nr;
    const int j0 = blockIdx.x * RS_OUT_PER_BLOCK + threadIdx.x;

    if (pi < 0) {   // equal rates: the item itself
        const int n = min(len, a.nr);
        if (blockIdx.x == 0 && threadIdx.x == 0) a.out_lens[b] = n;
#pragma unroll
        for (int r = 0; r < RS_OUT_PER_THREAD; ++r) {
            const int j = j0 + r * RS_THREADS;
            if (j < a.nr) y[j] = j < n ? __ldg(x + j) : 0.f;
        }
        return;
    }
    RsPair p{};
    if (pi < a.n_pairs) {
        const int32_t* d = a.pairs + RS_PAIR_WORDS * pi;
        p = RsPair{__ldg(d), __ldg(d + 1), __ldg(d + 2), __ldg(d + 3), __ldg(d + 4), __ldg(d + 5)};
    }
    const int n = pi < a.n_pairs ? min(rs_out_len(p, len), a.nr) : 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) a.out_lens[b] = n;
    const int jb = blockIdx.x * RS_OUT_PER_BLOCK;
    if (jb >= n) {   // the collate's zero padding only (uniform per block: no barrier below is skipped by part of it)
#pragma unroll
        for (int r = 0; r < RS_OUT_PER_THREAD; ++r) {
            const int j = j0 + r * RS_THREADS;
            if (j < a.nr) y[j] = 0.f;
        }
        return;
    }
    const int32_t* phases = a.phases + 3 * p.phase0;
    const float* taps = a.taps + p.tap0;
    if (STAGE) {
        int32_t* sp = rs_smem;
        float* st = reinterpret_cast<float*>(rs_smem + 3 * p.nw);
        for (int i = threadIdx.x; i < 3 * p.nw; i += RS_THREADS) sp[i] = __ldg(phases + i);
        for (int i = threadIdx.x; i < p.ntaps; i += RS_THREADS) st[i] = __ldg(taps + i);
        __syncthreads();
        phases = sp;
        taps = st;
    }
#pragma unroll
    for (int r = 0; r < RS_OUT_PER_THREAD; ++r) {
        const int j = j0 + r * RS_THREADS;
        if (j >= a.nr) break;
        float acc = 0.f;
        if (j < n) {
            const int q = j / p.nw, k = j - q * p.nw;
            const int first = STAGE ? phases[3 * k] : __ldg(phases + 3 * k);
            const int count = STAGE ? phases[3 * k + 1] : __ldg(phases + 3 * k + 1);
            const int off = STAGE ? phases[3 * k + 2] : __ldg(phases + 3 * k + 2);
            const long long s = (long long)q * p.orig - p.width + first;
            for (int i = 0; i < count; ++i) {
                const long long m = s + i;
                const float v = (m >= 0 && m < len) ? __ldg(x + m) : 0.f;
                const float w = STAGE ? taps[off + i] : __ldg(taps + off + i);
                acc = fmaf(w, v, acc);
            }
        }
        y[j] = acc;
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_resample(const b200_resample_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->wave && a->wave_lens && a->pair_idx && a->out && a->out_lens, "resample: null pointer");
    B200_REQUIRE(a->n_pairs >= 0 && a->max_pair_words >= 0, "resample: bad table n_pairs=%d max_pair_words=%d", a->n_pairs,
                 a->max_pair_words);
    B200_REQUIRE(a->n_pairs == 0 || (a->pairs && a->phases && a->taps), "resample: null table pointer");
    B200_REQUIRE(a->B >= 1 && a->B <= 65535 && a->nw >= 0 && a->nr >= 0, "resample: bad shape B=%d nw=%d nr=%d", a->B, a->nw, a->nr);
    const int blocks = (int)(((long long)a->nr + RS_OUT_PER_BLOCK - 1) / RS_OUT_PER_BLOCK);
    const dim3 grid(blocks > 0 ? blocks : 1, a->B);   // nr = 0: one block still writes out_lens
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = (size_t)a->max_pair_words * 4;
    if (smem <= RS_SMEM_MAX) {
        resample_kernel<true><<<grid, RS_THREADS, smem, st>>>(*a);
        return check_launch("resample_kernel<stage>");
    }
    resample_kernel<false><<<grid, RS_THREADS, 0, st>>>(*a);
    return check_launch("resample_kernel<global>");
}
