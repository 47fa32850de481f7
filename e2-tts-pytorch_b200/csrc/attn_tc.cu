// wgmma / TMA flash attention for the softclamped, key-masked, head-gated attention of the E2-TTS multistream block
// (x-transformers Attend as configured by the reference: SURVEY A.4 steps 4-5) — forward and backward, sm_90a.
//
// Forward: one CTA per (128-query tile, head, batch) on 64-key tiles, 384 threads:
//   warpgroup 0, one thread : TMA producer — Q once, then K_j / V_j tiles (64 keys x 64) into a 3-stage smem ring
//   warpgroups 1, 2         : 64 query rows each — S_j = Q K_j^T (wgmma m64n64k16 x4, both operands K-major from smem) into
//                             registers; softclamp (tanh) + exp2 + mask + dropout on the fragments; O += P_j V_j with P_j as the
//                             REGISTER A operand (wgmma m64n64k16, B = V MN-major) — P never touches shared memory.
//                             The softclamp bounds the logits to [-clamp, clamp], so exp() needs no running maximum: O accumulates
//                             over all key tiles and is normalised once by the row sum.
// mbarrier pipelines: q_full, kv_full/kv_empty[3].
//
// Unclamped mode (UNCLAMPED = true; x-transformers Attention without softclamp_logits): the same pipeline and fragment layout with an
// online softmax. Per key tile, masked keys go to -inf, the row maximum m is reduced over the quad, O and the row sum are rescaled by
// 2^((m_old - m_new) scale log2 e) and P = 2^(s scale log2 e - m_new scale log2 e); LSE = m scale + ln(l). The backward recomputes
// P from that LSE with no tanh factor. A row whose keys are all masked gives o = og = 0, lse = -inf and zero gradients, as the clamped
// kernels do.
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int TQ = 128, TKV = 128;
constexpr int TILE16 = 128 * 64 * 2;          // 16 KB: 128 rows x 64 bf16
constexpr int TILE8 = 64 * 64 * 2;            // 8 KB: 64 rows x 64 bf16
// A head row of DH bf16 is DH / 64 128-byte swizzle atoms: every Q / K / V / dO tile is stored as DH / 64 column blocks of 64
// (one TMA box each), and a K-major operand steps to the next block every 4 k-steps.
constexpr float LOG2E_F = 1.4426950408889634f;

struct AttnTcP {
    const unsigned int* maskbits;   // [B, words] key-validity bitmask (bit set = keep), words = ceil(Np / 32) padded to a multiple of 4
    int mask_words;
    const float* gate;              // [B*Np, H] or null
    __nv_bfloat16 *o, *og;
    float* lse;
    int B, H, Np, nkv;
    float scale_over_clamp, clamp, dropout_p, keep_scale;
    unsigned int drop_thresh;       // keep iff 16-bit hash >= thresh
    int drop_stride;                // even row pitch of the dropout counter space
    unsigned long long seed;
    const unsigned long long* seed_dev;   // optional device addend of the seed (CUDA-graph replays)
    float scale, scale_log2e;       // unclamped mode: the score scale, and scale * log2(e)
};

__device__ __forceinline__ float tanh_approx(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// tanh of a pair on the FMA pipe: odd degree-9 Taylor polynomial, |error| < 5e-6 for |x| <= 0.5 (tanh.approx is ~5e-4). The clamp
// argument score * scale / clamp is small in practice, so the callers take this path whenever a warp's whole tile fits the range and
// keep MUFU.TANH for outliers: with two MUFU operations per score the softmax math is otherwise bound by the MUFU pipe.
constexpr float TANH_POLY_MAX = 0.5f;
__device__ __forceinline__ float2 tanh_poly2(float2 x) {
    const float2 x2 = fmul2(x, x);
    float2 q = ffma2(x2, make_float2(62.f / 2835.f, 62.f / 2835.f), make_float2(-17.f / 315.f, -17.f / 315.f));
    q = ffma2(q, x2, make_float2(2.f / 15.f, 2.f / 15.f));
    q = ffma2(q, x2, make_float2(-1.f / 3.f, -1.f / 3.f));
    q = ffma2(q, x2, make_float2(1.f, 1.f));
    return fmul2(x, q);
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// key-validity bitmask: bit (n % 32) of word n / 32 is set iff key n participates (n < Np and mask[b, n] != 0)
__global__ void attn_maskbits_kernel(const unsigned char* mask, unsigned int* bits, int B, int Np, int words) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= B * words) return;
    const int b = w / words, w0 = (w % words) * 32;
    unsigned int v = 0;
    for (int i = 0; i < 32; ++i) {
        const int n = w0 + i;
        if (n < Np && (!mask || mask[(size_t)b * Np + n])) v |= 1u << i;
    }
    bits[w] = v;
}

// ------------------------------------------------------------------------------------------------ forward
constexpr int KV_STAGES = 3;

template <bool UNCLAMPED, int DH>
__global__ void __launch_bounds__(384, 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const AttnTcP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr int NA = DH / 64;                 // column blocks (swizzle atoms) per head row
    uint8_t* sQ = smem;                         // [NA] x 16 KB
    uint8_t* sK = sQ + NA * TILE16;             // [3][NA] x 8 KB
    uint8_t* sV = sK + KV_STAGES * NA * TILE8;  // [3][NA] x 8 KB
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * NA * TILE8);
    uint64_t* q_full = bars;                    // 1
    uint64_t* kv_full = bars + 1;               // 3
    uint64_t* kv_empty = bars + 4;              // 3 (one arrival per consumer warpgroup)

    const int wg = threadIdx.x >> 7;
    const int qt = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const int bh = b * p.H + hh;
    const int q0 = qt * TQ;
    const int nkv = (p.Np + 63) / 64;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // ---------------------------------------------------------------- TMA producer
            const int row_base = bh * p.Np;
            mbar_arrive_expect_tx(q_full, NA * TILE16);
#pragma unroll
            for (int a = 0; a < NA; ++a) tma_load_2d(sQ + a * TILE16, &tmQ, q_full, 64 * a, row_base + q0);
            int st = 0;
            uint32_t ph = 0;
            for (int j = 0; j < nkv; ++j) {
                mbar_wait(&kv_empty[st], ph ^ 1);
                mbar_arrive_expect_tx(&kv_full[st], 2 * NA * TILE8);
#pragma unroll
                for (int a = 0; a < NA; ++a) {
                    tma_load_2d(sK + (st * NA + a) * TILE8, &tmK, &kv_full[st], 64 * a, row_base + j * 64);
                    tma_load_2d(sV + (st * NA + a) * TILE8, &tmV, &kv_full[st], 64 * a, row_base + j * 64);
                }
                if (++st == KV_STAGES) { st = 0; ph ^= 1; }
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumer warpgroups: 64 query rows each
    regs_alloc<232>();
    const int cw = wg - 1, t = threadIdx.x & 127, lane = t & 31, wq = t >> 5;
    const int cq = 2 * (lane & 3);
    // fragment rows of this thread: r0 and r0 + 8 of the warpgroup's 64; columns 8 j + cq + {0, 1}
    const int r0 = cw * 64 + wq * 16 + (lane >> 2);
    const unsigned int* mb = p.maskbits + (size_t)b * p.mask_words;
    const uint32_t seedmix = drop_seed_word(p.seed, p.seed_dev);
    unsigned long long drop_row[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) drop_row[i] = ((unsigned long long)bh * p.Np + (unsigned long long)(q0 + r0 + 8 * i)) * (unsigned long long)p.drop_stride;
    const float2 soc2 = make_float2(p.scale_over_clamp, p.scale_over_clamp);
    const float2 cl2 = make_float2(p.clamp * LOG2E_F, p.clamp * LOG2E_F);
    const float soc = p.scale_over_clamp, soc2s = soc * soc;
    const float k1 = soc * p.clamp * LOG2E_F, k3 = k1 * soc2s * (-1.f / 3.f), k5 = k1 * soc2s * soc2s * (2.f / 15.f),
                k7 = k1 * soc2s * soc2s * soc2s * (-17.f / 315.f), k9 = k1 * soc2s * soc2s * soc2s * soc2s * (62.f / 2835.f);
    const float lim5 = 0.15f / fabsf(soc), lim9 = TANH_POLY_MAX / fabsf(soc);
    const uint32_t thr32 = drop_thresh32(p.drop_thresh);
    float l[2] = {0.f, 0.f};
    float m[2] = {-INFINITY, -INFINITY};   // unclamped mode: running row maximum of the raw scores
    float o[NA][32];   // O columns 64 a + 8 j + cq + {0, 1}
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[a][i] = 0.f;

    mbar_wait(q_full, 0);
    const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ + cw * TILE8), 16, 1024);
    int st = 0;
    uint32_t ph = 0;
    for (int j = 0; j < nkv; ++j) {
        mbar_wait(&kv_full[st], ph);
        float s[32];
        fence_regs(s);
        wgmma_fence();
        const uint64_t kdesc = make_smem_desc_sw128(smem_u32(sK + st * NA * TILE8), 16, 1024);
#pragma unroll
        for (int k = 0; k < DH / 16; ++k)
            wgmma_ss_n64<0, 0>(s, qdesc + (uint64_t)((k >> 2) * (TILE16 >> 4) + (k & 3) * 2), kdesc + (uint64_t)((k >> 2) * (TILE8 >> 4) + (k & 3) * 2),
                               k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        if constexpr (UNCLAMPED) {
            const unsigned int mw0 = mb[2 * j], mw1 = mb[2 * j + 1];
            if ((mw0 & mw1) != 0xffffffffu) {
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                    const unsigned int w = g < 4 ? mw0 : mw1;
                    const int bit = (8 * g + cq) & 31;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        if (!((w >> bit) & 1u)) s[4 * g + 2 * i] = -INFINITY;
                        if (!((w >> (bit + 1)) & 1u)) s[4 * g + 2 * i + 1] = -INFINITY;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float tm = m[i];
#pragma unroll
                for (int g = 0; g < 8; ++g) tm = fmaxf(tm, fmaxf(s[4 * g + 2 * i], s[4 * g + 2 * i + 1]));
                tm = fmaxf(tm, __shfl_xor_sync(0xffffffffu, tm, 1));
                tm = fmaxf(tm, __shfl_xor_sync(0xffffffffu, tm, 2));
                // every key this row has seen so far is masked: subtract 0 instead of -inf, so that P and the rescale factor are 0
                const float mt = tm == -INFINITY ? 0.f : tm;
                const float alpha = ex2_approx((m[i] - mt) * p.scale_log2e);
                const float nm = -mt * p.scale_log2e;
                m[i] = tm;
                float ls = 0.f;
#pragma unroll
                for (int g = 0; g < 8; ++g) {
#pragma unroll
                    for (int a = 0; a < NA; ++a) {
                        o[a][4 * g + 2 * i] *= alpha;
                        o[a][4 * g + 2 * i + 1] *= alpha;
                    }
                    s[4 * g + 2 * i] = ex2_approx(__fmaf_rn(s[4 * g + 2 * i], p.scale_log2e, nm));
                    s[4 * g + 2 * i + 1] = ex2_approx(__fmaf_rn(s[4 * g + 2 * i + 1], p.scale_log2e, nm));
                    ls += s[4 * g + 2 * i] + s[4 * g + 2 * i + 1];
                }
                l[i] = __fmaf_rn(l[i], alpha, ls);
            }
        } else {
            float amax = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) amax = fmaxf(amax, fabsf(s[i]));
            // clamp * log2(e) * tanh(u), u = s * scale / clamp, evaluated as an odd polynomial in the RAW score s with the constants folded
            // in: s * (k1 + s^2 (k3 + s^2 (k5 + ...))) — degree 5 for |u| <= 0.15 (exact to 1e-7), degree 9 for |u| <= 0.5; tanh.approx
            // only when a warp's tile leaves that range
            if (__all_sync(0xffffffffu, amax <= lim5)) {
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const float2 x = make_float2(s[i], s[i + 1]);
                    const float2 x2 = fmul2(x, x);
                    float2 q = ffma2(x2, make_float2(k5, k5), make_float2(k3, k3));
                    q = ffma2(q, x2, make_float2(k1, k1));
                    const float2 y = fmul2(x, q);
                    s[i] = ex2_approx(y.x);
                    s[i + 1] = ex2_approx(y.y);
                }
            } else if (__all_sync(0xffffffffu, amax <= lim9)) {
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const float2 x = make_float2(s[i], s[i + 1]);
                    const float2 x2 = fmul2(x, x);
                    float2 q = ffma2(x2, make_float2(k9, k9), make_float2(k7, k7));
                    q = ffma2(q, x2, make_float2(k5, k5));
                    q = ffma2(q, x2, make_float2(k3, k3));
                    q = ffma2(q, x2, make_float2(k1, k1));
                    const float2 y = fmul2(x, q);
                    s[i] = ex2_approx(y.x);
                    s[i + 1] = ex2_approx(y.y);
                }
            } else {   // mixed tile: the polynomial wherever it is in range, tanh.approx only for the outliers themselves
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const float x = s[i], x2 = x * x;
                    const float yp = x * __fmaf_rn(__fmaf_rn(__fmaf_rn(__fmaf_rn(k9, x2, k7), x2, k5), x2, k3), x2, k1);
                    const float y = fabsf(x) <= lim9 ? yp : tanh_approx(x * soc) * cl2.x;
                    s[i] = ex2_approx(y);
                }
            }
            const unsigned int mw0 = mb[2 * j], mw1 = mb[2 * j + 1];   // keys 64 j .. 64 j + 31, 64 j + 32 .. 64 j + 63
            if ((mw0 & mw1) != 0xffffffffu) {
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                    const unsigned int w = g < 4 ? mw0 : mw1;
                    const int bit = (8 * g + cq) & 31;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        if (!((w >> bit) & 1u)) s[4 * g + 2 * i] = 0.f;
                        if (!((w >> (bit + 1)) & 1u)) s[4 * g + 2 * i + 1] = 0.f;
                    }
                }
            }
#pragma unroll
            for (int g = 0; g < 8; ++g)
#pragma unroll
                for (int i = 0; i < 2; ++i) l[i] += s[4 * g + 2 * i] + s[4 * g + 2 * i + 1];
        }
        if (p.dropout_p > 0.f) {   // the 1/(1-p) factor is applied once, to the normalised output
#pragma unroll
            for (int g = 0; g < 8; ++g)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const DropWords h = drop_words(seedmix, (uint32_t)((drop_row[i] + (unsigned long long)(j * 64 + 8 * g + cq)) >> 1));
                    s[4 * g + 2 * i] = (h.a >= thr32) ? s[4 * g + 2 * i] : 0.f;
                    s[4 * g + 2 * i + 1] = (h.b >= thr32) ? s[4 * g + 2 * i + 1] : 0.f;
                }
        }
        // O += P V: the accumulator fragment of S is, 16 keys at a time, the register A fragment of the next MMA
#pragma unroll
        for (int a = 0; a < NA; ++a) fence_regs(o[a]);
        wgmma_fence();
        const uint64_t vdesc = make_smem_desc_sw128(smem_u32(sV + st * NA * TILE8), 64 * 128, 1024);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t a[4] = {pack_bf16(s[8 * kk], s[8 * kk + 1]), pack_bf16(s[8 * kk + 2], s[8 * kk + 3]),
                                   pack_bf16(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
            for (int na = 0; na < NA; ++na) wgmma_rs_n64<1>(o[na], a, vdesc + (uint64_t)(na * (TILE8 >> 4) + kk * 128), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int a = 0; a < NA; ++a) fence_regs(o[a]);
        if (t == 0) mbar_arrive(&kv_empty[st]);
        if (++st == KV_STAGES) { st = 0; ph ^= 1; }
    }
    // ---- epilogue: row sums over the quad, normalise, write O (ungated), Og (gated, head-merged) and LSE
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float lt = l[i];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const int qi = q0 + r0 + 8 * i;
        if (qi >= p.Np) continue;
        const float inv = lt > 0.f ? p.keep_scale / lt : 0.f;
        const float gt = p.gate ? p.gate[((size_t)b * p.Np + qi) * p.H + hh] : 1.f;
        __nv_bfloat16* orow = p.o + ((size_t)bh * p.Np + qi) * DH;
        __nv_bfloat16* grow = p.og + ((size_t)b * p.Np + qi) * (size_t)(p.H * DH) + hh * DH;
#pragma unroll
        for (int a = 0; a < NA; ++a)
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const uint32_t u = pack_bf16(o[a][4 * g + 2 * i] * inv, o[a][4 * g + 2 * i + 1] * inv);
                *reinterpret_cast<uint32_t*>(orow + 64 * a + 8 * g + cq) = u;
                // gate the bf16-rounded output (what the backward pass sees) for consistency
                *reinterpret_cast<uint32_t*>(grow + 64 * a + 8 * g + cq) = pack_bf16(bf16_lo(u) * gt, bf16_hi(u) * gt);
            }
        if ((lane & 3) == 0) {
            if constexpr (UNCLAMPED) p.lse[(size_t)bh * p.Np + qi] = __fmaf_rn(m[i], p.scale, logf(lt));
            else p.lse[(size_t)bh * p.Np + qi] = logf(lt);
        }
    }
}

// ================================================================================================ backward
// One CTA per (128-key tile, head, batch), 256 threads:
//   thread 0 also issues the TMA loads — K, V once; Q_i / dO_i tiles (64 queries) through a 3-stage ring, two tiles ahead
//   warpgroups 0, 1         : 64 keys each, per query tile i (all operands from smem, accumulators in registers):
//                             S^T = K Q_i^T, dP^T = V dO_i^T                 (wgmma m64n64k16, K-major operands)
//                             recompute softclamp + softmax from the saved LSE, dS^T = P^T (dP^T - delta)(1 - tanh^2) scale
//                             (unclamped mode: no tanh, dS^T = P^T (dP^T - delta) scale)
//                             dV += P^T dO_i, dK += dS^T Q_i                 (register A operands, B MN-major)
//                             and dS^T into a swizzled smem tile, double-buffered by the parity of the query tile.
// dQ is reduced once per CTA and query tile: after a named barrier, the warpgroup whose index equals the tile's parity computes
// dQ_i = dS_i K over all 128 keys from both dS^T tiles (A MN-major, 8 k-steps), stages the fp32 result in a swizzled smem tile and
// adds it into dq with one TMA tensor reduction (a [B*H, Np, 64] map, so rows >= Np are clipped and the next head is never touched).
// Barrier hand-offs per dS^T buffer b: DS_FULL (the other warpgroup arrives once its tile is written, the reducing one waits) and
// DS_FREE (the reducing warpgroup arrives once its dQ MMAs have read the buffer, the other one waits before it rewrites it two tiles on).
// The lse / delta of query tile i + 1 are loaded during tile i into smem, so no global load sits between the MMA wait and the score math.
struct AttnBwdTcP {
    const unsigned int* maskbits; int mask_words;
    const float *lse, *delta;
    __nv_bfloat16 *dk, *dv;
    int B, H, Np, nq;
    float scale, scale_over_clamp, clamp, dropout_p, keep_scale;
    unsigned int drop_thresh; int drop_stride;
    unsigned long long seed;
    const unsigned long long* seed_dev;   // optional device addend of the seed (CUDA-graph replays)
    float scale_log2e;              // unclamped mode: scale * log2(e)
};
constexpr int QDO_STAGES = 3, TQB = 64;
// named barriers of the backward consumers (ids 1, 2: per warpgroup)
constexpr int BAR_DS_FULL = 3, BAR_DS_FREE = 5;   // + dS^T buffer

// Backward prep, one DH / 8-lane group per (b, h, n): dO = dOg * gate, d_gate = <dOg, O>, delta = gate * d_gate = <dO, O>
struct AttnPrepP {
    const float* gate;              // [B*Np, H] or null
    const __nv_bfloat16* o;
    int B, H, Np;
    const __nv_bfloat16* dog;
    float* dgate;                   // or null
    __nv_bfloat16* dO_out;
    float* delta_out;
};
template <int DH>
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const AttnPrepP p) {
    constexpr int LANES = DH / 8, LOG2_LANES = DH == 64 ? 3 : 4;
    static_assert(LANES == 1 << LOG2_LANES, "head dim 64 or 128");
    const long long gidx = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long rowid = gidx >> LOG2_LANES;
    const int c = (int)(gidx & (LANES - 1));
    const long long total = (long long)p.B * p.H * p.Np;
    const bool ok = rowid < total;
    float dot = 0.f, gt = 1.f;
    long long b = 0, hh = 0, n = 0;
    if (ok) {
        n = rowid % p.Np; hh = (rowid / p.Np) % p.H; b = rowid / ((long long)p.Np * p.H);
        const uint4 dg = *reinterpret_cast<const uint4*>(p.dog + ((size_t)b * p.Np + n) * (size_t)(p.H * DH) + hh * DH + c * 8);
        const uint4 ov = *reinterpret_cast<const uint4*>(p.o + (size_t)rowid * DH + c * 8);
        gt = p.gate ? p.gate[((size_t)b * p.Np + n) * p.H + hh] : 1.f;
        const uint32_t dgv[4] = {dg.x, dg.y, dg.z, dg.w}, ovv[4] = {ov.x, ov.y, ov.z, ov.w};
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float a0 = bf16_lo(dgv[i]), a1 = bf16_hi(dgv[i]);
            dot += a0 * bf16_lo(ovv[i]) + a1 * bf16_hi(ovv[i]);
            w[i] = pack_bf16(a0 * gt, a1 * gt);
        }
        *reinterpret_cast<uint4*>(p.dO_out + (size_t)rowid * DH + c * 8) = make_uint4(w[0], w[1], w[2], w[3]);
    }
#pragma unroll
    for (int m = 1; m < LANES; m <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, m);
    if (ok && c == 0) {
        p.delta_out[rowid] = dot * gt;
        if (p.dgate) p.dgate[((size_t)b * p.Np + n) * p.H + hh] = dot;
    }
}

// P^T / dS^T of one query tile from the S^T / dP^T fragments (rows = keys kr, kr + 8; columns = queries qt0 + 8 g + cq + {0, 1}),
// for the column groups g = G0 .. G0 + NG - 1 (the head-dim-128 kernel splits the eight between its two warpgroups).
// UNCLAMPED: P = 2^(s scale log2 e - lse log2 e), dS = P (dP - delta) scale (POLY is then unused).
// sld: the tile's -lse log2 e (64 floats) then delta (64 floats), zero for queries >= Np.
// Dropout: the thread's keys kr, kr + 8 have the parity of lane >> 2, so lanes L and L ^ 4 hold the two keys of every hash pair at the
// same query columns. Each lane hashes one of its two columns (pair index drop_pair + 8 g half_stride + 4 i: the even-stride counter
// (bh Np + q) stride + key, halved, in 32 bits) and the word its partner needs crosses with one shuffle.
template <bool UNCLAMPED, bool POLY, bool DROP, int G0 = 0, int NG = 8>
__device__ __forceinline__ void bwd_score_math(const AttnBwdTcP& p, const float (&s)[32], const float (&dp)[32], const float* sld, int qt0, int cq,
                                               const bool (&kok)[2], bool kodd, uint32_t drop_pair, uint32_t seedmix,
                                               uint32_t (&ppk)[16], uint32_t (&dpk)[16]) {
    const uint32_t thr32 = drop_thresh32(p.drop_thresh);
    const uint32_t pair_g = 8u * ((uint32_t)p.drop_stride >> 1);
    const float clog = p.clamp * LOG2E_F;
#pragma unroll
    for (int g = G0; g < G0 + NG; ++g) {
        const float2 nl2 = *reinterpret_cast<const float2*>(sld + 8 * g + cq);
        const float2 dl2 = *reinterpret_cast<const float2*>(sld + 64 + 8 * g + cq);
        bool keepw[2][2];   // [key i][query column c]
        if constexpr (DROP) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const DropWords h = drop_words(seedmix, drop_pair + (uint32_t)g * pair_g + 4u * i);
                const uint32_t other = __shfl_xor_sync(0xffffffffu, kodd ? h.a : h.b, 4);
                const bool own = (kodd ? h.b : h.a) >= thr32, oth = other >= thr32;
                keepw[i][0] = kodd ? oth : own;
                keepw[i][1] = kodd ? own : oth;
            }
        }
        float pe[2][2], dsv[2][2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int qi = qt0 + 8 * g + cq + c;
            const bool qok = qi < p.Np;
            const float nlse2 = c ? nl2.y : nl2.x;
            const float dl = c ? dl2.y : dl2.x;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int e = 4 * g + 2 * i + c;
                float pv, dsc;
                if constexpr (UNCLAMPED) {
                    pv = ex2_approx(__fmaf_rn(s[e], p.scale_log2e, nlse2));
                    pv = (qok && kok[i]) ? pv : 0.f;
                    dsc = p.scale;
                } else {
                    const float x = s[e] * p.scale_over_clamp;
                    float th;
                    if constexpr (POLY) th = tanh_poly2(make_float2(x, 0.f)).x;
                    else th = fabsf(x) <= TANH_POLY_MAX ? tanh_poly2(make_float2(x, 0.f)).x : tanh_approx(x);   // outliers only
                    pv = ex2_approx(__fmaf_rn(th, clog, nlse2));
                    pv = (qok && kok[i]) ? pv : 0.f;
                    dsc = __fmaf_rn(th * -p.scale, th, p.scale);   // (1 - tanh^2) * scale = d(clamped logit)/d(raw score)
                }
                float tt, pd;
                if constexpr (DROP) {
                    const bool keep = keepw[i][c];
                    tt = __fmaf_rn(keep ? dp[e] : 0.f, p.keep_scale, -dl);
                    pd = keep ? pv : 0.f;   // dV uses the dropped probabilities, dS the un-dropped ones
                } else {
                    tt = dp[e] - dl;
                    pd = pv;
                }
                pe[i][c] = pd;
                dsv[i][c] = (pv * tt) * dsc;
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            ppk[2 * g + i] = pack_bf16(pe[i][0], pe[i][1]);
            dpk[2 * g + i] = pack_bf16(dsv[i][0], dsv[i][1]);
        }
    }
}

template <bool UNCLAMPED>
// Head dim 64. 256 threads and no register hand-over: with a third (producer) warpgroup, ptxas allocates every thread against 168 registers
// (3 warps per SM sub-partition) whatever setmaxnreg grants the consumers, and the consumer live set (S, dP, dV, dK fragments and the
// packed P / dS) spills there. One consumer thread issues the TMA loads instead.
__global__ void __launch_bounds__(256, 1)
attn_bwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmDQ, const AttnBwdTcP p) {
    constexpr int DH = 64;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sK = smem;                          // 16 KB (128 keys)
    uint8_t* sV = sK + TILE16;                   // 16 KB
    uint8_t* sQ = sV + TILE16;                   // [3] x 8 KB (64 queries)
    uint8_t* sDO = sQ + QDO_STAGES * TILE8;      // [3] x 8 KB
    uint8_t* sDS = sDO + QDO_STAGES * TILE8;     // [2 buffers][2 warpgroups] x 8 KB: dS^T (64 keys x 64 queries), 128B-swizzled
    uint8_t* sDQ = sDS + 4 * TILE8;              // [2 warpgroups] x 16 KB: fp32 dQ staging, two 64 x 32 halves, 128B-swizzled
    float* sLD = reinterpret_cast<float*>(sDQ + 2 * TILE16);   // [2 warpgroups][2 slots][-lse log2 e x 64 | delta x 64]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sLD + 2 * 2 * 128);
    uint64_t* kv_full = bars;                    // 1
    uint64_t* qdo_full = bars + 1;               // 3
    uint64_t* qdo_empty = bars + 4;              // 3 (one arrival per consumer warpgroup)

    const int wg = threadIdx.x >> 7;
    const int kt = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const int bh = b * p.H + hh;
    const int k0 = kt * TKV;
    const int nq = p.nq;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO); tma_prefetch_desc(&tmDQ);
        mbar_init(kv_full, 1);
        for (int i = 0; i < QDO_STAGES; ++i) { mbar_init(&qdo_full[i], 1); mbar_init(&qdo_empty[i], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    // TMA producer (thread 0): K, V once; query tile j into ring stage j % 3 once the tile j - 3 that used it has been released by
    // both warpgroups. Tiles 0 and 1 go out here, tile it + 2 at the top of iteration it.
    const int row_base = bh * p.Np;
    auto load_qdo = [&](int j) {
        const int s_j = j % QDO_STAGES;
        if (j >= QDO_STAGES) mbar_wait(&qdo_empty[s_j], (uint32_t)((j / QDO_STAGES) & 1) ^ 1u);
        mbar_arrive_expect_tx(&qdo_full[s_j], 2 * TILE8);
        const int qt_j = (j + kt) % nq;   // staggered query-tile order: the key-tile CTAs of one head never flush the same dQ rows together
        tma_load_2d(sQ + s_j * TILE8, &tmQ, &qdo_full[s_j], 0, row_base + qt_j * TQB);
        tma_load_2d(sDO + s_j * TILE8, &tmDO, &qdo_full[s_j], 0, row_base + qt_j * TQB);
    };
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(kv_full, 2 * TILE16);
        tma_load_2d(sK, &tmK, kv_full, 0, row_base + k0);
        tma_load_2d(sV, &tmV, kv_full, 0, row_base + k0);
        for (int j = 0; j < 2 && j < nq; ++j) load_qdo(j);
    }

    const int cw = wg, t = threadIdx.x & 127, lane = t & 31, wq = t >> 5;
    const int cq = 2 * (lane & 3);
    const int kr0 = cw * 64 + wq * 16 + (lane >> 2);   // fragment rows (keys) kr0, kr0 + 8 of the CTA's 128
    int key[2];
    bool kok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        key[i] = k0 + kr0 + 8 * i;
        kok[i] = key[i] < p.Np && ((p.maskbits[(size_t)b * p.mask_words + (key[i] >> 5)] >> (key[i] & 31)) & 1u);
    }
    const uint32_t seedmix = drop_seed_word(p.seed, p.seed_dev);
    const bool kodd = (lane >> 2) & 1;
    const bool active = k0 + cw * 64 < p.Np;   // a warpgroup whose 64 keys all lie at or past Np keeps only the barrier protocol
    const uint64_t kdesc = make_smem_desc_sw128(smem_u32(sK + cw * TILE8), 16, 1024);        // K-major A of S^T
    const uint64_t vdesc = make_smem_desc_sw128(smem_u32(sV + cw * TILE8), 16, 1024);        // K-major A of dP^T
    const uint64_t kmn = make_smem_desc_sw128(smem_u32(sK), 64 * 128, 1024);                 // MN-major B of dQ: all 128 keys
    uint8_t* dq_stage = sDQ + cw * TILE16;
    float* ld_own = sLD + cw * 256;
    // lse / delta of query tile `it` for this thread: threads 0-63 take -lse log2 e, threads 64-127 delta, 0 for queries >= Np
    const int ld_j = t & 63;
    const float* ld_src = (t < 64 ? p.lse : p.delta) + (size_t)bh * p.Np;
    auto ld_tile = [&](int it) {
        const int qi = ((it + kt) % nq) * TQB + ld_j;
        float v = 0.f;
        if (qi < p.Np) {
            v = __ldg(ld_src + qi);
            if (t < 64) v = -v * LOG2E_F;
        }
        return v;
    };
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }

    if (active) {
        ld_own[t] = ld_tile(0);
    } else {
        // dS^T = 0 for keys past Np in both buffers, written once: the dQ MMAs run over all 128 keys and add 0 x K for them
#pragma unroll
        for (int i = 0; i < 2 * TILE8 / 16 / 128; ++i) {
            uint8_t* tile = sDS + (2 * (i & 1) + cw) * TILE8;
            *reinterpret_cast<uint4*>(tile + ((i >> 1) * 128 + t) * 16) = make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();
    }
    named_bar_sync(1 + cw, 128);
    mbar_wait(kv_full, 0);
    int st = 0;
    uint32_t ph = 0;
    for (int it = 0; it < nq; ++it) {
        const int qt0 = ((it + kt) % nq) * TQB;
        const int buf = it & 1;               // dS^T buffer of this tile, and the warpgroup that reduces its dQ
        const bool reducer = cw == buf;
        if (threadIdx.x == 0 && it + 2 < nq) load_qdo(it + 2);
        const float ld_next = (active && it + 1 < nq) ? ld_tile(it + 1) : 0.f;
        mbar_wait(&qdo_full[st], ph);
        uint8_t* ds_tile = sDS + (2 * buf + cw) * TILE8;
        uint32_t ppk[16], dpk[16];   // bf16-packed P_drop^T and dS^T fragments
        if (active) {
            const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ + st * TILE8), 16, 1024);
            const uint64_t dodesc = make_smem_desc_sw128(smem_u32(sDO + st * TILE8), 16, 1024);
            float s[32], dp[32];
            fence_regs(s); fence_regs(dp);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_n64<0, 0>(s, kdesc + (uint64_t)(k * 2), qdesc + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_n64<0, 0>(dp, vdesc + (uint64_t)(k * 2), dodesc + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(s); fence_regs(dp);
            ld_own[(buf ^ 1) * 128 + t] = ld_next;   // read at tile it + 1, after this tile's closing barrier
            const float* sld = ld_own + buf * 128;
            const uint32_t drop_pair = ((uint32_t)bh * (uint32_t)p.Np + (uint32_t)(qt0 + cq + kodd)) * ((uint32_t)p.drop_stride >> 1) +
                                       ((uint32_t)key[0] >> 1);
            const bool drop = p.dropout_p > 0.f;
            if constexpr (UNCLAMPED) {
                if (drop) bwd_score_math<true, false, true>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                else bwd_score_math<true, false, false>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
            } else {
                float amax = 0.f;
#pragma unroll
                for (int e = 0; e < 32; ++e) amax = fmaxf(amax, fabsf(s[e]));
                const bool small = __all_sync(0xffffffffu, amax * fabsf(p.scale_over_clamp) <= TANH_POLY_MAX);   // same rule as the forward
                if (small) {
                    if (drop) bwd_score_math<false, true, true>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                    else bwd_score_math<false, true, false>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                } else {
                    if (drop) bwd_score_math<false, false, true>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                    else bwd_score_math<false, false, false>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                }
            }
        }
        if (!reducer && it >= 2) named_bar_sync(BAR_DS_FREE + buf, 256);   // the dQ MMAs of tile it - 2 have read this buffer
        if (active) {
            // dS^T into the warpgroup's swizzled smem tile (row = key, 64 queries = one 128-byte swizzle atom per row)
#pragma unroll
            for (int g = 0; g < 8; ++g)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int r = wq * 16 + (lane >> 2) + 8 * i;
                    *reinterpret_cast<uint32_t*>(ds_tile + r * 128 + ((g ^ (r & 7)) << 4) + cq * 2) = dpk[2 * g + i];
                }
            fence_proxy_async();
        }
        if (!reducer) named_bar_arrive(BAR_DS_FULL + buf, 256);
        if (active) {
            // dV += P^T dO_i, dK += dS^T Q_i (register A: 16 queries per MMA)
            const uint64_t domn = make_smem_desc_sw128(smem_u32(sDO + st * TILE8), 64 * 128, 1024);
            const uint64_t qmn = make_smem_desc_sw128(smem_u32(sQ + st * TILE8), 64 * 128, 1024);
            fence_regs(dv); fence_regs(dk);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t ap[4] = {ppk[4 * kk], ppk[4 * kk + 1], ppk[4 * kk + 2], ppk[4 * kk + 3]};
                wgmma_rs_n64<1>(dv, ap, domn + (uint64_t)(kk * 128), 1u);
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t ad[4] = {dpk[4 * kk], dpk[4 * kk + 1], dpk[4 * kk + 2], dpk[4 * kk + 3]};
                wgmma_rs_n64<1>(dk, ad, qmn + (uint64_t)(kk * 128), 1u);
            }
            wgmma_commit();
        }
        if (reducer) {
            // dQ_i = dS_i K over the CTA's keys: rows = queries, columns = head dims
            if (t == 0) bulk_wait_group_read<0>();   // the reduction of tile it - 2 has read the staging tile
            named_bar_sync(BAR_DS_FULL + buf, 256);
            const uint64_t dsdesc = make_smem_desc_sw128(smem_u32(sDS + 2 * buf * TILE8), 64 * 128, 1024);   // MN-major A (dS^T stored)
            float dq[32];
            fence_regs(dq);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) wgmma_ss_n64<1, 1>(dq, dsdesc + (uint64_t)(k * 128), kmn + (uint64_t)(k * 128), k > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(dq);
            if (it + 2 < nq) named_bar_arrive(BAR_DS_FREE + buf, 256);
            // stage as two 64 x 32 fp32 boxes in the 128B-swizzled layout of the tensor map (bank-conflict free float2 stores)
#pragma unroll
            for (int g = 0; g < 8; ++g)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int r = wq * 16 + (lane >> 2) + 8 * i;
                    const int chunk = 2 * (g & 3) + (cq >> 2);
                    *reinterpret_cast<float2*>(dq_stage + (g >> 2) * TILE8 + r * 128 + ((chunk ^ (r & 7)) << 4) + (cq & 3) * 4) =
                        make_float2(dq[4 * g + 2 * i], dq[4 * g + 2 * i + 1]);
                }
            fence_proxy_async();
        } else {
            wgmma_wait<0>();
        }
        fence_regs(dv); fence_regs(dk);
        if (t == 0) mbar_arrive(&qdo_empty[st]);
        named_bar_sync(1 + cw, 128);   // dQ staged; this tile's lse / delta slot read, the next one written
        if (reducer && t == 0) {
            tma_reduce_add_3d(&tmDQ, dq_stage, 0, qt0, bh);
            tma_reduce_add_3d(&tmDQ, dq_stage + TILE8, 32, qt0, bh);
            bulk_commit_group();
        }
        if (++st == QDO_STAGES) { st = 0; ph ^= 1; }
    }
    if (t == 0) bulk_wait_group<0>();
    // ---- dV (with the deferred 1/(1-p) of the dropped probabilities), dK: rows = keys
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (key[i] >= p.Np) continue;
        __nv_bfloat16* dvp = p.dv + ((size_t)bh * p.Np + key[i]) * DH;
        __nv_bfloat16* dkp = p.dk + ((size_t)bh * p.Np + key[i]) * DH;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            *reinterpret_cast<uint32_t*>(dvp + 8 * g + cq) = pack_bf16(dv[4 * g + 2 * i] * p.keep_scale, dv[4 * g + 2 * i + 1] * p.keep_scale);
            *reinterpret_cast<uint32_t*>(dkp + 8 * g + cq) = pack_bf16(dk[4 * g + 2 * i], dk[4 * g + 2 * i + 1]);
        }
    }
}

// Head dim 128. Doubling the head-dim-64 kernel does not fit: dK and dV of 64 keys x 128 dims would take 128 accumulator registers
// per thread next to S^T, dP^T and their packed operands (~290 in all), and the tiles ~256 KB of shared memory. So the two
// warpgroups share ONE 64-key tile and split the work instead of the keys — one CTA per (64-key tile, head, batch), 256 threads:
//   warpgroup 0 computes S^T = K Q_i^T, warpgroup 1 dP^T = V dO_i^T (m64n64k16, 8 k-steps over both column blocks of the head);
//   each hands the half of its fragment the other needs through shared memory (fp32, fragment order), so warpgroup 0 does the score
//   math of query columns 0-31 and warpgroup 1 of columns 32-63 (the same fragment positions, so the dropout hash, its lane pairing
//   and the score arithmetic are the head-dim-64 kernel's, element for element);
//   both write their P^T / dS^T columns into swizzled bf16 tiles, and warpgroup w then owns head dims 64 w .. 64 w + 63 of
//   dV += P^T dO_i, dK += dS^T Q_i and dQ_i = dS_i K (all operands from shared memory, 4 k-steps each), 96 accumulator registers.
//   Each warpgroup stages its 64 x 64 fp32 dQ block and adds it into dq with two TMA reductions (a [B*H, Np, 128] map, 32-float
//   boxes): one reduction per key tile, as in the head-dim-64 kernel.
// Per query tile: BAR_X (exchange halves written; also orders the lse / delta slot) and BAR_PDS (P^T / dS^T written, dQ staging free).
// Every warpgroup waits for its own MMAs before it reaches the next tile's BAR_X, so single exchange and P^T / dS^T buffers suffice.
constexpr int BAR_X = 3, BAR_PDS = 4;
// One warpgroup's half of the head-dim-128 score math for one query tile: warpgroup W holds S^T (W = 0) or dP^T (W = 1) in `acc`,
// hands the other warpgroup the fragment elements of its query columns through sX, takes its own from the other's, and writes
// P_drop^T and dS^T of query columns 32 W .. 32 W + 31 (column groups g = 4 W .. 4 W + 3) into the swizzled tiles.
template <bool UNCLAMPED, int W>
__device__ __forceinline__ void d128_score_half(const AttnBwdTcP& p, const float (&acc)[32], float* sX, float* sLD, int slot, float ld_next,
                                                bool last, uint8_t* sP, uint8_t* sDS, int t, int kr0, int qt0, int cq, const bool (&kok)[2],
                                                bool kodd, uint32_t drop_pair, uint32_t seedmix) {
    constexpr int KEEP = 16 * W, GIVE = 16 - KEEP;   // first fragment element this warpgroup scores / hands over
#pragma unroll
    for (int e = 0; e < 16; ++e) sX[(W * 16 + e) * 128 + t] = acc[GIVE + e];
    if (W == 0 && !last) sLD[(slot ^ 1) * 128 + t] = ld_next;   // read at the next tile, after its BAR_X
    named_bar_sync(BAR_X, 256);
    float oth[32];
#pragma unroll
    for (int e = 0; e < 16; ++e) oth[KEEP + e] = sX[((W ^ 1) * 16 + e) * 128 + t];
    const float* sld = sLD + slot * 128;
    const bool drop = p.dropout_p > 0.f;
    uint32_t ppk[16], dpk[16];
    auto score = [&](const float (&s)[32], const float (&dp)[32]) {
        if constexpr (UNCLAMPED) {
            if (drop) bwd_score_math<true, false, true, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
            else bwd_score_math<true, false, false, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
        } else {
            float amax = 0.f;
#pragma unroll
            for (int e = KEEP; e < KEEP + 16; ++e) amax = fmaxf(amax, fabsf(s[e]));
            if (__all_sync(0xffffffffu, amax * fabsf(p.scale_over_clamp) <= TANH_POLY_MAX)) {   // same rule as the forward
                if (drop) bwd_score_math<false, true, true, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                else bwd_score_math<false, true, false, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
            } else {
                if (drop) bwd_score_math<false, false, true, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
                else bwd_score_math<false, false, false, 4 * W, 4>(p, s, dp, sld, qt0, cq, kok, kodd, drop_pair, seedmix, ppk, dpk);
            }
        }
    };
    if constexpr (W == 0) score(acc, oth);
    else score(oth, acc);
#pragma unroll
    for (int g = 4 * W; g < 4 * W + 4; ++g)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = kr0 + 8 * i;
            const int off = r * 128 + ((g ^ (r & 7)) << 4) + cq * 2;
            *reinterpret_cast<uint32_t*>(sP + off) = ppk[2 * g + i];
            *reinterpret_cast<uint32_t*>(sDS + off) = dpk[2 * g + i];
        }
}

template <bool UNCLAMPED>
__global__ void __launch_bounds__(256, 1)
attn_bwd_d128_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                           const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmDQ, const AttnBwdTcP p) {
    constexpr int DH = 128;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sK = smem;                          // [2 column blocks] x 8 KB (64 keys)
    uint8_t* sV = sK + 2 * TILE8;                // [2] x 8 KB
    uint8_t* sQ = sV + 2 * TILE8;                // [3 stages][2] x 8 KB (64 queries)
    uint8_t* sDO = sQ + QDO_STAGES * 2 * TILE8;  // [3][2] x 8 KB
    uint8_t* sP = sDO + QDO_STAGES * 2 * TILE8;  // P_drop^T (64 keys x 64 queries), 128B-swizzled
    uint8_t* sDS = sP + TILE8;                   // dS^T, same layout
    uint8_t* sDQ = sDS + TILE8;                  // [2 warpgroups] x 16 KB: fp32 dQ staging, two 64 x 32 boxes each, 128B-swizzled
    float* sX = reinterpret_cast<float*>(sDQ + 2 * TILE16);   // [2 warpgroups][16 fragment elements][128 threads] fp32
    float* sLD = sX + 2 * 16 * 128;              // [2 slots][-lse log2 e x 64 | delta x 64]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sLD + 2 * 128);
    uint64_t* kv_full = bars;                    // 1
    uint64_t* qdo_full = bars + 1;               // 3
    uint64_t* qdo_empty = bars + 4;              // 3 (one arrival per consumer warpgroup)

    const int wg = threadIdx.x >> 7;
    const int kt = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const int bh = b * p.H + hh;
    const int k0 = kt * 64;
    const int nq = p.nq;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO); tma_prefetch_desc(&tmDQ);
        mbar_init(kv_full, 1);
        for (int i = 0; i < QDO_STAGES; ++i) { mbar_init(&qdo_full[i], 1); mbar_init(&qdo_empty[i], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    const int row_base = bh * p.Np;
    auto load_qdo = [&](int j) {
        const int s_j = j % QDO_STAGES;
        if (j >= QDO_STAGES) mbar_wait(&qdo_empty[s_j], (uint32_t)((j / QDO_STAGES) & 1) ^ 1u);
        mbar_arrive_expect_tx(&qdo_full[s_j], 4 * TILE8);
        const int qt_j = (j + kt) % nq;   // staggered query-tile order, as in the head-dim-64 kernel
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            tma_load_2d(sQ + (2 * s_j + a) * TILE8, &tmQ, &qdo_full[s_j], 64 * a, row_base + qt_j * TQB);
            tma_load_2d(sDO + (2 * s_j + a) * TILE8, &tmDO, &qdo_full[s_j], 64 * a, row_base + qt_j * TQB);
        }
    };
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(kv_full, 4 * TILE8);
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            tma_load_2d(sK + a * TILE8, &tmK, kv_full, 64 * a, row_base + k0);
            tma_load_2d(sV + a * TILE8, &tmV, kv_full, 64 * a, row_base + k0);
        }
        for (int j = 0; j < 2 && j < nq; ++j) load_qdo(j);
    }

    const int cw = wg, t = threadIdx.x & 127, lane = t & 31, wq = t >> 5;
    const int cq = 2 * (lane & 3);
    const int kr0 = wq * 16 + (lane >> 2);   // fragment rows (keys) kr0, kr0 + 8 of the CTA's 64
    int key[2];
    bool kok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        key[i] = k0 + kr0 + 8 * i;
        kok[i] = key[i] < p.Np && ((p.maskbits[(size_t)b * p.mask_words + (key[i] >> 5)] >> (key[i] & 31)) & 1u);
    }
    const uint32_t seedmix = drop_seed_word(p.seed, p.seed_dev);
    const bool kodd = (lane >> 2) & 1;
    // S^T (warpgroup 0): A = K, B = Q_i; dP^T (warpgroup 1): A = V, B = dO_i — both K-major over the 128 head dims
    const uint64_t adesc = make_smem_desc_sw128(smem_u32(cw == 0 ? sK : sV), 16, 1024);
    const uint64_t kmn = make_smem_desc_sw128(smem_u32(sK + cw * TILE8), 64 * 128, 1024);   // MN-major B of dQ: this warpgroup's dims
    const uint64_t pdesc = make_smem_desc_sw128(smem_u32(sP), 16, 1024);                     // K-major A of dV (P^T stored)
    const uint64_t dskm = make_smem_desc_sw128(smem_u32(sDS), 16, 1024);                     // K-major A of dK
    const uint64_t dsmn = make_smem_desc_sw128(smem_u32(sDS), 64 * 128, 1024);               // MN-major A of dQ
    uint8_t* dq_stage = sDQ + cw * TILE16;
    // lse / delta of query tile `it` (warpgroup 0 loads them): threads 0-63 take -lse log2 e, threads 64-127 delta, 0 for queries >= Np
    const int ld_j = t & 63;
    const float* ld_src = (t < 64 ? p.lse : p.delta) + (size_t)bh * p.Np;
    auto ld_tile = [&](int it) {
        const int qi = ((it + kt) % nq) * TQB + ld_j;
        float v = 0.f;
        if (qi < p.Np) {
            v = __ldg(ld_src + qi);
            if (t < 64) v = -v * LOG2E_F;
        }
        return v;
    };
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }

    if (cw == 0) sLD[t] = ld_tile(0);
    __syncthreads();
    mbar_wait(kv_full, 0);
    int st = 0;
    uint32_t ph = 0;
    for (int it = 0; it < nq; ++it) {
        const int qt0 = ((it + kt) % nq) * TQB;
        const int slot = it & 1;
        if (threadIdx.x == 0 && it + 2 < nq) load_qdo(it + 2);
        const float ld_next = (cw == 0 && it + 1 < nq) ? ld_tile(it + 1) : 0.f;
        mbar_wait(&qdo_full[st], ph);
        float acc[32];   // warpgroup 0: S^T, warpgroup 1: dP^T
        {
            const uint64_t bdesc = make_smem_desc_sw128(smem_u32((cw == 0 ? sQ : sDO) + 2 * st * TILE8), 16, 1024);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < DH / 16; ++k) {
                const uint64_t off = (uint64_t)((k >> 2) * (TILE8 >> 4) + (k & 3) * 2);
                wgmma_ss_n64<0, 0>(acc, adesc + off, bdesc + off, k > 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(acc);
        }
        const uint32_t drop_pair = ((uint32_t)bh * (uint32_t)p.Np + (uint32_t)(qt0 + cq + kodd)) * ((uint32_t)p.drop_stride >> 1) +
                                   ((uint32_t)key[0] >> 1);
        const bool last = it + 1 >= nq;
        if (cw == 0) d128_score_half<UNCLAMPED, 0>(p, acc, sX, sLD, slot, ld_next, last, sP, sDS, t, kr0, qt0, cq, kok, kodd, drop_pair, seedmix);
        else d128_score_half<UNCLAMPED, 1>(p, acc, sX, sLD, slot, ld_next, last, sP, sDS, t, kr0, qt0, cq, kok, kodd, drop_pair, seedmix);
        fence_proxy_async();
        if (t == 0) bulk_wait_group_read<0>();   // the reduction of the previous tile has read this warpgroup's dQ staging
        named_bar_sync(BAR_PDS, 256);
        // dV += P^T dO_i, dK += dS^T Q_i, dQ_i = dS_i K, each on this warpgroup's 64 head dims (column block cw)
        float dq[32];
        {
            const uint64_t domn = make_smem_desc_sw128(smem_u32(sDO + (2 * st + cw) * TILE8), 64 * 128, 1024);
            const uint64_t qmn = make_smem_desc_sw128(smem_u32(sQ + (2 * st + cw) * TILE8), 64 * 128, 1024);
            fence_regs(dv); fence_regs(dk); fence_regs(dq);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_n64<0, 1>(dv, pdesc + (uint64_t)(k * 2), domn + (uint64_t)(k * 128), 1u);
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_n64<0, 1>(dk, dskm + (uint64_t)(k * 2), qmn + (uint64_t)(k * 128), 1u);
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_n64<1, 1>(dq, dsmn + (uint64_t)(k * 128), kmn + (uint64_t)(k * 128), k > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(dv); fence_regs(dk); fence_regs(dq);
        }
        if (t == 0) mbar_arrive(&qdo_empty[st]);
        // stage as two 64 x 32 fp32 boxes in the 128B-swizzled layout of the tensor map (rows = queries)
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = kr0 + 8 * i;
                const int chunk = 2 * (g & 3) + (cq >> 2);
                *reinterpret_cast<float2*>(dq_stage + (g >> 2) * TILE8 + r * 128 + ((chunk ^ (r & 7)) << 4) + (cq & 3) * 4) =
                    make_float2(dq[4 * g + 2 * i], dq[4 * g + 2 * i + 1]);
            }
        fence_proxy_async();
        named_bar_sync(1 + cw, 128);
        if (t == 0) {
            tma_reduce_add_3d(&tmDQ, dq_stage, 64 * cw, qt0, bh);
            tma_reduce_add_3d(&tmDQ, dq_stage + TILE8, 64 * cw + 32, qt0, bh);
            bulk_commit_group();
        }
        if (++st == QDO_STAGES) { st = 0; ph ^= 1; }
    }
    if (t == 0) bulk_wait_group<0>();
    // ---- dV (with the deferred 1/(1-p) of the dropped probabilities), dK: rows = keys, columns 64 cw + 8 g + cq + {0, 1}
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (key[i] >= p.Np) continue;
        __nv_bfloat16* dvp = p.dv + ((size_t)bh * p.Np + key[i]) * DH + 64 * cw;
        __nv_bfloat16* dkp = p.dk + ((size_t)bh * p.Np + key[i]) * DH + 64 * cw;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            *reinterpret_cast<uint32_t*>(dvp + 8 * g + cq) = pack_bf16(dv[4 * g + 2 * i] * p.keep_scale, dv[4 * g + 2 * i + 1] * p.keep_scale);
            *reinterpret_cast<uint32_t*>(dkp + 8 * g + cq) = pack_bf16(dk[4 * g + 2 * i], dk[4 * g + 2 * i + 1]);
        }
    }
}

// ---------------------------------------------------------------------------------------------- host
typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                     const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled2 tensor_map_encoder() {
    static PFN_encodeTiled2 enc = nullptr;
    if (!enc) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            enc = reinterpret_cast<PFN_encodeTiled2>(fn);
    }
    return enc;
}

// bf16 [rows, dh] with boxes of 64 columns (one 128-byte swizzle atom) x box_rows rows
static int make_head_map(CUtensorMap* m, const void* ptr, long long rows, int dh, int box_rows) {
    const PFN_encodeTiled2 enc = tensor_map_encoder();
    B200_REQUIRE(enc, "cuTensorMapEncodeTiled entry point not available");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "attention: operand not 16-byte aligned");
    cuuint64_t gdim[2] = {(cuuint64_t)dh, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)dh * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

// fp32 dq [B*H, Np, dh] as a 3-D map with 64 x 32 boxes (128-byte rows, 128B swizzle; dh / 32 boxes per row): a box at rows >= Np
// is clipped by the hardware instead of running into the next head
static int make_dq_map(CUtensorMap* m, float* dq, int BH, int Np, int dh) {
    const PFN_encodeTiled2 enc = tensor_map_encoder();
    B200_REQUIRE(enc, "cuTensorMapEncodeTiled entry point not available");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(dq) & 15) == 0, "attn_bwd: dq not 16-byte aligned");
    cuuint64_t gdim[3] = {(cuuint64_t)dh, (cuuint64_t)Np, (cuuint64_t)BH};
    cuuint64_t gstride[2] = {dh * sizeof(float), (cuuint64_t)Np * dh * sizeof(float)};
    cuuint32_t box[3] = {32, TQB, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, dq, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (dq) failed (%d)", (int)r);
    return 0;
}

// The argument rules and parameter fields b200_attn_fwd and b200_attn_bwd share (their argument and parameter structs name them
// alike): dim_head, shape, logit clamp, dropout; then the key-validity bitmask, unless the caller has built it. `who` prefixes
// every refusal.
template <class Args, class P>
static int attn_setup(const Args* a, P& p, const char* who, cudaStream_t st) {
    B200_REQUIRE(a->dim_head == 64 || a->dim_head == 128, "%s: dim_head must be 64 or 128 (got %d)", who, a->dim_head);
    B200_REQUIRE(a->B > 0 && a->H > 0 && a->Np > 0 && a->B <= 65535 && a->H <= 65535, "%s: bad shape", who);
    if (a->unclamped) {
        B200_REQUIRE(a->softclamp == 0.f, "%s: unclamped attention needs softclamp == 0 (got %g)", who, a->softclamp);
    } else {
        B200_REQUIRE(a->softclamp > 0.f, "%s: softclamp value must be > 0, or set unclamped for attention without the logit soft-clamp", who);
    }
    B200_REQUIRE(a->dropout_p >= 0.f && a->dropout_p < 1.f, "%s: dropout must be in [0,1)", who);
    B200_REQUIRE(a->softclamp <= 64.f, "%s: softclamp %g > 64: the clamped wgmma kernel exponentiates the clamped logits without a "
                 "running maximum, which needs exp(+-softclamp) well inside fp32 / bf16 range (the reference uses 50)", who, a->softclamp);
    p.B = a->B; p.H = a->H; p.Np = a->Np;
    if (a->unclamped) {
        p.clamp = 0.f; p.scale_over_clamp = 0.f;
    } else {
        p.clamp = a->softclamp; p.scale_over_clamp = a->scale / a->softclamp;
    }
    p.scale = a->scale; p.scale_log2e = a->scale * LOG2E_F;
    p.dropout_p = a->dropout_p;
    p.drop_thresh = drop_thresh16(a->dropout_p);
    p.keep_scale = drop_keep_scale(p.drop_thresh);
    p.seed = a->seed; p.seed_dev = reinterpret_cast<const unsigned long long*>(a->seed_dev);
    p.drop_stride = (a->Np + 1) & ~1;
    p.mask_words = ((a->Np + TKV - 1) / TKV) * 4;
    p.maskbits = reinterpret_cast<const unsigned int*>(a->ws_maskbits);
    if (!a->maskbits_ready) {
        attn_maskbits_kernel<<<(a->B * p.mask_words + 127) / 128, 128, 0, st>>>(a->keymask, reinterpret_cast<unsigned int*>(a->ws_maskbits),
                                                                             a->B, a->Np, p.mask_words);
        return check_launch("attn_maskbits_kernel");
    }
    return 0;
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_attn_workspace_bytes(int32_t B, int32_t Np) {
    const int words = ((Np + 127) / 128) * 4;
    return (size_t)B * words * sizeof(unsigned int);
}

extern "C" int b200_attn_maskbits(const uint8_t* keymask, void* ws_maskbits, int32_t B, int32_t Np, b200_stream_t stream) {
    B200_REQUIRE(ws_maskbits && B > 0 && Np > 0, "attn_maskbits: bad arguments");
    const int words = ((Np + TKV - 1) / TKV) * 4;
    attn_maskbits_kernel<<<(B * words + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        keymask, reinterpret_cast<unsigned int*>(ws_maskbits), B, Np, words);
    return check_launch("attn_maskbits_kernel");
}

extern "C" int b200_attn_fwd(const b200_attn_fwd_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->q && a->k && a->v && a->o && a->og && a->lse && a->ws_maskbits, "attn_fwd: null pointer");
    AttnTcP p{};
    if (int rc = attn_setup(a, p, "attn_fwd", st)) return rc;
    p.nkv = (a->Np + TKV - 1) / TKV;
    p.gate = a->gate; p.o = (__nv_bfloat16*)a->o; p.og = (__nv_bfloat16*)a->og; p.lse = a->lse;
    CUtensorMap tq, tk, tv;
    const long long rows = (long long)a->B * a->H * a->Np;
    const int dh = a->dim_head, na = dh / 64;
    if (make_head_map(&tq, a->q, rows, dh, 128) || make_head_map(&tk, a->k, rows, dh, 64) || make_head_map(&tv, a->v, rows, dh, 64)) return -1;
    const int smem = na * (TILE16 + 2 * KV_STAGES * TILE8) + 128 + 1024;   // Q, K/V rings, barriers, alignment slack
    static DeviceOnce once[4];
    const auto kern = dh == 64 ? (a->unclamped ? attn_fwd_wgmma_kernel<true, 64> : attn_fwd_wgmma_kernel<false, 64>)
                               : (a->unclamped ? attn_fwd_wgmma_kernel<true, 128> : attn_fwd_wgmma_kernel<false, 128>);
    cudaError_t e = set_max_smem_once(once[(a->unclamped ? 1 : 0) + (dh == 128 ? 2 : 0)], kern, smem);
    B200_REQUIRE(e == cudaSuccess, "attn_fwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    dim3 grid((a->Np + TQ - 1) / TQ, a->H, a->B);
    kern<<<grid, 384, smem, st>>>(tq, tk, tv, p);
    return check_launch("attn_fwd_wgmma_kernel");
}

extern "C" int b200_attn_bwd(const b200_attn_bwd_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->q && a->k && a->v && a->o && a->d_og && a->lse && a->ws_dO && a->ws_delta && a->dq && a->dk && a->dv && a->ws_maskbits,
                 "attn_bwd: null pointer");
    AttnBwdTcP p{};
    if (int rc = attn_setup(a, p, "attn_bwd", st)) return rc;
    const AttnPrepP pp{a->gate, (const __nv_bfloat16*)a->o, a->B, a->H, a->Np, (const __nv_bfloat16*)a->d_og, a->d_gate,
                       (__nv_bfloat16*)a->ws_dO, a->ws_delta};
    const int dh = a->dim_head;
    const long long prep_threads = (long long)a->B * a->H * a->Np * (dh / 8);
    if (dh == 64) attn_bwd_prep_kernel<64><<<(unsigned)((prep_threads + 255) / 256), 256, 0, st>>>(pp);
    else attn_bwd_prep_kernel<128><<<(unsigned)((prep_threads + 255) / 256), 256, 0, st>>>(pp);
    if (int rc = check_launch("attn_bwd_prep_kernel")) return rc;
    p.nq = (a->Np + TQB - 1) / TQB;
    const size_t nelem = (size_t)a->B * a->H * a->Np * dh;
    cudaError_t e = cudaMemsetAsync(a->dq, 0, nelem * sizeof(float), st);
    B200_REQUIRE(e == cudaSuccess, "attn_bwd: memset: %s", cudaGetErrorString(e));
    p.lse = a->lse; p.delta = a->ws_delta;
    p.dk = (__nv_bfloat16*)a->dk; p.dv = (__nv_bfloat16*)a->dv;
    CUtensorMap tq, tk, tv, tdo, tdq;
    const long long rows = (long long)a->B * a->H * a->Np;
    const int kv_rows = dh == 64 ? TKV : 64;   // keys per CTA
    if (make_head_map(&tq, a->q, rows, dh, TQB) || make_head_map(&tk, a->k, rows, dh, kv_rows) || make_head_map(&tv, a->v, rows, dh, kv_rows) ||
        make_head_map(&tdo, a->ws_dO, rows, dh, TQB) || make_dq_map(&tdq, reinterpret_cast<float*>(a->dq), a->B * a->H, a->Np, dh)) return -1;
    dim3 grid((a->Np + kv_rows - 1) / kv_rows, a->H, a->B);
    if (dh == 64) {
        // K, V, Q/dO rings, dS^T tiles, dQ staging, lse / delta slots, barriers, alignment slack
        const int smem = 2 * TILE16 + 2 * QDO_STAGES * TILE8 + 4 * TILE8 + 2 * TILE16 + 2 * 2 * 128 * (int)sizeof(float) + 128 + 1024;
        static DeviceOnce once[2];
        const auto kern = a->unclamped ? attn_bwd_wgmma_kernel<true> : attn_bwd_wgmma_kernel<false>;
        cudaError_t e2 = set_max_smem_once(once[a->unclamped ? 1 : 0], kern, smem);
        B200_REQUIRE(e2 == cudaSuccess, "attn_bwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e2));
        kern<<<grid, 256, smem, st>>>(tq, tk, tv, tdo, tdq, p);
        return check_launch("attn_bwd_wgmma_kernel");
    }
    // K, V (2 column blocks each), Q/dO rings, P^T and dS^T tiles, dQ staging, exchange halves, lse / delta slots, barriers, alignment
    const int smem = 4 * TILE8 + 4 * QDO_STAGES * TILE8 + 2 * TILE8 + 2 * TILE16 + (2 * 16 * 128 + 2 * 128) * (int)sizeof(float) + 128 + 1024;
    static DeviceOnce once[2];
    const auto kern = a->unclamped ? attn_bwd_d128_wgmma_kernel<true> : attn_bwd_d128_wgmma_kernel<false>;
    cudaError_t e2 = set_max_smem_once(once[a->unclamped ? 1 : 0], kern, smem);
    B200_REQUIRE(e2 == cudaSuccess, "attn_bwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e2));
    kern<<<grid, 256, smem, st>>>(tq, tk, tv, tdo, tdq, p);
    return check_launch("attn_bwd_d128_wgmma_kernel");
}
