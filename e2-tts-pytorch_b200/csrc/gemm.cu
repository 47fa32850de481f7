// wgmma / TMA GEMM for sm_90a — the tensor-core core of the E2-TTS hot path.
//
//   D[M,N] = epilogue( sum_k A[m,k] * B[n,k] ),  bf16 operands, fp32 accumulation in registers.
//
// Structure (one persistent CTA per SM, 384 threads, warp-specialised):
//   warpgroup 0, one thread : TMA producer — cp.async.bulk.tensor 2-D tiles (128B swizzle) into a kStages smem ring
//   warpgroups 1, 2         : MMA + epilogue — each owns 64 * MH rows of the CTA tile: wgmma.m64nBNk16 from the smem ring into
//                             register accumulators, then the fused epilogue on the accumulator fragments. It decides twice: GLU or
//                             not, then TMA slices or fragment stores. A non-GLU output gets one element-wise pass in place
//                             (epilogue_pass: bias / act / AdaLN gate / row mask / residual from global memory), a GLU output takes
//                             h from one routine (glu_h_pair: activation, glu_mult, dropout), and either leaves by the same two paths:
//                             - TMA: 64 x 64 at a time through a 128B-swizzled smem staging slice (two per warpgroup, alternating) and
//                               a TMA tile store (bulk async groups), so the warpgroup moves on while the previous slice drains. A
//                               residual slice is TMA-loaded into the staging buffer its output slice will occupy (the tile's first
//                               two while its last k-blocks still run) and added there. GLU (K-major operands only): per 64 rows and
//                               128 packed columns, u + bias and gate + bias leave as two pre-activation slices and h, computed from
//                               the bf16 values just staged, as a third; the producer stages the tile's bias and glu_mult in smem.
//                             - fragments: bf16x2 / fp32 pairs stored from registers, fp32 split-K partials through vector atomics —
//                               for outputs without 16-byte aligned bases, N % 8 != 0, fp32, MN-major GLU and GLU without D2. The
//                               fragment GLU path is also the reference the TMA one is tested against, bit for bit.
// While a consumer warpgroup runs its epilogue the producer is already filling the ring with the next tile's operands.
// Operands may be K-major or MN-major (transposed storage) so that the backward contractions
// dX = dY*W and dW = dY^T*X read activations exactly as they lie in HBM — no transposes are materialised.
#include <stdlib.h>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int BM = 128;
constexpr int BK = 64;              // 64 bf16 = one 128-byte swizzle atom
constexpr int kGemmThreads = 384;   // warpgroup 0 TMA, warpgroups 1..2 MMA + epilogue
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int kSliceBytes = 64 * 64 * 2;   // one 64 x 64 bf16 output slice, 128B-swizzled (the TMA box layout)

struct GemmParams {
    int M, N, K;
    int tiles_m, tiles_n, num_work;
    int kb_total, kb_per_split, kb_a1;  // k-blocks; kb_a1 = number of k-blocks served by the first A source
    void* D; long long ldd; int d_fp32;
    void* D2; long long ldd2;
    const float* bias;
    const float* colscale; int rows_per_batch;
    const unsigned char* rowmask;
    const void* resid; long long ldr;
    int geglu; float dropout_p; unsigned long long seed;   // geglu: 0 none, else the GLU activation (GLU_GELU / GLU_SILU / GLU_RELU2)
    const unsigned long long* seed_dev;   // optional device addend of the seed (CUDA-graph replays)
    int atomic_out;
    int tma_store;   // bf16 output through the smem staging slices and TMA stores (tmD)
    int resid_tma;   // tma_store with a 16-byte aligned residual: its slices are TMA-loaded into the staging buffers (tmR)
    const float* glu_mult;   // optional [N/2] multiplier of the hidden units (x-transformers GLU mult_bias), hidden-unit order
    int glu_tma;     // GLU outputs through the staging slices and TMA stores (h: tmD, pre-activations: tmD2); bias / glu_mult staged per tile
};

constexpr int GLU_GELU = 1, GLU_SILU = 2, GLU_RELU2 = 3;
constexpr int ACT_GELU = 1;   // b200_gemm_args.act: plain exact-erf GELU of (z + bias), no GLU

// Tiles: (BM * MH) x BN. MH == 2 gives each consumer warpgroup 128 rows (two m64 MMAs per k-step share one B tile); BN == 256 gives it
// one m64n256 MMA per k-step. Both halve the smem -> tensor-core bytes per FLOP of the 128 x 128 tile; 128 fp32 accumulators per thread.
template <int BN, int MH>
struct GemmSmem {
    static constexpr int A_BYTES = MH * A_STAGE_BYTES;
    static constexpr int B_STAGE_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_STAGE_BYTES;
    static constexpr int kStages = (STAGE_BYTES <= 32768) ? 6 : 4;
    static constexpr int TILE_BYTES = kStages * STAGE_BYTES;
    static constexpr int STG_BYTES = 2 * 2 * kSliceBytes;        // two slices per consumer warpgroup: 32 KB
    static constexpr int BAR_BYTES = 256;   // full / empty per stage, one residual barrier per staging slice, GLU operands full / empty
    static_assert((2 * kStages + 4 + 2) * 8 <= BAR_BYTES, "GEMM mbarriers exceed their shared-memory slot");
    static constexpr int OPS_BYTES = BN * 4 + BN / 2 * 4;        // GLU tile operands: packed bias [BN] and glu_mult [BN / 2], fp32
    static constexpr int TOTAL = TILE_BYTES + STG_BYTES + BAR_BYTES + OPS_BYTES + 1024;  // + slack for manual 1024B alignment
    static_assert(TOTAL <= 227 * 1024, "GEMM shared memory exceeds the 227 KB a block may use");
};

// Exact (erf) GELU of x-transformers' GLU (A.2) for a PAIR of pre-activations:  gelu(x) = x Phi(x) = relu(x) - |x| Phi(-|x|), with the
// Gaussian tail written as Phi(-a) = 2^(-h(a)) and h a degree-7 polynomial (Chebyshev fit on [0, 6]; beyond, h keeps growing and
// a 2^-h < 6e-9): |error| < 5e-7 absolute on the GELU value in fp32 Horner arithmetic, 0.5 % of a bf16 half-ulp of the result.
// 7 paired FMAs + 2 MUFU.EX2 + ~5 more per PAIR; the Abramowitz-Stegun form it replaces cost 2 MUFU + ~13 scalar FMA-pipe instructions
// per element, and the GEGLU GEMM is bounded by its epilogue.
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
    const float2 a = make_float2(fabsf(x.x), fabsf(x.y));
    float2 t = ffma2(a, make_float2(-1.9449223600531695e-06f, -1.9449223600531695e-06f), make_float2(6.386057066265494e-05f, 6.386057066265494e-05f));
    t = ffma2(t, a, make_float2(-0.0009488713694736362f, -0.0009488713694736362f));
    t = ffma2(t, a, make_float2(0.008582375012338161f, 0.008582375012338161f));
    t = ffma2(t, a, make_float2(-0.0541183240711689f, -0.0541183240711689f));
    t = ffma2(t, a, make_float2(-0.4582974314689636f, -0.4582974314689636f));
    t = ffma2(t, a, make_float2(-1.1513246297836304f, -1.1513246297836304f));
    t = ffma2(t, a, make_float2(-0.9999869465827942f, -0.9999869465827942f));   // -h(a)
    float ex, ey;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(t.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ey) : "f"(t.y));
    return ffma2(make_float2(-a.x, -a.y), make_float2(ex, ey), make_float2(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f)));
}

// SiLU (x-transformers FeedForward(swish=True)) for a PAIR: silu(x) = x / (1 + 2^(-x log2 e)), one MUFU.EX2 and one MUFU.RCP (inside
// __fdividef) per element. The rounded exponent argument, ex2.approx (2^-22 relative), the add and __fdividef (2 ulp) keep the relative
// error below (8 + 1.5 |x|) 2^-24: under 4e-6 for |x| <= 40, 0.2 % of a bf16 half-ulp. Where 1 + 2^(-x log2 e) exceeds 2^126 (x < -87)
// the value is 0, and |silu(x)| < 1e-36 there; for large positive x the exponent underflows to 0 and silu(x) = x exactly.
// (The same arithmetic with an explicit rcp.approx and product makes the 128 x 256 tile spill 8 bytes; this form does not.)
__device__ __forceinline__ float2 silu2(float2 x) {
    const float2 t = fmul2(x, make_float2(-1.4426950408889634f, -1.4426950408889634f));
    float ex, ey;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(t.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ey) : "f"(t.y));
    const float2 d = fadd2(make_float2(ex, ey), make_float2(1.f, 1.f));
    return make_float2(__fdividef(x.x, d.x), __fdividef(x.y, d.y));
}

// ReLU^2 (x-transformers FeedForward(relu_squared=True)) for a PAIR: one max and one product per element, exactly 0 for x <= 0.
__device__ __forceinline__ float2 relu2_2(float2 x) {
    const float2 r = make_float2(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f));
    return fmul2(r, r);
}

template <int ACT>
__device__ __forceinline__ float2 glu_act2(float2 g) {
    if constexpr (ACT == GLU_GELU) return gelu_erf2(g);
    else if constexpr (ACT == GLU_SILU) return silu2(g);
    else return relu2_2(g);
}

// Output staging: each consumer warpgroup owns two 64 x 64 bf16 slices in shared memory (kSliceBytes each, 128B-swizzled: the TMA box
// layout) and fills them alternately; the warpgroup's n-th slice uses buffer n & 1. A thread writes its fragment rows r, r + 8 and, per
// 8-column group jj of the slice, the 4 bytes at column 8 jj + 2 (lane % 4) to 16-byte chunk (jj ^ (r & 7)) of the row — the TMA's 128B swizzle,
// and conflict-free: the 8 rows of a warp store land in 8 different chunks (r & 7 == lane / 4 for both rows). slice_addr gives that
// address; toff = (16 wq + lane / 4) * 128 + 4 (lane % 4), swz = (lane / 4) << 4.
__device__ __forceinline__ uint32_t slice_addr(uint32_t buf, uint32_t toff, uint32_t swz, int i, int jj) {
    return buf + toff + (uint32_t)i * 8 * 128 + (((uint32_t)jj << 4) ^ swz);
}
// toff of the GLU epilogue, from the lane index read inside it: computed once ahead of the tile loop, it would hold a register
// through the mainloop, and the 128 x 256 tile spills it.
__device__ __forceinline__ uint32_t slice_toff(int wq) {
    uint32_t l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return (uint32_t)(wq * 16 + (l >> 2)) * 128 + 4 * (l & 3);
}
// Waits until the buffer of slice n is free (the store issued from it two slices ago has read it); returns its shared address.
__device__ __forceinline__ uint32_t slice_acquire(uint8_t* my_stg, uint32_t n, int cw, int t) {
    if (t == 0) bulk_wait_group_read<1>();
    named_bar_sync(1 + cw, 128);
    return smem_u32(my_stg + (n & 1) * kSliceBytes);
}
// TMA-loads the residual's 64 x 64 slice at (column c0, row c1) into staging buffer b; completes on that buffer's barrier. The
// whole box counts: the TMA zero-fills what lies outside the tensor.
__device__ __forceinline__ void resid_load(const CUtensorMap* m, uint8_t* my_stg, uint64_t* my_rbar, uint32_t b, int c0, int c1) {
    mbar_arrive_expect_tx(&my_rbar[b], kSliceBytes);
    tma_load_2d(my_stg + b * kSliceBytes, m, &my_rbar[b], c0, c1);
}
// Orders the warpgroup's generic-proxy writes of slice n before the TMA (async proxy) reads them, then one thread stores the slice at
// (column c0, row c1) of `m`; rows and columns outside the tensor are clipped.
__device__ __forceinline__ void slice_store(const CUtensorMap* m, uint8_t* my_stg, uint32_t n, int cw, int t, int c0, int c1) {
    fence_proxy_async();
    named_bar_sync(1 + cw, 128);
    if (t == 0) {
        tma_store_2d(m, my_stg + (n & 1) * kSliceBytes, c0, c1);
        bulk_commit_group();
    }
}

// Fragment of an m64nBN accumulator: thread (wq, lane) holds rows 16 wq + lane / 4 (+ 8) and, for every 8-column group j,
// columns 8 j + 2 (lane % 4) + {0, 1}: acc[h][4 j + 2 i + c] = (row + 8 i, column + c) of the warpgroup's m64 block h.
__device__ __forceinline__ int frag_row(int tm, int cw, int wq, int lane, int MH, int h, int i) {
    return tm * BM * MH + (cw * MH + h) * 64 + wq * 16 + (lane >> 2) + 8 * i;
}

// GLU dropout state, built once per epilogue: P(drop) = thr32 / 2^32 on the hash words of the hidden-unit pairs of an [M, N / 2]
// hidden tensor; kept units are scaled by keep_scale. (The threshold is converted once per use: one shared conversion makes the
// 128 x 256 MN-major kernels spill.)
struct GluDrop { bool on; float keep_scale; uint32_t seed, thr32; };
__device__ __forceinline__ GluDrop glu_drop(const GemmParams& p) {
    const bool on = p.dropout_p > 0.f;
    return GluDrop{on, on ? drop_keep_scale(drop_thresh16(p.dropout_p)) : 1.f, on ? drop_seed_word(p.seed, p.seed_dev) : 0u,
                   drop_thresh32(drop_thresh16(p.dropout_p))};
}

// One packed pair of hidden units (hcol, hcol + 1) of `row`: h = u * act(gate) (* glu_mult) (* dropout keep / (1 - p)), bf16, from the
// bf16 pre-activation words (the rounded values the backward pass recomputes from). mult_pair() loads the glu_mult pair, when `mult`;
// pair() gives the dropout pair index (glu_drop_pair). Both are evaluated only inside their branches: loaded or computed ahead of
// them, they hold registers that make the GEMM kernels spill.
template <int ACT, class MultPair, class PairIdx>
__device__ __forceinline__ uint32_t glu_h_pair(uint32_t wu, uint32_t wgt, bool mult, MultPair mult_pair, const GluDrop& dr, PairIdx pair) {
    float2 h2 = fmul2(make_float2(bf16_lo(wu), bf16_hi(wu)), glu_act2<ACT>(make_float2(bf16_lo(wgt), bf16_hi(wgt))));
    if (mult) h2 = fmul2(h2, mult_pair());
    if (dr.on) {
        const DropWords hsh = drop_words(dr.seed, pair());
        h2 = fmul2(h2, make_float2(hsh.a >= dr.thr32 ? dr.keep_scale : 0.f, hsh.b >= dr.thr32 ? dr.keep_scale : 0.f));
    }
    return pack_bf16(h2.x, h2.y);
}

// GLU epilogue on the accumulator fragments: every 128 packed columns hold [0,64) = u, [64,128) = gate of the same 64 hidden units, so a
// thread holds both halves of each of its hidden units (fragment groups j and j + 8 of the 128-column group). D2 <- the bf16
// pre-activations, D <- h. The reference the TMA path (glu_store_slices) is tested against, and the path of MN-major operands and of
// calls whose h, pre-activation or glu_mult base is not 16-byte aligned or that give no D2.
template <int ACT, int BN, int MH>
__device__ __forceinline__ void glu_epilogue(const GemmParams& p, float (&acc)[MH][BN / 2], int tm, int tn, int cw, int wq, int lane) {
    const int cq = 2 * (lane & 3);
    const GluDrop dr = glu_drop(p);
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = frag_row(tm, cw, wq, lane, MH, h, i);
            if (row >= p.M) continue;
#pragma unroll
            for (int sub = 0; sub < BN / 128; ++sub) {
                const int colg = tn * BN + sub * 128;   // first packed column of the group (N % 128 == 0)
                if (colg >= p.N) continue;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int cu = colg + 8 * j + cq;           // packed column of u; the gate is 64 further
                    const int hcol = colg / 2 + 8 * j + cq;     // hidden-unit column
                    float2 u = make_float2(acc[h][4 * (sub * 16 + j) + 2 * i], acc[h][4 * (sub * 16 + j) + 2 * i + 1]);
                    float2 g = make_float2(acc[h][4 * (sub * 16 + 8 + j) + 2 * i], acc[h][4 * (sub * 16 + 8 + j) + 2 * i + 1]);
                    if (p.bias) {
                        u = fadd2(u, make_float2(__ldg(p.bias + cu), __ldg(p.bias + cu + 1)));
                        g = fadd2(g, make_float2(__ldg(p.bias + cu + 64), __ldg(p.bias + cu + 65)));
                    }
                    const uint32_t wu = pack_bf16(u.x, u.y), wgt = pack_bf16(g.x, g.y);
                    if (p.D2) {
                        __nv_bfloat16* d2 = reinterpret_cast<__nv_bfloat16*>(p.D2) + (long long)row * p.ldd2 + cu;
                        *reinterpret_cast<uint32_t*>(d2) = wu;
                        *reinterpret_cast<uint32_t*>(d2 + 64) = wgt;
                    }
                    const auto m = [&] { return make_float2(__ldg(p.glu_mult + hcol), __ldg(p.glu_mult + hcol + 1)); };
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.D) + (long long)row * p.ldd + hcol) =
                        glu_h_pair<ACT>(wu, wgt, p.glu_mult, m, dr, [&] { return glu_drop_pair(row, p.N / 2, hcol); });
                }
            }
        }
    }
}


// The tile's 64 x 64 output slices from the finished fragments, each through the warpgroup's next staging buffer and a TMA store.
// RESID: the buffer already holds the slice's residual, TMA-loaded by resid_load (the first two of a tile from the mainloop, the
// others here, one slice ahead); each pair is added in fp32 from the address it is written back to.
template <bool RESID, int BN, int MH>
__device__ __forceinline__ void store_slices(const GemmParams& p, float (&acc)[MH][BN / 2], const CUtensorMap* tmD, const CUtensorMap* tmR,
                                             uint8_t* my_stg, uint64_t* my_rbar, uint32_t& nslice, int tm, int tn, int cw, int wq, int lane,
                                             int t) {
    const uint32_t swz = (uint32_t)(lane >> 2) << 4;
    const uint32_t toff = (uint32_t)(wq * 16 + (lane >> 2)) * 128 + 4 * (lane & 3);
#pragma unroll
    for (int h = 0; h < MH; ++h) {
        const int rowb = tm * BM * MH + (cw * MH + h) * 64;
#pragma unroll
        for (int s = 0; s < BN / 64; ++s) {
            const int colb = tn * BN + s * 64;
            if (colb >= p.N) break;                  // uniform across the warpgroup
            uint32_t buf;
            if constexpr (RESID) {
                // the buffer holds this slice's residual once its barrier completes (each buffer's barrier completes once per two
                // slices of the warpgroup); it was free when the load was issued
                buf = smem_u32(my_stg + (nslice & 1) * kSliceBytes);
                mbar_wait(&my_rbar[nslice & 1], (nslice >> 1) & 1);
            } else {
                buf = slice_acquire(my_stg, nslice, cw, t);
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int j = s * 8 + jj;
                    const uint32_t a = slice_addr(buf, toff, swz, i, jj);
                    float v0 = acc[h][4 * j + 2 * i], v1 = acc[h][4 * j + 2 * i + 1];
                    if constexpr (RESID) {
                        const uint32_t r = ld_shared_u32(a);
                        v0 += bf16_lo(r); v1 += bf16_hi(r);
                    }
                    st_shared_u32(a, pack_bf16(v0, v1));
                }
            }
            slice_store(tmD, my_stg, nslice, cw, t, colb, rowb);
            if constexpr (RESID) {
                // the slice two further uses this buffer: 128 columns on (BN = 256), or these columns of the next m64 block (MH = 2)
                const bool more = MH == 1 ? (s + 2 < BN / 64 && colb + 128 < p.N) : (h + 1 < MH && tn * BN + 64 < p.N);
                if (t == 0 && more) {
                    bulk_wait_group_read<0>();       // the store just issued has read this buffer
                    resid_load(tmR, my_stg, my_rbar, nslice & 1, MH == 1 ? colb + 128 : colb, MH == 1 ? rowb : rowb + 64);
                }
            }
            ++nslice;
        }
    }
}

// GLU epilogue through the staging slices. Per 64-row band and 128-packed-column group, three 64 x 64 slices leave by TMA store:
// u + bias to D2 at packed column colg, gate + bias to D2 at colg + 64, then h to D at hidden column colg / 2. Hidden unit c of the
// group sits at the same slice position as its u and gate, so h is computed pair by pair from the bf16 u and gate the thread itself
// wrote to the two buffers (the rounded values the backward pass recomputes from) and written over u once u's store has read it.
// sbias / smult: the tile's packed bias and glu_mult slice, staged in shared memory by the producer; the dropout hashes are made in
// the h loop, one pair at a time. Bit-identical to glu_epilogue: both take h from glu_h_pair.
template <int ACT, int BN, int MH>
__device__ __forceinline__ void glu_store_slices(const GemmParams& p, float (&acc)[MH][BN / 2], const CUtensorMap* tmD, const CUtensorMap* tmD2,
                                                 uint8_t* my_stg, const float* sbias, const float* smult, uint32_t& nslice, int tm, int tn,
                                                 int cw, int wq, int lane, int t) {
    const uint32_t swz = (uint32_t)(lane >> 2) << 4;
    const uint32_t toff = slice_toff(wq);
    const int cq = 2 * (lane & 3);
    const GluDrop dr = glu_drop(p);
#pragma unroll
    for (int h = 0; h < MH; ++h) {
        const int rowb = tm * BM * MH + (cw * MH + h) * 64;
#pragma unroll
        for (int sub = 0; sub < BN / 128; ++sub) {
            const int colg = tn * BN + sub * 128;   // first packed column of the group (N % 128 == 0)
            if (colg >= p.N) break;                  // uniform across the warpgroup
            // u (half 0), then gate (half 1): + bias, rounded to bf16, out to D2
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const uint32_t buf = slice_acquire(my_stg, nslice, cw, t);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int j = sub * 16 + half * 8 + jj;
                        float2 v = make_float2(acc[h][4 * j + 2 * i], acc[h][4 * j + 2 * i + 1]);
                        if (p.bias) v = fadd2(v, *reinterpret_cast<const float2*>(sbias + 8 * j + cq));
                        st_shared_u32(slice_addr(buf, toff, swz, i, jj), pack_bf16(v.x, v.y));
                    }
                }
                slice_store(tmD2, my_stg, nslice, cw, t, colg + 64 * half, rowb);
                ++nslice;
            }
            // h into u's buffer: its store was issued two slices ago, the gate store one ago
            const uint32_t bu = slice_acquire(my_stg, nslice, cw, t);
            const uint32_t bg = smem_u32(my_stg + ((nslice + 1) & 1) * kSliceBytes);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = rowb + wq * 16 + (lane >> 2) + 8 * i;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int hl = sub * 64 + 8 * jj + cq;   // hidden-unit column within the tile
                    const uint32_t a = slice_addr(bu, toff, swz, i, jj);
                    const uint32_t wu = ld_shared_u32(a), wgt = ld_shared_u32(slice_addr(bg, toff, swz, i, jj));
                    const auto m = [&] { return *reinterpret_cast<const float2*>(smult + hl); };
                    st_shared_u32(a, glu_h_pair<ACT>(wu, wgt, p.glu_mult, m, dr, [&] { return glu_drop_pair(row, p.N / 2, tn * (BN / 2) + hl); }));
                }
            }
            slice_store(tmD, my_stg, nslice, cw, t, colg / 2, rowb);
            ++nslice;
        }
    }
}

// One bf16 pair / fp32 pair of the output: columns (col, col + 1) of `row`; col is even.
__device__ __forceinline__ void store_pair(const GemmParams& p, int row, int col, float v0, float v1) {
    const bool two = col + 1 < p.N;
    if (p.d_fp32) {
        float* dp = reinterpret_cast<float*>(p.D) + (long long)row * p.ldd + col;
        const bool vec = two && (reinterpret_cast<uintptr_t>(dp) & 7) == 0;
        if (p.atomic_out) {
            if (vec) atomicAdd(reinterpret_cast<float2*>(dp), make_float2(v0, v1));
            else { atomicAdd(dp, v0); if (two) atomicAdd(dp + 1, v1); }
        } else {
            if (vec) *reinterpret_cast<float2*>(dp) = make_float2(v0, v1);
            else { dp[0] = v0; if (two) dp[1] = v1; }
        }
    } else {
        __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(p.D) + (long long)row * p.ldd + col;
        if (two) *reinterpret_cast<uint32_t*>(dp) = pack_bf16(v0, v1);   // ldd % 8 == 0 and col even: 4-byte aligned
        else dp[0] = __float2bfloat16_rn(v0);
    }
}

// The element-wise epilogue of non-GLU outputs, in place on the fragments: bias -> act -> AdaLN gate (colscale) -> row mask -> +
// residual read from global memory (a residual TMA-loaded into the staging slices is added by store_slices instead). Rows >= M and
// columns >= N are left as they are: the stores skip or clip them.
template <int ACT, int BN, int MH>
__device__ __forceinline__ void epilogue_pass(const GemmParams& p, float (&acc)[MH][BN / 2], int tm, int tn, int cw, int wq, int lane) {
    const bool resid_ldg = p.resid && !p.resid_tma;
    if (!(ACT || p.bias || p.colscale || p.rowmask || resid_ldg)) return;   // plain outputs and split-K partials
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = frag_row(tm, cw, wq, lane, MH, h, i);
            if (row >= p.M) continue;
            const bool masked = p.rowmask && p.rowmask[row] == 0;
            const float* cs = p.colscale ? p.colscale + (long long)(row / p.rows_per_batch) * p.N : nullptr;
            const __nv_bfloat16* rp = resid_ldg ? reinterpret_cast<const __nv_bfloat16*>(p.resid) + (long long)row * p.ldr : nullptr;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = tn * BN + 8 * j + cq;
                if (col >= p.N) continue;
                const bool two = col + 1 < p.N;
                float v0 = acc[h][4 * j + 2 * i], v1 = acc[h][4 * j + 2 * i + 1];
                if (p.bias) { v0 += __ldg(p.bias + col); if (two) v1 += __ldg(p.bias + col + 1); }
                if constexpr (ACT == ACT_GELU) { const float2 g = gelu_erf2(make_float2(v0, v1)); v0 = g.x; v1 = g.y; }
                if (cs) { v0 *= __ldg(cs + col); if (two) v1 *= __ldg(cs + col + 1); }
                if (masked) { v0 = 0.f; v1 = 0.f; }
                if (rp) {
                    if (two) {
                        const uint32_t u = *reinterpret_cast<const uint32_t*>(rp + col);
                        v0 += bf16_lo(u); v1 += bf16_hi(u);
                    } else {
                        v0 += __bfloat162float(rp[col]);
                    }
                }
                acc[h][4 * j + 2 * i] = v0;
                acc[h][4 * j + 2 * i + 1] = v1;
            }
        }
    }
}

// The finished fragments of a non-GLU output, pair by pair from registers: fp32 outputs, split-K partials, and bf16 outputs the TMA
// cannot store (unaligned base or N % 8 != 0).
template <int BN, int MH>
__device__ __forceinline__ void store_frags(const GemmParams& p, float (&acc)[MH][BN / 2], int tm, int tn, int cw, int wq, int lane) {
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = frag_row(tm, cw, wq, lane, MH, h, i);
            if (row >= p.M) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = tn * BN + 8 * j + cq;
                if (col < p.N) store_pair(p, row, col, acc[h][4 * j + 2 * i], acc[h][4 * j + 2 * i + 1]);
            }
        }
    }
}

// Work item w -> output tile (tm, tn) and its k-blocks [kb0, kb1) (split-K: the split's share of them); the producer thread and the
// consumer warpgroups walk the same items.
struct WorkItem { int tm, tn, kb0, kb1; };
__device__ __forceinline__ WorkItem work_item(const GemmParams& p, int w) {
    const int rest = w / p.tiles_m;
    const int kb0 = rest / p.tiles_n * p.kb_per_split;
    return WorkItem{w % p.tiles_m, rest % p.tiles_n, kb0, min(p.kb_total, kb0 + p.kb_per_split)};
}

// ACT = ACT_GELU: GELU(z + bias) ahead of the rest of the epilogue (b200_gemm_args.act; instantiated for K-major A and B only).
// ACT = 0 compiles to the instructions the kernel had before it took the parameter.
template <int BN, bool A_MN, bool B_MN, int MH, int ACT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                  const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmD,
                  const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmD2, const GemmParams p) {
    using S = GemmSmem<BN, MH>;
    constexpr int kStages = S::kStages;
    constexpr int BMT = BM * MH;   // rows of the CTA tile
    constexpr int NACC = BN / 2;   // accumulators per thread and m64 block
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment by OFFSET, not by integer round-trip: the pointer keeps its shared-memory provenance
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* smA = smem;
    uint8_t* smB = smem + kStages * S::A_BYTES;
    uint8_t* stg = smem + S::TILE_BYTES;   // output staging slices: [warpgroup][2][64 x 128 B]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::TILE_BYTES + S::STG_BYTES);
    uint64_t* empty_bar = full_bar + kStages;
    uint64_t* resid_bar = empty_bar + kStages;   // [warpgroup][2]: the residual slice TMA-loaded into that staging buffer has landed
    uint64_t* ops_full = resid_bar + 4;          // glu_tma: the tile's bias / glu_mult have landed in sops
    uint64_t* ops_empty = ops_full + 1;          // glu_tma: both consumer warpgroups are done reading them (one arrival each)
    float* sops = reinterpret_cast<float*>(smem + S::TILE_BYTES + S::STG_BYTES + S::BAR_BYTES);   // [BN] bias, then [BN / 2] glu_mult
    // the GLU TMA path is built into the K-major kernels only (the model's FF-in); the others keep their instructions as they were
    constexpr bool kGluTma = !A_MN && !B_MN;
    const bool glu_ops = kGluTma && p.glu_tma && (p.bias || p.glu_mult);

    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmA2);
        tma_prefetch_desc(&tmB);
        if (p.tma_store) tma_prefetch_desc(&tmD);
        if (p.resid_tma) tma_prefetch_desc(&tmR);
        if (kGluTma && p.glu_tma) {
            tma_prefetch_desc(&tmD);
            tma_prefetch_desc(&tmD2);
        }
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup
        }
        for (int i = 0; i < 4; ++i) mbar_init(&resid_bar[i], 1);
        mbar_init(ops_full, 1);
        mbar_init(ops_empty, 2);
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // ------------------------------------------------------------ TMA producer
            int stage = 0;
            uint32_t phase = 0;
            uint32_t ntile = 0;
            for (int w = blockIdx.x; w < p.num_work; w += gridDim.x, ++ntile) {
                const WorkItem wi = work_item(p, w);
                const int arow = wi.tm * BMT;
                const int brow = wi.tn * BN;
                for (int kb = wi.kb0; kb < wi.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], S::STAGE_BYTES);
                    uint8_t* a_dst = smA + stage * S::A_BYTES;
                    uint8_t* b_dst = smB + stage * S::B_STAGE_BYTES;
                    const CUtensorMap* ma = kb < p.kb_a1 ? &tmA : &tmA2;
                    const int ka = kb < p.kb_a1 ? kb * BK : (kb - p.kb_a1) * BK;
                    if constexpr (!A_MN) {
#pragma unroll
                        for (int h = 0; h < MH; ++h) tma_load_2d(a_dst + h * A_STAGE_BYTES, ma, &full_bar[stage], ka, arow + h * BM);
                    } else {
#pragma unroll
                        for (int i = 0; i < BMT / 64; ++i) tma_load_2d(a_dst + i * (BK * 128), ma, &full_bar[stage], arow + i * 64, ka);
                    }
                    if constexpr (!B_MN) {
#pragma unroll
                        for (int h = 0; h < BN / 128; ++h) tma_load_2d(b_dst + h * (128 * BK * 2), &tmB, &full_bar[stage], kb * BK, brow + h * 128);
                    } else {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i) tma_load_2d(b_dst + i * (BK * 128), &tmB, &full_bar[stage], brow + i * 64, kb * BK);
                    }
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
                if (glu_ops) {
                    // after the tile's operands, so the ring is refilled ahead of the previous tile's epilogue; the next tile's
                    // k-blocks wait for ring slots that the consumers free only after that epilogue anyway
                    const int nb = min(BN, p.N - brow);   // packed columns of the tile (a multiple of 128)
                    mbar_wait(ops_empty, (ntile & 1) ^ 1);
                    mbar_arrive_expect_tx(ops_full, (p.bias ? nb * 4 : 0) + (p.glu_mult ? nb * 2 : 0));
                    if (p.bias) bulk_load_1d(sops, p.bias + brow, nb * 4, ops_full);
                    if (p.glu_mult) bulk_load_1d(sops + BN, p.glu_mult + brow / 2, nb * 2, ops_full);
                }
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumer warpgroups: MMA, then epilogue
    regs_alloc<232>();
    const int cw = wg - 1;                     // which 64 * MH rows of the CTA tile
    const int t = threadIdx.x & 127;
    const int lane = t & 31, wq = t >> 5;      // warp within the warpgroup: accumulator rows 16 * wq ..
    // K-major: 8-row groups 1024 B apart; MN-major: 64-element MN atoms BK*128 B apart (LBO), 8-k-row groups 1024 B apart (SBO).
    constexpr uint32_t a_lbo = A_MN ? BK * 128 : 16, b_lbo = B_MN ? BK * 128 : 16;
    constexpr uint32_t a_adv = A_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;   // per k16 step, in 16-B units
    constexpr uint32_t b_adv = B_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;
    float acc[MH][NACC];
    uint8_t* my_stg = stg + cw * 2 * kSliceBytes;
    uint64_t* my_rbar = resid_bar + cw * 2;
    uint32_t nslice = 0;                       // staging slices this warpgroup has filled so far (buffer = nslice & 1)
    int stage = 0;
    uint32_t phase = 0;
    uint32_t ntile = 0;
    for (int w = blockIdx.x; w < p.num_work; w += gridDim.x, ++ntile) {
        const auto [tm, tn, kb0, kb1] = work_item(p, w);
        // resid_tma: each residual slice is TMA-loaded into the staging buffer its output slice will use and completes on that buffer's
        // barrier. The tile's first two go out two k-blocks before its mainloop ends, once the previous tile's stores have left both
        // buffers; the third and fourth as soon as the store of the first and second has left its buffer.
        const int kb_resid = max(kb0, kb1 - 2);
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
#pragma unroll
            for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
            wgmma_fence();
            const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smB + stage * S::B_STAGE_BYTES), b_lbo, 1024);
#pragma unroll
            for (int h = 0; h < MH; ++h) {
                // the warpgroup's m64 block (cw * MH + h) lies 64 rows = 8 KB into the A tile in both layouts
                const uint64_t adesc = make_smem_desc_sw128(smem_u32(smA + stage * S::A_BYTES + (cw * MH + h) * 8192), a_lbo, 1024);
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
                    if constexpr (BN == 256) wgmma_ss_n256<A_MN, B_MN>(acc[h], adesc + (uint64_t)(k * a_adv), bdesc + (uint64_t)(k * b_adv), accum);
                    else wgmma_ss_n128<A_MN, B_MN>(acc[h], adesc + (uint64_t)(k * a_adv), bdesc + (uint64_t)(k * b_adv), accum);
                }
            }
            wgmma_commit();
            if (p.resid_tma && kb == kb_resid && t == 0) {
                const int r0 = tm * BMT + cw * MH * 64;
                bulk_wait_group_read<0>();
                resid_load(&tmR, my_stg, my_rbar, nslice & 1, tn * BN, r0);
                if (tn * BN + 64 < p.N) resid_load(&tmR, my_stg, my_rbar, (nslice + 1) & 1, tn * BN + 64, r0);
                else if (MH == 2) resid_load(&tmR, my_stg, my_rbar, (nslice + 1) & 1, tn * BN, r0 + 64);
            }
            wgmma_wait<1>();   // the MMAs of the previous k-block have retired: its smem slot may be refilled
#pragma unroll
            for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
            if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
        if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);

        // ---------------------------------------------------------------- epilogue from the accumulator fragments
        if (!p.geglu) {
            epilogue_pass<ACT, BN, MH>(p, acc, tm, tn, cw, wq, lane);
            // a copy of the slice loop per case keeps the plain path free of per-element residual branches
            if (p.resid_tma) store_slices<true, BN, MH>(p, acc, &tmD, &tmR, my_stg, my_rbar, nslice, tm, tn, cw, wq, lane, t);
            else if (p.tma_store) store_slices<false, BN, MH>(p, acc, &tmD, &tmR, my_stg, my_rbar, nslice, tm, tn, cw, wq, lane, t);
            else store_frags<BN, MH>(p, acc, tm, tn, cw, wq, lane);
        } else if (kGluTma && p.glu_tma) {
            if constexpr (kGluTma) {
                if (glu_ops) mbar_wait(ops_full, ntile & 1);
                if (p.geglu == GLU_GELU) glu_store_slices<GLU_GELU, BN, MH>(p, acc, &tmD, &tmD2, my_stg, sops, sops + BN, nslice, tm, tn, cw, wq, lane, t);
                else if (p.geglu == GLU_SILU) glu_store_slices<GLU_SILU, BN, MH>(p, acc, &tmD, &tmD2, my_stg, sops, sops + BN, nslice, tm, tn, cw, wq, lane, t);
                else glu_store_slices<GLU_RELU2, BN, MH>(p, acc, &tmD, &tmD2, my_stg, sops, sops + BN, nslice, tm, tn, cw, wq, lane, t);
                // the last slice_store's barrier is behind every read of sops by this warpgroup
                if (glu_ops && t == 0) mbar_arrive(ops_empty);
            }
        } else if (p.geglu == GLU_GELU) {   // one copy of the GLU epilogue per activation: no per-element branch on it
            glu_epilogue<GLU_GELU, BN, MH>(p, acc, tm, tn, cw, wq, lane);
        } else if (p.geglu == GLU_SILU) {
            glu_epilogue<GLU_SILU, BN, MH>(p, acc, tm, tn, cw, wq, lane);
        } else {
            glu_epilogue<GLU_RELU2, BN, MH>(p, acc, tm, tn, cw, wq, lane);
        }
    }
    if (t == 0) bulk_wait_group<0>();   // the staging slices stay valid until the last store has completed
}

// ---------------------------------------------------------------------------------------------- host

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

// 2-D bf16 tensor map: `inner` contiguous elements, `outer` rows of pitch `ld` elements; box = box_inner x box_outer with the swizzle
// whose span equals the box's row bytes: 64 elements / 128B swizzle for the operand tiles and every output, pre-activation and
// residual slice (the only box width in use; 32 elements would take the 64B swizzle).
// A descriptor is a pure function of (pointer, extents, pitch, box): the caching allocator hands the same addresses back every
// training step, so a small per-thread direct-mapped cache removes ~1500 driver encode calls per step from the host critical path.
struct MapKey { const void* ptr; int64_t inner, outer, ld; int box, box_inner; };
struct MapSlot { MapKey k; CUtensorMap m; bool valid; };
static int make_map_uncached(CUtensorMap* m, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_outer, int box_inner);
static int make_map(CUtensorMap* m, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_outer, int box_inner = 64) {
    constexpr int kSlots = 1024;
    static thread_local MapSlot cache[kSlots];
    uint64_t h = reinterpret_cast<uintptr_t>(ptr) >> 4;
    h = (h ^ (uint64_t)inner * 0x9E3779B97F4A7C15ull ^ (uint64_t)outer * 0xC2B2AE3D27D4EB4Full ^ (uint64_t)ld * 0x165667B19E3779F9ull ^ (uint64_t)(box_outer * 131 + box_inner)) * 0xFF51AFD7ED558CCDull;
    MapSlot& sl = cache[(h >> 40) % kSlots];
    if (sl.valid && sl.k.ptr == ptr && sl.k.inner == inner && sl.k.outer == outer && sl.k.ld == ld && sl.k.box == box_outer && sl.k.box_inner == box_inner) {
        *m = sl.m;
        return 0;
    }
    if (int rc = make_map_uncached(m, ptr, inner, outer, ld, box_outer, box_inner)) return rc;
    sl.k = MapKey{ptr, inner, outer, ld, box_outer, box_inner};
    sl.m = *m;
    sl.valid = true;
    return 0;
}
static int make_map_uncached(CUtensorMap* m, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_outer, int box_inner) {
    PFN_encodeTiled enc = get_encode_fn();
    B200_REQUIRE(enc, "cuTensorMapEncodeTiled entry point not available");
    B200_REQUIRE((ld % 8) == 0, "gemm: row pitch %lld not a multiple of 8 elements", (long long)ld);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "gemm: operand not 16-byte aligned");
    cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, box_inner == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

template <int BN, bool A_MN, bool B_MN, int MH, int ACT = 0>
static int launch_gemm(const CUtensorMap (&tm)[6], const GemmParams& p, cudaStream_t st) {
    using S = GemmSmem<BN, MH>;
    auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN, MH, ACT>;
    static DeviceOnce once;   // one flag per template instantiation and device
    {
        cudaError_t e = set_max_smem_once(once, kern, S::TOTAL);
        B200_REQUIRE(e == cudaSuccess, "gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    const int grid = p.num_work < num_sms() ? p.num_work : num_sms();
    kern<<<grid, kGemmThreads, S::TOTAL, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
    return check_launch("gemm_wgmma_kernel");
}

}  // namespace b200

using namespace b200;

extern "C" int b200_gemm(const b200_gemm_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->A && a->B && a->D, "gemm: null operand");
    B200_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "gemm: empty problem %lldx%lldx%lld", (long long)a->M, (long long)a->N, (long long)a->K);
    B200_REQUIRE(a->M < (1ll << 31) && a->N < (1ll << 31) && a->K < (1ll << 31), "gemm: dimension too large");
    const bool a_mn = a->a_mn_major != 0, b_mn = a->b_mn_major != 0;
    GemmParams p{};
    p.M = (int)a->M; p.N = (int)a->N; p.K = (int)a->K;
    // force_tile: 0 auto, 1 = 128x128, 2 = 256x128, 3 = 128x256 (auto: 128x256 for M >= 512, N >= 256; 256x128 for other M >= 256)
    const bool wide = a->force_tile == 3 || (a->force_tile == 0 && p.M >= 512 && p.N >= 256);
    const int BN = wide ? 256 : 128;
    const int MH = wide ? 1 : (a->force_tile == 1) ? 1 : ((a->force_tile == 2 || p.M >= 256) ? 2 : 1);
    const int tile_rows = BM * MH;
    p.tiles_m = (p.M + tile_rows - 1) / tile_rows;
    p.tiles_n = (p.N + BN - 1) / BN;
    p.kb_total = (p.K + BK - 1) / BK;
    p.kb_a1 = p.kb_total;
    if (a->A2) {
        B200_REQUIRE(a->K1 > 0 && a->K1 < a->K && (a->K1 % BK) == 0, "gemm: K1=%lld must be a multiple of %d inside (0,K)", (long long)a->K1, BK);
        p.kb_a1 = (int)(a->K1 / BK);
    }
    int split = a->split_k > 1 ? a->split_k : 1;
    if (a->split_k < 0) {
        // auto (weight gradients: few output tiles, very long K): fill the machine once — one work item per CTA —
        // while every split keeps >= 8 k-blocks so that the pipeline fill and the fp32 reduction of its partial tile stay amortised.
        const int units = num_sms();
        const int tiles = p.tiles_m * p.tiles_n;
        int s_fill = (units + tiles / 2) / tiles;                 // nearest number of splits that fills the units once
        while (s_fill > 1 && tiles * s_fill > units) --s_fill;     // never spill into a second, mostly empty round
        const int s_max = p.kb_total / 8;
        split = s_fill < 1 ? 1 : s_fill;
        if (split > s_max) split = s_max < 1 ? 1 : s_max;
        if (split > 64) split = 64;
    }
    if (split > p.kb_total) split = p.kb_total;
    p.kb_per_split = (p.kb_total + split - 1) / split;
    split = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
    p.num_work = p.tiles_m * p.tiles_n * split;
    p.atomic_out = split > 1;
    p.D = a->D; p.ldd = a->ldd; p.d_fp32 = a->d_fp32;
    p.D2 = a->D2; p.ldd2 = a->ldd2;
    p.bias = a->bias; p.colscale = a->colscale; p.rows_per_batch = (int)(a->rows_per_batch > 0 ? a->rows_per_batch : 1);
    p.rowmask = a->rowmask; p.resid = a->resid; p.ldr = a->ldr;
    B200_REQUIRE(a->geglu >= 0 && a->geglu <= GLU_RELU2, "gemm: geglu=%d is not an activation code (0 none, 1 GELU, 2 SiLU, 3 ReLU^2)", (int)a->geglu);
    B200_REQUIRE(!a->glu_mult || a->geglu, "gemm: glu_mult needs the GLU epilogue (geglu != 0)");
    p.geglu = a->geglu; p.dropout_p = a->dropout_p; p.seed = a->seed; p.seed_dev = reinterpret_cast<const unsigned long long*>(a->seed_dev);
    p.glu_mult = a->glu_mult;
    if (p.atomic_out) {
        B200_REQUIRE(a->d_fp32, "gemm: split-K requires an fp32 output");
        B200_REQUIRE(!a->bias && !a->colscale && !a->rowmask && !a->resid && !a->geglu, "gemm: split-K supports no epilogue");
        cudaError_t e = cudaMemset2DAsync(a->D, (size_t)a->ldd * 4, 0, (size_t)a->N * 4, (size_t)a->M, st);
        B200_REQUIRE(e == cudaSuccess, "gemm: memset: %s", cudaGetErrorString(e));
    }
    if (a->geglu) {
        B200_REQUIRE((a->N % 128) == 0 && !a->d_fp32 && !a->colscale && !a->rowmask && !a->resid, "gemm: GEGLU needs N %% 128 == 0, bf16 out, no other epilogue");
        B200_REQUIRE((a->ldd % 8) == 0 && (!a->D2 || (a->ldd2 % 8) == 0), "gemm: GEGLU output pitch must be a multiple of 8");
        B200_REQUIRE(!a->bias || (reinterpret_cast<uintptr_t>(a->bias) & 15) == 0, "gemm: GEGLU bias must be 16-byte aligned");
    }
    B200_REQUIRE(a->act == 0 || a->act == ACT_GELU, "gemm: act=%d is not an activation code (0 none, 1 GELU)", (int)a->act);
    if (a->act) {
        B200_REQUIRE(!a->geglu && a->split_k >= 0 && a->split_k <= 1 && !a->d_fp32, "gemm: act needs a bf16 output without GLU or split-K");
        B200_REQUIRE(!a_mn && !b_mn, "gemm: act is built for K-major operands only");
        B200_REQUIRE((reinterpret_cast<uintptr_t>(a->D) & 15) == 0, "gemm: act needs a 16-byte aligned output (TMA tile stores)");
    }
    if (!a->d_fp32) B200_REQUIRE((a->ldd % 8) == 0, "gemm: bf16 output pitch must be a multiple of 8");
    if (a->resid) B200_REQUIRE((a->ldr % 8) == 0, "gemm: residual pitch must be a multiple of 8");

    CUtensorMap tm[6];
    CUtensorMap &tA = tm[0], &tA2 = tm[1], &tB = tm[2], &tD = tm[3], &tR = tm[4], &tD2 = tm[5];
    int rc;
    const int64_t KA = a->A2 ? a->K1 : a->K;
    if (!a_mn) rc = make_map(&tA, a->A, KA, a->M, a->lda, BM);
    else rc = make_map(&tA, a->A, a->M, a->K, a->lda, BK);
    if (rc) return rc;
    if (a->A2) {
        if (!a_mn) rc = make_map(&tA2, a->A2, a->K - a->K1, a->M, a->lda2, BM);
        else rc = make_map(&tA2, a->A2, a->M, a->K - a->K1, a->lda2, BK);   // second run of K rows of an MN-major A (same M extent and box)
        if (rc) return rc;
    } else {
        tA2 = tA;
    }
    if (!b_mn) rc = make_map(&tB, a->B, a->K, a->N, a->ldb, 128);   // 128-row boxes: one per 128 output columns of the tile
    else rc = make_map(&tB, a->B, a->N, a->K, a->ldb, BK);
    if (rc) return rc;
    if (!a->d_fp32) B200_REQUIRE((reinterpret_cast<uintptr_t>(a->D) & 3) == 0, "gemm: bf16 output must be 4-byte aligned");
    // TMA tile stores and loads need 16-byte aligned bases (every pitch is a multiple of 16 bytes already), and the stores rows of
    // whole 16-byte units: a tile store does not clip the last partial unit of a row at column N, so with N % 8 != 0 it would write
    // the tile's columns past N into the output's padding. Other bf16 outputs store from the fragments, and other residuals are read
    // from global memory next to them.
    const auto a16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    // GLU outputs take the same path when both operands are K-major and h, the pre-activations and glu_mult have 16-byte aligned
    // bases (the producer bulk-copies the tile's bias and glu_mult into shared memory; the bias is 16-byte aligned already). N % 128 == 0 and the pitches are
    // multiples of 8 for every GLU problem.
    p.tma_store = !a->d_fp32 && !a->geglu && a16(a->D) && (p.N % 8) == 0;
    p.resid_tma = p.tma_store && a->resid && a16(a->resid);
    p.glu_tma = a->geglu && !a_mn && !b_mn && a->D2 && a16(a->D) && a16(a->D2) && (!a->glu_mult || a16(a->glu_mult));
    tD = tR = tD2 = tB;   // unused unless set below
    if (p.tma_store && (rc = make_map(&tD, a->D, a->N, a->M, a->ldd, 64))) return rc;
    if (p.resid_tma && (rc = make_map(&tR, a->resid, a->N, a->M, a->ldr, 64))) return rc;
    if (p.glu_tma && (rc = make_map(&tD, a->D, a->N / 2, a->M, a->ldd, 64))) return rc;
    if (p.glu_tma && (rc = make_map(&tD2, a->D2, a->N, a->M, a->ldd2, 64))) return rc;
    if (a->geglu && a->D2) B200_REQUIRE((reinterpret_cast<uintptr_t>(a->D2) & 3) == 0, "gemm: GEGLU pre-activation buffer must be 4-byte aligned");
    if (a->resid) B200_REQUIRE((reinterpret_cast<uintptr_t>(a->resid) & 3) == 0, "gemm: residual must be 4-byte aligned");

    {
        static const bool trace = getenv("B200_GEMM_TRACE") != nullptr;   // developer aid: log every problem shape
        if (trace)
            fprintf(stderr, "GEMMTRACE %d %d %d amn=%d bmn=%d split=%d geglu=%d two=%d mh=%d epi=%d%d%d%d store=%s\n", p.M, p.N, p.K, (int)a_mn,
                    (int)b_mn, split, p.geglu, a->A2 != nullptr, wide ? 3 : MH, p.bias != nullptr, p.colscale != nullptr, p.rowmask != nullptr,
                    p.resid != nullptr, (p.tma_store || p.glu_tma) ? "tma" : "frag");
    }
    if (a->act) {
        if (wide) return launch_gemm<256, false, false, 1, ACT_GELU>(tm, p, st);
        if (MH == 2) return launch_gemm<128, false, false, 2, ACT_GELU>(tm, p, st);
        return launch_gemm<128, false, false, 1, ACT_GELU>(tm, p, st);
    }
    if (wide) {
        if (!a_mn && !b_mn) return launch_gemm<256, false, false, 1>(tm, p, st);
        if (!a_mn && b_mn) return launch_gemm<256, false, true, 1>(tm, p, st);
        if (a_mn && !b_mn) return launch_gemm<256, true, false, 1>(tm, p, st);
        return launch_gemm<256, true, true, 1>(tm, p, st);
    }
    if (MH == 2) {
        if (!a_mn && !b_mn) return launch_gemm<128, false, false, 2>(tm, p, st);
        if (!a_mn && b_mn) return launch_gemm<128, false, true, 2>(tm, p, st);
        if (a_mn && !b_mn) return launch_gemm<128, true, false, 2>(tm, p, st);
        return launch_gemm<128, true, true, 2>(tm, p, st);
    }
    if (!a_mn && !b_mn) return launch_gemm<128, false, false, 1>(tm, p, st);
    if (!a_mn && b_mn) return launch_gemm<128, false, true, 1>(tm, p, st);
    if (a_mn && !b_mn) return launch_gemm<128, true, false, 1>(tm, p, st);
    return launch_gemm<128, true, true, 1>(tm, p, st);
}
