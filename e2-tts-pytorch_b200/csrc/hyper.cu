// Hyper-connection residual-stream kernels (S = 4 streams), fused with the consumer's (adaptive) RMSNorm.
//
// Replaces hyper_connections.HyperConnections as composed by the reference (SURVEY A.5; ctor e2_tts.py:607,
// 673-678, 709-713; calls :870-882, :900-939) together with the x-transformers RMSNorm / AdaptiveRMSNorm that
// consumes the branch input (A.1; :875, :881, :908, :937):
//   width : n^ = RMSNorm_{gamma+1}(r_s);  alpha = tanh(n^ A) * sa + alpha0;  beta = tanh(n^ b) * sb + beta0
//           mix_t = sum_s alpha[s,t] r_s;  branch = mix_0 (optionally normalised);  residual'_t = mix_{t+1}
//   depth : out_s = residual'_s + beta_s * y
// HBM layout: residual streams are (token, stream, d) bf16 so the 4 streams of a token are adjacent (the
// reference's '(b s) n d' puts them N'*d apart). One warp owns one token; all reductions are warp shuffles.
// These kernels are HBM-bound: width reads S*d and writes (S+1)*d bf16 per token (algorithmic minimum).
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int HS = 4;         // residual streams (reference default num_residual_streams = 4, e2_tts.py:547)
constexpr int HT = HS + 1;

struct HcP {
    const __nv_bfloat16* xres;  // [T, S, D]
    const float *gamma, *afn, *ascale, *salpha, *bfn, *bscale, *sbeta;
    int norm_mode;              // 0 none, 1 RMSNorm gain g[D], 2 adaptive gain (1+gamma)[B, D]
    const float* ng;
    int rows_per_batch, T, D;
    __nv_bfloat16 *branch, *res_out;
    float* beta_out;
    // fused preceding depth connection (optional): the streams entering this width connection are xres + beta_prev (x) y_prev and are
    // never materialised in HBM
    float* stats_out;              // forward: [T, 32] per-token reduction results (24 raw dots, branch norm factor, 4 sums of squares)
    const float* stats;            // backward: the same rows
    const __nv_bfloat16* y_prev;   // [T, D]
    const float* beta_prev;        // [T, S]
    __nv_bfloat16* d_y_prev;       // backward outputs of the fused depth connection
    float* d_beta_prev;
    // backward
    const __nv_bfloat16 *d_branch, *d_res;
    const float* d_beta;
    __nv_bfloat16* d_xres;
    float *g_gamma, *g_afn, *g_ascale, *g_salpha, *g_bfn, *g_bscale, *g_sbeta, *g_ng;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Reduce 32 per-lane values across the warp with recursive halving (31 shuffles instead of 160): on return
// lane l holds the warp-wide sum of v[l] in v[0].
template <int N>
__device__ __forceinline__ void warp_halve(float (&v)[32], int lane) {
    constexpr int o = N / 2;
    const bool hi = lane & o;
#pragma unroll
    for (int i = 0; i < o; ++i) {
        const float send = hi ? v[i] : v[i + o];
        const float keep = hi ? v[i + o] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
}
__device__ __forceinline__ float warp_reduce32(float (&v)[32], int lane) {
    warp_halve<32>(v, lane);
    warp_halve<16>(v, lane);
    warp_halve<8>(v, lane);
    warp_halve<4>(v, lane);
    warp_halve<2>(v, lane);
    return v[0];
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}

// fp32x2 pairs (elements 2i, 2i+1 of a bf16x2 word); ffma2 / fmul2 are in ptx.cuh.
typedef float2 f2;
__device__ __forceinline__ f2 splat(float a) { return make_float2(a, a); }
__device__ __forceinline__ float hsum(f2 a) { return a.x + a.y; }
__device__ __forceinline__ void unpack8p(const uint4& u, f2 (&f)[4]) {
    f[0] = make_float2(bf16_lo(u.x), bf16_hi(u.x)); f[1] = make_float2(bf16_lo(u.y), bf16_hi(u.y));
    f[2] = make_float2(bf16_lo(u.z), bf16_hi(u.z)); f[3] = make_float2(bf16_lo(u.w), bf16_hi(u.w));
}
__device__ __forceinline__ uint4 pack8p(const f2 (&f)[4]) {
    return make_uint4(pack_bf16(f[0].x, f[0].y), pack_bf16(f[1].x, f[1].y), pack_bf16(f[2].x, f[2].y), pack_bf16(f[3].x, f[3].y));
}
__device__ __forceinline__ f2 lo2(const float4& q) { return make_float2(q.x, q.y); }
__device__ __forceinline__ f2 hi2(const float4& q) { return make_float2(q.z, q.w); }

// Per-token forward state shared by the forward and backward kernels.
template <int VPT>
struct TokState {
    f2 r[HS][VPT][4];     // the 4 streams, element pairs (2i, 2i+1)
    float inv[HS];        // sqrt(D) / max(||r_s||, 1e-12)
    float alpha[HS][HT];  // broadcast to every lane
    // Lane-owned scalars. Lane l = s*HT + t (l < 20) owns alpha[s][t]; lane 20 + s owns beta[s]:
    float myraw;          //   raw dot product <r_s, (gamma+1) * A[:,t]>  (resp. b) left in this lane by the reduction
    float myinv;          //   inv of the lane's stream
    float myth;           //   tanh(myraw * myinv)
    float myval;          //   alpha[s][t] (resp. beta[s])
};
// token-invariant lane constants: the dynamic scale and static term of the scalar a lane owns
struct LaneConst { float scale, stat; };
__device__ __forceinline__ LaneConst lane_const(const HcP& p, int lane) {
    LaneConst lc;
    lc.scale = lane < HS * HT ? __ldg(p.ascale) : (lane < HS * HT + HS ? __ldg(p.bscale) : 0.f);
    lc.stat = lane < HS * HT ? __ldg(p.salpha + lane) : (lane < HS * HT + HS ? __ldg(p.sbeta + lane - HS * HT) : 0.f);
    return lc;
}

// Stage the per-feature parameters once per block, (gamma+1) folded in, as element PAIRS: for pair j of chunk c
//   part 0 = { A0[e0], A0[e1], A1[e0], A1[e1] },  part 1 = { A2.., A3.. },  part 2 = { A4[e0], A4[e1], b[e0], b[e1] }
// at sp[(j*3 + part) * nchunk + c]: the 32 lanes of a warp (consecutive chunks, same j/part) read 32 consecutive float4 —
// bank-conflict free (a naive per-feature layout is an 8-way conflict). 12 * nchunk float4 = 24 * D bytes.
__device__ __forceinline__ int sp_idx(int nchunk, int chunk, int j, int part) { return (j * 3 + part) * nchunk + chunk; }
__host__ __device__ inline size_t hc_param_smem(int D) { return (size_t)(D / 8) * 12 * sizeof(float4); }
__device__ __forceinline__ void stage_params(const HcP& p, float4* sp) {
    const int nchunk = p.D >> 3;
    for (int pi = threadIdx.x; pi < (p.D >> 1); pi += blockDim.x) {
        const int e0 = 2 * pi, e1 = e0 + 1;
        const float g0 = __ldg(p.gamma + e0) + 1.f, g1 = __ldg(p.gamma + e1) + 1.f;
        const float* a0 = p.afn + e0 * HT;
        const float* a1 = p.afn + e1 * HT;
        const int c = pi >> 2, j = pi & 3;
        sp[sp_idx(nchunk, c, j, 0)] = make_float4(g0 * __ldg(a0), g1 * __ldg(a1), g0 * __ldg(a0 + 1), g1 * __ldg(a1 + 1));
        sp[sp_idx(nchunk, c, j, 1)] = make_float4(g0 * __ldg(a0 + 2), g1 * __ldg(a1 + 2), g0 * __ldg(a0 + 3), g1 * __ldg(a1 + 3));
        sp[sp_idx(nchunk, c, j, 2)] = make_float4(g0 * __ldg(a0 + 4), g1 * __ldg(a1 + 4), g0 * __ldg(p.bfn + e0), g1 * __ldg(p.bfn + e1));
    }
    __syncthreads();
}

// FUSED: r_s = rsrc_s + bprev[s] * ysrc (the depth connection of the previous sub-block, fp32 — one rounding less than the unfused pair)
// STATS: the 24 raw dot products and 4 sums of squares of this token were saved by the forward kernel (32 fp32 per token, lane l owns
// word l) and arrive in `mine`: the backward pass then only LOADS the streams — no 28 x D FMAs, no smem parameter reads, no 32-value
// warp reduction on its critical path (~15 % of its instructions; the kernel is latency-bound with 8-16 warps per SM).
template <int VPT, bool FUSED, bool STATS>
__device__ __forceinline__ void token_forward(const HcP& p, const float4* __restrict__ sp, const __nv_bfloat16* __restrict__ rsrc,
                                              const __nv_bfloat16* __restrict__ ysrc, const float4 bprev, int lane,
                                              const LaneConst& lc, TokState<VPT>& st, float mine = 0.f) {   // rsrc: this token's [HS][D] block (HBM or smem copy)
    const int nchunk = p.D >> 3;
    const float bpv[HS] = {bprev.x, bprev.y, bprev.z, bprev.w};
    f2 ss2[HS], acc[HS][6];
#pragma unroll
    for (int s = 0; s < HS; ++s) {
        ss2[s] = splat(0.f);
#pragma unroll
        for (int k = 0; k < 6; ++k) acc[s][k] = splat(0.f);
    }
#pragma unroll
    for (int v = 0; v < VPT; ++v) {
        const int c = lane + 32 * v;
        if (c < nchunk) {
#pragma unroll
            for (int s = 0; s < HS; ++s) unpack8p(*reinterpret_cast<const uint4*>(rsrc + (size_t)s * p.D + c * 8), st.r[s][v]);
            if constexpr (FUSED) {
                f2 yv[4];
                unpack8p(*reinterpret_cast<const uint4*>(ysrc + c * 8), yv);
#pragma unroll
                for (int s = 0; s < HS; ++s)
#pragma unroll
                    for (int j = 0; j < 4; ++j) st.r[s][v][j] = ffma2(splat(bpv[s]), yv[j], st.r[s][v][j]);
            }
            if constexpr (!STATS)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 q0 = sp[sp_idx(nchunk, c, j, 0)], q1 = sp[sp_idx(nchunk, c, j, 1)], q2 = sp[sp_idx(nchunk, c, j, 2)];
#pragma unroll
                for (int s = 0; s < HS; ++s) {
                    const f2 rp = st.r[s][v][j];
                    ss2[s] = ffma2(rp, rp, ss2[s]);
                    acc[s][0] = ffma2(rp, lo2(q0), acc[s][0]); acc[s][1] = ffma2(rp, hi2(q0), acc[s][1]);
                    acc[s][2] = ffma2(rp, lo2(q1), acc[s][2]); acc[s][3] = ffma2(rp, hi2(q1), acc[s][3]);
                    acc[s][4] = ffma2(rp, lo2(q2), acc[s][4]); acc[s][5] = ffma2(rp, hi2(q2), acc[s][5]);
                }
            }
        } else {
#pragma unroll
            for (int s = 0; s < HS; ++s)
#pragma unroll
                for (int j = 0; j < 4; ++j) st.r[s][v][j] = splat(0.f);
        }
    }
    if constexpr (!STATS) {
        float red[32];
#pragma unroll
        for (int s = 0; s < HS; ++s) {
#pragma unroll
            for (int t = 0; t < HT; ++t) red[s * HT + t] = hsum(acc[s][t]);
            red[HS * HT + s] = hsum(acc[s][5]);
            red[24 + s] = 0.f;
            red[28 + s] = hsum(ss2[s]);   // the four sums of squares ride along in the same reduction
        }
        mine = warp_reduce32(red, lane);         // lane l owns total #l
    }
    const float sqrtD = sqrtf((float)p.D);
    float invs[HS];
#pragma unroll
    for (int s = 0; s < HS; ++s) {
        invs[s] = sqrtD / fmaxf(sqrtf(__shfl_sync(0xffffffffu, mine, 28 + s)), 1e-12f);
        st.inv[s] = invs[s];
    }
    // each lane applies inv_s, tanh, scale and static term to the ONE dot product it owns; only the 20 alphas are broadcast
    float myinv = invs[0];
    {
        const int s_of = lane < HS * HT ? lane / HT : lane - HS * HT;
#pragma unroll
        for (int s = 1; s < HS; ++s) myinv = (s_of == s) ? invs[s] : myinv;
    }
    const float th = tanhf(mine * myinv);
    st.myraw = mine;
    st.myinv = myinv;
    st.myth = th;
    st.myval = th * lc.scale + lc.stat;
#pragma unroll
    for (int s = 0; s < HS; ++s)
#pragma unroll
        for (int t = 0; t < HT; ++t) st.alpha[s][t] = __shfl_sync(0xffffffffu, st.myval, s * HT + t);
}

__device__ __forceinline__ const float* norm_gain(const HcP& p, long long tok) {
    return p.norm_mode == 2 ? p.ng + (size_t)(tok / p.rows_per_batch) * p.D : p.ng;
}
__device__ __forceinline__ void load_gain8(const float* g, f2 (&o)[4]) {   // 8 consecutive fp32 gains (32-byte aligned)
    const float4 a = __ldg(reinterpret_cast<const float4*>(g)), b = __ldg(reinterpret_cast<const float4*>(g) + 1);
    o[0] = lo2(a); o[1] = hi2(a); o[2] = lo2(b); o[3] = hi2(b);
}

// PF: every warp prefetches its NEXT token's 4 streams into a private shared-memory double buffer with one bulk (TMA) copy while
// it works on the current one. Without it the kernel alternates load and math phases with ~8 warps per SM and sits on
// long-scoreboard stalls.
template <int VPT, bool PF, bool FUSED>
__global__ void __launch_bounds__(256, (VPT <= 2) ? 2 : 1) hc_width_fwd_kernel(const HcP p) {
    extern __shared__ float4 sp[];
    __shared__ uint64_t bars[8][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long warp_global = (long long)blockIdx.x * 8 + warp;
    const long long nwarps = (long long)gridDim.x * 8;
    const int nchunk = p.D >> 3;
    // per-warp buffer of one token: [4 streams][D] bf16 (+ FUSED: y [D] bf16, beta_prev 4 x fp32)
    const uint32_t res_bytes = (uint32_t)(HS * p.D * 2), y_bytes = (uint32_t)(p.D * 2);
    const uint32_t tok_bytes = res_bytes + (FUSED ? y_bytes + 16u : 0u);
    uint8_t* wbuf = reinterpret_cast<uint8_t*>(sp) + hc_param_smem(p.D) + (size_t)warp * 2 * tok_bytes;
    auto prefetch = [&](long long tk, int buf) {
        uint8_t* dst = wbuf + (size_t)buf * tok_bytes;
        mbar_arrive_expect_tx(&bars[warp][buf], tok_bytes);
        bulk_load_1d(dst, p.xres + (size_t)tk * HS * p.D, res_bytes, &bars[warp][buf]);
        if constexpr (FUSED) {
            bulk_load_1d(dst + res_bytes, p.y_prev + (size_t)tk * p.D, y_bytes, &bars[warp][buf]);
            bulk_load_1d(dst + res_bytes + y_bytes, p.beta_prev + (size_t)tk * HS, 16u, &bars[warp][buf]);
        }
    };
    if (PF && lane == 0) {
        mbar_init(&bars[warp][0], 1);
        mbar_init(&bars[warp][1], 1);
        fence_barrier_init();
        if (warp_global < p.T) prefetch(warp_global, 0);
    }
    stage_params(p, sp);
    const LaneConst lc = lane_const(p, lane);
    int it = 0;
    for (long long tok = warp_global; tok < p.T; tok += nwarps, ++it) {
        const __nv_bfloat16* rsrc = p.xres + (size_t)tok * HS * p.D;
        const __nv_bfloat16* ysrc = FUSED ? p.y_prev + (size_t)tok * p.D : nullptr;
        const float* bsrc = FUSED ? p.beta_prev + (size_t)tok * HS : nullptr;
        if (PF) {
            const int buf = it & 1;
            const long long nxt = tok + nwarps;
            __syncwarp();   // every lane is done reading the other buffer (previous token)
            if (lane == 0 && nxt < p.T) prefetch(nxt, buf ^ 1);
            mbar_wait(&bars[warp][buf], (uint32_t)(it >> 1) & 1u);
            const uint8_t* src = wbuf + (size_t)buf * tok_bytes;
            rsrc = reinterpret_cast<const __nv_bfloat16*>(src);
            ysrc = reinterpret_cast<const __nv_bfloat16*>(src + res_bytes);
            bsrc = reinterpret_cast<const float*>(src + res_bytes + y_bytes);
        }
        const float4 bprev = FUSED ? *reinterpret_cast<const float4*>(bsrc) : make_float4(0.f, 0.f, 0.f, 0.f);
        TokState<VPT> st;
        token_forward<VPT, FUSED, false>(p, sp, rsrc, ysrc, bprev, lane, lc, st);
        if (p.stats_out && lane != 24) p.stats_out[(size_t)tok * 32 + lane] = st.myraw;   // word 24: the branch norm factor, below
        f2 br[VPT][4];
        f2 bss2 = splat(0.f);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                f2 acc = fmul2(splat(st.alpha[0][0]), st.r[0][v][j]);
#pragma unroll
                for (int s = 1; s < HS; ++s) acc = ffma2(splat(st.alpha[s][0]), st.r[s][v][j], acc);
                br[v][j] = acc;
                bss2 = ffma2(acc, acc, bss2);
            }
            if (c < nchunk) {
#pragma unroll
                for (int t = 1; t < HT; ++t) {
                    f2 o[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        f2 acc = fmul2(splat(st.alpha[0][t]), st.r[0][v][j]);
#pragma unroll
                        for (int s = 1; s < HS; ++s) acc = ffma2(splat(st.alpha[s][t]), st.r[s][v][j], acc);
                        o[j] = acc;
                    }
                    *reinterpret_cast<uint4*>(p.res_out + ((size_t)tok * HS + (t - 1)) * p.D + c * 8) = pack8p(o);
                }
            }
        }
        if (lane >= HS * HT && lane < HS * HT + HS) p.beta_out[(size_t)tok * HS + (lane - HS * HT)] = st.myval;   // lane-owned betas
        float c_norm = 1.f;
        const float* ng = nullptr;
        if (p.norm_mode) {
            c_norm = sqrtf((float)p.D) / fmaxf(sqrtf(warp_sum(hsum(bss2))), 1e-12f);
            ng = norm_gain(p, tok);
        }
        if (p.stats_out && lane == 24) p.stats_out[(size_t)tok * 32 + 24] = c_norm;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
                if (p.norm_mode) {
                    f2 g[4];
                    load_gain8(ng + c * 8, g);
#pragma unroll
                    for (int j = 0; j < 4; ++j) br[v][j] = fmul2(fmul2(br[v][j], splat(c_norm)), g[j]);
                }
                *reinterpret_cast<uint4*>(p.branch + (size_t)tok * p.D + c * 8) = pack8p(br[v]);
            }
        }
    }
}

// Backward:
//   (1) token kernel   : one warp per token — recompute the forward scalars, produce d_xres, the scalar parameter grads, d(norm gain)
//                        (register partial sums, one atomicAdd per column per block) and one bf16 row per (token, stream) of the
//                        coefficient matrix C = inv * d(tanh argument);
//   (2) wgmma GEMM     : G = R^T C over all (token, stream) rows (split-K), then hc_param_finalize_kernel turns G into
//                        d(dynamic_alpha_fn), d(dynamic_beta_fn), d(norm.gamma).
// grid.y = batch element: a block never straddles two batch elements (adaptive-gain gradient is per batch).
// Tokens per block are chosen by the host so that the whole grid is ONE wave of co-resident blocks (hc_tokens_per_block): with a fixed 64
// a grid of just over one wave leaves most of the machine idle in its second round.
// D <= 256 (VPT == 1) fits 128 registers, so two blocks (16 warps) share an SM: the per-token critical path (two warp-wide 32-value
// reductions, tanh, ~70 shuffles) is latency-bound, and at D = 256 the backward took 70 % of the D = 512 time for half the bytes.
// FUSED (preceding depth connection folded in): the streams are recomputed as xres + beta_prev (x) y_prev, and the kernel also emits the
// depth connection's gradients d_y_prev = sum_s beta_prev[s] d_r_s, d_beta_prev[s] = <d_r_s, y_prev> (d_xres is then d(residual') of the
// previous width connection) plus one extra coefficient row per token, C'[t] = sum_s beta_prev[s] C[(t,s)], so that the parameter GEMM
// R^T C = xres^T C + y_prev^T C' needs no materialised R.
template <int VPT, bool PF, bool FUSED>
__global__ void __launch_bounds__(256, (VPT == 1) ? 2 : 1) hc_width_bwd_kernel(const HcP p, __nv_bfloat16* __restrict__ cmat, int tok_per_block) {
    extern __shared__ float4 sp[];
    __shared__ float s_scal[32];
    __shared__ float s_gng[VPT * 256];   // d(norm gain) partial sums of this block (one batch element), VPT*256 >= D
    __shared__ uint64_t bars[8][2];
    if (threadIdx.x < 32) s_scal[threadIdx.x] = 0.f;
    for (int i = threadIdx.x; i < VPT * 256; i += 256) s_gng[i] = 0.f;
    const int D = p.D, nchunk = D >> 3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    const int n0 = blockIdx.x * tok_per_block;
    const int n1 = min(p.rows_per_batch, n0 + tok_per_block);
    // PF: per-warp double buffer {r [HS][D], d_res [HS][D], d_branch [D]} filled by bulk (TMA) copies one token ahead
    const uint32_t tok_bytes = (uint32_t)(HS * D * 2), br_bytes = (uint32_t)(D * 2);
    const uint32_t buf_bytes = 2 * tok_bytes + br_bytes + (FUSED ? br_bytes + 16u : 0u);   // FUSED: + y_prev [D], beta_prev [4] fp32
    uint8_t* wbuf = reinterpret_cast<uint8_t*>(sp) + hc_param_smem(D) + (size_t)warp * 2 * buf_bytes;
    auto prefetch = [&](int n, int buf) {
        const size_t tk = (size_t)b * p.rows_per_batch + n;
        uint8_t* dst = wbuf + (size_t)buf * buf_bytes;
        mbar_arrive_expect_tx(&bars[warp][buf], buf_bytes);
        bulk_load_1d(dst, p.xres + tk * HS * D, tok_bytes, &bars[warp][buf]);
        bulk_load_1d(dst + tok_bytes, p.d_res + tk * HS * D, tok_bytes, &bars[warp][buf]);
        bulk_load_1d(dst + 2 * tok_bytes, p.d_branch + tk * D, br_bytes, &bars[warp][buf]);
        if constexpr (FUSED) {
            bulk_load_1d(dst + 2 * tok_bytes + br_bytes, p.y_prev + tk * D, br_bytes, &bars[warp][buf]);
            bulk_load_1d(dst + 2 * tok_bytes + 2 * br_bytes, p.beta_prev + tk * HS, 16u, &bars[warp][buf]);
        }
    };
    if (PF && lane == 0) {
        mbar_init(&bars[warp][0], 1);
        mbar_init(&bars[warp][1], 1);
        fence_barrier_init();
        if (n0 + warp < n1) prefetch(n0 + warp, 0);
    }
    stage_params(p, sp);
    const LaneConst lc = lane_const(p, lane);
    float g_stat = 0.f, g_scale = 0.f;   // lane-owned: d(static_alpha[l] | static_beta[l-20]) and this lane's share of d(dynamic scale)
    const float invD = 1.f / (float)D;
    f2 gng2[VPT][4];                     // d(norm gain) of this lane's columns, summed over the warp's tokens
#pragma unroll
    for (int v = 0; v < VPT; ++v)
#pragma unroll
        for (int j = 0; j < 4; ++j) gng2[v][j] = splat(0.f);
    // where this lane's coefficient goes in the [T*S, 8] matrix handed to the parameter GEMM: row = stream, column = which tanh argument
    const int c_row = lane < HS * HT ? lane / HT : (lane < HS * HT + HS ? lane - HS * HT : (lane - 24) >> 1);
    const int c_col = lane < HS * HT ? lane % HT : (lane < HS * HT + HS ? HT : 6 + ((lane - 24) & 1));

    int it = 0;
    for (int n = n0 + warp; n < n1; n += 8, ++it) {
        const long long tok = (long long)b * p.rows_per_batch + n;
        const __nv_bfloat16* rsrc = p.xres + (size_t)tok * HS * D;
        const __nv_bfloat16* drsrc = p.d_res + (size_t)tok * HS * D;
        const __nv_bfloat16* dbsrc = p.d_branch + (size_t)tok * D;
        const __nv_bfloat16* ysrc = FUSED ? p.y_prev + (size_t)tok * D : nullptr;
        const float* bsrc = FUSED ? p.beta_prev + (size_t)tok * HS : nullptr;
        const float mystat = __ldg(p.stats + (size_t)tok * 32 + lane);   // issued before the wait for the token's tiles
        if (PF) {
            const int buf = it & 1;
            __syncwarp();   // every lane is done reading the other buffer (previous token)
            if (lane == 0 && n + 8 < n1) prefetch(n + 8, buf ^ 1);
            mbar_wait(&bars[warp][buf], (uint32_t)(it >> 1) & 1u);
            const uint8_t* src = wbuf + (size_t)buf * buf_bytes;
            rsrc = reinterpret_cast<const __nv_bfloat16*>(src);
            drsrc = reinterpret_cast<const __nv_bfloat16*>(src + tok_bytes);
            dbsrc = reinterpret_cast<const __nv_bfloat16*>(src + 2 * tok_bytes);
            ysrc = reinterpret_cast<const __nv_bfloat16*>(src + 2 * tok_bytes + br_bytes);
            bsrc = reinterpret_cast<const float*>(src + 2 * tok_bytes + 2 * br_bytes);
        }
        const float4 bprev = FUSED ? *reinterpret_cast<const float4*>(bsrc) : make_float4(0.f, 0.f, 0.f, 0.f);
        TokState<VPT> st;
        token_forward<VPT, FUSED, true>(p, sp, rsrc, ysrc, bprev, lane, lc, st, mystat);
        const float cn_saved = __shfl_sync(0xffffffffu, mystat, 24);

        // ---- branch (mix_0), its norm, and d(mix_0)
        f2 dm0[VPT][4];
        float cn = 1.f;
        {
            f2 br[VPT][4];
#pragma unroll
            for (int v = 0; v < VPT; ++v) {
                const int c = lane + 32 * v;
                if (c < nchunk) {
                    unpack8p(*reinterpret_cast<const uint4*>(dbsrc + c * 8), dm0[v]);   // dy for now
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) dm0[v][j] = splat(0.f);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    f2 acc = fmul2(splat(st.alpha[0][0]), st.r[0][v][j]);
#pragma unroll
                    for (int s = 1; s < HS; ++s) acc = ffma2(splat(st.alpha[s][0]), st.r[s][v][j], acc);
                    br[v][j] = acc;
                }
            }
            if (p.norm_mode) {
                cn = cn_saved;
                const float* ng = norm_gain(p, tok);
                f2 dot2 = splat(0.f);
#pragma unroll
                for (int v = 0; v < VPT; ++v) {
                    const int c = lane + 32 * v;
                    if (c < nchunk) {
                        f2 g[4];
                        load_gain8(ng + c * 8, g);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            gng2[v][j] = ffma2(fmul2(dm0[v][j], br[v][j]), splat(cn), gng2[v][j]);   // d gain += dy * normalised branch
                            dm0[v][j] = fmul2(g[j], dm0[v][j]);             // gain * dy
                            dot2 = ffma2(dm0[v][j], br[v][j], dot2);
                        }
                    }
                }
                const float dot = warp_sum(hsum(dot2));
                const f2 nk2 = splat(-((cn * cn * invD) * (cn * dot))), cn2 = splat(cn);   // same ordering: finite for an all-zero branch row
#pragma unroll
                for (int v = 0; v < VPT; ++v)
#pragma unroll
                    for (int j = 0; j < 4; ++j) dm0[v][j] = ffma2(dm0[v][j], cn2, fmul2(br[v][j], nk2));   // 0 beyond nchunk
            }
        }
        // ---- d_alpha[s][t] = <d_mix_t, r_s>; start d_r_s = sum_t alpha[s][t] d_mix_t
        f2 dr[HS][VPT][4];
        f2 red2[HS][HT];
#pragma unroll
        for (int s = 0; s < HS; ++s)
#pragma unroll
            for (int t = 0; t < HT; ++t) red2[s][t] = splat(0.f);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
#pragma unroll
            for (int s = 0; s < HS; ++s)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    dr[s][v][j] = fmul2(splat(st.alpha[s][0]), dm0[v][j]);
                    red2[s][0] = ffma2(dm0[v][j], st.r[s][v][j], red2[s][0]);
                }
            if (c < nchunk) {
#pragma unroll
                for (int t = 1; t < HT; ++t) {
                    f2 dm[4];
                    unpack8p(*reinterpret_cast<const uint4*>(drsrc + (size_t)(t - 1) * D + c * 8), dm);
#pragma unroll
                    for (int s = 0; s < HS; ++s)
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            dr[s][v][j] = ffma2(splat(st.alpha[s][t]), dm[j], dr[s][v][j]);
                            red2[s][t] = ffma2(dm[j], st.r[s][v][j], red2[s][t]);
                        }
                }
            }
        }
        float red[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
        for (int s = 0; s < HS; ++s)
#pragma unroll
            for (int t = 0; t < HT; ++t) red[s * HT + t] = hsum(red2[s][t]);
        const float mine = warp_reduce32(red, lane);     // lane s*HT+t owns d_alpha[s][t]; lanes >= 20 hold 0
        // ---- scalar backward, lane-owned (lane l < 20: alpha_l, lane 20+s: beta_s): d(static), d(scale), d(tanh argument)
        const bool is_beta = lane >= HS * HT && lane < HS * HT + HS;
        const float dval = is_beta ? (p.d_beta ? __ldg(p.d_beta + (size_t)tok * HS + (lane - HS * HT)) : 0.f) : mine;
        g_stat += dval;
        g_scale += dval * st.myth;
        const float mycoef = dval * lc.scale * (1.f - st.myth * st.myth);   // d_wc[s][t] (resp. d_dc[s]); 0 in lanes >= 24
        // row s of the coefficient matrix C[tok*S + s][8] = inv_s * { d_wc[s][0..4], d_dc[s], 0, 0 } (bf16): the parameter gradients
        // d(dynamic_alpha_fn | dynamic_beta_fn | norm.gamma) are the GEMM  R^T C  over all (token, stream) rows (see hc_param_finalize)
        cmat[((size_t)tok * HS + c_row) * 8 + c_col] = __float2bfloat16(mycoef * st.myinv);   // lanes >= 24 hold 0
        // ---- through n^ = r * inv * (gamma+1): u_s = sum_k coef[s][k] * P_k (P = the staged (gamma+1)-scaled A / b columns),
        //      d_r_s += inv_s * u_s - r_s * inv_s^3 / D * <u_s, r_s>.  <u_s, r_s> = sum_k coef[s][k] * <P_k, r_s>, and those raw dot
        //      products are what the forward reduction left in lanes 0..23 — no second pass over the features is needed.
        float nk3[HS], cw[HS][6];
        {
            const float term = mycoef * st.myraw;
            const float cws = mycoef * st.myinv;
#pragma unroll
            for (int s = 0; s < HS; ++s) {
                float Rs = __shfl_sync(0xffffffffu, term, HS * HT + s);
                cw[s][5] = __shfl_sync(0xffffffffu, cws, HS * HT + s);
#pragma unroll
                for (int t = 0; t < HT; ++t) {
                    Rs += __shfl_sync(0xffffffffu, term, s * HT + t);
                    cw[s][t] = __shfl_sync(0xffffffffu, cws, s * HT + t);
                }
                // (an all-zero stream has inv = sqrt(D) / 1e-12: inv^3 overflows fp32 and inf * 0 would poison the row — keep the product
                //  ordered so that the zero factor <u, r> is applied before the third power; x-transformers' F.normalize backward is finite too)
                nk3[s] = -((st.inv[s] * st.inv[s] * invD) * (st.inv[s] * Rs));
            }
        }
        const float bpv[HS] = {bprev.x, bprev.y, bprev.z, bprev.w};
        if constexpr (FUSED) {
            // coefficient row of the y_prev operand of the parameter GEMM: C'[tok][k] = sum_s beta_prev[s] * C[(tok, s)][k]  (k < 6, else 0)
            if (lane < 8) {
                float cp = 0.f;
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    const float ck = bpv[0] * cw[0][k] + bpv[1] * cw[1][k] + bpv[2] * cw[2][k] + bpv[3] * cw[3][k];
                    cp = (lane == k) ? ck : cp;
                }
                cmat[((size_t)p.T * HS + (size_t)tok) * 8 + lane] = __float2bfloat16(cp);
            }
        }
        f2 dbp[HS];   // FUSED: <d_r_s, y_prev> partial sums of this lane
#pragma unroll
        for (int s = 0; s < HS; ++s) dbp[s] = splat(0.f);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 q0 = sp[sp_idx(nchunk, c, j, 0)], q1 = sp[sp_idx(nchunk, c, j, 1)], q2 = sp[sp_idx(nchunk, c, j, 2)];
#pragma unroll
                    for (int s = 0; s < HS; ++s) {
                        f2 acc = ffma2(st.r[s][v][j], splat(nk3[s]), dr[s][v][j]);
                        acc = ffma2(splat(cw[s][0]), lo2(q0), acc); acc = ffma2(splat(cw[s][1]), hi2(q0), acc);
                        acc = ffma2(splat(cw[s][2]), lo2(q1), acc); acc = ffma2(splat(cw[s][3]), hi2(q1), acc);
                        acc = ffma2(splat(cw[s][4]), lo2(q2), acc); acc = ffma2(splat(cw[s][5]), hi2(q2), acc);
                        dr[s][v][j] = acc;
                    }
                }
#pragma unroll
                for (int s = 0; s < HS; ++s)
                    *reinterpret_cast<uint4*>(p.d_xres + ((size_t)tok * HS + s) * D + c * 8) = pack8p(dr[s][v]);
                if constexpr (FUSED) {
                    f2 yv[4], dy[4];
                    unpack8p(*reinterpret_cast<const uint4*>(ysrc + c * 8), yv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        dy[j] = fmul2(splat(bpv[0]), dr[0][v][j]);
                        dbp[0] = ffma2(dr[0][v][j], yv[j], dbp[0]);
#pragma unroll
                        for (int s = 1; s < HS; ++s) {
                            dy[j] = ffma2(splat(bpv[s]), dr[s][v][j], dy[j]);
                            dbp[s] = ffma2(dr[s][v][j], yv[j], dbp[s]);
                        }
                    }
                    *reinterpret_cast<uint4*>(p.d_y_prev + (size_t)tok * D + c * 8) = pack8p(dy);
                }
            }
        }
        if constexpr (FUSED) {
            float d0 = warp_sum(hsum(dbp[0])), d1 = warp_sum(hsum(dbp[1])), d2 = warp_sum(hsum(dbp[2])), d3 = warp_sum(hsum(dbp[3]));
            if (lane == 0) *reinterpret_cast<float4*>(p.d_beta_prev + (size_t)tok * HS) = make_float4(d0, d1, d2, d3);
        }
    }
    if (p.norm_mode) {
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    atomicAdd(&s_gng[c * 8 + 2 * j], gng2[v][j].x);
                    atomicAdd(&s_gng[c * 8 + 2 * j + 1], gng2[v][j].y);
                }
            }
        }
    }
    {
        if (lane < HS * HT + HS) atomicAdd(&s_scal[lane], g_stat);   // [0,20) static_alpha, [20,24) static_beta
        const float gas = warp_sum(lane < HS * HT ? g_scale : 0.f);
        const float gbs = warp_sum((lane >= HS * HT && lane < HS * HT + HS) ? g_scale : 0.f);
        if (lane == 0) {
            atomicAdd(&s_scal[24], gas);
            atomicAdd(&s_scal[25], gbs);
        }
    }
    __syncthreads();
    if (threadIdx.x < 20) atomicAdd(p.g_salpha + threadIdx.x, s_scal[threadIdx.x]);
    else if (threadIdx.x < 24) atomicAdd(p.g_sbeta + (threadIdx.x - 20), s_scal[threadIdx.x]);
    else if (threadIdx.x == 24) atomicAdd(p.g_ascale, s_scal[24]);
    else if (threadIdx.x == 25) atomicAdd(p.g_bscale, s_scal[25]);
    if (p.norm_mode) {
        float* dst = p.g_ng + (p.norm_mode == 2 ? (size_t)b * D : 0);
        for (int i = threadIdx.x; i < D; i += 256) atomicAdd(dst + i, s_gng[i]);
    }
}

// Parameter gradients from G[col][k] = sum_{token, stream} r[token, stream, col] * C[(token, stream)][k]  (fp32 [D, 8], produced by the
// wgmma GEMM  R^T C):  with n^ = r * inv * (gamma + 1) and C = inv * d(tanh argument),
//   d dynamic_alpha_fn[col][t] = (gamma+1) G[col][t],  d dynamic_beta_fn[col] = (gamma+1) G[col][5],
//   d norm.gamma[col]          = sum_t alpha_fn[col][t] G[col][t] + beta_fn[col] G[col][5].
// (The first versions marched 128-token slabs per thread pair on the CUDA cores: 48 us per call against ~15 us for the GEMM.)
__global__ void __launch_bounds__(256) hc_param_finalize_kernel(const HcP p, const float* __restrict__ G) {
    const int col = blockIdx.x * 256 + threadIdx.x;
    if (col >= p.D) return;
    const float4 g0 = *reinterpret_cast<const float4*>(G + (size_t)col * 8), g1v = *reinterpret_cast<const float4*>(G + (size_t)col * 8 + 4);
    const float g[6] = {g0.x, g0.y, g0.z, g0.w, g1v.x, g1v.y};
    const float gp1 = __ldg(p.gamma + col) + 1.f;
    float dgam = __ldg(p.bfn + col) * g[5];
#pragma unroll
    for (int t = 0; t < HT; ++t) {
        p.g_afn[col * HT + t] += gp1 * g[t];
        dgam += __ldg(p.afn + col * HT + t) * g[t];
    }
    p.g_bfn[col] += gp1 * g[5];
    p.g_gamma[col] += dgam;
}

// ------------------------------------------------------------------------------------------------ depth
struct HdP {
    const __nv_bfloat16 *res, *y;
    const float* beta;
    __nv_bfloat16* out;
    int T, D;
    const __nv_bfloat16* d_out;
    __nv_bfloat16* d_y;
    float* d_beta;
};

// out[t,s,:] = res[t,s,:] + beta[t,s] * y[t,:]     (one 16-byte chunk of y per thread, all 4 streams)
__global__ void __launch_bounds__(256) hc_depth_fwd_kernel(const HdP p) {
    const int nchunk = p.D >> 3;
    const long long total = (long long)p.T * nchunk;
    for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (long long)gridDim.x * 256) {
        const long long tok = idx / nchunk;
        const int c = (int)(idx % nchunk);
        float y[8];
        unpack8(*reinterpret_cast<const uint4*>(p.y + (size_t)tok * p.D + c * 8), y);
        const float4 be = *reinterpret_cast<const float4*>(p.beta + (size_t)tok * HS);
        const float bes[HS] = {be.x, be.y, be.z, be.w};
#pragma unroll
        for (int s = 0; s < HS; ++s) {
            float r[8];
            const size_t off = ((size_t)tok * HS + s) * p.D + c * 8;
            unpack8(*reinterpret_cast<const uint4*>(p.res + off), r);
#pragma unroll
            for (int e = 0; e < 8; ++e) r[e] += bes[s] * y[e];
            *reinterpret_cast<uint4*>(p.out + off) = pack8(r);
        }
    }
}

// d_y[t,:] = sum_s beta[t,s] d_out[t,s,:];  d_beta[t,s] = <d_out[t,s,:], y[t,:]>   (one warp per token)
__global__ void __launch_bounds__(256) hc_depth_bwd_kernel(const HdP p) {
    const int lane = threadIdx.x & 31;
    const int nchunk = p.D >> 3;
    const long long nwarps = (long long)gridDim.x * 8;
    for (long long tok = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); tok < p.T; tok += nwarps) {
        const float4 be = *reinterpret_cast<const float4*>(p.beta + (size_t)tok * HS);
        const float bes[HS] = {be.x, be.y, be.z, be.w};
        float db[HS] = {0.f, 0.f, 0.f, 0.f};
        for (int c = lane; c < nchunk; c += 32) {
            float y[8], dy[8];
            unpack8(*reinterpret_cast<const uint4*>(p.y + (size_t)tok * p.D + c * 8), y);
#pragma unroll
            for (int e = 0; e < 8; ++e) dy[e] = 0.f;
#pragma unroll
            for (int s = 0; s < HS; ++s) {
                float d[8];
                unpack8(*reinterpret_cast<const uint4*>(p.d_out + ((size_t)tok * HS + s) * p.D + c * 8), d);
#pragma unroll
                for (int e = 0; e < 8; ++e) { dy[e] += bes[s] * d[e]; db[s] += d[e] * y[e]; }
            }
            *reinterpret_cast<uint4*>(p.d_y + (size_t)tok * p.D + c * 8) = pack8(dy);
        }
#pragma unroll
        for (int s = 0; s < HS; ++s) db[s] = warp_sum(db[s]);
        if (lane == 0) *reinterpret_cast<float4*>(p.d_beta + (size_t)tok * HS) = make_float4(db[0], db[1], db[2], db[3]);
    }
}

// the dynamic shared-memory ceiling of a token kernel depends on D, which a process may vary between calls (text / audio streams):
// raise it once per (kernel instantiation, device) to the kernel's maximum instead of per call (SURVEY §8b: once_flag-guarded init)
template <auto kern>          // the kernel is a template VALUE: instantiations that share a function type still get their own flag
static int set_smem(size_t bytes) {
    static DeviceOnce once;
    constexpr int kMax = 200 * 1024;
    B200_REQUIRE(bytes <= (size_t)kMax, "hyper-connections: %zu B of shared memory exceed the kernel's ceiling", bytes);
    cudaError_t e = set_max_smem_once(once, kern, kMax);
    B200_REQUIRE(e == cudaSuccess, "hyper-connections: cudaFuncSetAttribute(%d B): %s", kMax, cudaGetErrorString(e));
    return 0;
}

static int fill_hc(HcP& p, const b200_hc_width_args* a) {
    B200_REQUIRE(a->num_streams == HS, "hyper-connections: only num_residual_streams=4 is built (got %d)", a->num_streams);
    B200_REQUIRE(a->D >= 8 && (a->D % 8) == 0 && a->D <= 1024, "hyper-connections: D=%d must be a multiple of 8 and <= 1024", a->D);
    B200_REQUIRE(a->T > 0 && a->rows_per_batch > 0 && (a->T % a->rows_per_batch) == 0, "hyper-connections: T must be a multiple of rows_per_batch");
    B200_REQUIRE(a->norm_mode >= 0 && a->norm_mode <= 2 && (a->norm_mode == 0 || a->norm_gain), "hyper-connections: bad norm mode");
    p.xres = (const __nv_bfloat16*)a->xres;
    p.gamma = a->norm_gamma; p.afn = a->dynamic_alpha_fn; p.ascale = a->dynamic_alpha_scale; p.salpha = a->static_alpha;
    p.bfn = a->dynamic_beta_fn; p.bscale = a->dynamic_beta_scale; p.sbeta = a->static_beta;
    p.norm_mode = a->norm_mode; p.ng = a->norm_gain; p.rows_per_batch = a->rows_per_batch; p.T = a->T; p.D = a->D;
    if (a->y_prev) {
        B200_REQUIRE(a->beta_prev, "hyper-connections: fused depth connection needs beta_prev next to y_prev");
        B200_REQUIRE((reinterpret_cast<uintptr_t>(a->y_prev) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->beta_prev) & 15) == 0,
                     "hyper-connections: y_prev / beta_prev must be 16-byte aligned");
        p.y_prev = (const __nv_bfloat16*)a->y_prev; p.beta_prev = a->beta_prev;
    }
    return 0;
}

}  // namespace b200

using namespace b200;

template <bool FUSED>
static int launch_hc_fwd(const HcP& p, const b200_hc_width_args* a, cudaStream_t st) {
    const size_t smem_par = hc_param_smem(a->D);
    if (a->D <= 512) {
        // prefetching variant: 2 blocks per SM, each warp owns a double buffer of one token {4 streams (+ y_prev, beta_prev)}
        const size_t tok = (size_t)HS * a->D * 2 + (FUSED ? (size_t)a->D * 2 + 16 : 0);
        const size_t smem = smem_par + 8 * 2 * tok;
        const int grid = (int)min((long long)(a->T + 7) / 8, (long long)num_sms() * 2);
        if (a->D <= 256) {
            if (int rc = set_smem<hc_width_fwd_kernel<1, true, FUSED>>(smem)) return rc;
            hc_width_fwd_kernel<1, true, FUSED><<<grid, 256, smem, st>>>(p);
        } else {
            if (int rc = set_smem<hc_width_fwd_kernel<2, true, FUSED>>(smem)) return rc;
            hc_width_fwd_kernel<2, true, FUSED><<<grid, 256, smem, st>>>(p);
        }
        return check_launch("hc_width_fwd_kernel");
    }
    const int grid = (int)min((long long)(a->T + 7) / 8, (long long)num_sms() * 8);
    if (a->D <= 256) hc_width_fwd_kernel<1, false, FUSED><<<grid, 256, smem_par, st>>>(p);
    else if (a->D <= 512) hc_width_fwd_kernel<2, false, FUSED><<<grid, 256, smem_par, st>>>(p);
    else hc_width_fwd_kernel<4, false, FUSED><<<grid, 256, smem_par, st>>>(p);
    return check_launch("hc_width_fwd_kernel");
}

extern "C" int b200_hc_width_fwd(const b200_hc_width_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->xres && a->branch && a->res_out && a->beta_out, "hc_width_fwd: null pointer");
    HcP p{};
    if (fill_hc(p, a)) return -1;
    p.branch = (__nv_bfloat16*)a->branch; p.res_out = (__nv_bfloat16*)a->res_out; p.beta_out = a->beta_out;
    p.stats_out = a->stats_out;
    return a->y_prev ? launch_hc_fwd<true>(p, a, st) : launch_hc_fwd<false>(p, a, st);
}

template <bool FUSED>
static int launch_hc_bwd(const HcP& p, const b200_hc_width_args* a, __nv_bfloat16* cmat, cudaStream_t st) {
    // one wave: as many blocks per batch element as fit the co-resident slots (8 warps x >= 1 token each), tokens rounded up to the warp count
    const int nbatch = a->T / a->rows_per_batch;
    const int slots = num_sms() * (a->D <= 256 ? 2 : 1);
    int per_batch = slots / nbatch > 0 ? slots / nbatch : 1;
    int tpb = (a->rows_per_batch + per_batch - 1) / per_batch;
    tpb = (tpb + 7) / 8 * 8;
    if (tpb < 32) tpb = 32;                     // amortise the per-block parameter staging
    dim3 grid((a->rows_per_batch + tpb - 1) / tpb, nbatch);
    const size_t smem_par = hc_param_smem(a->D);
    if (a->D <= 512) {
        // + per-warp {r, d_res, d_branch (, y_prev, beta_prev)} double buffers
        const size_t smem = smem_par + (size_t)8 * 2 * ((2 * HS + 1 + (FUSED ? 1 : 0)) * a->D * 2 + (FUSED ? 16 : 0));
        if (a->D <= 256) {
            if (int rc = set_smem<hc_width_bwd_kernel<1, true, FUSED>>(smem)) return rc;
            hc_width_bwd_kernel<1, true, FUSED><<<grid, 256, smem, st>>>(p, cmat, tpb);
        } else {
            if (int rc = set_smem<hc_width_bwd_kernel<2, true, FUSED>>(smem)) return rc;
            hc_width_bwd_kernel<2, true, FUSED><<<grid, 256, smem, st>>>(p, cmat, tpb);
        }
    } else if (a->D <= 256) hc_width_bwd_kernel<1, false, FUSED><<<grid, 256, smem_par, st>>>(p, cmat, tpb);
    else if (a->D <= 512) hc_width_bwd_kernel<2, false, FUSED><<<grid, 256, smem_par, st>>>(p, cmat, tpb);
    else hc_width_bwd_kernel<4, false, FUSED><<<grid, 256, smem_par, st>>>(p, cmat, tpb);
    return check_launch("hc_width_bwd_kernel");
}

extern "C" int b200_hc_width_bwd(const b200_hc_width_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->xres && a->d_branch && a->d_res && a->d_xres && a->g_norm_gamma && a->g_dynamic_alpha_fn && a->g_dynamic_alpha_scale &&
                 a->g_static_alpha && a->g_dynamic_beta_fn && a->g_dynamic_beta_scale && a->g_static_beta, "hc_width_bwd: null pointer");
    HcP p{};
    if (fill_hc(p, a)) return -1;
    B200_REQUIRE(a->norm_mode == 0 || a->g_norm_gain, "hc_width_bwd: missing gain gradient buffer");
    const bool fused = a->y_prev != nullptr;
    if (fused) {
        B200_REQUIRE(a->d_y_prev && a->d_beta_prev, "hc_width_bwd: fused depth connection needs d_y_prev and d_beta_prev");
        B200_REQUIRE(((int64_t)a->T * HS) % 64 == 0, "hc_width_bwd: fused depth connection needs T * S to be a multiple of 64 (T=%lld)", (long long)a->T);
        p.d_y_prev = (__nv_bfloat16*)a->d_y_prev; p.d_beta_prev = a->d_beta_prev;
    }
    p.d_branch = (const __nv_bfloat16*)a->d_branch; p.d_res = (const __nv_bfloat16*)a->d_res; p.d_beta = a->d_beta;
    p.d_xres = (__nv_bfloat16*)a->d_xres;
    p.g_gamma = a->g_norm_gamma; p.g_afn = a->g_dynamic_alpha_fn; p.g_ascale = a->g_dynamic_alpha_scale; p.g_salpha = a->g_static_alpha;
    p.g_bfn = a->g_dynamic_beta_fn; p.g_bscale = a->g_dynamic_beta_scale; p.g_sbeta = a->g_static_beta; p.g_ng = a->g_norm_gain;
    B200_REQUIRE(a->stats, "hc_width_bwd: the per-token reduction results saved by b200_hc_width_fwd (stats_out) are required");
    p.stats = a->stats;
    // workspace: coefficient matrix C bf16 [T*S (+ T fused rows), 8] (80 B per token), then G fp32 [D, 8] at byte offset 80 T
    // (16-byte aligned: finalize reads G as float4)
    B200_REQUIRE(a->ws_records && (reinterpret_cast<uintptr_t>(a->ws_records) & 15) == 0,
                 "hc_width_bwd: missing or misaligned workspace (T * 20 + D * 8 floats, 16-byte aligned)");
    __nv_bfloat16* cmat = reinterpret_cast<__nv_bfloat16*>(a->ws_records);
    float* G = a->ws_records + (size_t)a->T * 20;
    if (int rc = fused ? launch_hc_bwd<true>(p, a, cmat, st) : launch_hc_bwd<false>(p, a, cmat, st)) return rc;
    // G = R^T C on the tensor cores: A = residual streams [T*S, D] read MN-major (fused: followed by y_prev [T, D] against the C' rows),
    // B = C [T*S (+ T), 8] MN-major, split-K over the tokens
    b200_gemm_args g = {};
    g.A = a->xres; g.lda = a->D; g.a_mn_major = 1;
    g.B = cmat; g.ldb = 8; g.b_mn_major = 1;
    g.M = a->D; g.N = 8; g.K = (int64_t)a->T * HS;
    if (fused) { g.A2 = a->y_prev; g.lda2 = a->D; g.K1 = g.K; g.K += a->T; }
    g.D = G; g.ldd = 8; g.d_fp32 = 1;
    const int tiles = (a->D + 255) / 256;
    g.split_k = num_sms() / tiles > 1 ? num_sms() / tiles : 2;   // >= 2: the split-K path zeroes and accumulates G
    if (int rc = b200_gemm(&g, stream)) return rc;
    hc_param_finalize_kernel<<<(a->D + 255) / 256, 256, 0, st>>>(p, G);
    return check_launch("hc_param_finalize_kernel");
}

extern "C" int b200_hc_depth_fwd(const b200_hc_depth_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->res && a->y && a->beta && a->out, "hc_depth_fwd: null pointer");
    B200_REQUIRE(a->num_streams == HS && a->D % 8 == 0 && a->T > 0, "hc_depth_fwd: unsupported shape");
    HdP p{};
    p.res = (const __nv_bfloat16*)a->res; p.y = (const __nv_bfloat16*)a->y; p.beta = a->beta; p.out = (__nv_bfloat16*)a->out; p.T = a->T; p.D = a->D;
    const long long total = (long long)a->T * (a->D / 8);
    const int grid = (int)min((total + 255) / 256, (long long)num_sms() * 16);
    hc_depth_fwd_kernel<<<grid, 256, 0, st>>>(p);
    return check_launch("hc_depth_fwd_kernel");
}

extern "C" int b200_hc_depth_bwd(const b200_hc_depth_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->y && a->beta && a->d_out && a->d_y && a->d_beta, "hc_depth_bwd: null pointer");
    B200_REQUIRE(a->num_streams == HS && a->D % 8 == 0 && a->T > 0, "hc_depth_bwd: unsupported shape");
    HdP p{};
    p.y = (const __nv_bfloat16*)a->y; p.beta = a->beta; p.T = a->T; p.D = a->D;
    p.d_out = (const __nv_bfloat16*)a->d_out; p.d_y = (__nv_bfloat16*)a->d_y; p.d_beta = a->d_beta;
    const int grid = (int)min((long long)(a->T + 7) / 8, (long long)num_sms() * 8);
    hc_depth_bwd_kernel<<<grid, 256, 0, st>>>(p);
    return check_launch("hc_depth_bwd_kernel");
}
