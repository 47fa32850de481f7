// Fused softclamped multi-head attention (head_dim 64) for the E2-TTS multistream block, forward and backward.
//
// Replaces x-transformers Attend as the reference uses it (SURVEY A.4 steps 4-5; e2_tts.py:875,911):
//   sim = q k^T / sqrt(dh);  sim = 50*tanh(sim/50);  key-padding mask;  fp32 softmax;  dropout;  out = P v;
//   out *= sigmoid(head gate)   — without ever materialising the (B,h,N',N') score tensor.
// Flash-style tiling: 64 queries x 64 keys per step, online softmax in fp32 registers, bf16 mma.sync
// m16n8k16 tensor-core tiles fed by cp.async double-buffered, XOR-swizzled shared memory.
// Backward = recompute: a per-row prep kernel (dO = dOg*gate, delta = <dO,O>, d_gate), a dQ kernel
// (query-stationary) and a dK/dV kernel (key-stationary), including the (1 - tanh^2) softclamp factor.
// NOTE (DESIGN.md): these mma.sync kernels were the bring-up path. The product path is the wgmma kernels in attn_tc.cu;
// the entry points here are `*_legacy`: cross-checks for the tests, and the online-softmax fallback of b200_attn_fwd for
// softclamp values > 64 (the wgmma forward exponentiates without a running maximum). attn_bwd_prep_kernel is shared.
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int AT = 64;          // tile edge (queries per block, keys per step)
constexpr int AD = 64;          // head dim
constexpr int TILE_B = AT * AD * 2;  // 8 KB
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ uint32_t swz(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// load a 64 x 64 bf16 tile (rows row0.. of a [nrows, 64] matrix) into swizzled smem; rows >= nrows are zero-filled
__device__ __forceinline__ void load_tile(uint32_t sdst, const __nv_bfloat16* base, int row0, int nrows, int tid) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int idx = tid + i * 128;
        const int r = idx >> 3, c = idx & 7;
        const bool ok = (row0 + r) < nrows;
        const __nv_bfloat16* src = base + (size_t)(ok ? (row0 + r) : 0) * AD + c * 8;
        cp_async16(sdst + swz(r, c), src, ok);
    }
}
// A-operand fragments (16 rows x 64) for the 4 k-steps, rows [r0, r0+16) of a swizzled tile
__device__ __forceinline__ void load_a_frags(uint32_t stile, int r0, int lane, uint32_t (&a)[4][4]) {
    const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) ldsm4(stile + swz(row, ks * 2 + (lane >> 4)), a[ks][0], a[ks][1], a[ks][2], a[ks][3]);
}
// acc[nt] (16 x 64, 8 n-tiles) += A(16 x 64 over d) * T^T where T is a swizzled [64 rows][64 d] tile (rows become columns)
__device__ __forceinline__ void mma_a_tileT(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t stile, int lane) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            uint32_t b0, b1, b2, b3;
            const int row = np * 16 + (lane & 7) + (lane >> 4) * 8;
            ldsm4(stile + swz(row, ks * 2 + ((lane >> 3) & 1)), b0, b1, b2, b3);
            mma16816(acc[np * 2], a[ks], b0, b1);
            mma16816(acc[np * 2 + 1], a[ks], b2, b3);
        }
    }
}
// acc[dt] (16 x 64 over d) += P(16 x 64 over tile rows, as packed A fragments) * T where T is a swizzled [64 rows][64 d] tile
__device__ __forceinline__ void mma_p_tile(float (&acc)[8][4], const uint32_t (&pa)[4][4], uint32_t stile, int lane) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int dp = 0; dp < 4; ++dp) {
            uint32_t b0, b1, b2, b3;
            const int row = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
            ldsm4t(stile + swz(row, dp * 2 + (lane >> 4)), b0, b1, b2, b3);
            mma16816(acc[dp * 2], pa[kk], b0, b1);
            mma16816(acc[dp * 2 + 1], pa[kk], b2, b3);
        }
    }
}
__device__ __forceinline__ void pack_p(const float (&s)[8][4], uint32_t (&pa)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        pa[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
        pa[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
        pa[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pa[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
    }
}

struct AttnP {
    const __nv_bfloat16 *q, *k, *v;
    const unsigned char* keymask;
    const float* gate;
    __nv_bfloat16 *o, *og;
    float* lse;
    int B, H, Np;
    float scale, clamp, inv_clamp, dropout_p, keep_scale;
    unsigned int drop_thresh; int drop_stride;
    unsigned long long seed;
    const unsigned long long* seed_dev;
    // backward
    const __nv_bfloat16 *dog, *dO;
    const float* delta;
    float* dgate;
    __nv_bfloat16 *dq, *dk, *dv, *dO_out;
    float* delta_out;
};

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnP p) {
    pdl_wait();   // no global access before the previous kernel of the stream has completed (ptx.cuh)
    extern __shared__ __align__(128) uint8_t sm[];
    const uint32_t sQ = smem_u32(sm), sK = sQ + TILE_B, sV = sK + 2 * TILE_B;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const size_t head_off = ((size_t)b * p.H + hh) * p.Np * AD;
    const __nv_bfloat16 *Q = p.q + head_off, *K = p.k + head_off, *V = p.v + head_off;
    const unsigned char* km = p.keymask ? p.keymask + (size_t)b * p.Np : nullptr;
    const int nkt = (p.Np + AT - 1) / AT;

    load_tile(sQ, Q, qt * AT, p.Np, tid);
    load_tile(sK, K, 0, p.Np, tid);
    load_tile(sV, V, 0, p.Np, tid);
    cp_async_commit();

    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    uint32_t aq[4][4];
    const int qrow0 = qt * AT + warp * 16 + g, qrow1 = qrow0 + 8;
    const unsigned long long drop_base0 = (((unsigned long long)b * p.H + hh) * p.Np + qrow0) * (unsigned long long)p.drop_stride;
    const unsigned long long drop_base1 = drop_base0 + 8ull * p.drop_stride;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile(sK + (buf ^ 1) * TILE_B, K, (kt + 1) * AT, p.Np, tid);
            load_tile(sV + (buf ^ 1) * TILE_B, V, (kt + 1) * AT, p.Np, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (kt == 0) load_a_frags(sQ, warp * 16, lane, aq);

        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
        mma_a_tileT(s, aq, sK + buf * TILE_B, lane);

        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int key = kt * AT + nt * 8 + 2 * t + e;
                const bool ok = key < p.Np && (!km || km[key]);
                float a0 = p.clamp * tanh_fast(s[nt][e] * p.scale * p.inv_clamp);
                float a1 = p.clamp * tanh_fast(s[nt][2 + e] * p.scale * p.inv_clamp);
                a0 = ok ? a0 : -INFINITY;
                a1 = ok ? a1 : -INFINITY;
                s[nt][e] = a0; s[nt][2 + e] = a1;
                mx0 = fmaxf(mx0, a0); mx1 = fmaxf(mx1, a1);
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
        const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
        const float c0 = exp2f((m0 - ms0) * LOG2E), c1 = exp2f((m1 - ms1) * LOG2E);
        m0 = mn0; m1 = mn1;
        l0 *= c0; l1 *= c1;
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) { o[dt][0] *= c0; o[dt][1] *= c0; o[dt][2] *= c1; o[dt][3] *= c1; }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float p0 = exp2f((s[nt][e] - ms0) * LOG2E), p1 = exp2f((s[nt][2 + e] - ms1) * LOG2E);
                l0 += p0; l1 += p1;
                if (p.dropout_p > 0.f) {
                    const unsigned long long key = (unsigned long long)(kt * AT + nt * 8 + 2 * t + e);
                    p0 = dropout_keep16(p.seed + (p.seed_dev ? __ldg(p.seed_dev) : 0ull), drop_base0 + key, p.drop_thresh) ? p0 * p.keep_scale : 0.f;
                    p1 = dropout_keep16(p.seed + (p.seed_dev ? __ldg(p.seed_dev) : 0ull), drop_base1 + key, p.drop_thresh) ? p1 * p.keep_scale : 0.f;
                }
                s[nt][e] = p0; s[nt][2 + e] = p1;
            }
        }
        uint32_t pa[4][4];
        pack_p(s, pa);
        mma_p_tile(o, pa, sV + buf * TILE_B, lane);
        __syncthreads();
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
    if (t == 0) {
        if (qrow0 < p.Np) p.lse[((size_t)b * p.H + hh) * p.Np + qrow0] = m0 + logf(l0);
        if (qrow1 < p.Np) p.lse[((size_t)b * p.H + hh) * p.Np + qrow1] = m1 + logf(l1);
    }
    // stage O through smem (Q tile region is free now) for 16-byte coalesced stores
    uint8_t* so = sm;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
        const int r0 = warp * 16 + g, r1 = r0 + 8, ch = dt, off = (2 * t) * 2;
        *reinterpret_cast<uint32_t*>(so + swz(r0, ch) + off) = pack_bf16(o[dt][0] * inv0, o[dt][1] * inv0);
        *reinterpret_cast<uint32_t*>(so + swz(r1, ch) + off) = pack_bf16(o[dt][2] * inv1, o[dt][3] * inv1);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int idx = tid + i * 128, r = idx >> 3, c = idx & 7;
        const int n = qt * AT + r;
        if (n >= p.Np) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(so + swz(r, c));
        *reinterpret_cast<uint4*>(p.o + head_off + (size_t)n * AD + c * 8) = u;
        const float gt = p.gate ? p.gate[((size_t)b * p.Np + n) * p.H + hh] : 1.f;
        uint4 w;
        w.x = pack_bf16(bf16_lo(u.x) * gt, bf16_hi(u.x) * gt); w.y = pack_bf16(bf16_lo(u.y) * gt, bf16_hi(u.y) * gt);
        w.z = pack_bf16(bf16_lo(u.z) * gt, bf16_hi(u.z) * gt); w.w = pack_bf16(bf16_lo(u.w) * gt, bf16_hi(u.w) * gt);
        *reinterpret_cast<uint4*>(p.og + ((size_t)b * p.Np + n) * (size_t)(p.H * AD) + hh * AD + c * 8) = w;
    }
}

// ------------------------------------------------------------------------------------------------ backward prep
// one 8-lane group per (b, h, n): dO = dOg * gate, d_gate = <dOg, O>, delta = gate * d_gate
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const AttnP p) {
    pdl_wait();   // no global access before the previous kernel of the stream has completed (ptx.cuh)
    const long long gidx = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long rowid = gidx >> 3;
    const int c = (int)(gidx & 7);
    const long long total = (long long)p.B * p.H * p.Np;
    const bool ok = rowid < total;
    float dot = 0.f, gt = 1.f;
    long long b = 0, hh = 0, n = 0;
    if (ok) {
        n = rowid % p.Np; hh = (rowid / p.Np) % p.H; b = rowid / ((long long)p.Np * p.H);
        const uint4 dg = *reinterpret_cast<const uint4*>(p.dog + ((size_t)b * p.Np + n) * (size_t)(p.H * AD) + hh * AD + c * 8);
        const uint4 ov = *reinterpret_cast<const uint4*>(p.o + (size_t)rowid * AD + c * 8);
        gt = p.gate ? p.gate[((size_t)b * p.Np + n) * p.H + hh] : 1.f;
        const uint32_t dgv[4] = {dg.x, dg.y, dg.z, dg.w}, ovv[4] = {ov.x, ov.y, ov.z, ov.w};
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float a0 = bf16_lo(dgv[i]), a1 = bf16_hi(dgv[i]);
            dot += a0 * bf16_lo(ovv[i]) + a1 * bf16_hi(ovv[i]);
            w[i] = pack_bf16(a0 * gt, a1 * gt);
        }
        *reinterpret_cast<uint4*>(p.dO_out + (size_t)rowid * AD + c * 8) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    dot += __shfl_xor_sync(0xffffffffu, dot, 4);
    if (ok && c == 0) {
        p.delta_out[rowid] = dot * gt;
        if (p.dgate) p.dgate[((size_t)b * p.Np + n) * p.H + hh] = dot;
    }
}

// shared logic: recompute clamped logits / probabilities for a 16x64 accumulator block
// ------------------------------------------------------------------------------------------------ dQ
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const AttnP p) {
    pdl_wait();   // no global access before the previous kernel of the stream has completed (ptx.cuh)
    extern __shared__ __align__(128) uint8_t sm[];
    const uint32_t sQ = smem_u32(sm), sDO = sQ + TILE_B, sK = sDO + TILE_B, sV = sK + 2 * TILE_B;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const size_t bh = (size_t)b * p.H + hh;
    const size_t head_off = bh * p.Np * AD;
    const __nv_bfloat16 *Q = p.q + head_off, *K = p.k + head_off, *V = p.v + head_off, *DO = p.dO + head_off;
    const unsigned char* km = p.keymask ? p.keymask + (size_t)b * p.Np : nullptr;
    const int nkt = (p.Np + AT - 1) / AT;

    load_tile(sQ, Q, qt * AT, p.Np, tid);
    load_tile(sDO, DO, qt * AT, p.Np, tid);
    load_tile(sK, K, 0, p.Np, tid);
    load_tile(sV, V, 0, p.Np, tid);
    cp_async_commit();

    const int qrow0 = qt * AT + warp * 16 + g, qrow1 = qrow0 + 8;
    const float lse0 = qrow0 < p.Np ? p.lse[bh * p.Np + qrow0] : 0.f, lse1 = qrow1 < p.Np ? p.lse[bh * p.Np + qrow1] : 0.f;
    const float dl0 = qrow0 < p.Np ? p.delta[bh * p.Np + qrow0] : 0.f, dl1 = qrow1 < p.Np ? p.delta[bh * p.Np + qrow1] : 0.f;
    const unsigned long long drop_base0 = (bh * p.Np + qrow0) * (unsigned long long)p.drop_stride, drop_base1 = drop_base0 + 8ull * p.drop_stride;

    float dq[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }
    uint32_t aq[4][4], ado[4][4];

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile(sK + (buf ^ 1) * TILE_B, K, (kt + 1) * AT, p.Np, tid);
            load_tile(sV + (buf ^ 1) * TILE_B, V, (kt + 1) * AT, p.Np, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (kt == 0) { load_a_frags(sQ, warp * 16, lane, aq); load_a_frags(sDO, warp * 16, lane, ado); }

        float s[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
        mma_a_tileT(s, aq, sK + buf * TILE_B, lane);
        mma_a_tileT(dp, ado, sV + buf * TILE_B, lane);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kt * AT + nt * 8 + 2 * t + (e & 1);
                const bool ok = key < p.Np && (!km || km[key]);
                const float th = tanh_fast(s[nt][e] * p.scale * p.inv_clamp);
                const float sc = p.clamp * th;
                const float lse = (e < 2) ? lse0 : lse1, dl = (e < 2) ? dl0 : dl1;
                const float pr = ok ? exp2f((sc - lse) * LOG2E) : 0.f;
                float dpe = dp[nt][e];
                if (p.dropout_p > 0.f) {
                    const unsigned long long base = (e < 2) ? drop_base0 : drop_base1;
                    dpe = dropout_keep16(p.seed + (p.seed_dev ? __ldg(p.seed_dev) : 0ull), base + (unsigned long long)key, p.drop_thresh) ? dpe * p.keep_scale : 0.f;
                }
                s[nt][e] = pr * (dpe - dl) * (1.f - th * th) * p.scale;
            }
        }
        uint32_t pa[4][4];
        pack_p(s, pa);
        mma_p_tile(dq, pa, sK + buf * TILE_B, lane);
        __syncthreads();
    }
    uint8_t* so = sm;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
        const int r0 = warp * 16 + g, r1 = r0 + 8, off = (2 * t) * 2;
        *reinterpret_cast<uint32_t*>(so + swz(r0, dt) + off) = pack_bf16(dq[dt][0], dq[dt][1]);
        *reinterpret_cast<uint32_t*>(so + swz(r1, dt) + off) = pack_bf16(dq[dt][2], dq[dt][3]);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int idx = tid + i * 128, r = idx >> 3, c = idx & 7, n = qt * AT + r;
        if (n < p.Np) *reinterpret_cast<uint4*>(p.dq + head_off + (size_t)n * AD + c * 8) = *reinterpret_cast<const uint4*>(so + swz(r, c));
    }
}

// ------------------------------------------------------------------------------------------------ dK, dV
__global__ void __launch_bounds__(128) attn_bwd_dkv_kernel(const AttnP p) {
    pdl_wait();   // no global access before the previous kernel of the stream has completed (ptx.cuh)
    extern __shared__ __align__(128) uint8_t sm[];
    const uint32_t sK = smem_u32(sm), sV = sK + TILE_B, sQ = sV + TILE_B, sDO = sQ + 2 * TILE_B;
    float* s_lse = reinterpret_cast<float*>(sm + 6 * TILE_B);   // [2][64]
    float* s_dl = s_lse + 2 * AT;                               // [2][64]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int kb = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
    const size_t bh = (size_t)b * p.H + hh;
    const size_t head_off = bh * p.Np * AD;
    const __nv_bfloat16 *Q = p.q + head_off, *K = p.k + head_off, *V = p.v + head_off, *DO = p.dO + head_off;
    const unsigned char* km = p.keymask ? p.keymask + (size_t)b * p.Np : nullptr;
    const int nqt = (p.Np + AT - 1) / AT;

    auto load_q_stage = [&](int qt, int buf) {
        load_tile(sQ + buf * TILE_B, Q, qt * AT, p.Np, tid);
        load_tile(sDO + buf * TILE_B, DO, qt * AT, p.Np, tid);
        if (tid < AT) {
            const int n = qt * AT + tid;
            s_lse[buf * AT + tid] = n < p.Np ? p.lse[bh * p.Np + n] : 0.f;
            s_dl[buf * AT + tid] = n < p.Np ? p.delta[bh * p.Np + n] : 0.f;
        }
    };
    load_tile(sK, K, kb * AT, p.Np, tid);
    load_tile(sV, V, kb * AT, p.Np, tid);
    load_q_stage(0, 0);
    cp_async_commit();

    const int key0 = kb * AT + warp * 16 + g, key1 = key0 + 8;
    const bool kok0 = key0 < p.Np && (!km || km[key0]), kok1 = key1 < p.Np && (!km || km[key1]);
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }
    uint32_t ak[4][4], av[4][4];

    for (int qt = 0; qt < nqt; ++qt) {
        const int buf = qt & 1;
        if (qt + 1 < nqt) {
            load_q_stage(qt + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (qt == 0) { load_a_frags(sK, warp * 16, lane, ak); load_a_frags(sV, warp * 16, lane, av); }

        float s[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
        mma_a_tileT(s, ak, sQ + buf * TILE_B, lane);     // S^T[key, query]
        mma_a_tileT(dp, av, sDO + buf * TILE_B, lane);   // dP^T[key, query]
        float pd[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ql = nt * 8 + 2 * t + (e & 1);
                const int qn = qt * AT + ql;
                const bool ok = ((e < 2) ? kok0 : kok1) && qn < p.Np;
                const float th = tanh_fast(s[nt][e] * p.scale * p.inv_clamp);
                const float sc = p.clamp * th;
                float pr = ok ? exp2f((sc - s_lse[buf * AT + ql]) * LOG2E) : 0.f;
                float dpe = dp[nt][e];
                float prd = pr;
                if (p.dropout_p > 0.f) {
                    const unsigned long long idx = (bh * p.Np + (unsigned long long)qn) * (unsigned long long)p.drop_stride + (unsigned long long)((e < 2) ? key0 : key1);
                    const bool keep = dropout_keep16(p.seed + (p.seed_dev ? __ldg(p.seed_dev) : 0ull), idx, p.drop_thresh);
                    dpe = keep ? dpe * p.keep_scale : 0.f;
                    prd = keep ? pr * p.keep_scale : 0.f;
                }
                pd[nt][e] = prd;
                s[nt][e] = pr * (dpe - s_dl[buf * AT + ql]) * (1.f - th * th) * p.scale;
            }
        }
        uint32_t pa[4][4];
        pack_p(pd, pa);
        mma_p_tile(dv, pa, sDO + buf * TILE_B, lane);    // dV += P^T dO
        pack_p(s, pa);
        mma_p_tile(dk, pa, sQ + buf * TILE_B, lane);     // dK += dS^T Q
        __syncthreads();
    }
    // stage through smem (sQ/sDO stage 0 regions) for coalesced stores
    uint8_t* so_k = sm + 2 * TILE_B;
    uint8_t* so_v = sm + 4 * TILE_B;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
        const int r0 = warp * 16 + g, r1 = r0 + 8, off = (2 * t) * 2;
        *reinterpret_cast<uint32_t*>(so_k + swz(r0, dt) + off) = pack_bf16(dk[dt][0], dk[dt][1]);
        *reinterpret_cast<uint32_t*>(so_k + swz(r1, dt) + off) = pack_bf16(dk[dt][2], dk[dt][3]);
        *reinterpret_cast<uint32_t*>(so_v + swz(r0, dt) + off) = pack_bf16(dv[dt][0], dv[dt][1]);
        *reinterpret_cast<uint32_t*>(so_v + swz(r1, dt) + off) = pack_bf16(dv[dt][2], dv[dt][3]);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int idx = tid + i * 128, r = idx >> 3, c = idx & 7, n = kb * AT + r;
        if (n < p.Np) {
            *reinterpret_cast<uint4*>(p.dk + head_off + (size_t)n * AD + c * 8) = *reinterpret_cast<const uint4*>(so_k + swz(r, c));
            *reinterpret_cast<uint4*>(p.dv + head_off + (size_t)n * AD + c * 8) = *reinterpret_cast<const uint4*>(so_v + swz(r, c));
        }
    }
}

static int fill_common(AttnP& p, int B, int H, int Np, float scale, float clamp, float dropout_p, uint64_t seed, const uint64_t* seed_dev) {
    B200_REQUIRE(B > 0 && H > 0 && Np > 0, "attention: empty problem");
    B200_REQUIRE(B <= 65535 && H <= 65535, "attention: batch/heads exceed grid limits");
    B200_REQUIRE(clamp > 0.f, "attention: softclamp value must be > 0 (reference always clamps, e2_tts.py:548-551)");
    B200_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention: dropout must be in [0,1)");
    p.B = B; p.H = H; p.Np = Np; p.scale = scale; p.clamp = clamp; p.inv_clamp = 1.f / clamp;
    p.dropout_p = dropout_p; p.seed = seed; p.seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
    p.drop_thresh = (unsigned int)(dropout_p * 65536.f);
    p.keep_scale = 65536.f / (65536.f - (float)p.drop_thresh);
    p.drop_stride = (Np + 1) & ~1;
    return 0;
}

}  // namespace b200

using namespace b200;

// mma.sync forward (bring-up kernel): kept as a cross-check for the wgmma forward in attn_tc.cu.
extern "C" int b200_attn_fwd_legacy(const b200_attn_fwd_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->q && a->k && a->v && a->o && a->og && a->lse, "attn_fwd: null pointer");
    B200_REQUIRE(a->dim_head == 64, "attn_fwd: only dim_head 64 is built (got %d)", a->dim_head);
    AttnP p{};
    if (fill_common(p, a->B, a->H, a->Np, a->scale, a->softclamp, a->dropout_p, a->seed, a->seed_dev)) return -1;
    p.q = (const __nv_bfloat16*)a->q; p.k = (const __nv_bfloat16*)a->k; p.v = (const __nv_bfloat16*)a->v;
    p.keymask = a->keymask; p.gate = a->gate; p.o = (__nv_bfloat16*)a->o; p.og = (__nv_bfloat16*)a->og; p.lse = a->lse;
    dim3 grid((a->Np + AT - 1) / AT, a->H, a->B);
    B200_LAUNCH(attn_fwd_kernel, grid, 128, 5 * TILE_B, st, p);
    return check_launch("attn_fwd_kernel");
}

namespace b200 {
int launch_attn_bwd_prep(const b200_attn_bwd_args* a, cudaStream_t st) {
    AttnP p{};
    if (fill_common(p, a->B, a->H, a->Np, a->scale, a->softclamp, a->dropout_p, a->seed, a->seed_dev)) return -1;
    p.gate = a->gate; p.o = (__nv_bfloat16*)a->o; p.dog = (const __nv_bfloat16*)a->d_og; p.dO_out = (__nv_bfloat16*)a->ws_dO;
    p.delta_out = a->ws_delta; p.dgate = a->d_gate;
    const long long rows = (long long)a->B * a->H * a->Np;
    B200_LAUNCH(attn_bwd_prep_kernel, (unsigned)((rows * 8 + 255) / 256), 256, 0, st, p);
    return check_launch("attn_bwd_prep_kernel");
}
}  // namespace b200

// mma.sync backward (bring-up kernels, dq/dk/dv all bf16): kept as a cross-check for the wgmma backward.
extern "C" int b200_attn_bwd_legacy(const b200_attn_bwd_args* a, b200_stream_t stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B200_REQUIRE(a && a->q && a->k && a->v && a->o && a->d_og && a->lse && a->ws_dO && a->ws_delta && a->dq && a->dk && a->dv, "attn_bwd: null pointer");
    B200_REQUIRE(a->dim_head == 64, "attn_bwd: only dim_head 64 is built (got %d)", a->dim_head);
    AttnP p{};
    if (fill_common(p, a->B, a->H, a->Np, a->scale, a->softclamp, a->dropout_p, a->seed, a->seed_dev)) return -1;
    p.q = (const __nv_bfloat16*)a->q; p.k = (const __nv_bfloat16*)a->k; p.v = (const __nv_bfloat16*)a->v;
    p.keymask = a->keymask; p.gate = a->gate; p.o = (__nv_bfloat16*)a->o; p.lse = const_cast<float*>(a->lse);
    p.dog = (const __nv_bfloat16*)a->d_og; p.dO_out = (__nv_bfloat16*)a->ws_dO; p.delta_out = a->ws_delta; p.dgate = a->d_gate;
    p.dO = (const __nv_bfloat16*)a->ws_dO; p.delta = a->ws_delta;
    p.dq = (__nv_bfloat16*)a->dq; p.dk = (__nv_bfloat16*)a->dk; p.dv = (__nv_bfloat16*)a->dv;
    const long long rows = (long long)a->B * a->H * a->Np;
    B200_LAUNCH(attn_bwd_prep_kernel, (unsigned)((rows * 8 + 255) / 256), 256, 0, st, p);
    if (int rc = check_launch("attn_bwd_prep_kernel")) return rc;
    dim3 grid((a->Np + AT - 1) / AT, a->H, a->B);
    static DeviceOnce once_dkv, once_dq;
    B200_REQUIRE(set_max_smem_once(once_dkv, attn_bwd_dkv_kernel, 6 * TILE_B + 1024) == cudaSuccess &&
                 set_max_smem_once(once_dq, attn_bwd_dq_kernel, 6 * TILE_B) == cudaSuccess, "attn_bwd_legacy: cudaFuncSetAttribute failed");
    B200_LAUNCH(attn_bwd_dq_kernel, grid, 128, 6 * TILE_B, st, p);
    if (int rc = check_launch("attn_bwd_dq_kernel")) return rc;
    B200_LAUNCH(attn_bwd_dkv_kernel, grid, 128, 6 * TILE_B + 1024, st, p);
    return check_launch("attn_bwd_dkv_kernel");
}
