// HBM-bound fused kernels around the GEMM/attention core of the E2-TTS block: weight packing, the
// flow-matching stem (noise interpolation + cond masking), residual-stream assembly (abs-pos, registers,
// stream expand), rotary + value-residual + head-gate post-processing of the QKV projection, GEGLU backward,
// bias column sums, the final stream-reduce + RMSNorm, and the masked-MSE flow loss.
// All loads/stores are 16-byte vectorised and coalesced along the feature dimension.
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// ------------------------------------------------------------------------------------------------ weight packing
// One launch casts/permutes every fp32 nn.Parameter that feeds a tensor-core GEMM into its packed bf16 slot.
__device__ __forceinline__ int pack_row(const b200_pack_desc& d, int r) {
    if (d.mode != 1) return r;  // mode 1 = GEGLU interleave: [u(inner) ; gate(inner)] -> per 64 hidden units [u(64) | gate(64)]
    const int inner = d.rows >> 1;
    return r < inner ? (r >> 6) * 128 + (r & 63) : ((r - inner) >> 6) * 128 + 64 + ((r - inner) & 63);
}
__global__ void __launch_bounds__(256) pack_weights_kernel(const b200_pack_desc* descs) {
    const b200_pack_desc d = descs[blockIdx.y];
    if ((d.cols & 3) || (d.col_off & 3) || (d.ld_dst & 3)) {  // scalar path (1-D biases, odd widths)
        const long long total = (long long)d.rows * d.cols;
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
            const int r = (int)(i / d.cols), c = (int)(i % d.cols);
            const float v = d.src[i];
            const size_t off = (size_t)(d.row_off + pack_row(d, r)) * d.ld_dst + d.col_off + c;
            if (d.out_fp32) reinterpret_cast<float*>(d.dst)[off] = v;
            else reinterpret_cast<__nv_bfloat16*>(d.dst)[off] = __float2bfloat16(v);
        }
        return;
    }
    const long long total4 = ((long long)d.rows * d.cols) >> 2;
    const int c4 = d.cols >> 2;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total4; i += (long long)gridDim.x * 256) {
        const int r = (int)(i / c4), c = (int)(i % c4) * 4;
        const float4 v = *reinterpret_cast<const float4*>(d.src + (size_t)r * d.cols + c);
        const size_t off = (size_t)(d.row_off + pack_row(d, r)) * d.ld_dst + d.col_off + c;
        if (d.out_fp32) *reinterpret_cast<float4*>(reinterpret_cast<float*>(d.dst) + off) = v;
        else *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(d.dst) + off) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
    }
}

// ------------------------------------------------------------------------------------------------ stem
// A[row, 0:C] = w = (1-t) x0 + t x1 (or x given), A[row, Cp:Cp+C] = cond = span ? 0 : x1 (or cond given); pads are zero.
struct StemP {
    const float *x1, *x0, *times, *xin, *condin;
    const unsigned char* span;
    __nv_bfloat16* A;
    float* cond_out;
    int B, N, C, Cp;
    int concat;   // != 0: columns [0, C) = cond, [C, 2C) = x  (cat(cond, x), e2_tts.py:1265)
};
__global__ void __launch_bounds__(256) stem_prepare_kernel(const StemP p) {
    const long long total = (long long)p.B * p.N * p.Cp * 2;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int col = (int)(i % (2 * p.Cp));
        const long long row = i / (2 * p.Cp);
        int half = col / p.Cp, c = col % p.Cp;
        bool valid = c < p.C;
        if (p.concat) {
            valid = col < 2 * p.C;
            half = col < p.C ? 1 : 0;
            c = col < p.C ? col : col - p.C;
        }
        float v = 0.f;
        if (valid) {
            const size_t src = (size_t)row * p.C + c;
            if (p.xin) {
                v = half == 0 ? p.xin[src] : p.condin[src];
            } else {
                const float a = p.x1[src];
                if (half == 0) {
                    const float t = p.times[row / p.N];
                    v = (1.f - t) * p.x0[src] + t * a;
                } else {
                    v = p.span[row] ? 0.f : a;
                    if (p.cond_out) p.cond_out[src] = v;
                }
            }
        }
        p.A[i] = __float2bfloat16(v);
    }
}

// ------------------------------------------------------------------------------------------------ assemble
struct AsmP {
    const __nv_bfloat16* h;      // [B*N, D] or null
    const int* ids;              // [B, N] or null (embedding gather, fp32 table)
    const float *emb, *abs_pos, *registers;
    __nv_bfloat16* out;          // [B, R+N, S, D]
    int B, N, R, D, S;
    const __nv_bfloat16* d_out;
    __nv_bfloat16* d_h;
    float *d_tok, *d_abs_pos, *d_registers;
};
__global__ void __launch_bounds__(256) assemble_fwd_kernel(const AsmP p) {
    const int nchunk = p.D >> 3;
    const long long total = (long long)p.B * (p.R + p.N) * nchunk;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int c = (int)(i % nchunk);
        const long long tok = i / nchunk;
        const int n = (int)(tok % (p.R + p.N));
        const int b = (int)(tok / (p.R + p.N));
        float v[8];
        if (n < p.R) {
            const float4 a = *reinterpret_cast<const float4*>(p.registers + (size_t)n * p.D + c * 8);
            const float4 bq = *reinterpret_cast<const float4*>(p.registers + (size_t)n * p.D + c * 8 + 4);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = bq.x; v[5] = bq.y; v[6] = bq.z; v[7] = bq.w;
        } else {
            const int nn = n - p.R;
            if (p.h) {
                unpack8(*reinterpret_cast<const uint4*>(p.h + ((size_t)b * p.N + nn) * p.D + c * 8), v);
            } else {
                const int id = p.ids[(size_t)b * p.N + nn];
                const float* e = p.emb + (size_t)id * p.D + c * 8;
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = e[k];
            }
            if (p.abs_pos) {
                const float* a = p.abs_pos + (size_t)nn * p.D + c * 8;
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] += a[k];
            }
        }
        const uint4 u = pack8(v);
        for (int s = 0; s < p.S; ++s) *reinterpret_cast<uint4*>(p.out + ((size_t)tok * p.S + s) * p.D + c * 8) = u;
    }
}
// thread per (position, chunk): loops over batch; sums the S stream gradients
__global__ void __launch_bounds__(256) assemble_bwd_kernel(const AsmP p) {
    const int nchunk = p.D >> 3;
    const long long total = (long long)(p.R + p.N) * nchunk;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % nchunk), n = (int)(i / nchunk);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int b = 0; b < p.B; ++b) {
        float sum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const size_t tok = (size_t)b * (p.R + p.N) + n;
        for (int s = 0; s < p.S; ++s) {
            float v[8];
            unpack8(*reinterpret_cast<const uint4*>(p.d_out + (tok * p.S + s) * p.D + c * 8), v);
#pragma unroll
            for (int k = 0; k < 8; ++k) sum[k] += v[k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += sum[k];
        if (n >= p.R) {
            const size_t row = (size_t)b * p.N + (n - p.R);
            if (p.d_h) *reinterpret_cast<uint4*>(p.d_h + row * p.D + c * 8) = pack8(sum);
            if (p.d_tok) {
#pragma unroll
                for (int k = 0; k < 8; ++k) p.d_tok[row * p.D + c * 8 + k] = sum[k];
            }
        }
    }
    float* dst = n < p.R ? (p.d_registers ? p.d_registers + (size_t)n * p.D + c * 8 : nullptr)
                         : (p.d_abs_pos ? p.d_abs_pos + (size_t)(n - p.R) * p.D + c * 8 : nullptr);
    if (dst) {
#pragma unroll
        for (int k = 0; k < 8; ++k) dst[k] = acc[k];
    }
}
// embedding gradient: grid (vocab row, token slab); a block scans its slab for its id and adds its partial row
// (the hot filler id 0 is spread over all slabs instead of one serial block). d_emb is zeroed by the host wrapper.
__global__ void __launch_bounds__(256) embed_bwd_kernel(const float* d_tok, const int* ids, float* d_emb, int ntok, int D, int slab) {
    const int v = blockIdx.x;
    const int t0 = blockIdx.y * slab, t1 = min(ntok, t0 + slab);
    __shared__ int hits[256];
    __shared__ int nhit;
    for (int base = t0; base < t1; base += 256) {
        if (threadIdx.x == 0) nhit = 0;
        __syncthreads();
        const int t = base + threadIdx.x;
        if (t < t1 && ids[t] == v) hits[atomicAdd(&nhit, 1)] = t;
        __syncthreads();
        const int nh = nhit;
        for (int c = threadIdx.x; c < D; c += 256) {
            float acc = 0.f;
            for (int j = 0; j < nh; ++j) acc += d_tok[(size_t)hits[j] * D + c];
            if (nh) atomicAdd(d_emb + (size_t)v * D + c, acc);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ rotary table
__global__ void rotary_table_kernel(float* cs, float* sn, int Np, int half) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Np * half) return;
    const int n = i / half, j = i % half;
    const float inv = powf(10000.f, -(float)(2 * j) / (float)(2 * half));
    float s, c;
    sincosf((float)n * inv, &s, &c);
    cs[i] = c; sn[i] = s;
}

// ------------------------------------------------------------------------------------------------ qkv post
// qkvg [T, ld] = [q(I) | k(I) | v(I) | gate(h) | mix(h)] (raw GEMM output), or [q | k | v | mix(h)] without the head gate
// (no_gate), I = H * DH. Produces rotated q,k and the value-residual-mixed v in [B,H,Np,DH] (A.3, A.4 steps 1-3), plus sigmoid(head
// gate) [T,H] fp32. One DH / 8-lane group per (token, head), 8 elements (4 rotary pairs) per lane; the rotary table is [Np, DH / 2].
struct QkvP {
    const __nv_bfloat16* qkvg; int ld;
    const float *gate_b, *mix_b, *cs, *sn;
    const __nv_bfloat16* v_first;
    __nv_bfloat16 *q, *k, *v;
    float* gate;
    int B, H, Np;
    // backward
    const __nv_bfloat16 *dq, *dk, *dv, *dv_extra;
    const float* d_gate;
    __nv_bfloat16 *d_qkvg, *d_vfirst;
    int dq_fp32;
    int no_gate;
};
template <int DH>
__global__ void __launch_bounds__(256) qkv_post_fwd_kernel(const QkvP p) {
    constexpr int LANES = DH / 8, LOG2_LANES = DH == 64 ? 3 : 4;
    static_assert(LANES == 1 << LOG2_LANES, "head dim 64 or 128");
    const long long total = (long long)p.B * p.Np * p.H * LANES;
    const int I = p.H * DH;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int c = (int)(i & (LANES - 1));
        const int hh = (int)((i >> LOG2_LANES) % p.H);
        const long long tok = (i >> LOG2_LANES) / p.H;
        const int n = (int)(tok % p.Np), b = (int)(tok / p.Np);
        const __nv_bfloat16* row = p.qkvg + (size_t)tok * p.ld;
        const size_t dst = (((size_t)b * p.H + hh) * p.Np + n) * DH + c * 8;
        float cs[4], sn[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { cs[j] = p.cs[n * (DH / 2) + c * 4 + j]; sn[j] = p.sn[n * (DH / 2) + c * 4 + j]; }
        float x[8], y[8];
        unpack8(*reinterpret_cast<const uint4*>(row + hh * DH + c * 8), x);
#pragma unroll
        for (int j = 0; j < 4; ++j) { y[2 * j] = x[2 * j] * cs[j] - x[2 * j + 1] * sn[j]; y[2 * j + 1] = x[2 * j + 1] * cs[j] + x[2 * j] * sn[j]; }
        *reinterpret_cast<uint4*>(p.q + dst) = pack8(y);
        unpack8(*reinterpret_cast<const uint4*>(row + I + hh * DH + c * 8), x);
#pragma unroll
        for (int j = 0; j < 4; ++j) { y[2 * j] = x[2 * j] * cs[j] - x[2 * j + 1] * sn[j]; y[2 * j + 1] = x[2 * j + 1] * cs[j] + x[2 * j] * sn[j]; }
        *reinterpret_cast<uint4*>(p.k + dst) = pack8(y);
        unpack8(*reinterpret_cast<const uint4*>(row + 2 * I + hh * DH + c * 8), x);
        if (p.v_first) {
            const float mix = sigmoidf_(__bfloat162float(row[3 * I + (p.no_gate ? 0 : p.H) + hh]) + p.mix_b[hh]);
            float vf[8];
            unpack8(*reinterpret_cast<const uint4*>(p.v_first + dst), vf);
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] = x[j] * mix + vf[j] * (1.f - mix);
        }
        *reinterpret_cast<uint4*>(p.v + dst) = pack8(x);
        if (c == 0 && !p.no_gate) p.gate[(size_t)tok * p.H + hh] = sigmoidf_(__bfloat162float(row[3 * I + hh]) + p.gate_b[hh]);
    }
}
template <int DH>
__global__ void __launch_bounds__(256) qkv_post_bwd_kernel(const QkvP p) {
    constexpr int LANES = DH / 8, LOG2_LANES = DH == 64 ? 3 : 4;
    static_assert(LANES == 1 << LOG2_LANES, "head dim 64 or 128");
    const long long total = (long long)p.B * p.Np * p.H * LANES;
    const int I = p.H * DH;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const bool ok = i < total;
    float dmix = 0.f, mix = 0.f;
    int c = 0, hh = 0;
    long long tok = 0;
    if (ok) {
        c = (int)(i & (LANES - 1));
        hh = (int)((i >> LOG2_LANES) % p.H);
        tok = (i >> LOG2_LANES) / p.H;
        const int n = (int)(tok % p.Np), b = (int)(tok / p.Np);
        const __nv_bfloat16* row = p.qkvg + (size_t)tok * p.ld;
        __nv_bfloat16* drow = p.d_qkvg + (size_t)tok * p.ld;
        const size_t src = (((size_t)b * p.H + hh) * p.Np + n) * DH + c * 8;
        float cs[4], sn[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { cs[j] = p.cs[n * (DH / 2) + c * 4 + j]; sn[j] = p.sn[n * (DH / 2) + c * 4 + j]; }
        float x[8], y[8];
        if (p.dq_fp32) {
            const float4 a0 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.dq) + src);
            const float4 a1 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.dq) + src + 4);
            x[0] = a0.x; x[1] = a0.y; x[2] = a0.z; x[3] = a0.w; x[4] = a1.x; x[5] = a1.y; x[6] = a1.z; x[7] = a1.w;
        } else {
            unpack8(*reinterpret_cast<const uint4*>(p.dq + src), x);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { y[2 * j] = x[2 * j] * cs[j] + x[2 * j + 1] * sn[j]; y[2 * j + 1] = x[2 * j + 1] * cs[j] - x[2 * j] * sn[j]; }
        *reinterpret_cast<uint4*>(drow + hh * DH + c * 8) = pack8(y);
        unpack8(*reinterpret_cast<const uint4*>(p.dk + src), x);
#pragma unroll
        for (int j = 0; j < 4; ++j) { y[2 * j] = x[2 * j] * cs[j] + x[2 * j + 1] * sn[j]; y[2 * j + 1] = x[2 * j + 1] * cs[j] - x[2 * j] * sn[j]; }
        *reinterpret_cast<uint4*>(drow + I + hh * DH + c * 8) = pack8(y);
        unpack8(*reinterpret_cast<const uint4*>(p.dv + src), x);
        if (p.dv_extra) {
            float xe[8];
            unpack8(*reinterpret_cast<const uint4*>(p.dv_extra + src), xe);
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] += xe[j];
        }
        if (p.v_first) {
            mix = sigmoidf_(__bfloat162float(row[3 * I + (p.no_gate ? 0 : p.H) + hh]) + p.mix_b[hh]);
            float vr[8], vf[8], o[8];
            unpack8(*reinterpret_cast<const uint4*>(row + 2 * I + hh * DH + c * 8), vr);
            unpack8(*reinterpret_cast<const uint4*>(p.v_first + src), vf);
#pragma unroll
            for (int j = 0; j < 8; ++j) { dmix += x[j] * (vr[j] - vf[j]); o[j] = x[j] * (1.f - mix); x[j] *= mix; }
            *reinterpret_cast<uint4*>(p.d_vfirst + src) = pack8(o);
        }
        *reinterpret_cast<uint4*>(drow + 2 * I + hh * DH + c * 8) = pack8(x);
    }
#pragma unroll
    for (int m = 1; m < LANES; m <<= 1) dmix += __shfl_xor_sync(0xffffffffu, dmix, m);
    if (ok && c == 0) {
        __nv_bfloat16* drow = p.d_qkvg + (size_t)tok * p.ld;
        if (!p.no_gate) {
            const float g = p.gate[(size_t)tok * p.H + hh];
            drow[3 * I + hh] = __float2bfloat16(p.d_gate[(size_t)tok * p.H + hh] * g * (1.f - g));
        }
        const int mix_col = 3 * I + (p.no_gate ? 0 : p.H);
        if (p.v_first) drow[mix_col + hh] = __float2bfloat16(dmix * mix * (1.f - mix));
        // zero the pad columns (ld may exceed 3I + 2H) so that dW / colsum of the packed matrix stay clean
        if (hh == 0) {
            const int used = mix_col + (p.v_first ? p.H : 0);
            for (int j = used; j < p.ld; ++j) drow[j] = __float2bfloat16(0.f);
        }
    }
}

// ------------------------------------------------------------------------------------------------ GLU backward
// ug packed [T, 2*inner] ([u(64)|gate(64)] per 128 columns), dh [T, inner] -> dug packed; the bias gradient of the GLU
// projection (column sums of dug, packed order) is accumulated in the same pass (db must be zeroed by the caller), and with MULT the
// gradient of the hidden-unit multiplier (dmult[c] += sum_rows drop(dh) u act(g), zeroed by the caller, may be NULL).
// ACT: 1 exact erf GELU, 2 SiLU, 3 ReLU^2 (the activation codes of b200_gemm's GLU epilogue).
constexpr int GB_ROWS = 256;   // rows per block (8 row lanes x 32)
template <int ACT, bool MULT>
__global__ void __launch_bounds__(256) glu_bwd_kernel(const __nv_bfloat16* dh, const __nv_bfloat16* ug, __nv_bfloat16* dug, float* db,
                                                       const float* mult, float* dmult, long long T,
                                                       int inner, float dropout_p, unsigned long long seed, const unsigned long long* seed_dev) {
    __shared__ float red[8][32][17];
    const int nchunk = inner >> 3;
    const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cl;
    const uint32_t thr = drop_thresh16(dropout_p);
    const float ks = dropout_p > 0.f ? drop_keep_scale(thr) : 1.f;
    const uint32_t seedmix = drop_seed_word(seed, seed_dev);
    float su[8] = {0, 0, 0, 0, 0, 0, 0, 0}, sg[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    float sm[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // MULT only
    if (c < nchunk) {
        const int hcol = c * 8;
        float m[8];
        if constexpr (MULT) {
#pragma unroll
            for (int j = 0; j < 8; ++j) m[j] = __ldg(mult + hcol + j);
        }
        const long long r1 = min(T, (long long)(blockIdx.y + 1) * GB_ROWS);
        for (long long row = (long long)blockIdx.y * GB_ROWS + rl; row < r1; row += 8) {
            const size_t pu = (size_t)row * 2 * inner + (hcol >> 6) * 128 + (hcol & 63);
            float d[8], u[8], g[8], du[8], dg[8];
            unpack8(*reinterpret_cast<const uint4*>(dh + (size_t)row * inner + hcol), d);
            unpack8(*reinterpret_cast<const uint4*>(ug + pu), u);
            unpack8(*reinterpret_cast<const uint4*>(ug + pu + 64), g);
            if (dropout_p > 0.f) {   // same pair hash as the GLU epilogue of the forward GEMM
                const uint32_t pbase = glu_drop_pair(row, inner, hcol);
#pragma unroll
                for (int j = 0; j < 8; j += 2) {
                    const DropWords hsh = drop_words(seedmix, pbase + (j >> 1));
                    d[j] = (hsh.a >= drop_thresh32(thr)) ? d[j] * ks : 0.f;
                    d[j + 1] = (hsh.b >= drop_thresh32(thr)) ? d[j + 1] * ks : 0.f;
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a;                       // act(g), MULT only
                const float dd = MULT ? d[j] * m[j] : d[j];   // the gradient reaching u * act(g)
                if constexpr (ACT == 1) {
                    const float cdf = 0.5f * (1.f + erff(g[j] * 0.70710678118654752440f));
                    const float pdf = 0.3989422804014327f * __expf(-0.5f * g[j] * g[j]);
                    du[j] = dd * g[j] * cdf;
                    dg[j] = dd * u[j] * (cdf + g[j] * pdf);
                    a = g[j] * cdf;
                } else if constexpr (ACT == 2) {
                    const float s = 1.f / (1.f + __expf(-g[j]));   // sigmoid; 0 where exp(-g) overflows
                    a = g[j] * s;
                    du[j] = dd * a;
                    dg[j] = dd * u[j] * (s + a * (1.f - s));      // silu'(g) = s (1 + g (1 - s))
                } else {
                    const float r = fmaxf(g[j], 0.f);
                    a = r * r;
                    du[j] = dd * a;
                    dg[j] = dd * u[j] * (2.f * r);
                }
                if constexpr (MULT) sm[j] += d[j] * u[j] * a;
            }
            const uint4 pu4 = pack8(du), pg4 = pack8(dg);
            *reinterpret_cast<uint4*>(dug + pu) = pu4;
            *reinterpret_cast<uint4*>(dug + pu + 64) = pg4;
            float fu[8], fg[8];   // sum what the weight-gradient GEMM will actually read (bf16-rounded)
            unpack8(pu4, fu);
            unpack8(pg4, fg);
#pragma unroll
            for (int j = 0; j < 8; ++j) { su[j] += fu[j]; sg[j] += fg[j]; }
        }
    }
    if (db) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { red[rl][cl][j] = su[j]; red[rl][cl][8 + j] = sg[j]; }
        __syncthreads();
        for (int i = threadIdx.x; i < 32 * 16; i += 256) {
            const int cc = i >> 4, j = i & 15;
            const int chunk = blockIdx.x * 32 + cc;
            if (chunk >= nchunk) continue;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) s += red[k][cc][j];
            const int hcol = chunk * 8 + (j & 7);
            atomicAdd(db + (hcol >> 6) * 128 + (hcol & 63) + (j >= 8 ? 64 : 0), s);
        }
    }
    if (MULT && dmult) {
        if (db) __syncthreads();   // the bias reduction has read `red`
#pragma unroll
        for (int j = 0; j < 8; ++j) red[rl][cl][j] = sm[j];
        __syncthreads();
        for (int i = threadIdx.x; i < 32 * 8; i += 256) {
            const int cc = i >> 3, j = i & 7;
            const int chunk = blockIdx.x * 32 + cc;
            if (chunk >= nchunk) continue;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) s += red[k][cc][j];
            atomicAdd(dmult + chunk * 8 + j, s);
        }
    }
}

// ------------------------------------------------------------------------------------------------ column sums (bias grads)
// out[n] += sum_t X[t, n]  (X bf16 [T, ld]); out must be zeroed by the caller.
// A block is CL 8-column chunk lanes x (256 / CL) row lanes; narrow matrices (the 16 gate-logit columns of the packed qkv
// gradient) use a small CL so that all 256 threads stay busy. Each thread keeps four 16-byte loads in flight; row lanes are
// combined by warp shuffles, warps through shared memory, and one atomicAdd per column per block reaches HBM.
template <int CL>
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ X, long long T, int ncols, int ld,
                                                     float* __restrict__ out, int rows_per_block) {
    constexpr int RL = 256 / CL;
    __shared__ float red[8][CL * 8];
    const int cg = threadIdx.x % CL, rl = threadIdx.x / CL;
    const int col0 = (blockIdx.x * CL + cg) * 8;
    const long long r0 = (long long)blockIdx.y * rows_per_block;
    const long long r1 = min(T, r0 + rows_per_block);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (col0 + 8 <= ncols) {
        for (long long r = r0 + rl; r < r1; r += 4 * RL) {
            uint4 u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const long long rr = r + (long long)k * RL;
                u[k] = rr < r1 ? __ldg(reinterpret_cast<const uint4*>(X + (size_t)rr * ld + col0)) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float v[8];
                unpack8(u[k], v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        }
    } else if (col0 < ncols) {
        for (long long r = r0 + rl; r < r1; r += RL)
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (col0 + j < ncols) acc[j] += __bfloat162float(X[(size_t)r * ld + col0 + j]);
    }
    // row lanes that share a warp: lanes differing in bits >= log2(CL)
#pragma unroll
    for (int o = CL; o < 32; o <<= 1)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (CL == 32 || lane < CL) {
#pragma unroll
        for (int j = 0; j < 8; ++j) red[warp][(lane % CL) * 8 + j] = acc[j];
    }
    __syncthreads();
    // CL == 32: a warp owns one row-lane, the 8 warps are the 8 row lanes; CL < 32: every warp holds all CL chunks
    if (threadIdx.x < CL * 8) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
        const int col = blockIdx.x * CL * 8 + threadIdx.x;
        if (col < ncols) atomicAdd(out + col, s);
    }
}

// ------------------------------------------------------------------------------------------------ final norm (head)
// y[b*N+n, :] = RMSNorm_g( sum_s x[b, R+n, s, :] )   (e2_tts.py:943-952); one warp per token
struct FnP {
    const __nv_bfloat16* xres; const float* g; __nv_bfloat16* y;
    int B, N, R, D, S;
    const __nv_bfloat16* dy; __nv_bfloat16* d_xres; float* g_g;
    int rpb, rows_per_block; const float* gains; float* d_gains; const __nv_bfloat16* d_res;   // branch-norm mode (BRANCH = true) only
};

// Branch-norm mode: y[r] = F.normalize(x[r]) * sqrt(D) * gain, x bf16 [rows, D] (S = 1, R = 0). Block (x, b) owns rows
// [x * rows_per_block, (x + 1) * rows_per_block) of batch b, so the per-batch gain and its gradient are one row of [B, D] per block
// (shared-memory sums, one atomic per column and block); one warp per row. gain = gains[b] or g.
template <int VPT>
__device__ __forceinline__ void branch_norm_fwd(const FnP& p) {
    const int lane = threadIdx.x & 31, nchunk = p.D >> 3;
    const long long base = (long long)blockIdx.y * p.rpb;
    const float* gain = p.gains ? p.gains + (size_t)blockIdx.y * p.D : p.g;
    const int r1 = min(p.rpb, ((int)blockIdx.x + 1) * p.rows_per_block);
    for (int r = (int)blockIdx.x * p.rows_per_block + (threadIdx.x >> 5); r < r1; r += 8) {
        const size_t row = (size_t)(base + r);
        float x[VPT][8];
        float ss = 0.f;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) unpack8(*reinterpret_cast<const uint4*>(p.xres + row * p.D + c * 8), x[v]);
            else {
#pragma unroll
                for (int e = 0; e < 8; ++e) x[v][e] = 0.f;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) ss += x[v][e] * x[v][e];
        }
        const float cn = sqrtf((float)p.D) / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = x[v][e] * cn * __ldg(gain + c * 8 + e);
                *reinterpret_cast<uint4*>(p.y + row * p.D + c * 8) = pack8(o);
            }
        }
    }
}
// dx = cn * (gain dy - x <gain dy, x> / |x|^2) with cn = sqrt(D) / max(|x|, 1e-12) (the second term vanishes where the clamp holds,
// as in F.normalize's backward); d_gain += dy * x * cn
template <int VPT>
__device__ __forceinline__ void branch_norm_bwd(const FnP& p, float* sg) {
    const int lane = threadIdx.x & 31, nchunk = p.D >> 3;
    const long long base = (long long)blockIdx.y * p.rpb;
    const float* gain = p.gains ? p.gains + (size_t)blockIdx.y * p.D : p.g;
    const int r1 = min(p.rpb, ((int)blockIdx.x + 1) * p.rows_per_block);
    for (int r = (int)blockIdx.x * p.rows_per_block + (threadIdx.x >> 5); r < r1; r += 8) {
        const size_t row = (size_t)(base + r);
        float x[VPT][8], dy[VPT][8];
        float ss = 0.f, dot = 0.f;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
#pragma unroll
            for (int e = 0; e < 8; ++e) { x[v][e] = 0.f; dy[v][e] = 0.f; }
            if (c < nchunk) {
                unpack8(*reinterpret_cast<const uint4*>(p.xres + row * p.D + c * 8), x[v]);
                unpack8(*reinterpret_cast<const uint4*>(p.dy + row * p.D + c * 8), dy[v]);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    dy[v][e] *= __ldg(gain + c * 8 + e);   // from here on: gain * dy (the gain gradient divides it back out below)
                    dot += dy[v][e] * x[v][e];
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) ss += x[v][e] * x[v][e];
        }
        ss = warp_sum(ss);
        const float nrm = sqrtf(ss);
        const float cn = sqrtf((float)p.D) / fmaxf(nrm, 1e-12f);
        dot = warp_sum(dot);
        const float k = nrm > 1e-12f ? dot / ss : 0.f;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
                float o[8], dyr[8], dr[8];
                unpack8(*reinterpret_cast<const uint4*>(p.dy + row * p.D + c * 8), dyr);   // L1-resident re-read: the raw dy for the gain
                if (p.d_res) unpack8(*reinterpret_cast<const uint4*>(p.d_res + row * p.D + c * 8), dr);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    atomicAdd(&sg[c * 8 + e], dyr[e] * x[v][e] * cn);
                    o[e] = cn * (dy[v][e] - x[v][e] * k);
                    if (p.d_res) o[e] += dr[e];
                }
                *reinterpret_cast<uint4*>(p.d_xres + row * p.D + c * 8) = pack8(o);
            }
        }
    }
}

template <int VPT, bool BRANCH = false>
__global__ void __launch_bounds__(256) final_norm_fwd_kernel(const FnP p) {
    if constexpr (BRANCH) {
        branch_norm_fwd<VPT>(p);
        return;
    }
    const int lane = threadIdx.x & 31, nchunk = p.D >> 3;
    const long long ntok = (long long)p.B * p.N;
    for (long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); row < ntok; row += (long long)gridDim.x * 8) {
        const long long b = row / p.N, n = row % p.N;
        const size_t tok = (size_t)b * (p.R + p.N) + p.R + n;
        float x[VPT][8];
        float ss = 0.f;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
#pragma unroll
            for (int e = 0; e < 8; ++e) x[v][e] = 0.f;
            if (c < nchunk) {
                for (int s = 0; s < p.S; ++s) {
                    float t[8];
                    unpack8(*reinterpret_cast<const uint4*>(p.xres + (tok * p.S + s) * p.D + c * 8), t);
#pragma unroll
                    for (int e = 0; e < 8; ++e) x[v][e] += t[e];
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) ss += x[v][e] * x[v][e];
        }
        const float cn = sqrtf((float)p.D) / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = x[v][e] * cn * __ldg(p.g + c * 8 + e);
                *reinterpret_cast<uint4*>(p.y + (size_t)row * p.D + c * 8) = pack8(o);
            }
        }
    }
}
template <int VPT, bool BRANCH = false>
__global__ void __launch_bounds__(256) final_norm_bwd_kernel(const FnP p) {
    extern __shared__ float sg[];  // [D]
    for (int i = threadIdx.x; i < p.D; i += 256) sg[i] = 0.f;
    __syncthreads();
    if constexpr (BRANCH) {
        branch_norm_bwd<VPT>(p, sg);
        __syncthreads();
        float* out = p.gains ? p.d_gains + (size_t)blockIdx.y * p.D : p.g_g;
        for (int i = threadIdx.x; i < p.D; i += 256) atomicAdd(out + i, sg[i]);
        return;
    }
    const int lane = threadIdx.x & 31, nchunk = p.D >> 3;
    const long long ntok = (long long)p.B * (p.R + p.N);
    const float invD = 1.f / (float)p.D;
    for (long long tokl = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); tokl < ntok; tokl += (long long)gridDim.x * 8) {
        const long long b = tokl / (p.R + p.N), n = tokl % (p.R + p.N);
        const size_t tok = (size_t)tokl;
        if (n < p.R) {  // register rows are dropped before the reduce: zero gradient
            for (int c = lane; c < nchunk * p.S; c += 32) *reinterpret_cast<uint4*>(p.d_xres + tok * p.S * p.D + (size_t)c * 8) = make_uint4(0, 0, 0, 0);
            continue;
        }
        const size_t row = (size_t)b * p.N + (n - p.R);
        float x[VPT][8], dy[VPT][8];
        float ss = 0.f, dot = 0.f;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
#pragma unroll
            for (int e = 0; e < 8; ++e) { x[v][e] = 0.f; dy[v][e] = 0.f; }
            if (c < nchunk) {
                for (int s = 0; s < p.S; ++s) {
                    float t[8];
                    unpack8(*reinterpret_cast<const uint4*>(p.xres + (tok * p.S + s) * p.D + c * 8), t);
#pragma unroll
                    for (int e = 0; e < 8; ++e) x[v][e] += t[e];
                }
                unpack8(*reinterpret_cast<const uint4*>(p.dy + row * p.D + c * 8), dy[v]);
#pragma unroll
                for (int e = 0; e < 8; ++e) dot += __ldg(p.g + c * 8 + e) * dy[v][e] * x[v][e];
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) ss += x[v][e] * x[v][e];
        }
        const float cn = sqrtf((float)p.D) / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
        dot = warp_sum(dot);
        const float k2 = cn * cn * cn * invD * dot;
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int c = lane + 32 * v;
            if (c < nchunk) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    atomicAdd(&sg[c * 8 + e], dy[v][e] * x[v][e] * cn);
                    o[e] = cn * __ldg(p.g + c * 8 + e) * dy[v][e] - x[v][e] * k2;
                }
                const uint4 u = pack8(o);
                for (int s = 0; s < p.S; ++s) *reinterpret_cast<uint4*>(p.d_xres + (tok * p.S + s) * p.D + c * 8) = u;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < p.D; i += 256) atomicAdd(p.g_g + i, sg[i]);
}

// ------------------------------------------------------------------------------------------------ masked MSE flow loss
// sums[0] += sum_{span} (pred - (x1 - x0))^2, sums[1] += #span rows; pred_data = x0 + pred  (e2_tts.py:1580-1595)
struct LossP {
    const float *pred, *x1, *x0; const unsigned char* span; float* sums; float* pred_data;
    long long rows; int C;
    const float* dloss; __nv_bfloat16* dpred; int ldp;
    const float* vel_target; float vel_weight; float* loss_parts;   // velocity-consistency term (e2_tts.py:1556-1576), optional
};
__global__ void __launch_bounds__(256) flow_loss_fwd_kernel(const LossP p) {
    float acc = 0.f, cnt = 0.f, accv = 0.f;
    const long long total = p.rows * p.C;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const long long row = i / p.C;
        const float pr = p.pred[i], a0 = p.x0[i];
        if (p.pred_data) p.pred_data[i] = a0 + pr;
        if (p.span[row]) {
            const float d = pr - (p.x1[i] - a0);
            acc += d * d;
            if (i % p.C == 0) cnt += 1.f;
            if (p.vel_target) {
                const float dv = pr - p.vel_target[i];
                accv += dv * dv;
            }
        }
    }
    acc = warp_sum(acc); cnt = warp_sum(cnt); accv = warp_sum(accv);
    __shared__ float sa[8], sc[8], sv[8];
    if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = acc; sc[threadIdx.x >> 5] = cnt; sv[threadIdx.x >> 5] = accv; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f, c = 0.f, v = 0.f;
        for (int k = 0; k < 8; ++k) { a += sa[k]; c += sc[k]; v += sv[k]; }
        atomicAdd(p.sums, a);
        atomicAdd(p.sums + 1, c);
        if (p.vel_target) atomicAdd(p.sums + 2, v);
    }
}
// loss = flow + vel_weight * velocity (e2_tts.py:1586-1589); loss_parts (optional) = {flow, velocity} for the LossBreakdown
__global__ void flow_loss_finalize_kernel(const float* sums, float* loss, int C, int has_vel, float vel_weight, float* loss_parts) {
    const float den = sums[1] * (float)C;
    const float flow = sums[0] / den, vel = has_vel ? sums[2] / den : 0.f;
    *loss = flow + vel_weight * vel;
    if (loss_parts) { loss_parts[0] = flow; loss_parts[1] = vel; }
}
__global__ void __launch_bounds__(256) flow_loss_bwd_kernel(const LossP p) {
    const float scale = 2.f * (*p.dloss) / (p.sums[1] * (float)p.C);
    const long long total = p.rows * p.ldp;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const long long row = i / p.ldp;
        const int c = (int)(i % p.ldp);
        float v = 0.f;
        if (c < p.C && p.span[row]) {
            const size_t s = (size_t)row * p.C + c;
            v = p.pred[s] - (p.x1[s] - p.x0[s]);
            if (p.vel_target) v += p.vel_weight * (p.pred[s] - p.vel_target[s]);
            v *= scale;
        }
        p.dpred[i] = __float2bfloat16(v);
    }
}


// ------------------------------------------------------------------------------------------------ gate / mask backward
// Forward epilogue was y = mask * cs[b,:] * (x W^T + bias). Given dy and y: dz = dy * mask * cs, d_cs[b,:] += sum_rows dy * y / cs,
// and (optionally) d_bias[:] += sum_rows dz — the bias gradient rides along so that no separate column-sum pass re-reads dz.
// Each thread keeps ONE 8-column chunk and marches over rows, four rows (eight 16-byte loads) in flight.
// RESID: the epilogue also added resid (y = gated + resid): the gated value is read back as y - resid.
template <bool RESID = false>
__global__ void __launch_bounds__(256) rowgate_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y,
                                                           const float* __restrict__ cs, const unsigned char* __restrict__ mask,
                                                           __nv_bfloat16* __restrict__ dz, float* __restrict__ d_cs,
                                                           float* __restrict__ d_bias, int rows_per_batch, int D, int rows_per_block,
                                                           const __nv_bfloat16* __restrict__ resid = nullptr) {
    extern __shared__ float sacc[];  // [D] gate sums, then [D] bias sums
    float* sbias = sacc + D;
    const int b = blockIdx.y;
    const int r0 = blockIdx.x * rows_per_block, r1 = min(rows_per_batch, r0 + rows_per_block);
    const int nchunk = D >> 3;
    const int nrl = max(1, 256 / nchunk);            // row lanes
    const int c = threadIdx.x % nchunk, rl = threadIdx.x / nchunk;
    if (cs || d_bias) {
        for (int i = threadIdx.x; i < 2 * D; i += 256) sacc[i] = 0.f;
        __syncthreads();
    }
    for (int cc = c; cc < nchunk && rl < nrl; cc += 256) {   // (single pass unless D > 2048)
        float s8[8] = {1, 1, 1, 1, 1, 1, 1, 1}, acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, accb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (cs) {
#pragma unroll
            for (int j = 0; j < 8; ++j) s8[j] = __ldg(cs + (size_t)b * D + cc * 8 + j);
        }
        for (int r = r0 + rl; r < r1; r += 4 * nrl) {
            uint4 ug[4], uy[4];
            bool keep[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int rr = r + k * nrl;
                const bool ok = rr < r1;
                const size_t row = (size_t)b * rows_per_batch + (ok ? rr : r);
                ug[k] = __ldg(reinterpret_cast<const uint4*>(dy + row * D + cc * 8));
                uy[k] = cs ? __ldg(reinterpret_cast<const uint4*>(y + row * D + cc * 8)) : make_uint4(0, 0, 0, 0);
                keep[k] = ok && (!mask || mask[row]);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int rr = r + k * nrl;
                if (rr >= r1) break;
                const size_t row = (size_t)b * rows_per_batch + rr;
                float g[8], yv[8], o[8];
                unpack8(ug[k], g);
                unpack8(uy[k], yv);
                if constexpr (RESID) {
                    if (cs) {
                        float rv[8];
                        unpack8(__ldg(reinterpret_cast<const uint4*>(resid + row * D + cc * 8)), rv);
#pragma unroll
                        for (int j = 0; j < 8; ++j) yv[j] -= rv[j];
                    }
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[j] = keep[k] ? g[j] * s8[j] : 0.f;
                    acc[j] += keep[k] ? g[j] * yv[j] : 0.f;
                    accb[j] += o[j];
                }
                *reinterpret_cast<uint4*>(dz + row * D + cc * 8) = pack8(o);
            }
        }
        if (cs) {
#pragma unroll
            for (int j = 0; j < 8; ++j)   // d_cs = sum dy * z with z = y / cs: a gate that underflowed to 0 zeroed y as well (0/0), its gradient is taken as 0
                atomicAdd(&sacc[cc * 8 + j], fabsf(s8[j]) > 1e-30f ? acc[j] / s8[j] : 0.f);
        }
        if (d_bias) {
#pragma unroll
            for (int j = 0; j < 8; ++j) atomicAdd(&sbias[cc * 8 + j], accb[j]);
        }
    }
    if (cs || d_bias) {
        __syncthreads();
        if (cs) for (int i = threadIdx.x; i < D; i += 256) atomicAdd(d_cs + (size_t)b * D + i, sacc[i]);
        if (d_bias) for (int i = threadIdx.x; i < D; i += 256) atomicAdd(d_bias + i, sbias[i]);
    }
}

// fp32 -> bf16 cast with row pitch (used for small host-provided matrices)
__global__ void cast_rows_kernel(const float* src, __nv_bfloat16* dst, long long rows, int cols, int ld) {
    const long long total = rows * ld;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int c = (int)(i % ld);
        dst[i] = __float2bfloat16(c < cols ? src[(i / ld) * cols + c] : 0.f);
    }
}

static inline int grid_for(long long total, int per_block = 256) {
    long long g = (total + per_block - 1) / per_block;
    const long long cap = (long long)num_sms() * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace b200

using namespace b200;

extern "C" int b200_pack_weights(const b200_pack_desc* descs_dev, int32_t n, b200_stream_t stream) {
    B200_REQUIRE(descs_dev && n > 0, "pack_weights: empty table");
    pack_weights_kernel<<<dim3(32, n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(descs_dev);
    return check_launch("pack_weights_kernel");
}

extern "C" int b200_stem_prepare(const b200_stem_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->A && ((a->x1 && a->x0 && a->times && a->span) || (a->x_in && a->cond_in)), "stem_prepare: null pointer");
    B200_REQUIRE(a->C > 0 && a->Cp >= a->C && (a->Cp % 64) == 0, "stem_prepare: Cp must be a multiple of 64 >= C");
    StemP p{a->x1, a->x0, a->times, a->x_in, a->cond_in, a->span, (__nv_bfloat16*)a->A, a->cond_out, a->B, a->N, a->C, a->Cp, a->concat_cond};
    stem_prepare_kernel<<<grid_for((long long)a->B * a->N * a->Cp * 2), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("stem_prepare_kernel");
}

static int fill_asm(AsmP& p, const b200_assemble_args* a) {
    B200_REQUIRE(a && (a->h || (a->ids && a->emb)) && (a->registers || a->R == 0), "assemble: null pointer");   // R = 0: no register rows to read
    B200_REQUIRE(a->D % 8 == 0 && a->S >= 1 && a->B > 0 && a->N > 0 && a->R >= 0, "assemble: unsupported shape");
    p.h = (const __nv_bfloat16*)a->h; p.ids = a->ids; p.emb = a->emb; p.abs_pos = a->abs_pos; p.registers = a->registers;
    p.B = a->B; p.N = a->N; p.R = a->R; p.D = a->D; p.S = a->S;
    return 0;
}
extern "C" int b200_assemble_fwd(const b200_assemble_args* a, b200_stream_t stream) {
    AsmP p{};
    if (fill_asm(p, a)) return -1;
    B200_REQUIRE(a->out, "assemble_fwd: null output");
    p.out = (__nv_bfloat16*)a->out;
    assemble_fwd_kernel<<<grid_for((long long)a->B * (a->R + a->N) * (a->D / 8)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("assemble_fwd_kernel");
}
extern "C" int b200_assemble_bwd(const b200_assemble_args* a, b200_stream_t stream) {
    AsmP p{};
    if (fill_asm(p, a)) return -1;
    B200_REQUIRE(a->d_out, "assemble_bwd: null d_out");
    p.d_out = (const __nv_bfloat16*)a->d_out; p.d_h = (__nv_bfloat16*)a->d_h; p.d_tok = a->d_tok; p.d_abs_pos = a->d_abs_pos; p.d_registers = a->d_registers;
    const long long total = (long long)(a->R + a->N) * (a->D / 8);
    assemble_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("assemble_bwd_kernel");
}
extern "C" int b200_embed_bwd(const float* d_tok, const int32_t* ids, float* d_emb, int32_t ntok, int32_t D, int32_t vocab, b200_stream_t stream) {
    B200_REQUIRE(d_tok && ids && d_emb && ntok > 0 && D > 0 && vocab > 0, "embed_bwd: bad arguments");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(d_emb, 0, (size_t)vocab * D * sizeof(float), st);
    B200_REQUIRE(e == cudaSuccess, "embed_bwd: memset: %s", cudaGetErrorString(e));
    const int slab = 1024;
    embed_bwd_kernel<<<dim3(vocab, (ntok + slab - 1) / slab), 256, 0, st>>>(d_tok, ids, d_emb, ntok, D, slab);
    return check_launch("embed_bwd_kernel");
}
extern "C" int b200_rotary_table(float* cos_out, float* sin_out, int32_t Np, int32_t dim_head, b200_stream_t stream) {
    B200_REQUIRE(cos_out && sin_out && Np > 0, "rotary_table: bad arguments");
    B200_REQUIRE(dim_head == 64 || dim_head == 128, "rotary_table: dim_head must be 64 or 128 (got %d)", dim_head);
    const int half = dim_head / 2;
    rotary_table_kernel<<<(Np * half + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(cos_out, sin_out, Np, half);
    return check_launch("rotary_table_kernel");
}

static int fill_qkv(QkvP& p, const b200_qkv_post_args* a) {
    B200_REQUIRE(a && a->qkvg && a->rot_cos && a->rot_sin && (a->no_gate || (a->gate_bias && a->gate)), "qkv_post: null pointer");
    B200_REQUIRE(a->dim_head == 64 || a->dim_head == 128, "qkv_post: dim_head must be 64 or 128 (got %d)", a->dim_head);
    B200_REQUIRE(a->ld % 8 == 0 && a->ld >= 3 * a->H * a->dim_head + ((a->no_gate ? 0 : 1) + (a->v_first ? 1 : 0)) * a->H, "qkv_post: bad row pitch %d",
                 a->ld);
    B200_REQUIRE(!a->v_first || a->mix_bias, "qkv_post: value residual needs the mix bias");
    p.qkvg = (const __nv_bfloat16*)a->qkvg; p.ld = a->ld; p.gate_b = a->gate_bias; p.mix_b = a->mix_bias; p.cs = a->rot_cos; p.sn = a->rot_sin;
    p.v_first = (const __nv_bfloat16*)a->v_first; p.gate = a->gate; p.B = a->B; p.H = a->H; p.Np = a->Np;
    p.no_gate = a->no_gate;
    return 0;
}
extern "C" int b200_qkv_post_fwd(const b200_qkv_post_args* a, b200_stream_t stream) {
    QkvP p{};
    if (fill_qkv(p, a)) return -1;
    B200_REQUIRE(a->q && a->k && a->v, "qkv_post_fwd: null output");
    p.q = (__nv_bfloat16*)a->q; p.k = (__nv_bfloat16*)a->k; p.v = (__nv_bfloat16*)a->v;
    const long long threads = (long long)a->B * a->Np * a->H * (a->dim_head / 8);
    if (a->dim_head == 64) qkv_post_fwd_kernel<64><<<grid_for(threads), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    else qkv_post_fwd_kernel<128><<<grid_for(threads), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("qkv_post_fwd_kernel");
}
extern "C" int b200_qkv_post_bwd(const b200_qkv_post_args* a, b200_stream_t stream) {
    QkvP p{};
    if (fill_qkv(p, a)) return -1;
    B200_REQUIRE(a->dq && a->dk && a->dv && (a->no_gate || a->d_gate) && a->d_qkvg && (!a->v_first || a->d_vfirst), "qkv_post_bwd: null pointer");
    p.dq = (const __nv_bfloat16*)a->dq; p.dk = (const __nv_bfloat16*)a->dk; p.dv = (const __nv_bfloat16*)a->dv; p.d_gate = a->d_gate;
    p.d_qkvg = (__nv_bfloat16*)a->d_qkvg; p.d_vfirst = (__nv_bfloat16*)a->d_vfirst; p.dq_fp32 = a->dq_fp32; p.dv_extra = (const __nv_bfloat16*)a->dv_extra;
    const long long total = (long long)a->B * a->Np * a->H * (a->dim_head / 8);
    if (a->dim_head == 64) qkv_post_bwd_kernel<64><<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    else qkv_post_bwd_kernel<128><<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("qkv_post_bwd_kernel");
}

extern "C" int b200_glu_bwd(const b200_glu_bwd_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->dh && a->ug && a->dug, "glu_bwd: null pointer");
    B200_REQUIRE(a->T > 0 && a->inner > 0 && (a->inner % 64) == 0, "glu_bwd: inner must be a multiple of 64");
    B200_REQUIRE(a->act >= 1 && a->act <= 3, "glu_bwd: act=%d is not an activation code (1 GELU, 2 SiLU, 3 ReLU^2)", (int)a->act);
    B200_REQUIRE(!a->d_mult || a->mult, "glu_bwd: d_mult needs mult");
    dim3 grid((a->inner / 8 + 31) / 32, (unsigned)((a->T + GB_ROWS - 1) / GB_ROWS));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const auto dh = (const __nv_bfloat16*)a->dh, ug = (const __nv_bfloat16*)a->ug;
    const auto dug = (__nv_bfloat16*)a->dug;
    const auto sd = reinterpret_cast<const unsigned long long*>(a->seed_dev);
    auto kern = glu_bwd_kernel<1, false>;
    if (a->mult) kern = a->act == 1 ? glu_bwd_kernel<1, true> : a->act == 2 ? glu_bwd_kernel<2, true> : glu_bwd_kernel<3, true>;
    else kern = a->act == 1 ? glu_bwd_kernel<1, false> : a->act == 2 ? glu_bwd_kernel<2, false> : glu_bwd_kernel<3, false>;
    kern<<<grid, 256, 0, st>>>(dh, ug, dug, a->db_packed, a->mult, a->d_mult, a->T, a->inner, a->dropout_p, a->seed, sd);
    return check_launch("glu_bwd_kernel");
}

extern "C" int b200_geglu_bwd(const void* dh, const void* ug, void* dug, float* db_packed, int64_t T, int32_t inner, float dropout_p, uint64_t seed,
                              const uint64_t* seed_dev, b200_stream_t stream) {
    B200_REQUIRE(dh && ug && dug && T > 0 && inner > 0 && (inner % 64) == 0, "geglu_bwd: inner must be a multiple of 64");
    b200_glu_bwd_args a{};
    a.dh = dh; a.ug = ug; a.dug = dug; a.db_packed = db_packed;
    a.T = T; a.inner = inner; a.act = 1;
    a.dropout_p = dropout_p; a.seed = seed; a.seed_dev = seed_dev;
    return b200_glu_bwd(&a, stream);
}

extern "C" int b200_colsum(const void* X, int64_t T, int32_t ncols, int32_t ld, float* out, b200_stream_t stream) {
    B200_REQUIRE(X && out && T > 0 && ncols > 0 && ld >= ncols && (ld % 8) == 0, "colsum: bad arguments");
    const int nchunk = (ncols + 7) / 8;
    int cl = 32;
    while (cl > 2 && cl / 2 >= nchunk) cl >>= 1;     // chunk lanes per block: 32 for wide matrices, fewer when ncols < 256
    const int col_blocks = (nchunk + cl - 1) / cl;
    const int rl = 256 / cl;
    // about two blocks per SM, each thread marching over >= 4 rows; few enough blocks that the final atomics stay cheap
    long long slabs = (2LL * num_sms() + col_blocks - 1) / col_blocks;
    long long rows_per_block = (T + slabs - 1) / slabs;
    const long long min_rows = 4LL * rl;
    rows_per_block = ((rows_per_block + min_rows - 1) / min_rows) * min_rows;
    dim3 grid(col_blocks, (unsigned)((T + rows_per_block - 1) / rows_per_block));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const __nv_bfloat16* x = (const __nv_bfloat16*)X;
    switch (cl) {
        case 32: colsum_kernel<32><<<grid, 256, 0, st>>>(x, T, ncols, ld, out, (int)rows_per_block); break;
        case 16: colsum_kernel<16><<<grid, 256, 0, st>>>(x, T, ncols, ld, out, (int)rows_per_block); break;
        case 8: colsum_kernel<8><<<grid, 256, 0, st>>>(x, T, ncols, ld, out, (int)rows_per_block); break;
        case 4: colsum_kernel<4><<<grid, 256, 0, st>>>(x, T, ncols, ld, out, (int)rows_per_block); break;
        default: colsum_kernel<2><<<grid, 256, 0, st>>>(x, T, ncols, ld, out, (int)rows_per_block); break;
    }
    return check_launch("colsum_kernel");
}

// branch-norm mode (rows_per_batch > 0): validation shared by fwd / bwd, and the launch shape (block rows of one batch)
static int check_branch_norm(const b200_final_norm_args* a, FnP& p, dim3& grid) {
    B200_REQUIRE(a->D % 8 == 0 && a->D <= 1024, "final_norm: D must be a multiple of 8 and <= 1024");
    B200_REQUIRE(a->S == 1 && a->R == 0, "final_norm: branch-norm mode (rows_per_batch > 0) takes S == 1 and R == 0 (got S=%d, R=%d)", a->S, a->R);
    B200_REQUIRE(a->B > 0 && a->N > 0, "final_norm: unsupported shape");
    const long long rows = (long long)a->B * a->N;
    B200_REQUIRE(rows % a->rows_per_batch == 0 && rows / a->rows_per_batch <= 65535,
                 "final_norm: B*N (%lld) must be a multiple of rows_per_batch (%d), at most 65535 batches", rows, a->rows_per_batch);
    B200_REQUIRE(a->gains || a->g, "final_norm: branch-norm mode needs gains or g");
    // about four blocks per SM over all batches, 8 to 128 rows (a multiple of the 8 warps) per block
    const long long nb = rows / a->rows_per_batch;
    long long rb = (rows + 4LL * num_sms() - 1) / (4LL * num_sms());
    rb = min(128LL, max(8LL, (rb + 7) / 8 * 8));
    p = FnP{(const __nv_bfloat16*)a->xres, a->g, (__nv_bfloat16*)a->y, a->B, a->N, a->R, a->D, a->S, (const __nv_bfloat16*)a->dy,
            (__nv_bfloat16*)a->d_xres, a->g_g, a->rows_per_batch, (int)rb, a->gains, a->d_gains, (const __nv_bfloat16*)a->d_res};
    grid = dim3((unsigned)((a->rows_per_batch + rb - 1) / rb), (unsigned)nb);
    return 0;
}
extern "C" int b200_final_norm_fwd(const b200_final_norm_args* a, b200_stream_t stream) {
    B200_REQUIRE(a, "final_norm_fwd: null pointer");
    B200_REQUIRE(a->rows_per_batch >= 0, "final_norm: rows_per_batch must be >= 0 (got %d)", a->rows_per_batch);
    if (a->rows_per_batch > 0) {
        B200_REQUIRE(a->xres && a->y, "final_norm_fwd: null pointer");
        FnP p;
        dim3 grid;
        if (check_branch_norm(a, p, grid)) return -1;
        cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
        if (a->D <= 256) final_norm_fwd_kernel<1, true><<<grid, 256, 0, st>>>(p);
        else if (a->D <= 512) final_norm_fwd_kernel<2, true><<<grid, 256, 0, st>>>(p);
        else final_norm_fwd_kernel<4, true><<<grid, 256, 0, st>>>(p);
        return check_launch("final_norm_fwd_kernel");
    }
    B200_REQUIRE(!a->gains && !a->d_gains, "final_norm: gains / d_gains need rows_per_batch > 0 (branch-norm mode)");
    B200_REQUIRE(a->xres && a->g && a->y, "final_norm_fwd: null pointer");
    B200_REQUIRE(a->D % 8 == 0 && a->D <= 1024 && a->S >= 1, "final_norm: D must be a multiple of 8 and <= 1024");
    FnP p{(const __nv_bfloat16*)a->xres, a->g, (__nv_bfloat16*)a->y, a->B, a->N, a->R, a->D, a->S, nullptr, nullptr, nullptr};
    const int grid = (int)min(((long long)a->B * a->N + 7) / 8, (long long)num_sms() * 8);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (a->D <= 256) final_norm_fwd_kernel<1><<<grid, 256, 0, st>>>(p);
    else if (a->D <= 512) final_norm_fwd_kernel<2><<<grid, 256, 0, st>>>(p);
    else final_norm_fwd_kernel<4><<<grid, 256, 0, st>>>(p);
    return check_launch("final_norm_fwd_kernel");
}
extern "C" int b200_final_norm_bwd(const b200_final_norm_args* a, b200_stream_t stream) {
    B200_REQUIRE(a, "final_norm_bwd: null pointer");
    B200_REQUIRE(a->rows_per_batch >= 0, "final_norm: rows_per_batch must be >= 0 (got %d)", a->rows_per_batch);
    if (a->rows_per_batch > 0) {
        B200_REQUIRE(a->xres && a->dy && a->d_xres, "final_norm_bwd: null pointer");
        B200_REQUIRE(a->gains ? a->d_gains != nullptr : a->g_g != nullptr, "final_norm_bwd: gains need d_gains, g needs g_g");
        FnP p;
        dim3 grid;
        if (check_branch_norm(a, p, grid)) return -1;
        cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
        const size_t smem = (size_t)a->D * 4;
        if (a->D <= 256) final_norm_bwd_kernel<1, true><<<grid, 256, smem, st>>>(p);
        else if (a->D <= 512) final_norm_bwd_kernel<2, true><<<grid, 256, smem, st>>>(p);
        else final_norm_bwd_kernel<4, true><<<grid, 256, smem, st>>>(p);
        return check_launch("final_norm_bwd_kernel");
    }
    B200_REQUIRE(!a->gains && !a->d_gains && !a->d_res, "final_norm: gains / d_gains / d_res need rows_per_batch > 0 (branch-norm mode)");
    B200_REQUIRE(a->xres && a->g && a->dy && a->d_xres && a->g_g, "final_norm_bwd: null pointer");
    B200_REQUIRE(a->D % 8 == 0 && a->D <= 1024 && a->S >= 1, "final_norm: D must be a multiple of 8 and <= 1024");
    FnP p{(const __nv_bfloat16*)a->xres, a->g, nullptr, a->B, a->N, a->R, a->D, a->S, (const __nv_bfloat16*)a->dy, (__nv_bfloat16*)a->d_xres, a->g_g};
    const int grid = (int)min(((long long)a->B * (a->N + a->R) + 7) / 8, (long long)num_sms() * 4);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = (size_t)a->D * 4;
    if (a->D <= 256) final_norm_bwd_kernel<1><<<grid, 256, smem, st>>>(p);
    else if (a->D <= 512) final_norm_bwd_kernel<2><<<grid, 256, smem, st>>>(p);
    else final_norm_bwd_kernel<4><<<grid, 256, smem, st>>>(p);
    return check_launch("final_norm_bwd_kernel");
}

extern "C" int b200_flow_loss_fwd(const b200_flow_loss_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->pred && a->x1 && a->x0 && a->span && a->sums && a->loss, "flow_loss_fwd: null pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(a->sums, 0, 4 * sizeof(float), st);
    B200_REQUIRE(e == cudaSuccess, "flow_loss_fwd: memset: %s", cudaGetErrorString(e));
    LossP p{a->pred, a->x1, a->x0, a->span, a->sums, a->pred_data, a->rows, a->C, nullptr, nullptr, 0, a->vel_target, a->vel_weight, a->loss_parts};
    flow_loss_fwd_kernel<<<grid_for(a->rows * a->C), 256, 0, st>>>(p);
    if (int rc = check_launch("flow_loss_fwd_kernel")) return rc;
    flow_loss_finalize_kernel<<<1, 1, 0, st>>>(a->sums, a->loss, a->C, a->vel_target != nullptr, a->vel_weight, a->loss_parts);
    return check_launch("flow_loss_finalize_kernel");
}
extern "C" int b200_flow_loss_bwd(const b200_flow_loss_args* a, b200_stream_t stream) {
    B200_REQUIRE(a && a->pred && a->x1 && a->x0 && a->span && a->sums && a->dloss && a->dpred && a->ldp >= a->C && (a->ldp % 8) == 0, "flow_loss_bwd: bad arguments");
    LossP p{a->pred, a->x1, a->x0, a->span, a->sums, nullptr, a->rows, a->C, a->dloss, (__nv_bfloat16*)a->dpred, a->ldp, a->vel_target, a->vel_weight, nullptr};
    flow_loss_bwd_kernel<<<grid_for(a->rows * a->ldp), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("flow_loss_bwd_kernel");
}

extern "C" int b200_rowgate_bwd(const void* dy, const void* y, const float* cs, const uint8_t* mask, void* dz, float* d_cs,
                                float* d_bias, int32_t B, int32_t rows_per_batch, int32_t D, b200_stream_t stream) {
    B200_REQUIRE(dy && dz && B > 0 && B <= 65535 && rows_per_batch > 0 && D % 8 == 0, "rowgate_bwd: bad arguments");
    B200_REQUIRE(!cs || (y && d_cs), "rowgate_bwd: gate backward needs y and d_cs");
    const int rpb = 64;
    dim3 grid((rows_per_batch + rpb - 1) / rpb, B);
    rowgate_bwd_kernel<<<grid, 256, (size_t)D * 8, reinterpret_cast<cudaStream_t>(stream)>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, cs, mask, (__nv_bfloat16*)dz, d_cs, d_bias, rows_per_batch, D, rpb);
    return check_launch("rowgate_bwd_kernel");
}
extern "C" int b200_rowgate_resid_bwd(const void* dy, const void* y, const void* resid, const float* cs, const uint8_t* mask, void* dz,
                                      float* d_cs, float* d_bias, int32_t B, int32_t rows_per_batch, int32_t D, b200_stream_t stream) {
    B200_REQUIRE(dy && dz && B > 0 && B <= 65535 && rows_per_batch > 0 && D % 8 == 0, "rowgate_bwd: bad arguments");
    B200_REQUIRE(!cs || (y && d_cs), "rowgate_bwd: gate backward needs y and d_cs");
    B200_REQUIRE(resid, "rowgate_resid_bwd: null resid");
    const int rpb = 64;
    dim3 grid((rows_per_batch + rpb - 1) / rpb, B);
    rowgate_bwd_kernel<true><<<grid, 256, (size_t)D * 8, reinterpret_cast<cudaStream_t>(stream)>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, cs, mask, (__nv_bfloat16*)dz, d_cs, d_bias, rows_per_batch, D, rpb,
        (const __nv_bfloat16*)resid);
    return check_launch("rowgate_bwd_kernel");
}

// LinearFourierEmbed tail (e2_tts.py:368-386, attn_fourier_embed_input — a non-default switch of Transformer.__init__ :545-546):
//   z = linear(x) [T, df + dr]  ->  out [T, 2*df + dr] = cat(sin(z[:, :df]), cos(z[:, :df]), z[:, df:]);  the Linear itself is b200_gemm.
// One thread per 2 output columns; sin / cos in fp32 on the bf16 GEMM output (sincosf: arguments are not range-limited).
namespace b200 {
__global__ void __launch_bounds__(256) fourier_feat_fwd_kernel(const __nv_bfloat16* __restrict__ z, long long ldz, __nv_bfloat16* __restrict__ out,
                                                               long long T, int df, int dr) {
    const int dout = 2 * df + dr;
    const long long total = T * dout;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const long long t = i / dout;
        const int c = (int)(i % dout);
        const __nv_bfloat16* zr = z + t * ldz;
        float v;
        if (c < df) v = sinf(__bfloat162float(zr[c]));
        else if (c < 2 * df) v = cosf(__bfloat162float(zr[c - df]));
        else v = __bfloat162float(zr[c - df]);
        out[i] = __float2bfloat16(v);
    }
}
// dz[:, :df] = d_out[:, :df] * cos(z) - d_out[:, df:2df] * sin(z);  dz[:, df:] = d_out[:, 2df:]
__global__ void __launch_bounds__(256) fourier_feat_bwd_kernel(const __nv_bfloat16* __restrict__ d_out, const __nv_bfloat16* __restrict__ z,
                                                               long long ldz, __nv_bfloat16* __restrict__ dz, long long T, int df, int dr) {
    const int dout = 2 * df + dr, dz_cols = df + dr;
    const long long total = T * ldz;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const long long t = i / ldz;
        const int c = (int)(i % ldz);
        float v = 0.f;                      // pitch padding columns of dz are zeroed (they feed the dX / dW GEMMs as K rows)
        const __nv_bfloat16* g = d_out + t * dout;
        if (c < df) {
            float sn, cs;
            sincosf(__bfloat162float(z[i]), &sn, &cs);
            v = __bfloat162float(g[c]) * cs - __bfloat162float(g[c + df]) * sn;
        } else if (c < dz_cols) {
            v = __bfloat162float(g[c + df]);
        }
        dz[i] = __float2bfloat16(v);
    }
}
}  // namespace b200

extern "C" int b200_fourier_feat_fwd(const void* z, int64_t ldz, void* out, int64_t T, int32_t df, int32_t dr, b200_stream_t stream) {
    B200_REQUIRE(z && out && T > 0 && df >= 0 && dr >= 0 && df + dr > 0 && ldz >= df + dr, "fourier_feat_fwd: bad arguments");
    fourier_feat_fwd_kernel<<<grid_for(T * (2 * df + dr)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>((const __nv_bfloat16*)z,
                (long long)ldz, (__nv_bfloat16*)out, (long long)T, df, dr);
    return check_launch("fourier_feat_fwd_kernel");
}
extern "C" int b200_fourier_feat_bwd(const void* d_out, const void* z, int64_t ldz, void* dz, int64_t T, int32_t df, int32_t dr, b200_stream_t stream) {
    B200_REQUIRE(d_out && z && dz && T > 0 && df >= 0 && dr >= 0 && df + dr > 0 && ldz >= df + dr, "fourier_feat_bwd: bad arguments");
    fourier_feat_bwd_kernel<<<grid_for(T * ldz), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>((const __nv_bfloat16*)d_out,
                (const __nv_bfloat16*)z, (long long)ldz, (__nv_bfloat16*)dz, (long long)T, df, dr);
    return check_launch("fourier_feat_bwd_kernel");
}

// InterpolatedCharacterEmbed (e2_tts.py:414-482; E2TTS(interpolated_text=True) :1135, :1233): per sample, the embeddings of its Lt valid
// characters are stretched to its La audio frames by linear interpolation (F.interpolate 'bilinear', align_corners=False, :237-244, :459)
// and the stretched ABSOLUTE text positions linspace(0, Lt, La) (:460) go through abs_pos_mlp = Linear(1, d) -> SiLU -> Linear(d, d)
// (:424-429, :477). This kernel produces the two GEMM-side operands of  te = mask * (Linear2(h1) + lerp):
//   lerp [B*N, D] bf16 (rows n >= La: 0)  and  h1 = silu(pos * w1 + b1) [B*N, D] bf16 (pos = 0 for n >= La, as the reference's padding).
namespace b200 {
struct InterpP {
    const int* ids;        // [B, nt] compacted character ids (the first Lt[b] entries are valid)
    const int *Lt, *La;    // [B]
    const float *emb, *w1, *b1;
    int B, N, nt, D, V;
};
__device__ __forceinline__ void interp_coords(int n, int Lt, int La, int& i0, int& i1, float& lam, float& pos) {
    // area_pixel_compute_source_index(scale = Lt / La, align_corners = false): src = max((n + 0.5) * scale - 0.5, 0)
    const float scale = (float)Lt / (float)La;
    const float src = fmaxf(((float)n + 0.5f) * scale - 0.5f, 0.f);
    i0 = min((int)src, Lt - 1);
    i1 = i0 + (i0 < Lt - 1 ? 1 : 0);
    lam = src - (float)i0;
    // torch.linspace(0, Lt, La): step = Lt / (La - 1); first half counts up from 0, second half down from Lt
    const float step = La > 1 ? (float)Lt / (float)(La - 1) : 0.f;
    pos = (n < La / 2 || La == 1) ? (float)n * step : (float)Lt - (float)(La - 1 - n) * step;
}
__global__ void __launch_bounds__(256) interp_text_fwd_kernel(const InterpP p, __nv_bfloat16* __restrict__ lerp, __nv_bfloat16* __restrict__ h1) {
    const long long total = (long long)p.B * p.N * p.D;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int c = (int)(i % p.D);
        const long long row = i / p.D;
        const int n = (int)(row % p.N), b = (int)(row / p.N);
        const int Lt = p.Lt[b], La = min(p.La[b], p.N);
        float e = 0.f, pos = 0.f;
        if (n < La && Lt > 0) {
            int i0, i1; float lam;
            interp_coords(n, Lt, La, i0, i1, lam, pos);
            const int t0 = p.ids[(size_t)b * p.nt + i0], t1 = p.ids[(size_t)b * p.nt + i1];
            e = (1.f - lam) * __ldg(p.emb + (size_t)t0 * p.D + c) + lam * __ldg(p.emb + (size_t)t1 * p.D + c);
        }
        const float pre = pos * __ldg(p.w1 + c) + __ldg(p.b1 + c);
        lerp[i] = __float2bfloat16(e);
        h1[i] = __float2bfloat16(pre / (1.f + __expf(-pre)));
    }
}
// backward: d_emb[id] += weights * d_lerp (atomics into the zero-initialised table gradient); through SiLU and Linear(1, d):
// d_pre = d_h1 * silu'(pre), dw1[c] += sum_rows d_pre * pos, db1[c] += sum_rows d_pre. One thread per channel marching ROWS rows.
constexpr int INTERP_ROWS = 64;
__global__ void __launch_bounds__(256) interp_text_bwd_kernel(const InterpP p, const __nv_bfloat16* __restrict__ d_lerp, const __nv_bfloat16* __restrict__ d_h1,
                                                              float* __restrict__ d_emb, float* __restrict__ dw1, float* __restrict__ db1) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= p.D) return;
    const long long r0 = (long long)blockIdx.y * INTERP_ROWS, r1 = min((long long)p.B * p.N, r0 + INTERP_ROWS);
    const float w1 = __ldg(p.w1 + c), b1 = __ldg(p.b1 + c);
    float gw = 0.f, gb = 0.f;
    for (long long row = r0; row < r1; ++row) {
        const int n = (int)(row % p.N), b = (int)(row / p.N);
        const int Lt = p.Lt[b], La = min(p.La[b], p.N);
        float pos = 0.f;
        if (n < La && Lt > 0) {
            int i0, i1; float lam;
            interp_coords(n, Lt, La, i0, i1, lam, pos);
            const float g = __bfloat162float(d_lerp[row * p.D + c]);
            const int t0 = p.ids[(size_t)b * p.nt + i0], t1 = p.ids[(size_t)b * p.nt + i1];
            atomicAdd(d_emb + (size_t)t0 * p.D + c, (1.f - lam) * g);
            atomicAdd(d_emb + (size_t)t1 * p.D + c, lam * g);
        }
        const float pre = pos * w1 + b1;
        const float sg = 1.f / (1.f + __expf(-pre));
        const float dpre = __bfloat162float(d_h1[row * p.D + c]) * sg * (1.f + pre * (1.f - sg));
        gw += dpre * pos;
        gb += dpre;
    }
    atomicAdd(dw1 + c, gw);
    atomicAdd(db1 + c, gb);
}
}  // namespace b200

static int fill_interp(InterpP& p, const b200_interp_text_args* a) {
    B200_REQUIRE(a && a->ids && a->text_len && a->audio_len && a->emb && a->w1 && a->b1, "interp_text: null pointer");
    B200_REQUIRE(a->B > 0 && a->N > 0 && a->nt > 0 && a->D > 0 && a->vocab > 0, "interp_text: bad shape");
    p.ids = a->ids; p.Lt = a->text_len; p.La = a->audio_len; p.emb = a->emb; p.w1 = a->w1; p.b1 = a->b1;
    p.B = a->B; p.N = a->N; p.nt = a->nt; p.D = a->D; p.V = a->vocab;
    return 0;
}
extern "C" int b200_interp_text_fwd(const b200_interp_text_args* a, b200_stream_t stream) {
    InterpP p{};
    if (fill_interp(p, a)) return -1;
    B200_REQUIRE(a->lerp && a->h1, "interp_text_fwd: null output");
    interp_text_fwd_kernel<<<grid_for((long long)a->B * a->N * a->D), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p,
                (__nv_bfloat16*)a->lerp, (__nv_bfloat16*)a->h1);
    return check_launch("interp_text_fwd_kernel");
}
extern "C" int b200_interp_text_bwd(const b200_interp_text_args* a, b200_stream_t stream) {
    InterpP p{};
    if (fill_interp(p, a)) return -1;
    B200_REQUIRE(a->d_lerp && a->d_h1 && a->d_emb && a->d_w1 && a->d_b1, "interp_text_bwd: null pointer");
    const long long rows = (long long)a->B * a->N;
    dim3 grid((a->D + 255) / 256, (unsigned)((rows + INTERP_ROWS - 1) / INTERP_ROWS));
    interp_text_bwd_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, (const __nv_bfloat16*)a->d_lerp,
                (const __nv_bfloat16*)a->d_h1, a->d_emb, a->d_w1, a->d_b1);
    return check_launch("interp_text_bwd_kernel");
}

extern "C" int b200_cast_rows(const float* src, void* dst, int64_t rows, int32_t cols, int32_t ld, b200_stream_t stream) {
    B200_REQUIRE(src && dst && rows > 0 && cols > 0 && ld >= cols, "cast_rows: bad arguments");
    cast_rows_kernel<<<grid_for(rows * ld), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(src, (__nv_bfloat16*)dst, rows, cols, ld);
    return check_launch("cast_rows_kernel");
}
