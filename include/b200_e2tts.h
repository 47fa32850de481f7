/*
 * b200_e2tts.h — C ABI of libb200e2tts.so: the sm_90a (H100) kernels behind the E2-TTS flow-matching hot path.
 *
 * This is the drop-in boundary described in SURVEY.md §8(b): plain pointers and sizes, no torch types.
 * Every entry point replaces an eager PyTorch op chain of the reference (file:line cited per function,
 * relative to e2_tts_pytorch/e2_tts.py of the original project; "A.n" = SURVEY.md Appendix A, the unvendored
 * x-transformers / hyper-connections leaves the reference composes).
 *
 * Conventions
 *   - all pointers are DEVICE pointers owned by the caller (inputs, outputs, saved tensors, workspaces);
 *     the library never allocates device memory and keeps no pointer after the call returns;
 *   - every function enqueues work on `stream` and returns immediately: 0 on success, negative on error
 *     (unsupported shape/flag, CUDA launch failure); `b200_last_error()` returns a thread-local message;
 *   - activations are bf16 (row-major, innermost dim contiguous), parameters that feed tensor-core GEMMs
 *     are bf16 packed by `b200_pack_weight`, small vectors / parameter gradients are fp32;
 *   - no host synchronisation, no allocation: every call is CUDA-graph capturable and re-entrant.
 */
#ifndef B200_E2TTS_H
#define B200_E2TTS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* b200_stream_t; /* cudaStream_t */

const char* b200_last_error(void);
int b200_version(void);
/* number of kernels launched by this library since load (per process; used for bench "gpu_launches") */
uint64_t b200_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core GEMM (wgmma + TMA):  D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )
 * Replaces every nn.Linear on the path: to_q/to_k/to_v/to_out (A.4), FeedForward GLU proj + out (A.2),
 * skip_proj :649/:895-896, TextAudioCrossCondition :503-513, proj_in/cond_proj_in :1267-1277, to_pred
 * :1296, and all of their backward contractions (dX = dY*W, dW = dY^T*X).
 *
 * A: bf16. a_mn_major=0: A stored [M,K] (lda = row pitch in elements); 1: A stored [K,M] (M contiguous).
 *    Optional second K source: k in [0,K1) from A, k in [K1,K) from A2 (same major-ness as A) — the concat
 *    of skip / cross-condition inputs is never materialised. K1 % 64 == 0.
 * B: bf16. b_mn_major=0: stored [N,K] (an nn.Linear weight); 1: stored [K,N].
 * Row pitches must be multiples of 8 elements (16 B, TMA requirement); M, N, K otherwise arbitrary.
 * Epilogue (applied in this order, each optional):
 *   + bias[n] (fp32)   * colscale[(m / rows_per_batch), n] (fp32, AdaLNZero gate :346-351)
 *   zero rows where rowmask[m]==0 (A.4 step 6)   + resid[m,n] (bf16)
 *   geglu!=0: GLU (A.2); B rows are packed [u(64) | gate(64)] per 128-column tile (b200_pack_weight mode 2);
 *            D2[M,N] <- pre-activation (bf16), D[M,N/2] <- u * act(gate) [* glu_mult] * dropout, where geglu selects act:
 *            1 = exact erf GELU, 2 = SiLU (x-transformers swish=True), 3 = ReLU^2 (relu_squared=True); other values are refused.
 *            glu_mult (fp32 [N/2], hidden-unit order, NULL = none): x-transformers GLU(mult_bias=True); refused without geglu.
 *            The dropout keep set and D2 do not depend on the activation or on glu_mult.
 *   split_k>1: fp32 atomic accumulation into D (D is zeroed by the call); d_fp32 must be 1. split_k<0: the library picks the
 *            split that fills the SMs once for the tile shape it selects (weight-gradient GEMMs: few tiles, very long K).
 */
typedef struct {
    const void* A; int64_t lda;
    const void* A2; int64_t lda2; int64_t K1;
    const void* B; int64_t ldb;
    int64_t M, N, K;
    int32_t a_mn_major, b_mn_major;
    void* D; int64_t ldd; int32_t d_fp32;
    void* D2; int64_t ldd2;
    const float* bias;
    const float* colscale; int64_t rows_per_batch;
    const uint8_t* rowmask;
    const void* resid; int64_t ldr;
    int32_t geglu; float dropout_p; uint64_t seed;
    int32_t split_k;
    int32_t force_tile;   /* 0 = auto, 1 = 128 x 128 CTA tiles, 2 = 256 x 128 CTA tiles (two MMAs per k-step share one B tile),
                           * 3 = 128 x 256 CTA tiles (one m64n256 MMA per warpgroup and k-step); auto picks 3 for M >= 512, N >= 256 */
    const uint64_t* seed_dev;   /* optional DEVICE word added to `seed` when the kernel runs (see "dropout seeds" below); NULL = none */
    const float* glu_mult;      /* optional GLU hidden-unit multiplier (see geglu above); NULL = none */
    int32_t act;                /* 0: none; 1: exact-erf GELU of (z + bias) ahead of the rest of the epilogue (Vocos ConvNeXt pwconv1 ->
                                 * nn.GELU, vocos/modules.py ConvNeXtBlock), the GLU epilogue's GELU polynomial. Needs K-major A and B, a
                                 * bf16 16-byte aligned D (TMA tile stores); refused with geglu, split_k > 1 or d_fp32. */
} b200_gemm_args;
int b200_gemm(const b200_gemm_args* a, b200_stream_t stream);

/* Dropout seeds. Every seeded entry point (GEGLU dropout in b200_gemm / b200_geglu_bwd, attention dropout) takes a host `seed`
 * (a kernel ARGUMENT) and an optional `seed_dev`: a DEVICE word read when the kernel runs, effective seed = seed + *seed_dev.
 * A captured CUDA graph freezes kernel arguments, so the per-step randomness of a graphed training step
 * (e2_tts_pytorch_b200.GraphedTrainStep; the reference draws a fresh torch RNG state every step, trainer.py:263) comes from that
 * one word, which b200_seed_advance() steps in stream order as the first node of the graph. The pointer travels in the args of
 * each call (the library keeps no pointer after a call returns: two models, or two threads capturing at once, cannot interfere). */
int b200_seed_advance(uint64_t* seed_dev, b200_stream_t stream);   /* *seed_dev = splitmix64 step of *seed_dev (one thread) */

/* ------------------------------------------------------------------------------------------------
 * Fused softclamped attention, dim_head (= dh) 64 or 128; any other value is refused (x-transformers Attend as configured by the
 * reference: A.4 steps 4-5, call sites e2_tts.py:875, :911). q,k,v,o: bf16 [B,H,Np,dh]; keymask: u8 [B,Np] (1 = keep) or
 * NULL; gate: fp32 [B*Np, H] = sigmoid(to_v_head_gate(x)) or NULL; og: bf16 [B*Np, H*dh] gated, merged
 * heads (the input of to_out); lse: fp32 [B,H,Np] (natural log of the softmax denominator of the CLAMPED
 * logits). Dropout on P uses a counter-based hash of (seed, b,h,i,j) that backward recomputes.
 * Logits: softclamp * tanh(scale q.k / softclamp) with softclamp in (0, 64] (x-transformers softclamp_logits), or, when
 * `unclamped` != 0, plain scale q.k (an online softmax with a running row maximum; softclamp must then be 0, and lse is the
 * log-sum-exp of the unclamped logits). A query row whose keys are all masked gives o = og = 0, lse = -inf and zero gradients in
 * both modes (the model never produces one: its register keys are always valid).
 */
typedef struct {
    const void *q, *k, *v;
    const uint8_t* keymask;
    const float* gate;
    void *o, *og;
    float* lse;
    int32_t B, H, Np, dim_head;
    float scale, softclamp, dropout_p;
    uint64_t seed;
    void* ws_maskbits;   /* workspace of b200_attn_workspace_bytes(B, Np) bytes (key-validity bitmask built by the call) */
    const uint64_t* seed_dev;   /* optional device addend of `seed` (dropout seeds, above) */
    int32_t maskbits_ready;     /* != 0: ws_maskbits already holds b200_attn_maskbits(keymask) — every layer of a forward/backward shares
                                   one key mask, so the model builds the bitmask once instead of once per attention call */
    int32_t unclamped;          /* != 0: no logit soft-clamp (softclamp must be 0); 0: clamped by softclamp */
} b200_attn_fwd_args;
size_t b200_attn_workspace_bytes(int32_t B, int32_t Np);
/* key-validity bitmask of `keymask` (u8 [B,Np], NULL = all valid) into ws_maskbits, in the layout the wgmma kernels read */
int b200_attn_maskbits(const uint8_t* keymask, void* ws_maskbits, int32_t B, int32_t Np, b200_stream_t stream);
/* wgmma / TMA kernel; clamped: softclamp must be in (0, 64] (the clamped softmax is exponentiated without a running maximum);
 * unclamped: softclamp must be 0 */
int b200_attn_fwd(const b200_attn_fwd_args* a, b200_stream_t stream);

/* backward, dim_head (= dh) 64 or 128: d_og bf16 [B*Np, H*dh] -> dk,dv bf16 [B,H,Np,dh], dq FP32 [B,H,Np,dh] (accumulated with
 * TMA reductions across key tiles), d_gate fp32 [B*Np,H] (grad wrt the sigmoid gate VALUE;
 * may be NULL). ws_dO (bf16 [B,H,Np,dh]), ws_delta (fp32 [B,H,Np]) and ws_maskbits are caller workspaces. */
typedef struct {
    const void *q, *k, *v, *o, *d_og;
    const uint8_t* keymask;
    const float *gate, *lse;
    void* ws_dO; float* ws_delta;
    float* d_gate;
    void *dq, *dk, *dv;
    int32_t B, H, Np, dim_head;
    float scale, softclamp, dropout_p;
    uint64_t seed;
    void* ws_maskbits;
    const uint64_t* seed_dev;   /* optional device addend of `seed` (must be the forward's) */
    int32_t maskbits_ready;     /* as in b200_attn_fwd_args */
    int32_t unclamped;          /* as in b200_attn_fwd_args (must be the forward's) */
} b200_attn_bwd_args;
int b200_attn_bwd(const b200_attn_bwd_args* a, b200_stream_t stream);   /* wgmma / TMA kernel, dq fp32; softclamp, unclamped as in fwd */

/* ------------------------------------------------------------------------------------------------
 * Hyper-connections (A.5; e2_tts.py:607, 673-678, 709-713, 870-882, 900-939), S = 4 residual streams held
 * as bf16 [T, S, D] (token-major), fused with the consumer's RMSNorm / AdaptiveRMSNorm (A.1; :875,881,908,937).
 * width fwd : xres -> branch [T,D] (normalised when norm_mode != 0), res_out [T,S,D], beta_out [T,S] fp32.
 *   norm_mode 0: none (conv sub-block); 1: * sqrt(D)/||.|| * norm_gain[D]; 2: * norm_gain[t / rows_per_batch, D]
 *   (norm_gain = 1 + to_gamma(cond), produced by b200_small_linear).
 * width bwd : d_branch [T,D], d_res [T,S,D], d_beta [T,S] -> d_xres [T,S,D]; parameter gradients are ADDED
 *   (fp32 atomics) into the g_* buffers, which the caller zero-initialises: g_norm_gain is [D] (mode 1) or
 *   [T/rows_per_batch, D] (mode 2).
 * Fused depth connection (optional, y_prev != NULL): the streams entering the width connection are
 *   xres + beta_prev (x) y_prev — the depth connection `residual' + beta * branch_out` of the PREVIOUS sub-block
 *   (A.5 add_residual) — and are never written to HBM: xres is then that sub-block's residual' [T,S,D], y_prev its branch
 *   output bf16 [T,D], beta_prev its beta fp32 [T,S]. bwd additionally returns d_y_prev bf16 [T,D], d_beta_prev fp32 [T,S]
 *   (d_xres is d residual'); it needs T*S % 64 == 0. Otherwise use b200_hc_depth_* between the sub-blocks.
 */
typedef struct {
    const void* xres;
    const float *norm_gamma, *dynamic_alpha_fn, *dynamic_alpha_scale, *static_alpha, *dynamic_beta_fn, *dynamic_beta_scale, *static_beta;
    int32_t norm_mode; const float* norm_gain; int32_t rows_per_batch;
    int32_t T, D, num_streams;
    void *branch, *res_out; float* beta_out;                 /* forward outputs */
    const void *d_branch, *d_res; const float* d_beta;       /* backward inputs */
    void* d_xres;
    float *g_norm_gamma, *g_dynamic_alpha_fn, *g_dynamic_alpha_scale, *g_static_alpha, *g_dynamic_beta_fn, *g_dynamic_beta_scale,
        *g_static_beta, *g_norm_gain;
    float* ws_records;   /* bwd workspace: T * 20 + D * 8 floats, 16-byte aligned: bf16 coefficient matrix [T*S (+T), 8] (T * 20 floats,
                            the T fused C' rows included), then the fp32 [D, 8] result of the parameter GEMM at byte offset 80 T */
    float* stats_out;    /* fwd (optional): fp32 [T, 32] per-token reduction results; bwd REQUIRES them back in `stats` (caller-owned) */
    const float* stats;
    const void* y_prev; const float* beta_prev;              /* fused preceding depth connection (both or neither) */
    void* d_y_prev; float* d_beta_prev;                      /* its backward outputs */
} b200_hc_width_args;
int b200_hc_width_fwd(const b200_hc_width_args* a, b200_stream_t stream);
int b200_hc_width_bwd(const b200_hc_width_args* a, b200_stream_t stream);

/* depth: out[t,s,:] = res[t,s,:] + beta[t,s] * y[t,:] (out may alias res);
 * bwd: d_y[t,:] = sum_s beta[t,s] d_out[t,s,:], d_beta[t,s] = <d_out[t,s,:], y[t,:]> (d_res == d_out). */
typedef struct {
    const void *res, *y; const float* beta; void* out;
    const void* d_out; void* d_y; float* d_beta;
    int32_t T, D, num_streams;
} b200_hc_depth_args;
int b200_hc_depth_fwd(const b200_hc_depth_args* a, b200_stream_t stream);
int b200_hc_depth_bwd(const b200_hc_depth_args* a, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Weight packing: ONE launch casts every fp32 nn.Parameter that feeds a tensor-core GEMM into its bf16 slot
 * (reference keeps fp32 nn.Linear weights; names per SURVEY Appendix B). `descs_dev` is a DEVICE array.
 *   mode 0: dst[(row_off + r) * ld_dst + col_off + c] = src[r * cols + c]
 *   mode 1: GEGLU interleave (A.2 `proj` weight/bias: rows [u(inner); gate(inner)] -> per 64 hidden units
 *           [u(64) | gate(64)]), so one 128-column GEMM tile holds both halves of the same hidden units.
 *   cols, col_off, ld_dst must be multiples of 4.  out_fp32 != 0 keeps fp32 (packed biases).
 */
typedef struct {
    const float* src; void* dst;
    int32_t rows, cols, ld_dst, row_off, col_off, mode, out_fp32, _pad;
} b200_pack_desc;
int b200_pack_weights(const b200_pack_desc* descs_dev, int32_t n, b200_stream_t stream);

/* Flow-matching stem (e2_tts.py:1519-1543 and the operand of proj_in/cond_proj_in :1267-1277):
 *   training: A[row] = [ (1-t) x0 + t x1 | pad | where(span, 0, x1) | pad ] (bf16, 2*Cp columns), cond_out fp32
 *   direct  : x_in / cond_in given (sampling, transformer_with_pred_head).  Cp = C rounded up to 64.
 *   concat_cond != 0 (E2TTS(concat_cond=True), :1263-1265): A[row] = [ cond (C) | x (C) | pad ] = cat(cond, x), the operand of the
 *   single Linear(2C -> dim) proj_in of that variant (:1201). */
typedef struct {
    const float *x1, *x0, *times; const uint8_t* span;   /* training mode */
    const float *x_in, *cond_in;                          /* direct mode (x1 == NULL) */
    void* A; float* cond_out;
    int32_t B, N, C, Cp;
    int32_t concat_cond;
} b200_stem_args;
int b200_stem_prepare(const b200_stem_args* a, b200_stream_t stream);

/* Residual-stream assembly (e2_tts.py:760-771, 800-801, 818-821; CharacterEmbed :400-412):
 *   out[b, r, s, :]     = registers[r, :]                         r < R
 *   out[b, R+n, s, :]   = (h[b*N+n, :] | emb[ids[b,n], :]) + abs_pos[n, :]     for every stream s
 * bwd: d_h (bf16) or d_tok (fp32, for b200_embed_bwd), d_abs_pos [N,D], d_registers [R,D] (all overwritten). */
typedef struct {
    const void* h; const int32_t* ids; const float *emb, *abs_pos, *registers;
    void* out;
    const void* d_out; void* d_h; float *d_tok, *d_abs_pos, *d_registers;
    int32_t B, N, R, D, S;
} b200_assemble_args;
int b200_assemble_fwd(const b200_assemble_args* a, b200_stream_t stream);
int b200_assemble_bwd(const b200_assemble_args* a, b200_stream_t stream);
int b200_embed_bwd(const float* d_tok, const int32_t* ids, float* d_emb, int32_t ntok, int32_t D, int32_t vocab, b200_stream_t stream);

/* Rotary table cos/sin [Np, dim_head / 2], dim_head 64 or 128: inv_freq_i = 10000^(-2i / dim_head), positions 0..Np-1 including
 * registers (A.3; e2_tts.py:793, :798). */
int b200_rotary_table(float* cos_out, float* sin_out, int32_t Np, int32_t dim_head, b200_stream_t stream);

/* Post-processing of the fused [q|k|v|gate|mix] projection (A.4 steps 1-3, 5): interleaved-pair rotary on
 * q,k; v = lerp(v_first, v, sigmoid(mix)) when v_first != NULL; gate = sigmoid(gate_logit + bias) fp32 [T,H];
 * q,k,v written as [B,H,Np,dim_head], I = H * dim_head, dim_head 64 or 128 (rot_cos / rot_sin: the table of that dim_head).
 * bwd inverts all of it into d_qkvg (same packed layout) and d_vfirst.
 * no_gate != 0 (x-transformers Attention without gate_value_heads): the layout is [q|k|v|mix], the mix logits at column 3I;
 * gate, gate_bias and d_gate are then neither read nor written (may be NULL). */
typedef struct {
    const void* qkvg; int32_t ld;
    const float *gate_bias, *mix_bias, *rot_cos, *rot_sin;
    const void* v_first;
    void *q, *k, *v; float* gate;
    const void *dq, *dk, *dv; const float* d_gate;
    const void* dv_extra;   /* optional bf16 [B,H,Np,dim_head] added to dv (value-residual gradients of later layers into layer 0) */
    void *d_qkvg, *d_vfirst;
    int32_t B, H, Np, dim_head;
    int32_t dq_fp32;   /* bwd: dq is fp32 (wgmma attention backward) instead of bf16 */
    int32_t no_gate;   /* != 0: no head-gate column (layout above) */
} b200_qkv_post_args;
int b200_qkv_post_fwd(const b200_qkv_post_args* a, b200_stream_t stream);
int b200_qkv_post_bwd(const b200_qkv_post_args* a, b200_stream_t stream);

/* GEGLU backward on the packed pre-activations saved by b200_gemm(geglu=1) (A.2); db_packed (fp32 [2*inner], packed order,
 * zeroed by the caller, may be NULL) receives the bias gradient of the GLU projection in the same pass. */
int b200_geglu_bwd(const void* dh, const void* ug, void* dug, float* db_packed, int64_t T, int32_t inner, float dropout_p, uint64_t seed,
                   const uint64_t* seed_dev, b200_stream_t stream);
/* GLU backward of any activation of b200_gemm's GLU epilogue (A.2; b200_geglu_bwd is act = 1 with mult = NULL, bit for bit).
 * dh bf16 [T, inner] (gradient of the GLU output h = drop(u * act(g) [* mult])), ug bf16 packed pre-activations [T, 2*inner] ->
 * dug bf16 packed. db_packed (fp32 [2*inner], packed order, may be NULL) += column sums of the bf16 dug. mult (fp32 [inner],
 * hidden-unit order) may be NULL; d_mult (fp32 [inner], may be NULL, needs mult) += sum over rows of drop(dh) * u * act(g).
 * db_packed and d_mult are zeroed by the caller. act: 1 GELU, 2 SiLU, 3 ReLU^2. Dropout: the hash of the forward epilogue. */
typedef struct {
    const void* dh; const void* ug; void* dug; float* db_packed;
    const float* mult; float* d_mult;
    int64_t T; int32_t inner; int32_t act;
    float dropout_p; uint64_t seed; const uint64_t* seed_dev;
} b200_glu_bwd_args;
int b200_glu_bwd(const b200_glu_bwd_args* a, b200_stream_t stream);
/* out[n] += sum_t X[t,n] (bf16 X, fp32 out; caller zeroes out) — nn.Linear bias gradients. */
int b200_colsum(const void* X, int64_t T, int32_t ncols, int32_t ld, float* out, b200_stream_t stream);

/* Drop registers, sum the S streams, final RMSNorm (e2_tts.py:943-952). y bf16 [B*N, D].
 * Branch-norm mode (rows_per_batch > 0): the pre-norm of a plain residual sub-block (Transformer(num_residual_streams=1),
 *   e2_tts.py:870-882, 900-939): y[r] = F.normalize(x[r]) * sqrt(D) * gain, on rows x bf16 [B*N, D]; requires S == 1, R == 0 and
 *   (B*N) % rows_per_batch == 0. gains == NULL: RMSNorm, gain = g [D], bwd ADDS into g_g [D]; gains != NULL: AdaptiveRMSNorm,
 *   gain = gains[r / rows_per_batch] (fp32 [B*N / rows_per_batch, D], the 1 + gamma of b200_small_linear; g unused), bwd ADDS
 *   into d_gains (same shape, zeroed by the caller; g_g unused). A zero row gives y = 0 and the finite gradient of F.normalize
 *   (the norm clamped at 1e-12). bwd: d_res (optional bf16 [B*N, D]), the gradient of the residual path around the norm, is added
 *   into d_xres. All four fields zero: the final norm above. */
typedef struct {
    const void* xres; const float* g; void* y;
    const void* dy; void* d_xres; float* g_g;   /* bwd: d_xres [B,R+N,S,D] fully written, g_g accumulated */
    int32_t B, N, R, D, S;
    int32_t rows_per_batch; const float* gains; float* d_gains; const void* d_res;   /* branch-norm mode (above) */
} b200_final_norm_args;
int b200_final_norm_fwd(const b200_final_norm_args* a, b200_stream_t stream);
int b200_final_norm_bwd(const b200_final_norm_args* a, b200_stream_t stream);

/* Masked-MSE flow-matching loss (e2_tts.py:1535, 1580-1582, 1595) without the boolean gather / host sync:
 * flow = sum_{span}(pred - (x1 - x0))^2 / (count * C); pred_data = x0 + pred. sums is a 4-float workspace that
 * must be kept for backward; dpred is bf16 [rows, ldp] (pad columns zero) = dloss * d(loss)/d(pred).
 * Velocity-consistency term (e2_tts.py:1556-1576, 1586-1589), when vel_target != NULL (the EMA model's no-grad prediction at
 * t + delta, fp32 [rows, C]):  velocity = sum_{span}(pred - vel_target)^2 / (count * C),  loss = flow + vel_weight * velocity;
 * loss_parts (optional, 2 floats) receives {flow, velocity} for the reference's LossBreakdown. */
typedef struct {
    const float *pred, *x1, *x0; const uint8_t* span;
    float *sums, *loss, *pred_data;
    const float* dloss; void* dpred; int32_t ldp;
    int64_t rows; int32_t C;
    const float* vel_target; float vel_weight; float* loss_parts;
} b200_flow_loss_args;
int b200_flow_loss_fwd(const b200_flow_loss_args* a, b200_stream_t stream);
int b200_flow_loss_bwd(const b200_flow_loss_args* a, b200_stream_t stream);

/* Backward of the GEMM epilogue y = rowmask * colscale[b,:] * (z + bias) (AdaLNZero gate :346-351, A.4 step 6):
 * dz = dy * mask * cs (bf16), d_cs[b,:] += sum_rows dy * y / cs (fp32, caller zeroes), and when d_bias != NULL
 * d_bias[:] += sum_rows dz (fp32 [D], caller zeroes). cs/mask/d_bias may be NULL. */
int b200_rowgate_bwd(const void* dy, const void* y, const float* cs, const uint8_t* mask, void* dz, float* d_cs,
                     float* d_bias, int32_t B, int32_t rows_per_batch, int32_t D, b200_stream_t stream);
/* The same for an epilogue that also added a residual, y = rowmask * colscale * (z + bias) + resid (the fused residual add of a plain
 * residual sub-block): the gate gradient reads the branch value as y - resid (bf16 resid, required), so it carries the bf16 rounding
 * of the sum y (at most 2^-9 |y| per element). dz and d_bias are those of b200_rowgate_bwd; resid's own gradient is dy. */
int b200_rowgate_resid_bwd(const void* dy, const void* y, const void* resid, const float* cs, const uint8_t* mask, void* dz, float* d_cs,
                           float* d_bias, int32_t B, int32_t rows_per_batch, int32_t D, b200_stream_t stream);
int b200_cast_rows(const float* src, void* dst, int64_t rows, int32_t cols, int32_t ld, b200_stream_t stream);
/* InterpolatedCharacterEmbed (e2_tts.py:414-482; E2TTS(interpolated_text=True) :1135, :1233): the per-token front half of
 *   te[b, n] = mask[b, n] * ( lerp[b, n] + Linear2( silu( pos[b, n] * w1 + b1 ) ) )
 * ids: int32 [B, nt] COMPACTED character ids (the first text_len[b] are the valid ones, :445-447); audio_len[b] = frames of sample b
 * (mask.sum or N, :455-457). fwd writes lerp bf16 [B*N, D] = linear interpolation of the sample's embeddings to audio_len[b] frames
 * (F.interpolate 'bilinear', align_corners=False; rows beyond audio_len: 0) and h1 bf16 [B*N, D] = silu(pos * w1 + b1) with
 * pos = linspace(0, text_len, audio_len) (0 beyond). Linear2 (+ bias, + lerp as residual, row mask) is b200_gemm.
 * bwd: d_lerp, d_h1 bf16 [B*N, D] -> d_emb fp32 [vocab, D], d_w1, d_b1 fp32 [D] (all ADDED into zero-initialised buffers). */
typedef struct {
    const int32_t* ids; const int32_t *text_len, *audio_len;
    const float *emb, *w1, *b1;
    int32_t B, N, nt, D, vocab;
    void *lerp, *h1;                       /* forward outputs */
    const void *d_lerp, *d_h1;             /* backward inputs */
    float *d_emb, *d_w1, *d_b1;
} b200_interp_text_args;
int b200_interp_text_fwd(const b200_interp_text_args* a, b200_stream_t stream);
int b200_interp_text_bwd(const b200_interp_text_args* a, b200_stream_t stream);

/* LinearFourierEmbed (e2_tts.py:368-386; Transformer(attn_fourier_embed_input=True) :545-546, applied to the attention input :909):
 * the Linear(dim -> df + dr, no bias) is b200_gemm; this is its tail, z bf16 [T, df + dr] (row pitch ldz) ->
 * out bf16 [T, 2*df + dr] = cat(sin(z[:, :df]), cos(z[:, :df]), z[:, df:]). bwd: d_out -> dz bf16 [T, ldz] (padding columns zeroed). */
int b200_fourier_feat_fwd(const void* z, int64_t ldz, void* out, int64_t T, int32_t df, int32_t dr, b200_stream_t stream);
int b200_fourier_feat_bwd(const void* d_out, const void* z, int64_t ldz, void* dz, int64_t T, int32_t df, int32_t dr, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Small-batch fp32 linear (time conditioning path: time_cond_mlp e2_tts.py:621-625, all AdaptiveRMSNorm /
 * AdaLNZero to_gamma projections A.1 / :346-351 batched into one call, HLGaussLayer head A.6):
 *   Z[b,n] = sum_k X[b,k] W[n,k] + bias[n];  Y = act(Z).  B <= 64 rows.
 *   act: 0 identity, 1 SiLU, 2 sigmoid, 3 (1 + z), 4 softplus, 5 alternating per `seg` outputs: (1+z), sigmoid
 * bwd: dX (overwritten), dW, dbias (overwritten) from dY, Z. */
typedef struct {
    const float *X, *W, *bias; float *Z, *Y;
    const float* dY; float *dZ, *dX, *dW, *dbias;
    int32_t B, N, K, act, seg;
    int32_t seg_major;   /* != 0: Y/Z/dY/dZ are laid out [N/seg][B][seg] so every `seg`-wide output block is a contiguous [B, seg] matrix */
} b200_small_linear_args;
int b200_small_linear_fwd(const b200_small_linear_args* a, b200_stream_t stream);
int b200_small_linear_bwd(const b200_small_linear_args* a, b200_stream_t stream);
/* RandomFourierEmbed (e2_tts.py:355-364): out[b] = [t, sin(2 pi t w), cos(2 pi t w)], out [B, 2*half+1] */
int b200_fourier_embed(const float* times, const float* weights, float* out, int32_t B, int32_t half, b200_stream_t stream);

/* Masked depthwise conv k (odd, <= 31) + SiLU (DepthwiseConv e2_tts.py:295-328) on bf16 [B, Np, D]:
 *   y = m * silu(conv1d_depthwise(m * x) + bias), weight fp32 [D, k]. fwd also stores the bf16 pre-activation (conv + bias) into
 *   `pre` [B, Np, D] when it is non-null; bwd REQUIRES it (caller-owned, like every saved tensor) instead of recomputing the
 *   convolution. dweight/dbias are ADDED into zero-initialised fp32 buffers.
 *   residual != 0 (the plain residual sub-block x + DepthwiseConv(x, mask), e2_tts.py:870-872, 900-902): y = x + m * silu(...), the
 *   add itself unmasked (a masked row keeps x bit for bit) and rounded once; bwd dx = dy + the convolution's dx. y must not alias x. */
typedef struct {
    const void* x; const uint8_t* mask; const float *weight, *bias; void* y;
    const void* dy; void* dx; float *dweight, *dbias;
    int32_t B, Np, D, ksize;
    void* pre;
    int32_t residual;
} b200_dwconv_args;
int b200_dwconv_fwd(const b200_dwconv_args* a, b200_stream_t stream);
int b200_dwconv_bwd(const b200_dwconv_args* a, b200_stream_t stream);

/* HL-Gauss classification head of DurationPredictor(hl_gauss_loss=..., use_regression=False) (e2_tts.py:966-967 ctor arguments,
 * :1035-1040 HLGaussLayer, :1107 prediction, :1111 loss against lens.float(); hl-gauss-pytorch HLGaussLoss, SURVEY A.6) on fp32
 * logits [B, num_bins] (b200_small_linear, identity activation). One CTA per item; 1 <= B <= 64, 2 <= num_bins <= 4096.
 *   Edges s_j = min + j (max - min) / num_bins (s_N = max), centres (s_i + s_{i+1}) / 2, x_j = (s_j - y) / (sqrt(2) sigma) with
 *   y = target[b], clamped to [min, max] when clamp_to_range. Masses erf(x_{i+1}) - erf(x_i), taken through erfc where both lie on
 *   one side of 0; p = mass / (erf(x_N) - erf(x_0)), NaN where that fp32 difference of erf values is 0, as the reference's.
 * fwd, target != NULL (training): ce[b] = -sum_i p_i log_softmax(l)_i (max-shifted), diff [B, num_bins] = softmax - p (saved for the
 *   backward), *loss = mean_b ce[b], summed in item order by the last CTA (no float atomics: the same bits on every launch).
 *   ws_count: one zeroed 32-bit word, left zero again by the call (the last CTA is found by atomicInc wrapping at B - 1).
 * fwd, target == NULL (prediction): pred[b] = sum_i softmax(l)_i centre_i.
 * bwd: dlogits = (*dloss / B) * diff; dloss is read on the device (graph-capturable). */
typedef struct {
    const float *logits, *target;
    float *pred, *ce, *loss, *diff;
    uint32_t* ws_count;
    const float* dloss; float* dlogits;
    int32_t B, num_bins;
    float min_value, max_value, sigma;
    int32_t clamp_to_range;
} b200_hl_gauss_args;
int b200_hl_gauss_fwd(const b200_hl_gauss_args* a, b200_stream_t stream);
int b200_hl_gauss_bwd(const b200_hl_gauss_args* a, b200_stream_t stream);

/* Masked mean over the sequence (maybe_masked_mean e2_tts.py:212-224): x bf16 [B,N,D] -> out fp32 [B,D]; bwd. */
int b200_masked_mean_fwd(const void* x, const uint8_t* mask, float* out, int32_t B, int32_t N, int32_t D, b200_stream_t stream);
int b200_masked_mean_bwd(const float* dout, const uint8_t* mask, void* dx, int32_t B, int32_t N, int32_t D, b200_stream_t stream);

/* Fixed-grid ODE update out = y + a * f (torchdiffeq midpoint/euler as called at e2_tts.py:1421; SURVEY A.7). */
int b200_axpy(const float* y, const float* f, float a, float* out, int64_t n, b200_stream_t stream);
/* ------------------------------------------------------------------------------------------------
 * Runge–Kutta solver passes of E2TTS.sample for odeint_kwargs methods 'rk4', 'dopri5', 'bosh3', 'fehlberg2' and 'adaptive_heun'
 * (the odeint call at e2_tts.py:1421 with odeint_kwargs :1122-1126; torchdiffeq 0.2.x restated in SURVEY A.7). The ODE state is
 * the whole padded [B, max_duration, C] fp32 tensor of n elements; k0..k{S-1} are function evaluations (stage derivatives) of the
 * same size; the weights (tableau entry times the step size, rounded to fp32) are formed on the host. Memory-bound fp32 passes,
 * float4-vectorised when every pointer is 16-byte aligned, scalar otherwise and for the n % 4 tail. S is 1..7 (dopri5 has 7 stages).
 *
 * Reductions (step_error, norms) accumulate fp32 quotients squared in fp64: each block writes its partial sum to ws, one more block
 * adds the partials in a fixed order and writes the root mean square as fp32. The grid is min(ceil(n / 1024), ws_len) blocks
 * whatever the device, so the result is bit-identical from run to run; an n larger than the grid covers is wrapped by a grid-stride
 * loop. */

/* out = y0 + sum_j w_j k_j (the sum is formed first, then added to y0: torchdiffeq's y0 + k.matmul(beta * dt)). Replaces the stage
 * inputs of _runge_kutta_step (rk_common.py, `yi = y0 + k[..., :i + 1].matmul(beta_i * dt)`), its `y1` of a tableau without
 * first-same-as-last, and rk4_alt_step_func's update (fixed_grid.py / misc: (k1 + 3 (k2 + k3) + k4) dt / 8). out may alias y0. */
typedef struct {
    const float* y0;
    const float *k0, *k1, *k2, *k3, *k4, *k5, *k6;
    float w0, w1, w2, w3, w4, w5, w6;
    int32_t S;
    float* out;
    int64_t n;
} b200_ode_combine_args;
int b200_ode_combine(const b200_ode_combine_args* a, b200_stream_t stream);

/* The error estimate and its norm of one adaptive step (_adaptive_step, rk_common.py: `y1_error = k.matmul(dt * c_error)`,
 * `error_tol = atol + rtol * max(|y0|, |y1|)`, `error_ratio = rms_norm(y1_error / error_tol)`) in one pass:
 *   write_y1 != 0: y1 = y0 + sum_j s_j k_j is computed and stored (a tableau without first-same-as-last);
 *   write_y1 == 0: y1 is read (dopri5 / bosh3: the last stage input is the solution).
 * ratio[0] = sqrt(mean((sum_j e_j k_j / tol)^2)) in fp32. ws: ws_len doubles (1..65535). atol, rtol: finite, >= 0. */
typedef struct {
    const float* y0;
    const float *k0, *k1, *k2, *k3, *k4, *k5, *k6;
    float e0, e1, e2, e3, e4, e5, e6;
    float s0, s1, s2, s3, s4, s5, s6;
    int32_t S;
    float* y1;
    int32_t write_y1;
    float atol, rtol;
    double* ws;
    int32_t ws_len;
    float* ratio;
    int64_t n;
} b200_ode_step_error_args;
int b200_ode_step_error(const b200_ode_step_error_args* a, b200_stream_t stream);

/* The scaled norms of the initial step size (_select_initial_step, misc.py): scale = atol + |y0| rtol,
 *   out[0] = rms(a / scale) when a is non-null (d0 with a = y0),
 *   out[1] = rms((b - c) / scale), or rms(b / scale) when c is NULL (d1 with b = f0; d2 * h0 with b = f(t0 + h0, y0 + h0 f0), c = f0).
 * ws: 2 * ws_len doubles (ws_len 1..65535). atol, rtol: finite, >= 0. */
typedef struct {
    const float *y0, *a, *b, *c;
    float atol, rtol;
    double* ws;
    int32_t ws_len;
    float* out;
    int64_t n;
} b200_ode_norms_args;
int b200_ode_scaled_norms(const b200_ode_norms_args* a, b200_stream_t stream);

/* Dense output of the last accepted step at x = (t - t0) / (t1 - t0) (RKAdaptiveStepsizeODESolver._interp_fit + interp.py
 * _interp_fit / _interp_evaluate): y_mid = y0 + sum_j m_j k_j (m_j = dt c_mid_j), f0 = k0, f1 = k{S-1}, the quartic
 * e + x d + x^2 c + x^3 b + x^4 a with e = y0, d = dt f0, c = dt (f1 - 4 f0) - 11 y0 - 5 y1 + 16 y_mid,
 * b = dt (5 f0 - 3 f1) + 18 y0 + 14 y1 - 32 y_mid, a = 2 dt (f1 - f0) - 8 (y1 + y0) + 16 y_mid, all in fp32, without storing them. */
typedef struct {
    const float *y0, *y1;
    const float *k0, *k1, *k2, *k3, *k4, *k5, *k6;
    float m0, m1, m2, m3, m4, m5, m6;
    int32_t S;
    float dt, x;
    float* out;
    int64_t n;
} b200_ode_dense_args;
int b200_ode_dense_output(const b200_ode_dense_args* a, b200_stream_t stream);

/* Classifier-free guidance with the APG orthogonal projection in fp64 (e2_tts.py:1323-1330, project :113-124):
 * out = pred + (orth + par * keep) * strength per sample over all n*d elements. ws_red: 2*B doubles. */
int b200_cfg_combine(const float* pred, const float* null_pred, double* ws_red, float* out, int32_t B, int64_t per_sample,
                     float cfg_strength, int32_t remove_parallel, float keep_parallel_frac, b200_stream_t stream);
/* MelSpec (e2_tts.py:248-290, torchaudio MelSpectrogram with the reference's mel_spec_kwargs) -> log(clamp(mel, 1e-5)):
 * wave fp32 [B, nw] -> log-mel fp32 [B, n_mels, frames]; window fp32 [win_length] (the periodic Hann window, unpadded: its taps sit
 * at (n_fft - win_length)/2 .. of each n_fft frame, zeros elsewhere, as torch.stft pads it); fb fp32 [n_fft/2+1, n_mels] (HTK or
 * Slaney-scaled: any filterbank works, only its non-zero band per filter is read).
 *   center != 0: reflect-padded by n_fft/2 on both sides, frames = 1 + (nw + 2 (n_fft/2) - n_fft) / hop (= 1 + nw/hop for even
 *                n_fft); needs nw > n_fft/2.
 *   center == 0: valid frames only, frames = 1 + (nw - n_fft) / hop; needs nw >= n_fft.
 *   bin k: (|X_k| * norm_scale)^power (power 1: |X_k| exactly; normalize=True / 'window': norm_scale = 1/sqrt(sum window^2);
 *          'frame_length': 1/sqrt(n_fft); none: 1).
 * Refused before any launch: n_fft outside [64, 4096] or with a prime factor other than 2, 3 and 5; power <= 0 (a complex spectrum,
 * power=None, is not a log-mel); win_length outside [1, n_fft]; norm_scale <= 0. Power-of-two n_fft runs a radix-2 FFT, the others
 * a mixed-radix (4/2/3/5) Stockham FFT, both in shared memory.
 * ws_bands: caller workspace of 2 * n_mels int32 (8-byte aligned), filled by the call with each filter's non-zero bin range.
 * On-device collate (trainer.py:61-82 collate_fn + :101-131 HFDataset.__getitem__, SURVEY §8f row 3): wave_lens (optional int32 [B]) =
 * samples per sequence of a zero-padded ragged batch (a length past nw counts as nw) — sequence b yields the frame count above for
 * its own length (reflect-padded at its own end when centred), the remaining frames are the collate's zero padding. A sequence
 * too short for one frame (wave_lens[b] <= n_fft/2 centred — the reference's MelSpec raises on it — or < n_fft without centring) has
 * all its frames written as zeros. out_bnd != 0 writes [B, frames, n_mels] (the layout E2TTS.forward consumes, trainer.py:253
 * rearrange 'b d n -> b n d') instead of the reference MelSpec's [B, n_mels, frames]. */
typedef struct {
    const float *wave, *window, *fb; float* out;
    int32_t B, nw, n_fft, hop, n_mels;
    int32_t* ws_bands; const int32_t* wave_lens; int32_t out_bnd;
    int32_t win_length;   /* taps of `window`, 1..n_fft */
    int32_t center;
    float power;          /* > 0 */
    float norm_scale;     /* > 0; 1 = not normalised */
} b200_melspec_args;
int b200_melspec_ex(const b200_melspec_args* a, b200_stream_t stream);
/* The defaults of b200_melspec_ex (win_length = n_fft, center, power 1, norm_scale 1): same code, same bits. */
int b200_melspec(const float* wave, const float* window, const float* fb, float* out, int32_t B, int32_t nw, int32_t n_fft,
                 int32_t hop, int32_t n_mels, int32_t* ws_bands, const int32_t* wave_lens, int32_t out_bnd, b200_stream_t stream);

/* Resampling ahead of the mel (trainer.py:116-118: HFDataset.__getitem__ builds torchaudio.transforms.Resample(sample_rate, target)
 * for every item whose rate is not the target and applies it in fp32): a ragged batch of mixed rates in ONE launch.
 * wave fp32 [B, nw] with wave_lens int32 [B] (clamped to [0, nw]; samples at or past an item's length count as zero and are never
 * read); pair_idx int32 [B]: the item's rate pair in the table below, or < 0 to pass the item through unchanged (equal rates).
 * Rate pair p (orig', new': the rates reduced by their gcd; width: torchaudio's ceil(6 orig' / (0.99 min(orig', new')))):
 *   out[b, j] = sum_i taps[i] * x[s + i] over the band of phase k = j mod new', s = (j div new') orig' - width + first[k], the taps
 *   summed in increasing i by one fma chain (a fixed order: an item gives the same bits alone or in any batch);
 *   out_lens[b] = min(ceilf((float)((double)(new' L) / orig')), new' (L div orig' + 1), nr) for L = wave_lens[b] (torchaudio's
 *   length: its ceil runs in float32); a passed-through item has out_lens[b] = min(L, nr) and out[b, j] = x[j], bit for bit.
 *   out[b, j] = +0 for out_lens[b] <= j < nr. A pair_idx >= n_pairs gives out_lens[b] = 0.
 * The table is the banded form of torchaudio's fp32 taps (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99): per phase only
 * the contiguous run of non-zero taps, in three caller-built device arrays:
 *   pairs  int32 [n_pairs * 6]: orig', new', width, first phase (index into phases / 3), first tap (index into taps), taps of the pair;
 *   phases int32 [3 per phase]: first non-zero column of the phase's row in torchaudio's [new', 2 width + orig'] table, count, offset
 *          of its taps from the pair's first tap;
 *   taps   fp32: each pair's bands, phase after phase.
 * max_pair_words >= 3 new' + taps of every pair: when it is at most 12288 (48 KB) each block stages its item's pair in shared
 *   memory, otherwise the taps are read from global memory.
 * Refused before any launch: B < 1, nw < 0, nr < 0, n_pairs < 0, max_pair_words < 0, a missing pointer. */
typedef struct {
    const float* wave; const int32_t* wave_lens; const int32_t* pair_idx;
    const int32_t *pairs, *phases; const float* taps;
    float* out; int32_t* out_lens;
    int32_t B, nw, nr, n_pairs, max_pair_words;
} b200_resample_args;
int b200_resample(const b200_resample_args* a, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Vocos mel decoder (the reference's E2TTS(use_vocos=True): Vocos.from_pretrained e2_tts.py:1244, decode of each sampled mel
 * :1440-1451; published vocos package: VocosBackbone with ConvNeXt blocks, ISTFTHead with 'same' padding). Inference only.
 * A ragged batch is held as rows [B * T] (T = the longest item, row b * T + t = frame t of item b) with lens[b] frames per item
 * (int32 [B], 1 <= lens[b] <= T); every kernel treats item b as if it were decoded alone.
 *
 * im2col of the backbone's embed Conv1d(C -> dim, k 7, pad 3): mel fp32 [B, T, C] -> A bf16 [B * T, lda], column c * 7 + j =
 *   mel[b, t + j - 3, c], 0 outside [0, lens[b]) and on rows t >= lens[b]; columns 7C .. lda-1 are 0 (lda % 8 == 0, >= 7C). The embed
 *   is then one b200_gemm against the Conv1d weight viewed [dim, 7C]. db_to_amp != 0: each value is 10^(x / 20) (torchaudio
 *   DB_to_amplitude(x, ref=1, power=0.5), e2_tts.py:1444), formed in double and rounded to fp32, before the bf16 rounding. */
int b200_vocos_im2col(const float* mel, const int32_t* lens, void* A, int32_t B, int32_t T, int32_t C, int32_t lda, int32_t db_to_amp,
                      b200_stream_t stream);
/* LayerNorm over D channels (nn.LayerNorm(dim, eps) of the backbone: `norm`, `final_layer_norm`, each block's `norm`), bf16 x / y
 * [B * T, D] with fp32 math, D a multiple of 64 up to 1024; rows t >= lens[b] are written as zeros and never read.
 * b200_vocos_dwconv_ln first applies the block's masked depthwise Conv1d(k 7, pad 3) + bias (conv_w fp32 [D, 7], conv_b [D]), zero-
 * padded at the item's own ends; b200_vocos_ln is the LayerNorm alone (conv_w, conv_b unused). y must not alias x. */
typedef struct {
    const void* x; const int32_t* lens;
    const float *conv_w, *conv_b, *ln_w, *ln_b;
    void* y;
    int32_t B, T, D; float eps;
} b200_vocos_ln_args;
int b200_vocos_dwconv_ln(const b200_vocos_ln_args* a, b200_stream_t stream);
int b200_vocos_ln(const b200_vocos_ln_args* a, b200_stream_t stream);
/* ISTFTHead('same') after its Linear (vocos/heads.py ISTFTHead.forward + vocos/spectral_ops.py ISTFT): spec fp32 [B * T, n_fft + 2] =
 * [log-magnitude (n_fft/2 + 1) | phase (n_fft/2 + 1)]; S = min(exp(mag), 1e2) (cos p + i sin p); per frame irfft(S, n_fft) (the
 * imaginary parts of bins 0 and n_fft/2 are dropped) times window fp32 [n_fft], written to the caller's workspace frames fp32
 * [B * T, n_fft]; then each output sample sums its frames in increasing frame order (no atomics: deterministic), with the
 * overlap-added window^2 envelope of the item's own frames, trimmed by (n_fft - hop) / 2 at both ends: audio fp32 [B, T * hop],
 * item b holding lens[b] * hop samples and exact zeros after them. Refused: n_fft not a power of two in [64, 4096], hop outside
 * [1, n_fft], (n_fft - hop) odd. Lengths are read on the device and clamped to [0, T] (the host wrapper refuses lengths < 1
 * before any launch). Two launches. */
typedef struct {
    const float* spec; const float* window; const int32_t* lens;
    float* frames; float* audio;
    int32_t B, T, n_fft, hop;
} b200_vocos_istft_args;
int b200_vocos_istft(const b200_vocos_istft_args* a, b200_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Around the forward/backward step (SURVEY §8e, §8f row 1): multi-tensor gradient gather for ONE ncclAllReduce per step, global
 * gradient norm, and a fused clip + Adopt + EMA update. Parameters stay separate fp32 tensors (the reference's nn.Parameters);
 * gradients, optimizer state (m, v) and the EMA copy are flat fp32 buffers owned by the caller, addressed through a chunk table:
 * one entry per piece (<= 65536 elements) of a parameter, `ptr` = that piece inside the parameter (or its gradient tensor),
 * `flat_offset` = its element offset in the flat buffers (multiples of 4 keep the 16-byte vector path). One CTA per chunk.
 */
typedef struct { void* ptr; int64_t flat_offset; int32_t n; int32_t pidx; /* index of the parameter this piece belongs to */ } b200_chunk;
/* flat[flat_offset + i] = scale * ptr[i]; a NULL ptr (no gradient this step: the text stream when the text is dropped,
 * trainer.py:155 find_unused_parameters) zero-fills its slot. scale = 1/world_size gives DDP's gradient averaging (trainer.py:270).
 * used (optional, fp32 [n_params]): used[pidx] = 1 if the parameter had a gradient else 0 — summed by the same all-reduce when it
 * lies right behind the gradients, it tells the optimiser which parameters no rank touched (torch optimisers skip grad=None). */
int b200_flat_gather(const b200_chunk* chunks_dev, int32_t n_chunks, float* flat, float scale, float* used, b200_stream_t stream);
/* Gradient accumulation over micro-batches (trainer.py grad_accumulation_steps): flat[flat_offset + i] = fmaf(scale, ptr[i],
 * flat[flat_offset + i]), ONE fp32 rounding per element. A NULL ptr (no gradient on this micro-step) leaves its slot untouched;
 * used[pidx] (optional) is set to 1 where ptr is non-NULL and never cleared, so over the micro-steps it is the OR of the presence
 * flags (torch: p.grad is None only if no micro-step produced one). The 4-element padding between parameters is never written.
 * No allocation, no host sync: capturable. scale = 1 / (steps * world_size) gives accelerate's loss / steps and DDP's average. */
int b200_flat_accumulate(const b200_chunk* chunks_dev, int32_t n_chunks, float* flat, float scale, float* used, b200_stream_t stream);
/* ptr[i] = flat[flat_offset + i] (e.g. EMA weights into a module's parameters) */
int b200_flat_scatter(const b200_chunk* chunks_dev, int32_t n_chunks, const float* flat, b200_stream_t stream);
/* *out = sum x[i]^2 (out: ONE device float, overwritten): torch.nn.utils.clip_grad_norm_'s total norm, trainer.py:272-273.
 * Deterministic: the block partials are added in block order, so equal inputs give a bit-identical norm. The partials live in one
 * static device buffer, so calls on one device must be ordered (one stream, or events between streams). */
int b200_sumsq(const float* x, int64_t n, float* out, b200_stream_t stream);
/* One pass over every parameter (trainer.py:272-279):
 *   g    = grad * clamp(max_grad_norm / (sqrt(*gradnorm_sq) + 1e-6), max=1)  (clip_grad_norm_; skipped when gradnorm_sq == NULL;
 *                                                                          a NaN norm gives a NaN coefficient, an infinite one 0)
 *   w   *= 1 - lr * weight_decay                                              (Adopt's decoupled weight decay, when > 0)
 *   first gradient of a parameter : v = g^2, m = 0, parameter untouched     (Adopt initialises its state on first sight)
 *   afterwards                    : m += (1-beta1) (g / max(sqrt(v), eps) - m);  w -= lr m;  v += (1-beta2) (g^2 - v)
 *   (1-beta1, 1-beta2: one_minus_beta1 / one_minus_beta2 when non-zero — the complements formed in double and rounded once, as
 *   torch's lerp_(x, 1. - beta) applies them; 0 keeps 1.f - beta formed in fp32 on the device, which is 16 u off for beta 0.99)
 *   ("first" is tracked per chunk in chunk_state (int32 [n_chunks], zeroed once by the caller): a parameter that received no
 *   gradient on the first steps — the text stream while the text is dropped — is initialised when its first gradient arrives)
 *   ema_mode 1: ema += ema_weight (w - ema)   (ema-pytorch lerp, ema_weight = 1 - current decay);  2: ema = w (copy phase);  0: none
 * Adopt = adam-atan2-pytorch's `Adopt` (pyproject.toml:26, call site trainer.py:183) — the package is not part of the original project;
 * restated from the ADOPT algorithm it implements (Taniguchi et al. 2024, Alg. 2 without clipping) and pinned by a PyTorch
 * restatement in oracle/optim_oracle.py. chunk.ptr = the parameter piece. */
typedef struct {
    const b200_chunk* chunks_dev; int32_t n_chunks;
    const float* grad_flat; float *m_flat, *v_flat, *ema_flat;
    const float* gradnorm_sq; float max_grad_norm;
    float lr, beta1, beta2, eps, weight_decay;
    int32_t* chunk_state;
    int32_t ema_mode; float ema_weight;
    const float* used;   /* optional fp32 [n_params]: parameters with used[pidx] == 0 keep w, m, v (only their EMA moves) */
    float one_minus_beta1, one_minus_beta2;   /* optional: fp32(1 - beta) formed in double; 0 -> 1.f - beta on the device */
} b200_adopt_args;
int b200_adopt_step(const b200_adopt_args* a, b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
