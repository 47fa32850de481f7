"""torch.autograd.Function wrappers around the C-ABI kernels of libb200e2tts.so.

Each Function is one fused stage of the reference's multistream block (citations: /root/reference/
e2_tts_pytorch/e2_tts.py and SURVEY.md Appendix A). PyTorch only allocates the buffers, orders the launches on
the current stream and carries the autograd graph; no arithmetic on the path is done by torch ops.
Parameters stay ordinary fp32 nn.Parameters (reference-compatible state_dict); Functions receive them as
inputs (so autograd / DDP see per-parameter gradients) next to their packed bf16 copies.
"""
from __future__ import annotations

import math

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

BF16, F32 = torch.bfloat16, torch.float32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _c(t):
    return t if t is None or t.is_contiguous() else t.contiguous()


class _ZeroPool:
    """One zero-filled fp32 slab per training step for the ~300 small gradient accumulators the backward kernels add into
    (hyper-connection parameter grads, conv weight/bias grads, bias column sums, gate grads, abs-pos grads): ONE memset per step
    instead of 300 `torch.zeros` fill kernels. `begin()` is called by the
    model's forward when a backward will follow; a fresh slab is allocated every step (gradients handed to autograd alias it and
    must outlive the step), sized by the previous step's demand; anything that does not fit falls back to torch.zeros."""

    def __init__(self):
        self.buf, self.off, self.used, self.peak = None, 0, 0, 0

    def begin(self, device):
        self.peak = max(self.peak, self.used)
        self.used, self.off = 0, 0
        self.buf = torch.zeros(int(self.peak * 1.1) + 4096, device=device, dtype=F32) if self.peak else None

    def zeros(self, shape, device):
        n = 1
        for d in (shape if isinstance(shape, (tuple, list, torch.Size)) else (shape,)):
            n *= int(d)
        n_al = (n + 31) // 32 * 32      # 128-byte aligned slices
        self.used += n_al
        if self.buf is None or self.buf.device != device or self.off + n_al > self.buf.numel():
            return torch.zeros(shape, device=device, dtype=F32)
        out = self.buf[self.off:self.off + n].view(shape)
        self.off += n_al
        return out


zero_pool = _ZeroPool()


def _zeros(shape, device):
    return zero_pool.zeros(shape, device)


def gemm(A, B, M, N, K, *, lda=None, ldb=None, A2=None, lda2=0, K1=0, a_mn=False, b_mn=False, out=None, ldd=None,
         out_fp32=False, D2=None, ldd2=0, bias=None, colscale=None, rows_per_batch=0, rowmask=None, resid=None, ldr=0,
         geglu=False, dropout_p=0.0, seed=0, split_k=1, force_tile=0, seed_dev=None, glu_mult=None, act=0):
    """D[M,N] = epilogue(sum_k A[m,k] B[n,k]) on the wgmma GEMM (include/b200_e2tts.h: b200_gemm). geglu: the GLU activation code
    (GLU_GELU, GLU_SILU, GLU_RELU2; True is GELU), glu_mult: fp32 [N/2] multiplier of the hidden units. act: ACT_GELU applies the
    exact-erf GELU to (z + bias) without a GLU."""
    dev = A.device
    n_out = N // 2 if geglu else N
    if ldd is None:
        ldd = n_out if out_fp32 else (n_out + 7) // 8 * 8
    if out is None:
        out = torch.empty((M, ldd), device=dev, dtype=F32 if out_fp32 else BF16)
    args = lib.make_args_positional('b200_gemm_args', _GEMM_FIELDS, (
        A, lda if lda is not None else (M if a_mn else K), A2, lda2, K1,
        B, ldb if ldb is not None else (N if b_mn else K), M, N, K, int(a_mn), int(b_mn),
        out, ldd, int(out_fp32), D2, ldd2, bias, colscale, rows_per_batch,
        rowmask, resid, ldr, int(geglu), float(dropout_p), int(seed), int(split_k), int(force_tile), seed_dev, glu_mult, int(act)))
    lib.call('b200_gemm', args, _stream())
    return out


_GEMM_FIELDS = ('A', 'lda', 'A2', 'lda2', 'K1', 'B', 'ldb', 'M', 'N', 'K', 'a_mn_major', 'b_mn_major', 'D', 'ldd', 'd_fp32', 'D2', 'ldd2',
                'bias', 'colscale', 'rows_per_batch', 'rowmask', 'resid', 'ldr', 'geglu', 'dropout_p', 'seed', 'split_k', 'force_tile', 'seed_dev',
                'glu_mult', 'act')

# GLU activation codes of b200_gemm's GLU epilogue and b200_glu_bwd (x-transformers FeedForward: default, swish=True, relu_squared=True)
GLU_GELU, GLU_SILU, GLU_RELU2 = 1, 2, 3
ACT_GELU = 1   # b200_gemm_args.act


def grad_weight(dY, X, T, n_out, n_in, *, ldy=None, ldx=None, out=None, ldd=None):
    """dW[n_out, n_in] = dY[T, n_out]^T X[T, n_in]  — both operands MN-major, fp32 out, split-K."""
    return gemm(dY, X, n_out, n_in, T, lda=ldy if ldy is not None else n_out, ldb=ldx if ldx is not None else n_in,
                a_mn=True, b_mn=True, out=out, ldd=ldd, out_fp32=True, split_k=-1)   # -1: the library fills the SMs for the tile it picks


def colsum(X, T, ncols, ld):
    out = _zeros(ncols, X.device)
    lib.call('b200_colsum', X, T, ncols, ld, out, _stream())
    return out


def pack_weights(table_dev, n):
    lib.call('b200_pack_weights', table_dev, n, _stream())


def rotary_table(Np, device, dim_head=64):
    """cos / sin fp32 [Np, dim_head / 2] of the rotary embedding (A.3), dim_head 64 or 128"""
    cs = torch.empty((Np, dim_head // 2), device=device, dtype=F32)
    sn = torch.empty((Np, dim_head // 2), device=device, dtype=F32)
    lib.call('b200_rotary_table', cs, sn, Np, dim_head, _stream())
    return cs, sn


# ---------------------------------------------------------------------------------------------------- hyper-connections
def _hc_width_fwd(xres, y_prev, beta_prev, params, norm_gain, norm_mode, rows_per_batch, want_stats):
    gamma, afn, ascale, salpha, bfn, bscale, sbeta = params
    T, S, D = xres.shape
    branch = torch.empty((T, D), device=xres.device, dtype=BF16)
    res = torch.empty_like(xres)
    beta = torch.empty((T, S), device=xres.device, dtype=F32)
    stats = torch.empty((T, 32), device=xres.device, dtype=F32) if want_stats else None   # 128 B per token: the backward's reductions
    a = lib.make_args('b200_hc_width_args', xres=xres, norm_gamma=gamma, dynamic_alpha_fn=afn, dynamic_alpha_scale=ascale,
                      static_alpha=salpha, dynamic_beta_fn=bfn, dynamic_beta_scale=bscale, static_beta=sbeta,
                      norm_mode=norm_mode, norm_gain=norm_gain, rows_per_batch=rows_per_batch, T=T, D=D, num_streams=S,
                      branch=branch, res_out=res, beta_out=beta, y_prev=y_prev, beta_prev=beta_prev, stats_out=stats)
    lib.call('b200_hc_width_fwd', a, _stream())
    return branch, res, beta, stats


def _hc_width_bwd(xres, y_prev, beta_prev, stats, params, norm_gain, norm_mode, rpb, d_branch, d_res, d_beta):
    gamma, afn, ascale, salpha, bfn, bscale, sbeta = params
    T, S, D = xres.shape
    dev = xres.device
    d_xres = torch.empty_like(xres)
    d_y = torch.empty_like(y_prev) if y_prev is not None else None
    d_bp = torch.empty_like(beta_prev) if y_prev is not None else None
    if d_branch is None:
        d_branch = torch.zeros((T, D), device=dev, dtype=BF16)
    if d_res is None:
        d_res = torch.zeros_like(xres)
    # one zero-filled fp32 slab for all parameter-gradient accumulators
    n_gain = 0 if norm_mode == 0 else norm_gain.numel()
    sizes = [D, D * (S + 1), 1, S * (S + 1), D, 1, S, n_gain]
    slab = _zeros(sum(sizes), dev)
    parts, o = [], 0
    for n in sizes:
        parts.append(slab[o:o + n])
        o += n
    g_gamma, g_afn, g_as, g_sal, g_bfn, g_bs, g_sbe, g_gain = parts
    a = lib.make_args('b200_hc_width_args', xres=xres, norm_gamma=gamma, dynamic_alpha_fn=afn, dynamic_alpha_scale=ascale,
                      static_alpha=salpha, dynamic_beta_fn=bfn, dynamic_beta_scale=bscale, static_beta=sbeta,
                      norm_mode=norm_mode, norm_gain=norm_gain, rows_per_batch=rpb, T=T, D=D, num_streams=S,
                      d_branch=_c(d_branch), d_res=_c(d_res), d_beta=_c(d_beta), d_xres=d_xres,
                      g_norm_gamma=g_gamma, g_dynamic_alpha_fn=g_afn, g_dynamic_alpha_scale=g_as, g_static_alpha=g_sal,
                      g_dynamic_beta_fn=g_bfn, g_dynamic_beta_scale=g_bs, g_static_beta=g_sbe,
                      g_norm_gain=g_gain if norm_mode else None, ws_records=torch.empty(T * 20 + D * 8, device=dev, dtype=F32),
                      y_prev=y_prev, beta_prev=beta_prev, d_y_prev=d_y, d_beta_prev=d_bp, stats=stats)
    lib.call('b200_hc_width_bwd', a, _stream())
    pg = (g_gamma, g_afn.view(D, S + 1), g_as.view(()), g_sal.view(S, S + 1), g_bfn, g_bs.view(()), g_sbe,
          g_gain.view_as(norm_gain) if norm_mode else None)
    return d_xres, d_y, d_bp, pg


class HcWidth(Function):
    """HyperConnections width connection + consumer (Adaptive)RMSNorm (A.5, A.1; e2_tts.py:870-882, 900-939)."""

    @staticmethod
    def forward(ctx, xres, gamma, afn, ascale, salpha, bfn, bscale, sbeta, norm_gain, norm_mode, rows_per_batch):
        *out, stats = _hc_width_fwd(xres, None, None, (gamma, afn, ascale, salpha, bfn, bscale, sbeta), norm_gain, norm_mode, rows_per_batch,
                                    any(ctx.needs_input_grad))
        ctx.save_for_backward(xres, stats, gamma, afn, ascale, salpha, bfn, bscale, sbeta, norm_gain)
        ctx.meta = (norm_mode, rows_per_batch)
        return tuple(out)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_branch, d_res, d_beta):
        xres, stats, *params, norm_gain = ctx.saved_tensors
        norm_mode, rpb = ctx.meta
        d_xres, _, _, pg = _hc_width_bwd(xres, None, None, stats, params, norm_gain, norm_mode, rpb, d_branch, d_res, d_beta)
        return (d_xres, *pg, None, None)


def hc_can_fuse(T, S):
    """The fused depth -> width backward feeds the parameter GEMM with two K runs (residual' rows, then branch rows): the first run must
    end on a 64-row k-block boundary (include/b200_e2tts.h, b200_hc_width_args)."""
    return (T * S) % 64 == 0


class HcDepthWidth(Function):
    """Depth connection of sub-block k (residual' + beta * branch_out, A.5 add_residual) FUSED into the width connection of sub-block
    k+1 (e2_tts.py:870-882, 900-939 apply them back to back): the updated streams are formed in registers and never written to HBM
    (forward: one [T,S,D] write + read less per sub-block; backward: the depth gradients come out of the width backward kernel)."""

    @staticmethod
    def forward(ctx, rest_prev, y_prev, beta_prev, gamma, afn, ascale, salpha, bfn, bscale, sbeta, norm_gain, norm_mode, rows_per_batch):
        y_prev, beta_prev = _c(y_prev), _c(beta_prev)
        *out, stats = _hc_width_fwd(rest_prev, y_prev, beta_prev, (gamma, afn, ascale, salpha, bfn, bscale, sbeta), norm_gain, norm_mode,
                                    rows_per_batch, any(ctx.needs_input_grad))
        ctx.save_for_backward(rest_prev, y_prev, beta_prev, stats, gamma, afn, ascale, salpha, bfn, bscale, sbeta, norm_gain)
        ctx.meta = (norm_mode, rows_per_batch)
        return tuple(out)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_branch, d_res, d_beta):
        rest_prev, y_prev, beta_prev, stats, *params, norm_gain = ctx.saved_tensors
        norm_mode, rpb = ctx.meta
        d_rest, d_y, d_bp, pg = _hc_width_bwd(rest_prev, y_prev, beta_prev, stats, params, norm_gain, norm_mode, rpb, d_branch, d_res, d_beta)
        return (d_rest, d_y, d_bp, *pg, None, None)


class HcDepth(Function):
    """HyperConnections depth connection: residual' + beta * branch_out (A.5)."""

    @staticmethod
    def forward(ctx, res, y, beta):
        T, S, D = res.shape
        out = torch.empty_like(res)
        a = lib.make_args('b200_hc_depth_args', res=res, y=y, beta=beta, out=out, T=T, D=D, num_streams=S)
        lib.call('b200_hc_depth_fwd', a, _stream())
        ctx.save_for_backward(y, beta)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        y, beta = ctx.saved_tensors
        d_out = _c(d_out)
        T, S, D = d_out.shape
        d_y = torch.empty_like(y)
        d_beta = torch.empty_like(beta)
        a = lib.make_args('b200_hc_depth_args', y=y, beta=beta, d_out=d_out, d_y=d_y, d_beta=d_beta, T=T, D=D, num_streams=S)
        lib.call('b200_hc_depth_bwd', a, _stream())
        return d_out, d_y, d_beta


# ---------------------------------------------------------------------------------------------------- depthwise conv
class DwConv(Function):
    """DepthwiseConv (e2_tts.py:295-328): mask -> depthwise conv k -> SiLU -> mask, on bf16 [B, Np, D]. residual=True: the plain
    residual sub-block x + DepthwiseConv(x, mask) (:870-872, 900-902) in the same launch; masked rows keep x."""

    @staticmethod
    def forward(ctx, x, weight, bias, mask, B, Np, residual=False):
        D = x.shape[-1]
        w2 = weight.reshape(D, -1)
        y = torch.empty_like(x)
        pre = torch.empty_like(x) if any(ctx.needs_input_grad[:3]) else None   # bf16 pre-activation: backward does not redo the convolution
        a = lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w2, bias=bias, y=y, B=B, Np=Np, D=D, ksize=w2.shape[1], pre=pre,
                          residual=int(residual))
        lib.call('b200_dwconv_fwd', a, _stream())
        ctx.save_for_backward(x, weight, bias, mask, pre)
        ctx.meta = (B, Np)
        ctx.residual = int(residual)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight, bias, mask, pre = ctx.saved_tensors
        B, Np = ctx.meta
        residual = ctx.residual
        D = x.shape[-1]
        w2 = weight.reshape(D, -1)
        dx = torch.empty_like(x)
        dw = _zeros(w2.shape, w2.device)
        db = _zeros(bias.shape, bias.device)
        a = lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w2, bias=bias, dy=_c(dy), dx=dx, dweight=dw, dbias=db,
                          B=B, Np=Np, D=D, ksize=w2.shape[1], pre=pre, residual=residual)
        lib.call('b200_dwconv_bwd', a, _stream())
        return dx, dw.view_as(weight), db, None, None, None, None


class BranchNorm(Function):
    """Pre-norm of a plain residual sub-block (Transformer(num_residual_streams=1), e2_tts.py:874-882, 906-939) on bf16 rows x [T, D]:
    RMSNorm(g) (:875, 881 and the DurationPredictor) or, with `gains` (fp32 [B, D] = 1 + to_gamma(cond), one row per Np rows),
    AdaptiveRMSNorm (:908, 937); the branch-norm mode of b200_final_norm_*. Returns (normed branch input, x): the second output IS x,
    handed on as the sub-block's residual, so that its gradient (the residual add's dy) joins the norm's gradient inside the
    backward kernel instead of in an autograd sum."""

    @staticmethod
    def forward(ctx, x, g, gains, B, Np):
        T, D = x.shape
        y = torch.empty_like(x)
        a = lib.make_args('b200_final_norm_args', xres=x, g=None if gains is not None else g, y=y, B=B, N=Np, R=0, D=D, S=1,
                          rows_per_batch=Np, gains=gains)
        lib.call('b200_final_norm_fwd', a, _stream())
        ctx.save_for_backward(x, g if gains is None else None, gains)
        ctx.meta = (B, Np)
        ctx.set_materialize_grads(False)
        return y, x.view_as(x)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, d_res):
        x, g, gains = ctx.saved_tensors
        B, Np = ctx.meta
        T, D = x.shape
        if dy is None:
            return d_res, None, None, None, None
        dx = torch.empty_like(x)
        d_g = _zeros(g.shape, g.device) if g is not None else None
        d_gains = _zeros(gains.shape, gains.device) if gains is not None else None
        a = lib.make_args('b200_final_norm_args', xres=x, g=g, dy=_c(dy), d_xres=dx, g_g=d_g, B=B, N=Np, R=0, D=D, S=1,
                          rows_per_batch=Np, gains=gains, d_gains=d_gains, d_res=_c(d_res))
        lib.call('b200_final_norm_bwd', a, _stream())
        return dx, d_g, d_gains, None, None


# ---------------------------------------------------------------------------------------------------- attention
def _maskbits_ws(B, Np, device):
    return torch.empty(((Np + 127) // 128) * 4 * B, device=device, dtype=torch.int32)   # b200_attn_workspace_bytes(B, Np)


def _clamp_args(softclamp):
    """softclamp None: attention without the logit soft-clamp (the running-maximum kernels)"""
    return dict(softclamp=0.0, unclamped=1) if softclamp is None else dict(softclamp=softclamp, unclamped=0)


def _attn_core_fwd(q, k, v, gate, mask, dropout_p, seed, softclamp, seed_dev, maskbits=None):
    """b200_attn_fwd on q, k, v bf16 [B, H, Np, dh] (dh 64 or 128) -> og (gated, head-merged bf16 [B*Np, H*dh]), o (bf16 [B, H, Np, dh]), lse (fp32
    [B, H, Np]). `maskbits` is attn_maskbits(mask), shared by every layer of a step; without it the call builds its own. `gate` may be
    None (no head gate), `softclamp` None (no logit soft-clamp)."""
    B, H, Np, dh = q.shape
    o = torch.empty_like(q)
    og = torch.empty((B * Np, H * dh), device=q.device, dtype=BF16)
    lse = torch.empty((B, H, Np), device=q.device, dtype=F32)
    a = lib.make_args('b200_attn_fwd_args', q=q, k=k, v=v, keymask=mask, gate=gate, o=o, og=og, lse=lse, B=B, H=H, Np=Np, dim_head=dh,
                      scale=dh ** -0.5, dropout_p=dropout_p, seed=seed,
                      ws_maskbits=maskbits if maskbits is not None else _maskbits_ws(B, Np, q.device), seed_dev=seed_dev,
                      maskbits_ready=int(maskbits is not None), **_clamp_args(softclamp))
    lib.call('b200_attn_fwd', a, _stream())
    return og, o, lse


def _attn_core_bwd(d_og, q, k, v, o, lse, gate, mask, dropout_p, seed, softclamp, seed_dev, maskbits=None):
    """b200_attn_bwd -> dq (fp32: accumulated across key tiles with atomics), dk, dv (bf16 [B, H, Np, dh]), d_gate (fp32 [B*Np, H],
    None without a gate)."""
    B, H, Np, dh = q.shape
    dq = torch.empty(q.shape, device=q.device, dtype=F32)
    dk, dv, ws_dO = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    ws_delta = torch.empty_like(lse)
    d_gate = torch.empty_like(gate) if gate is not None else None
    a = lib.make_args('b200_attn_bwd_args', q=q, k=k, v=v, o=o, d_og=_c(d_og), keymask=mask, gate=gate, lse=lse, ws_dO=ws_dO,
                      ws_delta=ws_delta, d_gate=d_gate, dq=dq, dk=dk, dv=dv, B=B, H=H, Np=Np, dim_head=dh, scale=dh ** -0.5,
                      dropout_p=dropout_p, seed=seed,
                      ws_maskbits=maskbits if maskbits is not None else _maskbits_ws(B, Np, q.device), seed_dev=seed_dev,
                      maskbits_ready=int(maskbits is not None), **_clamp_args(softclamp))
    lib.call('b200_attn_bwd', a, _stream())
    return dq, dk, dv, d_gate


class AttnCore(Function):
    """Softclamped, key-masked, head-gated flash attention (A.4 steps 4-5) on given q, k, v. Returns the gated, head-merged output.
    The model runs the same kernels inside Attention; this node serves the attention-core tests and benchmarks. gate None: no head
    gate; softclamp None: no logit soft-clamp."""

    @staticmethod
    def forward(ctx, q, k, v, gate, mask, dropout_p, seed, softclamp, seed_dev):
        og, o, lse = _attn_core_fwd(q, k, v, gate, mask, dropout_p, seed, softclamp, seed_dev)
        ctx.save_for_backward(q, k, v, gate, mask, o, lse)
        ctx.meta = (dropout_p, seed, softclamp, seed_dev)
        return og

    @staticmethod
    @once_differentiable
    def backward(ctx, d_og):
        q, k, v, gate, mask, o, lse = ctx.saved_tensors
        dq, dk, dv, d_gate = _attn_core_bwd(d_og, q, k, v, o, lse, gate, mask, *ctx.meta)
        return dq, dk, dv, d_gate, None, None, None, None, None


class Attention(Function):
    """Fused attention stage: ONE GEMM for to_q/to_k/to_v (+ head-gate and value-residual-mix logits), rotary + value
    residual + gate post-processing, wgmma flash attention (softclamp, key mask, dropout, head gate). Returns the gated
    head-merged output (input of to_out) and this layer's values (the first layer's feed every later layer, e2_tts.py:878,916).
    One autograd node: q/k/v never enter the graph, and dq stays fp32 from the attention backward into the rotary inverse.
    wg, bg None: no head gate (x-transformers gate_value_heads=False; packed rows [q|k|v|mix]); softclamp None: no logit soft-clamp.
    dim_head: 64 or 128, H heads of it (I = H * dim_head); cs / sn the rotary table of that head dim."""

    @staticmethod
    def forward(ctx, xn, wq, wk, wv, wg, bg, wm, bm, v_first, wpack, cs, sn, mask, B, Np, H, dropout_p, seed, softclamp, seed_dev, maskbits=None,
                dim_head=64):
        ctx.set_materialize_grads(False)   # only the first layer's values are consumed downstream: no zero-filled d_v for the others
        T, Din = xn.shape
        I = H * dim_head
        dev = xn.device
        has_mix = wm is not None
        has_gate = wg is not None
        ncat = 3 * I + (int(has_gate) + int(has_mix)) * H
        ld = (ncat + 7) // 8 * 8
        qkvg = gemm(xn, wpack, T, ncat, Din, ldd=ld)
        q = torch.empty((B, H, Np, dim_head), device=dev, dtype=BF16)
        k, v = torch.empty_like(q), torch.empty_like(q)
        gate = torch.empty((T, H), device=dev, dtype=F32) if has_gate else None
        a = lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=bg, mix_bias=bm, rot_cos=cs, rot_sin=sn, v_first=v_first,
                          q=q, k=k, v=v, gate=gate, B=B, H=H, Np=Np, dim_head=dim_head, no_gate=int(not has_gate))
        lib.call('b200_qkv_post_fwd', a, _stream())
        og, o, lse = _attn_core_fwd(q, k, v, gate, mask, dropout_p, seed, softclamp, seed_dev, maskbits)
        ctx.maskbits = maskbits
        ctx.save_for_backward(xn, qkvg, gate, v_first, wpack, cs, sn, bg, bm, q, k, v, o, lse, mask)
        ctx.meta = (B, Np, H, ncat, ld, has_mix, dropout_p, seed, softclamp, seed_dev, has_gate)
        return og, v

    @staticmethod
    @once_differentiable
    def backward(ctx, d_og, d_v_extra):
        xn, qkvg, gate, v_first, wpack, cs, sn, bg, bm, q, k, v, o, lse, mask = ctx.saved_tensors
        B, Np, H, ncat, ld, has_mix, dropout_p, seed, softclamp, seed_dev, has_gate = ctx.meta
        dh = q.shape[-1]
        if d_og is None:   # (only the values were used: not a case the model produces, kept for completeness)
            d_og = torch.zeros((xn.shape[0], H * dh), device=xn.device, dtype=BF16)
        T, Din = xn.shape
        I = H * dh
        dev = xn.device
        dq, dk, dv, d_gate = _attn_core_bwd(d_og, q, k, v, o, lse, gate, mask, dropout_p, seed, softclamp, seed_dev, ctx.maskbits)
        d_qkvg = torch.empty((T, ld), device=dev, dtype=BF16)
        d_vfirst = torch.empty_like(v_first) if v_first is not None else None
        a = lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=bg, mix_bias=bm, rot_cos=cs, rot_sin=sn, v_first=v_first,
                          gate=gate, dq=dq, dk=dk, dv=dv, dv_extra=_c(d_v_extra), d_gate=d_gate, d_qkvg=d_qkvg, d_vfirst=d_vfirst,
                          B=B, H=H, Np=Np, dim_head=dh, dq_fp32=1, no_gate=int(not has_gate))
        lib.call('b200_qkv_post_bwd', a, _stream())
        dx = gemm(d_qkvg, wpack, T, Din, ncat, lda=ld, ldb=Din, b_mn=True)
        dW = grad_weight(d_qkvg, xn, T, ncat, Din, ldy=ld)
        # only the head-gate / value-residual-mix logits have biases (none at all: the first layer without a head gate)
        db = colsum(d_qkvg[:, 3 * I:], T, ld - 3 * I, ld) if ld > 3 * I else None
        m0 = H if has_gate else 0                           # first mix column past 3 I
        return (dx, dW[:I], dW[I:2 * I], dW[2 * I:3 * I], dW[3 * I:3 * I + H] if has_gate else None, db[:H] if has_gate else None,
                dW[3 * I + m0:3 * I + m0 + H] if has_mix else None, db[m0:m0 + H] if has_mix else None,
                d_vfirst, None, None, None, None, None, None, None, None, None, None, None, None, None)


def attn_maskbits(mask_u8, B, Np, device):
    """Key-validity bitmask shared by every attention call of one forward/backward (all layers see the same key mask)."""
    ws = _maskbits_ws(B, Np, device)
    lib.call('b200_attn_maskbits', mask_u8, ws, B, Np, _stream())
    return ws


def _rowgate_bwd(dy, y, cs, mask, B, rpb, D, want_bias=False):
    """dz = dy * mask * cs ; d_cs (fp32 [B, D]) ; optionally d_bias = colsum(dz) — backward of the fused GEMM epilogue."""
    if cs is None and mask is None:
        return (dy, None, None) if want_bias else (dy, None)
    dz = torch.empty_like(dy)
    d_cs = _zeros(cs.shape, cs.device) if cs is not None else None
    d_bias = _zeros(D, dy.device) if want_bias else None
    lib.call('b200_rowgate_bwd', dy, y, cs, mask, dz, d_cs, d_bias, B, rpb, D, _stream())
    return (dz, d_cs, d_bias) if want_bias else (dz, d_cs)


class FourierLinear(Function):
    """LinearFourierEmbed (e2_tts.py:368-386): cat(sin(f), cos(f), rest) of Linear(dim -> df + dr, no bias)(x) — the attention-input
    transform of Transformer(attn_fourier_embed_input=True) (:545-546, :639, applied at :909)."""

    @staticmethod
    def forward(ctx, x, w, wpack, df, dr):
        T, D = x.shape
        n = df + dr
        ld = (n + 7) // 8 * 8
        z = gemm(x, wpack, T, n, D, ldd=ld)
        out = torch.empty((T, 2 * df + dr), device=x.device, dtype=BF16)
        lib.call('b200_fourier_feat_fwd', z, ld, out, T, df, dr, _stream())
        ctx.save_for_backward(x, wpack, z)
        ctx.meta = (df, dr, ld)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        x, wpack, z = ctx.saved_tensors
        df, dr, ld = ctx.meta
        T, D = x.shape
        n = df + dr
        dz = torch.empty((T, ld), device=x.device, dtype=BF16)
        lib.call('b200_fourier_feat_bwd', _c(d_out), z, ld, dz, T, df, dr, _stream())
        dx = gemm(dz, wpack, T, D, n, lda=ld, b_mn=True)
        dW = grad_weight(dz, x, T, n, D, ldy=ld)
        return dx, dW, None, None, None


def _rowgate_resid_bwd(dy, y, resid, cs, mask, B, rpb, D, want_bias=False):
    """_rowgate_bwd for an epilogue that also added `resid` (the gate gradient reads the branch value as y - resid)."""
    if cs is None:
        return _rowgate_bwd(dy, y, cs, mask, B, rpb, D, want_bias)
    dz = torch.empty_like(dy)
    d_cs = _zeros(cs.shape, cs.device)
    d_bias = _zeros(D, dy.device) if want_bias else None
    lib.call('b200_rowgate_resid_bwd', dy, y, _c(resid), cs, mask, dz, d_cs, d_bias, B, rpb, D, _stream())
    return (dz, d_cs, d_bias) if want_bias else (dz, d_cs)


class OutProj(Function):
    """Attention to_out (no bias) with the fused epilogue: zero padded rows (A.4 step 6) and AdaLNZero gate (:346-351).
    resid (bf16 [T, Dout], optional): the plain residual sub-block's add, x + gated output (:878, 916), in the same epilogue; its
    gradient is dy itself."""

    @staticmethod
    def forward(ctx, og, w, wpack, colscale, mask, B, Np, resid=None):
        T, I = og.shape
        Dout = w.shape[0]
        y = gemm(og, wpack, T, Dout, I, colscale=colscale, rows_per_batch=Np, rowmask=mask, resid=resid, ldr=Dout if resid is not None else 0)
        ctx.save_for_backward(og, wpack, colscale, mask, y)
        ctx.meta = (B, Np)
        ctx.has_resid, ctx.resid = resid is not None, (resid if colscale is not None else None)   # the gated backward reads y - resid
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        og, wpack, colscale, mask, y = ctx.saved_tensors
        B, Np = ctx.meta
        has_resid, resid = ctx.has_resid, ctx.resid
        T, I = og.shape
        Dout = y.shape[1]
        dy = _c(dy)
        if resid is not None:
            dz, d_cs = _rowgate_resid_bwd(dy, y, resid, colscale, mask, B, Np, Dout)
        else:
            dz, d_cs = _rowgate_bwd(dy, y, colscale, mask, B, Np, Dout)
        d_og = gemm(dz, wpack, T, I, Dout, b_mn=True)
        dW = grad_weight(dz, og, T, Dout, I)
        return d_og, dW, None, d_cs, None, None, None, (dy if has_resid else None)


class FeedForward(Function):
    """x-transformers FeedForward(glu=True) (A.2): GLU GEMM (+dropout) -> out GEMM (+bias, AdaLNZero gate). resid (bf16 [T, Din],
    optional): the plain residual sub-block's add (:882, 939) in the out GEMM's epilogue; its gradient is dy itself.
    act: the GLU activation code (GLU_GELU, GLU_SILU, GLU_RELU2); mult (fp32 [inner], optional): GLU(mult_bias=True), h = u act(g) mult;
    b2 None: the output Linear without bias (FeedForward(no_bias=True))."""

    @staticmethod
    def forward(ctx, xn, w1, b1, w2, b2, w1pack, b1pack, w2pack, colscale, B, Np, dropout_p, seed, seed_dev, resid=None, act=GLU_GELU,
                mult=None):
        T, Din = xn.shape
        inner = w2.shape[1]
        ug = torch.empty((T, 2 * inner), device=xn.device, dtype=BF16)
        h = gemm(xn, w1pack, T, 2 * inner, Din, D2=ug, ldd2=2 * inner, bias=b1pack, geglu=act, dropout_p=dropout_p, seed=seed, seed_dev=seed_dev,
                 glu_mult=mult)
        y = gemm(h, w2pack, T, Din, inner, bias=b2, colscale=colscale, rows_per_batch=Np, resid=resid, ldr=Din if resid is not None else 0)
        ctx.save_for_backward(xn, ug, h, y, w1pack, w2pack, colscale)
        ctx.meta = (B, Np, dropout_p, seed, inner, seed_dev, act, b2 is not None)
        ctx.mult = mult
        ctx.has_resid, ctx.resid = resid is not None, (resid if colscale is not None else None)   # the gated backward reads y - resid
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        xn, ug, h, y, w1pack, w2pack, colscale = ctx.saved_tensors
        B, Np, dropout_p, seed, inner, seed_dev, act, has_b2 = ctx.meta
        has_resid, resid, mult = ctx.has_resid, ctx.resid, ctx.mult
        T, Din = xn.shape
        dy = _c(dy)
        db2 = None
        if colscale is not None and resid is not None:
            dz, d_cs, *db2 = _rowgate_resid_bwd(dy, y, resid, colscale, None, B, Np, Din, want_bias=has_b2)
        elif colscale is not None:
            # y = cs * (h W2^T + b2): recover the pre-gate value through y / cs inside the kernel
            dz, d_cs, *db2 = _rowgate_bwd(dy, y, colscale, None, B, Np, Din, want_bias=has_b2)   # bias grad rides along
        else:
            dz, d_cs = dy, None
            db2 = [colsum(dz, T, Din, Din)] if has_b2 else []
        db2 = db2[0] if db2 else None
        dh = gemm(dz, w2pack, T, inner, Din, b_mn=True)
        dW2 = grad_weight(dz, h, T, Din, inner)
        dug = torch.empty_like(ug)
        db1p = _zeros(2 * inner, xn.device)
        d_mult = None
        if act == GLU_GELU and mult is None:
            lib.call('b200_geglu_bwd', dh, ug, dug, db1p, T, inner, float(dropout_p), int(seed), seed_dev, _stream())
        else:
            d_mult = _zeros(inner, xn.device) if mult is not None and ctx.needs_input_grad[16] else None
            lib.call('b200_glu_bwd', lib.make_args('b200_glu_bwd_args', dh=dh, ug=ug, dug=dug, db_packed=db1p, mult=mult, d_mult=d_mult, T=T,
                                                   inner=inner, act=int(act), dropout_p=float(dropout_p), seed=int(seed),
                                                   seed_dev=seed_dev), _stream())
        dx = gemm(dug, w1pack, T, Din, 2 * inner, b_mn=True)
        dW1p = grad_weight(dug, xn, T, 2 * inner, Din)
        nb = inner // 64
        dW1 = dW1p.view(nb, 2, 64, Din).transpose(0, 1).reshape(2 * inner, Din)   # undo the GEGLU interleave (layout only)
        db1 = db1p.view(nb, 2, 64).transpose(0, 1).reshape(2 * inner)
        return dx, dW1, db1, dW2, db2, None, None, None, d_cs, None, None, None, None, None, (dy if has_resid else None), None, d_mult


# ---------------------------------------------------------------------------------------------------- cross-stream GEMMs
class CrossCondition(Function):
    """TextAudioCrossCondition (e2_tts.py:486-513) on all S streams, concat never materialised (two-source K)."""

    @staticmethod
    def forward(ctx, xs, ts, w_ta, w_at, wstack):
        ctx.set_materialize_grads(False)   # the text stream's last output has no consumer: its gradient stays None instead of a zero fill
        T, S, D = xs.shape
        Dt = ts.shape[-1]
        R = T * S
        x2, t2 = xs.view(R, D), ts.view(R, Dt)
        xo = gemm(x2, wstack, R, D, D + Dt, lda=D, A2=t2, lda2=Dt, K1=D, ldb=D + Dt, resid=x2, ldr=D)
        if w_at is not None:
            to = gemm(x2, wstack[D:], R, Dt, D + Dt, lda=D, A2=t2, lda2=Dt, K1=D, ldb=D + Dt, resid=t2, ldr=Dt)
        else:
            to = ts.view(R, Dt)
        ctx.save_for_backward(xs, ts, wstack)
        ctx.has_at = w_at is not None
        return xo.view(T, S, D), to.view(T, S, Dt)

    @staticmethod
    @once_differentiable
    def backward(ctx, dxo, dto):
        xs, ts, wstack = ctx.saved_tensors
        T, S, D = xs.shape
        Dt = ts.shape[-1]
        R, Kc = T * S, D + Dt
        x2, t2 = xs.view(R, D), ts.view(R, Dt)
        if dxo is None:
            dxo = torch.zeros_like(xs)
        if dto is None and ctx.has_at:
            dto = torch.zeros_like(ts)
        dxo2, dto2 = _c(dxo).view(R, D), (_c(dto).view(R, Dt) if dto is not None else None)
        dWta = torch.empty((D, Kc), device=xs.device, dtype=F32)
        grad_weight(dxo2, x2, R, D, D, out=dWta, ldd=Kc)
        grad_weight(dxo2, t2, R, D, Dt, out=dWta[:, D:], ldd=Kc)
        if ctx.has_at:
            dx = gemm(dxo2, wstack, R, D, Kc, lda=D, A2=dto2, lda2=Dt, K1=D, ldb=Kc, b_mn=True, resid=dxo2, ldr=D)
            dt = gemm(dxo2, wstack[:, D:], R, Dt, Kc, lda=D, A2=dto2, lda2=Dt, K1=D, ldb=Kc, b_mn=True, resid=dto2, ldr=Dt)
            dWat = torch.empty((Dt, Kc), device=xs.device, dtype=F32)
            grad_weight(dto2, x2, R, Dt, D, out=dWat, ldd=Kc)
            grad_weight(dto2, t2, R, Dt, Dt, out=dWat[:, D:], ldd=Kc)
        else:
            dx = gemm(dxo2, wstack, R, D, D, lda=D, ldb=Kc, b_mn=True, resid=dxo2, ldr=D)
            dt = gemm(dxo2, wstack[:, D:], R, Dt, D, lda=D, ldb=Kc, b_mn=True, resid=dto2, ldr=Dt if dto2 is not None else 0)
            dWat = None
        return dx.view(T, S, D), dt.view(T, S, Dt), dWta, dWat, None


class SkipProj(Function):
    """U-Net skip: Linear(2d -> d, no bias) on cat(x, skip) for every stream (e2_tts.py:649, 887-896)."""

    @staticmethod
    def forward(ctx, xs, skip, w, wpack):
        T, S, D = xs.shape
        R = T * S
        out = gemm(xs.view(R, D), wpack, R, D, 2 * D, lda=D, A2=skip.view(R, D), lda2=D, K1=D, ldb=2 * D)
        ctx.save_for_backward(xs, skip, wpack)
        return out.view(T, S, D)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        xs, skip, wpack = ctx.saved_tensors
        T, S, D = xs.shape
        R = T * S
        dy2 = _c(dy).view(R, D)
        dx = gemm(dy2, wpack, R, D, D, ldb=2 * D, b_mn=True)
        dskip = gemm(dy2, wpack[:, D:], R, D, D, ldb=2 * D, b_mn=True)
        dW = torch.empty((D, 2 * D), device=xs.device, dtype=F32)
        grad_weight(dy2, xs.view(R, D), R, D, D, out=dW, ldd=2 * D)
        grad_weight(dy2, skip.view(R, D), R, D, D, out=dW[:, D:], ldd=2 * D)
        return dx.view(T, S, D), dskip.view(T, S, D), dW, None


# ---------------------------------------------------------------------------------------------------- stem / head
class StemLinear(Function):
    """proj_in(x) + cond_proj_in(cond) as ONE K = 2*Cp GEMM over the packed [w | cond] operand (e2_tts.py:1267-1277);
    with w_cond=None it is the DurationPredictor's single proj_in (:1057)."""

    @staticmethod
    def forward(ctx, A, w_in, b_in, w_cond, b_cond, wpack):
        T, Kp = A.shape
        D = wpack.shape[0]
        bias = b_in + b_cond if b_cond is not None else b_in
        h = gemm(A, wpack, T, D, Kp, bias=bias)
        ctx.save_for_backward(A)
        ctx.meta = (D, w_in.shape[1], w_cond is not None)
        return h

    @staticmethod
    @once_differentiable
    def backward(ctx, d_h):
        (A,) = ctx.saved_tensors
        D, C, has_cond = ctx.meta
        T, Kp = A.shape
        d_h = _c(d_h)
        dWp = grad_weight(d_h, A, T, D, Kp)
        db = colsum(d_h, T, D, D)
        half = Kp // 2
        return None, dWp[:, :C], db, (dWp[:, half:half + C] if has_cond else None), (db if has_cond else None), None


class Assemble(Function):
    """+ abs_pos, register prepend, expand to S residual streams (e2_tts.py:760-771, 800-801, 818-821). h bf16 [B*N, D]."""

    @staticmethod
    def forward(ctx, h, abs_pos, registers, B, N, S):
        D = h.shape[1]
        R = registers.shape[0]
        out = torch.empty((B * (R + N), S, D), device=h.device, dtype=BF16)
        a = lib.make_args('b200_assemble_args', h=h, abs_pos=abs_pos, registers=registers, out=out, B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_assemble_fwd', a, _stream())
        ctx.save_for_backward(registers)
        ctx.meta = (B, N, S, D, abs_pos.shape[0] if abs_pos is not None else 0)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        (registers,) = ctx.saved_tensors
        B, N, S, D, max_len = ctx.meta
        R = registers.shape[0]
        dev = registers.device
        d_h = torch.empty((B * N, D), device=dev, dtype=BF16)
        d_abs = _zeros((max_len, D), dev) if max_len else None
        d_reg = torch.empty((R, D), device=dev, dtype=F32)
        a = lib.make_args('b200_assemble_args', h=d_h, registers=registers, d_out=_c(d_out), d_h=d_h, d_abs_pos=d_abs, d_registers=d_reg,
                          B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_assemble_bwd', a, _stream())
        return d_h, d_abs, d_reg, None, None, None


class TextStem(Function):
    """CharacterEmbed gather + text register prepend + stream expand (e2_tts.py:400-412, 800-801, 821)."""

    @staticmethod
    def forward(ctx, ids, emb, registers, B, N, S):
        D = emb.shape[1]
        R = registers.shape[0]
        out = torch.empty((B * (R + N), S, D), device=emb.device, dtype=BF16)
        a = lib.make_args('b200_assemble_args', ids=ids, emb=emb, registers=registers, out=out, B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_assemble_fwd', a, _stream())
        ctx.save_for_backward(ids, emb, registers)
        ctx.meta = (B, N, S)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        ids, emb, registers = ctx.saved_tensors
        B, N, S = ctx.meta
        V, D = emb.shape
        R = registers.shape[0]
        dev = emb.device
        d_tok = torch.empty((B * N, D), device=dev, dtype=F32)
        d_reg = torch.empty((R, D), device=dev, dtype=F32)
        a = lib.make_args('b200_assemble_args', ids=ids, emb=emb, registers=registers, d_out=_c(d_out), d_tok=d_tok, d_registers=d_reg,
                          B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_assemble_bwd', a, _stream())
        d_emb = torch.empty_like(emb)
        lib.call('b200_embed_bwd', d_tok, ids, d_emb, B * N, D, V, _stream())
        return None, d_emb, d_reg, None, None, None


class InterpText(Function):
    """InterpolatedCharacterEmbed (e2_tts.py:414-482): te = mask * (interpolate(embed(valid chars), audio_len) + abs_pos_mlp(linspace(0, Lt, La))).
    b200_interp_text_fwd stretches the embeddings and evaluates Linear(1, d) + SiLU per token; Linear(d, d) + bias + the stretched
    embeddings (residual) + the row mask are ONE wgmma GEMM with its fused epilogue, over w2p, the packed bf16 copy of w2.
    Returns bf16 [B*N, d]."""

    @staticmethod
    def forward(ctx, ids_c, text_len, audio_len, mask_u8, emb, w1, b1, w2, w2p, b2, B, N):
        V, D = emb.shape
        dev = emb.device
        nt = ids_c.shape[1]
        lerp = torch.empty((B * N, D), device=dev, dtype=BF16)
        h1 = torch.empty((B * N, D), device=dev, dtype=BF16)
        a = lib.make_args('b200_interp_text_args', ids=ids_c, text_len=text_len, audio_len=audio_len, emb=emb, w1=w1, b1=b1,
                          B=B, N=N, nt=nt, D=D, vocab=V, lerp=lerp, h1=h1)
        lib.call('b200_interp_text_fwd', a, _stream())
        te = gemm(h1, w2p, B * N, D, D, bias=b2, rowmask=mask_u8, resid=lerp, ldr=D)
        ctx.save_for_backward(ids_c, text_len, audio_len, mask_u8, emb, w1, b1, w2p, h1)
        ctx.meta = (B, N)
        return te

    @staticmethod
    @once_differentiable
    def backward(ctx, d_te):
        ids_c, text_len, audio_len, mask_u8, emb, w1, b1, w2p, h1 = ctx.saved_tensors
        B, N = ctx.meta
        V, D = emb.shape
        T = B * N
        dz, _ = _rowgate_bwd(_c(d_te), d_te, None, mask_u8, B, N, D)        # dz = d_te * mask (the epilogue's row mask)
        d_h1 = gemm(dz, w2p, T, D, D, b_mn=True)
        dW2 = grad_weight(dz, h1, T, D, D)
        db2 = colsum(dz, T, D, D)
        d_emb, dw1, db1 = _zeros((V, D), emb.device), _zeros(D, emb.device), _zeros(D, emb.device)
        a = lib.make_args('b200_interp_text_args', ids=ids_c, text_len=text_len, audio_len=audio_len, emb=emb, w1=w1, b1=b1,
                          B=B, N=N, nt=ids_c.shape[1], D=D, vocab=V, d_lerp=dz, d_h1=d_h1, d_emb=d_emb, d_w1=dw1, d_b1=db1)
        lib.call('b200_interp_text_bwd', a, _stream())
        return None, None, None, None, d_emb, dw1.view_as(w1), db1, dW2, None, db2, None, None


class FinalNorm(Function):
    """drop registers -> sum residual streams -> final RMSNorm (e2_tts.py:943-952). -> bf16 [B*N, D]"""

    @staticmethod
    def forward(ctx, xres, g, B, N, R):
        T, S, D = xres.shape
        y = torch.empty((B * N, D), device=xres.device, dtype=BF16)
        a = lib.make_args('b200_final_norm_args', xres=xres, g=g, y=y, B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_final_norm_fwd', a, _stream())
        ctx.save_for_backward(xres, g)
        ctx.meta = (B, N, R)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        xres, g = ctx.saved_tensors
        B, N, R = ctx.meta
        T, S, D = xres.shape
        d_xres = torch.empty_like(xres)
        g_g = _zeros(g.shape, g.device)
        a = lib.make_args('b200_final_norm_args', xres=xres, g=g, dy=_c(dy), d_xres=d_xres, g_g=g_g, B=B, N=N, R=R, D=D, S=S)
        lib.call('b200_final_norm_bwd', a, _stream())
        return d_xres, g_g, None, None, None


class PredHead(Function):
    """to_pred Linear(d -> C) with fp32 output (e2_tts.py:1214, 1296)."""

    @staticmethod
    def forward(ctx, y, w, b, wpack):
        T, D = y.shape
        C = w.shape[0]
        pred = gemm(y, wpack, T, C, D, bias=b, out_fp32=True, ldd=C)
        ctx.save_for_backward(y, wpack)
        ctx.C = C
        return pred

    @staticmethod
    @once_differentiable
    def backward(ctx, dpred):
        y, wpack = ctx.saved_tensors
        T, D = y.shape
        C = ctx.C
        ldp = (C + 7) // 8 * 8
        dp = torch.empty((T, ldp), device=y.device, dtype=BF16)
        lib.call('b200_cast_rows', _c(dpred), dp, T, C, ldp, _stream())
        return PredHead._bwd_from_bf16(dp, ldp, y, wpack, T, D, C)

    @staticmethod
    def _bwd_from_bf16(dp, ldp, y, wpack, T, D, C):
        dy = gemm(dp, wpack, T, D, C, lda=ldp, ldb=D, b_mn=True)
        dW = grad_weight(dp, y, T, C, D, ldy=ldp)
        db = colsum(dp, T, C, ldp)
        return dy, dW, db, None


class FlowLossHead(Function):
    """to_pred + masked-MSE flow-matching loss fused at the output stage (e2_tts.py:1296, 1535, 1580-1582, 1595), optionally with the
    velocity-consistency term against `vel_target` (:1556-1576, the EMA model's no-grad prediction at t + delta).
    Returns (loss, pred fp32 [B,N,C], pred_data = x0 + pred, parts = [flow, velocity]); only `loss` is differentiable."""

    @staticmethod
    def forward(ctx, y, w, b, wpack, x1, x0, span, vel_target, vel_weight):
        T, D = y.shape
        C = w.shape[0]
        pred = gemm(y, wpack, T, C, D, bias=b, out_fp32=True, ldd=C)
        return FlowLossHead._loss(ctx, y, wpack, pred, x1, x0, span, vel_target, vel_weight, C)

    @staticmethod
    def _loss(ctx, y, wpack, pred, x1, x0, span, vel_target, vel_weight, C):
        T = pred.shape[0]
        sums = torch.empty(4, device=y.device, dtype=F32)
        loss = torch.empty((), device=y.device, dtype=F32)
        parts = torch.empty(2, device=y.device, dtype=F32)
        pred_data = torch.empty_like(pred)
        a = lib.make_args('b200_flow_loss_args', pred=pred, x1=x1, x0=x0, span=span, sums=sums, loss=loss, pred_data=pred_data, rows=T, C=C,
                          vel_target=_c(vel_target), vel_weight=float(vel_weight), loss_parts=parts)
        lib.call('b200_flow_loss_fwd', a, _stream())
        ctx.save_for_backward(y, wpack, pred, x1, x0, span, sums, vel_target)
        ctx.C, ctx.vel_weight = C, float(vel_weight)
        ctx.mark_non_differentiable(pred, pred_data, parts)
        return loss, pred, pred_data, parts

    @staticmethod
    @once_differentiable
    def backward(ctx, dloss, _dpred, _dpd, _dparts):
        y, wpack, pred, x1, x0, span, sums, vel_target = ctx.saved_tensors
        T, D = y.shape
        C = ctx.C
        ldp = (C + 7) // 8 * 8
        dp = torch.empty((T, ldp), device=y.device, dtype=BF16)
        a = lib.make_args('b200_flow_loss_args', pred=pred, x1=x1, x0=x0, span=span, sums=sums, dloss=_c(dloss.to(F32)), dpred=dp, ldp=ldp,
                          rows=T, C=C, vel_target=_c(vel_target), vel_weight=ctx.vel_weight)
        lib.call('b200_flow_loss_bwd', a, _stream())
        dy, dW, db, _ = PredHead._bwd_from_bf16(dp, ldp, y, wpack, T, D, C)
        return dy, dW, db, None, None, None, None, None, None


# ---------------------------------------------------------------------------------------------------- conditioning path
class SmallLinear(Function):
    """fp32 small-batch linear + activation (time_cond_mlp e2_tts.py:621-625; batched to_gamma projections A.1/:346-351;
    HLGaussLayer head A.6). seg_major=True returns [N/seg, B, seg] so each seg block is a contiguous [B, seg] matrix."""

    @staticmethod
    def forward(ctx, X, W, bias, act, seg, seg_major):
        Bn, K = X.shape
        N = W.shape[0]
        shape = (N // seg, Bn, seg) if seg_major else (Bn, N)
        Z = torch.empty(shape, device=X.device, dtype=F32)
        Y = torch.empty(shape, device=X.device, dtype=F32)
        a = lib.make_args('b200_small_linear_args', X=X, W=W, bias=bias, Z=Z, Y=Y, B=Bn, N=N, K=K, act=act, seg=seg, seg_major=int(seg_major))
        lib.call('b200_small_linear_fwd', a, _stream())
        ctx.save_for_backward(X, W, Z)
        ctx.meta = (act, seg, seg_major, bias is not None)
        return Y

    @staticmethod
    @once_differentiable
    def backward(ctx, dY):
        X, W, Z = ctx.saved_tensors
        act, seg, seg_major, has_bias = ctx.meta
        Bn, K = X.shape
        N = W.shape[0]
        dZ = torch.empty_like(Z)
        dX = torch.empty_like(X)
        dW = torch.empty_like(W)
        db = torch.empty(N, device=X.device, dtype=F32)
        a = lib.make_args('b200_small_linear_args', X=X, W=W, Z=Z, dY=_c(dY), dZ=dZ, dX=dX, dW=dW, dbias=db, B=Bn, N=N, K=K, act=act, seg=seg,
                          seg_major=int(seg_major))
        lib.call('b200_small_linear_bwd', a, _stream())
        return dX, dW, db if has_bias else None, None, None, None


def fourier_embed(times, weights):
    """RandomFourierEmbed (e2_tts.py:355-364); `weights` is a buffer, times carries no gradient on the path."""
    Bn, half = times.shape[0], weights.shape[0]
    out = torch.empty((Bn, 2 * half + 1), device=times.device, dtype=F32)
    lib.call('b200_fourier_embed', times, weights, out, Bn, half, _stream())
    return out


class MaskedMean(Function):
    """maybe_masked_mean (e2_tts.py:212-224) over bf16 [B, N, D] -> fp32 [B, D]."""

    @staticmethod
    def forward(ctx, x, mask, B, N):
        D = x.shape[-1]
        out = torch.empty((B, D), device=x.device, dtype=F32)
        lib.call('b200_masked_mean_fwd', x, mask, out, B, N, D, _stream())
        ctx.save_for_backward(mask)
        ctx.meta = (B, N, D)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        (mask,) = ctx.saved_tensors
        B, N, D = ctx.meta
        dx = torch.empty((B * N, D), device=dout.device, dtype=BF16)
        lib.call('b200_masked_mean_bwd', _c(dout), mask, dx, B, N, D, _stream())
        return dx, None, None, None


def stem_prepare(B, N, C, Cp, *, x1=None, x0=None, times=None, span=None, x_in=None, cond_in=None, want_cond=False, concat=False):
    """Flow-matching input stage (e2_tts.py:1519-1543): builds the bf16 GEMM operand [w | cond] (2*Cp columns); concat=True lays it out
    as cat(cond, w) for the single proj_in of E2TTS(concat_cond=True) (:1263-1265)."""
    dev = (x1 if x1 is not None else x_in).device
    A = torch.empty((B * N, 2 * Cp), device=dev, dtype=BF16)
    cond_out = torch.empty((B, N, C), device=dev, dtype=F32) if want_cond else None
    a = lib.make_args('b200_stem_args', x1=x1, x0=x0, times=times, span=span, x_in=x_in, cond_in=cond_in, A=A, cond_out=cond_out,
                      B=B, N=N, C=C, Cp=Cp, concat_cond=int(concat))
    lib.call('b200_stem_prepare', a, _stream())
    return A, cond_out


class CondPack(Function):
    """The packed to_gamma stack as an autograd node: W_out, b_out hold every per-layer to_gamma weight (AdaptiveRMSNorm A.1,
    AdaLNZero e2_tts.py:341) as one fp32 [4L*d, d] matrix and the AdaLNZero biases in the odd d-wide segments of one [4L*d]
    vector, already written by the model's weight pack; backward hands each parameter its slice of the packed gradients."""

    @staticmethod
    def forward(ctx, W_out, b_out, d, n_w, *params):
        ctx.meta = (d, n_w, len(params) - n_w)
        return W_out, b_out

    @staticmethod
    @once_differentiable
    def backward(ctx, dW, db):
        d, n_w, n_b = ctx.meta
        gw = [dW[j * d:(j + 1) * d] if dW is not None else None for j in range(n_w)]
        gb = [db[(2 * m + 1) * d:(2 * m + 2) * d] if db is not None else None for m in range(n_b)]
        return (None, None, None, None, *gw, *gb)


class CastRows(Function):
    """fp32 [rows, cols] -> bf16 (generic Transformer.forward entry, e2_tts.py:731)."""

    @staticmethod
    def forward(ctx, x):
        rows, cols = x.shape
        ctx.dtype = x.dtype
        return cast_rows(x.to(F32), rows, cols, cols)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dtype)


def cast_rows(src_f32, rows, cols, ld):
    out = torch.empty((rows, ld), device=src_f32.device, dtype=BF16)
    lib.call('b200_cast_rows', _c(src_f32), out, rows, cols, ld, _stream())
    return out


def axpy(y, f, a):
    """y + a * f (fp32), the fixed-grid ODE update of E2TTS.sample (e2_tts.py:1421)."""
    out = torch.empty_like(y)
    lib.call('b200_axpy', _c(y), _c(f), float(a), out, y.numel(), _stream())
    return out


def cfg_combine(pred, null_pred, strength, remove_parallel, keep_frac):
    """CFG + APG projection (e2_tts.py:1323-1330)."""
    B = pred.shape[0]
    pred, null_pred = _c(pred.to(F32)), _c(null_pred.to(F32))
    ws = torch.empty(2 * B, device=pred.device, dtype=torch.float64)
    out = torch.empty_like(pred)
    lib.call('b200_cfg_combine', pred, null_pred, ws, out, B, pred.numel() // B, strength, int(remove_parallel), keep_frac, _stream())
    return out


ODE_MAX_SOURCES = 7


def _ode_sources(ks, ws, prefix):
    """k0..k{S-1} and their fp32 weights as keyword arguments of the b200_ode_* structs"""
    if not 1 <= len(ks) == len(ws) <= ODE_MAX_SOURCES:
        raise ValueError(f'{len(ks)} sources with {len(ws)} weights: want 1..{ODE_MAX_SOURCES} of each')
    kw = {f'k{j}': _c(k) for j, k in enumerate(ks)}
    kw.update({f'{prefix}{j}': float(w) for j, w in enumerate(ws)})
    return kw, len(ks)


def ode_combine(y0, ks, ws, out=None):
    """y0 + sum_j ws[j] * ks[j] (fp32): stage inputs and updates of the Runge–Kutta methods of E2TTS.sample (SURVEY A.7)."""
    out = torch.empty_like(y0) if out is None else out
    kw, S = _ode_sources(ks, ws, 'w')
    lib.call('b200_ode_combine', lib.make_args('b200_ode_combine_args', y0=_c(y0), S=S, out=out, n=y0.numel(), **kw), _stream())
    return out


def ode_step_error(y0, ks, err_w, y1, atol, rtol, ws, ratio, sol_w=None):
    """The error ratio rms((sum_j err_w[j] ks[j]) / (atol + rtol max(|y0|, |y1|))) of one adaptive step into `ratio` (fp32 [1]);
    with `sol_w`, y1 = y0 + sum_j sol_w[j] ks[j] is written first. ws: fp64 workspace of the reduction."""
    kw, S = _ode_sources(ks, err_w, 'e')
    kw.update({f's{j}': float(w) for j, w in enumerate(sol_w or ())})
    lib.call('b200_ode_step_error', lib.make_args('b200_ode_step_error_args', y0=_c(y0), S=S, y1=y1, write_y1=int(sol_w is not None),
                                                  atol=float(atol), rtol=float(rtol), ws=ws, ws_len=ws.numel(), ratio=ratio,
                                                  n=y0.numel(), **kw), _stream())
    return ratio


def ode_scaled_norms(y0, a, b, c, atol, rtol, ws, out):
    """out[0] = rms(a / scale) (a may be None), out[1] = rms((b - c) / scale) (c None: rms(b / scale)), scale = atol + |y0| rtol:
    the norms of the initial step size. ws: fp64 workspace of 2 * ws_len doubles, out: fp32 [2]."""
    lib.call('b200_ode_scaled_norms', lib.make_args('b200_ode_norms_args', y0=_c(y0), a=_c(a), b=_c(b), c=_c(c), atol=float(atol),
                                                    rtol=float(rtol), ws=ws, ws_len=ws.numel() // 2, out=out, n=y0.numel()), _stream())
    return out


def ode_dense_output(y0, y1, ks, mid_w, dt, x, out=None):
    """The quartic dense output of an accepted step at x = (t - t0) / (t1 - t0), with y_mid = y0 + sum_j mid_w[j] ks[j]."""
    out = torch.empty_like(y0) if out is None else out
    kw, S = _ode_sources(ks, mid_w, 'm')
    lib.call('b200_ode_dense_output', lib.make_args('b200_ode_dense_args', y0=_c(y0), y1=_c(y1), S=S, dt=float(dt), x=float(x), out=out,
                                                    n=y0.numel(), **kw), _stream())
    return out


def melspec_frames(nw, n_fft, hop, center=True):
    """frames of a wave of nw samples: reflect-padded by n_fft // 2 on both sides (center) or valid frames only (torch.stft)"""
    pad = n_fft // 2 if center else 0
    return 1 + (nw + 2 * pad - n_fft) // hop


def melspec(wave, window, fb, n_fft, hop, wave_lens=None, out_bnd=False, center=True, power=1.0, norm_scale=1.0):
    """MelSpec front-end (e2_tts.py:248-290): fp32 [B, nw] -> [B, n_mels, frames] (or [B, frames, n_mels] with out_bnd); wave_lens
    (int32 [B]) makes it the on-device collate of a zero-padded ragged batch (trainer.py:61-82). window: the unpadded window of
    win_length <= n_fft taps; center, power and norm_scale as b200_melspec_ex documents them."""
    B, nw = wave.shape
    n_mels = fb.shape[1]
    frames = melspec_frames(nw, n_fft, hop, center)
    out = torch.empty((B, frames, n_mels) if out_bnd else (B, n_mels, frames), device=wave.device, dtype=F32)
    bands = torch.empty(2 * n_mels, device=wave.device, dtype=torch.int32)
    a = lib.make_args('b200_melspec_args', wave=wave, window=_c(window), fb=_c(fb), out=out, B=B, nw=nw, n_fft=n_fft, hop=hop,
                      n_mels=n_mels, ws_bands=bands, wave_lens=wave_lens, out_bnd=int(out_bnd), win_length=window.shape[0],
                      center=int(center), power=float(power), norm_scale=float(norm_scale))
    lib.call('b200_melspec_ex', a, _stream())
    return out


# ------------------------------------------------------------------------------------------------ resampling (trainer.py:116-118)
# torchaudio.transforms.Resample(orig, new) with the defaults the reference's HFDataset uses: sinc_interp_hann, lowpass_filter_width 6,
# rolloff 0.99, taps built in float64 and cached as float32.
RESAMPLE_LOWPASS_WIDTH, RESAMPLE_ROLLOFF = 6, 0.99


def resample_pair(orig, new):
    """(orig', new'): the rates reduced by their gcd, as torchaudio reduces them"""
    g = math.gcd(orig, new)
    return orig // g, new // g


def resample_length(n, orig, new):
    """torchaudio's output length for n samples: ceil(torch.as_tensor(new' n / orig')), a float32 ceil (one short of the exact
    ceiling at some lengths), never more than the new' (n // orig' + 1) samples its strided convolution produces"""
    o, w = resample_pair(orig, new)
    return min(int(torch.ceil(torch.as_tensor(w * n / o))), w * (n // o + 1))


def resample_taps(orig, new):
    """The banded form of torchaudio's fp32 tap table for orig -> new: (orig', new', width, first int32 [new'], count int32 [new'],
    taps fp32 [sum count]). Phase k of the full table [new', 2 width + orig'] is zero outside columns first[k] .. first[k] + count[k]
    - 1. The values are torchaudio's construction (_get_sinc_resample_kernel with dtype=None: the phase offsets -k / new' divided in
    float32, everything else in float64, rounded once to float32), evaluated only on the columns around each phase's centre: every
    other column has its time clamped to +-lowpass_filter_width, where the tap is 0 in fp32, and that is checked here."""
    o, n = resample_pair(orig, new)
    lw, base = RESAMPLE_LOWPASS_WIDTH, min(o, n) * RESAMPLE_ROLLOFF
    width = math.ceil(lw * o / base)
    cols_total = 2 * width + o
    span = math.ceil(lw * o / base) + 2
    centre = torch.arange(n, dtype=torch.float64) * o / n + width        # column where phase k's time is 0
    m = (centre - span).floor().long().clamp(min=0)[:, None] + torch.arange(2 * span + 2)
    inside = m < cols_total
    t = torch.arange(0, -n, -1)[:, None] / n + (m - width).to(torch.float64) / o
    t *= base
    t = t.clamp_(-lw, lw)
    window = torch.cos(t * math.pi / lw / 2) ** 2
    t *= math.pi
    taps = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    taps *= window * (base / o)
    taps = torch.where(inside, taps.to(torch.float32), 0.0)
    nz = taps != 0
    if bool((nz[:, 0] & (m[:, 0] > 0)).any() or (nz[:, -1] & (m[:, -1] < cols_total - 1)).any()):
        raise RuntimeError(f'resample_taps({orig}, {new}): a non-zero tap at the edge of the evaluated columns')
    col = torch.arange(m.shape[1])
    lo = torch.where(nz, col, m.shape[1]).min(1).values
    hi = torch.where(nz, col, -1).max(1).values
    first = m.gather(1, lo[:, None])[:, 0]
    count = hi - lo + 1
    keep = (col >= lo[:, None]) & (col <= hi[:, None])
    return o, n, width, first.to(torch.int32), count.to(torch.int32), taps[keep].contiguous()


RESAMPLE_PAIR_WORDS = 6    # per rate pair: orig', new', width, phase offset, tap offset, taps; per phase: first tap, count, tap offset


class ResampleTable:
    """The rate pairs of one b200_resample launch packed into one int32 tensor (taps as their fp32 bits): [pairs | phases | taps],
    in the layout include/b200_e2tts.h documents. `index[(orig, new)]` is the pair's slot (the b200_resample pair_idx value)."""

    def __init__(self, pairs, device=None):
        self.index, words, phases, taps = {}, [], [], []
        n_phases = n_taps = 0
        self.max_pair_words = 0
        for p in pairs:
            o, n, width, first, count, t = resample_taps(*p)
            self.index[p] = len(words)
            words.append([o, n, width, n_phases, n_taps, t.numel()])
            off = torch.cumsum(count, 0, dtype=torch.int32) - count
            phases.append(torch.stack([first, count, off], 1).flatten())
            taps.append(t.view(torch.int32))
            self.max_pair_words = max(self.max_pair_words, 3 * n + t.numel())
            n_phases += n
            n_taps += t.numel()
        self.n_pairs, self.n_phases, self.n_taps = len(words), n_phases, n_taps
        head = torch.tensor(words, dtype=torch.int32).flatten()
        self.data = torch.cat([head, *phases, *taps]).to(device)

    def pointers(self):
        base = self.data.data_ptr()
        return base, base + 4 * RESAMPLE_PAIR_WORDS * self.n_pairs, base + 4 * (RESAMPLE_PAIR_WORDS * self.n_pairs + 3 * self.n_phases)


def resample(wave, wave_lens, pair_idx, table, nr):
    """b200_resample (trainer.py:116-118, torchaudio.transforms.Resample per item): fp32 [B, nw] with wave_lens int32 [B] -> (fp32
    [B, nr], out_lens int32 [B]). pair_idx int32 [B]: the item's slot in `table` (a ResampleTable on the wave's device), or -1 to
    pass the item through. Samples at or past wave_lens[b] count as zero and are never read; out[b, j] = +0 for j >= out_lens[b]."""
    B, nw = wave.shape
    out = torch.empty((B, nr), device=wave.device, dtype=F32)
    out_lens = torch.empty(B, device=wave.device, dtype=torch.int32)
    pairs, phases, taps = table.pointers()
    a = lib.make_args('b200_resample_args', wave=_c(wave), wave_lens=wave_lens, pair_idx=pair_idx, pairs=pairs, phases=phases, taps=taps,
                      out=out, out_lens=out_lens, B=B, nw=nw, nr=nr, n_pairs=table.n_pairs, max_pair_words=table.max_pair_words)
    lib.call('b200_resample', a, _stream())
    return out, out_lens


# ---------------------------------------------------------------------------------------------------------- Vocos decoder (inference)


def vocos_im2col(mel, lens, lda, db_to_amp=False):
    """mel fp32 [B, T, C], lens int32 [B] -> bf16 [B * T, lda]: the k-7 embed Conv1d's operand (b200_vocos_im2col)."""
    B, T, C = mel.shape
    out = torch.empty((B * T, lda), device=mel.device, dtype=BF16)
    lib.call('b200_vocos_im2col', _c(mel), lens, out, B, T, C, lda, int(bool(db_to_amp)), _stream())
    return out


def vocos_ln(x, lens, weight, bias, eps, B, T, D, conv_w=None, conv_b=None):
    """LayerNorm of bf16 rows [B * T, D] (b200_vocos_ln), after the masked depthwise k-7 conv when conv_w is given
    (b200_vocos_dwconv_ln); rows past an item's length are zeros."""
    y = torch.empty((B * T, D), device=x.device, dtype=BF16)
    a = lib.make_args('b200_vocos_ln_args', x=x, lens=lens, conv_w=conv_w, conv_b=conv_b, ln_w=weight, ln_b=bias, y=y, B=B, T=T, D=D,
                      eps=float(eps))
    lib.call('b200_vocos_dwconv_ln' if conv_w is not None else 'b200_vocos_ln', a, _stream())
    return y


def vocos_istft(spec, window, lens, B, T, n_fft, hop):
    """ISTFTHead('same') after its Linear: spec fp32 [B * T, n_fft + 2] -> audio fp32 [B, T * hop] (b200_vocos_istft)."""
    frames = torch.empty((B * T, n_fft), device=spec.device, dtype=F32)
    audio = torch.empty((B, T * hop), device=spec.device, dtype=F32)
    a = lib.make_args('b200_vocos_istft_args', spec=spec, window=window, lens=lens, frames=frames, audio=audio, B=B, T=T, n_fft=n_fft,
                      hop=hop)
    lib.call('b200_vocos_istft', a, _stream())
    return audio
