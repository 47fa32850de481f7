"""Hyper-connection launches and the depthwise-convolution float64 reference, shared by the kernel tests of csrc/hyper.cu and
csrc/small.cu (tests/test_gpu_attention_hyper_kernels.py, tests/test_gpu_conv_melspec_kernels.py) and the tests of the nodes and the
plain-residual backbone built on them."""
import torch
import torch.nn.functional as F

from kernel_checks import BF16, F32, F64, U, Rv, add, dev, gamma, mul, nans, neg, sig_err, stream

S = 4                         # residual streams (the only count the library builds)


# ================================================================================================================ hyper-connections
def hc_params(D, seed):
    g = torch.Generator().manual_seed(seed)
    P = dict(gamma=torch.randn(D, generator=g) * 0.1, afn=torch.randn(D, S + 1, generator=g) * 0.05, ascale=torch.tensor(0.5),
             salpha=torch.randn(S, S + 1, generator=g) * 0.5 + 0.3, bfn=torch.randn(D, generator=g) * 0.05, bscale=torch.tensor(0.7),
             sbeta=torch.randn(S, generator=g) * 0.3 + 1)
    return {k: v.to(dev()) for k, v in P.items()}


def hc_inputs(T, D, rpb, mode, fused, seed, zero_tokens=()):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(T, S, D, generator=g) * 1.5).to(BF16)
    y = torch.randn(T, D, generator=g).to(BF16) if fused else None
    bp = (1 + 0.3 * torch.randn(T, S, generator=g)) if fused else None
    for tok, streams in zero_tokens:
        x[tok, list(streams)] = 0
    ng = None
    if mode == 2:
        ng = 1 + 0.2 * torch.randn(T // rpb, D, generator=g)
    elif mode == 1:
        ng = 1 + 0.2 * torch.randn(D, generator=g)
    d_branch = torch.randn(T, D, generator=g).to(BF16)
    d_res = torch.randn(T, S, D, generator=g).to(BF16)
    d_beta = torch.randn(T, S, generator=g)
    to = lambda t: None if t is None else t.to(dev()).contiguous()
    return dict(x=to(x), y=to(y), bp=to(bp), ng=to(ng), d_branch=to(d_branch), d_res=to(d_res), d_beta=to(d_beta))


def hc_common(P, x, mode, ng, rpb, y, bp):
    T, _, D = x.shape
    return dict(xres=x, norm_gamma=P['gamma'], dynamic_alpha_fn=P['afn'], dynamic_alpha_scale=P['ascale'], static_alpha=P['salpha'],
                dynamic_beta_fn=P['bfn'], dynamic_beta_scale=P['bscale'], static_beta=P['sbeta'], norm_mode=mode, norm_gain=ng,
                rows_per_batch=rpb, T=T, D=D, num_streams=S, y_prev=y, beta_prev=bp)


def hc_fwd(pkg, P, x, mode, ng, rpb, y=None, bp=None):
    T, _, D = x.shape
    out = dict(branch=nans((T, D), BF16), res=nans((T, S, D), BF16), beta=nans((T, S), F32), stats=nans((T, 32), F32))
    a = pkg.lib.make_args('b200_hc_width_args', **hc_common(P, x, mode, ng, rpb, y, bp), branch=out['branch'], res_out=out['res'],
                          beta_out=out['beta'], stats_out=out['stats'])
    pkg.lib.call('b200_hc_width_fwd', a, stream())
    return out


# ======================================================================================================== depthwise conv
CV_TN = 64                    # token tile of b200_dwconv_fwd / _bwd
FDIV = 4 * U                  # __fdividef: 2 ulp, i.e. at most 4u relative


def cdiv(a, b):
    return -(-a // b)


def corr(t, w):
    """out[b, n, c] = sum_k w[c, k] t[b, n + k - ks/2, c] (zero outside the sequence): F.conv1d's depthwise cross-correlation
    with padding ks/2, on [B, Np, D]"""
    ks, Np = w.shape[1], t.shape[1]
    tp = F.pad(t, (0, 0, ks // 2, ks // 2))
    return sum(w[:, k] * tp[:, k:k + Np] for k in range(ks))


def tap_sums(d, t, ks):
    """out[c, k] = sum_{b, n} d[b, n, c] t[b, n + k - ks/2, c]: the weight gradient of corr"""
    Np = t.shape[1]
    tp = F.pad(t, (0, 0, ks // 2, ks // 2))
    return torch.stack([(d * tp[:, k:k + Np]).sum((0, 1)) for k in range(ks)], 1)


def dw_mask(Np, spec, g):
    """one batch row's validity: 'all', 'none', an int L (tokens n < L valid: a suffix mask, or with L >= 32 the model's register
    prefix followed by a ragged audio suffix) or 'holes' (random interior holes, a single valid token between two masked ones and
    masked tokens on both sides of a tile edge)"""
    if spec == 'all':
        return torch.ones(Np, dtype=torch.bool)
    if spec == 'none':
        return torch.zeros(Np, dtype=torch.bool)
    if isinstance(spec, int):
        return torch.arange(Np) < spec
    m = torch.rand(Np, generator=g) > 0.25
    if Np >= 3:
        c = Np // 2
        m[c - 1], m[c], m[c + 1] = False, True, False
    if Np > 66:
        m[63], m[64] = False, False
    return m


def model_mask(B, Np, g, R=32):
    """the model's layer mask: R register tokens, then each clip's audio length (ragged, the longest fills the row)"""
    lens = torch.randint(Np // 3, Np - R + 1, (B,), generator=g)
    lens[0] = Np - R
    return [R + int(n) for n in lens]


def dw_ref(x, m, w, b, dy, pre):
    """float64 restatement on the host, [B, Np, D] (a channel subset is exact: the convolution is per channel).
    x, dy, pre: the bf16 values the kernel read; m: bool [B, Np]; w [D, k], b [D]: the fp32 parameters.

    pre = conv(m x) + b: the kernel's fp32 value is bias + k FMAs (the zero-padded taps of the 31-wide window add exact zeros),
        within gamma(k + 1) (|b| + sum|w||m x|) = e_pre; then one bf16 rounding (check_b).
    y = m silu(pre): the kernel evaluates __fdividef(p, 1 + __expf(-p)) at its fp32 p. |silu'| <= 1.1 carries e_pre; at |p| <= P =
        |pre| + e_pre the evaluation errs by <= P (sig_err(P) + 4u) (sig_err: the __expf and 1 + e rounding and a rounded
        quotient; __fdividef's 2 ulp add 4u). This absolute bound also covers p < -87.3, where 1 + e exceeds 2^126 and __fdividef
        returns 0 for a true value below 1e-36. Masked rows are exactly +0.
    d_pre = dy silu'(pre_bf16), from the saved bf16 pre the kernel reads, so the designed rounding of pre is not an error of the
        backward: s = __fdividef(1, 1 + __expf(-p)) within sig_err(|p|) + 4u, then the fp32 evaluation of s (1 + p (1 - s)) and the
        product with dy, one rounding per operation (Rv). Masked rows and rows outside the sequence: exactly 0.
    dx = flipped conv of d_pre: k FMAs from 0, gamma(k) sum|w||d_pre| plus sum|w| e_dpre carried, then bf16; masked rows +0.
    dW[c, k] = sum d_pre x[n + k - k/2], dbias = sum d_pre over B Np tokens (register sums, shared atomics, global atomics into
        the initial value: any order) within gamma(B Np64 + 1) sum|terms| (Np64: Np rounded up to whole tiles; the initial value is
        one term) plus the carried sum e_dpre |x|."""
    ks = w.shape[1]
    mx = torch.where(m[..., None], x, torch.zeros((), dtype=F64))
    aw = w.abs()
    conv = corr(mx, w) + b
    e_pre = gamma(ks + 1) * (b.abs() + corr(mx.abs(), aw))
    P = conv.abs() + e_pre
    y = torch.where(m[..., None], F.silu(conv), torch.zeros((), dtype=F64))
    e_y = 1.1 * e_pre + P * (sig_err(P) + FDIV)
    p = torch.where(m[..., None], pre, torch.zeros((), dtype=F64))
    s = torch.sigmoid(p)
    one = Rv(torch.ones_like(p))
    t = mul(Rv(s, sig_err(p) + FDIV), add(one, mul(Rv(p), add(one, neg(Rv(s, sig_err(p) + FDIV))))))
    dp = mul(Rv(torch.where(m[..., None], dy, torch.zeros((), dtype=F64))), t)
    dpv = torch.where(m[..., None], dp.v, torch.zeros((), dtype=F64))
    edp = torch.where(m[..., None], dp.e, torch.zeros((), dtype=F64))
    wf = w.flip(1)
    dx = corr(dpv, wf)
    e_dx = gamma(ks) * corr(dpv.abs() + edp, wf.abs()) + corr(edp, wf.abs())
    return dict(conv=conv, e_pre=e_pre, y=y, e_y=e_y, dpre=dpv, e_dpre=edp, dx=dx, e_dx=e_dx,
                dW=tap_sums(dpv, mx, ks), dWabs=tap_sums(dpv.abs() + edp, mx.abs(), ks), dWcar=tap_sums(edp, mx.abs(), ks),
                db=dpv.sum((0, 1)), dbabs=(dpv.abs() + edp).sum((0, 1)), dbcar=edp.sum((0, 1)))
