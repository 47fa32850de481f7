"""Hyper-connection launches, their host launch rules and float64 checks, and the depthwise-convolution float64 reference, shared by
the kernel tests of csrc/hyper.cu and csrc/small.cu (tests/test_gpu_attention_hyper_kernels.py, tests/test_gpu_conv_melspec_kernels.py,
tests/test_gpu_geometry.py) and the tests of the nodes and the plain-residual backbone built on them.

The hyper-connection references come from the oracle (float64 autograd of O.hyper_width / O.hyper_depth, the kernels'
max(||r||, 1e-12) semantics) and from `hc_restate`, the width kernels' operations in their order as Rv; the bound classes are those of
tests/kernel_checks.py."""
import math

import torch
import torch.nn.functional as F

from kernel_checks import (BF16, F32, F64, U, Rv, _rnd, add, check_e, chk_b, chk_f, dev, dot, dots, exact, fma, gamma, h64, mono, mul,
                           nans, neg, ones_rv, sig_err, sms, stream, to_bf16)
from oracle import e2tts_oracle as O

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


# host rules of hyper.cu
def hc_fwd_launch(T, D):
    pf = D <= 512
    vpt = 1 if D <= 256 else (2 if D <= 512 else 4)
    grid = min((T + 7) // 8, sms() * (2 if pf else 8))
    return pf, vpt, grid * 8                     # prefetching?, 16-byte chunks per lane, warps (one token each per pass)


def hc_bwd_launch(T, D, rpb):
    nbatch = T // rpb
    slots = sms() * (2 if D <= 256 else 1)
    per_batch = max(slots // nbatch, 1)
    tpb = -(-rpb // per_batch)
    tpb = max(-(-tpb // 8) * 8, 32)
    return nbatch, slots, tpb


def depth_fwd_threads(T, D):
    return min(-(-T * (D // 8) // 256), sms() * 16) * 256


def depth_bwd_warps(T):
    return min(-(-T // 8), sms() * 8) * 8


def hc_bwd(pkg, P, x, mode, ng, rpb, stats, d_branch, d_res, d_beta, y=None, bp=None):
    T, _, D = x.shape
    fused = y is not None
    out = dict(d_xres=nans((T, S, D), BF16), d_y=nans((T, D), BF16) if fused else None, d_bp=nans((T, S), F32) if fused else None)
    g = {k: torch.zeros_like(v) for k, v in P.items()}     # the kernel ADDS into the parameter gradients
    g_ng = torch.zeros_like(ng) if mode else None
    ws = nans((T * 20 + D * 8,), F32)                      # the workspace size of include/b200_e2tts.h
    a = pkg.lib.make_args('b200_hc_width_args', **hc_common(P, x, mode, ng, rpb, y, bp), d_branch=d_branch, d_res=d_res, d_beta=d_beta,
                          d_xres=out['d_xres'], g_norm_gamma=g['gamma'], g_dynamic_alpha_fn=g['afn'], g_dynamic_alpha_scale=g['ascale'],
                          g_static_alpha=g['salpha'], g_dynamic_beta_fn=g['bfn'], g_dynamic_beta_scale=g['bscale'], g_static_beta=g['sbeta'],
                          g_norm_gain=g_ng, ws_records=ws, stats=stats, d_y_prev=out['d_y'], d_beta_prev=out['d_bp'])
    pkg.lib.call('b200_hc_width_bwd', a, stream())
    out.update({'g_' + k: v for k, v in g.items()}, g_ng=g_ng)
    return out


def hc_oracle(P, inp, mode, rpb, use_dbeta):
    """float64 autograd of O.hyper_depth (fused) + O.hyper_width + the consumer's RMSNorm on the exact kernel inputs"""
    x, y, bp, ng = inp['x'], inp['y'], inp['bp'], inp['ng']
    T, _, D = x.shape
    sd = {'p.norm.gamma': P['gamma'], 'p.dynamic_alpha_fn': P['afn'], 'p.dynamic_alpha_scale': P['ascale'], 'p.static_alpha': P['salpha'],
          'p.dynamic_beta_fn': P['bfn'], 'p.dynamic_beta_scale': P['bscale'], 'p.static_beta': P['sbeta']}
    sd = {k: h64(v).requires_grad_() for k, v in sd.items()}
    xr = h64(x).view(1, T, S, D).requires_grad_()
    leaves = [xr]
    r = xr
    if y is not None:
        yr, bpr = h64(y).view(1, T, D).requires_grad_(), h64(bp).view(1, T, S).requires_grad_()
        leaves += [yr, bpr]
        r = O.hyper_depth(xr, bpr, yr)
    b0, rest, be = O.hyper_width(sd, 'p', r, S)
    ngr = None
    if mode:
        ngr = h64(ng).requires_grad_()
        gain = ngr.repeat_interleave(rpb, 0)[None] if mode == 2 else ngr
        b0 = F.normalize(b0, dim=-1) * D ** 0.5 * gain
    loss = (b0 * h64(inp['d_branch']).view(1, T, D)).sum() + (rest * h64(inp['d_res']).view(1, T, S, D)).sum()
    if use_dbeta:
        loss = loss + (be * h64(inp['d_beta']).view(1, T, S)).sum()
    leaves += list(sd.values()) + ([ngr] if mode else [])
    grads = torch.autograd.grad(loss, leaves, allow_unused=True)           # without d_beta the beta parameters get no gradient
    grads = [torch.zeros_like(l) if g is None else g for l, g in zip(leaves, grads)]
    names = ['d_xres'] + (['d_y', 'd_bp'] if y is not None else []) + ['g_gamma', 'g_afn', 'g_ascale', 'g_salpha', 'g_bfn', 'g_bscale',
                                                                        'g_sbeta'] + (['g_ng'] if mode else [])
    ref = dict(zip(names, grads))
    ref.update(branch=b0.detach()[0], res=rest.detach()[0], beta=be.detach()[0])
    return ref


def hc_restate(P, inp, mode, rpb, use_dbeta):
    """the width kernels' operations in their order, as Rv (forward, then backward from the forward's saved per-token results)"""
    x, y, bp, ng = inp['x'], inp['y'], inp['bp'], inp['ng']
    T, _, D = x.shape
    X = exact(x)
    R = X
    if y is not None:                                                # fused: r = fma(beta_prev, y_prev, xres) in fp32
        Y, BP = exact(y), exact(bp)
        R = fma(BP[:, :, None], Y[:, None, :], X)
    A = exact(torch.cat([P['afn'], P['bfn'][:, None]], 1))          # [D, 6]: the 5 alpha columns, then beta
    G1 = _rnd(h64(P['gamma']) + 1, 0)                                # gamma + 1
    Pk = mul(G1[:, None], A)                                         # staged (gamma + 1) A
    raw = dot('nsd,dk->nsk', R, Pk, D)
    ss = dot('nsd,nsd->ns', R, R, D)
    nrm = mono(ss, lambda t: t.clamp(min=0).sqrt().clamp(min=1e-12), gamma(2), lo=0)   # sqrtf; fmaxf against the fp32 1e-12
    inv = mono(nrm, lambda t: math.sqrt(D) / t, gamma(2))             # sqrtf(D), division
    arg = mul(raw, inv[:, :, None])
    th = mono(arg, torch.tanh, 4 * U)                                # tanhf: 2 ulp
    scale = Rv(torch.tensor([float(P['ascale'])] * 5 + [float(P['bscale'])], dtype=F64))
    stat = exact(torch.cat([P['salpha'], P['sbeta'][:, None]], 1))
    val = add(mul(th, scale), stat)                                  # th * scale + stat (fused or not: two roundings at most)
    alpha, beta = val[:, :, :5], val[:, :, 5]
    mix = dot('nsk,nsd->nkd', alpha, R, S)
    br = mix[:, 0]
    gain = None
    if mode:
        bss = dot('nd,nd->n', br, br, D)
        cn = mono(mono(bss, lambda t: t.clamp(min=0).sqrt().clamp(min=1e-12), gamma(2), lo=0), lambda t: math.sqrt(D) / t, gamma(2))
        gain = exact(ng).reshape(-1, D)
        gain = gain[torch.arange(T) // rpb] if mode == 2 else gain[torch.zeros(T, dtype=torch.long)]
        branch = mul(mul(br, cn[:, None]), gain)
    else:
        cn = Rv(torch.ones(T, dtype=F64))
        branch = br
    fw = dict(branch=branch, res=mix[:, 1:], beta=beta, raw=raw, cn=cn, ss=ss)

    # backward (hc_width_bwd_kernel), from the saved raw dots, sums of squares and branch norm factor
    dy = exact(inp['d_branch'])
    invD = Rv(torch.tensor(1.0 / D, dtype=F64), gamma(1) / D)
    bw = {}
    if mode:
        terms = mul(mul(dy, br), cn[:, None])                         # d gain += (dy * branch) * cn
        if mode == 2:
            bw['g_ng'] = dot('bnd,bn->bd', terms.reshape(T // rpb, rpb, D), ones_rv(T // rpb, rpb), rpb)
        else:
            bw['g_ng'] = dot('nd,n->d', terms, ones_rv(T), T)
        dmg = mul(gain, dy)
        dt = dot('nd,nd->n', dmg, br, D)
        nk2 = neg(mul(mul(mul(cn, cn), invD), mul(cn, dt)))         # -((cn cn invD) (cn dot))
        dm0 = fma(dmg, cn[:, None], mul(br, nk2[:, None]))
    else:
        dm0 = dy
    DR = exact(inp['d_res'])
    DM = Rv(torch.cat([dm0.v[:, None], DR.v], 1), torch.cat([dm0.e[:, None], DR.e], 1))   # d mix_t, t = 0..4
    dal = dot('nkd,nsd->nsk', DM, R, D)                               # d alpha[s][t] = <d mix_t, r_s>
    dr = dot('nsk,nkd->nsd', alpha, DM, S + 1)
    dbeta = exact(inp['d_beta']) if use_dbeta else Rv(torch.zeros(T, S, dtype=F64))
    dval = Rv(torch.cat([dal.v, dbeta.v[:, :, None]], 2), torch.cat([dal.e, dbeta.e[:, :, None]], 2))
    om = add(Rv(torch.ones((), dtype=F64)), neg(mul(th, th)))         # 1 - th th
    coef = mul(mul(dval, scale), om)
    cw = mul(coef, inv[:, :, None])
    Rs = dot('nsk,nsk->ns', coef, raw, 6)
    nk3 = neg(mul(mul(mul(inv, inv), invD), mul(inv, Rs)))          # -((inv inv invD) (inv Rs))
    # d r_s = dr + r nk3 + sum_k cw_k P_k: eight terms
    rn = Rv(R.v * nk3.v[:, :, None], R.mag() * nk3.e[:, :, None] + R.e * nk3.v.abs()[:, :, None])
    cp = Rv(torch.einsum('nsk,dk->nsd', cw.v, Pk.v),
            torch.einsum('nsk,dk->nsd', cw.mag(), Pk.e) + torch.einsum('nsk,dk->nsd', cw.e, Pk.v.abs()))
    mags = dr.mag() + R.mag() * nk3.mag()[:, :, None] + torch.einsum('nsk,dk->nsd', cw.mag(), Pk.mag())
    dxr = Rv(dr.v + rn.v + cp.v, dr.e + rn.e + cp.e + gamma(8) * mags)
    bw['d_xres'] = dxr
    C = to_bf16(cw)                                                   # the bf16 coefficient rows of the parameter GEMM
    pairs = [('nsd,nsk->dk', X, C)]
    K = T * S
    if y is not None:
        bw['d_y'] = dot('ns,nsd->nd', BP, dxr, S)
        bw['d_bp'] = dot('nsd,nd->ns', dxr, Y, D)
        Cp = to_bf16(dot('ns,nsk->nk', BP, cw, S))                    # C' rows: sum_s beta_prev[s] C[(tok, s)]
        pairs.append(('nd,nk->dk', Y, Cp))
        K += T
    Gm = dots(pairs, K)
    bw['g_afn'] = mul(G1[:, None], Gm[:, :5])
    bw['g_bfn'] = mul(G1, Gm[:, 5])
    bw['g_gamma'] = dot('dk,dk->d', A, Gm, 6)
    bw['g_salpha'] = dot('nsk,n->sk', dval[:, :, :5], ones_rv(T), T)
    bw['g_sbeta'] = dot('ns,n->s', dbeta, ones_rv(T), T)
    bw['g_ascale'] = dot('nsk,nsk->', dval[:, :, :5], th[:, :, :5], 20 * T)
    bw['g_bscale'] = dot('ns,ns->', dbeta, th[:, :, 5], 4 * T)
    return fw, bw


def depth_check(pkg, name, res, y, beta, d_out):
    """b200_hc_depth_fwd / _bwd: out = res + beta y (B), d_y = sum_s beta d_out (B), d_beta = <d_out, y> (F)"""
    T, _, D = res.shape
    out = nans((T, S, D), BF16)
    a = pkg.lib.make_args('b200_hc_depth_args', res=res, y=y, beta=beta, out=out, T=T, D=D, num_streams=S)
    pkg.lib.call('b200_hc_depth_fwd', a, stream())
    d_y, d_beta = nans((T, D), BF16), nans((T, S), F32)
    a = pkg.lib.make_args('b200_hc_depth_args', y=y, beta=beta, d_out=d_out, d_y=d_y, d_beta=d_beta, T=T, D=D, num_streams=S)
    pkg.lib.call('b200_hc_depth_bwd', a, stream())
    torch.cuda.synchronize()
    rr, yr, br = h64(res).requires_grad_(), h64(y).requires_grad_(), h64(beta).requires_grad_()
    o = O.hyper_depth(rr, br, yr)
    gy, gb = torch.autograd.grad(o, [yr, br], h64(d_out))
    Rr, Y, Bt, DO = exact(res), exact(y), exact(beta), exact(d_out)
    chk_b(f'{name} depth out', out, add(mul(Bt[:, :, None], Y[:, None, :]), Rr), o.detach())   # res + beta y: two roundings at most
    chk_b(f'{name} depth d_y', d_y, dot('ns,nsd->nd', Bt, DO, S), gy)
    chk_f(f'{name} depth d_beta', d_beta, dot('nsd,nd->ns', DO, Y, D), gb)
    return out, d_y, d_beta


def check_hc_case(pkg, name, T, D, rpb, mode, fused, use_dbeta, zeros, iso):
    """b200_hc_width_fwd / _bwd (unfused or fused) on T tokens of width D against hc_oracle and hc_restate, every output NaN-
    prefilled; from T = 64 on, the depth kernels on its outputs (depth_check); `iso` = (b0, b1): a launch on those batch elements
    reproduces the big launch's per-token results bit for bit. Asserts the sides of the launch thresholds the case name promises."""
    pf, vpt, fwd_warps = hc_fwd_launch(T, D)
    nbatch, slots, tpb = hc_bwd_launch(T, D, rpb)
    if name.startswith('d8-'):
        assert D // 8 == 1                                  # one 16-byte chunk: only lane 0 holds data
    if D == 264:
        assert D // 8 == 33 and vpt == 2                     # lane 0 owns chunks 0 and 32
    if 'rpb33' in name or 'rpb1056x7' in name:
        assert rpb % tpb != 0, (rpb, tpb)                    # the last block of each batch element is partial
    if 'rpb1-' in name:
        assert nbatch > slots                                # more batch elements than resident blocks
    if T in (1, 7):
        assert fwd_warps == 8 and tpb == 32                  # one block, fewer tokens than its 8 warps
    if T < 0.4 * D:
        assert T * 20 < D * 8                                # the parameter GEMM result is larger than the coefficient rows
    if fused:
        assert (T * S) % 64 == 0
    if T in (7, 99):
        assert (T * S) % 64 != 0 and not fused
    if T >= 16000:                                            # every grid-stride / persistent loop makes a second pass
        assert fwd_warps < T and depth_fwd_threads(T, D) < T * D // 8 and depth_bwd_warps(T) < T
    P = hc_params(D, 7 + D)
    inp = hc_inputs(T, D, rpb, mode, fused, seed=T + D + mode, zero_tokens=zeros)
    x, y, bp, ng = inp['x'], inp['y'], inp['bp'], inp['ng']
    fw = hc_fwd(pkg, P, x, mode, ng, rpb, y, bp)
    bw = hc_bwd(pkg, P, x, mode, ng, rpb, fw['stats'], inp['d_branch'], inp['d_res'], inp['d_beta'] if use_dbeta else None, y, bp)
    torch.cuda.synchronize()
    ref = hc_oracle(P, inp, mode, rpb, use_dbeta)
    rf, rb = hc_restate(P, inp, mode, rpb, use_dbeta)
    for k in ('branch', 'res', 'd_xres') + (('d_y',) if fused else ()):
        assert bool(torch.isfinite((fw if k in fw else bw)[k].float()).all()), f'{name} {k}: not finite'
    chk_b(f'{name} branch', fw['branch'], rf['branch'], ref['branch'])
    chk_b(f'{name} res_out', fw['res'], rf['res'], ref['res'])
    chk_f(f'{name} beta', fw['beta'], rf['beta'], ref['beta'])
    st = fw['stats'].cpu()
    chk_f(f'{name} stats raw alpha dots', st[:, :20].reshape(T, S, 5), rf['raw'][:, :, :5], rf['raw'].v[:, :, :5])
    chk_f(f'{name} stats raw beta dots', st[:, 20:24], rf['raw'][:, :, 5], rf['raw'].v[:, :, 5])
    chk_f(f'{name} stats branch norm factor', st[:, 24], rf['cn'], rf['cn'].v)
    check_e(f'{name} stats words 25-27', st[:, 25:28], torch.zeros(T, 3))
    chk_f(f'{name} stats sums of squares', st[:, 28:], rf['ss'], rf['ss'].v)
    chk_b(f'{name} d_xres', bw['d_xres'], rb['d_xres'], ref['d_xres'])
    if fused:
        chk_b(f'{name} d_y_prev', bw['d_y'], rb['d_y'], ref['d_y'])
        chk_f(f'{name} d_beta_prev', bw['d_bp'], rb['d_bp'], ref['d_bp'])
    for k in ('g_gamma', 'g_afn', 'g_ascale', 'g_salpha', 'g_bfn', 'g_bscale', 'g_sbeta') + (('g_ng',) if mode else ()):
        chk_f(f'{name} {k}', bw[k], rb[k], ref[k])
    if T >= 64:
        # the depth connection on this case's outputs (d_out = d_res), at the same token count: the big cases wrap its loops
        depth_check(pkg, name, fw['res'], inp['d_branch'], fw['beta'], inp['d_res'])
    if iso is not None:
        # token isolation (E): a launch on batch elements [b0, b1) reproduces the big launch's per-token results bit for bit
        b0, b1 = iso
        t0, t1 = b0 * rpb, b1 * rpb
        sl = lambda t: None if t is None else t[t0:t1].contiguous()
        ngs = ng[b0:b1].contiguous() if mode == 2 else ng
        fs = hc_fwd(pkg, P, sl(x), mode, ngs, rpb, sl(y), sl(bp))
        bs = hc_bwd(pkg, P, sl(x), mode, ngs, rpb, fs['stats'], sl(inp['d_branch']), sl(inp['d_res']),
                    sl(inp['d_beta']) if use_dbeta else None, sl(y), sl(bp))
        torch.cuda.synchronize()
        for k in ('branch', 'res', 'beta', 'stats'):
            check_e(f'{name} isolation {k}', fs[k], fw[k][t0:t1])
        for k in ('d_xres',) + (('d_y', 'd_bp') if fused else ()):
            check_e(f'{name} isolation {k}', bs[k], bw[k][t0:t1])


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
