"""Element-wise float64 bounds for the attention (csrc/attn_tc.cu) and hyper-connection (csrc/hyper.cu) kernels.

Method of tests/kernel_checks.py: every output of b200_attn_maskbits / b200_attn_fwd / b200_attn_bwd (with its prep kernel) and
b200_hc_width_fwd / _bwd (unfused and fused) / b200_hc_depth_fwd / _bwd is compared element by element with a float64 restatement
computed on the host from the exact bf16 / fp32 tensors the kernel received. The C ABI is called directly with NaN-prefilled output
buffers, so an element the kernel never writes fails. Every bound is E (bit-identical), F (fp32) or B (one bf16 rounding of an F
value, check_b).

The F bounds are carried by `Rv` (tests/kernel_checks.py). Figures for functions: tanhf 2 ulp, logf 1 ulp (CUDA C++ Programming
Guide, appendix "Mathematical Functions"); sqrtf and / correctly rounded. The attention restatement, its error model and the
figures for the instructions it uses are those of tests/attn_ref.py.
The reference values come from the oracle (float64 autograd of O.hyper_width / O.hyper_depth, kernels' max(||r||, 1e-12) semantics)
and, for attention, from the float64 restatement itself, which is checked against float64 autograd of the softmax attention where
the case is small enough. Each restatement must agree with that reference to a thousandth of its own bound.
Where a case exists to reach a path behind a threshold, the test asserts which side of it the case is on, from the device's SM count
and the host rules of hyper.cu and attn_tc.cu restated below.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from attn_ref import (TQ, assert_regime, attn_bwd, attn_fwd, attn_inputs, autograd64, dropout_keep, host_maskbits,
                      restate)
from hyper_conv_ref import S, hc_common, hc_fwd, hc_inputs, hc_params
from kernel_checks import (BF16, F32, F64, U, Rv, _rnd, add, agree, check_b, check_e, check_f, chk_b, chk_f, dev, dot, dots,
                           exact, fma, gamma, h64, mono, mul, nans, neg, ones_rv, pkg, sms, stream, to_bf16)
from model_checks import whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


# ================================================================================================================ hyper-connections
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


# (name, T, D, rows_per_batch, norm mode, fused, d_beta given, zero tokens, isolation slice in batch elements)
HC_CASES = [
    ('d8-t1', 1, 8, 1, 2, False, True, (), None),
    ('d8-t7', 7, 8, 7, 1, False, True, ((3, (0,)),), None),
    ('d128-t7', 7, 128, 7, 0, False, True, (), None),
    ('d512-t7', 7, 512, 7, 2, False, True, (), None),
    ('d512-t204', 204, 512, 204, 2, False, True, (), None),
    ('d1024-t16-fused', 16, 1024, 16, 2, True, True, (), None),
    ('d128-t16-fused-m1', 16, 128, 8, 1, True, True, (), None),
    ('d264-rpb33-m0', 99, 264, 33, 0, False, True, (), None),
    ('d264-rpb33-m1', 99, 264, 33, 1, False, True, (), None),
    ('d264-rpb33-m2', 99, 264, 33, 2, False, False, (), (1, 2)),
    ('d512-rpb1-m0', 400, 512, 1, 0, True, True, (), None),
    ('d512-rpb1-m1', 400, 512, 1, 1, False, True, (), None),
    ('d512-rpb1-m2', 400, 512, 1, 2, False, True, (), (150, 250)),
    ('d256-rpb1056-m0', 2112, 256, 1056, 0, False, True, (), None),
    ('d128-rpb1056-m1', 2112, 128, 1056, 1, True, True, (), None),
    ('d1024-rpb1056x7-m2', 7392, 1024, 1056, 2, False, True, (), None),
    ('d512-zero-streams', 64, 512, 32, 2, False, True, ((3, (1,)), (10, (0, 1, 2, 3))), None),
    ('d1024-zero-streams-m1', 16, 1024, 16, 1, False, False, ((5, (2,)), (9, (0, 1, 2, 3))), None),
    ('d512-t16896-fused', 16896, 512, 1056, 2, True, True, (), (3, 5)),
    ('d1024-t16640', 16640, 1024, 2080, 2, False, True, (), (2, 4)),
]


@pytest.mark.parametrize('name,T,D,rpb,mode,fused,use_dbeta,zeros,iso', HC_CASES, ids=[c[0] for c in HC_CASES])
def test_hyper_connection_kernels(pkg, name, T, D, rpb, mode, fused, use_dbeta, zeros, iso):
    pf, vpt, fwd_warps = hc_fwd_launch(T, D)
    nbatch, slots, tpb = hc_bwd_launch(T, D, rpb)
    if name.startswith('d8'):
        assert D // 8 == 1                                   # one 16-byte chunk: only lane 0 holds data
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


def test_hyper_cases_reach_every_instantiation():
    """the width kernels are built for (VPT, prefetching, fused) = (1 | 2, yes, *) at D <= 512 and (4, no, *) above"""
    reached = {(hc_fwd_launch(1, c[2])[1], hc_fwd_launch(1, c[2])[0], c[5]) for c in HC_CASES}
    assert reached == {(v, v < 4, f) for v in (1, 2, 4) for f in (False, True)}


def test_hyper_depth_short(pkg):
    """the depth kernels alone at T = 1 and 7 (fewer tokens than a block) and D = 8 / 264 (one chunk; a partial lane pass)"""
    for T, D in ((1, 8), (7, 264), (7, 1024)):
        g = torch.Generator().manual_seed(T * D)
        res = torch.randn(T, S, D, generator=g).to(BF16).to(dev())
        y = torch.randn(T, D, generator=g).to(BF16).to(dev())
        beta = (1 + 0.3 * torch.randn(T, S, generator=g)).to(dev())
        d_out = torch.randn(T, S, D, generator=g).to(BF16).to(dev())
        assert depth_bwd_warps(T) >= T and depth_fwd_threads(T, D) >= T * D // 8
        depth_check(pkg, f'T{T} D{D}', res, y, beta, d_out)


def test_whole_model_single_short_clip(pkg):
    """E2TTS(dim=512), one clip of 100 frames: T = B (N + 32) = 132 tokens < 0.4 D, so the hyper-connection backward's parameter
    GEMM result (D * 8 floats) is larger than its coefficient rows (T * 20 floats)"""
    T, D = 1 * (100 + 32), 512
    assert T * 20 < D * 8
    whole_model(pkg, dict(dim=512, depth=2, heads=8), B=1, N=100, lens=[100], seed=70)


# ================================================================================================================ attention
# (name, B, H, N', logit regime, softclamp, dropout, per-batch masks, gate, isolation)
ATTN_CASES = [
    ('n33-b1-h1', 1, 1, 33, 'mixed', 50.0, 0.0, ('edges',), True, False),
    ('n63-b4-h3', 4, 3, 63, 'deg5', 50.0, 0.0, ('edges', 'tail', 'random', 'none'), True, False),
    ('n64-b2-h8', 2, 8, 64, 'deg9', 50.0, 0.0, ('edges', 'tail'), True, False),
    ('n65-b1-h16', 1, 16, 65, 'mixed', 50.0, 0.0, ('edges',), True, True),
    ('n127-b3-h3', 3, 3, 127, 'tanh', 50.0, 0.0, ('tail', 'edges', 'random'), True, True),
    ('n128-b4-h1-nogate', 4, 1, 128, 'deg9', 50.0, 0.0, ('edges', 'tail', 'random', 'none'), False, False),
    ('n129-b2-h8', 2, 8, 129, 'mixed', 50.0, 0.0, ('edges', 'tail'), True, True),
    ('n331-b2-h3-clamp64', 2, 3, 331, 'sat', 64.0, 0.0, ('edges', 'random'), True, False),
    ('n331-b2-h3-dropout', 2, 3, 331, 'mixed', 50.0, 0.1, ('edges', 'tail'), True, False),
    ('n65-b2-h3-dropout', 2, 3, 65, 'deg9', 50.0, 0.1, ('tail', 'edges'), True, False),
    ('n1056-b2-h8', 2, 8, 1056, 'mixed', 50.0, 0.0, ('tail', 'random'), True, False),
    ('n2080-b1-h2', 1, 2, 2080, 'deg5', 50.0, 0.0, ('tail',), True, False),
    ('n1056-b1-h3-unmasked', 1, 3, 1056, 'deg9', 50.0, 0.0, ('none',), True, False),
]


@pytest.mark.parametrize('name,B,H,Np,regime,clamp,p_drop,masks,use_gate,iso', ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def test_attention_kernels(pkg, name, B, H, Np, regime, clamp, p_drop, masks, use_gate, iso):
    seed = 1234567 + Np
    q, k, v, gate, m, mask, dog = attn_inputs(B, H, Np, regime, masks, use_gate, seed=Np * 31 + H)
    uvalid = assert_regime(regime, q, k, m, clamp)
    if Np == 33:
        assert B * H * Np < TQ                                      # the whole tensor is smaller than one 128-row TMA box
    if p_drop > 0:
        assert Np % 2 == 1                                          # odd N': the dropout row pitch is N' + 1
    fw = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, clamp, p_drop, seed, d_gate=True)
    torch.cuda.synchronize()
    mb = fw['ws'].cpu()
    assert torch.equal(mb, host_maskbits(m, Np)), f'{name}: key bitmask'
    r = restate(q, k, v, gate, m, clamp, p_drop, seed, dog, fw['o'], fw['lse'])
    if B * H * Np * Np <= 3_000_000:
        ag = autograd64(q, k, v, gate, m, clamp, p_drop, seed, dog)
        for key in ('o', 'lse', 'dq', 'dk', 'dv'):
            agree(f'{name} {key} (restatement vs float64 autograd)', r[key], ag[key])
    check_b(f'{name} o', fw['o'], r['o'].v, r['o'].e)
    check_b(f'{name} og', fw['og'], r['og'].v.permute(0, 2, 1, 3).reshape(B * Np, H * 64),
            r['og'].e.permute(0, 2, 1, 3).reshape(B * Np, H * 64))
    check_f(f'{name} lse', fw['lse'], r['lse'].v, r['lse'].e)
    dgo = r['dgate_own'].permute(0, 2, 1).reshape(B * Np, H)
    check_f(f'{name} d_gate', bw['d_gate'], dgo, r['dgate_e'].permute(0, 2, 1).reshape(B * Np, H))
    g4 = h64(gate).view(B, Np, H).permute(0, 2, 1) if gate is not None else torch.ones(B, H, Np, dtype=F64)
    check_f(f'{name} delta', bw['ws_delta'], r['dgate_own'] * g4, gamma(65) * r['dgate_e'] / gamma(64) * g4)
    check_b(f'{name} ws_dO', bw['ws_dO'], r['dO'].v, U * r['dO'].v.abs())
    check_b(f'{name} dv', bw['dv'], r['dv'].v, r['dv'].e)
    check_b(f'{name} dk', bw['dk'], r['dk'].v, r['dk'].e)
    check_f(f'{name} dq', bw['dq'], r['dq'].v, r['dq'].e)
    if iso:
        # isolation (E): each (b, h) of the launch equals a B = 1, H = 1 launch on that slice. The degree-5 / degree-9 choice is made
        # per warp over the rows the TMA boxes read, which reach into the next head; outside the degree-5 range both launches make
        # the same per-element choice, so every warp tile of these cases must lie beyond it
        assert regime != 'deg5' and bool((uvalid > 0.15 * (1 + 1e-3)).all())
        for b in range(B):
            for hh in range(H):
                sl = lambda t: t[b:b + 1, hh:hh + 1].contiguous()
                gs = gate.view(B, Np, H)[b, :, hh:hh + 1].contiguous() if gate is not None else None
                ms = mask[b:b + 1].contiguous() if mask is not None else None
                dogs = dog.view(B, Np, H, 64)[b, :, hh].contiguous()
                f1 = attn_fwd(pkg, sl(q), sl(k), sl(v), gs, ms, clamp, p_drop, seed)
                b1 = attn_bwd(pkg, sl(q), sl(k), sl(v), f1['o'], f1['lse'], gs, ms, dogs, clamp, p_drop, seed, d_gate=True)
                torch.cuda.synchronize()
                tag = f'{name} isolation b{b} h{hh}'
                check_e(f'{tag} o', f1['o'], sl(fw['o']))
                check_e(f'{tag} og', f1['og'], fw['og'].view(B, Np, H, 64)[b, :, hh])
                check_e(f'{tag} lse', f1['lse'], fw['lse'][b:b + 1, hh:hh + 1])
                check_e(f'{tag} dk', b1['dk'], sl(bw['dk']))
                check_e(f'{tag} dv', b1['dv'], sl(bw['dv']))
                check_e(f'{tag} d_gate', b1['d_gate'], bw['d_gate'].view(B, Np, H)[b, :, hh:hh + 1])
                check_f(f'{tag} dq', b1['dq'], r['dq'].v[b:b + 1, hh:hh + 1], r['dq'].e[b:b + 1, hh:hh + 1])


def test_attention_shared_bitmask_and_device_seed(pkg):
    """maskbits_ready = 1 with the bitmask of ops.attn_maskbits, and seed + *seed_dev, reproduce the per-call bitmask and the summed
    seed bit for bit (E)"""
    B, H, Np, clamp, p_drop = 3, 2, 193, 50.0, 0.1
    q, k, v, gate, m, mask, dog = attn_inputs(B, H, Np, 'mixed', ('edges', 'tail', 'random'), True, seed=99)
    base, addend = 0x0123456789ABCDEF, 0xFEDCBA9876543211
    total = (base + addend) % 2 ** 64
    ref_f = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, total)
    ref_b = attn_bwd(pkg, q, k, v, ref_f['o'], ref_f['lse'], gate, mask, dog, clamp, p_drop, total)
    shared = pkg.ops.attn_maskbits(mask, B, Np, dev())
    torch.cuda.synchronize()
    assert torch.equal(shared.cpu(), host_maskbits(m, Np))
    sd = torch.tensor([addend - 2 ** 64 if addend >= 2 ** 63 else addend], dtype=torch.int64, device=dev())
    f = attn_fwd(pkg, q, k, v, gate, None, clamp, p_drop, base, ws=shared, ready=1, seed_dev=sd)   # keymask unused when ready
    b = attn_bwd(pkg, q, k, v, f['o'], f['lse'], gate, None, dog, clamp, p_drop, base, ws=shared, ready=1, seed_dev=sd)
    torch.cuda.synchronize()
    assert torch.equal(shared.cpu(), host_maskbits(m, Np))          # a ready bitmask is only read
    for key in ('o', 'og', 'lse'):
        check_e(f'shared bitmask + device seed {key}', f[key], ref_f[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_dO', 'ws_delta'):
        check_e(f'shared bitmask + device seed {key}', b[key], ref_b[key])
    keep = dropout_keep(total, B, H, Np, p_drop)
    assert 0.05 < 1 - float(keep.double().mean()) < 0.15              # the summed seed's dropout pattern is the one applied
    r = restate(q, k, v, gate, m, clamp, p_drop, total, dog, f['o'], f['lse'])
    check_b('device seed o', f['o'], r['o'].v, r['o'].e)
    check_f('device seed dq', b['dq'], r['dq'].v, r['dq'].e)
