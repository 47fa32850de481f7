"""GPU: attention without the logit soft-clamp (the running-maximum instantiations of csrc/attn_tc.cu) and without the head gate (the
[q|k|v|mix] layout of b200_qkv_post), from the kernels up to the whole model.

Kernels: element-wise float64 bounds in the method of tests/test_gpu_attention_hyper_kernels.py (its Rv helpers, imported). The
forward's online softmax is bounded per score term: its exponent 2^((s - m) scale log2 e) is evaluated from fp32 s with fp32 roundings
of scale log2 e, m scale log2 e and the fma, and is rescaled by one factor 2^((m_old - m_new) scale log2 e) per key tile, each an
ex2.approx (2 ulp) of a rounded argument of magnitude <= 2 max|s| scale log2 e. The kernel's final row maximum differs from the exact
one by at most the score error; that common factor cancels in o and lse. Exact properties are held bit for bit."""
import math

import pytest
import torch

from attn_variants import variant_oracle
from oracle import e2tts_oracle as O
from test_gpu_attention_hyper_kernels import (EX2_REL, F64, FTZ, SCALE, BF16, F32, LOG2E, Rv, U, _rnd, agree, attn_bwd, attn_fwd, dev,
                                              dot, exact, ex2_rv, h64, host_maskbits, mono, mul, nans, ones_rv, stream, to_bf16)
from test_gpu_leaf_kernels import check_b, check_e, check_f, gamma
from conftest import rel_l2
from test_gpu_parity_full import _dropout_keep, _whole_model

pytestmark = pytest.mark.gpu

SL2 = SCALE * LOG2E


@pytest.fixture(scope='module')
def pkg():
    import e2_tts_pytorch_b200 as pkg
    assert torch.cuda.is_available()
    pkg.lib.load()
    return pkg


def ufwd(pkg, q, k, v, gate, mask, p_drop, seed, **kw):
    a = dict(q=q, k=k, v=v, gate=gate, mask=mask, clamp=0.0, p_drop=p_drop, seed=seed)
    return _with_unclamped(pkg, lambda: attn_fwd(pkg, **a, **kw))


def ubwd(pkg, q, k, v, o, lse, gate, mask, dog, p_drop, seed, **kw):
    a = dict(q=q, k=k, v=v, o=o, lse=lse, gate=gate, mask=mask, dog=dog, clamp=0.0, p_drop=p_drop, seed=seed)
    return _with_unclamped(pkg, lambda: attn_bwd(pkg, **a, **kw))


def _with_unclamped(pkg, fn):
    """the launch helpers of the clamped tests, with unclamped = 1 added to the argument struct they build"""
    make = pkg.lib.make_args

    def patched(name, **fields):
        if name in ('b200_attn_fwd_args', 'b200_attn_bwd_args'):
            fields['unclamped'] = 1
        return make(name, **fields)
    pkg.lib.make_args = patched
    try:
        return fn()
    finally:
        pkg.lib.make_args = make


# ------------------------------------------------------------------------------------------------------------------ inputs
def inputs(B, H, Np, kind, seed, gate=True):
    """kind: 'big' (|scale s| > 90 somewhere), 'grow' (the row maximum grows from key tile to key tile), 'first_tile' (keys 0..63 of
    every batch element masked), 'all_masked' (batch element 1 has no valid key), 'random'"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    q, k = rn(B, H, Np, 64), rn(B, H, Np, 64)
    m = torch.rand(B, Np, generator=g) > 0.25
    if kind == 'big':
        q, k = q * 6.0, k * 6.0                                       # |s| up to ~ 36 * 64 ^ 0.5 * 4: scale s beyond 90
    elif kind == 'grow':
        d = torch.where(rn(1, H, 1, 64) > 0, 1.0, -1.0)
        q = d * 2.0 + 0.1 * q
        k = d * (torch.arange(Np, dtype=torch.float32) / 16.0)[None, None, :, None] + 0.1 * k   # s grows with the key index
        m[:, -1] = True                                             # (the last key tile holds a valid key)
    elif kind == 'first_tile':
        m[:, :64] = False
        m[:, 64] = True
    elif kind == 'all_masked':
        m[1] = False
    v = rn(B, H, Np, 64)
    gt = torch.rand(B * Np, H, generator=g) if gate else None
    dog = rn(B * Np, H * 64)
    to = lambda t: None if t is None else t.to(dev()).contiguous()
    return to(q.to(BF16)), to(k.to(BF16)), to(v.to(BF16)), to(gt), m, to(m.to(torch.uint8)), to(dog.to(BF16))


# ------------------------------------------------------------------------------------------------------------------ restatement
def restate(q, k, v, gate, m, p_drop, seed, dog, o_k, lse_k):
    """forward and backward of the unclamped instantiations as Rv on [B, H, Np(query), Np(key)]; rows without a valid key are left to
    the caller (their exact outputs are 0 / -inf)"""
    B, H, Np, _ = q.shape
    nkv = -(-Np // 64)
    Q, K, V = exact(q), exact(k), exact(v)
    thr = int(p_drop * 65536)
    ks = 65536 / (65536 - thr)
    ksR = Rv(torch.tensor(ks, dtype=F64), U * ks if p_drop > 0 else 0.0)
    valid = m[:, None, None, :].expand(B, H, Np, Np)
    row_ok = valid.any(-1, keepdim=True)
    keep = _dropout_keep(seed, B, H, Np, p_drop).to(F64) if p_drop > 0 else torch.ones(B, H, Np, Np, dtype=F64)
    s = dot('bhid,bhjd->bhij', Q, K, 64)
    neg = torch.full_like(s.v, -math.inf)
    M = torch.where(valid, s.v, neg).amax(-1, keepdim=True)
    M = torch.where(row_ok, M, torch.zeros_like(M))
    Mabs = torch.where(valid, s.v.abs() + s.e, torch.zeros_like(s.v)).amax(-1, keepdim=True)
    # exponent error of one term in log2 units: its own score error, the fp32 roundings of scale log2 e, -m scale log2 e and the fma,
    # and the arguments of the rescale factors it goes through (one rounding of m_old - m_new, one of the product, per tile)
    A = SL2 * (s.e + 4 * U * (s.v.abs() + Mabs)) + nkv * SL2 * 3 * U * 2 * Mabs
    r = torch.exp2(A) * (1 + EX2_REL) ** (nkv + 1) - 1
    pv = torch.where(valid, torch.exp2(SL2 * (s.v - M)), torch.zeros_like(s.v))
    p = Rv(pv, torch.where(valid, pv * r + FTZ, torch.zeros_like(pv)))
    l = dot('bhij,j->bhi', p, ones_rv(Np), Np + 2 * nkv)                 # + the rescaling multiplies, one per tile
    l1 = Rv(torch.where(row_ok[..., 0], l.v, torch.ones_like(l.v)), l.e)
    lnl = mono(l1, torch.log, 2 * U)
    lse = Rv(M[..., 0] * SCALE + lnl.v, lnl.e + U * (M[..., 0].abs() * SCALE + lnl.v.abs()) * 2)
    pk = to_bf16(Rv(p.v * keep, p.e * keep))
    oacc = dot('bhij,bhjd->bhid', pk, V, Np + 2 * nkv)
    inv = mono(l1, lambda t: ks / t, gamma(2))
    o = mul(oacc, inv[..., None])
    G = Rv(h64(gate).view(B, Np, H).permute(0, 2, 1)[..., None]) if gate is not None else Rv(torch.ones(B, H, Np, 1, dtype=F64))
    og = mul(to_bf16(o), G)
    # backward: P from the kernel's lse
    DOG = Rv(h64(dog).view(B, Np, H, 64).permute(0, 2, 1, 3))
    dO = to_bf16(mul(DOG, G))
    ok64 = h64(o_k)
    delta = Rv((dO.v * o.v).sum(-1),
               G.v[..., 0].abs() * ((DOG.v.abs() * (ok64 - o.v).abs()).sum(-1) + gamma(65) * (DOG.v.abs() * ok64.abs()).sum(-1)))
    dP = dot('bhid,bhjd->bhij', dO, V, 64)
    lk = torch.where(row_ok[..., 0], h64(lse_k), torch.zeros_like(lse.v))
    dlse = (lk - torch.where(row_ok[..., 0], lse.v, torch.zeros_like(lse.v))).abs()
    arg_v = SL2 * s.v - torch.where(row_ok, lse.v[..., None], torch.zeros_like(M)) * LOG2E
    arg_e = SL2 * s.e + LOG2E * dlse[..., None] + gamma(2) * (SL2 * s.v.abs() + LOG2E * lk.abs()[..., None])
    pb = ex2_rv(_rnd(arg_v, arg_e), valid)
    dsc = Rv(torch.tensor(SCALE, dtype=F64))
    if p_drop > 0:
        tt = _rnd(keep * ks * dP.v - delta.v[..., None], keep * (ks * dP.e + dP.v.abs() * ksR.e) + delta.e[..., None])
    else:
        tt = _rnd(dP.v - delta.v[..., None], dP.e + delta.e[..., None])
    ds = to_bf16(mul(mul(pb, tt), dsc))
    dk = dot('bhij,bhid->bhjd', ds, Q, Np)
    dq = dot('bhij,bhjd->bhid', ds, K, Np)
    dv = mul(dot('bhij,bhid->bhjd', to_bf16(Rv(pb.v * keep, pb.e * keep)), dO, Np), ksR)
    return dict(o=o, og=og, lse=lse, dq=dq, dk=dk, dv=dv, row_ok=row_ok[..., 0])


def autograd64(q, k, v, gate, m, p_drop, seed, dog):
    """float64 autograd of the unclamped softmax attention (rows with a valid key)"""
    B, H, Np, _ = q.shape
    qr, kr, vr = (h64(t).requires_grad_() for t in (q, k, v))
    sim = torch.einsum('bhid,bhjd->bhij', qr, kr) * SCALE
    valid = m[:, None, None, :].expand_as(sim)
    row_ok = valid.any(-1, keepdim=True)
    sim = torch.where(row_ok, sim.masked_fill(~valid, -math.inf), torch.zeros_like(sim))   # (no NaN through rows without a valid key)
    lse = torch.logsumexp(sim, -1)
    attn = torch.where(row_ok, torch.softmax(sim, -1), torch.zeros_like(sim))
    if p_drop > 0:
        attn = attn * _dropout_keep(seed, B, H, Np, p_drop) * (65536 / (65536 - int(p_drop * 65536)))
    o = attn @ vr
    g = h64(gate).view(B, Np, H).permute(0, 2, 1)[..., None] if gate is not None else 1.0
    dog4 = h64(dog).view(B, Np, H, 64).permute(0, 2, 1, 3)
    dq, dk, dv = torch.autograd.grad(o * g, [qr, kr, vr], dog4)
    return dict(o=o.detach(), lse=lse.detach(), dq=dq, dk=dk, dv=dv)


# (name, B, H, N', inputs, dropout, gate)
CASES = [
    ('n33-b1-h1-big', 1, 1, 33, 'big', 0.0, True),
    ('n65-b2-h16-grow', 2, 16, 65, 'grow', 0.0, True),
    ('n128-b4-h2-first-tile-masked', 4, 2, 128, 'first_tile', 0.0, False),
    ('n331-b3-h3-all-masked', 3, 3, 331, 'all_masked', 0.0, True),
    ('n331-b2-h3-dropout', 2, 3, 331, 'big', 0.1, True),
    ('n1056-b2-h4-grow', 2, 4, 1056, 'grow', 0.0, True),
    ('n2080-b1-h2', 1, 2, 2080, 'random', 0.0, False),
]


@pytest.mark.parametrize('name,B,H,Np,kind,p_drop,use_gate', CASES, ids=[c[0] for c in CASES])
def test_unclamped_attention_kernels(pkg, name, B, H, Np, kind, p_drop, use_gate):
    seed = 7654321 + Np
    q, k, v, gate, m, mask, dog = inputs(B, H, Np, kind, seed=Np * 17 + H, gate=use_gate)
    s64 = h64(q) @ h64(k).transpose(-1, -2)
    if kind == 'big':
        assert float((s64.abs() * SCALE).max()) > 90                  # 2^(clamp log2 e) of the clamped kernel's approach would overflow
    if kind == 'grow':
        sm = torch.where(m[:, None, None, :], s64, torch.tensor(-math.inf, dtype=F64))
        first, last = sm[..., :64].amax(-1), sm[..., 64 * ((Np - 1) // 64):].amax(-1)
        assert bool((last > first).all())                            # every row's maximum moves on the last key tile
    fw = ufwd(pkg, q, k, v, gate, mask, p_drop, seed)
    bw = ubwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, p_drop, seed)
    torch.cuda.synchronize()
    assert torch.equal(fw['ws'].cpu(), host_maskbits(m, Np))
    r = restate(q, k, v, gate, m, p_drop, seed, dog, fw['o'], fw['lse'])
    ok = r['row_ok']                                                  # [B, H, Np]
    if B * H * Np * Np <= 3_000_000:
        ag = autograd64(q, k, v, gate, m, p_drop, seed, dog)
        for key in ('o', 'lse', 'dq', 'dk', 'dv'):
            sel = ok if key in ('o', 'lse', 'dq') else torch.ones_like(ok)
            agree(f'{name} {key} (restatement vs float64 autograd)', Rv(r[key].v[sel], r[key].e[sel]), ag[key][sel])
    # rows without a valid key: o = og = 0, lse = -inf, zero dq; their keys (all masked) get zero dk, dv
    okq = ok[..., None].expand(B, H, Np, 64)
    zero = torch.zeros(B, H, Np, 64, dtype=F64)
    check_b(f'{name} o', fw['o'], torch.where(okq, r['o'].v, zero), torch.where(okq, r['o'].e, zero))
    ogv = torch.where(okq, r['og'].v, zero).permute(0, 2, 1, 3).reshape(B * Np, H * 64)
    oge = torch.where(okq, r['og'].e, zero).permute(0, 2, 1, 3).reshape(B * Np, H * 64)
    check_b(f'{name} og', fw['og'], ogv, oge)
    lse_k = fw['lse'].cpu()
    assert bool(torch.isneginf(lse_k[~ok]).all()), f'{name}: lse of rows without a valid key'
    check_f(f'{name} lse', lse_k[ok].contiguous(), r['lse'].v[ok], r['lse'].e[ok])
    check_b(f'{name} dv', bw['dv'], r['dv'].v, r['dv'].e)
    check_b(f'{name} dk', bw['dk'], r['dk'].v, r['dk'].e)
    check_f(f'{name} dq', bw['dq'], torch.where(okq, r['dq'].v, zero), torch.where(okq, r['dq'].e, zero))
    if kind == 'all_masked':
        for t in ('o', 'og', 'dk', 'dv', 'dq'):
            src = fw if t in ('o', 'og') else bw
            x = src[t].view(B, Np, H, 64)[1] if t == 'og' else src[t][1]
            assert bool((x == 0).all()), f'{name}: {t} of the batch element without a valid key'


def test_unclamped_isolation_shared_bitmask_device_seed(pkg):
    """(E) a (b, h) slice launched alone equals the big launch; the shared bitmask and seed + *seed_dev equal the per-call ones"""
    B, H, Np, p_drop = 2, 3, 193, 0.1
    q, k, v, gate, m, mask, dog = inputs(B, H, Np, 'grow', seed=5)
    base, addend = 0x0123456789ABCDEF, 0x0EDCBA9876543211
    total = base + addend
    fw = ufwd(pkg, q, k, v, gate, mask, p_drop, total)
    bw = ubwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, p_drop, total)
    shared = pkg.ops.attn_maskbits(mask, B, Np, dev())
    sd = torch.tensor([addend], dtype=torch.int64, device=dev())
    f2 = ufwd(pkg, q, k, v, gate, None, p_drop, base, ws=shared, ready=1, seed_dev=sd)
    b2 = ubwd(pkg, q, k, v, f2['o'], f2['lse'], gate, None, dog, p_drop, base, ws=shared, ready=1, seed_dev=sd)
    torch.cuda.synchronize()
    for key in ('o', 'og', 'lse'):
        check_e(f'shared bitmask + device seed {key}', f2[key], fw[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_dO', 'ws_delta'):
        check_e(f'shared bitmask + device seed {key}', b2[key], bw[key])
    # with dropout, a slice launched alone has the dropout counters of (b, h) = (0, 0) of the big launch
    sl = lambda t: t[0:1, 0:1].contiguous()
    gs = gate.view(B, Np, H)[0, :, 0:1].contiguous()
    dogs = dog.view(B, Np, H, 64)[0, :, 0].contiguous()
    f1 = ufwd(pkg, sl(q), sl(k), sl(v), gs, mask[0:1].contiguous(), p_drop, total)
    b1 = ubwd(pkg, sl(q), sl(k), sl(v), f1['o'], f1['lse'], gs, mask[0:1].contiguous(), dogs, p_drop, total)
    torch.cuda.synchronize()
    check_e('isolation o', f1['o'], sl(fw['o']))
    check_e('isolation lse', f1['lse'], fw['lse'][0:1, 0:1])
    check_e('isolation dk', b1['dk'], sl(bw['dk']))
    check_e('isolation dv', b1['dv'], sl(bw['dv']))


def test_unclamped_isolation_without_dropout(pkg):
    """(E) every (b, h) slice launched alone equals the big launch"""
    B, H, Np = 2, 3, 193
    q, k, v, gate, m, mask, dog = inputs(B, H, Np, 'big', seed=6)
    fw = ufwd(pkg, q, k, v, gate, mask, 0.0, 1)
    bw = ubwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, 0.0, 1)
    for b in range(B):
        for hh in range(H):
            sl = lambda t: t[b:b + 1, hh:hh + 1].contiguous()
            gs = gate.view(B, Np, H)[b, :, hh:hh + 1].contiguous()
            dogs = dog.view(B, Np, H, 64)[b, :, hh].contiguous()
            f1 = ufwd(pkg, sl(q), sl(k), sl(v), gs, mask[b:b + 1].contiguous(), 0.0, 1)
            b1 = ubwd(pkg, sl(q), sl(k), sl(v), f1['o'], f1['lse'], gs, mask[b:b + 1].contiguous(), dogs, 0.0, 1)
            torch.cuda.synchronize()
            tag = f'isolation b{b} h{hh}'
            check_e(f'{tag} o', f1['o'], sl(fw['o']))
            check_e(f'{tag} og', f1['og'], fw['og'].view(B, Np, H, 64)[b, :, hh])
            check_e(f'{tag} lse', f1['lse'], fw['lse'][b:b + 1, hh:hh + 1])
            check_e(f'{tag} dk', b1['dk'], sl(bw['dk']))
            check_e(f'{tag} dv', b1['dv'], sl(bw['dv']))
            check_e(f'{tag} d_gate', b1['d_gate'], bw['d_gate'].view(B, Np, H)[b, :, hh:hh + 1])


def test_unclamped_equals_clamped_at_zero_logits(pkg):
    """(E) with q = 0 every logit is 0 in both modes: the clamped and the unclamped kernels compute the same P = 2^0 = 1 and the same
    dropout keep pattern for the same seed, so every output is bit-identical"""
    B, H, Np, p_drop, seed = 2, 3, 331, 0.1, 0xC0FFEE
    q, k, v, gate, m, mask, dog = inputs(B, H, Np, 'random', seed=8)
    q = torch.zeros_like(q)
    fc = attn_fwd(pkg, q, k, v, gate, mask, 50.0, p_drop, seed)
    bc = attn_bwd(pkg, q, k, v, fc['o'], fc['lse'], gate, mask, dog, 50.0, p_drop, seed)
    fu = ufwd(pkg, q, k, v, gate, mask, p_drop, seed)
    bu = ubwd(pkg, q, k, v, fu['o'], fu['lse'], gate, mask, dog, p_drop, seed)
    torch.cuda.synchronize()
    for key in ('o', 'og', 'lse'):
        check_e(f'zero logits {key}', fu[key], fc[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_delta'):   # (dq is summed over key tiles with atomics, in no fixed order)
        check_e(f'zero logits {key}', bu[key], bc[key])
    keep = _dropout_keep(seed, B, H, Np, p_drop)
    assert 0.05 < 1 - float(keep.double().mean()) < 0.15


# ------------------------------------------------------------------------------------------------------------------ qkv_post
@pytest.mark.parametrize('H,mix', [(8, True), (8, False), (16, True), (3, True)])
def test_qkv_post_no_gate_bit_exact(pkg, H, mix):
    """(E) [q|k|v|mix] gives the q, k, v and the d_qkvg columns of [q|k|v|gate|mix] with the same data, bit for bit; pad columns are 0"""
    B, Np, I = 2, 97, H * 64
    g = torch.Generator().manual_seed(H + 10 * mix)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev())
    ldg = (3 * I + (2 if mix else 1) * H + 7) // 8 * 8
    ldn = (3 * I + (1 if mix else 0) * H + 7) // 8 * 8
    T = B * Np
    full = rn(T, ldg).to(BF16)
    nog = torch.zeros(T, ldn, device=dev(), dtype=BF16)
    nog[:, :3 * I] = full[:, :3 * I]
    if mix:
        nog[:, 3 * I:3 * I + H] = full[:, 3 * I + H:3 * I + 2 * H]
    cs, sn = pkg.ops.rotary_table(Np, dev())
    gb, mb = rn(H), rn(H) if mix else None
    vf = rn(B, H, Np, 64).to(BF16) if mix else None
    out = {}
    for tag, qkvg, ld, ng in (('gate', full, ldg, 0), ('nogate', nog, ldn, 1)):
        q, k, v = (nans((B, H, Np, 64), BF16) for _ in range(3))
        gate = nans((T, H), F32) if not ng else None
        a = pkg.lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=None if ng else gb, mix_bias=mb, rot_cos=cs, rot_sin=sn,
                              v_first=vf, q=q, k=k, v=v, gate=gate, B=B, H=H, Np=Np, dim_head=64, no_gate=ng)
        pkg.lib.call('b200_qkv_post_fwd', a, stream())
        out[tag] = dict(q=q, k=k, v=v, gate=gate)
    gen = torch.Generator().manual_seed(3)
    dq = torch.randn(B, H, Np, 64, generator=gen).to(dev())
    dk, dv, dve = (torch.randn(B, H, Np, 64, generator=gen).to(dev()).to(BF16) for _ in range(3))
    dgate = torch.randn(T, H, generator=gen).to(dev())
    for tag, qkvg, ld, ng in (('gate', full, ldg, 0), ('nogate', nog, ldn, 1)):
        d = nans((T, ld), BF16)
        dvf = nans((B, H, Np, 64), BF16) if mix else None
        a = pkg.lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=None if ng else gb, mix_bias=mb, rot_cos=cs, rot_sin=sn,
                              v_first=vf, gate=out[tag]['gate'], dq=dq, dk=dk, dv=dv, dv_extra=dve, d_gate=None if ng else dgate,
                              d_qkvg=d, d_vfirst=dvf, B=B, H=H, Np=Np, dim_head=64, dq_fp32=1, no_gate=ng)
        pkg.lib.call('b200_qkv_post_bwd', a, stream())
        out[tag].update(d=d, dvf=dvf)
    torch.cuda.synchronize()
    for key in ('q', 'k', 'v'):
        check_e(f'no-gate {key}', out['nogate'][key], out['gate'][key])
    dn, dg = out['nogate']['d'], out['gate']['d']
    check_e('no-gate d_qkv', dn[:, :3 * I], dg[:, :3 * I])
    if mix:
        check_e('no-gate d_mix', dn[:, 3 * I:3 * I + H], dg[:, 3 * I + H:3 * I + 2 * H])
        check_e('no-gate d_vfirst', out['nogate']['dvf'], out['gate']['dvf'])
    used = 3 * I + (H if mix else 0)
    assert bool((dn[:, used:].float() == 0).all())


# ------------------------------------------------------------------------------------------------------------------ autograd node
@pytest.mark.parametrize('gate,clamp', [(False, 50.0), (True, None), (False, None)])
def test_attention_node_variants(pkg, gate, clamp):
    """ops.Attention at the cfg2 widths (d512, 8 heads) without gate and/or clamp: og and v equal the composition of b200_qkv_post and
    the attention kernels it wraps (E), and its parameter gradients agree with float64 autograd of the x-transformers attention to
    bf16 accuracy (cosine >= 0.999)"""
    from attn_variants import attention as xt_attention
    ops = pkg.ops
    B, Np, H, Din = 2, 160, 8, 512
    T, I = B * Np, H * 64
    g = torch.Generator().manual_seed(11 + gate)
    rn = lambda *s: torch.randn(*s, generator=g)
    xn = rn(T, Din).to(BF16).to(dev()).requires_grad_()
    ws = {n: (rn(*s) * Din ** -0.5).to(dev()).requires_grad_() for n, s in (('q', (I, Din)), ('k', (I, Din)), ('v', (I, Din)))}
    wg = (rn(H, Din) * 0.05).to(dev()).requires_grad_() if gate else None
    bg = rn(H).to(dev()).requires_grad_() if gate else None
    rows = [ws['q'], ws['k'], ws['v']] + ([wg] if gate else [])
    wpack = torch.cat(rows).to(BF16).contiguous()
    cs, sn = ops.rotary_table(Np, dev())
    mask = torch.ones(B, Np, dtype=torch.uint8, device=dev())
    mask[1, 120:] = 0
    og, v = ops.Attention.apply(xn, ws['q'], ws['k'], ws['v'], wg, bg, None, None, None, wpack, cs, sn, mask, B, Np, H, 0.0, 1, clamp, None)
    assert og.grad_fn.meta[10] == gate
    dog = (rn(T, I) * mask.cpu().view(T, 1)).to(BF16).to(dev())   # masked query rows: no gradient (the reference zeroes their output)
    og.backward(dog)
    torch.cuda.synchronize()
    # float64 autograd of the same attention on the same (bf16) operands
    sd = {f'a.to_{c}.weight': h64(ws[c]).requires_grad_() for c in 'qkv'}
    sd['a.to_out.weight'] = torch.eye(I, dtype=F64)
    if gate:
        sd['a.to_v_head_gate.weight'] = h64(wg).requires_grad_()
        sd['a.to_v_head_gate.bias'] = h64(bg).requires_grad_()
    x64 = h64(xn).view(B, Np, Din).requires_grad_()
    freqs = O.rotary_freqs(Np, 64, 'cpu').to(F64)
    ref, _ = xt_attention(sd, 'a', x64, mask.cpu().bool(), freqs, None, H, 64, clamp)
    ref = ref * mask.cpu()[..., None]
    (ref * h64(dog).view(B, Np, I)).sum().backward()
    ok = mask.cpu().bool().view(-1)
    assert rel_l2(og.float().cpu()[ok], ref.detach().view(T, I).float()[ok]) < 2e-2
    pairs = [(xn.grad, x64.grad.view(T, Din))] + [(ws[c].grad, sd[f'a.to_{c}.weight'].grad) for c in 'qkv']
    if gate:
        pairs += [(wg.grad, sd['a.to_v_head_gate.weight'].grad), (bg.grad, sd['a.to_v_head_gate.bias'].grad)]
    for got, want in pairs:
        got, want = got.double().cpu().flatten(), want.double().flatten()
        assert float(got @ want / (got.norm() * want.norm())) >= 0.999


# ------------------------------------------------------------------------------------------------------------------ whole model
ATTN_SETTINGS = {'plain': dict(), 'gate_only': dict(gate_value_heads=True), 'clamp30': dict(softclamp_logits=True, logit_softclamp_value=30.)}


@pytest.mark.parametrize('setting', list(ATTN_SETTINGS))
def test_e2tts_cfg2_shape_attn_kwargs_vs_oracle(pkg, setting):
    """BASELINE cfg2's model (d512, depth 8, 8 heads, N = 1024, ragged B = 2) with these attn_kwargs: conditioning probe < 1.5 %, loss
    within 1e-2, prediction rel-L2 within 3e-2, every gradient cosine >= 0.99 (the bounds of tests/test_gpu_parity_full.py)"""
    kw = ATTN_SETTINGS[setting]
    with variant_oracle(kw):
        _whole_model(pkg, dict(dim=512, depth=8, heads=8), B=2, N=1024, lens=[1024, 800], seed=40, model_kw=dict(attn_kwargs=kw))


def _small(pkg, seed, kw, cls='E2TTS'):
    import random
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dim=128, depth=2, heads=2, dropout=0., max_seq_len=256, attn_kwargs=kw)
    model = pkg.E2TTS(transformer=t, use_vocos=False) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=t)
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1)
    model.load_state_dict(sd)
    return model.to(dev()), sd


def test_sample_32_steps_plain_attention_vs_oracle(pkg):
    model, sd = _small(pkg, 60, dict())
    torch.manual_seed(61)
    cond = torch.randn(2, 24, 100)
    text = ['Hello', 'Goodbye']
    y0 = torch.randn(2, 64, 100)
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(cond.to(dev()), text=text, duration=64, steps=32, cfg_strength=1.0, return_raw_output=True)
    with variant_oracle(dict()):
        want = O.e2tts_sample(sd, O.TransformerCfg(dim=128, depth=2, heads=2), cond, O.list_str_to_tensor(text), duration=64, y0=y0,
                              steps=32, cfg_strength=1.0)
    assert out.shape == want.shape
    assert rel_l2(out.cpu(), want) < 5e-2


@pytest.mark.parametrize('setting', ['plain', 'gate_only'])
def test_graphed_step_matches_eager(pkg, setting):
    """GraphedTrainStep replays the eager step's gradients with these attn_kwargs"""
    model, _ = _small(pkg, 3, ATTN_SETTINGS[setting])
    model.train()
    model.cond_drop_prob = 0.0
    B, N = 2, 96
    mel = torch.randn(B, N, 100, device=dev())
    text = pkg.list_str_to_tensor(['Hello', 'Goodbye']).to(dev())
    x0, times = torch.randn(B, N, 100, device=dev()), torch.rand(B, device=dev())
    span = torch.zeros(B, N, dtype=torch.bool, device=dev())
    span[:, 20:70] = True
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        out = model(mel, text=text)
        out.loss.backward()
        want = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        for p in model.parameters():
            p.grad = None
        del out
        step = pkg.GraphedTrainStep(model, mel, text=text)
        step()
    torch.cuda.synchronize()
    for n, p in model.named_parameters():
        if n in want:
            assert p.grad is not None, n
            assert rel_l2(p.grad.float().cpu(), want[n].float().cpu()) < 2e-3 or float(want[n].norm()) == 0, n


def test_duration_predictor_plain_attention_vs_oracle(pkg):
    """DurationPredictor(attn_kwargs=dict()): loss within 1e-2 of the oracle, gradient cosines >= 0.99"""
    model, sd = _small(pkg, 41, dict(), cls='DurationPredictor')
    model.train()
    mel = torch.randn(3, 72, 100)
    lens = torch.tensor([72, 50, 31])
    text = ['abc', 'hello world', 'x']
    rand_frac = torch.tensor([0.3, 0.6, 0.9])
    with pkg.inject_randomness(duration_rand_frac=rand_frac.to(dev())):
        loss = model(mel.to(dev()), text=text, lens=lens.to(dev()))
    loss.backward()
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    with variant_oracle(dict()):
        ref = O.duration_forward(osd, O.TransformerCfg(cond_on_time=False, dim=128, depth=2, heads=2), mel, O.list_str_to_tensor(text),
                                 lens=lens, rand_frac=rand_frac)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-2 * abs(float(ref))
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None or float(gr.norm()) < 1e-4 * total:
            continue
        got = p.grad.double().cpu().flatten()
        assert float(got @ gr.double().flatten() / (got.norm() * gr.double().norm())) >= 0.99, k
