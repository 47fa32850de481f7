"""GPU: attention without the logit soft-clamp (the running-maximum instantiations of csrc/attn_tc.cu) and without the head gate (the
[q|k|v|mix] layout of b200_qkv_post), from the kernels up to the whole model.

Kernels: element-wise float64 bounds of the restatement of tests/attn_ref.py with clamp None, whose docstring bounds the forward's
online softmax per score term. Exact properties are held bit for bit."""
import math

import pytest
import torch

from attn_ref import attn_bwd, attn_fwd, autograd64, dropout_keep, host_maskbits, restate, unclamped_inputs
from conftest import rel_l2
from kernel_checks import BF16, F32, F64, Rv, agree, check_b, check_e, check_f, dev, h64, nans, pkg, stream
from model_checks import duration_vs_oracle, graphed_matches_eager, sample_vs_oracle, small_model, step_inputs, whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

SCALE = 0.125   # 64 ** -0.5


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
    q, k, v, gate, m, mask, dog = unclamped_inputs(B, H, Np, kind, seed=Np * 17 + H, gate=use_gate)
    s64 = h64(q) @ h64(k).transpose(-1, -2)
    if kind == 'big':
        assert float((s64.abs() * SCALE).max()) > 90                  # 2^(clamp log2 e) of the clamped kernel's approach would overflow
    if kind == 'grow':
        sm = torch.where(m[:, None, None, :], s64, torch.tensor(-math.inf, dtype=F64))
        first, last = sm[..., :64].amax(-1), sm[..., 64 * ((Np - 1) // 64):].amax(-1)
        assert bool((last > first).all())                            # every row's maximum moves on the last key tile
    fw = attn_fwd(pkg, q, k, v, gate, mask, None, p_drop, seed)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, None, p_drop, seed, d_gate=True)
    torch.cuda.synchronize()
    assert torch.equal(fw['ws'].cpu(), host_maskbits(m, Np))
    r = restate(q, k, v, gate, m, None, p_drop, seed, dog, fw['o'], fw['lse'])
    ok = r['row_ok']                                                  # [B, H, Np]
    if B * H * Np * Np <= 3_000_000:
        ag = autograd64(q, k, v, gate, m, None, p_drop, seed, dog)
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
    q, k, v, gate, m, mask, dog = unclamped_inputs(B, H, Np, 'grow', seed=5)
    base, addend = 0x0123456789ABCDEF, 0x0EDCBA9876543211
    total = base + addend
    fw = attn_fwd(pkg, q, k, v, gate, mask, None, p_drop, total)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, None, p_drop, total)
    shared = pkg.ops.attn_maskbits(mask, B, Np, dev())
    sd = torch.tensor([addend], dtype=torch.int64, device=dev())
    f2 = attn_fwd(pkg, q, k, v, gate, None, None, p_drop, base, ws=shared, ready=1, seed_dev=sd)
    b2 = attn_bwd(pkg, q, k, v, f2['o'], f2['lse'], gate, None, dog, None, p_drop, base, ws=shared, ready=1, seed_dev=sd)
    torch.cuda.synchronize()
    for key in ('o', 'og', 'lse'):
        check_e(f'shared bitmask + device seed {key}', f2[key], fw[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_dO', 'ws_delta'):
        check_e(f'shared bitmask + device seed {key}', b2[key], bw[key])
    # with dropout, a slice launched alone has the dropout counters of (b, h) = (0, 0) of the big launch
    sl = lambda t: t[0:1, 0:1].contiguous()
    gs = gate.view(B, Np, H)[0, :, 0:1].contiguous()
    dogs = dog.view(B, Np, H, 64)[0, :, 0].contiguous()
    f1 = attn_fwd(pkg, sl(q), sl(k), sl(v), gs, mask[0:1].contiguous(), None, p_drop, total)
    b1 = attn_bwd(pkg, sl(q), sl(k), sl(v), f1['o'], f1['lse'], gs, mask[0:1].contiguous(), dogs, None, p_drop, total)
    torch.cuda.synchronize()
    check_e('isolation o', f1['o'], sl(fw['o']))
    check_e('isolation lse', f1['lse'], fw['lse'][0:1, 0:1])
    check_e('isolation dk', b1['dk'], sl(bw['dk']))
    check_e('isolation dv', b1['dv'], sl(bw['dv']))


def test_unclamped_isolation_without_dropout(pkg):
    """(E) every (b, h) slice launched alone equals the big launch"""
    B, H, Np = 2, 3, 193
    q, k, v, gate, m, mask, dog = unclamped_inputs(B, H, Np, 'big', seed=6)
    fw = attn_fwd(pkg, q, k, v, gate, mask, None, 0.0, 1)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, None, 0.0, 1)
    for b in range(B):
        for hh in range(H):
            sl = lambda t: t[b:b + 1, hh:hh + 1].contiguous()
            gs = gate.view(B, Np, H)[b, :, hh:hh + 1].contiguous()
            dogs = dog.view(B, Np, H, 64)[b, :, hh].contiguous()
            f1 = attn_fwd(pkg, sl(q), sl(k), sl(v), gs, mask[b:b + 1].contiguous(), None, 0.0, 1)
            b1 = attn_bwd(pkg, sl(q), sl(k), sl(v), f1['o'], f1['lse'], gs, mask[b:b + 1].contiguous(), dogs, None, 0.0, 1)
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
    q, k, v, gate, m, mask, dog = unclamped_inputs(B, H, Np, 'random', seed=8)
    q = torch.zeros_like(q)
    fc = attn_fwd(pkg, q, k, v, gate, mask, 50.0, p_drop, seed)
    bc = attn_bwd(pkg, q, k, v, fc['o'], fc['lse'], gate, mask, dog, 50.0, p_drop, seed)
    fu = attn_fwd(pkg, q, k, v, gate, mask, None, p_drop, seed)
    bu = attn_bwd(pkg, q, k, v, fu['o'], fu['lse'], gate, mask, dog, None, p_drop, seed)
    torch.cuda.synchronize()
    for key in ('o', 'og', 'lse'):
        check_e(f'zero logits {key}', fu[key], fc[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_delta'):   # (dq is summed over key tiles with atomics, in no fixed order)
        check_e(f'zero logits {key}', bu[key], bc[key])
    keep = dropout_keep(seed, B, H, Np, p_drop)
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
    ref, _ = O.attention(sd, 'a', x64, mask.cpu().bool(), freqs, None, H, 64, clamp, gate)
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
    whole_model(pkg, dict(dim=512, depth=8, heads=8, attn_kwargs=kw), B=2, N=1024, lens=[1024, 800], seed=40)


def test_sample_32_steps_plain_attention_vs_oracle(pkg):
    sample_vs_oracle(pkg, 60, dict(dim=128, depth=2, heads=2, attn_kwargs=dict()))


@pytest.mark.parametrize('setting', ['plain', 'gate_only'])
def test_graphed_step_matches_eager(pkg, setting):
    """GraphedTrainStep replays the eager step's gradients with these attn_kwargs"""
    model, _ = small_model(pkg, 3, dim=128, depth=2, heads=2, attn_kwargs=ATTN_SETTINGS[setting])
    graphed_matches_eager(pkg, model, *step_inputs(pkg))


def test_duration_predictor_plain_attention_vs_oracle(pkg):
    """DurationPredictor(attn_kwargs=dict()): loss within 1e-2 of the oracle, gradient cosines >= 0.99"""
    duration_vs_oracle(pkg, 41, dict(dim=128, depth=2, heads=2, attn_kwargs=dict()))
