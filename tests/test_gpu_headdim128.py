"""GPU: attention with 128-wide heads (Transformer dim_head / text_dim_head = 128) and a text stream with its own head count, from the
kernels up to the whole model.

Kernels: b200_attn_fwd / b200_attn_bwd at dim_head 128 (the <*, 128> forward instantiations and attn_bwd_d128_wgmma_kernel), clamped
and unclamped, with and without the head gate, against the element-wise float64 bounds of the restatement of tests/attn_ref.py;
outputs start NaN-filled. At head dim 128 its dot products run over 128 terms and the score scale is 128 ** -0.5. Rows whose keys
are all masked give o = og = 0, lse = -inf and zero gradients.
Then b200_qkv_post_* and b200_rotary_table at dim_head 128, the ops.Attention / AttnCore nodes, and whole models against the oracle
within the bounds of tests/model_checks.py."""
import math

import pytest
import torch

from attn_ref import attn_bwd, attn_fwd, autograd64, d128_inputs, dropout_keep, host_maskbits, restate
from conftest import rel_l2
from kernel_checks import BF16, F32, F64, U, Rv, agree, check_b, check_e, check_f, dev, gamma, h64, nans, pkg, stream
from model_checks import duration_vs_oracle, graphed_matches_eager, sample_vs_oracle, small_model, step_inputs, whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

DH = 128


# (name, B, H, N', logits, softclamp (None: unclamped), dropout, gate, masked)
CASES = [
    ('n1-b2-h1', 2, 1, 1, 'small', 50.0, 0.0, True, False),
    ('n33-b3-h2-masked', 3, 2, 33, 'mixed', 50.0, 0.0, True, True),
    ('n64-b1-h3-nogate', 1, 3, 64, 'small', 50.0, 0.0, False, False),
    ('n65-b2-h1-unclamped-masked', 2, 1, 65, 'big', None, 0.0, True, True),
    ('n128-b2-h2-unclamped-nogate', 2, 2, 128, 'small', None, 0.0, False, False),
    ('n129-b3-h2-masked', 3, 2, 129, 'mixed', 50.0, 0.0, False, True),
    ('n129-b2-h2-dropout', 2, 2, 129, 'mixed', 50.0, 0.1, True, True),
    ('n65-b2-h1-unclamped-dropout', 2, 1, 65, 'big', None, 0.1, False, True),
    ('n1056-b2-h4', 2, 4, 1056, 'mixed', 50.0, 0.0, True, True),
    ('n1056-b1-h2-unclamped', 1, 2, 1056, 'big', None, 0.0, True, False),
    ('n2080-b1-h1', 1, 1, 2080, 'small', 50.0, 0.0, True, False),
]


@pytest.mark.parametrize('name,B,H,Np,kind,clamp,p_drop,use_gate,masked', CASES, ids=[c[0] for c in CASES])
def test_attention_kernels_d128(pkg, name, B, H, Np, kind, clamp, p_drop, use_gate, masked):
    seed = 97531 + Np
    q, k, v, gate, m, mask, dog = d128_inputs(B, H, Np, kind, use_gate, masked, seed=Np * 13 + H)
    fw = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, clamp, p_drop, seed)
    torch.cuda.synchronize()
    assert torch.equal(fw['ws'].cpu(), host_maskbits(m, Np)), f'{name}: key bitmask'
    r = restate(q, k, v, gate, m, clamp, p_drop, seed, dog, fw['o'], fw['lse'])
    ok = r['row_ok']
    if B * H * Np * Np <= 3_000_000:
        ag = autograd64(q, k, v, gate, m, clamp, p_drop, seed, dog)
        for key in ('o', 'lse', 'dq', 'dk', 'dv'):
            sel = ok if key in ('o', 'lse', 'dq') else torch.ones_like(ok)
            agree(f'{name} {key} (restatement vs float64 autograd)', Rv(r[key].v[sel], r[key].e[sel]), ag[key][sel])
    okq = ok[..., None].expand(B, H, Np, DH)
    zero = torch.zeros(B, H, Np, DH, dtype=F64)
    sel = lambda t: (torch.where(okq, t.v, zero), torch.where(okq, t.e, zero))
    check_b(f'{name} o', fw['o'], *sel(r['o']))
    merge = lambda t: t.permute(0, 2, 1, 3).reshape(B * Np, H * DH)
    ogv, oge = sel(r['og'])
    check_b(f'{name} og', fw['og'], merge(ogv), merge(oge))
    lse_k = fw['lse'].cpu()
    assert bool(torch.isneginf(lse_k[~ok]).all()), f'{name}: lse of rows without a valid key'
    check_f(f'{name} lse', lse_k[ok].contiguous(), r['lse'].v[ok], r['lse'].e[ok])
    if gate is not None:
        okg = ok.permute(0, 2, 1).reshape(B * Np, H)
        dgo = torch.where(okg, r['dgate_own'].permute(0, 2, 1).reshape(B * Np, H), 0.)
        check_f(f'{name} d_gate', bw['d_gate'], dgo, r['dgate_e'].permute(0, 2, 1).reshape(B * Np, H))
    check_b(f'{name} ws_dO', bw['ws_dO'], r['dO'].v, U * r['dO'].v.abs())
    check_b(f'{name} dv', bw['dv'], r['dv'].v, r['dv'].e)
    check_b(f'{name} dk', bw['dk'], r['dk'].v, r['dk'].e)
    check_f(f'{name} dq', bw['dq'], *sel(r['dq']))
    if masked and B > 1:   # batch element 1 has no valid key
        for t, src in (('o', fw), ('dk', bw), ('dv', bw), ('dq', bw)):
            assert bool((src[t][1] == 0).all()), f'{name}: {t} of the batch element without a valid key'
        assert bool((fw['og'].view(B, Np, H, DH)[1] == 0).all())


@pytest.mark.parametrize('clamp', [50.0, None])
def test_dropout_kept_set_equals_dim_head_64(pkg, clamp):
    """with q = 0 every logit is 0, so o = keep_scale * sum over kept keys of v / (number of valid keys): the forward at dim_head 128
    on v = [v64 | v'] gives, in its first 64 columns, bit for bit what the dim_head-64 kernel gives on v64 with the same seed — the
    kept set is indexed by (b, h, query, key) whatever the head width"""
    B, H, Np, p_drop, seed = 2, 3, 193, 0.1, 0xBADC0DE
    q, k, v, gate, m, mask, dog = d128_inputs(B, H, Np, 'small', True, True, seed=3)
    q = torch.zeros_like(q)
    f128 = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed)
    sl = lambda t: t[..., :64].contiguous()
    f64 = attn_fwd(pkg, sl(q), sl(k), sl(v), gate, mask, clamp, p_drop, seed)
    torch.cuda.synchronize()
    check_e('kept set: o', sl(f128['o']), f64['o'])
    check_e('kept set: lse', f128['lse'], f64['lse'])
    keep = dropout_keep(seed, B, H, Np, p_drop)
    assert 0.05 < 1 - float(keep.double().mean()) < 0.15


# ------------------------------------------------------------------------------------------------------------------ qkv_post, rotary
def test_rotary_table_d128(pkg):
    for Np in (1, 97, 2080):
        cs, sn = pkg.ops.rotary_table(Np, dev(), 128)
        torch.cuda.synchronize()
        assert cs.shape == (Np, 64)
        f = O.rotary_freqs(Np, 128, 'cpu').double()[:, ::2]      # interleaved pairs share one frequency
        fd = torch.arange(Np, dtype=F64)[:, None] * (10000.0 ** (-torch.arange(0, 128, 2, dtype=F64) / 128))[None]
        assert float((f - fd).abs().max()) <= 1e-6 * max(Np, 1)
        # fp32 argument n * inv_freq (two roundings) through sincosf (a few ulp)
        err = 4 * U * fd.abs() + 8 * U
        check_f(f'rotary cos Np {Np}', cs, torch.cos(fd), err)
        check_f(f'rotary sin Np {Np}', sn, torch.sin(fd), err)


@pytest.mark.parametrize('no_gate,mix', [(False, True), (True, False), (False, False)])
def test_qkv_post_d128(pkg, no_gate, mix):
    B, Np, H = 2, 97, 3
    I = H * DH
    g = torch.Generator().manual_seed(11 + 2 * no_gate + mix)
    ncat = 3 * I + (0 if no_gate else H) + (H if mix else 0)
    ld = (ncat + 7) // 8 * 8
    T = B * Np
    qkvg = torch.randn(T, ld, generator=g).to(BF16)
    gb, mb = torch.randn(H, generator=g), torch.randn(H, generator=g)
    vf = torch.randn(B, H, Np, DH, generator=g).to(BF16) if mix else None
    cs, sn = pkg.ops.rotary_table(Np, dev(), DH)
    to = lambda t: None if t is None else t.to(dev()).contiguous()
    q, k, v = (nans((B, H, Np, DH), BF16) for _ in range(3))
    gate = None if no_gate else nans((T, H), F32)
    a = pkg.lib.make_args('b200_qkv_post_args', qkvg=to(qkvg), ld=ld, gate_bias=None if no_gate else to(gb), mix_bias=to(mb) if mix else None,
                          rot_cos=cs, rot_sin=sn, v_first=to(vf), q=q, k=k, v=v, gate=gate, B=B, H=H, Np=Np, dim_head=DH, no_gate=int(no_gate))
    pkg.lib.call('b200_qkv_post_fwd', a, stream())
    # backward
    dq = torch.randn(B, H, Np, DH, generator=g)
    dk, dv = (torch.randn(B, H, Np, DH, generator=g).to(BF16) for _ in range(2))
    d_gate = torch.randn(T, H, generator=g)
    d_qkvg = nans((T, ld), BF16)
    d_vf = nans((B, H, Np, DH), BF16) if mix else None
    a = pkg.lib.make_args('b200_qkv_post_args', qkvg=to(qkvg), ld=ld, gate_bias=None if no_gate else to(gb), mix_bias=to(mb) if mix else None,
                          rot_cos=cs, rot_sin=sn, v_first=to(vf), gate=gate, dq=to(dq), dk=to(dk), dv=to(dv), d_gate=None if no_gate else to(d_gate),
                          d_qkvg=d_qkvg, d_vfirst=d_vf, B=B, H=H, Np=Np, dim_head=DH, dq_fp32=1, no_gate=int(no_gate))
    pkg.lib.call('b200_qkv_post_bwd', a, stream())
    torch.cuda.synchronize()
    # float64 reference on the kernel's own rotary table
    X = h64(qkvg)
    heads = lambda t: t.view(B, Np, H, DH).permute(0, 2, 1, 3)
    c64, s64 = h64(cs).repeat_interleave(2, -1), h64(sn).repeat_interleave(2, -1)

    def rot(t):
        t2 = t.reshape(*t.shape[:-1], -1, 2)
        r = torch.stack((-t2[..., 1], t2[..., 0]), -1).reshape(t.shape)
        return t * c64 + r * s64

    def rot_t(t):   # the transpose of rot (the backward)
        t2 = t.reshape(*t.shape[:-1], -1, 2)
        r = torch.stack((t2[..., 1], -t2[..., 0]), -1).reshape(t.shape)
        return t * c64 + r * s64
    qr, kr = rot(heads(X[:, :I])), rot(heads(X[:, I:2 * I]))
    vr = heads(X[:, 2 * I:3 * I])
    mcol = 3 * I + (0 if no_gate else H)
    if mix:
        mx = torch.sigmoid(X[:, mcol:mcol + H] + mb.double()).view(B, Np, H).permute(0, 2, 1)[..., None]
        vmix = vr * mx + h64(vf) * (1 - mx)
    else:
        vmix = vr
    bnd = lambda t: 4 * U * (t.abs() + 1e-30) + 2 * U * (t.abs())   # two products and a sum in fp32, one bf16 rounding checked by check_b
    check_b('qkv_post q', q, qr, bnd(qr) + 4 * U * (heads(X[:, :I]).abs() * 2))
    check_b('qkv_post k', k, kr, bnd(kr) + 4 * U * (heads(X[:, I:2 * I]).abs() * 2))
    check_b('qkv_post v', v, vmix, 4 * U * (vr.abs() + (h64(vf).abs() if mix else 0)) + 1e-7)
    if not no_gate:
        gt = torch.sigmoid(X[:, 3 * I:3 * I + H] + gb.double())
        check_f('qkv_post gate', gate, gt, 4 * U * gt + 1e-7)
    dqk = lambda t: rot_t(h64(t))
    DQ = dqk(dq.to(BF16).float()) if False else rot_t(dq.double())
    d = h64(d_qkvg)
    merge = lambda t: t.permute(0, 2, 1, 3).reshape(T, I)
    check_b('qkv_post d_q', d_qkvg[:, :I], merge(DQ), merge(4 * U * (dq.double().abs().repeat(1, 1, 1, 1) * 2)))
    DK = rot_t(h64(dk))
    check_b('qkv_post d_k', d_qkvg[:, I:2 * I], merge(DK), merge(4 * U * h64(dk).abs() * 2))
    DV = h64(dv) * (mx if mix else 1.0)
    check_b('qkv_post d_v', d_qkvg[:, 2 * I:3 * I], merge(DV), merge(4 * U * h64(dv).abs()))
    if mix:
        check_b('qkv_post d_vfirst', d_vf, h64(dv) * (1 - mx), 4 * U * h64(dv).abs())
        dmix = (h64(dv) * (vr - h64(vf))).sum(-1) * (mx * (1 - mx))[..., 0]
        dmix_e = gamma(DH + 4) * (h64(dv).abs() * (vr.abs() + h64(vf).abs())).sum(-1) * (mx * (1 - mx))[..., 0] + 1e-7
        check_b('qkv_post d_mix', d_qkvg[:, mcol:mcol + H], dmix.permute(0, 2, 1).reshape(T, H), dmix_e.permute(0, 2, 1).reshape(T, H))
    if not no_gate:
        dg = d_gate.double() * gt * (1 - gt)
        check_b('qkv_post d_gate logit', d_qkvg[:, 3 * I:3 * I + H], dg, 8 * U * dg.abs() + 1e-7)
    used = mcol + (H if mix else 0)
    assert bool((d[:, used:] == 0).all()), 'pad columns of d_qkvg'


# ------------------------------------------------------------------------------------------------------------------ autograd nodes
@pytest.mark.parametrize('B,Np,H,Din,has_mix,has_gate,clamp', [
    (2, 1056, 4, 512, True, True, 50.0),     # cfg2's attention widths at head dim 128
    (3, 37, 1, 96, False, True, 50.0),
    (2, 129, 3, 192, True, False, None),
])
def test_attention_node_d128(pkg, B, Np, H, Din, has_mix, has_gate, clamp):
    """ops.Attention (one GEMM for q/k/v/gate/mix, rotary, value mix, attention, head gate) at head dim 128 against float64 autograd of
    the same composition: rel-L2 of the output and of every gradient within the bf16 budget of tests/test_gpu_autograd_nodes.py"""
    ops = pkg.ops
    g = torch.Generator().manual_seed(B * Np + H)
    I = H * DH
    T = B * Np
    rn = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc)
    xn = rn(T, Din).to(BF16)
    wq, wk, wv = (rn(I, Din, sc=Din ** -0.5).to(BF16) for _ in range(3))
    wg, bg = (rn(H, Din, sc=Din ** -0.5), rn(H)) if has_gate else (None, None)
    wm, bm = (rn(H, Din, sc=Din ** -0.5), rn(H)) if has_mix else (None, None)
    vf = rn(B, H, Np, DH).to(BF16) if has_mix else None
    m = torch.rand(B, Np, generator=g) > 0.2
    m[:, 0] = True
    dog = rn(T, I).to(BF16)
    # the values a first layer (no mix) returns feed every later layer: their gradient arrives as d_v_extra
    dv_extra = None if has_mix else rn(B, H, Np, DH).to(BF16)
    params = [wq, wk, wv] + ([wg] if has_gate else []) + ([wm] if has_mix else [])
    ncat = 3 * I + (int(has_gate) + int(has_mix)) * H
    wpack = torch.cat([p.to(BF16) for p in params]).to(dev()).contiguous()
    to = lambda t: None if t is None else t.to(dev()).contiguous().requires_grad_(t.is_floating_point())
    leaves = dict(xn=to(xn), wq=to(wq), wk=to(wk), wv=to(wv), wg=to(wg), bg=to(bg), wm=to(wm), bm=to(bm), vf=to(vf))
    cs, sn = ops.rotary_table(Np, dev(), DH)
    mask = m.to(torch.uint8).to(dev())
    L = leaves
    og, v = ops.Attention.apply(L['xn'], L['wq'], L['wk'], L['wv'], L['wg'], L['bg'], L['wm'], L['bm'], L['vf'], wpack, cs, sn, mask, B, Np,
                                H, 0.0, 1, clamp, None, None, DH)
    torch.autograd.backward([og] if has_mix else [og, v], [dog.to(dev())] if has_mix else [dog.to(dev()), dv_extra.to(dev())])
    torch.cuda.synchronize()
    # float64 reference
    R = {k: (None if t is None else t.detach().cpu().double().requires_grad_()) for k, t in leaves.items()}
    x = R['xn']
    heads = lambda t: t.view(B, Np, H, DH).permute(0, 2, 1, 3)
    q, k, vv = heads(x @ R['wq'].t()), heads(x @ R['wk'].t()), heads(x @ R['wv'].t())
    v_out = vv
    if has_mix:
        mx = torch.sigmoid(x @ R['wm'].t() + R['bm']).view(B, Np, H).permute(0, 2, 1)[..., None]
        vv = vv * mx + R['vf'] * (1 - mx)
    c64, s64 = h64(cs).repeat_interleave(2, -1), h64(sn).repeat_interleave(2, -1)

    def rot(t):
        t2 = t.reshape(*t.shape[:-1], -1, 2)
        return t * c64 + torch.stack((-t2[..., 1], t2[..., 0]), -1).reshape(t.shape) * s64
    q, k = rot(q), rot(k)
    sim = q @ k.transpose(-1, -2) * DH ** -0.5
    if clamp is not None:
        sim = torch.tanh(sim / clamp) * clamp
    sim = sim.masked_fill(~m[:, None, None, :], -math.inf)
    o = torch.softmax(sim, -1) @ vv
    if has_gate:
        o = o * torch.sigmoid(x @ R['wg'].t() + R['bg']).view(B, Np, H).permute(0, 2, 1)[..., None]
    og_ref = o.permute(0, 2, 1, 3).reshape(T, I)
    outs, grads = [og_ref], [h64(dog)]
    if not has_mix:
        outs.append(v_out)
        grads.append(h64(dv_extra))
    torch.autograd.backward(outs, grads)
    assert rel_l2(og.float().cpu(), og_ref.detach()) < 1e-2
    if not has_mix:
        assert rel_l2(v.float().cpu(), v_out.detach()) < 1e-2
    for key, t in leaves.items():
        if t is None or t.grad is None:
            continue
        assert R[key].grad is not None, key
        e = rel_l2(t.grad.float().cpu(), R[key].grad)
        assert e < 2e-2, (key, e)


def test_attn_core_node_d128(pkg):
    """AttnCore at head dim 128 against float64 autograd (cfg2's 4 x 128 heads at N' = 1056 with a masked batch element)"""
    B, H, Np = 2, 4, 1056
    q, k, v, gate, m, mask, dog = d128_inputs(B, H, Np, 'small', True, True, seed=21)
    m[1] = torch.rand(Np) > 0.5
    m[1, 0] = True
    mask = m.to(torch.uint8).to(dev())
    leaves = [t.clone().requires_grad_() for t in (q, k, v, gate)]
    og = pkg.ops.AttnCore.apply(*leaves, mask, 0.0, 0, 50.0, None)
    og.backward(dog)
    torch.cuda.synchronize()
    R = [h64(t).requires_grad_() for t in (q, k, v, gate)]
    sim = torch.tanh(R[0] @ R[1].transpose(-1, -2) * DH ** -0.5 / 50.0) * 50.0
    o = torch.softmax(sim.masked_fill(~m[:, None, None, :], -math.inf), -1) @ R[2]
    o = (o * R[3].view(B, Np, H).permute(0, 2, 1)[..., None]).permute(0, 2, 1, 3).reshape(B * Np, H * DH)
    o.backward(h64(dog))
    assert rel_l2(og.float().cpu(), o.detach()) < 1e-2
    for name, a, b in zip('qkvg', leaves, R):
        assert rel_l2(a.grad.float().cpu(), b.grad) < 2e-2, name


# ------------------------------------------------------------------------------------------------------------------ whole models
def test_e2tts_d512_depth8_heads4x128_vs_oracle(pkg):
    """cfg2's width (d512, depth 8) with 4 heads of 128 (I = 512, as 8 x 64): N = 1024 ragged, loss, prediction and every gradient"""
    whole_model(pkg, dict(dim=512, depth=8, heads=4, dim_head=128), B=2, N=1024, lens=[1024, 800], seed=40)


def test_e2tts_mixed_geometry_vs_oracle(pkg):
    """audio 8 x 64, text 2 x 128: two rotary tables, two qkv packings"""
    whole_model(pkg, dict(dim=512, depth=2, heads=8, dim_head=64, text_heads=2, text_dim_head=128), B=2, N=224, lens=[224, 170], seed=41)


def test_e2tts_plain_residual_unclamped_d128_vs_oracle(pkg):
    """dim_head 128 with num_residual_streams=1 and attn_kwargs=dict() (no clamp, no head gate), at cfg2's shape like the 64-wide
    tests of these switches"""
    whole_model(pkg, dict(dim=512, depth=8, heads=4, dim_head=128, num_residual_streams=1, attn_kwargs=dict()), B=2, N=1024,
                lens=[1024, 800], seed=40)


SMALL = dict(dim=128, depth=2, heads=1, dim_head=128, text_heads=2, text_dim_head=64)


def test_sample_32_steps_d128_vs_oracle(pkg):
    sample_vs_oracle(pkg, 90, SMALL)


def test_duration_predictor_d128_vs_oracle(pkg):
    duration_vs_oracle(pkg, 92, SMALL)


def test_graphed_step_matches_eager_d128(pkg):
    """GraphedTrainStep replays the eager step's gradients at head dim 128 (audio) / 64 (text, 2 heads)"""
    model, _ = small_model(pkg, 93, **SMALL)
    graphed_matches_eager(pkg, model, *step_inputs(pkg))
