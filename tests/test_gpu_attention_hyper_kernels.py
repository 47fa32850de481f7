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
from hyper_conv_ref import S, check_hc_case, depth_bwd_warps, depth_check, depth_fwd_threads, hc_fwd_launch
from kernel_checks import (BF16, F32, F64, U, Rv, _rnd, add, agree, check_b, check_e, check_f, chk_b, chk_f, dev, dot, dots,
                           exact, fma, gamma, h64, mono, mul, nans, neg, ones_rv, pkg, sms, stream, to_bf16)
from model_checks import whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


# ================================================================================================================ hyper-connections
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
    check_hc_case(pkg, name, T, D, rpb, mode, fused, use_dbeta, zeros, iso)


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
