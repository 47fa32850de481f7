"""Leaf parity tests for the elementwise, conditioning and loss-head kernels (csrc/elementwise.cu, csrc/small.cu).

Each entry point runs on the GPU and is compared, element by element, with a float64 restatement of the same operation computed
on the host from the exact bf16 / fp32 tensors the kernel received (backward references: float64 autograd of that expression).
Where the oracle (oracle/e2tts_oracle.py) has the leaf, the reference is built on it.

Every bound is E (bit-identical), F (fp32) or B (one bf16 rounding of an F value), the classes of tests/kernel_checks.py; the helpers
below carry the derivations. Where a case exists to reach a code path behind a size threshold, the test asserts that it is on the
intended side.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_checks import BF16, F32, F64, U, U16, bf16_ulp, check_b, check_e, check_f, check_zero, dev, gamma, gen, pkg, sig_err
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


def bfr(t):
    """round to bf16 (host copy): the exact values a bf16 kernel input holds"""
    return t.to(BF16)


# ---------------------------------------------------------------------------------------------------------------------- small linear
SL_XS_MAX = 12 * 1024    # floats of X the forward stages in shared memory (csrc/small.cu)
SL_SLAB = 256            # largest dX slab of output features per block


def _sl_launch(N, num_sms):
    """the host side of b200_small_linear_*: outputs per warp of the forward, output features per dX block"""
    npw = 1
    while npw < 8 and (N + 8 * npw * 2 - 1) // (8 * npw * 2) >= 2 * num_sms:
        npw *= 2
    slab = SL_SLAB
    while slab > 32 and (N + slab - 1) // slab < num_sms:
        slab >>= 1
    return npw, slab


def _act64(act, z):
    if act == 1:
        return F.silu(z)
    if act == 2:
        return torch.sigmoid(z)
    if act == 3:
        return 1 + z
    if act == 4:
        return F.softplus(z)     # threshold 20: z itself above it, as the kernel
    return z


# max |act'| and max |act''| (silu' peaks at 1.0998, silu''(0) = 1/2, sigmoid'' <= 1/(6 sqrt 3), softplus'' = sigmoid' <= 1/4)
ACT_D1 = {0: 1.0, 1: 1.1, 2: 0.25, 3: 1.0, 4: 1.0}
ACT_D2 = {0: 0.0, 1: 0.5, 2: 0.0963, 3: 0.0, 4: 0.25}
# act(z) evaluated in fp32 is within u (a |y| + b) of act of the fp32 z: sigmoid = 1 / (1 + expf(-z)) with expf <= 2 ulp (4u relative)
# -> <= 4u sigma (1 - sigma) / sigma + 2u (add, division) <= 6u relative; silu multiplies once more (7u); 1 + z rounds once;
# softplus: expf's 4u moves log1p(e) by <= 4u e / (1 + e) <= 4u, log1pf <= 1 ulp (2u relative); above 20 it is z itself.
ACT_EVAL = {0: (0, 0), 1: (7, 0), 2: (6, 0), 3: (1, 0), 4: (2, 4)}


def _per_col(act, seg, N):
    """activation of every output feature; act 5 alternates (1 + z) and sigmoid per seg-wide block (csrc/small.cu act_of)"""
    if act != 5:
        return torch.full((N,), act)
    return torch.where((torch.arange(N) // seg) % 2 == 1, 2, 3)


def _check_small_linear(ops, X, W, bias, act, seg=1, seg_major=False, seed=0, tag=''):
    """ops.SmallLinear forward + backward against float64 autograd of act(X W^T + bias).
    Z is an fp32 inner product of K terms plus the bias: within gamma(K + 1) sum|x w| + |b| (bZ). Y adds act' * bZ and ACT_EVAL.
    Backward: dZ = dY act'(Z) with the kernel's Z, so dZ moves by |dY| (max|act''| bZ + the fp32 evaluation of act'), where every
    act' the kernel uses (s, s (1 - s), s (1 + z (1 - s))) is within 16u (1 + |z|): s within 6u, 1 - s within 7u, each further product
    or sum one rounding; plus u|dZ| for the product. dW, dX, dbias are sums of B, N, B products of dZ: gamma(n) sum|terms| plus the
    dZ error carried through."""
    B, K = X.shape
    N = W.shape[0]
    acts = _per_col(act, seg, N)
    g = gen(seed)
    dY = torch.randn(B, N, generator=g)
    lay = (lambda t: t.reshape(B, N // seg, seg).permute(1, 0, 2).contiguous()) if seg_major else (lambda t: t)
    unlay = (lambda t: t.permute(1, 0, 2).reshape(B, N)) if seg_major else (lambda t: t)
    leaves = [X.to(dev()).requires_grad_(), W.to(dev()).requires_grad_()] + ([bias.to(dev()).requires_grad_()] if bias is not None else [])
    Y = ops.SmallLinear.apply(leaves[0], leaves[1], leaves[2] if bias is not None else None, act, seg, seg_major)
    assert Y.shape == lay(dY).shape
    grads = torch.autograd.grad(Y, leaves, lay(dY).to(dev()))
    torch.cuda.synchronize()
    rl = [t.detach().cpu().to(F64).requires_grad_() for t in leaves]
    Z = rl[0] @ rl[1].t() + (rl[2] if bias is not None else 0)
    Y64 = sum(torch.where(acts == a, _act64(a, Z), torch.zeros_like(Z)) for a in acts.unique().tolist())
    rg = torch.autograd.grad(Y64, rl + [Z], dY.to(F64))
    dZ64 = rg[-1]
    Zd, Yd = Z.detach(), Y64.detach()
    d1 = torch.tensor([ACT_D1[int(a)] for a in acts], dtype=F64)
    d2 = torch.tensor([ACT_D2[int(a)] for a in acts], dtype=F64)
    ea = torch.tensor([ACT_EVAL[int(a)][0] for a in acts], dtype=F64)
    eb = torch.tensor([ACT_EVAL[int(a)][1] for a in acts], dtype=F64)
    nonlin = torch.tensor([int(a) in (1, 2, 4) for a in acts], dtype=F64)
    aX, aW = X.to(F64).abs(), W.to(F64).abs()
    bZ = gamma(K + 1) * (aX @ aW.t() + (bias.to(F64).abs() if bias is not None else 0))
    check_f(f'{tag}act{act} Y', unlay(Y), Yd, d1 * bZ + U * (ea * Yd.abs() + eb))
    adY = dY.to(F64).abs()
    bdZ = adY * (d2 * bZ + nonlin * 16 * U * (1 + Zd.abs())) + U * dZ64.abs()
    adZ = dZ64.abs()
    check_f(f'{tag}act{act} dX', grads[0], rg[0], gamma(N) * (adZ @ aW) + bdZ @ aW)
    check_f(f'{tag}act{act} dW', grads[1], rg[1], gamma(B) * (adZ.t() @ aX) + bdZ.t() @ aX)
    if bias is not None:
        check_f(f'{tag}act{act} dbias', grads[2], rg[2], gamma(B) * adZ.sum(0) + bdZ.sum(0))
    return Zd


# (B, K, where the forward reads X, which dX path runs): every combination of the two thresholds
SL_CASES = [
    (1, 129, 'smem', 'generic'), (1, 512, 'smem', 'vec'), (1, 1024, 'smem', 'generic'),
    (16, 129, 'smem', 'generic'), (16, 512, 'smem', 'vec'), (16, 1024, 'global', 'generic'),
    (17, 129, 'smem', 'generic'), (17, 512, 'smem', 'vec'), (17, 1024, 'global', 'generic'),
    (32, 129, 'smem', 'generic'), (32, 512, 'global', 'vec'), (32, 1024, 'global', 'generic'),
    (64, 129, 'smem', 'generic'), (64, 512, 'global', 'vec'), (64, 1024, 'global', 'generic'),
]


@pytest.mark.parametrize('B,K,xpath,dxpath', SL_CASES, ids=[f'B{b}-K{k}-{x}-{d}' for b, k, x, d in SL_CASES])
def test_small_linear(pkg, B, K, xpath, dxpath):
    """every activation (act 5 with 32-wide segments); z spans about +-30 so softplus crosses its threshold of 20 and sigmoid
    saturates; B > 16 takes two or more 16-row batch passes."""
    assert (B * K <= SL_XS_MAX) == (xpath == 'smem')
    assert (K % 4 == 0 and K <= 512) == (dxpath == 'vec')
    g = gen(1000 + 7 * B + K)
    N = 96
    X = torch.randn(B, K, generator=g)
    W = torch.randn(N, K, generator=g) * (10 / math.sqrt(K))     # z ~ N(bias, 10^2)
    bias = torch.randn(N, generator=g)
    W[:2] *= 0.1                                                 # features 0 and 1 sit at z ~ +-25: past the softplus threshold,
    bias[0], bias[1] = 25.0, -25.0                               # sigmoid saturated at both ends
    for act in range(6):
        Z = _check_small_linear(pkg.ops, X, W, bias, act, seg=32 if act == 5 else 1, seed=act, tag=f'B{B} K{K} ')
    assert bool((Z > 20).any()) and bool((Z < -20).any()) and bool((Z.abs() < 20).any())


@pytest.mark.parametrize('B', [4, 32])
def test_small_linear_seg_major_gains(pkg, B, d=512, L=18):
    """the batched gain projection of a deep d = 512 stack: act 5, seg = d, seg-major output, N = 4 L d; large enough that a warp
    computes several outputs and the dX slab is the full 256 features"""
    N = 4 * L * d
    npw, slab = _sl_launch(N, torch.cuda.get_device_properties(0).multi_processor_count)
    assert npw > 1 and slab == SL_SLAB
    g = gen(77 + B)
    X = torch.randn(B, d, generator=g)
    W = torch.randn(N, d, generator=g) * (4 / math.sqrt(d))
    bias = torch.randn(N, generator=g)
    _check_small_linear(pkg.ops, X, W, bias, 5, seg=d, seg_major=True, seed=B, tag='gains ')


@pytest.mark.parametrize('B', [2, 16])
def test_small_linear_seg_major_gains_depth24_d1024(pkg, B):
    """the same projection at the width and depth of the d1024 depth-24 models: N = 4 * 24 * 1024 = 98 304 gains"""
    test_small_linear_seg_major_gains(pkg, B, d=1024, L=24)


def test_small_linear_duration_head(pkg):
    """the DurationPredictor head: N = 1, softplus, B = 32 rows of K = 512 (X read from global memory, two batch passes);
    the rows are placed so that z runs from -30 to 30"""
    B, K = 32, 512
    assert B * K > SL_XS_MAX and B > 16
    g = gen(5)
    W = torch.randn(1, K, generator=g, dtype=F64) / math.sqrt(K)
    bias = torch.tensor([0.25], dtype=F64)
    X = torch.randn(B, K, generator=g, dtype=F64)
    target = torch.linspace(-30, 30, B, dtype=F64)
    X = X + ((target - bias - X @ W[0]) / (W[0] @ W[0]))[:, None] * W[0][None]
    Z = _check_small_linear(pkg.ops, X.float(), W.float(), bias.float(), 4, seed=9, tag='duration ')
    assert bool((Z > 20).any()) and bool((Z < 20).any())


# ---------------------------------------------------------------------------------------------------------------------- time MLP
@pytest.mark.parametrize('d', [128, 512, 1024])
def test_fourier_embed_and_time_mlp(pkg, d):
    """RandomFourierEmbed + Linear(d + 1, d) + SiLU, the time-MLP lines of O.transformer_forward (e2_tts.py:355-364, 621-625).
    Fourier features: the kernel forms f = ((t w) 2) pi_f: pi_f is within u of pi and two products round, so f is within 3u|f|;
    sincosf adds <= 2 ulp (4u relative). The MLP is checked from the kernel's own features (its K = d + 1 takes the generic dX path)."""
    half = d // 2
    g = gen(d)
    times = torch.cat([torch.tensor([0.0, 1.0]), torch.rand(2, generator=g)])
    w = torch.randn(half, generator=g)
    four = pkg.ops.fourier_embed(times.to(dev()), w.to(dev()))
    f = times.to(F64)[:, None] * w.to(F64)[None] * 2 * math.pi
    ref = torch.cat((times.to(F64)[:, None], f.sin(), f.cos()), -1)
    fb = 3 * U * f.abs()
    check_f('fourier t', four[:, 0], ref[:, 0], 0.0)
    check_f('fourier sin', four[:, 1:half + 1], ref[:, 1:half + 1], fb + 4 * U * ref[:, 1:half + 1].abs())
    check_f('fourier cos', four[:, half + 1:], ref[:, half + 1:], fb + 4 * U * ref[:, half + 1:].abs())
    check_f('fourier at t = 0', four[0, 1:], torch.cat([torch.zeros(half), torch.ones(half)]).to(F64), 0.0)
    K = d + 1
    assert K % 4 != 0                         # dX generic path
    lin = torch.nn.Linear(K, d)
    _check_small_linear(pkg.ops, four.cpu(), lin.weight.detach(), lin.bias.detach(), 1, seed=d, tag='time mlp ')


# ---------------------------------------------------------------------------------------------------------------------- rotary
@pytest.mark.parametrize('Np', [1, 33, 1056, 2080])
def test_rotary_table(pkg, Np):
    """cos/sin of n * 10000^(-2j/64) against float64 (the angles of O.rotary_freqs, without its fp32 rounding). The kernel's
    exponent -(2j)/64 is exact, powf is within 4 ulp (8u relative) and n * inv rounds once: the angle is within 9u n inv; sincosf
    adds <= 2 ulp. Rotating a q/k pair by an angle off by delta moves it by delta * |pair|: the bound stays under 2^-9, a quarter of
    the bf16 spacing 2^-7 at the pair's scale, so the table cannot move a rotated bf16 value by a full ulp."""
    cs, sn = pkg.ops.rotary_table(Np, dev())
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=F64) / 64))
    ang = torch.arange(Np, dtype=F64)[:, None] * inv[None]
    of = O.rotary_freqs(Np, 64, torch.device('cpu')).to(F64)         # the oracle's layout: interleaved duplicates of the angles
    assert torch.equal(of[:, 0::2], of[:, 1::2])
    assert torch.allclose(of[:, 0::2], ang, rtol=1e-6, atol=0)
    eang = 9 * U * ang
    assert float(eang.max()) <= 2.0 ** -9
    check_f('rotary cos', cs, ang.cos(), eang + 4 * U * ang.cos().abs())
    check_f('rotary sin', sn, ang.sin(), eang + 4 * U * ang.sin().abs())


# ---------------------------------------------------------------------------------------------------------------------- qkv post
def _rot(t, c, s):
    """O.apply_rotary with given cos/sin (interleaved pairs)"""
    t2 = t.reshape(*t.shape[:-1], -1, 2)
    r = torch.stack((-t2[..., 1], t2[..., 0]), -1).reshape(t.shape)
    return t * c + r * s


def _rot_abs(t, c, s):
    """|x0 c| + |x1 s| (resp. |x1 c| + |x0 s|): a rotated component is two products and one add, <= 2u of this"""
    t2 = t.abs().reshape(*t.shape[:-1], -1, 2)
    r = torch.stack((t2[..., 1], t2[..., 0]), -1).reshape(t.shape)
    return t.abs() * c.abs() + r * s.abs()


@pytest.mark.parametrize('H,Np', [(2, 33), (3, 1056), (8, 33), (16, 1056)])
def test_qkv_post(pkg, H, Np):
    """rotary on q, k; value-residual mix; head gate; and the backward as the model calls it (fp32 dq), with and without v_first and
    the layer-0 value-residual gradient dv_extra. Pad columns of d_qkvg (row pitch > 3I + (1 or 2) H) must be exactly 0."""
    lib, ops = pkg.lib, pkg.ops
    g = gen(40 + H + Np)
    B, I = 2, 64 * H
    T = B * Np
    cs, sn = ops.rotary_table(Np, dev())
    c64 = cs.cpu().to(F64).repeat_interleave(2, -1)
    s64 = sn.cpu().to(F64).repeat_interleave(2, -1)
    heads = lambda t: t.reshape(B, Np, H, 64).permute(0, 2, 1, 3)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(T, I)
    padded = False
    for vf_on, extra_on in ((False, True), (True, False), (False, False)):
        used = 3 * I + (2 if vf_on else 1) * H
        ld = (used + 7) // 8 * 8
        padded |= ld > used
        qkvg = bfr(torch.randn(T, ld, generator=g) * torch.cat([torch.ones(3 * I), 2 * torch.ones(ld - 3 * I)]))
        gb, mb = torch.randn(H, generator=g), torch.randn(H, generator=g)
        vf = bfr(torch.randn(B, H, Np, 64, generator=g)) if vf_on else None
        dq = torch.randn(B, H, Np, 64, generator=g)
        dk, dv = bfr(torch.randn(B, H, Np, 64, generator=g)), bfr(torch.randn(B, H, Np, 64, generator=g))
        dve = bfr(torch.randn(B, H, Np, 64, generator=g)) if extra_on else None
        dgate = torch.randn(T, H, generator=g)
        D = {k: (v.to(dev()) if v is not None else None) for k, v in dict(qkvg=qkvg, gb=gb, mb=mb, vf=vf, dq=dq, dk=dk, dv=dv, dve=dve,
                                                                          dgate=dgate).items()}
        q, k, v = (torch.empty(B, H, Np, 64, device=dev(), dtype=BF16) for _ in range(3))
        gate = torch.empty(T, H, device=dev(), dtype=F32)
        a = lib.make_args('b200_qkv_post_args', qkvg=D['qkvg'], ld=ld, gate_bias=D['gb'], mix_bias=D['mb'] if vf_on else None, rot_cos=cs,
                          rot_sin=sn, v_first=D['vf'], q=q, k=k, v=v, gate=gate, B=B, H=H, Np=Np, dim_head=64)
        lib.call('b200_qkv_post_fwd', a, ops._stream())
        d_qkvg = torch.full((T, ld), 7.0, device=dev(), dtype=BF16)      # sentinel: every column must be written
        d_vf = torch.empty_like(D['vf']) if vf_on else None
        a = lib.make_args('b200_qkv_post_args', qkvg=D['qkvg'], ld=ld, gate_bias=D['gb'], mix_bias=D['mb'] if vf_on else None, rot_cos=cs,
                          rot_sin=sn, v_first=D['vf'], gate=gate, dq=D['dq'], dk=D['dk'], dv=D['dv'], dv_extra=D['dve'], d_gate=D['dgate'],
                          d_qkvg=d_qkvg, d_vfirst=d_vf, B=B, H=H, Np=Np, dim_head=64, dq_fp32=1)
        lib.call('b200_qkv_post_bwd', a, ops._stream())
        # float64 reference
        X = qkvg.to(F64).requires_grad_()
        xq, xk, xv = heads(X[:, :I]), heads(X[:, I:2 * I]), heads(X[:, 2 * I:3 * I])
        ga = X[:, 3 * I:3 * I + H] + gb.to(F64)
        qr, kr = _rot(xq, c64, s64), _rot(xk, c64, s64)
        gr = torch.sigmoid(ga)
        leaves = [X]
        if vf_on:
            ma = X[:, 3 * I + H:3 * I + 2 * H] + mb.to(F64)
            mix = torch.sigmoid(ma).reshape(B, Np, H).permute(0, 2, 1)[..., None]
            VF = vf.to(F64).requires_grad_()
            leaves.append(VF)
            vr = xv * mix + VF * (1 - mix)
        else:
            vr = xv
        gdv = dv.to(F64) + (dve.to(F64) if extra_on else 0)
        rg = torch.autograd.grad([qr, kr, vr, gr], leaves, [dq.to(F64), dk.to(F64), gdv, dgate.to(F64)])
        Xd = X.detach()
        tag = f'H{H} Np{Np} vf={vf_on} extra={extra_on}'
        check_b(f'q {tag}', q.cpu(), qr.detach(), 2 * U * _rot_abs(heads(Xd[:, :I]), c64, s64))
        check_b(f'k {tag}', k.cpu(), kr.detach(), 2 * U * _rot_abs(heads(Xd[:, I:2 * I]), c64, s64))
        check_f(f'gate {tag}', gate.cpu(), gr.detach(), sig_err(ga.detach()))
        dX = rg[0]
        check_b(f'd_qkvg q {tag}', d_qkvg[:, :I].cpu(), dX[:, :I], rows(2 * U * _rot_abs(dq.to(F64), c64, s64)))
        check_b(f'd_qkvg k {tag}', d_qkvg[:, I:2 * I].cpu(), dX[:, I:2 * I], rows(2 * U * _rot_abs(dk.to(F64), c64, s64)))
        eg = sig_err(ga.detach())
        gd = gr.detach()
        check_b(f'd_qkvg gate logit {tag}', d_qkvg[:, 3 * I:3 * I + H].cpu(), dX[:, 3 * I:3 * I + H],
                dgate.to(F64).abs() * eg * (1 + eg) + 3 * U * (dgate.to(F64) * gd * (1 - gd)).abs())
        ax = gdv.abs()
        e_add = U * ax if extra_on else 0.0          # dv + dv_extra rounds once
        if vf_on:
            em = sig_err(ma.detach()).reshape(B, Np, H).permute(0, 2, 1)[..., None]
            md = mix.detach()
            vfd = vf.to(F64)
            xvd = xv.detach()
            check_b(f'v {tag}', v.cpu(), vr.detach(), xvd.abs() * em + vfd.abs() * (em + U) + 2 * U * ((xvd * md).abs() + (vfd * (1 - md)).abs()))
            check_b(f'd_qkvg v {tag}', d_qkvg[:, 2 * I:3 * I].cpu(), dX[:, 2 * I:3 * I], rows(ax * (em + 2 * U)))
            check_b(f'd_vfirst {tag}', d_vf.cpu(), rg[1], ax * (em + 3 * U))
            # dmix = sum_64 x (vr - vf): three roundings per term and a 64-term sum -> gamma(67) S; times mix (1 - mix) <= 1/4, which
            # itself is within em (1 + em); the two products and 1 - mix round (3u)
            S = (ax * (xvd - vfd).abs()).sum(-1, keepdim=True)
            dmix = (gdv * (xvd - vfd)).sum(-1, keepdim=True)
            ref_m = dX[:, 3 * I + H:3 * I + 2 * H]
            atol = S * gamma(67) / 4 + dmix.abs() * em * (1 + em)
            check_b(f'd_qkvg mix logit {tag}', d_qkvg[:, 3 * I + H:3 * I + 2 * H].cpu(), ref_m,
                    atol[..., 0].permute(0, 2, 1).reshape(T, H) + 3 * U * ref_m.abs())
        else:
            check_e(f'v {tag}', v.cpu(), heads(qkvg[:, 2 * I:3 * I]).contiguous())
            check_b(f'd_qkvg v {tag}', d_qkvg[:, 2 * I:3 * I].cpu(), dX[:, 2 * I:3 * I], rows(e_add * torch.ones_like(ax)))
        check_zero(f'd_qkvg pads {tag}', d_qkvg[:, used:])
    assert padded == (H in (2, 3))


# ---------------------------------------------------------------------------------------------------------------------- assemble
@pytest.mark.parametrize('S', [1, 4])
@pytest.mark.parametrize('R', [0, 32])
@pytest.mark.parametrize('D', [64, 512, 1024])
def test_assemble_and_text_stem(pkg, D, R, S):
    """ops.Assemble (+ abs_pos or none, registers, S streams) and ops.TextStem (embedding gather) forward and backward. The text spans
    several 1024-token slabs of embed_bwd, the filler id 0 repeats more than 256 times inside one slab, id vocab - 1 occurs, some
    vocabulary rows are never hit (their gradient stays exactly 0), and rows >= N of d_abs_pos stay 0."""
    ops = pkg.ops
    g = gen(D + R + S)
    B, N, max_len, V = 4, 600, 640, 257
    assert B * N > 2 * 1024
    h = bfr(torch.randn(B * N, D, generator=g))
    abs_pos = torch.randn(max_len, D, generator=g)
    regs = torch.randn(R, D, generator=g)
    d_out = bfr(torch.randn(B * (R + N), S, D, generator=g))
    dsum = d_out.to(F64).view(B, R + N, S, D)
    asum = dsum.abs()
    d_tok = dsum[:, R:].sum(2)                        # [B, N, D]
    a_tok = asum[:, R:].sum(2)

    def expand(tok):                                  # [B, N, D] fp32 -> the [B (R + N), S, D] bf16 residual streams
        full = torch.cat((regs[None].expand(B, R, D), tok), 1)
        return full[:, :, None].expand(B, R + N, S, D).to(BF16).reshape(B * (R + N), S, D)

    for with_abs in (True, False):
        tag = f'D{D} R{R} S{S} abs_pos={with_abs}'
        leaves = [h.to(dev()).requires_grad_(), abs_pos.to(dev()).requires_grad_() if with_abs else None, regs.to(dev()).requires_grad_()]
        out = ops.Assemble.apply(leaves[0], leaves[1], leaves[2], B, N, S)
        tok = h.float().view(B, N, D) + (abs_pos[:N] if with_abs else 0)
        check_e(f'assemble out {tag}', out, expand(tok))
        grads = torch.autograd.grad(out, [t for t in leaves if t is not None], d_out.to(dev()))
        check_b(f'd_h {tag}', grads[0].cpu(), d_tok.reshape(B * N, D), gamma(S - 1) * a_tok.reshape(B * N, D))
        if with_abs:
            check_f(f'd_abs_pos {tag}', grads[1][:N], d_tok.sum(0), gamma(B * S - 1) * a_tok.sum(0))
            check_zero(f'd_abs_pos rows >= N {tag}', grads[1][N:])
        check_f(f'd_registers {tag}', grads[-1], dsum[:, :R].sum((0, 2)), gamma(B * S - 1) * asum[:, :R].sum((0, 2)))
    # text stem
    ids = torch.randint(0, V, (B, N), generator=g)
    ids[(ids >= 5) & (ids < 10)] = 10                 # rows 5..9 never hit
    ids[0, 100:500] = 0                               # filler: 400 hits of id 0 inside the first slab
    ids[3, N - 1] = V - 1
    assert int((ids.view(-1)[:1024] == 0).sum()) > 256
    emb = torch.randn(V, D, generator=g)
    leaves = [emb.to(dev()).requires_grad_(), regs.to(dev()).requires_grad_()]
    out = ops.TextStem.apply(ids.to(torch.int32).to(dev()), leaves[0], leaves[1], B, N, S)
    tag = f'text D{D} R{R} S{S}'
    check_e(f'text stem out {tag}', out, expand(emb[ids]))
    d_emb, d_reg = torch.autograd.grad(out, leaves, d_out.to(dev()))
    flat = ids.view(-1)
    ref = torch.zeros(V, D, dtype=F64).index_add_(0, flat, d_tok.reshape(B * N, D))
    aref = torch.zeros(V, D, dtype=F64).index_add_(0, flat, a_tok.reshape(B * N, D))
    hits = torch.bincount(flat, minlength=V).to(F64)[:, None]
    check_f(f'd_emb {tag}', d_emb, ref, torch.tensor([gamma(int(n) * S) for n in hits[:, 0]], dtype=F64)[:, None] * aref)
    check_zero(f'd_emb unused rows {tag}', d_emb[5:10])
    assert float(hits[V - 1]) >= 1
    check_f(f'text d_registers {tag}', d_reg, dsum[:, :R].sum((0, 2)), gamma(B * S - 1) * asum[:, :R].sum((0, 2)))


# ---------------------------------------------------------------------------------------------------------------------- interpolated text
class _f64_default:
    def __enter__(self):
        self.old = torch.get_default_dtype()
        torch.set_default_dtype(F64)       # O.interpolated_character_embed's linspace then runs in float64

    def __exit__(self, *a):
        torch.set_default_dtype(self.old)


def test_interp_text_packed_operand(pkg):
    """ops.InterpText against O.interpolated_character_embed: downsampling (Lt 50 -> La 20), equal lengths, a single character,
    a single frame, upsampling; La < N, so every sample has padded rows, which must be exactly 0."""
    ops = pkg.ops
    g = gen(11)
    LT_LA = [(50, 20), (20, 20), (1, 37), (7, 1), (9, 41)]
    B, N, D, V, nt = len(LT_LA), 48, 80, 257, 56
    text = torch.full((B, nt), -1, dtype=torch.long)
    for b, (lt, _) in enumerate(LT_LA):
        text[b, :lt] = torch.randint(0, V, (lt,), generator=g)
    text[0, 3] = V - 1
    Lt = torch.tensor([lt for lt, _ in LT_LA])
    La = torch.tensor([la for _, la in LT_LA])
    assert int(La.max()) < N
    mask = torch.arange(N)[None] < La[:, None]
    emb = torch.randn(V, D, generator=g)
    w1, b1 = torch.randn(D, 1, generator=g) * 0.3, torch.randn(D, generator=g)
    w2, b2 = torch.randn(D, D, generator=g) / math.sqrt(D), torch.randn(D, generator=g) * 0.1
    ids_c = torch.zeros(B, nt, dtype=torch.int32)
    ids_c[:, :] = text.clamp(min=0).to(torch.int32)          # the valid ids are already first
    params = [t.to(dev()).requires_grad_() for t in (emb, w1, b1, w2, b2)]
    w2p = params[3].detach().to(BF16)        # the model passes its weight pack's copy: the same round to nearest even
    te = ops.InterpText.apply(ids_c.to(dev()), Lt.to(torch.int32).to(dev()), La.to(torch.int32).to(dev()), mask.to(torch.uint8).to(dev()),
                              *params[:4], w2p, params[4], B, N)
    d_te = bfr(torch.randn(B * N, D, generator=g))
    grads = torch.autograd.grad(te, params, d_te.to(dev()))
    names = ['embed.weight', 'abs_pos_mlp.1.weight', 'abs_pos_mlp.1.bias', 'abs_pos_mlp.3.weight', 'abs_pos_mlp.3.bias']
    sd = {'embed_text.' + n: t.to(F64).requires_grad_() for n, t in zip(names, (emb, w1, b1, w2, b2))}
    with _f64_default():
        ref = O.interpolated_character_embed(sd, text, N, mask)
    rgrads = torch.autograd.grad(ref, list(sd.values()), d_te.to(F64).view(B, N, D))
    ref = ref.detach().reshape(B * N, D)
    # per-row quantities of the kernel's arithmetic, float64
    m = mask.reshape(-1)
    n_ = torch.arange(N, dtype=F64).repeat(B)
    lt_, la_ = Lt.repeat_interleave(N).to(F64), La.repeat_interleave(N).to(F64)
    src = ((n_ + 0.5) * lt_ / la_ - 0.5).clamp(min=0)
    e_src = 3 * U * (src + 1)                       # scale = Lt / La and two more operations round: <= 3u (|src| + 1)
    step = torch.where(la_ > 1, lt_ / (la_ - 1).clamp(min=1), torch.zeros_like(lt_))
    pos = torch.where((n_ < la_ // 2) | (la_ == 1), n_ * step, lt_ - (la_ - 1 - n_) * step) * m
    e_pos = 3 * U * lt_                             # step rounds, one product, one subtraction: <= 3u Lt
    # interpolated embedding: Lipschitz in src with the largest step between neighbouring characters of the sample
    E = emb.to(F64)
    lip = torch.zeros(B, D, dtype=F64)
    for b, (lt, _) in enumerate(LT_LA):
        if lt > 1:
            lip[b] = (E[text[b, 1:lt]] - E[text[b, :lt - 1]]).abs().amax(0)
    lip = lip.repeat_interleave(N, 0)
    lerp_ref = torch.zeros(B * N, D, dtype=F64)
    with _f64_default():
        for b, (lt, la) in enumerate(LT_LA):
            e = E[text[b, :lt]]
            lerp_ref[b * N:b * N + la] = F.interpolate(e.t()[None, :, :, None], (la, 1), mode='bilinear')[0, :, :, 0].t()
    # lerp = bf16((1 - lam) e0 + lam e1): src error through the Lipschitz constant, four roundings (1 - lam, two products, add)
    e_lerp = U16 * lerp_ref.abs() + (1 + U16) * (lip * e_src[:, None] + 4 * U * E.abs().amax(0)[None])
    # h1 = bf16(silu(pos w1 + b1)): pre within |w1| e_pos + 2u (|pos w1| + |b1|); silu = pre / (1 + __expf(-pre)) within
    # (2 (2 + 1.173 |pre|) + 2) u relative, silu' <= 1.1
    pre = pos[:, None] * w1.to(F64)[:, 0][None] + b1.to(F64)[None]
    h1 = F.silu(pre)
    e_pre = w1.to(F64)[:, 0].abs()[None] * e_pos[:, None] + 2 * U * ((pos[:, None] * w1.to(F64)[:, 0][None]).abs() + b1.to(F64).abs()[None])
    e_h1 = U16 * h1.abs() + (1 + U16) * (1.1 * e_pre + h1.abs() * (2 * (2 + 1.173 * pre.abs()) + 2) * U)
    # Linear2 on the tensor cores: bf16 w2 (2^-8 relative), h1 within e_h1, an fp32 accumulator allowed a full ulp per addition
    # (gamma(2D)); the epilogue adds bias and residual (2u of the magnitudes)
    aw2 = w2.to(F64).abs()
    e_gemm = (e_h1 @ aw2.t()) * (1 + U16) + (h1.abs() @ aw2.t()) * (U16 + gamma(2 * D))
    lin = h1 @ w2.to(F64).t()
    atol = e_lerp + e_gemm + 2 * U * (lin.abs() + b2.to(F64).abs()[None] + lerp_ref.abs())
    check_b('te', te[m.to(dev())].cpu(), ref[m], atol[m])
    check_zero('te padded rows', te[~m.to(dev())])
    # backward. dz = d_te * mask (exact); d_emb: each row adds (1 - lam) g and lam g; a rounding that moves src across an integer
    # hands its weight to the neighbouring id, so ids i0 - 1 .. i0 + 1 may each see 2 e_src of the row's |g| besides the product
    # roundings; i0 and i1 = i0 + 1 receive the row's terms, whose atomic sum carries gamma(2 B N)
    dz = (d_te.to(F64) * m[:, None])
    ag = dz.abs()
    w_err = 2 * e_src + 2 * U
    ids_rows = [text[b, :lt] for b, (lt, _) in enumerate(LT_LA)]
    aemb = torch.zeros(V, D, dtype=F64)
    for b, (lt, la) in enumerate(LT_LA):
        r = slice(b * N, b * N + la)
        i0 = src[r].floor().clamp(max=lt - 1).long()
        for j in range(-1, 2):
            idx = ids_rows[b][(i0 + j).clamp(0, lt - 1)]
            aemb.index_add_(0, idx, ag[r] * (w_err[r][:, None] + (0 if j < 0 else 1) * gamma(2 * B * N)))
    check_f('d_emb', grads[0], rgrads[0], aemb)
    # d_h1 = bf16(dz W2) (tensor cores, bf16 W2); dpre = d_h1 silu'(pre) with silu' through __expf: sigma within sig_err(pre),
    # silu' = s (1 + pre (1 - s)) within sig_err (1 + 2|pre|) + 4u (1 + |pre|), and pre within e_pre moves it by <= 1/2 e_pre
    dh1 = dz @ w2.to(F64)
    e_dh1 = U16 * dh1.abs() + (1 + U16) * ((ag @ aw2) * (U16 + gamma(2 * D)))
    sp = torch.sigmoid(pre) * (1 + pre * (1 - torch.sigmoid(pre)))
    e_sp = sig_err(pre) * (1 + 2 * pre.abs()) + 4 * U * (1 + pre.abs()) + 0.5 * e_pre
    dpre = dh1 * sp
    e_dpre = 1.1 * e_dh1 + dh1.abs() * e_sp + U * dpre.abs()
    nrow = B * N
    check_f('d_b1', grads[2], rgrads[2], e_dpre.sum(0) + gamma(nrow) * dpre.abs().sum(0))
    check_f('d_w1', grads[1][:, 0], rgrads[1][:, 0],
            (e_dpre * pos[:, None] + dpre.abs() * e_pos[:, None]).sum(0) + gamma(nrow + 1) * (dpre * pos[:, None]).abs().sum(0))
    # Linear2 gradients: dW2 = dz^T h1 with the kernel's bf16 h1; db2 = column sums of dz
    check_f('d_w2', grads[3], rgrads[3], ag.t() @ e_h1 + gamma(2 * nrow) * (ag.t() @ h1.abs()))
    check_f('d_b2', grads[4], rgrads[4], gamma(nrow) * ag.sum(0))


# ---------------------------------------------------------------------------------------------------------------------- final norm
@pytest.mark.parametrize('S', [1, 4])
@pytest.mark.parametrize('R', [0, 32])
@pytest.mark.parametrize('D', [128, 264, 512, 1024, 192, 384, 640, 768, 896])
def test_final_norm(pkg, D, R, S):
    """ops.FinalNorm against O.rmsnorm(xres[:, R:].sum(2), g): all three per-thread widths (D <= 256, <= 512, <= 1024) and
    D = 264, whose 33 chunks leave most lanes of a warp's second pass idle; D = 192, 384, 640, 768, 896 (24, 48, 80, 96, 112 chunks):
    model widths that leave lanes of the last pass of their width idle. Register rows of d_xres are exactly 0.
    x = the fp32 sum of S bf16 streams, within dx = gamma(S - 1) sum|streams|. cn = sqrt(D) / ||x||: the D squares and their sum
    carry gamma(D + 1) of ||x||^2 (half of it for ||x||), sqrtf(D), sqrtf and the division 3u, and dx moves ||x|| by ||dx|| (rc)."""
    g = gen(D * 10 + R + S)
    B, N = 2, 50
    T = B * (R + N)
    xres = bfr(torch.randn(T, S, D, generator=g) * 3)       # scale 3: cn = sqrt(D) / ||x|| is far from 1
    gg = 1 + 0.2 * torch.randn(D, generator=g)
    dy = bfr(torch.randn(B * N, D, generator=g))
    leaves = [xres.to(dev()).requires_grad_(), gg.to(dev()).requires_grad_()]
    y = pkg.ops.FinalNorm.apply(leaves[0], leaves[1], B, N, R)
    d_xres, g_g = torch.autograd.grad(y, leaves, dy.to(dev()))
    X = xres.to(F64).requires_grad_()
    G = gg.to(F64).requires_grad_()
    yr = O.rmsnorm(X.view(B, R + N, S, D)[:, R:].sum(2), G).reshape(B * N, D)
    rx, rgg = torch.autograd.grad(yr, [X, G], dy.to(F64))
    x = xres.to(F64).view(B, R + N, S, D)[:, R:].sum(2).reshape(B * N, D)
    dx = gamma(S - 1) * xres.to(F64).abs().view(B, R + N, S, D)[:, R:].sum(2).reshape(B * N, D)
    nrm = x.norm(dim=-1, keepdim=True)
    cn = D ** 0.5 / nrm
    rc = gamma(D + 1) / 2 + 3 * U + dx.norm(dim=-1, keepdim=True) / nrm
    ag = gg.to(F64).abs()[None]
    ydet = yr.detach()
    check_b(f'y D{D} R{R} S{S}', y.cpu(), ydet, cn * ag * dx + ydet.abs() * (rc + 2 * U))
    # d_x = cn g dy - x k2, k2 = cn^3 / D * sum(g dy x): the dot carries gamma(D + 2) sum|g dy x| and dx, k2 3 rc and 4 roundings,
    # the two products and the subtraction 3u
    d64 = dy.to(F64)
    gdx = gg.to(F64)[None] * d64
    dot = (gdx * x).sum(-1, keepdim=True)
    k2 = cn ** 3 / D * dot
    e_dot = gamma(D + 2) * (gdx * x).abs().sum(-1, keepdim=True) + (gdx.abs() * dx).sum(-1, keepdim=True)
    e_k2 = k2.abs() * (3 * rc + 4 * U) + cn ** 3 / D * e_dot
    t1, t2 = (cn * gdx).abs(), (x * k2).abs()
    atol = t1 * (rc + 2 * U) + x.abs() * e_k2 + dx * k2.abs() + 3 * U * (t1 + t2)
    rxd = rx.view(B, R + N, S, D)
    got = d_xres.view(B, R + N, S, D).cpu()
    for s in range(S):
        check_b(f'd_xres D{D} R{R} S{S} stream {s}', got[:, R:, s].reshape(B * N, D), rxd[:, R:, s].reshape(B * N, D), atol)
    check_zero(f'd_xres register rows D{D} R{R} S{S}', got[:, :R])
    # g_g = sum_rows dy x cn: 2B N rows of products, each with the cn and x errors
    e_g = (d64.abs() * (dx * cn + x.abs() * cn * rc)).sum(0) + gamma(B * N + 2) * (d64 * x * cn).abs().sum(0)
    check_f(f'g_g D{D} R{R} S{S}', g_g, rgg, e_g)


# ---------------------------------------------------------------------------------------------------------------------- flow loss
@pytest.mark.parametrize('dloss', [1.0, 0.37])
@pytest.mark.parametrize('with_vel', [False, True])
def test_flow_loss(pkg, with_vel, dloss):
    """b200_flow_loss_fwd/bwd: masked MSE (e2_tts.py:1580-1582, O.e2tts_forward) with the span in one sample only, optionally the
    velocity-consistency term (weight 0.7); C = 100 with a 104-column dpred whose pad columns must be exactly 0.
    loss: every term is (pr - (x1 - x0))^2 with two roundings in the difference and one square (5u relative); all terms are
    positive, so the sum carries gamma(n) of itself; the division and the weighted add round (2u)."""
    lib, ops = pkg.lib, pkg.ops
    g = gen(int(dloss * 100) + with_vel)
    B, N, C = 3, 77, 100
    ldp = 104
    rows = B * N
    pred, x1, x0 = (torch.randn(rows, C, generator=g) for _ in range(3))
    vt = torch.randn(rows, C, generator=g) if with_vel else None
    span = torch.zeros(B, N, dtype=torch.bool)
    span[1, 10:60] = True
    w32 = float(np.float32(0.7))
    Dv = {k: (v.to(dev()) if v is not None else None) for k, v in dict(pred=pred, x1=x1, x0=x0, vt=vt).items()}
    span_d = span.to(torch.uint8).reshape(-1).to(dev())
    sums = torch.empty(4, device=dev())
    loss = torch.empty((), device=dev())
    parts = torch.empty(2, device=dev())
    pred_data = torch.empty_like(Dv['pred'])
    a = lib.make_args('b200_flow_loss_args', pred=Dv['pred'], x1=Dv['x1'], x0=Dv['x0'], span=span_d, sums=sums, loss=loss, pred_data=pred_data,
                      rows=rows, C=C, vel_target=Dv['vt'], vel_weight=0.7, loss_parts=parts)
    lib.call('b200_flow_loss_fwd', a, ops._stream())
    dl = torch.tensor(dloss, dtype=F32)
    dl_d = dl.to(dev())
    dpred = torch.full((rows, ldp), 7.0, device=dev(), dtype=BF16)
    a = lib.make_args('b200_flow_loss_args', pred=Dv['pred'], x1=Dv['x1'], x0=Dv['x0'], span=span_d, sums=sums, dloss=dl_d, dpred=dpred,
                      ldp=ldp, rows=rows, C=C, vel_target=Dv['vt'], vel_weight=0.7)
    lib.call('b200_flow_loss_bwd', a, ops._stream())
    check_e('pred_data', pred_data, x0 + pred)
    P = pred.to(F64).requires_grad_()
    sm = span.reshape(-1)
    d = P - (x1.to(F64) - x0.to(F64))
    flow = (d ** 2)[sm].mean()
    n = int(sm.sum()) * C
    vel = ((P - vt.to(F64)) ** 2)[sm].mean() if with_vel else torch.zeros((), dtype=F64)
    tot = flow + w32 * vel
    (dP,) = torch.autograd.grad(tot, [P], torch.tensor(float(dl), dtype=F64))
    flow, vel, tot = flow.detach(), vel.detach(), tot.detach()
    e_flow = float(flow) * (gamma(n) + 6 * U)
    e_vel = float(vel) * (gamma(n) + 6 * U)
    check_f('loss_parts', parts, torch.stack([flow, vel]), torch.tensor([e_flow, e_vel], dtype=F64))
    check_f('loss', loss, tot, e_flow + w32 * e_vel + 2 * U * float(tot))
    # dpred = bf16(scale (d + w (pr - vt))), scale = 2 dloss / (count C): d rounds twice, pr - vt once, the weight product and the sum
    # once each, scale once (its operands are exact), the final product once
    dd = d.detach()
    dv_ = (pred.to(F64) - vt.to(F64)) if with_vel else torch.zeros_like(dd)
    v = dd + w32 * dv_
    scale = 2 * float(dl) / n
    atol = abs(scale) * (2 * U * dd.abs() + 3 * U * w32 * dv_.abs() + 3 * U * v.abs())
    check_b('dpred', dpred[:, :C].cpu()[sm], dP[sm], atol[sm])
    check_zero('dpred outside the span', dpred[:, :C][~sm.to(dev())])
    check_zero('dpred pad columns', dpred[:, C:])


# ---------------------------------------------------------------------------------------------------------------------- rowgate
@pytest.mark.parametrize('rpb', [1, 63, 64, 65, 1056])
@pytest.mark.parametrize('D', [8, 264, 512, 1024])
def test_rowgate_bwd(pkg, D, rpb):
    """backward of the GEMM epilogue y = mask * cs[b] * z (AdaLNZero gate, row mask): dz, d_cs (against sum dy z with the exact
    pre-gate z) and the fused bias sum; cs and/or mask absent; 64-row blocks with rows_per_batch around 64; D = 264 leaves row lanes
    idle (256 is not a multiple of 33 chunks). A gate that is exactly 0 gets d_cs = 0 (documented: y = 0 there, y / cs is 0 / 0)."""
    ops = pkg.ops
    if D == 264:
        assert 256 % (D // 8) != 0
    g = gen(D + rpb)
    B = 2
    T = B * rpb
    z = torch.randn(T, D, generator=g)
    cs = torch.rand(B, D, generator=g) * 0.8 + 0.1
    cs[0, 3] = 0.0
    mask = torch.rand(T, generator=g) > 0.2
    mask[0] = True
    dy = bfr(torch.randn(T, D, generator=g))
    bidx = torch.arange(T) // rpb
    for use_cs, use_mask in ((True, True), (True, False), (False, True)):
        mk = mask if use_mask else torch.ones(T, dtype=torch.bool)
        csr = cs[bidx] if use_cs else torch.ones(T, D)
        y = (z * csr * mk[:, None]).to(BF16)                # what the forward GEMM epilogue stored
        for want_bias in (False, True):
            tag = f'D{D} rpb{rpb} cs={use_cs} mask={use_mask} bias={want_bias}'
            out = ops._rowgate_bwd(dy.to(dev()), y.to(dev()), cs.to(dev()) if use_cs else None,
                                   mask.to(torch.uint8).to(dev()) if use_mask else None, B, rpb, D, want_bias)
            dz = out[0]
            g64 = dy.to(F64) * mk[:, None]
            if use_cs:
                check_b(f'dz {tag}', dz.cpu(), g64 * csr.to(F64), U * (g64 * csr.to(F64)).abs())
                # d_cs = (sum dy y) / cs with y = bf16(cs z): every term within (2^-8 + u) |dy z|, the sum gamma(rpb), the division u
                t = (g64 * z.to(F64)).view(B, rpb, D)
                ref = t.sum(1)
                bound = t.abs().sum(1) * (U16 + 2 * U + gamma(rpb + 1) * (1 + U16 + U))
                check_f(f'd_cs {tag}', out[1][cs.to(dev()) != 0], ref[cs != 0], bound[cs != 0])
                check_zero(f'd_cs at a zero gate {tag}', out[1][0, 3:4])
            else:
                check_e(f'dz {tag}', dz.cpu(), torch.where(mk[:, None], dy, torch.zeros_like(dy)))   # masked rows: +0
            if want_bias:
                tb = g64 * (csr.to(F64) if use_cs else 1)
                check_f(f'd_bias {tag}', out[-1], tb.sum(0), gamma(T + 1) * tb.abs().sum(0))


# ---------------------------------------------------------------------------------------------------------------------- colsum
def _colsum_cl(ncols):
    """chunk lanes per block chosen by b200_colsum"""
    nchunk, cl = (ncols + 7) // 8, 32
    while cl > 2 and cl // 2 >= nchunk:
        cl >>= 1
    return cl


COLSUM_COLS = [(8, 8, 2), (16, 16, 2), (32, 32, 4), (64, 64, 8), (100, 104, 16), (264, 264, 32), (512, 512, 32), (4096, 4096, 32)]


@pytest.mark.parametrize('T', [1, 7, 2112, 16899])
@pytest.mark.parametrize('ncols,ld,cl', COLSUM_COLS, ids=[f'{n}-ld{l}-CL{c}' for n, l, c in COLSUM_COLS])
def test_colsum(pkg, ncols, ld, cl, T):
    """ops.colsum against float64 column sums: every chunk-lane instantiation (CL 32/16/8/4/2), the scalar tail (ncols % 8 != 0),
    and a column slice of a wider matrix, as Attention.backward passes. F: gamma(T - 1) sum|X| per column."""
    assert _colsum_cl(ncols) == cl
    g = gen(ncols + T)
    off = 3 * 64 * 2                                   # a slice starting at a 16-byte aligned column, like d_qkvg[:, 3I:]
    full = bfr(torch.randn(T, off + ld, generator=g) * 4)
    Xd = full.to(dev())
    for name, X, pitch in (('contiguous', Xd[:, off:].contiguous(), ld), ('slice', Xd[:, off:], off + ld)):
        got = pkg.ops.colsum(X, T, ncols, pitch)
        ref = full[:, off:off + ncols].to(F64)
        check_f(f'colsum {name} ncols{ncols} T{T}', got, ref.sum(0), gamma(T - 1) * ref.abs().sum(0))


# ---------------------------------------------------------------------------------------------------------------------- GEGLU backward
@pytest.mark.parametrize('T', [1, 257])
@pytest.mark.parametrize('inner', [64, 2048, 320])
def test_geglu_bwd(pkg, inner, T):
    """b200_geglu_bwd (dropout 0) against float64 autograd of u * gelu(g) with the exact erf GELU, on the packed [u(64) | g(64)]
    layout; the packed bias gradient is the column sum of what the kernel wrote (the bf16 values the weight GEMM reads).
    cdf = 0.5 (1 + erff(g c)): erff <= 2 ulp (4u), the argument's two roundings move erf by <= 2u * max(x erf'(x)) < 1u, the add 2u:
    cdf within 3.5u; pdf = 0.39894f __expf(-g^2 / 2) within (2 (2 + 1.173 a) + 2a + 2) u relative, a = g^2 / 2 (the argument's two
    products round: 2u a; the constant and the product round: 2u)."""
    lib, ops = pkg.lib, pkg.ops
    g = gen(inner + T)
    nb = inner // 64
    ug = bfr(torch.randn(T, 2 * inner, generator=g) * 2)
    dh = bfr(torch.randn(T, inner, generator=g))
    perm = torch.arange(2 * inner).view(nb, 2, 64)
    iu, ig = perm[:, 0].reshape(-1), perm[:, 1].reshape(-1)          # packed columns of u and of g for hidden unit h
    for with_db in (False, True):
        dug = torch.empty(T, 2 * inner, device=dev(), dtype=BF16)
        db = torch.zeros(2 * inner, device=dev()) if with_db else None
        lib.call('b200_geglu_bwd', dh.to(dev()), ug.to(dev()), dug, db, T, inner, 0.0, 0, None, ops._stream())
        u = ug[:, iu].to(F64).requires_grad_()
        gg = ug[:, ig].to(F64).requires_grad_()
        du, dg = torch.autograd.grad(u * F.gelu(gg), [u, gg], dh.to(F64))
        ud, gd, d = u.detach(), gg.detach(), dh.to(F64)
        cdf = 0.5 * (1 + torch.erf(gd / math.sqrt(2)))
        pdf = torch.exp(-0.5 * gd ** 2) / math.sqrt(2 * math.pi)
        e_cdf = 3.5 * U
        a = 0.5 * gd ** 2
        e_pdf = pdf * (2 * (2 + 1.173 * a) + 2 * a + 2) * U
        got = dug.cpu()
        check_b(f'du inner{inner} T{T}', got[:, iu], du, (d * gd).abs() * e_cdf + 2 * U * du.abs())
        inner_t = cdf + gd * pdf
        atol = (d * ud).abs() * (e_cdf + gd.abs() * (e_pdf + U * pdf) + U * inner_t.abs()) + 2 * U * dg.abs()
        check_b(f'dg inner{inner} T{T}', got[:, ig], dg, atol)
        if with_db:
            ref = got.to(F64).sum(0)
            check_f(f'db inner{inner} T{T}', db, ref, gamma(T - 1) * got.to(F64).abs().sum(0))


# ---------------------------------------------------------------------------------------------------------------------- stem
@pytest.mark.parametrize('concat', [False, True])
def test_stem_prepare(pkg, concat):
    """ops.stem_prepare in training mode (t = 0, 1 and random) and direct mode, C = 100 padded to Cp = 128: the cond half, cond_out,
    the direct copies and the pad columns are exact; the lerp (1 - t) x0 + t x1 may be contracted into an FMA, so it is compared with
    the unfused fp32 torch expression within one bf16 step (plus the fp32 discrepancy of the two evaluations, which matters only where
    the lerp cancels), and with float64 as a B bound (1 - t, two products, one add: 3u)."""
    ops = pkg.ops
    g = gen(3 + concat)
    B, N, C, Cp = 3, 50, 100, 128
    x1, x0 = torch.randn(B, N, C, generator=g), torch.randn(B, N, C, generator=g)
    times = torch.cat([torch.tensor([0.0, 1.0]), torch.rand(1, generator=g)])
    span = torch.rand(B, N, generator=g) > 0.5
    A, cond = ops.stem_prepare(B, N, C, Cp, x1=x1.to(dev()), x0=x0.to(dev()), times=times.to(dev()),
                               span=span.to(torch.uint8).to(dev()), want_cond=True, concat=concat)
    A = A.cpu().view(B, N, 2 * Cp)
    t = times[:, None, None]
    cond_ref = torch.where(span[..., None], torch.zeros_like(x1), x1)
    check_e('cond_out', cond.cpu(), cond_ref)
    w_cols, c_cols = (slice(C, 2 * C), slice(0, C)) if concat else (slice(0, C), slice(Cp, Cp + C))
    pads = [slice(2 * C, 2 * Cp)] if concat else [slice(C, Cp), slice(Cp + C, 2 * Cp)]
    check_e('cond half', A[..., c_cols], cond_ref.to(BF16))
    for p in pads:
        check_zero('pad columns', A[..., p])
    lerp32 = ((1 - t) * x0 + t * x1).to(BF16)
    got = A[..., w_cols]
    t64 = times.to(F64)[:, None, None]
    mag = (1 - t64) * x0.to(F64).abs() + t64 * x1.to(F64).abs()
    # fused or not, each fp32 evaluation is within 3u mag of the exact lerp, so the two differ by <= 6u mag; rounding to bf16 is
    # monotonic, which adds at most one bf16 step (where the lerp cancels, 6u mag can exceed that step)
    diff = (got.to(F64) - lerp32.to(F64)).abs()
    lim = bf16_ulp(torch.maximum(got.to(F64).abs(), lerp32.to(F64).abs())) + 6 * U * mag
    assert bool((diff <= lim).all()), f'lerp: {int((diff > lim).sum())} elements differ from the fp32 expression by more than one bf16 step'
    ref = (1 - t64) * x0.to(F64) + t64 * x1.to(F64)
    check_b('lerp', got, ref, 3 * U * mag)
    check_e('lerp at t = 0', got[0], x0[0].to(BF16))
    check_e('lerp at t = 1', got[1], x1[1].to(BF16))
    # direct mode (sampling): both halves are copies
    xin, cin = torch.randn(B, N, C, generator=g), torch.randn(B, N, C, generator=g)
    A, _ = ops.stem_prepare(B, N, C, Cp, x_in=xin.to(dev()), cond_in=cin.to(dev()), concat=concat)
    A = A.cpu().view(B, N, 2 * Cp)
    check_e('direct x', A[..., w_cols], xin.to(BF16))
    check_e('direct cond', A[..., c_cols], cin.to(BF16))
    for p in pads:
        check_zero('direct pad columns', A[..., p])


# ---------------------------------------------------------------------------------------------------------------------- masked mean
@pytest.mark.parametrize('D', [100, 512])
def test_masked_mean(pkg, D):
    """ops.MaskedMean (maybe_masked_mean, the formula of O.duration_forward: sum / den.clamp(min=1)) with rows that are all valid,
    have one valid token, have none (output and gradient exactly 0) and a random mask; and without a mask.
    fwd: gamma(N - 1) sum|x| / den plus the division's u; bwd: one division (u) then bf16."""
    ops = pkg.ops
    g = gen(D)
    B, N = 4, 1024
    x = bfr(torch.randn(B * N, D, generator=g))
    mask = torch.zeros(B, N, dtype=torch.bool)
    mask[0] = True
    mask[1, 517] = True
    mask[3] = torch.rand(N, generator=g) > 0.5
    dout = torch.randn(B, D, generator=g)
    for use_mask in (True, False):
        m = mask if use_mask else torch.ones(B, N, dtype=torch.bool)
        xl = x.to(dev()).requires_grad_()
        out = ops.MaskedMean.apply(xl, mask.to(torch.uint8).to(dev()) if use_mask else None, B, N)
        (dx,) = torch.autograd.grad(out, [xl], dout.to(dev()))
        X = x.to(F64).view(B, N, D).requires_grad_()
        den = m.to(F64).sum(1).clamp(min=1)
        ref = (X * m[..., None]).sum(1) / den[:, None]
        (rdx,) = torch.autograd.grad(ref, [X], dout.to(F64))
        ax = (x.to(F64).view(B, N, D).abs() * m[..., None]).sum(1)
        check_f(f'masked mean mask={use_mask}', out, ref.detach(), gamma(N - 1) * ax / den[:, None] + U * ref.detach().abs())
        check_b(f'masked mean dx mask={use_mask}', dx.cpu(), rdx.reshape(B * N, D), U * rdx.reshape(B * N, D).abs())
        if use_mask:
            check_zero('masked mean with no valid token', out[2])
            check_zero('masked mean dx with no valid token', dx.view(B, N, D)[2])


# ---------------------------------------------------------------------------------------------------------------------- cast / pack
def test_cast_rows(pkg):
    """ops.cast_rows: round to nearest even, ties, subnormals, overflow to inf, signed zeros; pad columns exactly 0."""
    g = gen(1)
    rows, cols, ld = 37, 100, 104
    src = torch.randn(rows, cols, generator=g) * torch.logspace(-40, 38, rows)[:, None].float()
    special = torch.tensor([0x3F808000, 0x3F818000, 0xBF808000, 0x3F80FFFF, 0x00000001, 0x00008000, 0x00018000, 0x807FFFFF,
                            0x00800000, 0x7F7FFFFF, 0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x3F7FFFFF, 0x33800000],
                           dtype=torch.int64).to(torch.int32)
    src[0, :special.numel()] = special.view(F32)
    out = pkg.ops.cast_rows(src.to(dev()), rows, cols, ld)
    check_e('cast', out[:, :cols], src.to(BF16))
    check_zero('cast pad columns', out[:, cols:])


def test_weight_pack(pkg):
    """modules.WeightPack / b200_pack_weights: mode 0 with row and column offsets, mode 1 (GEGLU interleave) for a weight and a 1-D
    bias, fp32 output, the scalar path (cols % 4 != 0: 1-D biases, 3-D conv weights, odd column offsets). The destinations are filled
    with a sentinel first: every byte outside the described slots must be untouched."""
    mods = pkg.modules
    g = gen(2)
    inner, d = 128, 48
    w_geglu = torch.randn(2 * inner, d, generator=g)
    b_geglu = torch.randn(2 * inner, generator=g)
    w_plain = torch.randn(40, 64, generator=g)
    w_conv = torch.randn(24, 1, 31, generator=g)
    w_odd = torch.randn(10, 5, generator=g)
    dst_bf = torch.full((300, 200), -12345.0, dtype=BF16)
    dst_f32 = torch.full((600,), 1e30)
    dst_conv = torch.full((30, 40), 3.0, dtype=BF16)
    D = {k: v.to(dev()) for k, v in dict(w_geglu=w_geglu, b_geglu=b_geglu, w_plain=w_plain, w_conv=w_conv, w_odd=w_odd,
                                         dst_bf=dst_bf, dst_f32=dst_f32, dst_conv=dst_conv).items()}
    tab = mods.WeightPack(dev())
    tab.add(D['w_plain'], D['dst_bf'], row_off=7, col_off=64)
    tab.add(D['w_geglu'], D['dst_bf'], row_off=44, col_off=132, mode=1)
    tab.add(D['w_odd'], D['dst_bf'], row_off=290, col_off=3)
    tab.add(D['b_geglu'], D['dst_f32'], row_off=300, mode=1)
    tab.add(D['w_conv'], D['dst_conv'], row_off=2, col_off=5)
    tab.run()
    inter = lambda t: t.reshape(2, inner // 64, 64, *t.shape[1:]).transpose(0, 1).reshape(t.shape)
    want_bf = dst_bf.clone()
    want_bf[7:47, 64:128] = w_plain.to(BF16)
    want_bf[44:44 + 2 * inner, 132:132 + d] = inter(w_geglu).to(BF16)
    want_bf[290:300, 3:8] = w_odd.to(BF16)
    want_f32 = dst_f32.clone()
    want_f32[300:300 + 2 * inner] = inter(b_geglu)
    want_conv = dst_conv.clone()
    want_conv[2:26, 5:36] = w_conv.reshape(24, 31).to(BF16)
    check_e('pack bf16', D['dst_bf'], want_bf)
    check_e('pack fp32 bias', D['dst_f32'], want_f32)
    check_e('pack conv', D['dst_conv'], want_conv)


# ---------------------------------------------------------------------------------------------------------------------- fourier features
@pytest.mark.parametrize('df,dr', [(64, 0), (48, 32), (8, 120)])
def test_fourier_feat(pkg, df, dr):
    """b200_fourier_feat_fwd/bwd (LinearFourierEmbed tail, O.linear_fourier_embed): cat(sin z, cos z, rest) with |z| up to 100 and a
    row pitch ldz > df + dr (pad columns of dz exactly 0). sinf/cosf/sincosf are within 2 ulp (4u relative) at any argument;
    dz = g_s cos - g_c sin adds two products and a subtraction (2u)."""
    lib, ops = pkg.lib, pkg.ops
    g = gen(df + dr)
    T = 300
    ldz = (df + dr + 7) // 8 * 8 + 8
    z = bfr((torch.rand(T, ldz, generator=g) * 2 - 1) * 100)
    out = torch.empty(T, 2 * df + dr, device=dev(), dtype=BF16)
    zd = z.to(dev())
    lib.call('b200_fourier_feat_fwd', zd, ldz, out, T, df, dr, ops._stream())
    d_out = bfr(torch.randn(T, 2 * df + dr, generator=g))
    dz = torch.full((T, ldz), 7.0, device=dev(), dtype=BF16)
    lib.call('b200_fourier_feat_bwd', d_out.to(dev()), zd, ldz, dz, T, df, dr, ops._stream())
    Z = z[:, :df + dr].to(F64).requires_grad_()
    f, rest = Z[:, :df], Z[:, df:]
    ref = torch.cat((f.sin(), f.cos(), rest), -1)
    (rdz,) = torch.autograd.grad(ref, [Z], d_out.to(F64))
    ref = ref.detach()
    got = out.cpu()
    check_b('fourier sin/cos', got[:, :2 * df], ref[:, :2 * df], 4 * U * ref[:, :2 * df].abs())
    check_e('fourier rest', got[:, 2 * df:], z[:, df:df + dr])
    fd = f.detach()
    gs, gc = d_out[:, :df].to(F64), d_out[:, df:2 * df].to(F64)
    atol = 6 * U * ((gs * fd.cos()).abs() + (gc * fd.sin()).abs())
    dzc = dz.cpu()
    check_b('fourier dz', dzc[:, :df], rdz[:, :df], atol)
    check_e('fourier dz rest', dzc[:, df:df + dr], d_out[:, 2 * df:])
    check_zero('fourier dz pad columns', dzc[:, df + dr:])


# ---------------------------------------------------------------------------------------------------------------------- ODE / CFG
@pytest.mark.parametrize('per', [1000, 5000])
def test_axpy_and_cfg_combine(pkg, per):
    """ops.axpy (y + a f: one product, one add, 2u of the magnitudes) and ops.cfg_combine against e2_tts.py:1323-1330 with O.project
    in float64: remove_parallel on/off, keep_parallel_frac 0 and 0.3, a sample with pred == null_pred, a sample with pred == 0 (the
    norm clamp), per-sample sizes below and above one 2048-element block.
    cfg: the projection coefficient is formed in float64 (relative error <= 2 per 2^-53); parallel and orthogonal parts are rounded to
    fp32 (u each), orth + par * keep adds two fp32 roundings, the final pred + update * strength is formed in double and rounded once."""
    ops = pkg.ops
    g = gen(per)
    B = 4
    assert (per > 2048) == (per == 5000)
    pred = torch.randn(B, per, generator=g)
    null = torch.randn(B, per, generator=g)
    null[1] = pred[1]
    pred[2] = 0.0
    y, f = torch.randn(B * per, generator=g), torch.randn(B * per, generator=g)
    a = -0.3
    out = ops.axpy(y.to(dev()), f.to(dev()), a)
    a32 = float(np.float32(a))
    ref = y.to(F64) + a32 * f.to(F64)
    check_f('axpy', out, ref, 2 * U * ((a32 * f.to(F64)).abs() + y.to(F64).abs()))
    strength = 2.0
    for remove_parallel in (False, True):
        for keep in (0.0, 0.3):
            k32 = float(np.float32(keep))
            got = ops.cfg_combine(pred.to(dev()), null.to(dev()), strength, remove_parallel, keep)
            P, Q = pred.to(F64), null.to(F64)
            upd = P - Q
            tag = f'per{per} remove_parallel={remove_parallel} keep={keep}'
            if remove_parallel:
                par, orth = O.project(upd, P)
                ref = P + (orth + par * k32) * strength
                e64 = 4 * per * 2.0 ** -53 * (1 + k32) * par.abs()
                bound = strength * (U * orth.abs() + U * k32 * par.abs() + 2 * U * (orth.abs() + k32 * par.abs()) + e64) + U * ref.abs()
            else:
                ref = P + upd * strength
                bound = U * ref.abs()
            check_f(f'cfg {tag}', got, ref, bound)
            check_e(f'cfg pred == null {tag}', got[1].cpu(), pred[1])
            check_f(f'cfg pred == 0 {tag}', got[2], -Q[2] * strength, U * (Q[2] * strength).abs())
