"""GPU: Transformer(num_residual_streams=1), the plain residual backbone (e2_tts.py:547, :607 with disable=True).

Kernels, element-wise against float64 with NaN-filled outputs (the method of kernel_checks.py, the depthwise reference of hyper_conv_ref.py):
  * the branch-norm mode of b200_final_norm_* (RMSNorm(g) and per-batch AdaptiveRMSNorm gains, the residual gradient d_res, zero rows);
  * the residual mode of b200_dwconv_* (y = x + the masked conv, dx = dy + the conv's dx).
Bit-exact properties: masked rows of the residual convolution keep x (and pass dy); its pre-activation equals the plain launch's;
the branch norm's forward equals the final norm's with one stream and no registers.
Nodes at the config-2 widths (ops.BranchNorm, ops.DwConv / OutProj / FeedForward with a residual): the residual's gradient is dy
itself. Model: the cfg2-shape E2TTS against the fp32 oracle with one stream, DurationPredictor, 32-step sample(), a
graphed training step, and no hyper-connection entry point launched."""
import pytest
import torch

from conftest import rel_l2
from hyper_conv_ref import CV_TN, cdiv, dw_mask, dw_ref, model_mask
from kernel_checks import BF16, F64, U, U16, check_b, check_e, check_f, dev, gamma, gen, h64, nans, pkg, stream
from model_checks import duration_vs_oracle, graphed_matches_eager, sample_vs_oracle, small_model, step_inputs, whole_model

pytestmark = pytest.mark.gpu


# ================================================================================================================ branch norm
def bn_launch(pkg, x, B, Np, rpb, g=None, gains=None, dy=None, d_res=None, g0=None):
    """one forward and (with dy) one backward launch of the branch-norm mode into NaN-filled outputs; gradient accumulators start at g0"""
    T, D = x.shape
    y = nans((T, D), BF16)
    pkg.lib.call('b200_final_norm_fwd', pkg.lib.make_args('b200_final_norm_args', xres=x, g=g, gains=gains, y=y, B=B, N=Np, R=0, D=D, S=1,
                                                        rows_per_batch=rpb), stream())
    if dy is None:
        return y
    dx = nans((T, D), BF16)
    acc = g0.clone()
    pkg.lib.call('b200_final_norm_bwd', pkg.lib.make_args(
        'b200_final_norm_args', xres=x, g=g, gains=gains, dy=dy, d_xres=dx, g_g=None if gains is not None else acc,
        d_gains=acc if gains is not None else None, d_res=d_res, B=B, N=Np, R=0, D=D, S=1, rows_per_batch=rpb), stream())
    return y, dx, acc


def bn_check(name, x, gain_rows, dy, d_res, y, dx, acc, acc0, rpb):
    """x, dy, d_res: the bf16 values the kernel read ([T, D]); gain_rows: fp32 gain of every row [T, D]; acc: the gain gradient
    ([D] for g, [T / rpb, D] for gains) added onto acc0.
    y = x cn gain, cn = sqrt(D) / max(|x|, 1e-12): the squares and their sum carry gamma(D + 1) of |x|^2 (half of that for |x|),
    sqrtf(D), sqrtf and the division 3u (rc); the two products 2u.
    dx = cn (gain dy - x k) + d_res with k = <gain dy, x> / |x|^2 (0 where the clamp holds): the gain dy products 1u, the dot
    gamma(D + 2) sum|gain dy x|, |x|^2 gamma(D + 1) and the division 1u; x k, the subtraction, the product with cn and the add of
    d_res one rounding each; cn carries rc.
    gain gradient = sum_rows dy x cn, each term within (rc + 2u), summed over at most T + 1 terms in any order."""
    x64, gr, dy64 = h64(x), gain_rows.to(F64), h64(dy)
    T, D = x64.shape
    ss = (x64 * x64).sum(-1, keepdim=True)
    nrm = ss.sqrt()
    live = nrm > 1e-12
    cn = D ** 0.5 / nrm.clamp(min=1e-12)
    rc = gamma(D + 1) / 2 + 3 * U
    yr = x64 * cn * gr
    check_b(f'{name} y', y.cpu(), yr, yr.abs() * (rc + 2 * U))
    gdy = gr * dy64
    dot = (gdy * x64).sum(-1, keepdim=True)
    k = torch.where(live, dot / ss.clamp(min=1e-300), torch.zeros((), dtype=F64))
    e_k = torch.where(live, k.abs() * (gamma(D + 1) + U) + gamma(D + 2) * (gdy * x64).abs().sum(-1, keepdim=True) / ss.clamp(min=1e-300),
                      torch.zeros((), dtype=F64))
    inner = gdy - x64 * k
    e_inner = 3 * U * (gdy.abs() + (x64 * k).abs()) + x64.abs() * e_k
    dr = h64(d_res) if d_res is not None else torch.zeros_like(x64)
    dxr = cn * inner + dr
    check_b(f'{name} dx', dx.cpu(), dxr, cn * e_inner + (cn * inner).abs() * (rc + 2 * U) + U * dxr.abs())
    term = dy64 * x64 * cn
    if acc.dim() == 1:
        want, e = term.sum(0), (term.abs() * (rc + 2 * U)).sum(0) + gamma(T + 1) * (term.abs().sum(0) + acc0.abs().to(F64).cpu())
    else:
        tb = term.view(-1, rpb, D)
        want, e = tb.sum(1), (tb.abs() * (rc + 2 * U)).sum(1) + gamma(rpb + 1) * (tb.abs().sum(1) + acc0.abs().to(F64).cpu())
    check_f(f'{name} gain grad', acc, want + acc0.to(F64).cpu(), e)
    return yr, dxr


# D, batches, rows per batch: every per-thread width, a batch that is not a multiple of the block's rows, a batch of one block
# row, and a cfg2 row count (T = 2 x 1056)
# D = 192, 384, 640, 768, 896: model widths off the powers of two, whose last 16-byte-chunk pass leaves lanes of the warp idle
BN_CASES = [(128, 3, 37), (256, 2, 1056), (512, 4, 150), (1024, 3, 77), (512, 1, 8), (264, 2, 45),
            (192, 2, 99), (384, 3, 50), (640, 2, 45), (768, 2, 1056), (896, 1, 77)]


@pytest.mark.parametrize('gain_mode', ['g', 'gains'])
@pytest.mark.parametrize('D,B,Np', BN_CASES)
def test_branch_norm_kernels(pkg, D, B, Np, gain_mode):
    """rows of x: scale 3 (cn far from 1), one all-zero row per batch element (F.normalize's clamp: y = 0, finite dx = cn gain dy)"""
    g = gen(D * 7 + B * 3 + Np + (gain_mode == 'gains'))
    T = B * Np
    x = (torch.randn(T, D, generator=g) * 3).to(BF16)
    for b in range(B):
        x[b * Np + (b * 5) % Np] = 0
    dy = torch.randn(T, D, generator=g).to(BF16)
    d_res = torch.randn(T, D, generator=g).to(BF16)
    if gain_mode == 'g':
        gg = 1 + 0.2 * torch.randn(D, generator=g)
        kw, rows, acc0 = dict(g=gg.to(dev())), gg[None].expand(T, D), torch.randn(D, generator=g)
    else:
        gains = 1 + 0.3 * torch.randn(B, D, generator=g)
        kw, rows, acc0 = dict(gains=gains.to(dev())), gains.repeat_interleave(Np, 0), torch.randn(B, D, generator=g)
    y, dx, acc = bn_launch(pkg, x.to(dev()), B, Np, Np, dy=dy.to(dev()), d_res=d_res.to(dev()), g0=acc0.to(dev()), **kw)
    torch.cuda.synchronize()
    for nm, t in (('y', y), ('dx', dx), ('gain grad', acc)):
        assert bool(torch.isfinite(t).all()), f'{nm}: non-finite elements'
    bn_check(f'D{D} B{B} Np{Np} {gain_mode}', x, rows, dy, d_res, y, dx, acc, acc0, Np)
    zero = (x.view(torch.int16) == 0).all(-1)
    assert int(zero.sum()) == B
    assert bool((y.cpu()[zero].float() == 0).all()), 'y of zero rows'   # +-0: the sign of the gain, as in F.normalize(0) * gain
    # without d_res, dx is the norm's gradient alone
    _, dx0, _ = bn_launch(pkg, x.to(dev()), B, Np, Np, dy=dy.to(dev()), g0=acc0.to(dev()), **kw)
    bn_check(f'D{D} B{B} Np{Np} {gain_mode} no d_res', x, rows, dy, None, y, dx0, acc, acc0, Np)


def test_branch_norm_reference_matches_autograd():
    """bn_check's formulas against float64 autograd of the oracle's AdaptiveRMSNorm (F.normalize * sqrt(D) * gain), zero row included"""
    g = gen(5)
    x = torch.randn(6, 64, generator=g, dtype=F64)
    x[2] = 0
    gain = torch.randn(6, 64, generator=g, dtype=F64)
    dy, dr = torch.randn(6, 64, generator=g, dtype=F64), torch.randn(6, 64, generator=g, dtype=F64)
    xr = x.clone().requires_grad_()
    yr = F_norm(xr) * 8.0 * gain
    gx, = torch.autograd.grad(yr, [xr], dy)
    ss = (x * x).sum(-1, keepdim=True)
    cn = 8.0 / ss.sqrt().clamp(min=1e-12)
    k = torch.where(ss.sqrt() > 1e-12, (gain * dy * x).sum(-1, keepdim=True) / ss.clamp(min=1e-300), torch.zeros((), dtype=F64))
    check_f('dx', cn * (gain * dy - x * k) + dr, gx + dr, 1e-9 * (1 + gx.abs()))


def F_norm(x):
    return torch.nn.functional.normalize(x, dim=-1)


def test_branch_norm_forward_equals_final_norm(pkg):
    """g mode: the same per-row arithmetic as the final norm with one stream and no registers, bit for bit"""
    g = gen(9)
    B, Np, D = 2, 1056, 512
    x = (torch.randn(B * Np, D, generator=g) * 2).to(BF16).to(dev())
    gg = (1 + 0.2 * torch.randn(D, generator=g)).to(dev())
    y = bn_launch(pkg, x, B, Np, Np, g=gg)
    yf = nans((B * Np, D), BF16)
    pkg.lib.call('b200_final_norm_fwd', pkg.lib.make_args('b200_final_norm_args', xres=x, g=gg, y=yf, B=B, N=Np, R=0, D=D, S=1), stream())
    check_e('branch norm y vs final norm y', y, yf)


# ================================================================================================================ residual conv
def rc_launch(pkg, x, mask, w, b, dy, residual, dw0, db0):
    B, Np, D = x.shape
    y, pre = nans((B, Np, D), BF16), nans((B, Np, D), BF16)
    pkg.lib.call('b200_dwconv_fwd', pkg.lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w, bias=b, y=y, B=B, Np=Np, D=D,
                                                      ksize=w.shape[1], pre=pre, residual=residual), stream())
    dx, dw, db = nans((B, Np, D), BF16), dw0.clone(), db0.clone()
    pkg.lib.call('b200_dwconv_bwd', pkg.lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w, bias=b, dy=dy, dx=dx, dweight=dw,
                                                      dbias=db, B=B, Np=Np, D=D, ksize=w.shape[1], pre=pre, residual=residual), stream())
    return y, pre, dx, dw, db


# name, B, Np, D, per-row masks ('model': registers + ragged audio), channel subset
RC_CASES = [
    ('suffix-holes', 3, 200, 136, ['holes', 150, 'none'], False),
    ('tile-edges', 3, 130, 72, [63, 64, 'all'], False),
    ('cfg2-audio', 16, 1056, 512, 'model', True),
    ('cfg2-text', 16, 1056, 256, 'model', True),
]


@pytest.mark.parametrize('name,B,Np,D,masks,subset', RC_CASES, ids=[c[0] for c in RC_CASES])
def test_residual_dwconv_kernels(pkg, name, B, Np, D, masks, subset):
    """y = x + m silu(conv(m x) + b): the plain kernel's fp32 value (dw_ref's e_y) plus x, one fp32 add, then bf16;
    dx = dy + the conv's dx (dw_ref's e_dx), one fp32 add, then bf16. Masked rows: y = x and dx = dy bit for bit. The
    pre-activation equals the plain launch's bit for bit; the weight / bias gradients are held to dw_ref's bounds."""
    ks = 31
    seed = sum(map(ord, name))
    g = gen(seed)
    if masks == 'model':
        masks = model_mask(B, Np, gen(seed + 1))
    m = torch.stack([dw_mask(Np, s, g) for s in masks])
    x = torch.randn(B, Np, D, generator=g).to(BF16)
    w = torch.randn(D, ks, generator=g) / ks ** 0.5 + 0.1 * torch.arange(ks) / ks
    b = torch.randn(D, generator=g) * 0.5
    dy = torch.randn(B, Np, D, generator=g).to(BF16)
    dw0, db0 = torch.randn(D, ks, generator=g), torch.randn(D, generator=g)
    md = m.to(torch.uint8).to(dev())
    args = (x.to(dev()), md, w.to(dev()), b.to(dev()), dy.to(dev()))
    y, pre, dx, dw, db = rc_launch(pkg, *args, 1, dw0.to(dev()), db0.to(dev()))
    y0, pre0, dx0, dw_0, db_0 = rc_launch(pkg, *args, 0, dw0.to(dev()), db0.to(dev()))
    torch.cuda.synchronize()
    for nm, t in (('y', y), ('pre', pre), ('dx', dx), ('dweight', dw), ('dbias', db)):
        assert bool(torch.isfinite(t).all()), f'{name} {nm}: non-finite elements'
    check_e(f'{name} pre', pre, pre0)
    bad = ~m
    check_e(f'{name} masked y == x', y.cpu()[bad], x[bad])
    check_e(f'{name} masked dx == dy', dx.cpu()[bad], dy[bad])
    c = torch.arange(D)
    if subset:
        c = torch.cat([torch.arange(0, 64), torch.arange(D // 2, D // 2 + 64), torch.arange(D - 64, D)]).unique()
    r = dw_ref(h64(x[..., c]), m, h64(w[c]), h64(b[c]), h64(dy[..., c]), h64(pre[..., c]))
    mm = m[..., None].expand(B, Np, len(c))
    xs, dys = h64(x[..., c]), h64(dy[..., c])
    yr, dxr = xs + r['y'], dys + r['dx'] * m[..., None]
    check_b(f'{name} y', y.cpu()[..., c][mm], yr[mm], (r['e_y'] + U * (yr.abs() + r['e_y']))[mm])
    check_b(f'{name} dx', dx.cpu()[..., c][mm], dxr[mm], (r['e_dx'] + U * (dxr.abs() + r['e_dx']))[mm])
    # the weight / bias gradients are the plain launch's (fp32 atomics: same terms, any order), as in check_dwconv
    n = B * cdiv(Np, CV_TN) * CV_TN + 1
    check_f(f'{name} dweight', dw.cpu()[c], h64(dw0[c]) + r['dW'], gamma(n) * (r['dWabs'] + h64(dw0[c]).abs()) + r['dWcar'])
    check_f(f'{name} dbias', db.cpu()[c], h64(db0[c]) + r['db'], gamma(n) * (r['dbabs'] + h64(db0[c]).abs()) + r['dbcar'])


# ================================================================================================================ nodes
def cfg2_widths():
    import bench
    c = bench.CONFIGS[2]
    return c['dim'], c['heads']


def test_nodes_with_residual(pkg):
    """at the cfg2 widths (d512 audio, 256 text), B = 2, Np = 1056, with a mask: BranchNorm hands x on as its second output and the
    gradient arriving there joins d x; DwConv(residual) is the kernel; OutProj / FeedForward with resid: y - resid is the resid-less
    node's output up to the rounding of the sum, the resid gradient IS dy, and with no gate every other gradient equals the
    resid-less node's bit for bit; with the AdaLNZero gate, d_cs stays within the rounding of y."""
    d, H = cfg2_widths()
    B, Np, I = 2, 1056, H * 64
    T = B * Np
    g = gen(17)
    mask = torch.ones(B, Np, dtype=torch.bool)
    mask[1, 800:] = False
    md = mask.to(torch.uint8).to(dev())
    # BranchNorm: both outputs used
    for D in (d, d // 2):
        x = (torch.randn(T, D, generator=g) * 2).to(BF16).to(dev()).requires_grad_()
        gains = (1 + 0.2 * torch.randn(B, D, generator=g)).to(dev()).requires_grad_()
        xn, xr = pkg.ops.BranchNorm.apply(x, None, gains, B, Np)
        assert xr.data_ptr() == x.data_ptr()
        dy1, dy2 = torch.randn(T, D, device=dev()).to(BF16), torch.randn(T, D, device=dev()).to(BF16)
        gx, gg = torch.autograd.grad([xn, xr], [x, gains], [dy1, dy2])
        _, dxk, acck = bn_launch(pkg, x.detach(), B, Np, Np, gains=gains.detach(), dy=dy1, d_res=dy2, g0=torch.zeros(B, D, device=dev()))
        check_e(f'BranchNorm dx D{D}', gx, dxk)
        assert rel_l2(gg.cpu(), acck.cpu()) < 1e-5, f'BranchNorm d_gains D{D}'   # atomics: the order of the sums varies
    # OutProj with and without the gate
    og = (torch.randn(T, I, generator=g) * 0.5).to(BF16).to(dev())
    w = (torch.randn(d, I, generator=g) / I ** 0.5).to(dev())
    wpack = w.to(BF16)
    resid = torch.randn(T, d, generator=g).to(BF16).to(dev())
    dy = torch.randn(T, d, generator=g).to(BF16).to(dev())
    for gated in (False, True):
        cs = torch.sigmoid(torch.randn(B, d, generator=g) - 2).to(dev()).requires_grad_() if gated else None
        leaves = [og.clone().requires_grad_(), w.clone().requires_grad_(), resid.clone().requires_grad_()]
        y = pkg.ops.OutProj.apply(leaves[0], leaves[1], wpack, cs, md, B, Np, leaves[2])
        grads = torch.autograd.grad(y, leaves + ([cs] if gated else []), dy)
        l0 = [og.clone().requires_grad_(), w.clone().requires_grad_()]
        y0 = pkg.ops.OutProj.apply(l0[0], l0[1], wpack, cs, md, B, Np)
        g0 = torch.autograd.grad(y0, l0 + ([cs] if gated else []), dy)
        check_e(f'OutProj gated={gated} d_resid == dy', grads[2], dy)
        bound = U16 * (h64(y).abs() + h64(y0).abs()) + 1e-30
        check_f(f'OutProj gated={gated} y - resid', h64(y) - h64(resid), h64(y0), bound)
        check_e(f'OutProj gated={gated} masked rows == resid', y[~mask.flatten().to(dev())], resid[~mask.flatten().to(dev())])
        if not gated:
            check_e('OutProj d_og', grads[0], g0[0])
            assert rel_l2(grads[1].cpu(), g0[1].cpu()) < 1e-5, 'OutProj dW'   # split-K atomics: the order of the sums varies
        else:
            # d_cs[b] = sum_rows dy (y - resid) / cs against sum_rows dy y0 / cs: each (y - resid) within 2^-8 (|y| + |y0|) of y0, and
            # both fp32 sums within gamma(Np + 1) of their terms
            ady, ay, ay0, ar = h64(dy).abs(), h64(y).abs(), h64(y0).abs(), h64(resid).abs()
            per_b = lambda t: t.view(B, Np, d).sum(1)
            e = (U16 * per_b(ady * (ay + ay0)) + 2 * gamma(Np + 1) * per_b(ady * (ay + ay0 + ar))) / h64(cs.detach())
            check_f('OutProj d_cs', grads[3], h64(g0[2]), e)
    # FeedForward with resid (text width: no gate, the text stream's call)
    Dt, inner = d // 2, 2 * d
    xn = torch.randn(T, Dt, generator=g).to(BF16).to(dev())
    w1, b1 = (torch.randn(2 * inner, Dt, generator=g) / Dt ** 0.5).to(dev()), (0.1 * torch.randn(2 * inner, generator=g)).to(dev())
    w2, b2 = (torch.randn(Dt, inner, generator=g) / inner ** 0.5).to(dev()), (0.1 * torch.randn(Dt, generator=g)).to(dev())
    nb = inner // 64
    w1p = w1.view(2, nb, 64, Dt).transpose(0, 1).reshape(2 * inner, Dt).to(BF16).contiguous()
    b1p = b1.view(2, nb, 64).transpose(0, 1).reshape(2 * inner).contiguous()
    w2p = w2.to(BF16)
    resid_t = torch.randn(T, Dt, generator=g).to(BF16).to(dev())
    dyt = torch.randn(T, Dt, generator=g).to(BF16).to(dev())
    outs = []
    for r in (resid_t, None):
        leaves = [xn.clone().requires_grad_(), w1.clone().requires_grad_(), b1.clone().requires_grad_(), w2.clone().requires_grad_(),
                  b2.clone().requires_grad_()] + ([r.clone().requires_grad_()] if r is not None else [])
        y = pkg.ops.FeedForward.apply(*leaves[:5], w1p, b1p, w2p, None, B, Np, 0.0, 0, None, *leaves[5:])
        outs.append((y, torch.autograd.grad(y, leaves, dyt)))
    (y, gr), (y0, g0) = outs
    check_e('FeedForward d_resid == dy', gr[5], dyt)
    check_e('FeedForward dx', gr[0], g0[0])
    for i, nm in ((1, 'dW1'), (2, 'db1'), (3, 'dW2'), (4, 'db2')):   # split-K / column-sum atomics: the order of the sums varies
        assert rel_l2(gr[i].cpu(), g0[i].cpu()) < 1e-5, f'FeedForward {nm}'
    check_f('FeedForward y - resid', h64(y) - h64(resid_t), h64(y0), U16 * (h64(y).abs() + h64(y0).abs()) + 1e-30)


# ================================================================================================================ model
def test_e2tts_cfg2_shape_plain_residual_vs_oracle(pkg):
    """BASELINE cfg2's model (d512, depth 8, 8 heads, N = 1024, ragged B = 2) with num_residual_streams=1: conditioning probe < 1.5 %,
    loss within 1e-2, prediction rel-L2 within 3e-2, every gradient cosine >= 0.99 (the bounds of tests/model_checks.py)"""
    whole_model(pkg, dict(dim=512, depth=8, heads=8, num_residual_streams=1), B=2, N=1024, lens=[1024, 800], seed=40)


SMALL = dict(dim=128, depth=2, heads=2, num_residual_streams=1)


def test_sample_32_steps_plain_residual_vs_oracle(pkg):
    sample_vs_oracle(pkg, 70, SMALL)


def test_graphed_step_matches_eager_and_launches_no_hyper_connection(pkg, monkeypatch):
    """GraphedTrainStep replays the eager step's gradients; neither launches a hyper-connection entry point"""
    model, _ = small_model(pkg, 3, **SMALL)
    mel, text, rnd = step_inputs(pkg)
    called = set()
    real_call = pkg.lib.call

    def recording_call(name, *a):
        called.add(name)
        return real_call(name, *a)
    monkeypatch.setattr(pkg.lib, 'call', recording_call)
    graphed_matches_eager(pkg, model, mel, text, rnd)
    assert not any(n.startswith('b200_hc_') for n in called), sorted(n for n in called if n.startswith('b200_hc_'))
    assert {'b200_final_norm_fwd', 'b200_final_norm_bwd', 'b200_dwconv_fwd', 'b200_dwconv_bwd', 'b200_rowgate_resid_bwd'} <= called


def test_duration_predictor_plain_residual_vs_oracle(pkg):
    """DurationPredictor(num_residual_streams=1): loss within 1e-2 of the oracle, gradient cosines >= 0.99"""
    duration_vs_oracle(pkg, 41, SMALL)
