"""GPU parity tests (run with -m gpu on an H100): every CUDA stage through the C ABI against the oracle
(oracle/e2tts_oracle.py, fp32) on identical seeded inputs, then the whole model against the golden vectors
minted from the reference's own e2_tts.py.

Tolerances (bf16 tensor-core path vs fp32 oracle, SURVEY §8c): per-leaf rel-L2 <= 2e-2, whole-model pred
rel-L2 <= 3e-2, loss rel <= 1e-2, parameter-gradient cosine >= 0.99, ODE end point rel-L2 <= 5e-2,
log-mel abs <= 1e-3.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_l2
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

LEAF_TOL = 2e-2


@pytest.fixture(scope='module')
def pkg():
    import e2_tts_pytorch_b200 as pkg
    assert torch.cuda.is_available()
    pkg.lib.load()
    return pkg


def dev():
    return torch.device('cuda:0')


def bf(t):
    return t.to(torch.bfloat16).contiguous()


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def check(name, got, want, tol=LEAF_TOL):
    e = rel_l2(got.float().cpu(), want.float().cpu())
    assert e < tol, f'{name}: rel-L2 {e:.4g} >= {tol}'


# ---------------------------------------------------------------------------------------------------------------------
def test_gemm_modes(pkg):
    torch.manual_seed(0)
    ops = pkg.ops
    M, N, K = 304, 264, 192
    A, B = bf(torch.randn(M, K, device=dev())), bf(torch.randn(N, K, device=dev()))
    ref = A.float() @ B.float().t()
    check('nt', ops.gemm(A, B, M, N, K)[:, :N], ref, 1e-2)
    Bt = B.t().contiguous()   # [K, N]
    check('b mn-major', ops.gemm(A, Bt, M, N, K, b_mn=True)[:, :N], ref, 1e-2)
    At = A.t().contiguous()   # [K, M]
    got = ops.gemm(At, Bt, M, N, K, lda=M, ldb=N, a_mn=True, b_mn=True, out_fp32=True, split_k=3)
    check('dW split-k', got, ref, 1e-3)
    A1, A2 = A[:, :128].contiguous(), A[:, 128:].contiguous()
    check('two-source', ops.gemm(A1, B, M, N, K, lda=128, A2=A2, lda2=64, K1=128)[:, :N], ref, 1e-2)
    # K = 104 ends in a partial 64-wide k-block; fp32 output with a bias at N = 100 (row pitch not a multiple of 8)
    M, N, K = 300, 200, 104
    A, B = bf(torch.randn(M, K, device=dev())), bf(torch.randn(N, K, device=dev()))
    check('k tail', ops.gemm(A, B, M, N, K)[:, :N], A.float() @ B.float().t(), 1e-2)
    M, N, K = 200, 100, 128
    A, B = bf(torch.randn(M, K, device=dev())), bf(torch.randn(N, K, device=dev()))
    bias = torch.randn(N, device=dev())
    check('fp32 + bias', ops.gemm(A, B, M, N, K, bias=bias, out_fp32=True), A.float() @ B.float().t() + bias, 1e-3)


def test_hyper_width_depth(pkg):
    torch.manual_seed(1)
    ops = pkg.ops
    B, n, S, D = 2, 40, 4, 128
    T = B * n
    x = (torch.randn(T, S, D, device=dev()) * 1.5).to(torch.bfloat16).requires_grad_()
    P = dict(gamma=torch.randn(D) * 0.1, afn=torch.randn(D, S + 1) * 0.05, ascale=torch.tensor(0.5), salpha=torch.randn(S, S + 1) * 0.5 + 0.3,
             bfn=torch.randn(D) * 0.05, bscale=torch.tensor(0.7), sbeta=torch.randn(S) * 0.3 + 1)
    P = {k: v.to(dev()).requires_grad_() for k, v in P.items()}
    gain = (1 + 0.2 * torch.randn(B, D, device=dev())).requires_grad_()
    y = bf(torch.randn(T, D, device=dev())).requires_grad_()
    for mode, ng in ((2, gain), (1, gain[0].detach().clone().requires_grad_()), (0, None)):
        br, res, beta = ops.HcWidth.apply(x, P['gamma'], P['afn'], P['ascale'], P['salpha'], P['bfn'], P['bscale'], P['sbeta'], ng, mode, n)
        out = ops.HcDepth.apply(res, y, beta)
        wb, wo = torch.randn_like(br, dtype=torch.float32), torch.randn_like(out, dtype=torch.float32)
        loss = (br.float() * wb).sum() + (out.float() * wo).sum()
        leaves = [x, y] + list(P.values()) + ([ng] if ng is not None else [])
        grads = torch.autograd.grad(loss, leaves)
        # oracle
        xr = x.detach().float().view(B, n, S, D).requires_grad_()
        yr = y.detach().float().view(B, n, D).requires_grad_()
        sd = {'p.norm.gamma': P['gamma'], 'p.dynamic_alpha_fn': P['afn'], 'p.dynamic_alpha_scale': P['ascale'], 'p.static_alpha': P['salpha'],
              'p.dynamic_beta_fn': P['bfn'], 'p.dynamic_beta_scale': P['bscale'], 'p.static_beta': P['sbeta']}
        sd = {k: v.detach().clone().requires_grad_() for k, v in sd.items()}
        ngr = ng.detach().clone().requires_grad_() if ng is not None else None
        b0, rest, be = O.hyper_width(sd, 'p', xr, S)
        if mode == 2:
            b0 = F.normalize(b0, dim=-1) * D ** 0.5 * ngr[:, None, :]
        elif mode == 1:
            b0 = F.normalize(b0, dim=-1) * D ** 0.5 * ngr
        o = O.hyper_depth(rest, be, yr)
        lr = (b0 * wb.view(B, n, D)).sum() + (o * wo.view(B, n, S, D)).sum()
        rleaves = [xr, yr] + list(sd.values()) + ([ngr] if ng is not None else [])
        rgrads = torch.autograd.grad(lr, rleaves)
        check(f'branch m{mode}', br, b0.reshape(T, D))
        check(f'out m{mode}', out, o.reshape(T, S, D))
        check(f'beta m{mode}', beta, be.reshape(T, S), 1e-3)
        names = ['d_xres', 'd_y', 'gamma', 'afn', 'ascale', 'salpha', 'bfn', 'bscale', 'sbeta', 'gain']
        for nm, a, b in zip(names, grads, rgrads):
            check(f'{nm} m{mode}', a.reshape(-1), b.reshape(-1), 3e-2)


@pytest.mark.parametrize('D,ks,Np', [(128, 31, 100), (64, 7, 100), (512, 31, 333), (264, 31, 70), (128, 31, 40)])
def test_dwconv(pkg, D, ks, Np):
    """fwd + (dx, dw, db) vs the oracle; Np = 333 spans two blocks of four 64-token tiles, D = 264 leaves a partial channel tile,
    Np = 40 is shorter than one tile, so the 15-row halo runs past both ends of the sequence."""
    torch.manual_seed(2)
    ops = pkg.ops
    B = 2
    x = bf(torch.randn(B * Np, D, device=dev())).requires_grad_()
    w = (torch.randn(D, 1, ks, device=dev()) * 0.2).requires_grad_()
    b = (torch.randn(D, device=dev()) * 0.1).requires_grad_()
    mask = torch.ones(B, Np, dtype=torch.bool, device=dev())
    mask[1, int(Np * 0.7):] = False
    y = ops.DwConv.apply(x, w, b, mask.to(torch.uint8).contiguous(), B, Np)
    wo = torch.randn_like(y, dtype=torch.float32)
    g = torch.autograd.grad((y.float() * wo).sum(), [x, w, b])
    xr, wr, br_ = x.detach().float().view(B, Np, D).requires_grad_(), w.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    yr = O.depthwise_conv({'c.dw_conv1d.0.weight': wr, 'c.dw_conv1d.0.bias': br_}, 'c', xr, mask)
    gr = torch.autograd.grad((yr * wo.view(B, Np, D)).sum(), [xr, wr, br_])
    check('y', y, yr.reshape(B * Np, D))
    for nm, a, c in zip(['dx', 'dw', 'db'], g, gr):
        check(nm, a.reshape(-1), c.reshape(-1), 3e-2)


@pytest.mark.parametrize('value_residual,Np', [(False, 96), (True, 150)])
def test_attention_node(pkg, value_residual, Np):
    """Attention (the model's node) + OutProj vs oracle.attention (rotary, softclamp, key mask, value residual, head gate)."""
    torch.manual_seed(3)
    ops, mods = pkg.ops, pkg.modules
    B, H, d = 2, 2, 128
    T = B * Np
    attn = mods.Attention(d, H, 64, value_residual).to(dev())
    with torch.no_grad():
        attn.to_v_head_gate.weight.normal_(0, 0.05)
        attn.to_v_head_gate.bias.normal_(0, 1)
    x = bf(torch.randn(T, d, device=dev())).requires_grad_()
    mask = torch.ones(B, Np, dtype=torch.bool, device=dev())
    mask[0, Np - 17:] = False
    mu8 = mask.to(torch.uint8).contiguous()
    vf = bf(torch.randn(B, H, Np, 64, device=dev())).requires_grad_() if value_residual else None
    mix = attn.to_value_residual_mix
    ws = [attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, attn.to_v_head_gate.weight] + ([mix[0].weight] if value_residual else [])
    wpack = bf(torch.cat([w.detach() for w in ws], 0))
    opack = bf(attn.to_out.weight.detach())
    cs, sn = ops.rotary_table(Np, dev())
    gatecs = (torch.rand(B, d, device=dev()) * 0.8 + 0.1).requires_grad_()
    og, v = ops.Attention.apply(x, attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, attn.to_v_head_gate.weight, attn.to_v_head_gate.bias,
                                mix[0].weight if value_residual else None, mix[0].bias if value_residual else None, vf, wpack, cs, sn, mu8,
                                B, Np, H, 0.0, 0, 50.0, None)
    y = ops.OutProj.apply(og, attn.to_out.weight, opack, gatecs, mu8, B, Np)
    wo = torch.randn_like(y, dtype=torch.float32)
    params = [p for p in attn.parameters()]
    leaves = [x, gatecs] + params + ([vf] if value_residual else [])
    grads = torch.autograd.grad((y.float() * wo).sum(), leaves)
    # oracle
    sd = {'a.' + k_: p.detach().clone().requires_grad_() for k_, p in attn.named_parameters()}
    xr = x.detach().float().view(B, Np, d).requires_grad_()
    gr_ = gatecs.detach().clone().requires_grad_()
    vfr = vf.detach().float().requires_grad_() if value_residual else None
    out, vals = O.attention(sd, 'a', xr, mask, O.rotary_freqs(Np, 64, dev()), vfr, H, 64, 50.0)
    out = out * gr_[:, None, :]
    rparams = [sd['a.' + k_] for k_, _ in attn.named_parameters()]
    rleaves = [xr, gr_] + rparams + ([vfr] if value_residual else [])
    rgrads = torch.autograd.grad((out * wo.view(B, Np, d)).sum(), rleaves)
    check('attn out', y, out.reshape(T, d))
    if not value_residual:
        check('orig values', v, vals)
    names = ['dx', 'd_gate_cs'] + [k_ for k_, _ in attn.named_parameters()] + ['d_vfirst']
    for nm, a, c in zip(names, grads, rgrads):
        check(nm, a.reshape(-1), c.reshape(-1), 4e-2)


def test_feedforward_cross_skip(pkg):
    torch.manual_seed(4)
    ops, mods = pkg.ops, pkg.modules
    B, Np, d, dt, S = 2, 72, 128, 64, 4
    T = B * Np
    ff = mods.FeedForward(d, 4, 0.).to(dev())
    lin1, lin2 = ff.ff[0].proj, ff.ff[2]
    inner = lin2.weight.shape[1]
    nb = inner // 64
    w1p = bf(lin1.weight.detach().view(2, nb, 64, d).transpose(0, 1).reshape(2 * inner, d))
    b1p = lin1.bias.detach().view(2, nb, 64).transpose(0, 1).reshape(2 * inner).contiguous()
    w2p = bf(lin2.weight.detach())
    x = bf(torch.randn(T, d, device=dev())).requires_grad_()
    cs = (torch.rand(B, d, device=dev()) * 0.8 + 0.1).requires_grad_()
    y = ops.FeedForward.apply(x, lin1.weight, lin1.bias, lin2.weight, lin2.bias, w1p, b1p, w2p, cs, B, Np, 0.0, 0, None)
    wo = torch.randn_like(y, dtype=torch.float32)
    leaves = [x, cs, lin1.weight, lin1.bias, lin2.weight, lin2.bias]
    grads = torch.autograd.grad((y.float() * wo).sum(), leaves)
    sd = {'f.ff.0.proj.weight': lin1.weight, 'f.ff.0.proj.bias': lin1.bias, 'f.ff.2.weight': lin2.weight, 'f.ff.2.bias': lin2.bias}
    sd = {k: v.detach().clone().requires_grad_() for k, v in sd.items()}
    xr, csr = x.detach().float().view(B, Np, d).requires_grad_(), cs.detach().clone().requires_grad_()
    yr = O.feedforward(sd, 'f', xr) * csr[:, None, :]
    rgrads = torch.autograd.grad((yr * wo.view(B, Np, d)).sum(), [xr, csr] + list(sd.values()))
    check('ff out', y, yr.reshape(T, d))
    for nm, a, c in zip(['dx', 'dcs', 'dW1', 'db1', 'dW2', 'db2'], grads, rgrads):
        check('ff ' + nm, a.reshape(-1), c.reshape(-1), 3e-2)

    # cross-condition and skip on S-stream tensors
    for has_at in (True, False):
        cc = mods.TextAudioCrossCondition(d, dt, cond_audio_to_text=has_at).to(dev())
        with torch.no_grad():
            for p in cc.parameters():
                p.normal_(0, 0.05)
        xs = bf(torch.randn(T, S, d, device=dev())).requires_grad_()
        ts = bf(torch.randn(T, S, dt, device=dev())).requires_grad_()
        stack = bf(torch.cat([cc.text_to_audio.weight.detach()] + ([cc.audio_to_text.weight.detach()] if has_at else []), 0))
        xo, to = ops.CrossCondition.apply(xs, ts, cc.text_to_audio.weight, cc.audio_to_text.weight if has_at else None, stack)
        w_x, w_t = torch.randn_like(xo, dtype=torch.float32), torch.randn_like(to, dtype=torch.float32)
        leaves = [xs, ts] + list(cc.parameters())
        grads = torch.autograd.grad((xo.float() * w_x).sum() + (to.float() * w_t).sum(), leaves)
        xr, tr = xs.detach().float().requires_grad_(), ts.detach().float().requires_grad_()
        ps = [p.detach().clone().requires_grad_() for p in cc.parameters()]
        at = torch.cat((xr, tr), -1)
        xor_ = xr + at @ ps[0].t()
        tor_ = tr + at @ ps[1].t() if has_at else tr
        rgrads = torch.autograd.grad((xor_ * w_x).sum() + (tor_ * w_t).sum(), [xr, tr] + ps)
        check('cross x', xo, xor_)
        check('cross t', to, tor_)
        for nm, a, c in zip(['dxs', 'dts', 'dWta', 'dWat'], grads, rgrads):
            check(f'cross {nm} at={has_at}', a.reshape(-1), c.reshape(-1), 3e-2)
    lin = torch.nn.Linear(2 * d, d, bias=False).to(dev())
    xs = bf(torch.randn(T, S, d, device=dev())).requires_grad_()
    sk = bf(torch.randn(T, S, d, device=dev())).requires_grad_()
    out = ops.SkipProj.apply(xs, sk, lin.weight, bf(lin.weight.detach()))
    w_o = torch.randn_like(out, dtype=torch.float32)
    grads = torch.autograd.grad((out.float() * w_o).sum(), [xs, sk, lin.weight])
    xr, sr, wr = xs.detach().float().requires_grad_(), sk.detach().float().requires_grad_(), lin.weight.detach().clone().requires_grad_()
    outr = torch.cat((xr, sr), -1) @ wr.t()
    rgrads = torch.autograd.grad((outr * w_o).sum(), [xr, sr, wr])
    check('skip', out, outr)
    for nm, a, c in zip(['dx', 'dskip', 'dW'], grads, rgrads):
        check('skip ' + nm, a.reshape(-1), c.reshape(-1), 3e-2)


def test_attention_dropout_is_consistent(pkg):
    """dropout > 0: forward/backward use the same counter-based mask (finite-difference-free check: the gradient of
    sum(og * w) wrt v equals P_drop^T (w * gate), which must match a second forward with v perturbed along a direction)."""
    torch.manual_seed(5)
    ops = pkg.ops
    B, H, Np = 1, 2, 80
    q, k, v = (bf(torch.randn(B, H, Np, 64, device=dev())) for _ in range(3))
    gate = torch.rand(B * Np, H, device=dev())
    v1 = v.clone().requires_grad_()
    og = ops.AttnCore.apply(q, k, v1, gate, None, 0.3, 1234, 50.0, None)
    w = torch.randn_like(og, dtype=torch.float32)
    (dv,) = torch.autograd.grad((og.float() * w).sum(), [v1])
    dirn = bf(torch.randn_like(v.float()))
    og2 = ops.AttnCore.apply(q, k, bf(v.float() + 0.5 * dirn.float()), gate, None, 0.3, 1234, 50.0, None)
    lhs = ((og2.float() - og.float()) * w).sum() / 0.5
    rhs = (dv.float() * dirn.float()).sum()
    assert abs(float(lhs - rhs)) <= 0.05 * abs(float(rhs)) + 0.5, (float(lhs), float(rhs))
    og3 = ops.AttnCore.apply(q, k, v, gate, None, 0.3, 99, 50.0, None)
    assert rel_l2(og3.float().cpu(), og.float().cpu()) > 1e-2   # a different seed gives a different mask


# ---------------------------------------------------------------------------------------------------------------------
def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize('case', ['text', 'drop'])
def test_e2tts_forward_backward_vs_golden(pkg, case):
    g = _load('e2tts_d128_L2.pt')
    c = g['cases'][case]
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=g['max_seq_len'], **g['transformer']), use_vocos=False)
    model.load_state_dict(g['state_dict'])
    model.to(dev()).train()
    with pkg.inject_randomness(x0=c['x0'].to(dev()), times=c['times'].to(dev()), span_mask=c['span_mask'].to(dev()),
                               drop_text_cond=c['drop_text_cond']):
        out = model(g['mel'].to(dev()), text=g['text'], lens=g['lens'].to(dev()))
    out.loss.backward()
    assert rel_l2(out.cond.cpu(), c['cond']) == 0.0
    e_pred = rel_l2(out.pred_flow.float().cpu(), c['pred'])
    assert e_pred < 3e-2, e_pred
    assert abs(float(out.loss) - float(c['loss'])) <= 1e-2 * abs(float(c['loss']))
    assert rel_l2(out.pred_data.float().cpu(), c['pred_data']) < 3e-2
    worst = (1.0, None)
    for k, p in model.named_parameters():
        if k not in c['grads']:
            if p.grad is not None:
                assert float(p.grad.abs().max()) == 0.0, f'{k} should be unused'
            continue
        assert p.grad is not None, k
        gr = c['grads'][k]
        if case == 'drop':
            got = torch.stack((p.grad.norm(), p.grad.sum())).cpu()
            assert abs(float(got[0] - gr[0])) <= 0.1 * float(gr[0]) + 1e-6, (k, got, gr)
        else:
            cs_ = cos(p.grad.cpu(), gr)
            if gr.norm() > 1e-6 * max(1.0, gr.numel() ** 0.5):
                worst = min(worst, (cs_, k))
                assert cs_ >= 0.99, (k, cs_)
    print('worst grad cosine', worst)


def test_duration_predictor_vs_golden(pkg):
    """DurationPredictor fwd+bwd against the reference-minted golden (B=4; re-minted in round 2 on a well-conditioned prefix draw,
    oracle/make_golden.py): loss <= 1e-2, every parameter gradient cosine >= 0.99 and norm within 25 % (the loosest parameter is
    hyper_conns.0.1.0.static_beta, the 4-element parameter the old fixture was ill-conditioned for)."""
    g, e = _load('duration_d128_L2.pt'), _load('e2tts_d128_L2.pt')
    dp = pkg.DurationPredictor(transformer=dict(dropout=0., max_seq_len=256, **e['transformer']))
    dp.load_state_dict(g['state_dict'])
    dp.to(dev()).train()
    with pkg.inject_randomness(duration_rand_frac=g['rand_frac'].to(dev())):
        loss = dp(g['mel'].to(dev()), text=g['text'], lens=g['lens'].to(dev()))
    loss.backward()
    assert abs(float(loss) - float(g['loss'])) <= 1e-2 * abs(float(g['loss']))
    total = float(torch.cat([v.flatten() for v in g['grads'].values()]).norm())
    worst = (1.0, None)
    for k, p in dp.named_parameters():
        if k not in g['grads']:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, f'{k} should be unused'
            continue
        gr = g['grads'][k]
        if float(gr.norm()) < 1e-4 * total:
            continue
        cs_ = cos(p.grad.cpu(), gr)
        worst = min(worst, (cs_, k))
        assert cs_ >= 0.99, (k, cs_)
        assert 0.8 <= float(p.grad.norm()) / float(gr.norm()) <= 1.25, (k, float(p.grad.norm()), float(gr.norm()))
    print('duration: worst grad cosine', worst)
    dp.eval()
    with torch.no_grad():
        pred = dp(g['mel'].to(dev()), text=g['text'], lens=g['lens'].to(dev()), return_loss=False)
    assert rel_l2(pred.cpu(), g['pred']) < 2e-2


def test_sample_vs_golden(pkg):
    g, e = _load('sample_d128_L2.pt'), _load('e2tts_d128_L2.pt')
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=e['max_seq_len'], **e['transformer']), use_vocos=False)
    model.load_state_dict(e['state_dict'])
    model.to(dev())
    with pkg.inject_randomness(y0=g['y0'].to(dev())):
        out = model.sample(g['cond'].to(dev()), text=e['text'], duration=g['duration'], steps=g['steps'], cfg_strength=g['cfg_strength'],
                           return_raw_output=True)
    assert out.shape == g['out'].shape
    assert rel_l2(out.cpu(), g['out']) < 5e-2


def test_melspec_vs_golden(pkg):
    g = _load('melspec.pt')
    ms = pkg.MelSpec().to(dev())
    out = ms(g['wave'].to(dev()))
    assert out.shape == g['mel'].shape
    assert float((out.cpu() - g['mel']).abs().max()) < 1e-3


def test_transformer_public_forward_and_readme_snippet(pkg):
    """README usage (reference README.md:30-63) through the public API, at a reduced size; also Transformer.forward."""
    torch.manual_seed(0)
    dp = pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2)).to(dev())
    mel = torch.randn(2, 64, 100, device=dev())
    text = ['Hello', 'Goodbye']
    loss = dp(mel, text=text)
    loss.backward()
    e2 = pkg.E2TTS(duration_predictor=dp, transformer=dict(dim=128, depth=2, heads=2), use_vocos=False).to(dev())
    out = e2(mel, text=text)
    out.loss.backward()
    assert torch.isfinite(out.loss)
    assert all(torch.isfinite(p.grad).all() for p in e2.transformer.parameters() if p.grad is not None)
    sampled = e2.sample(mel[:, :5], text=text, steps=3, return_raw_output=True)
    assert sampled.ndim == 3 and sampled.shape[-1] == 100
    tr = e2.transformer
    y = tr(torch.randn(2, 40, 128, device=dev()), times=torch.rand(2, device=dev()), mask=None, text_embed=torch.randn(2, 40, 64, device=dev()))
    assert y.shape == (2, 40, 128) and torch.isfinite(y).all()


def test_full_size_properties(pkg):
    """BASELINE cfg2 shape (d512 L8, B16 x N1024) is too big for the CPU oracle: check size-independent properties —
    finite loss/grads, loss invariance to batch order, and linearity of the flow target (pred_data - x0 == pred)."""
    torch.manual_seed(0)
    model = pkg.E2TTS(transformer=dict(dim=512, depth=8, dropout=0.), use_vocos=False).to(dev())
    B, N = 4, 1024
    mel = torch.randn(B, N, 100, device=dev())
    text = ['Hello', 'Goodbye'] * (B // 2)
    x0, times = torch.randn_like(mel), torch.rand(B, device=dev())
    span = torch.zeros(B, N, dtype=torch.bool, device=dev())
    span[:, 100:900] = True
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        out = model(mel, text=text)
    out.loss.backward()
    assert torch.isfinite(out.loss)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
    assert rel_l2((out.pred_data - x0).cpu(), out.pred_flow.cpu()) < 1e-5
    perm = torch.tensor([2, 3, 0, 1], device=dev())
    with pkg.inject_randomness(x0=x0[perm], times=times[perm], span_mask=span[perm], drop_text_cond=False):
        out2 = model(mel[perm], text=[text[i] for i in perm.tolist()])
    assert abs(float(out2.loss) - float(out.loss)) <= 2e-3 * abs(float(out.loss))
    assert rel_l2(out2.pred_flow.cpu(), out.pred_flow[perm].cpu()) < 5e-3


def test_feedforward_dropout_mask_is_consistent_between_forward_and_backward(pkg):
    """GEGLU dropout (counter-based pair hash in the GEMM epilogue, recomputed by geglu_bwd): directional-derivative check."""
    torch.manual_seed(8)
    ops, mods = pkg.ops, pkg.modules
    B, Np, d = 2, 96, 128
    T = B * Np
    ff = mods.FeedForward(d, 4, 0.).to(dev())
    lin1, lin2 = ff.ff[0].proj, ff.ff[2]
    inner = lin2.weight.shape[1]
    nb = inner // 64
    w1p = bf(lin1.weight.detach().view(2, nb, 64, d).transpose(0, 1).reshape(2 * inner, d))
    b1p = lin1.bias.detach().view(2, nb, 64).transpose(0, 1).reshape(2 * inner).contiguous()
    w2p = bf(lin2.weight.detach())
    x = bf(torch.randn(T, d, device=dev()))
    run = lambda xx, seed: ops.FeedForward.apply(xx, lin1.weight, lin1.bias, lin2.weight, lin2.bias, w1p, b1p, w2p, None, B, Np, 0.3, seed, None)
    x1 = x.clone().requires_grad_()
    y1 = run(x1, 77)
    w = torch.randn_like(y1, dtype=torch.float32)
    (dx,) = torch.autograd.grad((y1.float() * w).sum(), [x1])
    dirn = bf(torch.randn_like(x.float()))
    eps = 0.0625   # central difference: the GEGLU is nonlinear, second-order terms cancel
    xp, xm = bf(x.float() + eps * dirn.float()), bf(x.float() - eps * dirn.float())
    step = (xp.float() - xm.float())          # the perturbation actually applied after bf16 rounding
    lhs = float(((run(xp, 77).float() - run(xm, 77).float()) * w).sum())
    rhs = float((dx.float() * step).sum())
    assert abs(lhs - rhs) <= 0.1 * abs(rhs) + 2.0, (lhs, rhs)
    assert rel_l2(run(x, 77).float().cpu(), y1.float().cpu()) == 0.0          # deterministic for a fixed seed
    assert rel_l2(run(x, 78).float().cpu(), y1.float().cpu()) > 1e-2          # and seed-dependent


def test_graphed_train_step_matches_eager_step(pkg):
    """e2_tts_pytorch_b200.GraphedTrainStep replays forward + backward as one CUDA graph: with the step's randomness pinned
    (inject_randomness) and dropout off, loss and parameter gradients must equal the eager step; with dropout on, two replays
    must draw different masks (the device seed word) and stay finite."""
    torch.manual_seed(0)
    B, N = 2, 96
    model = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, dropout=0.0), use_vocos=False).to(dev())
    model.train()
    model.cond_drop_prob = 0.0
    mel = torch.randn(B, N, 100, device=dev())
    text = pkg.list_str_to_tensor(['Hello', 'Goodbye']).to(dev())
    x0 = torch.randn(B, N, 100, device=dev())
    times = torch.rand(B, device=dev())
    span = torch.zeros(B, N, dtype=torch.bool, device=dev())
    span[:, 20:70] = True
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        out = model(mel, text=text)
        out.loss.backward()
        want_loss = float(out.loss)
        want = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        for p in model.parameters():
            p.grad = None
        del out   # an alive eager graph keeps its AccumulateGrad nodes (bound to the default stream) and would drag stream 0 into the capture
        step = pkg.GraphedTrainStep(model, mel, text=text)
        got_loss = float(step())
    assert step.launches_per_step > 50
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (got_loss, want_loss)
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(want)
    worst = max(rel_l2(got[n].float().cpu(), want[n].float().cpu()) for n in want if float(want[n].norm()) > 0)
    assert worst < 2e-3, f'graphed vs eager gradients: worst rel-L2 {worst:.3g}'   # fp32 atomics reorder between runs
    # a new batch flows through the static input; the loss changes
    got2 = float(step(torch.randn(B, N, 100, device=dev())))
    assert got2 == got2 and got2 != got_loss
    # dropout on: the device seed word re-draws the masks on every replay
    model_d = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, dropout=0.3), use_vocos=False).to(dev())
    model_d.train()
    model_d.cond_drop_prob = 0.0
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        step_d = pkg.GraphedTrainStep(model_d, mel, text=text)
        l1, l2 = float(step_d()), float(step_d())
    assert l1 == l1 and l2 == l2 and l1 != l2, (l1, l2)
