"""The HL-Gauss classification head of DurationPredictor(hl_gauss_loss=..., use_regression=False) on the GPU: b200_hl_gauss_fwd /
_bwd against a float64 restatement of their operation sequence, and whole models against the oracle.

Kernel (NaN-filled outputs, element-wise float64 bounds carried by kernel_checks.Rv, the method of tests/kernel_checks.py): the bin
edges s_j = fmaf(j, bin, min) and sqrt(2) sigma are single fp32 operations, restated exactly on the host (s_j) or with their exact
distance from sqrt(2) sigma (s2). x_j = (s_j - y) / s2 rounds twice; erff carries 2 ulp, erfcf 4 ulp, expf 2 ulp and logf 1 ulp
(CUDA C++ Programming Guide, "Mathematical Functions"; an ulp is at most 2u of the value), plus 2^-146 absolute for erfcf's subnormal
results; the tail masses are differences of erfc values on the side of 0 both edges lie on, and the float64 restatement takes them
the same way, so its own error stays far below the bound. Sums of n terms are within gamma(n) of the exact sum in any order.
Exact properties: the loss is the fp32 sum of the per-item cross-entropies in item order divided by B, d_logits is fl(fl(dloss / B)
diff) bit for bit, the counter word is 0 again after the launch, an item launched alone has the bits it has in the batch, and two
launches give the same bits. NaN where both cdf ends round to the same value (targets >= 8 sigma outside an unclamped support)."""
import copy
import math
import random

import pytest
import torch

from conftest import rel_l2
import hl_gauss_ref as H
from kernel_checks import F32, F64, U, Rv, add, check_e, check_f, dev, gamma, mono, mul, neg, pkg  # noqa: F401
from model_checks import cos
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

FLOOR = 2.0 ** -146   # erfcf's absolute error on subnormal results
SQRT2_F = torch.tensor(1.41421356, dtype=F32)


def div(a, b):
    q = a.v / b.v
    return Rv(q, (a.e + q.abs() * b.e) / (b.v.abs() - b.e) + U * (q.abs() + (a.e + q.abs() * b.e) / (b.v.abs() - b.e)))


def total(a, dim):
    """a sum of n terms along dim, any order"""
    n = a.v.shape[dim]
    s = Rv(a.v.sum(dim), a.e.sum(dim))
    return Rv(s.v, s.e + gamma(n) * a.mag().sum(dim))


def erf_diff(a, b):
    """erf(b) - erf(a), a <= b, through erfc where both lie on one side of 0 (the kernel's branches)"""
    erfc = lambda x: Rv(mono(x, torch.special.erfc, 8 * U).v, mono(x, torch.special.erfc, 8 * U).e + FLOOR)   # noqa: E731
    pos, neg_ = a.v >= 0, b.v <= 0
    d_pos = add(erfc(a), neg(erfc(b)))
    d_neg = add(erfc(neg(b)), neg(erfc(neg(a))))
    d_mid = add(mono(b, torch.special.erf, 4 * U), neg(mono(a, torch.special.erf, 4 * U)))
    v = torch.where(pos, d_pos.v, torch.where(neg_, d_neg.v, d_mid.v))
    e = torch.where(pos, d_pos.e, torch.where(neg_, d_neg.e, d_mid.e))
    return Rv(v, e)


def edges(lo, hi, nb):
    """the kernel's fp32 edges, exactly: bin = fl((hi - lo) / nb), s_j = fl(j bin + lo), s_nb = hi"""
    lo32, hi32 = torch.tensor(lo, dtype=F32), torch.tensor(hi, dtype=F32)
    bin_ = (hi32 - lo32) / nb
    j = torch.arange(nb + 1, dtype=F64)
    s = (j * bin_.double() + lo32.double()).to(F32)   # the product is exact in float64, so this is fmaf's one rounding
    s[nb] = hi32
    return s


def restate(logits, target, lo, hi, nb, sigma, clamp):
    """float64 restatement with bounds: (ce [B], diff [B, nb], the rows the reference makes NaN); target None: the prediction [B]"""
    l = logits.double().cpu()
    m = l.max(-1, keepdim=True).values
    d = Rv(l - m, U * (l - m).abs())
    e = mono(d, torch.exp, 4 * U)
    S = total(e, -1)
    s = edges(lo, hi, nb).double()
    if target is None:
        c = ((s[:-1].float() + s[1:].float()) * 0.5).double()   # fp32 add and an exact halving, as in the kernel
        sm = div(e, Rv(S.v[:, None], S.e[:, None]))
        return total(mul(sm, Rv(c[None].expand_as(sm.v))), -1)
    y = target.double().cpu()
    if clamp:
        y = y.clamp(lo, hi)
    s2_32 = torch.tensor(sigma, dtype=F32) * SQRT2_F
    s2 = Rv(torch.tensor(math.sqrt(2.) * sigma, dtype=F64), (s2_32.double() - math.sqrt(2.) * sigma).abs())
    dv = s[None] - y[:, None]
    x = div(Rv(dv, U * dv.abs()), Rv(s2.v.expand_as(dv), s2.e.expand_as(dv)))
    mass = erf_diff(x[:, :-1], x[:, 1:])
    z = erf_diff(x[:, :1], x[:, -1:])
    x32 = dv.float() / s2_32   # fp32 erf rounds to +-1 beyond |x| = 3.92: the NaN rows lie far beyond that, the others well inside
    nan_rows = torch.special.erf(x32[:, -1]) - torch.special.erf(x32[:, 0]) == 0
    p = div(mass, z)
    logS = mono(S, torch.log, 2 * U)
    lp = add(d, neg(Rv(logS.v[:, None], logS.e[:, None])))
    ce = neg(total(mul(p, lp), -1))
    sm = div(e, Rv(S.v[:, None], S.e[:, None]))
    return ce, add(sm, neg(p)), nan_rows


def check_e_nan(name, got, want):
    """bit for bit where want is a number, NaN where it is NaN"""
    got, want = got.detach().cpu(), want.detach().cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f'{name}: NaN pattern differs'
    check_e(name, got[~nan], want[~nan])


def launch(pkg, logits, target, lo, hi, sigma, clamp, count=None):
    B, nb = logits.shape
    t = lambda *shape: torch.full(shape, float('nan'), device=dev(), dtype=F32)   # noqa: E731
    out = dict(ce=t(B), loss=t(1), diff=t(B, nb), pred=t(B))
    count = torch.zeros(1, device=dev(), dtype=torch.int32) if count is None else count
    a = pkg.lib.make_args('b200_hl_gauss_args', logits=logits, target=target, ce=out['ce'], loss=out['loss'], diff=out['diff'],
                          pred=out['pred'], ws_count=count, B=B, num_bins=nb, min_value=lo, max_value=hi, sigma=sigma, clamp_to_range=int(clamp))
    pkg.lib.call('b200_hl_gauss_fwd', a, pkg.ops._stream())
    torch.cuda.synchronize()
    return out, count


def inputs(B, nb, seed):
    """logits up to +-80 (randn * 6, and +-80 spikes), targets at edges, centres, min, max, beyond the support by 1 and 3 sigma, and
    >= 8 sigma outside (NaN without clamp); bin size 2, sigma 1.5"""
    lo, hi, sigma = 0., 2. * nb, 1.5
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, nb, generator=g) * 6
    k = torch.randint(0, nb, (B,), generator=g)
    logits[torch.arange(B), k] = torch.where(torch.rand(B, generator=g) < 0.5, 80., -80.)
    s = edges(lo, hi, nb)
    pool = [lo, hi, float(s[nb // 2]), float(s[1]), float(s[nb - 1]), float(s[0] + s[1]) / 2, float(s[nb - 1] + s[nb]) / 2,
            hi + sigma, lo - 3 * sigma, hi + 3 * sigma, hi + 10 * sigma, lo - 12 * sigma, float(torch.rand(1, generator=g)) * hi]
    target = torch.tensor([pool[(i * 5 + seed) % len(pool)] for i in range(B)], dtype=F32)
    if B == 1:
        target[0] = pool[seed % 3]
    return logits, target, lo, hi, sigma


SHAPES = [(B, nb) for nb in (2, 3, 100, 1000, 4096) for B in (1, 7, 64)]


@pytest.mark.parametrize('B,nb', SHAPES)
@pytest.mark.parametrize('clamp', [False, True])
def test_hl_gauss_fwd_bwd(pkg, B, nb, clamp):
    logits, target, lo, hi, sigma = inputs(B, nb, seed=B + nb)
    L, T = logits.to(dev()), target.to(dev())
    out, count = launch(pkg, L, T, lo, hi, sigma, clamp)
    ce, diff, nan_rows = restate(logits, target, lo, hi, nb, sigma, clamp)
    tag = f'B{B} nb{nb} clamp={clamp}'
    if clamp:
        assert not nan_rows.any()
    got_ce, got_diff = out['ce'].cpu(), out['diff'].cpu()
    assert bool(torch.isnan(got_ce[nan_rows]).all()), f'{tag}: the reference gives NaN here'
    assert bool(torch.isnan(got_diff[nan_rows]).all())
    ok = ~nan_rows
    check_f(f'ce {tag}', got_ce[ok], ce.v[ok], ce.e[ok])
    check_f(f'diff {tag}', got_diff[ok], diff.v[ok], diff.e[ok])
    # loss: the fp32 sum in item order, / B, bit for bit; NaN with any NaN item
    t = torch.zeros((), dtype=F32)
    for j in range(B):
        t = t + got_ce[j]
    want = (t / B).reshape(1)
    if bool(nan_rows.any()):
        assert bool(torch.isnan(out['loss']).all())
    else:
        check_e(f'loss {tag}', out['loss'], want)
    check_e('counter back to 0', count, torch.zeros(1, dtype=torch.int32))
    # two launches: the same bits (the counter word reused)
    again, _ = launch(pkg, L, T, lo, hi, sigma, clamp, count=count)
    for k in ('ce', 'loss', 'diff'):
        assert torch.equal(again[k].cpu().view(torch.int32), out[k].cpu().view(torch.int32)), k
    # each item alone: the bits it has in the batch
    for b in sorted({0, B // 2, B - 1}):
        one, _ = launch(pkg, L[b:b + 1].contiguous(), T[b:b + 1].contiguous(), lo, hi, sigma, clamp)
        assert torch.equal(one['ce'].cpu().view(torch.int32), got_ce[b:b + 1].view(torch.int32)), b
        assert torch.equal(one['loss'].cpu().view(torch.int32), got_ce[b:b + 1].view(torch.int32)), b
        assert torch.equal(one['diff'].cpu().view(torch.int32), got_diff[b:b + 1].view(torch.int32)), b
    # backward: fl(fl(dloss / B) * diff), bit for bit, dloss read on the device
    dloss = torch.tensor([0.7], device=dev())
    dl = torch.full((B, nb), float('nan'), device=dev())
    a = pkg.lib.make_args('b200_hl_gauss_args', diff=out['diff'], dloss=dloss, dlogits=dl, B=B, num_bins=nb, min_value=lo, max_value=hi,
                          sigma=sigma)
    pkg.lib.call('b200_hl_gauss_bwd', a, pkg.ops._stream())
    torch.cuda.synchronize()
    g = torch.tensor(0.7, dtype=F32) / B
    check_e_nan(f'd_logits {tag}', dl, g * got_diff)


@pytest.mark.parametrize('B,nb', SHAPES)
def test_hl_gauss_predict(pkg, B, nb):
    logits, _, lo, hi, sigma = inputs(B, nb, seed=7 * B + nb)
    out, _ = launch(pkg, logits.to(dev()), None, lo, hi, sigma, False)
    pred = restate(logits, None, lo, hi, nb, sigma, False)
    check_f(f'pred B{B} nb{nb}', out['pred'].cpu(), pred.v, pred.e)
    assert bool(torch.isnan(out['loss']).all()) and bool(torch.isnan(out['ce']).all())   # prediction mode writes nothing else


def test_node_and_predict_helper(pkg):
    """ops.HLGaussLoss / hl_gauss_predict: the same bits as the entry point, the gradient through autograd is b200_hl_gauss_bwd's"""
    logits, target, lo, hi, sigma = inputs(7, 100, seed=3)
    spec = pkg.ops.HLGaussSpec(lo, hi, 100, sigma=sigma)
    L = logits.to(dev()).requires_grad_()
    loss = pkg.ops.HLGaussLoss.apply(L, target.to(dev()), spec)
    out, _ = launch(pkg, logits.to(dev()), target.to(dev()), lo, hi, sigma, False)
    nan = bool(torch.isnan(out['loss']).all())
    assert nan == bool(torch.isnan(loss)) and (nan or float(loss) == float(out['loss']))
    loss.backward(torch.tensor(2.0, device=dev()))
    check_e_nan('d_logits', L.grad, (torch.tensor(2.0, dtype=F32) / 7) * out['diff'].cpu())
    pred = pkg.ops.hl_gauss_predict(logits.to(dev()), spec)
    ref, _ = launch(pkg, logits.to(dev()), None, lo, hi, sigma, False)
    check_e('pred', pred, ref['pred'])


# ---------------------------------------------------------------------------------------------------------------------- whole models
HL = dict(min_value=0., max_value=128., num_bins=64, sigma=3.)
TKW = dict(dim=128, depth=2, heads=2)


def hl_model(pkg, seed, hl=HL, tkw=TKW, cls='DurationPredictor'):
    """a DurationPredictor with the HL-Gauss head (or an E2TTS driving one) on the GPU, zero-initialised tensors randomised"""
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dropout=0., max_seq_len=256, **tkw)
    dp = dict(transformer=copy.deepcopy(t), hl_gauss_loss=hl, use_regression=False)
    model = pkg.DurationPredictor(**dp) if cls == 'DurationPredictor' else pkg.E2TTS(transformer=t, duration_predictor=dp, use_vocos=False)
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1)
    model.load_state_dict(sd)
    return model.to(dev()), sd


def dp_inputs():
    g = torch.Generator().manual_seed(5)
    return torch.randn(3, 72, 100, generator=g), torch.tensor([72, 50, 31]), ['abc', 'hello world', 'x'], torch.tensor([0.3, 0.6, 0.9])


def eager_step(pkg, model, mel, lens, text, frac):
    for p in model.parameters():
        p.grad = None
    with pkg.inject_randomness(duration_rand_frac=frac.to(dev())):
        loss = model(mel.to(dev()), text=text, lens=lens.to(dev()))
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def test_duration_predictor_step_vs_oracle(pkg):
    """training loss within 1e-2, gradients present with cosine >= 0.99 where not negligible; predictions within 1e-3 of the range"""
    model, sd = hl_model(pkg, 71)
    model.train()
    mel, lens, text, frac = dp_inputs()
    loss, grads = eager_step(pkg, model, mel, lens, text, frac)
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = H.duration_forward(osd, O.TransformerCfg(cond_on_time=False, **TKW), mel, O.list_str_to_tensor(text), lens=lens, rand_frac=frac,
                             hl_gauss=HL)
    ref.backward()
    print(f'HL-Gauss duration predictor: loss {loss:.6f} (oracle {float(ref):.6f})')
    assert abs(loss - float(ref)) <= 1e-2 * abs(float(ref))
    tot = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    assert 'hl_gauss_layer.to_pred.0.weight' in grads
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None:
            assert k not in grads or float(grads[k].abs().max()) == 0.0, k
            continue
        if float(gr.norm()) < 1e-4 * tot:
            continue
        assert cos(grads[k].cpu(), gr) >= 0.99, k
    model.eval()
    with torch.no_grad():
        pred = model(mel.to(dev()), text=text, lens=lens.to(dev()), return_loss=False)
        want = H.duration_forward(sd, O.TransformerCfg(cond_on_time=False, **TKW), mel, O.list_str_to_tensor(text), lens=lens,
                                  return_loss=False, hl_gauss=HL)
    assert pred.dtype == F32 and pred.shape == (3,)
    print(f'HL-Gauss predictions: max |GPU - oracle| {float((pred.cpu() - want).abs().max()):.4g} frames')
    assert float((pred.cpu() - want).abs().max()) <= 1e-3 * (HL['max_value'] - HL['min_value'])


def test_nan_target_gives_nan_loss(pkg):
    """a length 10 sigma beyond an unclamped support: the reference's loss is NaN, so is the model's"""
    hl = dict(min_value=0., max_value=40., num_bins=16, sigma=2.)
    model, _ = hl_model(pkg, 72, hl=hl)
    model.train()
    mel, lens, text, frac = dp_inputs()
    loss, _ = eager_step(pkg, model, mel, torch.tensor([72, 30, 31]), text, frac)
    assert math.isnan(loss)
    loss, _ = eager_step(pkg, model, mel, torch.tensor([40, 30, 31]), text, frac)
    assert math.isfinite(loss)


def test_graphed_step_matches_eager(pkg):
    """GraphedTrainStep replays the eager step (prefix fractions pinned): loss within 1e-3, gradients within rel-L2 2e-3"""
    model, _ = hl_model(pkg, 73)
    model.train()
    mel, lens, text, frac = dp_inputs()
    want_loss, want = eager_step(pkg, model, mel, lens, text, frac)
    for p in model.parameters():
        p.grad = None
    with pkg.inject_randomness(duration_rand_frac=frac.to(dev())):
        step = pkg.GraphedTrainStep(model, mel.to(dev()), text=text, lens=lens.to(dev()))
        got_loss = float(step())
    torch.cuda.synchronize()
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (got_loss, want_loss)
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(want)
    for n in want:
        assert rel_l2(got[n].float().cpu(), want[n].float().cpu()) < 2e-3 or float(want[n].norm()) == 0, n


def test_bucketed_micro_step(pkg):
    """one BucketedTrainStep micro-step of a ragged batch (72 frames padded to the 96 bucket): the eager step at the padded shape, loss
    within 1e-3 and the accumulated gradients (k = 1) within rel-L2 2e-3; the loss also within 1e-3 of the unpadded eager step's"""
    model, _ = hl_model(pkg, 74)
    model.train()
    mel, lens, text, frac = dp_inputs()
    unpadded_loss, _ = eager_step(pkg, model, mel, lens, text, frac)
    want_loss, want = eager_step(pkg, model, torch.nn.functional.pad(mel, (0, 0, 0, 96 - 72)), lens, text, frac)
    for p in model.parameters():
        p.grad = None
    with pkg.inject_randomness(duration_rand_frac=frac.to(dev())):
        steps = pkg.BucketedTrainStep(model, batch_size=3, buckets=(64, 96), warmup=1)
        got_loss = float(steps(mel.to(dev()), text=text, lens=lens.to(dev())))
    torch.cuda.synchronize()
    assert steps.sync_gradients
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (got_loss, want_loss)
    assert abs(got_loss - unpadded_loss) <= 1e-3 * abs(unpadded_loss), (got_loss, unpadded_loss)
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(want)
    for n in want:
        assert rel_l2(got[n].float().cpu(), want[n].float().cpu()) < 2e-3 or float(want[n].norm()) == 0, n


def test_checkpointed_step_matches_plain(pkg):
    """Transformer(checkpoint_activations=True) under the HL-Gauss head: the plain step's loss and gradients"""
    model, _ = hl_model(pkg, 75)
    model.train()
    mel, lens, text, frac = dp_inputs()
    runs = []
    for ckpt in (False, True):
        model.transformer.checkpoint_activations = ckpt
        runs.append(eager_step(pkg, model, mel, lens, text, frac))
    (l0, g0), (l1, g1) = runs
    assert abs(l1 - l0) <= 1e-5 * abs(l0), (l0, l1)
    assert set(g0) == set(g1)
    for n in g0:
        assert rel_l2(g1[n].float().cpu(), g0[n].float().cpu()) < 2e-3 or float(g0[n].norm()) == 0, n


def test_sample_durations_vs_oracle(pkg):
    """E2TTS.sample without `duration`: the HL-Gauss predictions .long() equal the oracle's, except where the oracle's float64
    prediction lies within the bound (1e-3 of the range) of an integer, where +-1 is allowed; the sample is as long as the longest
    duration and matches the oracle's ODE on those durations"""
    hl = dict(min_value=0., max_value=96., num_bins=48)
    model, sd = hl_model(pkg, 76, hl=hl, cls='E2TTS')
    torch.manual_seed(77)
    cond = torch.randn(2, 24, 100)
    text = ['Hello', 'Goodbye then']
    ids = O.list_str_to_tensor(text)
    lens = torch.maximum((ids != -1).sum(-1), torch.full((2,), 24))
    dsd = {k[len('duration_predictor.'):]: v.double() for k, v in sd.items() if k.startswith('duration_predictor.')}
    old = torch.get_default_dtype()
    torch.set_default_dtype(F64)
    try:
        with torch.no_grad():
            want = H.duration_forward(dsd, O.TransformerCfg(cond_on_time=False, **TKW), cond.double(), ids, lens=lens, return_loss=False,
                                      hl_gauss=hl)
    finally:
        torch.set_default_dtype(old)
    with torch.no_grad():
        got = model.duration_predictor(cond.to(dev()), text=ids.to(dev()), lens=lens.to(dev()), return_loss=False).cpu()
    bound = 1e-3 * (hl['max_value'] - hl['min_value'])
    print(f'sample durations: predictions {got.tolist()} (oracle {want.tolist()})')
    assert float((got.double() - want).abs().max()) <= bound, (got, want)
    near = (want - want.round()).abs() <= bound
    dur_got, dur_want = got.long(), want.long()
    assert bool(((dur_got == dur_want) | (near & ((dur_got - dur_want).abs() <= 1))).all()), (got, want)
    duration = torch.maximum(lens + 1, dur_got)
    y0 = torch.randn(2, int(duration.max()), 100)
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(cond.to(dev()), text=text, steps=4, return_raw_output=True)
    assert out.shape == (2, int(duration.max()), 100)
    ref = O.e2tts_sample(sd, O.TransformerCfg(**TKW), cond, ids, duration=duration, y0=y0, steps=4, cfg_strength=1.0)
    assert rel_l2(out.cpu(), ref) < 5e-2
