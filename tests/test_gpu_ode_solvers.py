"""GPU: the Runge–Kutta solver of E2TTS.sample (e2-tts-pytorch_b200/ode.py, csrc/ode.cu; SURVEY A.7). The four solver kernels
against float64 element-wise bounds; the solver's step control on an analytic function against the float64 restatement of
tests/ode_ref.py (same evaluation times, same accept / reject decisions, same result); whole-model sample() with every new method
against the oracle with the same method."""
import math

import pytest
import torch

import ode_ref
from conftest import rel_l2
from kernel_checks import dev, pkg
from model_checks import small_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
CFG5 = 8 * 2048 * 100            # the state of bench.py cfg5: B8 x 2048 frames x 100 mel channels
SIZES = [1, 3, 4, 5, 127, CFG5 + 3]


def nan_like(t):
    return torch.full_like(t, float('nan'))


def randn(n, seed, scale=1.0):
    return torch.randn(n, generator=torch.Generator().manual_seed(seed)) * scale


def weights(S, seed):
    w = randn(S, seed).tolist()
    w[S // 2] = 0.0                      # a zero and (from the draw) negative weights
    return [float(torch.tensor(v, dtype=torch.float32)) for v in w]


def fma_bound(y0, ks, ws):
    """|error| of the fp32 sum y0 + sum_j w_j k_j: one rounding per term, on the running magnitude"""
    mag = y0.double().abs() + sum(abs(w) * k.double().abs() for w, k in zip(ws, ks))
    return (len(ks) + 2) * EPS * mag + 1e-30


# ---------------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize('n', SIZES)
@pytest.mark.parametrize('S', range(1, 8))
def test_combine_vs_float64(pkg, n, S):
    if n == CFG5 + 3 and S not in (1, 7):
        pytest.skip('the large size at one and seven sources')
    y0, ks = randn(n, S), [randn(n, 100 * S + j) for j in range(S)]
    ws = weights(S, S)
    want = y0.double() + sum(w * k.double() for w, k in zip(ws, ks))
    yd, kd = y0.to(dev()), [k.to(dev()) for k in ks]
    out = nan_like(yd)
    pkg.ops.ode_combine(yd, kd, ws, out=out)
    err = (out.cpu().double() - want).abs()
    assert bool((err <= fma_bound(y0, ks, ws)).all()), float(err.max())
    # unaligned views take the scalar path: same bound
    if n > 4:
        off = nan_like(yd)
        pkg.ops.ode_combine(yd[1:], [k[1:] for k in kd], ws, out=off[1:])
        err = (off[1:].cpu().double() - want[1:]).abs()
        assert bool((err <= fma_bound(y0[1:], [k[1:] for k in ks], ws)).all())


def error_ratio64(y0, ks, ew, y1, atol, rtol):
    err = sum(w * k.double() for w, k in zip(ew, ks))
    tol = atol + rtol * torch.maximum(y0.double().abs(), y1.double().abs())
    return float((err / tol).pow(2).mean().sqrt())


@pytest.mark.parametrize('n', SIZES)
@pytest.mark.parametrize('write_y1', [0, 1])
def test_step_error_vs_float64(pkg, n, write_y1):
    S = 7 if n > 200 else 3 + write_y1
    y0, ks = randn(n, 1), [randn(n, 10 + j, 0.5) for j in range(S)]
    ew, sw = weights(S, 3), weights(S, 4)
    atol, rtol = 1e-3, 1e-2
    y1_want = y0.double() + sum(w * k.double() for w, k in zip(sw, ks))
    yd, kd = y0.to(dev()), [k.to(dev()) for k in ks]
    ws = torch.empty(1024, dtype=torch.float64, device=dev())
    ratio = torch.full((1,), float('nan'), device=dev())
    if write_y1:
        y1 = nan_like(yd)
        pkg.ops.ode_step_error(yd, kd, ew, y1, atol, rtol, ws, ratio, sol_w=sw)
        assert bool(((y1.cpu().double() - y1_want).abs() <= fma_bound(y0, ks, sw)).all())
    else:
        y1 = y1_want.float().to(dev())
        pkg.ops.ode_step_error(yd, kd, ew, y1, atol, rtol, ws, ratio)
    got = float(ratio)
    want = error_ratio64(y0, ks, ew, y1.cpu(), atol, rtol)
    # fp32 error sum and quotient (a few ulp each, relative to the error's term magnitudes) under an fp64 mean square
    assert abs(got - want) <= 1e-5 * want + 1e-30, (got, want)
    # deterministic: the same bits on repeat, and a grid of 3 blocks wrapping the whole state adds the same sum
    again = torch.full((1,), float('nan'), device=dev())
    pkg.ops.ode_step_error(yd, kd, ew, y1, atol, rtol, ws, again, sol_w=sw if write_y1 else None)
    assert torch.equal(again, ratio)
    small = torch.empty(3, dtype=torch.float64, device=dev())
    wrapped = torch.full((1,), float('nan'), device=dev())
    pkg.ops.ode_step_error(yd, kd, ew, y1, atol, rtol, small, wrapped, sol_w=sw if write_y1 else None)
    assert abs(float(wrapped) - got) <= 1e-6 * got


@pytest.mark.parametrize('n', SIZES)
def test_scaled_norms_vs_float64(pkg, n):
    y0, f0, f1 = randn(n, 1), randn(n, 2), randn(n, 3)
    atol, rtol = 1e-4, 1e-3
    scale = atol + y0.double().abs() * rtol
    rms = lambda x: float((x / scale).pow(2).mean().sqrt())
    yd, f0d, f1d = y0.to(dev()), f0.to(dev()), f1.to(dev())
    ws = torch.empty(2 * 1024, dtype=torch.float64, device=dev())
    out = torch.full((2,), float('nan'), device=dev())
    d0, d1 = pkg.ops.ode_scaled_norms(yd, yd, f0d, None, atol, rtol, ws, out).tolist()
    _, d2 = pkg.ops.ode_scaled_norms(yd, None, f1d, f0d, atol, rtol, ws, out).tolist()
    for got, want in ((d0, rms(y0.double())), (d1, rms(f0.double())), (d2, rms(f1.double() - f0.double()))):
        assert abs(got - want) <= 1e-5 * want, (got, want)


@pytest.mark.parametrize('n', SIZES)
@pytest.mark.parametrize('method', ['dopri5', 'bosh3', 'adaptive_heun'])
def test_dense_output_vs_float64(pkg, n, method):
    tab = pkg.ode.TABLEAUX[method]
    S = len(tab.alpha) + 1
    y0, y1, ks = randn(n, 1), randn(n, 2), [randn(n, 10 + j) for j in range(S)]
    dt, x = 0.0625, 0.7
    mw = [float(torch.tensor(float(c) * dt, dtype=torch.float32)) for c in tab.c_mid]
    D = lambda t: t.double()
    coeff = ode_ref.interp_fit(D(y0), D(y1), D(y0) + sum(w * D(k) for w, k in zip(mw, ks)), D(ks[0]), D(ks[-1]), dt)
    want = ode_ref.interp_evaluate(coeff, x)
    mag = ode_ref.interp_evaluate([c.abs() for c in ode_ref.interp_fit(D(y0).abs(), D(y1).abs(), D(y0).abs() + sum(
        abs(w) * D(k).abs() for w, k in zip(mw, ks)), D(ks[0]).abs(), D(ks[-1]).abs(), dt)], x)
    out = pkg.ops.ode_dense_output(y0.to(dev()), y1.to(dev()), [k.to(dev()) for k in ks], mw, dt, x, out=nan_like(y0.to(dev())))
    err = (out.cpu().double() - want).abs()
    assert bool((err <= 64 * EPS * (mag + 32 * (D(y0).abs() + D(y1).abs()))).all()), float(err.max())
    # at x = 0 the quartic is y0 and at x = 1 it is y1, to the rounding of the terms
    for xx, end in ((0.0, y0), (1.0, y1)):
        o = pkg.ops.ode_dense_output(y0.to(dev()), y1.to(dev()), [k.to(dev()) for k in ks], mw, dt, xx).cpu()
        assert float((o - end).abs().max()) <= 1e-4 * max(1.0, float(end.abs().max()))


# ---------------------------------------------------------------------------------------------------------------------- step control
SHAPE = (3, 41, 7)                   # 861 elements: float4 body and a scalar tail


def analytic(lam):
    return lambda t, y: lam * y + torch.cos(3 * t)


# An explicit first step: the automatic one of a smooth problem is so small that its error ratio is fp32 rounding (the float64
# restatement sees ~0, the fp32 state ~1e-5), and the next step size, ratio^(-1 / order), follows that rounding.
@pytest.mark.parametrize('method, rtol, atol, options', [
    ('dopri5', 1e-5, 1e-6, dict(first_step=0.2)), ('bosh3', 1e-3, 1e-4, dict(first_step=0.1)),
    ('fehlberg2', 1e-3, 1e-4, dict(first_step=0.1)), ('adaptive_heun', 1e-3, 1e-4, dict(first_step=0.2, safety=0.5)),
    ('dopri5', 1e-6, 1e-7, dict(first_step=0.5, safety=0.8, ifactor=5.0, dfactor=0.3)),     # rejects its first step
])
def test_step_control_vs_float64_restatement(pkg, method, rtol, atol, options):
    lam = torch.linspace(-2.0, 0.5, math.prod(SHAPE)).reshape(SHAPE)
    y0 = randn(math.prod(SHAPE), 5).reshape(SHAPE)
    steps = 3
    stats = {}
    got = pkg.ode.odeint(analytic(lam.to(dev())), y0.to(dev()), steps, method, rtol=rtol, atol=atol, options=options, stats=stats)
    want = ode_ref.odeint(analytic(lam.double()), y0.double(), torch.linspace(0, 1, steps).double(), method=method, rtol=rtol, atol=atol,
                          options=options)[-1]
    log = ode_ref.LOG
    assert (stats['nfe'], stats['accepted'], stats['rejected']) == (log['nfe'], log['accepted'], log['rejected'])
    if options.get('first_step') == 0.5:
        assert stats['rejected'] >= 1 and stats['ratios'][0] > 1
    # the decisions are not near ties, so agreeing on them is not luck
    assert all(abs(r - 1) > 0.01 for r in stats['ratios']), stats['ratios']
    t32 = torch.tensor(log['times'], dtype=torch.float64).float().double()
    assert torch.allclose(torch.tensor(stats['times'], dtype=torch.float64), t32, rtol=1e-4, atol=1e-6)
    err = (got.cpu().double() - want).abs().max() / want.abs().max()
    assert float(err) < 2e-5, float(err)


def test_rk4_step_control_vs_float64_restatement(pkg):
    lam = torch.linspace(-2.0, 0.5, math.prod(SHAPE)).reshape(SHAPE)
    y0 = randn(math.prod(SHAPE), 6).reshape(SHAPE)
    stats = {}
    got = pkg.ode.odeint(analytic(lam.to(dev())), y0.to(dev()), 9, 'rk4', stats=stats)
    want = ode_ref.odeint(analytic(lam.double()), y0.double(), torch.linspace(0, 1, 9), method='rk4')[-1]
    assert stats['nfe'] == ode_ref.LOG['nfe'] == 32
    assert torch.allclose(torch.tensor(stats['times']), torch.tensor(ode_ref.LOG['times']), rtol=0, atol=0)
    assert float((got.cpu().double() - want).abs().max() / want.abs().max()) < 2e-5


def test_underflow_and_max_num_steps(pkg):
    fn, y0 = analytic(torch.ones(SHAPE, device=dev())), torch.ones(SHAPE, device=dev())
    with pytest.raises(AssertionError, match=r'max_num_steps exceeded \(2>=2\)'):
        pkg.ode.odeint(fn, y0, 2, 'bosh3', rtol=1e-9, atol=1e-9, options=dict(max_num_steps=2))
    nan_fn = lambda t, y: y * float('nan')
    with pytest.raises(AssertionError, match='underflow in dt nan'):
        pkg.ode.odeint(nan_fn, y0, 2, 'dopri5', rtol=1e-3, atol=1e-3, options=dict(first_step=0.1))


# ---------------------------------------------------------------------------------------------------------------------- whole model
SMALL = dict(dim=128, depth=2, heads=2)
# The function evaluations are bf16 transformers (rel-L2 ~1e-2 from the fp32 oracle), so the accept / reject decisions and step sizes
# agree only where the error ratios stand well above that noise: first steps large enough that no ratio is near 0 (where the step
# growth ratio^(-1 / order) follows the noise) and tolerances where no ratio is near 1 (the oracle's ratios are printed).
METHODS = [
    dict(method='rk4'),
    dict(method='dopri5', atol=1e-3, rtol=1e-3, options=dict(first_step=0.5)),
    dict(method='bosh3', atol=1e-2, rtol=1e-2, options=dict(first_step=0.5)),
    dict(method='fehlberg2', atol=1e-3, rtol=1e-3, options=dict(first_step=0.5)),
    dict(method='adaptive_heun', atol=1e-2, rtol=1e-2, options=dict(first_step=0.1)),
]


def counted(model):
    """count the model's transformer passes and record the times they see (one function evaluation = one pass per model at
    cfg_strength 1)"""
    log = dict(calls=0, times=[])
    inner = model.transformer_with_pred_head

    def wrapped(*a, **k):
        log['calls'] += 1
        log['times'].append(float(k['times']))
        return inner(*a, **k)

    model.transformer_with_pred_head = wrapped
    return log


@pytest.mark.parametrize('kw', METHODS, ids=[k['method'] for k in METHODS])
def test_sample_vs_oracle(pkg, kw, monkeypatch):
    model, sd = small_model(pkg, 60, **SMALL)
    model.odeint_kwargs = kw
    torch.manual_seed(61)
    cond, text, y0 = torch.randn(2, 24, 100), ['Hello', 'Goodbye'], torch.randn(2, 64, 100)
    log = counted(model)
    packs, pack_weights = [], pkg.ops.pack_weights
    monkeypatch.setattr(pkg.ops, 'pack_weights', lambda *a, **k: (packs.append(1), pack_weights(*a, **k))[1])
    outs = []
    for _ in range(2):
        with pkg.inject_randomness(y0=y0.to(dev())):
            outs.append(model.sample(cond.to(dev()), text=text, duration=64, steps=4, cfg_strength=1.0, return_raw_output=True))
    want = ode_ref.e2tts_sample(sd, O.TransformerCfg(**SMALL), cond, O.list_str_to_tensor(text), duration=64, y0=y0, steps=4,
                                cfg_strength=1.0, odeint_kwargs=kw)
    e = rel_l2(outs[0].cpu(), want)
    nfe = log['calls'] // 4                       # two sample() calls, a text and a null pass per evaluation
    print(f"{kw['method']}: rel-L2 {e:.3g}, nfe {nfe} (oracle {ode_ref.LOG['nfe']}), ratios {ode_ref.LOG['ratios']}")
    assert e < 5e-2
    assert nfe == ode_ref.LOG['nfe']
    assert len(packs) == 2                        # one weight-pack launch per sample()
    assert torch.equal(outs[0], outs[1])          # a repeated call: the same bits and the same evaluation times
    half = log['calls'] // 2
    assert log['times'][:half] == log['times'][half:]


def test_dopri5_ragged_durations_and_null_model(pkg):
    model, sd = small_model(pkg, 70, **SMALL)
    weak, wsd = small_model(pkg, 80, **SMALL)
    kw = dict(method='dopri5', atol=1e-3, rtol=1e-3, options=dict(first_step=0.5))
    model.odeint_kwargs = kw
    torch.manual_seed(71)
    cond, text = torch.randn(2, 20, 100), ['Hello', 'Goodbye then']
    duration = torch.tensor([48, 33])
    y0 = torch.randn(2, 48, 100)
    log = counted(model)
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(cond.to(dev()), text=text, duration=duration.to(dev()), steps=3, cfg_strength=1.5, cfg_null_model=weak,
                           return_raw_output=True)
    want = ode_ref.e2tts_sample(sd, O.TransformerCfg(**SMALL), cond, O.list_str_to_tensor(text), duration=duration, y0=y0, steps=3,
                                cfg_strength=1.5, odeint_kwargs=kw, null_sd=wsd)
    e = rel_l2(out.cpu(), want)
    print(f'dopri5 ragged + null model: rel-L2 {e:.3g}, nfe {log["calls"]} (oracle {ode_ref.LOG["nfe"]})')
    assert e < 5e-2
    assert log['calls'] == ode_ref.LOG['nfe']     # the null model's passes are its own
    # rows past each item's duration are part of the state (its norms run over them): the kernels' predictions there follow the oracle
    mask = O.lens_to_mask(duration, 48)
    assert rel_l2(out.cpu()[1][~mask[1]], want[1][~mask[1]]) < 5e-2


def test_automatic_first_step(pkg):
    """the initial step-size selection of a whole model: h0 = 0.01 d0 / d1 from the norms of y0 and f(t0, y0) agrees with the oracle's;
    the first step min(100 h0, h1) and the growth after it depend on f differenced over h0 and on an error ratio near 0, where the bf16
    evaluations' noise shows: the step counts of both sides are printed, not compared"""
    model, sd = small_model(pkg, 60, **SMALL)
    kw = dict(method='dopri5', atol=1e-3, rtol=1e-3)
    model.odeint_kwargs = kw
    torch.manual_seed(61)
    cond, text, y0 = torch.randn(2, 24, 100), ['Hello', 'Goodbye'], torch.randn(2, 64, 100)
    stats, odeint = {}, pkg.ode.odeint
    pkg.ode.odeint = lambda *a, **k: odeint(*a, **{**k, 'stats': stats})
    try:
        with pkg.inject_randomness(y0=y0.to(dev())):
            out = model.sample(cond.to(dev()), text=text, duration=64, steps=4, cfg_strength=1.0, return_raw_output=True)
    finally:
        pkg.ode.odeint = odeint
    want = ode_ref.e2tts_sample(sd, O.TransformerCfg(**SMALL), cond, O.list_str_to_tensor(text), duration=64, y0=y0, steps=4,
                                cfg_strength=1.0, odeint_kwargs=kw)
    log = ode_ref.LOG
    print(f"kernels: nfe {stats['nfe']}, times {[round(t, 5) for t in stats['times'][:4]]}, ratios {stats['ratios']}")
    print(f"oracle:  nfe {log['nfe']}, times {[round(t, 5) for t in log['times'][:4]]}, ratios {log['ratios']}")
    assert rel_l2(out.cpu(), want) < 5e-2
    assert abs(stats['times'][1] - log['times'][1]) <= 1e-2 * log['times'][1]      # t0 + h0
