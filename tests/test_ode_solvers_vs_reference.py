"""CPU: the Runge–Kutta methods of E2TTS.sample's `odeint_kwargs` (rk4, dopri5, bosh3, fehlberg2, adaptive_heun; SURVEY A.7). The
package's tableaux (exact fractions) against the order conditions and against the restatement of tests/ode_ref.py; the restated
solvers' dense output, convergence orders, step control and assertions; the oracle's sample with each method against what the original
E2TTS.sample computed (tests/golden/reference/ode_*.pt, tools/make_ode_golden.py); the parsing of odeint_kwargs; the C-ABI validation of
the solver kernels."""
import math
from fractions import Fraction as Fr
from functools import lru_cache

import pytest
import torch

import ode_ref
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg
from e2_tts_pytorch_b200 import ode

ORDERS = dict(rk4=4, dopri5=5, bosh3=3, fehlberg2=2, adaptive_heun=2)


# ---------------------------------------------------------------------------------------------------------------------- tableaux
@lru_cache(None)
def trees(n):
    """rooted trees with n nodes, each a sorted tuple of its subtrees"""
    return tuple(sorted(forests(n - 1))) if n > 1 else ((),)


@lru_cache(None)
def forests(m):
    """multisets of rooted trees with m nodes in all, as sorted tuples"""
    if m == 0:
        return frozenset({()})
    out = set()
    for k in range(1, m + 1):
        for t in trees(k):
            for f in forests(m - k):
                out.add(tuple(sorted(f + (t,))))
    return frozenset(out)


def size(t):
    return 1 + sum(size(c) for c in t)


def gamma(t):
    return size(t) * math.prod(gamma(c) for c in t)


def phi(A, t):
    """per stage i: the elementary weight prod over subtrees c of sum_j A[i][j] phi_j(c)"""
    subs = [phi(A, c) for c in t]
    return [math.prod(sum(A[i][j] * s[j] for j in range(len(A))) for s in subs) for i in range(len(A))]


def order_of(A, b, up_to):
    """the largest p <= up_to with sum_i b_i phi_i(t) = 1 / gamma(t) for every tree of order <= p"""
    for p in range(1, up_to + 1):
        if any(sum(bi * f for bi, f in zip(b, phi(A, t))) != Fr(1, gamma(t)) for t in trees(p)):
            return p - 1
    return up_to


def matrix(tab):
    S = len(tab.alpha) + 1
    return [[Fr(0)] * S] + [list(row) + [Fr(0)] * (S - len(row)) for row in tab.beta]


def test_tree_counts():
    assert [len(trees(n)) for n in range(1, 7)] == [1, 1, 2, 4, 9, 20]


@pytest.mark.parametrize('method', list(ode.TABLEAUX))
def test_tableau_consistency_and_order(method):
    tab = ode.TABLEAUX[method]
    S = len(tab.alpha) + 1
    assert len(tab.beta) == S - 1 and len(tab.c_sol) == len(tab.c_err) == len(tab.c_mid) == S
    for a, row in zip(tab.alpha, tab.beta):
        assert sum(row) == a                       # row sums are the stage nodes
    assert sum(tab.c_sol) == 1 and sum(tab.c_err) == 0
    A = matrix(tab)
    assert order_of(A, tab.c_sol, tab.order + 1) == tab.order    # exactly the nominal order
    c_hat = [s - e for s, e in zip(tab.c_sol, tab.c_err)]
    assert order_of(A, c_hat, tab.order) == dict(dopri5=4, bosh3=2, fehlberg2=1, adaptive_heun=1)[method]
    assert tab.fsal == (method in ('dopri5', 'bosh3'))


@pytest.mark.parametrize('method', list(ode.TABLEAUX))
def test_package_tableaux_match_the_restatement(method):
    tab, (alpha, beta, c_sol, c_err, c_mid, order) = ode.TABLEAUX[method], ode_ref.TABLEAUX[method]
    close = lambda u, v: len(u) == len(v) and all(abs(float(p) - q) <= 1e-15 * max(1.0, abs(q)) for p, q in zip(u, v))
    assert close(tab.alpha, alpha) and close(tab.c_sol, c_sol) and close(tab.c_err, c_err) and close(tab.c_mid, c_mid)
    assert all(close(r, q) for r, q in zip(tab.beta, beta)) and tab.order == order


def test_rk4_is_the_three_eighths_rule():
    """rk4_alt_step_func: nodes 0, 1/3, 2/3, 1, rows [1/3], [-1/3, 1], [1, -1, 1], weights 1/8, 3/8, 3/8, 1/8 — fourth order"""
    A = [[Fr(0)] * 4, [Fr(1, 3), 0, 0, 0], [Fr(-1, 3), Fr(1), 0, 0], [Fr(1), Fr(-1), Fr(1), 0]]
    assert order_of(A, [Fr(1, 8), Fr(3, 8), Fr(3, 8), Fr(1, 8)], 5) == 4


# ---------------------------------------------------------------------------------------------------------------------- solvers
def exp_sin(t):   # y' = cos(t) y, y(0) = 1
    return torch.exp(torch.sin(t))


def fn_exp_sin(t, y):
    return torch.cos(t) * y


def fixed_steps(method, n):
    """the restated solver at t = 1 with n equal steps: tolerances so loose every step is accepted and ifactor 1 keeps dt = 1/n"""
    y0 = torch.ones(3, dtype=torch.float64)
    if method == 'rk4':
        return ode_ref.odeint(fn_exp_sin, y0, torch.linspace(0, 1, n + 1, dtype=torch.float64), method='rk4')[-1]
    opts = dict(first_step=1.0 / n, ifactor=1.0)
    return ode_ref.odeint(fn_exp_sin, y0, torch.tensor([0.0, 1.0], dtype=torch.float64), method=method, rtol=1e9, atol=1e9, options=opts)[-1]


def test_dense_output_end_points():
    g = torch.Generator().manual_seed(0)
    y0, y1, ym, f0, f1 = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(5))
    coeff = ode_ref.interp_fit(y0, y1, ym, f0, f1, torch.tensor(0.37, dtype=torch.float64))
    assert torch.allclose(ode_ref.interp_evaluate(coeff, torch.tensor(0.0, dtype=torch.float64)), y0, rtol=0, atol=1e-13)
    assert torch.allclose(ode_ref.interp_evaluate(coeff, torch.tensor(1.0, dtype=torch.float64)), y1, rtol=0, atol=1e-12)


def test_dense_output_is_fourth_order_on_linear_problem():
    """dopri5's interpolant at the middle of one step of y' = -y: its local error falls as h^5"""
    errs = []
    for h in (0.2, 0.1, 0.05):
        y0 = torch.ones(1, dtype=torch.float64)
        y = ode_ref.odeint(lambda t, y: -y, y0, torch.tensor([0.0, h / 2], dtype=torch.float64), method='dopri5', rtol=1e9, atol=1e9,
                           options=dict(first_step=h))[-1]
        assert ode_ref.LOG['accepted'] == 1
        errs.append(abs(float(y) - math.exp(-h / 2)))
    rates = [math.log2(a / b) for a, b in zip(errs[:-1], errs[1:])]
    assert all(abs(r - 5) < 0.3 for r in rates), rates


@pytest.mark.parametrize('method', list(ORDERS))
def test_convergence_order(method):
    want = exp_sin(torch.tensor(1.0, dtype=torch.float64))
    n0 = 4 if method == 'dopri5' else 16
    errs = [float((fixed_steps(method, n) - want).abs().max()) for n in (n0, 2 * n0, 4 * n0)]
    rates = [math.log2(a / b) for a, b in zip(errs[:-1], errs[1:])]
    assert all(abs(r - ORDERS[method]) < 0.3 for r in rates), (method, errs, rates)


@pytest.mark.parametrize('method', list(ode.TABLEAUX))
def test_adaptive_error_falls_as_rtol_tightens(method):
    want = exp_sin(torch.tensor(1.0, dtype=torch.float64))
    errs, nfes = [], []
    for rtol in (1e-3, 1e-5, 1e-7):
        y = ode_ref.odeint(fn_exp_sin, torch.ones(4, dtype=torch.float64), torch.linspace(0, 1, 3, dtype=torch.float64), method=method,
                           rtol=rtol, atol=rtol * 1e-2)[-1]
        errs.append(float((y - want).abs().max()))
        nfes.append(ode_ref.LOG['nfe'])
    assert min(errs[:2]) > errs[2] and errs[2] < 1e-4, errs   # (at loose tolerances the error of an easy problem may not fall)
    assert nfes[0] < nfes[1] < nfes[2]


def test_rejected_first_step():
    y = ode_ref.odeint(fn_exp_sin, torch.ones(2, dtype=torch.float64), torch.tensor([0.0, 1.0], dtype=torch.float64), method='dopri5',
                       rtol=1e-8, atol=1e-10, options=dict(first_step=1.0))[-1]
    assert ode_ref.LOG['ratios'][0] > 1 and ode_ref.LOG['rejected'] >= 1
    assert float((y - exp_sin(torch.tensor(1.0, dtype=torch.float64))).abs().max()) < 1e-6


def test_underflow_and_max_num_steps_assertions():
    y0, t = torch.ones(2, dtype=torch.float64), torch.tensor([1.0, 2.0], dtype=torch.float64)
    with pytest.raises(AssertionError, match=r'underflow in dt 1e-20'):
        ode_ref.odeint(fn_exp_sin, y0, t, method='dopri5', rtol=1e-6, atol=1e-8, options=dict(first_step=1e-20))
    with pytest.raises(AssertionError, match=r'max_num_steps exceeded \(2>=2\)'):
        ode_ref.odeint(fn_exp_sin, y0, t, method='bosh3', rtol=1e-9, atol=1e-9, options=dict(max_num_steps=2))


def test_steps_one_returns_y0():
    y0 = torch.randn(5, dtype=torch.float64)
    for method in ORDERS:
        assert torch.equal(ode_ref.odeint(fn_exp_sin, y0, torch.zeros(1, dtype=torch.float64), method=method, rtol=1e-3, atol=1e-3)[-1], y0)


# ---------------------------------------------------------------------------------------------------------------------- oracle vs original
@pytest.mark.parametrize('name', list(ode_ref.ODE_CASES))
def test_sample_vs_reference(name):
    """the oracle's E2TTS.sample with each method (ragged durations, a cfg_null_model) against the original's E2TTS.sample on the same
    restated solver: the output, the number of function evaluations and the times they were made at"""
    c, g = ode_ref.ODE_CASES[name], RC.load('ode_' + name)
    cond = RC.randn((c['cond'][0], c['cond'][1], 100), c['seed'] + 1000)
    duration = c['duration'] if isinstance(c['duration'], int) else torch.tensor(c['duration'])
    null_sd = RC.state_dict('E2TTS', c['null_seed'], ode_ref.ODE_KW) if 'null_seed' in c else None
    got = ode_ref.e2tts_sample(RC.state_dict('E2TTS', c['seed'], ode_ref.ODE_KW), O.TransformerCfg(**ode_ref.ODE_KW), cond,
                               O.list_str_to_tensor(c['text']), duration=duration, y0=RC.randn(g['shape'], 3000 + c['seed']),
                               steps=c['steps'], cfg_strength=c['cfg_strength'], odeint_kwargs=c['odeint_kwargs'], null_sd=null_sd)
    log = ode_ref.LOG
    assert tuple(got.shape) == g['shape']
    assert RC.compact_rel_l2(got, g['out']) < 1e-4
    assert (log['nfe'], log['accepted'], log['rejected']) == (g['nfe'], g['accepted'], g['rejected'])
    # the step sizes follow the error ratios, which move with the last bits of the two fp32 computations
    assert torch.allclose(torch.tensor(log['times'], dtype=torch.float64), g['times'], rtol=0, atol=2e-3)


# ---------------------------------------------------------------------------------------------------------------------- parsing
SMALL = dict(dim=128, depth=2, heads=2)


def e2tts(**odeint_kwargs):
    return pkg.E2TTS(transformer=SMALL, use_vocos=False, odeint_kwargs=odeint_kwargs)


@pytest.mark.parametrize('kw', [
    dict(method='rk4'), dict(method='rk4', atol=1e-3, rtol=1e-3),
    *[dict(method=m) for m in ode.TABLEAUX],
    *[dict(method=m, atol=1e-4, rtol=1e-3) for m in ode.TABLEAUX],
    dict(method='dopri5', atol=1, rtol=0.0, options=dict(first_step=0.1, safety=0.8, ifactor=5.0, dfactor=0.1, max_num_steps=50)),
    dict(method='bosh3', options=dict(first_step=None)), dict(method='fehlberg2', options=None),
    dict(atol=1e-5, rtol=1e-5), dict(method='midpoint', atol=1e-5, rtol=1e-5), dict(method='euler'),
])
def test_supported_odeint_kwargs_construct(kw):
    m = e2tts(**kw)
    assert pkg.modules._parse_odeint_kwargs(m.odeint_kwargs)['method'] == kw.get('method', 'midpoint')


def test_parsed_defaults_are_torchdiffeqs():
    p = pkg.modules._parse_odeint_kwargs(dict(method='dopri5'))
    assert p == dict(method='dopri5', rtol=1e-7, atol=1e-9, options={})


@pytest.mark.parametrize('kw, key', [
    *[(dict(method=m), "'method'") for m in ('dopri8', 'heun2', 'heun3', 'explicit_adams', 'implicit_adams', 'fixed_adams',
                                              'scipy_solver', 'no_such_method')],
    *[(dict(method='dopri5', options={o: 0.1}), repr(o)) for o in ('step_size', 'step_t', 'jump_t', 'grid_points', 'perturb', 'norm',
                                                                    'min_step', 'max_step', 'interp')],
    (dict(method='rk4', options=dict(step_size=0.1)), "'step_size'"),
    (dict(method='dopri5', atol=torch.tensor(1e-3)), "'atol'"),
    (dict(method='bosh3', rtol=torch.full((4,), 1e-3)), "'rtol'"),
    (dict(method='dopri5', options=dict(first_step=torch.tensor(0.1))), "'first_step'"),
    (dict(method='adaptive_heun', event_fn=lambda t, y: y), "'event_fn'"),
])
def test_refused_odeint_kwargs_name_the_key(kw, key):
    with pytest.raises(NotImplementedError, match=key.replace('(', r'\(')) as e:
        e2tts(**kw)
    assert 'e2_tts.py:1122-1126' in str(e.value)


@pytest.mark.parametrize('kw', [dict(method='dopri5', rtol=-1e-3), dict(method='dopri5', atol=float('nan')),
                                dict(method='bosh3', options=dict(max_num_steps=0)), dict(method='bosh3', options=dict(safety=0.0))])
def test_out_of_range_values_raise(kw):
    with pytest.raises(ValueError):
        e2tts(**kw)


def test_sample_checks_reassigned_odeint_kwargs():
    """odeint_kwargs is a plain attribute: sample() parses it again before any work (and before needing a GPU)"""
    m = e2tts(method='dopri5')
    m.odeint_kwargs = dict(method='dopri8')
    with pytest.raises(NotImplementedError, match='dopri8'):
        m.sample(torch.randn(1, 8, 100), duration=16, return_raw_output=True)


# ---------------------------------------------------------------------------------------------------------------------- C ABI
def test_solver_entry_points_validate_without_gpu():
    """bad arguments are refused before the device is touched (placeholder pointers, never read)"""
    lib = pkg.lib
    lib.load()
    P = 256
    cases = [
        ('b200_ode_combine', 'b200_ode_combine_args', dict(y0=P, out=P, n=8, S=0), 'S=0'),
        ('b200_ode_combine', 'b200_ode_combine_args', dict(y0=P, out=P, n=8, S=8, **{f'k{j}': P for j in range(7)}), 'S=8'),
        ('b200_ode_combine', 'b200_ode_combine_args', dict(y0=P, out=P, n=8, S=2, k0=P), 'k1 is null'),
        ('b200_ode_combine', 'b200_ode_combine_args', dict(y0=P, out=P, n=0, S=1, k0=P), 'bad arguments'),
        ('b200_ode_step_error', 'b200_ode_step_error_args', dict(y0=P, y1=P, ws=P, ratio=P, n=8, S=1, k0=P, ws_len=0, rtol=1e-3), 'ws_len'),
        ('b200_ode_step_error', 'b200_ode_step_error_args', dict(y0=P, y1=P, ws=P, ratio=P, n=8, S=1, k0=P, ws_len=4, atol=-1.0), 'atol'),
        ('b200_ode_step_error', 'b200_ode_step_error_args', dict(y0=P, y1=P, ws=P, ratio=None, n=8, S=1, k0=P, ws_len=4), 'bad arguments'),
        ('b200_ode_scaled_norms', 'b200_ode_norms_args', dict(y0=P, b=P, ws=P, out=P, n=8, ws_len=70000), 'ws_len'),
        ('b200_ode_scaled_norms', 'b200_ode_norms_args', dict(y0=P, b=P, ws=P, out=P, n=8, ws_len=4, rtol=float('inf')), 'rtol'),
        ('b200_ode_scaled_norms', 'b200_ode_norms_args', dict(y0=P, ws=P, out=P, n=8, ws_len=4), 'bad arguments'),
        ('b200_ode_dense_output', 'b200_ode_dense_args', dict(y0=P, y1=P, out=P, n=8, S=2, k0=P, k1=P, x=float('nan')), 'x=nan'),
        ('b200_ode_dense_output', 'b200_ode_dense_args', dict(y0=P, y1=None, out=P, n=8, S=2, k0=P, k1=P), 'bad arguments'),
    ]
    n0 = lib.launch_count()
    for fn, struct, kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg.replace('(', r'\(')):
            lib.call(fn, lib.make_args(struct, **kw), None)
    assert lib.launch_count() == n0
    with pytest.raises(ValueError, match='8 sources'):
        pkg.ops.ode_combine(torch.zeros(4), [torch.zeros(4)] * 8, [1.0] * 8)
