"""Runge–Kutta solvers of E2TTS.sample's `odeint_kwargs` besides its fixed-grid midpoint / euler loop (e2_tts.py:1421 calls
torchdiffeq's odeint): torchdiffeq 0.2.x's fixed-grid 'rk4' (rk4_alt_step_func, the 3/8 rule) and the embedded adaptive methods of its
RKAdaptiveStepsizeODESolver, 'dopri5', 'bosh3', 'fehlberg2' and 'adaptive_heun' (SURVEY.md Appendix A.7). The tableaux and the step
control live here on the host; every pass over the ODE state runs in the b200_ode_* kernels (ops.ode_*).

The state is the whole padded [B, max_duration, C] fp32 tensor, so one step size serves the batch and every norm runs over every
element. Step-control times are float64 host floats; stage times, step sizes and tableau weights are rounded to fp32 where torchdiffeq
casts them to the state's dtype. An adaptive step reads back its fp32 error ratio (one 4-byte scalar, where torchdiffeq synchronises
too) and copies the step's stage times to the device right after it, while the device is idle.
"""
from __future__ import annotations

import math
from fractions import Fraction as Fr
from typing import NamedTuple

import numpy as np
import torch

from . import ops

F32 = np.float32
WS_LEN = 1024        # reduction blocks of the error / norm passes (ops.ode_step_error, ops.ode_scaled_norms)


class Tableau(NamedTuple):
    """Butcher tableau of an embedded method as torchdiffeq holds it: stage nodes alpha, stage rows beta, solution weights c_sol,
    error weights c_err (= c_sol - the embedded solution's weights), dense-output midpoint weights c_mid, and the order that sets the
    step-size exponent."""
    alpha: tuple
    beta: tuple
    c_sol: tuple
    c_err: tuple
    c_mid: tuple
    order: int

    @property
    def fsal(self):
        """first-same-as-last: the last stage input is the solution (torchdiffeq: c_sol[-1] == 0 and c_sol[:-1] == beta[-1])"""
        return self.c_sol[-1] == 0 and tuple(self.c_sol[:-1]) == tuple(self.beta[-1])


_DP_SOL = (Fr(35, 384), Fr(0), Fr(500, 1113), Fr(125, 192), Fr(-2187, 6784), Fr(11, 84), Fr(0))
_DP_HAT = (Fr(1951, 21600), Fr(0), Fr(22642, 50085), Fr(451, 720), Fr(-12231, 42400), Fr(649, 6300), Fr(1, 60))
TABLEAUX = {
    'dopri5': Tableau(
        alpha=(Fr(1, 5), Fr(3, 10), Fr(4, 5), Fr(8, 9), Fr(1), Fr(1)),
        beta=((Fr(1, 5),),
              (Fr(3, 40), Fr(9, 40)),
              (Fr(44, 45), Fr(-56, 15), Fr(32, 9)),
              (Fr(19372, 6561), Fr(-25360, 2187), Fr(64448, 6561), Fr(-212, 729)),
              (Fr(9017, 3168), Fr(-355, 33), Fr(46732, 5247), Fr(49, 176), Fr(-5103, 18656)),
              _DP_SOL[:6]),
        c_sol=_DP_SOL,
        c_err=tuple(s - h for s, h in zip(_DP_SOL, _DP_HAT)),
        c_mid=tuple(Fr(1, 2) * m for m in (Fr(6025192743, 30085553152), Fr(0), Fr(51252292925, 65400821598),
                                          Fr(-2691868925, 45128329728), Fr(187940372067, 1594534317056),
                                          Fr(-1776094331, 19743644256), Fr(11237099, 235043384))),
        order=5),
    'bosh3': Tableau(
        alpha=(Fr(1, 2), Fr(3, 4), Fr(1)),
        beta=((Fr(1, 2),), (Fr(0), Fr(3, 4)), (Fr(2, 9), Fr(1, 3), Fr(4, 9))),
        c_sol=(Fr(2, 9), Fr(1, 3), Fr(4, 9), Fr(0)),
        c_err=(Fr(2, 9) - Fr(7, 24), Fr(1, 3) - Fr(1, 4), Fr(4, 9) - Fr(1, 3), Fr(-1, 8)),
        c_mid=(Fr(0), Fr(1, 2), Fr(0), Fr(0)),
        order=3),
    'fehlberg2': Tableau(
        alpha=(Fr(1, 2), Fr(1)),
        beta=((Fr(1, 2),), (Fr(1, 256), Fr(255, 256))),
        c_sol=(Fr(1, 512), Fr(255, 256), Fr(1, 512)),
        c_err=(Fr(-1, 512), Fr(0), Fr(1, 512)),
        c_mid=(Fr(0), Fr(1, 2), Fr(0)),
        order=2),
    'adaptive_heun': Tableau(
        alpha=(Fr(1),),
        beta=((Fr(1),),),
        c_sol=(Fr(1, 2), Fr(1, 2)),
        c_err=(Fr(1, 2), Fr(-1, 2)),
        c_mid=(Fr(1, 2), Fr(0)),
        order=2),
}
ADAPTIVE_METHODS = tuple(TABLEAUX)
# torchdiffeq's defaults for keys a user's odeint_kwargs leaves out (odeint signature; RKAdaptiveStepsizeODESolver.__init__)
DEFAULT_TOL = dict(rtol=1e-7, atol=1e-9)
DEFAULT_OPTIONS = dict(first_step=None, safety=0.9, ifactor=10.0, dfactor=0.2, max_num_steps=2 ** 31 - 1)


def _f32(v):
    return F32(float(v))


def _weights(coefs, dt32):
    """tableau entries times the fp32 step, each product rounded to fp32 (torchdiffeq: `beta_i * dt` on fp32 tensors)"""
    return [float(F32(_f32(c) * dt32)) for c in coefs]


def _nonzero(ks, *weight_lists):
    """drop the sources whose weights are all exactly zero (they add nothing and cost a read of the state)"""
    keep = [j for j in range(len(ks)) if any(w[j] != 0.0 for w in weight_lists)]
    return [ks[j] for j in keep], *([w[j] for j in keep] for w in weight_lists)


def grid(steps):
    """torchdiffeq's output grid t = linspace(0, 1, steps) in fp32 (e2_tts.py:1419), as host floats"""
    return torch.linspace(0, 1, steps).tolist()


def rk4_times(steps):
    """the stage times of fixed-grid rk4 on t = linspace(0, 1, steps), four per step, fp32 as on torchdiffeq's fp32 grid"""
    ts = [F32(t) for t in grid(steps)]
    third, two_thirds = F32(1 / 3), F32(2 / 3)
    times = []
    for t0, t1 in zip(ts[:-1], ts[1:]):
        dt = F32(t1 - t0)
        times += [t0, F32(t0 + F32(dt * third)), F32(t0 + F32(dt * two_thirds)), t1]
    return times


def rk4(fn, y0, steps, stats=None, tt=None):
    """Fixed-grid rk4 (torchdiffeq rk4_alt_step_func, the 3/8 rule) on t = linspace(0, 1, steps): per step
    k1 = f(t0, y0), k2 = f(t0 + dt/3, y0 + dt k1/3), k3 = f(t0 + 2dt/3, y0 + dt (k2 - k1/3)), k4 = f(t1, y0 + dt (k1 - k2 + k3)),
    y1 = y0 + (k1 + 3 (k2 + k3) + k4) dt/8; times and dt in fp32 as on torchdiffeq's fp32 grid. tt: rk4_times(steps) already on the
    device (a CUDA-graph capture cannot copy them there)."""
    ts = [F32(t) for t in grid(steps)]
    third = F32(1 / 3)
    times = rk4_times(steps)
    if tt is None:
        tt = torch.tensor(times, dtype=torch.float32).to(y0.device)   # every stage time in one copy: no host synchronisation per step
    y, stage, ring = y0, torch.empty_like(y0), [torch.empty_like(y0), torch.empty_like(y0)]
    for i, (t0, t1) in enumerate(zip(ts[:-1], ts[1:])):
        dt = F32(t1 - t0)
        w3, d = float(F32(dt * third)), float(dt)
        k1 = fn(tt[4 * i], y)
        k2 = fn(tt[4 * i + 1], ops.ode_combine(y, [k1], [w3], out=stage))
        k3 = fn(tt[4 * i + 2], ops.ode_combine(y, [k1, k2], [-w3, d], out=stage))
        k4 = fn(tt[4 * i + 3], ops.ode_combine(y, [k1, k2, k3], [d, -d, d], out=stage))
        e, m = float(F32(dt * F32(0.125))), float(F32(dt * F32(0.375)))
        y = ops.ode_combine(y, [k1, k2, k3, k4], [e, m, m, e], out=ring[i % 2])
    if stats is not None:
        stats.update(nfe=4 * (len(ts) - 1), times=[float(t) for t in times])
    return y


def _optimal_step_size(dt, ratio, safety, ifactor, dfactor, order):
    """torchdiffeq rk_common._optimal_step_size in float64 (a NaN ratio gives a NaN step, which the next step's underflow check
    reports, as torchdiffeq's tensors do)"""
    if ratio == 0:
        return dt * ifactor
    if math.isnan(ratio):
        return math.nan
    if ratio < 1:
        dfactor = 1.0
    return dt * min(ifactor, max(safety / ratio ** (1.0 / order), dfactor))


def adaptive(fn, y0, steps, method, rtol, atol, first_step=None, safety=0.9, ifactor=10.0, dfactor=0.2, max_num_steps=2 ** 31 - 1,
             stats=None):
    """torchdiffeq's RKAdaptiveStepsizeODESolver on t = linspace(0, 1, steps): returns the dense output at t = 1 of the last
    accepted step. Steps are not clipped at the output times; `max_num_steps` counts steps per output interval. Raises
    AssertionError with torchdiffeq's messages on an underflowing step size or too many steps."""
    tab = TABLEAUX[method]
    S = len(tab.alpha) + 1
    dev = y0.device
    ts = grid(steps)
    ws = torch.empty(2 * WS_LEN, dtype=torch.float64, device=dev)
    scal = torch.empty(2, dtype=torch.float32, device=dev)
    ring = [torch.empty_like(y0), torch.empty_like(y0)]   # y1 of the step being taken / y0 of the state, alternating on accept
    stage = torch.empty_like(y0)
    log = dict(nfe=0, accepted=0, rejected=0, ratios=[], times=[])

    def f(t32, y, t_dev=None):
        log['nfe'] += 1
        log['times'].append(float(t32))
        return fn(torch.tensor(float(t32), dtype=torch.float32).to(dev) if t_dev is None else t_dev, y)

    t0 = ts[0]
    f0 = f(_f32(t0), y0)
    if first_step is None:   # _select_initial_step with order - 1, i.e. the exponent 1 / order
        d0, d1 = ops.ode_scaled_norms(y0, y0, f0, None, atol, rtol, ws, scal).tolist()
        h0 = 1e-6 if d0 < 1e-5 or d1 < 1e-5 else 0.01 * d0 / d1
        f1 = f(_f32(t0 + h0), ops.ode_combine(y0, [f0], [float(_f32(h0))], out=stage))
        d2 = ops.ode_scaled_norms(y0, None, f1, f0, atol, rtol, ws, scal)[1].item() / h0
        if d1 <= 1e-15 and d2 <= 1e-15:
            h1 = max(1e-6, h0 * 1e-3)
        else:
            h1 = (0.01 / max(d1, d2)) ** (1.0 / tab.order)
        dt = min(100 * h0, h1)
        del f1
    else:
        dt = float(first_step)

    y, t1, last, spare = y0, t0, None, 0
    for next_t in ts[1:]:
        n_steps = 0
        while next_t > t1:
            if n_steps >= max_num_steps:
                raise AssertionError(f'max_num_steps exceeded ({n_steps}>={max_num_steps})')
            t0 = t1
            if not t0 + dt > t0:
                raise AssertionError(f'underflow in dt {dt}')
            t_end = t0 + dt
            t0_32, dt32, t1_32 = _f32(t0), _f32(dt), _f32(t_end)
            y1 = ring[spare]
            stage_t = [t1_32 if a == 1 else F32(t0_32 + F32(_f32(a) * dt32)) for a in tab.alpha]
            tt = torch.tensor(stage_t, dtype=torch.float32).to(dev)   # the device is idle here (after the ratio read back)
            ks = [f0]
            for i, row in enumerate(tab.beta):
                out = y1 if (tab.fsal and i == S - 2) else stage
                src, w = _nonzero(ks, _weights(row, dt32))
                ks.append(f(stage_t[i], ops.ode_combine(y, src, w, out=out), tt[i]))
            err_w = _weights(tab.c_err, dt32)
            sol_w = None if tab.fsal else _weights(tab.c_sol, dt32)
            src, *wl = _nonzero(ks, err_w, *([sol_w] if sol_w else []))
            ops.ode_step_error(y, src, wl[0], y1, atol, rtol, ws, scal[:1], sol_w=wl[1] if sol_w else None)
            ratio = float(scal[0].item())   # the accept / reject decision: one 4-byte read back per step
            log['ratios'].append(ratio)
            n_steps += 1
            if ratio <= 1:
                last = (y, y1, ks, dt32, t0, t_end)
                y, f0, t1, spare = y1, ks[-1], t_end, 1 - spare
                log['accepted'] += 1
            else:
                t1 = t0
                log['rejected'] += 1
            dt = _optimal_step_size(dt, ratio, safety, ifactor, dfactor, tab.order)
    if stats is not None:
        stats.update(log)
    if last is None:          # steps == 1: the trajectory is y0 alone
        return y0
    ya, yb, ks, dt32, ta, tb = last
    x = _f32((ts[-1] - ta) / (tb - ta))
    return ops.ode_dense_output(ya, yb, ks, _weights(tab.c_mid, dt32), float(dt32), float(x))


def odeint(fn, y0, steps, method, rtol=DEFAULT_TOL['rtol'], atol=DEFAULT_TOL['atol'], options=None, stats=None):
    """The state at t = 1 of torchdiffeq.odeint(fn, y0, linspace(0, 1, steps), method=method, rtol=rtol, atol=atol,
    options=options) for method 'rk4' or one of ADAPTIVE_METHODS. `stats`, a dict, receives nfe, the evaluation times and, for the
    adaptive methods, accepted / rejected step counts and every error ratio."""
    if method == 'rk4':
        return rk4(fn, y0, steps, stats)
    return adaptive(fn, y0, steps, method, float(rtol), float(atol), **{**DEFAULT_OPTIONS, **(options or {})}, stats=stats)
