"""torchdiffeq 0.2.x's Runge–Kutta solvers restated in plain PyTorch (SURVEY.md Appendix A.7), in the dtype of the state: the
fixed-grid 'rk4' (rk4_alt_step_func, the 3/8 rule) and the adaptive 'dopri5', 'bosh3', 'fehlberg2' and 'adaptive_heun' of
RKAdaptiveStepsizeODESolver; 'midpoint' / 'euler' are the leaf of oracle/ref_leaves/torchdiffeq.py. TEST INFRASTRUCTURE: the package's
solver (e2-tts-pytorch_b200/ode.py) is held to this module, and tools/make_ode_golden.py runs the original E2TTS.sample on it.

Also here: `e2tts_sample`, the oracle's E2TTS.sample (oracle/e2tts_oracle.py) with any of these methods and a `cfg_null_model`, and
the cases of the goldens tests/golden/reference/ode_*.pt."""
import math

import torch
import torch.nn.functional as F

from oracle import e2tts_oracle as O
from oracle.ref_leaves.torchdiffeq import odeint as fixed_grid_odeint

# (alpha, beta rows, c_sol, c_error, c_mid, order), as torchdiffeq writes them
TABLEAUX = {
    'dopri5': (
        [1 / 5, 3 / 10, 4 / 5, 8 / 9, 1., 1.],
        [[1 / 5],
         [3 / 40, 9 / 40],
         [44 / 45, -56 / 15, 32 / 9],
         [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729],
         [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656],
         [35 / 384, 0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84]],
        [35 / 384, 0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84, 0],
        [35 / 384 - 1951 / 21600, 0, 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720, -2187 / 6784 - -12231 / 42400,
         11 / 84 - 649 / 6300, -1. / 60.],
        [6025192743 / 30085553152 / 2, 0, 51252292925 / 65400821598 / 2, -2691868925 / 45128329728 / 2,
         187940372067 / 1594534317056 / 2, -1776094331 / 19743644256 / 2, 11237099 / 235043384 / 2],
        5),
    'bosh3': ([1 / 2, 3 / 4, 1.], [[1 / 2], [0., 3 / 4], [2 / 9, 1 / 3, 4 / 9]], [2 / 9, 1 / 3, 4 / 9, 0.],
              [2 / 9 - 7 / 24, 1 / 3 - 1 / 4, 4 / 9 - 1 / 3, -1 / 8], [0., 0.5, 0., 0.], 3),
    'fehlberg2': ([1 / 2, 1.], [[1 / 2], [1 / 256, 255 / 256]], [1 / 512, 255 / 256, 1 / 512], [-1 / 512, 0, 1 / 512], [0., 0.5, 0.], 2),
    'adaptive_heun': ([1.], [[1.]], [0.5, 0.5], [0.5, -0.5], [0.5, 0.], 2),
}


def rms(x):
    return float(x.abs().pow(2).mean().sqrt())


def interp_fit(y0, y1, y_mid, f0, f1, dt):
    """the quartic's coefficients [e, d, c, b, a] of the dense output (torchdiffeq interp._interp_fit)"""
    return [y0, dt * f0, dt * (f1 - 4 * f0) - 11 * y0 - 5 * y1 + 16 * y_mid, dt * (5 * f0 - 3 * f1) + 18 * y0 + 14 * y1 - 32 * y_mid,
            2 * dt * (f1 - f0) - 8 * (y1 + y0) + 16 * y_mid]


def interp_evaluate(coeff, x):
    """e + x d + x^2 c + x^3 b + x^4 a, powers of x formed by repeated products (torchdiffeq interp._interp_evaluate)"""
    total, xp = coeff[0] + x * coeff[1], x
    for c in coeff[2:]:
        xp = xp * x
        total = total + xp * c
    return total


class Log(dict):
    """what a solve did: nfe, the times fn saw (as floats), accepted / rejected steps and every error ratio"""

    def __init__(self):
        super().__init__(nfe=0, times=[], accepted=0, rejected=0, ratios=[])


def _rk4(fn, y0, t):
    ys, y = [y0], y0
    for t0, t1 in zip(t[:-1], t[1:]):
        dt = t1 - t0
        k1 = fn(t0, y)
        k2 = fn(t0 + dt * (1 / 3), y + dt * k1 * (1 / 3))
        k3 = fn(t0 + dt * (2 / 3), y + dt * (k2 - k1 * (1 / 3)))
        k4 = fn(t1, y + dt * (k1 - k2 + k3))
        y = y + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
        ys.append(y)
    return ys


def _adaptive(fn, y0, t, method, rtol, atol, first_step=None, safety=0.9, ifactor=10.0, dfactor=0.2, max_num_steps=2 ** 31 - 1):
    alpha, beta, c_sol, c_err, c_mid, order = TABLEAUX[method]
    dt_ = y0.dtype
    T = lambda v: torch.tensor(v, dtype=dt_)                        # a host value cast to the state's dtype (_runge_kutta_step)
    c_sol_t, c_err_t, c_mid_t = T(c_sol), T(c_err), T(c_mid)
    beta_t = [T(b) for b in beta]
    fsal = c_sol[-1] == 0 and list(c_sol[:-1]) == list(beta[-1])
    ts = [float(v) for v in t.double()]                              # step control in float64

    f0 = fn(T(ts[0]), y0)
    if first_step is None:                                          # _select_initial_step(order - 1): exponent 1 / order
        scale = atol + y0.abs() * rtol
        d0, d1 = rms(y0 / scale), rms(f0 / scale)
        h0 = 1e-6 if d0 < 1e-5 or d1 < 1e-5 else 0.01 * d0 / d1
        f1 = fn(T(ts[0] + h0), y0 + T(h0) * f0)
        d2 = rms((f1 - f0) / scale) / h0
        h1 = max(1e-6, h0 * 1e-3) if d1 <= 1e-15 and d2 <= 1e-15 else (0.01 / max(d1, d2)) ** (1.0 / order)
        dt = min(100 * h0, h1)
    else:
        dt = float(first_step)

    y, t_start, t_end, coeff = y0, ts[0], ts[0], None
    out = [y0]
    for next_t in ts[1:]:
        n_steps = 0
        while next_t > t_end:
            assert n_steps < max_num_steps, 'max_num_steps exceeded ({}>={})'.format(n_steps, max_num_steps)
            t0 = t_end
            t1 = t0 + dt
            assert t0 + dt > t0, 'underflow in dt {}'.format(dt)
            t0c, dtc, t1c = T(t0), T(dt), T(t1)
            k = [f0]
            for a, b in zip(alpha, beta_t):
                ti = t1c if a == 1 else t0c + T(a) * dtc
                yi = y + torch.stack(k, -1).matmul(b * dtc)
                k.append(fn(ti, yi))
            K = torch.stack(k, -1)
            y1 = yi if fsal else y + K.matmul(dtc * c_sol_t)
            err = K.matmul(dtc * c_err_t)
            ratio = rms(err / (atol + rtol * torch.max(y.abs(), y1.abs())))
            LOG['ratios'].append(ratio)
            if ratio <= 1:
                coeff = interp_fit(y, y1, y + K.matmul(dtc * c_mid_t), k[0], k[-1], dtc)
                t_start, t_end, y, f0 = t0, t1, y1, k[-1]
                LOG['accepted'] += 1
            else:
                t_start, t_end = t0, t0
                LOG['rejected'] += 1
            if ratio == 0:
                dt = dt * ifactor
            elif math.isnan(ratio):
                dt = math.nan
            else:
                dt = dt * min(ifactor, max(safety / ratio ** (1.0 / order), 1.0 if ratio < 1 else dfactor))
            n_steps += 1
        out.append(interp_evaluate(coeff, T((next_t - t_start) / (t_end - t_start))))
    return out


LOG = Log()


def odeint(fn, y0, t, *, method='midpoint', rtol=1e-7, atol=1e-9, options=None):
    """torchdiffeq.odeint(fn, y0, t, method=..., rtol=..., atol=..., options=...) -> the trajectory at t; LOG records the solve
    (reset on every call)."""
    if method in ('midpoint', 'euler'):
        return fixed_grid_odeint(fn, y0, t, method=method)
    LOG.__init__()

    def f(tt, y):
        LOG['nfe'] += 1
        LOG['times'].append(float(tt))
        return fn(tt, y)

    if method == 'rk4':
        return torch.stack(_rk4(f, y0, t))
    assert method in TABLEAUX, method
    return torch.stack(_adaptive(f, y0, t, method, float(rtol), float(atol), **(options or {})))


@torch.no_grad()
def e2tts_sample(sd, cfg, cond, text, *, duration, y0, steps=32, cfg_strength=1.0, lens=None, max_duration=4096, odeint_kwargs=None,
                 null_sd=None):
    """O.e2tts_sample (E2TTS.sample :1332-1431 with y0 injected) solved by `odeint` with `odeint_kwargs`; null_sd = the state dict of
    a `cfg_null_model` (:1318-1321: its prediction WITH text is the null prediction)."""
    b, cn, _ = cond.shape
    if lens is None:
        lens = torch.full((b,), cn, dtype=torch.long)
    if text is not None:
        lens = torch.maximum((text != -1).sum(-1), lens)
    cond_mask = O.lens_to_mask(lens, int(lens.amax()))
    if isinstance(duration, int):
        duration = torch.full((b,), duration, dtype=torch.long)
    duration = torch.maximum(lens + 1, duration).clamp(max=max_duration)
    md = int(duration.amax())
    cond = F.pad(cond, (0, 0, 0, md - cn))
    cond_mask = F.pad(cond_mask, (0, md - cond_mask.shape[-1]), value=False)[..., None]
    mask = O.lens_to_mask(duration, md)
    step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))

    def fn(tt, y):
        if null_sd is None:
            return O.cfg_pred(sd, cfg, y, step_cond, tt, mask, text, cfg_strength)
        pred = O.transformer_with_pred_head(sd, cfg, y, step_cond, tt, mask, text, False)
        if cfg_strength < 1e-5:
            return pred
        null = O.transformer_with_pred_head(null_sd, cfg, y, step_cond, tt, mask, text, False)
        _, orth = O.project(pred - null, pred)
        return pred + orth * cfg_strength

    y = odeint(fn, y0, torch.linspace(0, 1, steps), **(odeint_kwargs or dict(method='midpoint')))[-1]
    return torch.where(cond_mask, cond, y)


# Goldens of the original E2TTS.sample on this module's solvers (tools/make_ode_golden.py): weights seed (null_seed: a cfg_null_model),
# cond (batch, frames), text, duration, steps, cfg_strength, odeint_kwargs; y0 = first draw of generator 3000 + seed
ODE_KW = dict(dim=128, depth=2, heads=2)
ODE_CASES = {
    'rk4': dict(seed=81, cond=(2, 20), text=['Hello', 'Goodbye'], duration=40, steps=4, cfg_strength=1.0, odeint_kwargs=dict(method='rk4')),
    'dopri5_ragged_null': dict(seed=82, null_seed=83, cond=(2, 20), text=['Hello', 'Goodbye then'], duration=[40, 29], steps=3,
                               cfg_strength=1.5, odeint_kwargs=dict(method='dopri5', atol=1e-3, rtol=1e-3)),
    'dopri5_options': dict(seed=84, cond=(2, 16), text=['abc', 'de'], duration=32, steps=2, cfg_strength=1.0,
                           odeint_kwargs=dict(method='dopri5', atol=1e-4, rtol=1e-3,
                                              options=dict(first_step=0.25, safety=0.8, ifactor=4.0, dfactor=0.3, max_num_steps=100))),
    'bosh3': dict(seed=85, cond=(2, 16), text=['Hello', 'x'], duration=[32, 24], steps=2, cfg_strength=1.0,
                  odeint_kwargs=dict(method='bosh3', atol=1e-3, rtol=1e-3)),
    'fehlberg2': dict(seed=86, cond=(2, 16), text=['Hello', 'x'], duration=32, steps=5, cfg_strength=0.0,
                      odeint_kwargs=dict(method='fehlberg2', atol=1e-2, rtol=1e-2)),
    'adaptive_heun': dict(seed=87, cond=(2, 16), text=['Hello', 'x'], duration=[28, 32], steps=2, cfg_strength=1.0,
                          odeint_kwargs=dict(method='adaptive_heun', atol=1e-2, rtol=1e-2)),
}
