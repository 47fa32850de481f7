"""E2TTS.sample() with each odeint method (midpoint, rk4 and the adaptive Runge–Kutta methods): per method the number of function
evaluations (NFE, each a text pass and a null pass at cfg_strength 1), accepted / rejected steps, wall time per sample(), time per NFE
against midpoint's, the solver kernels' share of the GPU kernel time (torch.profiler, a run of its own) and the rel-L2 distance to a
tight-tolerance dopri5 solution of the same ODE. Seeded random model; card name and power limit are read in the same run.

    python tools/ode_bench.py [--reps 3] [--out ode_bench.json] [--no-cfg5]

Shapes: d512 depth8 h8, B8, prompt 256 -> 1024 frames (rtol = atol = 1e-3), and the cfg5 shape of bench.py (d1024 depth24 h16, B8,
prompt 256 -> 2048 frames) for midpoint and dopri5 only, one timed call each.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import e2_tts_pytorch_b200 as pkg  # noqa: E402
from oracle import e2tts_oracle as O  # noqa: E402

TOL = dict(atol=1e-3, rtol=1e-3)
METHODS = {
    'midpoint': dict(method='midpoint'),
    'rk4': dict(method='rk4'),
    'dopri5': dict(method='dopri5', **TOL),
    'bosh3': dict(method='bosh3', **TOL),
    'fehlberg2': dict(method='fehlberg2', **TOL),
    'adaptive_heun': dict(method='adaptive_heun', **TOL),
}
TIGHT = dict(method='dopri5', atol=1e-6, rtol=1e-6)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f'{torch.cuda.get_device_name(0)} (power limit not readable)'


def build(dim, depth, heads, seq, seed=0):
    torch.manual_seed(seed)
    random.seed(seed)
    m = pkg.E2TTS(transformer=dict(dim=dim, depth=depth, heads=heads, dropout=0., max_seq_len=seq), use_vocos=False)
    m.load_state_dict(O.randomize_zero_init({k: v.clone() for k, v in m.state_dict().items()}, seed=seed + 1, dyn_scale=0.05))
    return m.cuda()


class Counter:
    """transformer passes of sample() and the adaptive solver's step statistics"""

    def __init__(self, model):
        self.calls, self.stats = 0, {}
        inner, odeint = model.transformer_with_pred_head, pkg.ode.odeint

        def count(*a, **k):
            self.calls += 1
            return inner(*a, **k)

        def solve(*a, **k):
            return odeint(*a, **{**k, 'stats': self.stats})

        model.transformer_with_pred_head = count
        pkg.ode.odeint = solve


def run(model, inp, kw, steps):
    model.odeint_kwargs = kw
    with pkg.inject_randomness(y0=inp['y0']):
        return model.sample(inp['cond'], text=inp['text'], duration=inp['duration'], steps=steps, cfg_strength=1.0, return_raw_output=True)


def timed(model, inp, kw, steps, reps):
    run(model, inp, kw, steps)                      # warm-up: every shape of the timed calls
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = run(model, inp, kw, steps)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return out, ts[len(ts) // 2]


def solver_share(model, inp, kw, steps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, inp, kw, steps)
        torch.cuda.synchronize()
    total = solver = 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        if e.device_type == torch.autograd.DeviceType.CUDA:   # kernels only (host ops would count their kernels twice)
            total += t
            if 'ode_' in e.key:
                solver += t
    return solver / total if total else float('nan'), solver / 1e3


def bench(label, dim, depth, heads, seq, methods, reps, steps=32):
    model = build(dim, depth, heads, seq)
    g = torch.Generator().manual_seed(1)
    B, prompt = 8, 256
    inp = dict(cond=torch.randn(B, prompt, 100, generator=g).cuda(), y0=torch.randn(B, seq, 100, generator=g).cuda(),
               text=['Hello there'] * B, duration=seq)
    counter = Counter(model)
    ref = run(model, inp, TIGHT, steps).float()
    ref_nfe = counter.calls // 2
    rows, mid_per_nfe = [], None
    for name in methods:
        kw = METHODS[name]
        out, wall = timed(model, inp, kw, steps, reps)
        counter.calls, counter.stats = 0, {}
        run(model, inp, kw, steps)
        nfe = counter.calls // 2
        share, solver_ms = solver_share(model, inp, kw, steps)
        per_nfe = wall / nfe
        mid_per_nfe = per_nfe if name == 'midpoint' else mid_per_nfe
        row = dict(shape=label, method=name, nfe=nfe, accepted=counter.stats.get('accepted'), rejected=counter.stats.get('rejected'),
                   wall_s=round(wall, 4), ms_per_nfe=round(1e3 * per_nfe, 3),
                   per_nfe_vs_midpoint=round(per_nfe / mid_per_nfe, 4) if mid_per_nfe else None,
                   solver_kernel_share=share, solver_kernel_ms=round(solver_ms, 3),
                   rel_l2_vs_tight_dopri5=float((out.float() - ref).norm() / ref.norm()))
        print(json.dumps(row), flush=True)
        rows.append(row)
    del model
    torch.cuda.empty_cache()
    return dict(shape=label, tight_dopri5_nfe=ref_nfe, rows=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-cfg5', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'ode_bench measures on the GPU'
    res = dict(card=card(), tolerance=TOL, cfg_strength=1.0, results=[])
    print('card (name, power limit, max SM clock):', res['card'], flush=True)
    res['results'].append(bench('d512 depth8 h8, B8, 256 -> 1024 frames', 512, 8, 8, 1024, list(METHODS), a.reps))
    if not a.no_cfg5:
        res['results'].append(bench('cfg5: d1024 depth24 h16, B8, 256 -> 2048 frames', 1024, 24, 16, 2048, ['midpoint', 'dopri5'], 1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
