"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) with the Runge–Kutta
`odeint_kwargs` of the cases of tests/ode_ref.py, its `odeint` being the restated torchdiffeq solvers of that module, and store what
E2TTS.sample computed as tests/golden/reference/ode_<case>.pt: the output in the record format of oracle/make_reference_golden.py,
the number of function evaluations, the accepted / rejected steps and the times the solver evaluated at. Writes only those files.
Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_ode_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import ode_ref  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference  # noqa: E402


def model(ref, seed):
    m = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **ode_ref.ODE_KW), use_vocos=False)
    m.load_state_dict(RC.state_dict('E2TTS', seed, ode_ref.ODE_KW))
    return m.eval()


def main():
    ref = load_reference()
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in ode_ref.ODE_CASES.items():
        m = model(ref, c['seed'])
        m.odeint_kwargs = c['odeint_kwargs']
        null = model(ref, c['null_seed']) if 'null_seed' in c else None
        cond = RC.randn((c['cond'][0], c['cond'][1], 100), c['seed'] + 1000)
        duration = c['duration'] if isinstance(c['duration'], int) else torch.tensor(c['duration'])
        ref.torch, ref.odeint = RC.noise(torch, 3000 + c['seed']), ode_ref.odeint   # y0 = the first draw of that generator
        try:
            with torch.no_grad():
                want = m.sample(cond, text=c['text'], duration=duration, steps=c['steps'], cfg_strength=c['cfg_strength'],
                                cfg_null_model=null, return_raw_output=True)
        finally:
            ref.torch, ref.odeint = torch, sys.modules['torchdiffeq'].odeint
        log = ode_ref.LOG
        obj = dict(shape=tuple(want.shape), out=RC.compact(want), nfe=log['nfe'], accepted=log['accepted'], rejected=log['rejected'],
                   times=torch.tensor(log['times'], dtype=torch.float64))
        path = os.path.join(RC.GOLDEN, f'ode_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB: nfe {log["nfe"]}, accepted {log["accepted"]}, '
              f'rejected {log["rejected"]}')


if __name__ == '__main__':
    main()
