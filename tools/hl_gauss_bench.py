"""The HL-Gauss classification head (DurationPredictor(hl_gauss_loss=dict(min_value=0, max_value=4096, num_bins=1024),
use_regression=False)) against the regression head of bench.py's cfg4: DurationPredictor d512 depth 8 h8, B32 x 1024 frames, one
GraphedTrainStep (forward + backward replayed as one CUDA graph) per head, the two alternating round by round in one process, on the
card's name and power limit read in the same run. The head adds B x num_bins work after the depth-8 stack.

Prints one JSON line (and writes it to --out when given).

    python tools/hl_gauss_bench.py [--rounds 7] [--steps 20] [--bins 1024] [--max-value 4096] [--out results/hl_gauss.json]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CFG4 = dict(dim=512, depth=8, heads=8, batch=32, seq=1024)


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'unavailable ({e})'
    return name, q


def make_step(pkg, mel, text, **head):
    torch.manual_seed(0)
    random.seed(0)
    c = CFG4
    model = pkg.DurationPredictor(transformer=dict(dim=c['dim'], depth=c['depth'], heads=c['heads'], max_seq_len=c['seq']), **head)
    model.cuda().train()
    return model, pkg.GraphedTrainStep(model, mel, text=text)


def time_steps(step, n):
    """n graph replays -> device ms per step"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7, help='alternating rounds of both heads')
    ap.add_argument('--steps', type=int, default=20, help='timed replays per head per round')
    ap.add_argument('--bins', type=int, default=1024)
    ap.add_argument('--max-value', type=float, default=4096.)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    import e2_tts_pytorch_b200 as pkg
    c = CFG4
    g = torch.Generator().manual_seed(0)
    mel = torch.randn(c['batch'], c['seq'], 100, generator=g).cuda()
    text = [''.join(random.Random(i).choices('abcdefghij klmnop', k=c['seq'] // 8)) for i in range(c['batch'])]
    heads = {'regression': {},
             'hl_gauss': dict(hl_gauss_loss=dict(min_value=0., max_value=args.max_value, num_bins=args.bins), use_regression=False)}
    steps = {name: make_step(pkg, mel, text, **kw) for name, kw in heads.items()}
    for _, step in steps.values():
        time_steps(step, 3)
    ms = {name: [] for name in heads}
    for _ in range(args.rounds):
        for name, (_, step) in steps.items():
            ms[name].append(time_steps(step, args.steps))
    res = dict(mode=f"GraphedTrainStep replays, DurationPredictor d{c['dim']} depth{c['depth']} h{c['heads']}, B{c['batch']} x {c['seq']}, "
                    'the two heads alternating')
    res['gpu'], res['power_limit'] = gpu_info()
    for name in heads:
        res[name] = dict(step_ms_median=round(statistics.median(ms[name]), 3), step_ms_range=[round(min(ms[name]), 3), round(max(ms[name]), 3)],
                         loss=float(steps[name][1]()))
    res['hl_gauss']['head'] = f'{args.bins} bins over [0, {args.max_value:g}]'
    res['time_ratio'] = round(res['hl_gauss']['step_ms_median'] / res['regression']['step_ms_median'], 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
