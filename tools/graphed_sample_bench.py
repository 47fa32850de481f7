"""E2TTS.sample() against GraphedSampler on the same model and inputs: the 32-step midpoint ODE with classifier-free guidance
(cfg_strength 1, no cfg_null_model: GraphedSampler runs each function evaluation as one batched pass over 2B items).

  a  d512 depth 8 h8, B1, prompt 100 -> 600 frames   (one utterance: where the host sets the latency)
  b  d512 depth 8 h8, B8, prompt 100 -> 600 frames
  c  d1024 depth 24 h16, B8, prompt 256 -> 2048 frames (bench.py cfg5)

Per workload the two paths alternate in one process (eager, graphed, eager, ...), `--repeats` calls each after one warm-up call of
each; every call is timed on the host clock and ends in a synchronise. Reports the median ms per call and generated mel frames per
second (B x frames / call time), the sampler's capture time, the rel-L2 between the two outputs (same y0), the card name and its power
limit read in the same run. Prints one JSON line (and writes it to --out when given).

    python tools/graphed_sample_bench.py [--repeats 5] [--only a,b,c] [--out results/graphed_sample_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    'a': dict(dim=512, depth=8, heads=8, batch=1, prompt=100, frames=600, buckets=(512, 640, 768, 1024)),
    'b': dict(dim=512, depth=8, heads=8, batch=8, prompt=100, frames=600, buckets=(512, 640, 768, 1024)),
    'c': dict(dim=1024, depth=24, heads=16, batch=8, prompt=256, frames=2048, buckets=(1024, 2048)),
}
STEPS = 32
TEXT = ['the quick brown fox jumps over the lazy dog', 'a short line of text to speak']


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'unavailable ({e})'
    return name, q


def run(pkg, w, repeats):
    dev = torch.device('cuda')
    torch.manual_seed(0)
    model = pkg.E2TTS(transformer=dict(dim=w['dim'], depth=w['depth'], heads=w['heads'], dropout=0., max_seq_len=max(w['buckets'])),
                      use_vocos=False).to(dev).eval()
    B, n = w['batch'], w['frames']
    cond = torch.randn(B, w['prompt'], 100, device=dev)
    text = [TEXT[i % 2] for i in range(B)]
    t0 = time.perf_counter()
    sampler = pkg.GraphedSampler(model, B, w['buckets'], steps=STEPS, cfg_strength=1.0)
    torch.cuda.synchronize()
    capture_s = time.perf_counter() - t0
    paths = {
        'eager': lambda: model.sample(cond, text=text, duration=n, steps=STEPS, cfg_strength=1.0, return_raw_output=True),
        'graphed': lambda: sampler(cond, text=text, duration=n, return_raw_output=True),
    }
    outs = {}
    for name, f in paths.items():          # warm-up, and the outputs of one seed
        torch.manual_seed(1)
        outs[name] = f()
    torch.cuda.synchronize()
    err = float((outs['graphed'] - outs['eager']).double().norm() / outs['eager'].double().norm())
    times = {k: [] for k in paths}
    for _ in range(repeats):
        for name, f in paths.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t)
    res = dict(capture_s=round(capture_s, 2), rel_l2_graphed_vs_eager=err)
    for name, ts in times.items():
        ms = 1e3 * statistics.median(ts)
        res[name] = dict(ms_per_call=round(ms, 2), frames_per_s=round(B * n / (ms / 1e3), 1), all_ms=[round(1e3 * t, 2) for t in ts])
    res['speedup'] = round(res['eager']['ms_per_call'] / res['graphed']['ms_per_call'], 3)
    del sampler, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--only', default='a,b,c')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('graphed_sample_bench: needs a GPU')
    import e2_tts_pytorch_b200 as pkg
    gpu, power = gpu_info()
    result = dict(gpu=gpu, power_limit_and_max_sm_clock=power, ode=f'{STEPS}-step midpoint, cfg_strength 1', repeats=args.repeats)
    for key in args.only.split(','):
        w = WORKLOADS[key]
        result[key] = dict(workload=w, **run(pkg, w, args.repeats))
        print(key, json.dumps(result[key]), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
