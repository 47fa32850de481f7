"""Time MelSpec.collate — the on-device data path: one kernel launch over a ragged batch of waves — for the reference's
mel_spec_kwargs: the defaults, each switch alone, n_fft 1200 (mixed-radix FFT) against 1024 and 2048 (radix-2), and the 16 kHz
front-end (n_fft 400). 32 items of 2-15 s (seeded lengths) per batch, already on the GPU; CUDA events around `iters` calls after
warm-up, the configurations alternated over `repeats` rounds; reports the median and spread per configuration, with the card's
name and power limit.

    python tools/melspec_bench.py [--iters 50] [--repeats 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import e2_tts_pytorch_b200 as pkg  # noqa: E402

CONFIGS = {
    'defaults (n_fft 1024, 24 kHz)': dict(),
    'win_length=800': dict(win_length=800),
    'center=False': dict(center=False),
    'power=2': dict(power=2),
    'power=1.5': dict(power=1.5),
    'normalize=True': dict(normalize=True),
    "norm='slaney'": dict(norm='slaney'),
    'n_fft=1024 hop 300': dict(filter_length=1024, win_length=1024, hop_length=300),
    'n_fft=1200 hop 300': dict(filter_length=1200, win_length=1200, hop_length=300),
    'n_fft=2048 hop 300': dict(filter_length=2048, win_length=2048, hop_length=300),
    'n_fft=400 hop 160, 16 kHz, 80 mels': dict(filter_length=400, win_length=400, hop_length=160, n_mel_channels=80, sampling_rate=16000),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'melspec_bench.py measures on the GPU'
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    seconds = 2 + 13 * torch.rand(32, generator=g)
    runs = {}
    for name, kw in CONFIGS.items():
        ms = pkg.MelSpec(**kw).to(dev)
        lens = (seconds * ms.sampling_rate).long()
        waves = torch.randn(32, int(lens.max()), generator=g) * 0.3
        waves = waves * (torch.arange(waves.shape[1])[None] < lens[:, None])
        runs[name] = (ms, waves.to(dev), lens.to(dev))
    for ms, w, l in runs.values():      # warm-up: module load, the once-per-device shared-memory opt-in
        for _ in range(5):
            ms.collate(w, l)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(args.repeats):
        for name, (ms, w, l) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                ms.collate(w, l)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.iters)
    gpu, limit = card()
    res = dict(gpu=gpu, power_limit_and_max_sm_clock=limit, batch='32 items of 2-15 s', iters=args.iters, repeats=args.repeats,
               results={})
    for name, t in times.items():
        ms, w, l = runs[name]
        frames = int(ms.collate(w, l)['mel_lengths'].sum())
        med = statistics.median(t)
        res['results'][name] = dict(ms_median=round(med, 4), ms_min=round(min(t), 4), ms_max=round(max(t), 4), frames=frames,
                                    us_per_kframe=round(1e3 * med / frames * 1e3, 3))
        print(f'{name:40s} {med:8.4f} ms  (min {min(t):.4f}, max {max(t):.4f})  {frames} frames')
    print(f'{gpu}; power limit, max SM clock: {limit}')
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
