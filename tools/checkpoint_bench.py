"""Activation checkpointing (Transformer(checkpoint_activations=True)) against the plain step: eager E2TTS training steps (forward +
`loss.backward()`), the two modes alternating round by round in one process after a warm-up, on the card's name and power limit read
in the same run.

  cfg2  E2TTS d512 depth 8 h8, B16 x 1024 frames: step ms (CUDA events, median over rounds) and peak memory per mode
  cfg3  E2TTS d1024 depth 24 h16, 2048 frames: the same at B4, then the largest batch that fits each mode (the first batch of
        --batches that runs out of memory ends the search for that mode)

Prints one JSON line (and writes it to --out when given).

    python tools/checkpoint_bench.py [--rounds 5] [--steps 5] [--warmup 3] [--batches 4,6,8,10,12,16,20,24] [--out results/ckpt.json]
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

CFG = {'cfg2': dict(dim=512, depth=8, heads=8, batch=16, seq=1024), 'cfg3': dict(dim=1024, depth=24, heads=16, batch=4, seq=2048)}


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'unavailable ({e})'
    return name, q


def make(pkg, c):
    torch.manual_seed(0)
    random.seed(0)
    return pkg.E2TTS(transformer=dict(dim=c['dim'], depth=c['depth'], heads=c['heads'], max_seq_len=c['seq']), use_vocos=False,
                     cond_drop_prob=0.0).cuda().train()


def batch(B, N):
    g = torch.Generator().manual_seed(B * 7919 + N)
    text = [''.join(random.Random(i).choices('abcdefghij klmnop', k=N // 8)) for i in range(B)]
    return torch.randn(B, N, 100, generator=g).cuda(), text


def run_steps(model, mel, text, n):
    """n eager steps -> device ms per step"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        out = model(mel, text=text)
        out.loss.backward()
        del out
        for p in model.parameters():
            p.grad = None
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def peak(model, mel, text):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    run_steps(model, mel, text, 1)
    return torch.cuda.max_memory_allocated() / 2 ** 30


def compare(pkg, c, B, args):
    model = make(pkg, c)
    mel, text = batch(B, c['seq'])
    res = {}
    for ckpt in (False, True):
        model.transformer.checkpoint_activations = ckpt
        run_steps(model, mel, text, args.warmup)
        res[ckpt] = dict(ms=[], peak_gib=peak(model, mel, text))
    for _ in range(args.rounds):
        for ckpt in (False, True):
            model.transformer.checkpoint_activations = ckpt
            res[ckpt]['ms'].append(run_steps(model, mel, text, args.steps))
    del model, mel
    torch.cuda.empty_cache()
    out = {}
    for ckpt, name in ((False, 'plain'), (True, 'checkpointed')):
        ms = res[ckpt]['ms']
        out[name] = dict(step_ms_median=round(statistics.median(ms), 2), step_ms_range=[round(min(ms), 2), round(max(ms), 2)],
                         peak_gib=round(res[ckpt]['peak_gib'], 2))
    out['time_ratio'] = round(out['checkpointed']['step_ms_median'] / out['plain']['step_ms_median'], 3)
    return out


def largest_batch(pkg, c, ckpt, batches):
    model = make(pkg, c)
    model.transformer.checkpoint_activations = ckpt
    best = None
    for B in batches:
        try:
            mel, text = batch(B, c['seq'])
            run_steps(model, mel, text, 1)
            best = dict(batch=B, peak_gib=round(peak(model, mel, text), 2))
        except torch.OutOfMemoryError:
            break
        finally:
            mel = None
            for p in model.parameters():
                p.grad = None
            torch.cuda.empty_cache()
    del model
    torch.cuda.empty_cache()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5, help='alternating rounds of both modes')
    ap.add_argument('--steps', type=int, default=5, help='timed steps per mode per round')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--batches', default='4,6,8,10,12,16,20,24', help='cfg3 batch sizes tried, in order, for the largest that fits')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    import e2_tts_pytorch_b200 as pkg
    res = dict(mode='eager E2TTS training steps (forward + backward), dropout 0.1, the two modes alternating')
    res['gpu'], res['power_limit'] = gpu_info()
    for name in ('cfg2', 'cfg3'):
        c = CFG[name]
        res[name] = dict(shape=f"d{c['dim']} depth{c['depth']} h{c['heads']}, B{c['batch']} x {c['seq']}", **compare(pkg, c, c['batch'], args))
        print(name, json.dumps(res[name]), flush=True)
    batches = [int(b) for b in args.batches.split(',')]
    res['cfg3']['largest_batch'] = {('checkpointed' if ckpt else 'plain'): largest_batch(pkg, CFG['cfg3'], ckpt, batches)
                                    for ckpt in (False, True)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
