"""Graphed training on ragged batches against the eager loop: cfg2 (E2TTS d512 depth 8 h8) at batch 16 on a seeded stream of ragged
batches — clip lengths uniform over 188..1407 frames (2-15 s at 24 kHz, hop 256), cond_drop_prob 0.25, gradient accumulation k = 4.

  eager     : the reference's loop — each batch padded to its longest clip, `(loss / k).backward()`, p.grad accumulated by autograd
  bucketed  : BucketedTrainStep(buckets=(256, 512, 768, 1024, 1408)) — one graph replay + in-graph accumulate per micro-step

Per micro-step: device ms (CUDA events around the whole window: the GPU timeline, idle gaps included) and end-to-end ms (host clock
around the window, batch upload included, ending in a synchronise); valid mel-frames/s; padding overhead (frames computed over the
frames of the longest clip of each batch, and over the valid frames); capture time; peak memory of one bucket against all buckets.
Prints one JSON line (and writes it to --out when given).

    python tools/bucketed_step_bench.py [--steps 40] [--warmup 8] [--out results/bucketed_step_bench.json]
"""
import argparse
import json
import os
import random
import string
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BUCKETS = (256, 512, 768, 1024, 1408)
B, K, P_DROP = 16, 4, 0.25
LO, HI = 188, 1407


def batches(n, seed):
    """n host batches: (mel [B, longest, 100] pinned, lens [B], text list[str]); the same stream for every loop"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        lens = torch.randint(LO, HI + 1, (B,), generator=g)
        n_max = int(lens.max())
        mel = torch.randn(B, n_max, 100, generator=g)
        mel *= (torch.arange(n_max)[None, :, None] < lens[:, None, None])     # the collate's zero padding
        text = [''.join(random.Random(int(l) * 7 + i).choices(string.ascii_lowercase + ' ', k=int(l) // 8)) for i, l in enumerate(lens)]
        out.append((mel.pin_memory(), lens, text))
    return out


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'unavailable ({e})'
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40, help='timed micro-steps per loop (a multiple of k = 4)')
    ap.add_argument('--warmup', type=int, default=8)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    import e2_tts_pytorch_b200 as pkg
    dev = torch.device('cuda')
    torch.manual_seed(0)
    random.seed(0)
    model = pkg.E2TTS(transformer=dict(dim=512, depth=8, heads=8), use_vocos=False, cond_drop_prob=P_DROP).to(dev).train()
    warm, timed = batches(args.warmup, 1), batches(args.steps, 2)
    res = dict(workload=f'cfg2 E2TTS d512 depth8 h8, B{B}, clip lengths uniform {LO}..{HI} frames, cond_drop_prob {P_DROP}, k={K}',
               buckets=list(BUCKETS), micro_steps=args.steps)
    res['gpu'], res['power_limit_and_max_sm_clock'] = gpu_info()

    # ---------------------------------------------------------------- eager loop
    def eager(batch, i):
        mel, lens, text = batch
        out = model(mel.to(dev, non_blocking=True), text=text, lens=lens.to(dev, non_blocking=True))
        (out.loss / K).backward()
        loss = out.loss.detach()
        del out
        if (i + 1) % K == 0:
            for p in model.parameters():
                p.grad = None        # the optimiser step would consume them here
        return loss

    def window(fn, data):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for i, b in enumerate(data):
            fn(b, i)
        e1.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        return e0.elapsed_time(e1) / len(data), 1e3 * wall / len(data)

    for i, b in enumerate(warm):
        eager(b, i)
    torch.cuda.reset_peak_memory_stats()
    dev_ms, e2e_ms = window(eager, timed)
    res['eager'] = dict(device_ms=round(dev_ms, 2), end_to_end_ms=round(e2e_ms, 2),
                        peak_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    for p in model.parameters():
        p.grad = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # ---------------------------------------------------------------- memory of one bucket against all
    r0 = torch.cuda.memory_reserved()
    one = pkg.BucketedTrainStep(model, B, (BUCKETS[-1],), grad_accumulation_steps=K)
    torch.cuda.synchronize()
    res['one_bucket'] = dict(bucket=BUCKETS[-1], graphs=len(one.graphs), reserved_gib=round((torch.cuda.memory_reserved() - r0) / 2 ** 30, 2),
                             capture_s=round(one.capture_seconds, 2))
    del one
    for p in model.parameters():
        p.grad = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r0 = torch.cuda.memory_reserved()
    step = pkg.BucketedTrainStep(model, B, BUCKETS, grad_accumulation_steps=K)
    torch.cuda.synchronize()
    res['all_buckets'] = dict(graphs=len(step.graphs), reserved_gib=round((torch.cuda.memory_reserved() - r0) / 2 ** 30, 2),
                              capture_s=round(step.capture_seconds, 2), launches_per_micro_step=step.launches_per_step)

    # ---------------------------------------------------------------- bucketed loop
    def bucketed(batch, i):
        mel, lens, text = batch
        loss = step(mel.to(dev, non_blocking=True), text=text, lens=lens.to(dev, non_blocking=True))
        assert step.sync_gradients == ((i + 1) % K == 0)
        return loss

    for i, b in enumerate(warm):
        bucketed(b, i)
    torch.cuda.reset_peak_memory_stats()
    dev_ms_g, e2e_ms_g = window(bucketed, timed)
    res['bucketed'] = dict(device_ms=round(dev_ms_g, 2), end_to_end_ms=round(e2e_ms_g, 2),
                           peak_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))

    valid = sum(int(l.sum()) for _, l, _ in timed)
    longest = sum(B * int(l.max()) for _, l, _ in timed)
    padded = sum(B * step.plan.bucket(int(l.max())) for _, l, _ in timed)
    res['valid_frames_per_s'] = dict(eager=round(valid / (args.steps * e2e_ms / 1e3)), bucketed=round(valid / (args.steps * e2e_ms_g / 1e3)))
    res['padding'] = dict(bucket_over_longest=round(padded / longest - 1, 4), bucket_over_valid=round(padded / valid - 1, 4),
                          longest_over_valid=round(longest / valid - 1, 4))
    res['speedup_end_to_end'] = round(e2e_ms / e2e_ms_g, 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
