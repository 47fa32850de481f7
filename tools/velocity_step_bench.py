"""Training steps with the velocity-consistency term (E2TTS(velocity_consistency_weight=0.1) and an EMA teacher in eval mode): cfg2
(E2TTS d512 depth 8 h8, dropout 0.1), the teacher a deep copy of the model.

  eager          : model(mel, text=..., velocity_consistency_model=teacher) + backward, B16 x 1024 frames
  graphed        : GraphedTrainStep(model, mel) without a teacher, B16 x 1024
  graphed+teacher: GraphedTrainStep(model, mel, velocity_consistency_model=teacher), B16 x 1024
  bucketed       : BucketedTrainStep(velocity_consistency_model=teacher) on the ragged workload of tools/bucketed_step_bench.py
                   (clip lengths uniform 188..1407, cond_drop_prob 0.25, k = 4, buckets 256..1408), velocity on and off

The paths alternate in one process: each round times one sample of every path (CUDA events around `--inner` calls, per-call ms).
Reports the median and the 10th / 90th percentiles per path, the peak memory each path allocates above what is already allocated, the memory each step's
graph pool reserved at construction, the launches per replay, and the card's name, power limit and max SM clock read in the same
run. Prints one JSON line (and writes it to --out when given).

    python tools/velocity_step_bench.py [--rounds 15] [--inner 4] [--out results/velocity_step_bench.json]
"""
import argparse
import copy
import json
import os
import random
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bucketed_step_bench import BUCKETS, B, K, P_DROP, batches, gpu_info  # noqa: E402

N, WEIGHT = 1024, 0.1


def reserved_by(build):
    """-> (the object build() returns, bytes it left reserved)"""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r0 = torch.cuda.memory_reserved()
    obj = build()
    torch.cuda.synchronize()
    return obj, torch.cuda.memory_reserved() - r0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=15, help='timed samples per path')
    ap.add_argument('--inner', type=int, default=4, help='calls per sample (a multiple of k = 4 keeps bucketed windows whole)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    import e2_tts_pytorch_b200 as pkg
    dev = torch.device('cuda')
    torch.manual_seed(0)
    random.seed(0)
    model = pkg.E2TTS(transformer=dict(dim=512, depth=8, heads=8), use_vocos=False, cond_drop_prob=0.0,
                      velocity_consistency_weight=WEIGHT).to(dev).train()
    teacher = copy.deepcopy(model).eval()
    res = dict(workload=f'cfg2 E2TTS d512 depth8 h8 dropout 0.1, velocity_consistency_weight {WEIGHT}, teacher in eval mode; '
                        f'fixed: B{B} x {N}; ragged: B{B}, clip lengths uniform 188..1407, cond_drop_prob {P_DROP}, k={K}',
               buckets=list(BUCKETS), rounds=args.rounds, inner=args.inner)
    res['gpu'], res['power_limit_and_max_sm_clock'] = gpu_info()
    g = torch.Generator().manual_seed(3)
    mel = torch.randn(B, N, 100, generator=g).to(dev)
    text = pkg.list_str_to_tensor([''.join(random.Random(i).choices('abcdefgh ', k=120)) for i in range(B)]).to(dev)

    def eager(_i):
        out = model(mel, text=text, velocity_consistency_model=teacher)
        out.loss.backward()
        del out
        for p in model.parameters():
            p.grad = None

    for i in range(3):
        eager(i)
    torch.cuda.synchronize()
    plain, res_plain = reserved_by(lambda: pkg.GraphedTrainStep(model, mel, text=text))
    with_t, res_t = reserved_by(lambda: pkg.GraphedTrainStep(model, mel, text=text, velocity_consistency_model=teacher))
    model.cond_drop_prob = P_DROP
    bucketed, res_b = reserved_by(lambda: pkg.BucketedTrainStep(model, B, BUCKETS, grad_accumulation_steps=K,
                                                                velocity_consistency_model=teacher))
    model.cond_drop_prob = 0.0
    res['graph_pool_reserved_gib'] = {'graphed': round(res_plain / 2 ** 30, 2), 'graphed+teacher': round(res_t / 2 ** 30, 2),
                                      'bucketed (+teacher)': round(res_b / 2 ** 30, 2)}
    res['launches_per_replay'] = {'graphed': plain.launches_per_step, 'graphed+teacher': with_t.launches[True],
                                  'graphed+teacher, velocity off': with_t.launches[False],
                                  'bucketed 1408 text, velocity on / off': [bucketed.launches[1408, False, True], bucketed.launches[1408, False, False]]}
    res['bucketed_capture_s'] = round(bucketed.capture_seconds, 2)

    ragged = batches(args.rounds * args.inner + 8, 2)
    cursor = {'on': 0, 'off': 0}

    def ragged_step(velocity):
        key = 'on' if velocity else 'off'

        def run(_i):
            m, lens, txt = ragged[cursor[key] % len(ragged)]
            cursor[key] += 1
            model.cond_drop_prob = P_DROP
            bucketed(m.to(dev, non_blocking=True), text=txt, lens=lens.to(dev, non_blocking=True), velocity=velocity)
            model.cond_drop_prob = 0.0
        return run

    paths = {
        'eager+teacher': eager,
        'graphed': lambda i: plain(),
        'graphed+teacher': lambda i: with_t(),
        'bucketed+teacher': ragged_step(True),
        'bucketed, velocity off': ragged_step(False),
    }
    for fn in paths.values():          # warm-up of every path (and every bucket the ragged stream reaches first)
        for i in range(args.inner):
            fn(i)
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    peak = {k: 0 for k in paths}
    for _ in range(args.rounds):
        for name, fn in paths.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.inner):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.inner)
            peak[name] = max(peak[name], torch.cuda.max_memory_allocated() - base)

    def pct(xs, q):
        xs = sorted(xs)
        return xs[min(len(xs) - 1, int(round(q * (len(xs) - 1))))]

    res['ms_per_call'] = {k: dict(median=round(statistics.median(v), 2), p10=round(pct(v, 0.1), 2), p90=round(pct(v, 0.9), 2))
                          for k, v in times.items()}
    res['allocated_outside_calls_gib'] = round(torch.cuda.memory_allocated() / 2 ** 30, 2)   # models, static step tensors, graph outputs
    res['peak_allocated_during_call_gib'] = {k: round(v / 2 ** 30, 2) for k, v in peak.items()}   # above what was allocated before it
    m = res['ms_per_call']
    res['speedup_graphed+teacher_over_eager+teacher'] = round(m['eager+teacher']['median'] / m['graphed+teacher']['median'], 3)
    res['teacher_cost_graphed'] = round(m['graphed+teacher']['median'] / m['graphed']['median'] - 1, 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
