"""Developer tool (GPU): what the feed-forward variants of `ff_kwargs` cost, in one process.
  1. The FF-in GLU GEMM (bias, dropout 0.1, pre-activations saved, as in the training step) per activation, and GELU with the GLU
     multiplier, at the cfg2 audio / text and cfg3 audio / text shapes (CUDA events, operands cycled so that L2 does not hold them).
  2. BASELINE cfg2's graphed training step (dropout 0.1, text on every step) with the default feed-forward, SwiGLU (swish=True) and
     ReLU^2 (relu_squared=True), timed in alternating rounds.
Prints both tables and one JSON line, with the GPU's name and power limit read in the same run.
usage: python tools/ff_bench.py [rounds] [steps_per_round] [warmup]"""
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import e2_tts_pytorch_b200 as pkg  # noqa: E402
from e2_tts_pytorch_b200 import ops  # noqa: E402

NSET = 6
ACTS = {'gelu': dict(act=ops.GLU_GELU), 'silu': dict(act=ops.GLU_SILU), 'relu2': dict(act=ops.GLU_RELU2),
        'gelu+mult': dict(act=ops.GLU_GELU, mult=True)}
SETTINGS = {'default': dict(), 'swiglu': dict(swish=True), 'relu2': dict(relu_squared=True)}
med = lambda v: sorted(v)[len(v) // 2]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip() if q.returncode == 0 else f'unavailable ({q.stderr.strip()[:80]})')


def gemm_table(dev, reps=40, rounds=3):
    shapes = {}
    for c in (2, 3):
        cfg = bench.CONFIGS[c]
        T = cfg['batch'] * (cfg['seq'] + 32)
        d = cfg['dim']
        shapes[f'cfg{c} audio'] = (T, 8 * d, d)
        shapes[f'cfg{c} text'] = (T, 4 * d, d // 2)
    out = {}
    for sname, (M, N, K) in shapes.items():
        sets = []
        for _ in range(NSET):
            sets.append(((torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16), (torch.randn(N, K, device=dev) * 0.05).to(torch.bfloat16),
                         torch.empty(M, N // 2, device=dev, dtype=torch.bfloat16), torch.empty(M, N, device=dev, dtype=torch.bfloat16),
                         torch.randn(N, device=dev) * 0.1, 1 + 0.1 * torch.randn(N // 2, device=dev)))
        times = {a: [] for a in ACTS}
        for r in range(rounds):   # activations alternate within each round
            for a in (list(ACTS) if r % 2 == 0 else list(ACTS)[::-1]):
                kw = ACTS[a]

                def run(i):
                    A, W, h, ug, b, m = sets[i % NSET]
                    ops.gemm(A, W, M, N, K, out=h, D2=ug, ldd2=N, bias=b, geglu=kw['act'], dropout_p=0.1, seed=5 + i,
                             glu_mult=m if kw.get('mult') else None)
                for i in range(5):
                    run(i)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
                ev[0].record()
                for i in range(reps):
                    run(i)
                    ev[i + 1].record()
                torch.cuda.synchronize()
                times[a] += [ev[i].elapsed_time(ev[i + 1]) * 1e3 for i in range(reps)]
        out[sname] = dict(shape=[M, N, K], **{a: round(med(t), 1) for a, t in times.items()})
        print(f'FF-in GLU GEMM {sname} {M}x{N}x{K} (median us): ' + ', '.join(f'{a} {out[sname][a]}' for a in ACTS), flush=True)
    return out


def step_table(dev, rounds, per_round, warmup):
    cfg = bench.CONFIGS[2]
    B, N = cfg['batch'], cfg['seq']
    torch.manual_seed(1)
    mel = torch.randn(B, N, 100, device=dev)
    text = pkg.list_str_to_tensor([bench.TEXT[i % 2] for i in range(B)]).to(dev)
    steps = {}
    for s, kw in SETTINGS.items():
        torch.manual_seed(0)
        random.seed(0)
        model = pkg.E2TTS(transformer=dict(dim=cfg['dim'], depth=cfg['depth'], heads=cfg['heads'], dropout=0.1, ff_kwargs=kw),
                          use_vocos=False).to(dev)
        model.cond_drop_prob = 0.0
        model.train()
        steps[s] = pkg.GraphedTrainStep(model, mel, text=text)
        torch.cuda.synchronize()
    for s in SETTINGS:
        for _ in range(warmup):
            steps[s]()
    torch.cuda.synchronize()
    times = {s: [] for s in SETTINGS}
    round_medians = {s: [] for s in SETTINGS}
    for r in range(rounds):
        order = list(SETTINGS) if r % 2 == 0 else list(SETTINGS)[::-1]
        for s in order:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(per_round + 1)]
            ev[0].record()
            for i in range(per_round):
                steps[s]()
                ev[i + 1].record()
            torch.cuda.synchronize()
            t = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(per_round))
            times[s] += t
            round_medians[s].append(t[len(t) // 2])
    res = {}
    for s in SETTINGS:
        res[s] = dict(median_ms=round(med(times[s]), 3), round_median_min_ms=round(min(round_medians[s]), 3),
                      round_median_max_ms=round(max(round_medians[s]), 3), timed_steps=len(times[s]),
                      launches_per_step=steps[s].launches_per_step)
        r = res[s]
        print(f'cfg2 graphed step, {s}: median {r["median_ms"]:.2f} ms over {r["timed_steps"]} steps '
              f'(round medians {r["round_median_min_ms"]:.2f}-{r["round_median_max_ms"]:.2f}), {r["launches_per_step"]} launches', flush=True)
    return res


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    per_round = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    warmup = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    assert torch.cuda.is_available(), 'ff_bench.py times H100 kernels: it needs a GPU'
    dev = torch.device('cuda:0')
    res = dict(card=card(), gemm_us=gemm_table(dev), step=step_table(dev, rounds, per_round, warmup))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
