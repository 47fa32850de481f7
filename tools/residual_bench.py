"""Developer tool (GPU): step time of BASELINE cfg2's training step (E2TTS d512 depth 8 h8, B16 x N1024, dropout 0.1, text on every
step) with num_residual_streams=1 (plain residual) and 4 (hyper-connections, the reference default), both replayed through
GraphedTrainStep and timed in alternating rounds within one process, so that both see the same card and the same neighbours.
Prints, per setting, the median device time per step over every timed step, the spread of the round medians and the kernel launches
per step, with the GPU's name and power limit read in the same run.
usage: python tools/residual_bench.py [rounds] [steps_per_round] [warmup]"""
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


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip() if q.returncode == 0 else f'unavailable ({q.stderr.strip()[:80]})')


def build(streams, dev, mel, text):
    cfg = bench.CONFIGS[2]
    torch.manual_seed(0)
    random.seed(0)
    model = pkg.E2TTS(transformer=dict(dim=cfg['dim'], depth=cfg['depth'], heads=cfg['heads'], dropout=0.1, num_residual_streams=streams),
                      use_vocos=False).to(dev)
    model.cond_drop_prob = 0.0
    model.train()
    step = pkg.GraphedTrainStep(model, mel, text=text)
    return model, step


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    per_round = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    warmup = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    assert torch.cuda.is_available(), 'residual_bench.py times the H100 step: it needs a GPU'
    dev = torch.device('cuda:0')
    cfg = bench.CONFIGS[2]
    B, N = cfg['batch'], cfg['seq']
    torch.manual_seed(1)
    mel = torch.randn(B, N, 100, device=dev)
    text = pkg.list_str_to_tensor([bench.TEXT[i % 2] for i in range(B)]).to(dev)
    steps = {}
    for s in (1, 4):
        _, steps[s] = build(s, dev, mel, text)
        torch.cuda.synchronize()
    for s in (1, 4):
        for _ in range(warmup):
            steps[s]()
    torch.cuda.synchronize()
    times = {1: [], 4: []}
    round_medians = {1: [], 4: []}
    for r in range(rounds):
        for s in ((1, 4) if r % 2 == 0 else (4, 1)):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(per_round + 1)]
            ev[0].record()
            for i in range(per_round):
                steps[s]()
                ev[i + 1].record()
            torch.cuda.synchronize()
            t = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(per_round))
            times[s] += t
            round_medians[s].append(t[len(t) // 2])
    med = lambda v: sorted(v)[len(v) // 2]
    res = dict(config=cfg['name'] + ', dropout 0.1, CUDA graph', card=card(), rounds=rounds, steps_per_round=per_round)
    for s in (1, 4):
        res[f'S{s}'] = dict(median_ms=round(med(times[s]), 3), round_median_min_ms=round(min(round_medians[s]), 3),
                            round_median_max_ms=round(max(round_medians[s]), 3), timed_steps=len(times[s]),
                            launches_per_step=steps[s].launches_per_step, mel_frames_per_s=round(B * N / (med(times[s]) * 1e-3)))
    res['S1_over_S4'] = round(res['S1']['median_ms'] / res['S4']['median_ms'], 4)
    for s in (1, 4):
        r = res[f'S{s}']
        print(f'num_residual_streams={s}: median {r["median_ms"]:.2f} ms/step over {r["timed_steps"]} steps '
              f'(round medians {r["round_median_min_ms"]:.2f}-{r["round_median_max_ms"]:.2f}), {r["launches_per_step"]} launches/step')
    print(json.dumps(res))


if __name__ == '__main__':
    main()
