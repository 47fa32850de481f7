"""Developer tool (GPU): 64- against 128-wide attention heads at the same inner width I = heads * dim_head.
  1. attention kernels alone (b200_attn_fwd + b200_attn_bwd through ops.AttnCore, softclamp 50, dropout 0.1, head gate): 8 x 64 against
     4 x 128 at cfg2's shape (B 16, N' 1056, I 512) and 16 x 64 against 8 x 128 at cfg3's (B 4, N' 2080, I 1024);
  2. BASELINE cfg2's training step (E2TTS d512 depth 8, B16 x N1024, dropout 0.1) with heads=8, dim_head=64 and heads=4, dim_head=128,
     both replayed through GraphedTrainStep.
Each pair is timed in alternating rounds within one process (CUDA events), so that both see the same card and the same neighbours.
Prints, per setting, the median time over every timed call and the spread of the round medians, with the GPU's name, power limit and
SM clock read in the same run.
usage: python tools/headdim_bench.py [rounds] [calls_per_round] [warmup]"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import torch  # noqa: E402

import bench  # noqa: E402
import e2_tts_pytorch_b200 as pkg  # noqa: E402
from residual_bench import card  # noqa: E402


def alternate(fns, rounds, per_round, warmup):
    """fns: {label: callable}; -> {label: dict(median_ms, round_median_min_ms, round_median_max_ms, calls)}"""
    for f in fns.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    rmed = {k: [] for k in fns}
    labels = list(fns)
    for r in range(rounds):
        for k in (labels if r % 2 == 0 else labels[::-1]):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(per_round + 1)]
            ev[0].record()
            for i in range(per_round):
                fns[k]()
                ev[i + 1].record()
            torch.cuda.synchronize()
            t = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(per_round))
            times[k] += t
            rmed[k].append(t[len(t) // 2])
    med = lambda v: sorted(v)[len(v) // 2]
    return {k: dict(median_ms=round(med(times[k]), 4), round_median_min_ms=round(min(rmed[k]), 4),
                    round_median_max_ms=round(max(rmed[k]), 4), calls=len(times[k])) for k in fns}


def attn_call(B, H, dh, Np, dev):
    g = torch.Generator(device=dev).manual_seed(H * dh)
    bf = lambda *s: (torch.randn(*s, device=dev, generator=g)).to(torch.bfloat16)
    q, k, v = (bf(B, H, Np, dh).requires_grad_() for _ in range(3))
    gate = torch.rand(B * Np, H, device=dev, generator=g).requires_grad_()
    mask = torch.ones(B, Np, dtype=torch.uint8, device=dev)
    mask[B // 2:, Np - Np // 5:] = 0
    dog = bf(B * Np, H * dh)

    def run():
        og = pkg.ops.AttnCore.apply(q, k, v, gate, mask, 0.1, 7, 50.0, None)
        og.backward(dog)
    return run


def step_call(heads, dim_head, dev, mel, text):
    cfg = bench.CONFIGS[2]
    torch.manual_seed(0)
    random.seed(0)
    model = pkg.E2TTS(transformer=dict(dim=cfg['dim'], depth=cfg['depth'], heads=heads, dim_head=dim_head, dropout=0.1), use_vocos=False).to(dev)
    model.cond_drop_prob = 0.0
    model.train()
    return pkg.GraphedTrainStep(model, mel, text=text)


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    per_round = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    warmup = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    assert torch.cuda.is_available(), 'headdim_bench.py times the H100: it needs a GPU'
    dev = torch.device('cuda:0')
    res = dict(card=card(), rounds=rounds, calls_per_round=per_round)
    for name, B, Np, I in (('cfg2', 16, 1056, 512), ('cfg3', 4, 2080, 1024)):
        fns = {f'{I // dh}x{dh}': attn_call(B, I // dh, dh, Np, dev) for dh in (64, 128)}
        res[f'attention fwd+bwd {name} (B {B}, N\' {Np}, I {I})'] = alternate(fns, rounds, per_round, warmup)
        del fns
        torch.cuda.empty_cache()
    cfg = bench.CONFIGS[2]
    torch.manual_seed(1)
    mel = torch.randn(cfg['batch'], cfg['seq'], 100, device=dev)
    text = pkg.list_str_to_tensor([bench.TEXT[i % 2] for i in range(cfg['batch'])]).to(dev)
    steps = {'8x64': step_call(8, 64, dev, mel, text), '4x128': step_call(4, 128, dev, mel, text)}
    torch.cuda.synchronize()
    res[cfg['name'] + ' training step, dropout 0.1, CUDA graph'] = alternate(steps, rounds, per_round, warmup)
    res['card_after'] = card()
    for key, val in res.items():
        if isinstance(val, dict) and all(isinstance(r, dict) and 'median_ms' in r for r in val.values()):
            print(key)
            for lab, r in val.items():
                print(f'  {lab}: median {r["median_ms"]:.3f} ms over {r["calls"]} calls (round medians {r["round_median_min_ms"]:.3f}-'
                      f'{r["round_median_max_ms"]:.3f})')
    print(json.dumps(res))


if __name__ == '__main__':
    main()
