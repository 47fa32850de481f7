"""Developer tool (GPU): per-shape-group timing of the GEMMs of one training step.

    python tools/gemm_step_bench.py [--config 2|3|4] [--reps 7] [--profile DIR]

Records every `ops.gemm` call of one eager step the way bench.py's roofline pass does (live operands), groups the calls by
(M, N, K, operand majors, split-K, epilogue), and replays each group as one CUDA graph between one CUDA-event pair (median of
`--reps` replays). Prints one row per group: calls per step, µs per step, TF/s, share of the family total; then the whole list
replayed as one graph (bench.py's `roofline` figure). `B200_LIB=<path>` runs another build of the same ABI, for A/B tables.

`--profile DIR` instead runs one eager step under torch.profiler (CUDA activities) and prints the device time per kernel family
(GEMM, attention forward / backward, hyper-connections, geglu_bwd, the rest); the trace goes to DIR.
"""
import argparse
import os
import random
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

CONFIGS = {2: dict(dim=512, depth=8, heads=8, batch=16, seq=1024, kind='train'),
           3: dict(dim=1024, depth=24, heads=16, batch=4, seq=2048, kind='train'),
           4: dict(dim=512, depth=8, heads=8, batch=32, seq=1024, kind='duration')}


def make_step(cfg, dev):
    import e2_tts_pytorch_b200 as pkg
    torch.manual_seed(0)
    random.seed(0)
    tkw = dict(dim=cfg['dim'], depth=cfg['depth'], heads=cfg['heads'], dropout=0.1)
    if cfg['kind'] == 'duration':
        model = pkg.DurationPredictor(transformer=tkw).to(dev)
    else:
        model = pkg.E2TTS(transformer=tkw, use_vocos=False).to(dev)
        model.cond_drop_prob = 0.0
    model.train()
    mel = torch.randn(cfg['batch'], cfg['seq'], 100, device=dev)
    text = pkg.list_str_to_tensor([['Hello', 'Goodbye'][i % 2] for i in range(cfg['batch'])]).to(dev)

    def step():
        out = model(mel, text=text)
        (out if cfg['kind'] == 'duration' else out.loss).backward()
        for p in model.parameters():
            p.grad = None
    return step


def group_key(M, N, K, kw):
    epi = ''.join(c for c, on in (('b', kw.get('bias') is not None), ('g', kw.get('colscale') is not None),
                                  ('m', kw.get('rowmask') is not None), ('r', kw.get('resid') is not None),
                                  ('G', bool(kw.get('geglu'))), ('d', kw.get('D2') is not None),
                                  ('2', kw.get('A2') is not None), ('f', bool(kw.get('out_fp32')))) if on) or '-'
    majors = ('T' if kw.get('a_mn') else 'N') + ('T' if kw.get('b_mn') else 'N')
    return (M, N, K, majors, kw.get('split_k', 1), epi)


def time_graph(gemm, calls, reps):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for c in calls:   # warm the descriptor cache and the one-time kernel attributes off the capture
            gemm(c[0], c[1], c[2], c[3], c[4], **c[5])
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for c in calls:
            gemm(c[0], c[1], c[2], c[3], c[4], **c[5])
    g.replay()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3)
    del g
    times.sort()
    return times[len(times) // 2]


def gemm_table(cfg, dev, reps):
    from e2_tts_pytorch_b200 import ops
    step = make_step(cfg, dev)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    calls = []
    orig = ops.gemm

    def recorded(A, Bm, M, N, K, **kw):
        out = orig(A, Bm, M, N, K, **kw)
        kw2 = dict(kw)
        kw2['out'] = out
        calls.append((A, Bm, M, N, K, kw2))
        return out
    ops.gemm = recorded
    try:
        step()
    finally:
        ops.gemm = orig
    torch.cuda.synchronize()
    groups = OrderedDict()
    for c in calls:
        groups.setdefault(group_key(c[2], c[3], c[4], c[5]), []).append(c)
    rows = []
    for key, cs in groups.items():
        us = time_graph(orig, cs, reps)
        flops = sum(2.0 * c[2] * c[3] * c[4] for c in cs)
        rows.append((key, len(cs), us, flops))
    total_us = time_graph(orig, calls, reps)
    total_flops = sum(r[3] for r in rows)
    sum_us = sum(r[2] for r in rows)
    rows.sort(key=lambda r: -r[2])
    print(f'{"M":>6} {"N":>5} {"K":>6} {"maj":>3} {"split":>5} {"epi":>5} {"calls":>5} {"us/step":>9} {"TF/s":>6} {"share":>6}')
    for (M, N, K, maj, split, epi), n, us, fl in rows:
        print(f'{M:6d} {N:5d} {K:6d} {maj:>3} {split:5d} {epi:>5} {n:5d} {us:9.1f} {fl / us / 1e6:6.1f} {us / sum_us:6.1%}')
    print(f'groups: {len(rows)}, calls: {len(calls)}, sum of groups {sum_us:.1f} us; whole list as one graph {total_us:.1f} us = '
          f'{total_flops / total_us / 1e6:.1f} TF/s ({total_flops / 1e12:.2f} TFLOP)')
    print('epi: b bias, g AdaLN gate (colscale), m row mask, r residual, G GEGLU, d saved GEGLU pre-activations, 2 two-source K, f fp32 out')


FAMILIES = (('gemm', ('gemm_wgmma',)), ('attn_fwd', ('attn_fwd',)), ('attn_bwd', ('attn_bwd', 'attn_prep')), ('hc', ('hc_',)),
            ('geglu_bwd', ('geglu_bwd',)))


def profile_step(cfg, dev, outdir):
    from torch.profiler import ProfilerActivity, profile
    step = make_step(cfg, dev)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    os.makedirs(outdir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(outdir, 'step.pt.trace.json'))
    fam, per_kernel = OrderedDict((f, 0.0) for f, _ in FAMILIES), {}
    fam['other'] = 0.0
    for ev in prof.key_averages():
        us = getattr(ev, 'device_time_total', None)
        if us is None:
            us = ev.cuda_time_total
        if us <= 0 or ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per_kernel[ev.key] = per_kernel.get(ev.key, 0.0) + us
        f = next((f for f, pats in FAMILIES if any(p in ev.key for p in pats)), 'other')
        fam[f] += us
    total = sum(fam.values())
    print(f'device time of one eager step: {total / 1e3:.2f} ms (kernels and memsets, summed over streams)')
    for f, us in fam.items():
        print(f'  {f:10s} {us / 1e3:8.2f} ms {us / total:6.1%}')
    print('top kernels:')
    for k, us in sorted(per_kernel.items(), key=lambda kv: -kv[1])[:25]:
        print(f'  {us / 1e3:8.2f} ms  {k[:110]}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', type=int, default=2, choices=sorted(CONFIGS))
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--profile', metavar='DIR', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    print(f'{torch.cuda.get_device_name(dev)}, lib {os.environ.get("B200_LIB", "in-tree")}, cfg{args.config}', flush=True)
    if args.profile:
        profile_step(CONFIGS[args.config], dev, args.profile)
    else:
        gemm_table(CONFIGS[args.config], dev, args.reps)


if __name__ == '__main__':
    main()
