"""Time Vocos.decode at cfg5's output shape (B 8, 2048 frames, vocos-mel-24khz geometry, seeded random weights from tests/vocos_ref.py):
median time per call over alternating rounds, kernel launches per call, and the GEMM share of the kernel time (torch.profiler, in a
separate pass). As a comparison point in the same process, the fp32 torch restatement run eagerly on the same GPU, item by item as the
reference's sample() loop does (e2_tts.py:1440-1451). Prints one JSON line; writes under --out if given.

    python tools/vocos_bench.py [--rounds 5] [--calls 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import vocos_ref as V  # noqa: E402

import e2_tts_pytorch_b200 as pkg  # noqa: E402


def timed(fn, calls):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=2048)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    g = V.MEL_24KHZ
    with tempfile.TemporaryDirectory() as d:
        sd = V.write_checkpoint(d, g, 1)
        voc = pkg.Vocos.from_pretrained(d).to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    B, T = args.batch, args.frames
    mel = (torch.randn(B, T, g['input_channels'], generator=torch.Generator().manual_seed(0)) * 2 - 4).to(dev)
    lens = torch.full((B,), T, dtype=torch.int32)

    def kernels():
        return voc.decode_padded(mel, lens, db_to_amp=True)

    def eager():
        with torch.no_grad():
            return [V.decode(sd, g, torch.pow(torch.pow(10.0, 0.1 * mel[b]), 0.5).t()[None]) for b in range(B)]

    for fn in (kernels, eager):   # warm every shape of the timed window
        fn()
    n0 = pkg.lib.launch_count()
    kernels()
    torch.cuda.synchronize()
    launches = pkg.lib.launch_count() - n0
    k_ms, e_ms = [], []
    for _ in range(args.rounds):   # alternate the two so drift on a shared host hits both
        k_ms.append(timed(kernels, args.calls))
        e_ms.append(timed(eager, max(1, args.calls // 5)))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            kernels()
        torch.cuda.synchronize()
    total = gemm = 0.
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        total += t
        if 'gemm_wgmma_kernel' in ev.key:
            gemm += t
    flop = 2 * B * T * (7 * g['input_channels'] * g['dim'] + g['num_layers'] * 2 * g['dim'] * g['intermediate_dim'] +
                        g['dim'] * (g['n_fft'] + 2))
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps(dict(card=card, batch=B, frames=T, kernels_ms_median=statistics.median(k_ms), kernels_ms_rounds=k_ms,
                          eager_fp32_ms_median=statistics.median(e_ms), eager_fp32_ms_rounds=e_ms, launches_per_call=launches,
                          gemm_share_of_kernel_time=gemm / total if total else None, gemm_tflop_per_call=flop / 1e12)))


if __name__ == '__main__':
    main()
