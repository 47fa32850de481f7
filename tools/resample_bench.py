"""Time MelSpec.collate with resampling — one b200_resample launch over a mixed-rate ragged batch, then the mel launch — against
  (a) torchaudio.transforms.Resample, one per rate pair, moved to the GPU and applied item by item, then the same collate; and
  (b) the reference dataset's per-item CPU path (trainer.py:116-122: Resample, then the MelSpectrogram + log of its MelSpec, per
      item, at the host thread count reported), then the padding of collate_fn.
Workload: 32 items of 2-15 s (seeded) at 16, 22.05, 44.1 and 48 kHz in turn, into 24 kHz; the waves are already on the GPU for the
GPU paths and on the host for (b). CUDA events around `iters` calls after warm-up, the paths alternated over `repeats` rounds;
medians and spreads. The resample kernel is also timed alone and reported as achieved HBM bandwidth (4 B read per input sample,
4 B written per output sample, the zero padding included) against the H100 SXM data-sheet 3.35 TB/s, with the card's name and power
limit read in the same run.

    python tools/resample_bench.py [--iters 20] [--repeats 5] [--cpu-repeats 3] [--out result.json]
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
import e2_tts_pytorch_b200 as pkg  # noqa: E402

RATES = (16000, 22050, 44100, 48000)
TARGET = 24000
HBM_PEAK = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def gpu_time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def summary(ts):
    return dict(median_ms=statistics.median(ts), min_ms=min(ts), max_ms=max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--cpu-repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'resample_bench.py measures on the GPU'
    import torchaudio
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    seconds = 2 + 13 * torch.rand(32, generator=g)
    rates = [RATES[i % len(RATES)] for i in range(32)]
    host = [torch.randn(int(s * r), generator=g) * 0.3 for s, r in zip(seconds.tolist(), rates)]
    waves = [w.to(dev) for w in host]
    ms = pkg.MelSpec().to(dev)

    ta_gpu = {r: torchaudio.transforms.Resample(r, TARGET).to(dev) for r in set(rates)}
    ta_cpu = {r: torchaudio.transforms.Resample(r, TARGET) for r in set(rates)}
    mel_cpu = torchaudio.transforms.MelSpectrogram(sample_rate=TARGET, n_fft=1024, win_length=1024, hop_length=256, n_mels=100,
                                                   power=1, center=True, normalized=False, norm=None)

    def ours():
        return ms.collate(waves, sample_rates=rates)

    def torchaudio_gpu():
        return ms.collate([ta_gpu[r](w) for w, r in zip(waves, rates)])

    def reference_cpu():
        mels = [mel_cpu(ta_cpu[r](w)[None]).clamp(min=1e-5).log()[0] for w, r in zip(host, rates)]
        n = max(m.shape[-1] for m in mels)
        return torch.stack([torch.nn.functional.pad(m, (0, n - m.shape[-1])) for m in mels])

    # the resample launch alone, on the padded batch collate builds
    lens = torch.tensor([w.shape[0] for w in host], dtype=torch.int32)
    padded = torch.zeros(32, int(lens.max()))
    for i, w in enumerate(host):
        padded[i, :w.shape[0]] = w
    padded, lens_d = padded.to(dev), lens.to(dev)
    table = ms._rate_table(rates, dev)
    idx = torch.tensor([table.index[(r, TARGET)] for r in rates], dtype=torch.int32, device=dev)
    nr = max(pkg.ops.resample_length(int(n), r, TARGET) for n, r in zip(lens.tolist(), rates))

    def kernel():
        return pkg.ops.resample(padded, lens_d, idx, table, nr)

    out, out_lens = kernel()
    in_samples, out_samples = int(lens.sum()), 32 * nr
    ref_lens = torch.tensor([pkg.ops.resample_length(int(n), r, TARGET) for n, r in zip(lens.tolist(), rates)], dtype=torch.int32)
    assert torch.equal(out_lens.cpu(), ref_lens)
    a, b = ours(), torchaudio_gpu()
    assert torch.equal(a['mel_lengths'], b['mel_lengths'])
    diff_vs_torchaudio = float((a['mel'] - b['mel']).abs().max())

    for fn in (ours, torchaudio_gpu, kernel):
        for _ in range(3):
            fn()
    reference_cpu()
    torch.cuda.synchronize()
    times = {'collate_resample': [], 'torchaudio_gpu_per_item_then_collate': [], 'resample_kernel_alone': []}
    cpu_times = []
    for r in range(args.repeats):
        times['collate_resample'].append(gpu_time(ours, args.iters))
        times['torchaudio_gpu_per_item_then_collate'].append(gpu_time(torchaudio_gpu, args.iters))
        times['resample_kernel_alone'].append(gpu_time(kernel, args.iters * 5))
        if r < args.cpu_repeats:
            t0 = time.perf_counter()
            reference_cpu()
            cpu_times.append((time.perf_counter() - t0) * 1e3)
    gpu, limit = card()
    k = statistics.median(times['resample_kernel_alone']) * 1e-3
    bytes_moved = 4 * (in_samples + out_samples)
    res = dict(gpu=gpu, power_limit_and_max_sm_clock=limit, batch='32 items of 2-15 s at 16 / 22.05 / 44.1 / 48 kHz -> 24 kHz',
               audio_seconds=float(seconds.sum()), iters=args.iters, repeats=args.repeats,
               results={k_: summary(v) for k_, v in times.items()},
               reference_cpu_per_item=dict(summary(cpu_times), host_threads=torch.get_num_threads(), rounds=len(cpu_times)),
               resample_kernel=dict(input_samples=in_samples, output_samples_incl_padding=out_samples, bytes=bytes_moved,
                                    achieved_GBps=bytes_moved / k / 1e9, share_of_3p35TBps=bytes_moved / k / HBM_PEAK),
               max_abs_mel_diff_vs_torchaudio_gpu_path=diff_vs_torchaudio)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
