"""The reference dataset's resampling (trainer.py:116-118: torchaudio.transforms.Resample(sample_rate, target) in fp32, per item)
restated in float64: torchaudio's tap construction, its output length, the resample itself, and the element-wise bound of the CUDA
kernel (csrc/resample.cu) around it; plus the golden cases that pin collate() to the reference's HFDataset + collate_fn
(tools/make_resample_golden.py, tests/golden/reference/resample_<case>.pt).

torchaudio (functional._get_sinc_resample_kernel with dtype=None, _apply_sinc_resample_kernel): the rates reduced by their gcd to
orig', new'; base = 0.99 min(orig', new'); width = ceil(6 orig' / base); phase k, column c of the [new', 2 width + orig'] table is
    t = (float32(-k / new') + (c - width) / orig') * base, clamped to [-6, 6];
    tap = (t == 0 ? 1 : sin(pi t) / (pi t)) * cos(pi t / 12)^2 * base / orig'   (float64, rounded once to float32)
— the phase offset is an int64 arange divided by new', which torch does in float32 before promoting. Output j = q new' + k sums
tap[k, c] x[q orig' - width + c] over c, x zero outside the item; the output has ceil(float32(new' L / orig')) samples.
"""
import math

import numpy as np
import torch

from kernel_checks import F64, gamma

LOWPASS, ROLLOFF = 6, 0.99


def reduced(orig, new):
    g = math.gcd(orig, new)
    return orig // g, new // g


def table_width(orig, new):
    o, n = reduced(orig, new)
    return math.ceil(LOWPASS * o / (min(o, n) * ROLLOFF))


def taps_full(orig, new, phases=None):
    """torchaudio's fp32 table [new', 2 width + orig'], or only the rows `phases` of it (the table of a large coprime pair does not
    fit in memory; each element is computed on its own, so a row subset has the same bits)"""
    o, n = reduced(orig, new)
    base = min(o, n) * ROLLOFF
    width = table_width(orig, new)
    idx = torch.arange(-width, width + o, dtype=F64)[None] / o
    kt = torch.arange(0, -n, -1)[:, None] / n
    if phases is not None:
        kt = kt[torch.as_tensor(phases)]
    t = (kt + idx) * base
    t = t.clamp(-LOWPASS, LOWPASS)
    window = torch.cos(t * math.pi / LOWPASS / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.tensor(1.0, dtype=F64), t.sin() / t)
    k = k * (window * (base / o))
    return k.to(torch.float32)


def expand_banded(first, count, taps, ncols):
    """the package's banded table (ops.resample_taps) as a full [new', ncols] fp32 table, +0 outside the bands"""
    full = torch.zeros((first.shape[0], ncols), dtype=torch.float32)
    off = 0
    for k in range(first.shape[0]):
        c, f = int(count[k]), int(first[k])
        full[k, f:f + c] = taps[off:off + c]
        off += c
    return full


def banded(full):
    """(first, count, taps) of a full fp32 table: each phase's run from its first to its last non-zero tap"""
    nz = full != 0
    col = torch.arange(full.shape[1])
    lo = torch.where(nz, col, full.shape[1]).min(1).values
    hi = torch.where(nz, col, -1).max(1).values
    keep = (col >= lo[:, None]) & (col <= hi[:, None])
    return lo, hi - lo + 1, full[keep]


def out_length(n, orig, new):
    """torchaudio's ceil(torch.as_tensor(new' n / orig')): the quotient rounded to float32 before the ceil"""
    o, w = reduced(orig, new)
    return min(math.ceil(np.float32(w * n / o)), w * (n // o + 1))


def resample64(x, orig, new, first, count, taps, bound=False):
    """float64 resample of the fp32 samples x [L] with the banded fp32 taps (exact products, exact sums) -> [out_length]; with bound,
    also the kernel's element-wise bound gamma_K sum |w x| over the K non-zero taps of the output's phase (one fma chain: K
    roundings)"""
    o, n = reduced(orig, new)
    L = x.shape[0]
    nout = out_length(L, orig, new)
    width = table_width(orig, new)
    x64 = x.to(F64)
    j = torch.arange(nout)
    k, q = j % n, j // n
    kmax = int(count.max())
    i = torch.arange(kmax)
    off = torch.cumsum(count, 0) - count
    valid = i[None] < count[k][:, None]
    m = (q * o - width + first[k])[:, None] + i[None]
    xv = torch.where(valid & (m >= 0) & (m < L), x64[m.clamp(0, max(L - 1, 0))] if L else torch.zeros(()), torch.zeros((), dtype=F64))
    w = torch.where(valid, taps.to(F64)[(off[k][:, None] + i[None]).clamp(max=taps.numel() - 1)], torch.zeros((), dtype=F64))
    y = (w * xv).sum(1)
    if not bound:
        return y
    return y, gamma(count[k].to(F64)) * (w * xv).abs().sum(1)


def resample_item(x, orig, new, bound=False):
    """resample64 of one item with torchaudio's taps restated here (the item itself when the rates are equal, bound 0)"""
    if orig == new:
        y = x.to(F64)
        return (y, torch.zeros_like(y)) if bound else y
    first, count, taps = banded(taps_full(orig, new))
    return resample64(x, orig, new, first, count, taps, bound)


# ------------------------------------------------------------------------------------------------------------- golden cases
# name -> target rate and items (rate, samples, seed): every item within HFDataset's 0.3-20 s window. The waves are
# randn(samples, seed) * 0.3, stored by the dataset as float32 arrays. `quirk`: 400 055 samples at 44.1 kHz resample to 217 717
# samples (float32 ceil), not the exact 217 718: the same 851 frames (no length within 20 s at the common rates moves the frame
# count), but the last frames reflect the wave about its last sample.
RESAMPLE_CASES = {
    'mixed24k': dict(target=24000, items=[(16000, 8000, 1), (22050, 7000, 2), (24000, 7300, 3), (44100, 15435, 4), (48000, 14881, 5)]),
    'mixed16k': dict(target=16000, items=[(22050, 6700, 6), (44100, 13300, 7), (16000, 5001, 8), (48000, 15000, 9), (24000, 7777, 10)]),
    'quirk': dict(target=24000, items=[(44100, 400055, 11), (48000, 14500, 12), (22050, 6616, 13)]),
}
MEL_SAMPLE = 8192     # stored mel elements per case (seeded flat indices, oracle.reference_cases.sample_index)
TAIL = 5              # last frames of each item stored in full: the frames whose reflect padding reaches the item's end


def case_wave(rate, samples, seed):
    return (torch.randn(samples, generator=torch.Generator().manual_seed(seed)) * 0.3).to(torch.float32)


def case_waves(name):
    c = RESAMPLE_CASES[name]
    return [case_wave(*it) for it in c['items']], [it[0] for it in c['items']], c['target']
