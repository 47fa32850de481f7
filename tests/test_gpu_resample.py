"""GPU: b200_resample (csrc/resample.cu), the resampling of a ragged mixed-rate batch ahead of the mel, and MelSpec.collate with
sample_rates.

Kernel: called through the C ABI with NaN-filled outputs and NaN past each item's length in the input; every output is held to the
float64 restatement of tests/resample_ref.py (exact products and sums of the fp32 taps and samples) within gamma_K sum |w x| over the
K non-zero taps of its phase, the lengths to torchaudio's float32-ceil length, the padding to +0. Exact properties: equal-rate items
are bit copies, an item launched alone gives the bits it gets in a batch, a CUDA graph replay gives the eager bits. Module: collate
with sample_rates is ops.resample followed by the ragged collate, bit for bit; it matches the reference's HFDataset + collate_fn
(tests/golden/reference/resample_*.pt); without resampling it is the same code path as without sample_rates: no extra launch.
"""
import math

import pytest
import torch

from kernel_checks import F32, check_e, check_f, dev, gen, pkg, stream  # noqa: F401 (pkg: the fixture)
from oracle import reference_cases as RC
from resample_ref import MEL_SAMPLE, RESAMPLE_CASES, TAIL, case_waves, out_length, resample64, table_width

pytestmark = pytest.mark.gpu

RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000, 88200, 96000)
PAIRS = [(r, t) for t in (24000, 16000) for r in RATES if r != t] + [(44101, 24000)]


def launch(pkg, wave, lens, idx, table, nr):
    """b200_resample with NaN-filled outputs and out_lens preset to -1"""
    B, nw = wave.shape
    out = torch.full((B, nr), float('nan'), device=dev(), dtype=F32)
    out_lens = torch.full((B,), -1, device=dev(), dtype=torch.int32)
    pairs, phases, taps = table.pointers()
    a = pkg.lib.make_args('b200_resample_args', wave=wave, wave_lens=lens, pair_idx=idx, pairs=pairs, phases=phases, taps=taps, out=out,
                          out_lens=out_lens, B=B, nw=nw, nr=nr, n_pairs=table.n_pairs, max_pair_words=table.max_pair_words)
    pkg.lib.call('b200_resample', a, stream())
    return out, out_lens


def ragged(lengths, seed, nw=None):
    """seeded items at 0.3 rms in a [B, nw] buffer, NaN past each item's length (never to be read)"""
    nw = nw or max(max(lengths), 1)
    g = gen(seed)
    wave = torch.full((len(lengths), nw), float('nan'))
    for i, n in enumerate(lengths):
        wave[i, :n] = torch.randn(n, generator=g) * 0.3
    return wave


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device=dev())


def check_item(pkg, name, got, got_len, x, orig, new, nr):
    """one output row against the restatement with the package's banded taps; +0 past its length"""
    _, _, _, first, count, taps = pkg.ops.resample_taps(orig, new)
    n = min(out_length(x.shape[0], orig, new), nr)
    assert int(got_len) == n, (name, int(got_len), n)
    ref, bound = resample64(x, orig, new, first.long(), count.long(), taps, bound=True)
    check_f(name, got[:n], ref[:n], bound[:n])
    check_e(f'{name} padding', got[n:], torch.zeros_like(got[n:]))


def lengths_for(orig, new):
    o = orig // math.gcd(orig, new)
    w = table_width(orig, new)
    ls = [0, 1, w - 1, o, 3 * o, 3 * o + 1, 4801]
    if (orig, new) in ((44100, 24000), (22050, 24000)):
        ls.append(400055)                   # float32-ceil length
    if orig == 48000:
        ls.append(20 * 48000)               # 20 s at 48 kHz
    return ls


@pytest.mark.parametrize('orig,new', PAIRS, ids=[f'{o}-{n}' for o, n in PAIRS])
def test_resample_kernel_bounds(pkg, orig, new):
    """lengths 0, 1, < width, multiples of orig', a float32-ceil length and 20 s at 48 kHz in one ragged launch: every output within
    the element-wise bound, out_lens torchaudio's, +0 padding, and the NaN past each item's length never read"""
    lens = lengths_for(orig, new)
    wave = ragged(lens, seed=orig + new)
    table = pkg.ops.ResampleTable([(orig, new)], device=dev())
    nr = max(out_length(n, orig, new) for n in lens)
    out, out_lens = launch(pkg, wave.to(dev()), i32(lens), i32([0] * len(lens)), table, nr)
    torch.cuda.synchronize()
    out, out_lens = out.cpu(), out_lens.cpu()
    assert not bool(torch.isnan(out).any())
    for i, n in enumerate(lens):
        check_item(pkg, f'{orig}->{new} len {n}', out[i], out_lens[i], wave[i, :n], orig, new, nr)


MIXED = [(44100, 400055 // 8), (22050, 7001), (16000, 16000 * 2 + 5), (24000, 12345), (48000, 15000), (44101, 9999), (8000, 1),
         (96000, 0), (24000, 0)]


def mixed_batch(pkg, target=24000, seed=3):
    lens = [n for _, n in MIXED]
    wave = ragged(lens, seed)
    pairs = sorted({(r, target) for r, _ in MIXED if r != target})
    table = pkg.ops.ResampleTable(pairs, device=dev())
    idx = [table.index[(r, target)] if r != target else -1 for r, _ in MIXED]
    nr = max(out_length(n, r, target) if r != target else n for r, n in MIXED)
    return wave, lens, table, idx, nr


def test_mixed_batch_one_launch(pkg):
    """every rate pair and equal-rate items in ONE launch (one b200 launch counted): each item within its bound, equal-rate items
    bit copies, NaN past each length never read, +0 padding"""
    wave, lens, table, idx, nr = mixed_batch(pkg)
    wd = wave.to(dev())
    n0 = pkg.lib.launch_count()
    out, out_lens = launch(pkg, wd, i32(lens), i32(idx), table, nr)
    assert pkg.lib.launch_count() - n0 == 1
    out, out_lens = out.cpu(), out_lens.cpu()
    assert not bool(torch.isnan(out).any())
    for i, (r, n) in enumerate(MIXED):
        if r == 24000:
            assert int(out_lens[i]) == n
            check_e(f'item {i} copy', out[i, :n], wave[i, :n])
            check_e(f'item {i} padding', out[i, n:], torch.zeros_like(out[i, n:]))
        else:
            check_item(pkg, f'item {i} ({r} Hz, {n})', out[i], out_lens[i], wave[i, :n], r, 24000, nr)


def test_each_item_alone_is_bit_identical(pkg):
    """an item launched alone (B = 1, its own width) gives the bits of the batched launch"""
    wave, lens, table, idx, nr = mixed_batch(pkg, seed=4)
    wd = wave.to(dev())
    out, out_lens = launch(pkg, wd, i32(lens), i32(idx), table, nr)
    for i, n in enumerate(lens):
        alone = wd[i:i + 1, :max(n, 1)].contiguous()
        m = int(out_lens[i])
        o1, l1 = launch(pkg, alone, i32([n]), i32([idx[i]]), table, max(m, 1))
        assert int(l1[0]) == m
        check_e(f'item {i}', o1[0, :m], out[i, :m])


def test_graph_replay_gives_the_eager_bits(pkg):
    wave, lens, table, idx, nr = mixed_batch(pkg, seed=5)
    wd, ld, xd = wave.to(dev()), i32(lens), i32(idx)
    eager, eager_lens = pkg.ops.resample(wd, ld, xd, table, nr)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pkg.ops.resample(wd, ld, xd, table, nr)      # warm-up off the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, out_lens = pkg.ops.resample(wd, ld, xd, table, nr)
    out.fill_(float('nan'))
    out_lens.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    check_e('graph replay', out, eager)
    check_e('graph replay lengths', out_lens, eager_lens)


# ======================================================================================================== MelSpec.collate
def test_collate_is_resample_then_ragged_collate(pkg):
    """collate(waves, sample_rates) = ops.resample, then today's ragged collate of its output, bit for bit — for a list and for a
    padded tensor with lengths; n_frames_max from the longest resampled item (list) or from the padded width (tensor)"""
    ms = pkg.MelSpec().to(dev())
    keys = set(ms.state_dict())
    rates = [r for r, _ in MIXED[:6]]
    lens = [n for _, n in MIXED[:6]]
    wave = ragged(lens, seed=6).nan_to_num(0.0)
    waves = [wave[i, :n] for i, n in enumerate(lens)]
    batch = ms.collate(waves, sample_rates=rates)
    assert set(ms.state_dict()) == keys
    table = ms._resample_table
    idx = i32([table.index[(r, 24000)] if r != 24000 else -1 for r in rates])
    nr = max(out_length(n, r, 24000) if r != 24000 else n for r, n in zip(rates, lens))
    out, out_lens = pkg.ops.resample(wave.to(dev()), i32(lens), idx, table, nr)
    want = ms.collate([out[i, :int(n)] for i, n in enumerate(out_lens.tolist())])
    check_e('list mel', batch['mel'], want['mel'])
    assert torch.equal(batch['mel_lengths'].cpu(), want['mel_lengths'].cpu())
    # padded tensor + lengths: the output width is the padded width resampled at the slowest conversion present
    b2 = ms.collate(wave.to(dev()), lens=torch.tensor(lens), sample_rates=torch.tensor(rates))
    nr2 = max(out_length(wave.shape[1], r, 24000) if r != 24000 else wave.shape[1] for r in set(rates))
    out2, out_lens2 = pkg.ops.resample(wave.to(dev()), i32(lens), idx, table, nr2)
    want2 = ms.collate(out2, lens=out_lens2)
    assert b2['mel'].shape[1] == ms.frames(nr2)
    check_e('tensor mel', b2['mel'], want2['mel'])
    assert torch.equal(b2['mel_lengths'].cpu(), want2['mel_lengths'].cpu())
    assert torch.equal(b2['mel_lengths'].cpu()[:len(lens)], batch['mel_lengths'].cpu())


@pytest.mark.parametrize('name', list(RESAMPLE_CASES))
def test_collate_vs_reference(pkg, name):
    """collate(waves as stored, sample_rates) against the reference's HFDataset + collate_fn: mel_lengths exactly, the mel (sampled
    elements and each item's last frames) within the mel golden tolerance 1e-3"""
    g = RC.load('resample_' + name)
    waves, rates, target = case_waves(name)
    ms = pkg.MelSpec(sampling_rate=target).to(dev())
    batch = ms.collate(waves, sample_rates=rates)
    assert torch.equal(batch['mel_lengths'].cpu(), g['mel_lengths'])
    mel = batch['mel'].transpose(1, 2).cpu()
    assert tuple(mel.shape) == g['mel_shape']
    got = mel.flatten()[RC.sample_index(mel.numel(), MEL_SAMPLE)]
    assert float((got - g['mel_values']).abs().max()) < 1e-3
    tail = torch.stack([mel[b, :, n - TAIL:n] for b, n in enumerate(g['mel_lengths'].tolist())])
    assert float((tail - g['mel_tail']).abs().max()) < 1e-3


def test_default_path_is_unchanged(pkg):
    """sample_rates=None and rates all equal to sampling_rate take today's path: the same bits, the same launches, no resampling"""
    ms = pkg.MelSpec().to(dev())
    g = gen(8)
    waves = [torch.randn(n, generator=g) * 0.3 for n in (24000, 7001, 12000)]
    n0 = pkg.lib.launch_count()
    base = ms.collate(waves)
    per_call = pkg.lib.launch_count() - n0
    for rates in (24000, [24000, 24000, 24000], torch.tensor([24000] * 3)):
        n0 = pkg.lib.launch_count()
        b = ms.collate(waves, sample_rates=rates)
        assert pkg.lib.launch_count() - n0 == per_call
        check_e('mel', b['mel'], base['mel'])
        assert torch.equal(b['mel_lengths'], base['mel_lengths'])
    assert ms._resample_table is None and 'resample_taps' not in dict(ms.named_buffers())
    n0 = pkg.lib.launch_count()
    ms.collate(waves, sample_rates=[24000, 44100, 24000])
    assert pkg.lib.launch_count() - n0 == per_call + 1
