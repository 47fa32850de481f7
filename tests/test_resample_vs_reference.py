"""CPU: resampling ahead of the mel (trainer.py:116-118, torchaudio.transforms.Resample per item). The float64 restatement of
tests/resample_ref.py against torchaudio (taps bit for bit, the resample in float64, the float32 length) and, with the existing
float64 mel restatement, against what the reference's HFDataset + collate_fn computed (tests/golden/reference/resample_*.pt,
tools/make_resample_golden.py); the package's banded tap tables against the restated ones; the refusals of MelSpec.collate and of
the C ABI (before any launch); the state_dict of a MelSpec that holds tap tables."""
import pytest
import torch

from mel_kwargs_ref import mel_of_module
from oracle import reference_cases as RC
from resample_ref import (MEL_SAMPLE, RESAMPLE_CASES, TAIL, banded, case_waves, expand_banded, out_length, reduced, resample64,
                          resample_item, table_width, taps_full)

import e2_tts_pytorch_b200 as pkg

RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000, 88200, 96000)
PAIRS = [(r, t) for t in (24000, 16000) for r in RATES if r != t]


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('orig,new', PAIRS, ids=[f'{o}-{n}' for o, n in PAIRS])
def test_taps_bit_identical_to_torchaudio(orig, new):
    """the restated table equals torchaudio.transforms.Resample(orig, new).kernel bit for bit (zeros' signs included); the package's
    banded table holds exactly its non-zero runs"""
    ta = pytest.importorskip('torchaudio')
    t = ta.transforms.Resample(orig, new)
    want = t.kernel[:, 0]
    full = taps_full(orig, new)
    assert t.width == table_width(orig, new) and torch.equal(_bits(full), _bits(want))
    o, n, width, first, count, taps = pkg.ops.resample_taps(orig, new)
    assert (o, n, width) == (*reduced(orig, new), t.width)
    f2, c2, t2 = banded(full)
    assert torch.equal(first.long(), f2) and torch.equal(count.long(), c2) and torch.equal(_bits(taps), _bits(t2))
    assert torch.equal(expand_banded(first, count, taps, full.shape[1]), full)     # +0 == -0: the rest is zeros


def test_taps_of_a_coprime_pair():
    """44 101 -> 24 000 (24 000 phases of 44 125 stored taps; torchaudio's table would take 8.5 GB in float64): the banded table
    against the restated rows of 128 seeded phases and the first and last phase"""
    o, n, width, first, count, taps = pkg.ops.resample_taps(44101, 24000)
    assert (o, n, width) == (44101, 24000, table_width(44101, 24000)) and first.shape == (24000,)
    rows = sorted(set(torch.randperm(n, generator=torch.Generator().manual_seed(0))[:128].tolist()) | {0, n - 1})
    full = taps_full(44101, 24000, rows)
    off = torch.cumsum(count.long(), 0) - count.long()
    for r, k in enumerate(rows):
        f, c = int(first[k]), int(count[k])
        band = taps[int(off[k]):int(off[k]) + c]
        assert torch.equal(_bits(full[r, f:f + c]), _bits(band)), k
        assert bool((full[r, :f] == 0).all() and (full[r, f + c:] == 0).all()), k
    assert int(count.max()) <= 25


def test_band_widths():
    """non-zero taps per phase: at most 25 for the common rates into 24 kHz, 49 from 96 kHz, 37 for 48 -> 16 kHz"""
    widest = {p: int(pkg.ops.resample_taps(*p)[4].max()) for p in PAIRS}
    assert max(widest[(r, 24000)] for r in (16000, 22050, 44100, 48000)) <= 25
    assert widest[(96000, 24000)] == 49 and widest[(48000, 16000)] == 37


FLOAT64_PAIRS = [(44100, 24000), (22050, 24000), (16000, 24000), (48000, 16000), (8000, 24000), (96000, 16000)]


@pytest.mark.parametrize('orig,new', FLOAT64_PAIRS, ids=[f'{o}-{n}' for o, n in FLOAT64_PAIRS])
def test_restated_resample_vs_torchaudio(orig, new):
    """the float64 restatement equals torchaudio's _apply_sinc_resample_kernel run in float64 with the transform's taps to 1e-12;
    the float32 transform (what the dataset runs) stays within the kernel's bound around it"""
    ta = pytest.importorskip('torchaudio')
    from torchaudio.functional.functional import _apply_sinc_resample_kernel
    t = ta.transforms.Resample(orig, new)
    g = torch.Generator().manual_seed(orig + new)
    for L in (1, 7, orig // 100 + 3, 5 * orig // 100 + 17):
        x = torch.randn(L, generator=g) * 0.3
        want = _apply_sinc_resample_kernel(x.double(), orig, new, t.gcd, t.kernel.double(), t.width)
        got, bound = resample_item(x, orig, new, bound=True)
        assert got.shape == want.shape, (L, got.shape, want.shape)
        assert float((got - want).abs().max()) <= 1e-12 * (1 + float(want.abs().max()))
        d = (t(x).double() - got).abs()
        assert bool((d <= bound).all()), (L, float((d / bound.clamp(min=1e-300)).max()))


def test_lengths_vs_torchaudio():
    """output lengths over a sweep of lengths, the float32-ceil lengths included (400 055 at 44.1 kHz: 217 717, one short of the
    exact ceiling), from the restatement and from ops.resample_length"""
    ta = pytest.importorskip('torchaudio')
    for orig, new in [(44100, 24000), (22050, 24000), (48000, 16000), (44101, 24000), (8000, 24000)]:
        o, n = reduced(orig, new)
        lengths = list(range(0, 300)) + [o - 1, o, o + 1, 10 * o, 10 * o + 1, 400055, 240832 + 147 * 3]
        t = ta.transforms.Resample(orig, new) if o < 1000 else None
        quirks = 0
        for L in lengths:
            want = (t(torch.zeros(L)).shape[-1] if L else 0) if t is not None else None   # torchaudio cannot view an empty wave
            got = out_length(L, orig, new)
            assert pkg.ops.resample_length(L, orig, new) == got
            if want is not None:
                assert got == want, (orig, new, L, got, want)
            quirks += got != -(-n * L // o)
        if (orig, new) == (44100, 24000):
            assert out_length(400055, orig, new) == 217717 and quirks >= 1


@pytest.mark.parametrize('name', list(RESAMPLE_CASES))
def test_float64_pipeline_vs_reference(name):
    """restated resample, then the float64 mel restatement, then the zero padding of collate_fn: the reference's mel_lengths
    exactly, its mel (sampled elements and each item's last frames) within 1e-4"""
    g = RC.load('resample_' + name)
    waves, rates, target = case_waves(name)
    assert g['items'] == RESAMPLE_CASES[name]['items'] and g['target'] == target
    ms = pkg.MelSpec(sampling_rate=target)
    mels = [mel_of_module(ms, resample_item(w, r, target)[None])[0] for w, r in zip(waves, rates)]
    lens = torch.tensor([m.shape[1] for m in mels])
    assert torch.equal(lens, g['mel_lengths'])
    mel = torch.stack([torch.nn.functional.pad(m, (0, int(lens.max()) - m.shape[1])) for m in mels])
    assert tuple(mel.shape) == g['mel_shape']
    got = mel.flatten()[RC.sample_index(mel.numel(), MEL_SAMPLE)]
    assert float((got - g['mel_values'].double()).abs().max()) < 1e-4
    tail = torch.stack([mel[b, :, n - TAIL:n] for b, n in enumerate(lens.tolist())])
    assert float((tail - g['mel_tail'].double()).abs().max()) < 1e-4


def test_cases_reach_every_rate():
    """16, 22.05, 24, 44.1 and 48 kHz items into 24 kHz and into 16 kHz, items at the target rate, and a float32-ceil length"""
    for target in (24000, 16000):
        rates = {r for c in RESAMPLE_CASES.values() if c['target'] == target for r, _, _ in c['items']}
        assert {16000, 22050, 24000, 44100, 48000} <= rates
    for c in RESAMPLE_CASES.values():
        for r, n, _ in c['items']:
            assert 0.3 <= n / r <= 20
    assert any(out_length(n, r, c['target']) != -(-reduced(r, c['target'])[1] * n // reduced(r, c['target'])[0])
               for c in RESAMPLE_CASES.values() for r, n, _ in c['items'])


@pytest.mark.parametrize('rates', [[22050.5, 24000], [0, 24000], [-16000, 24000], [16000], 'x', [True, 24000],
                                   torch.tensor([[16000, 24000]]), [float('nan'), 24000]],
                         ids=['fractional', 'zero', 'negative', 'count', 'str', 'bool', '2d', 'nan'])
def test_collate_refuses_bad_rates(rates):
    """sample_rates that are not positive integers, one per item, raise ValueError before anything runs"""
    ms = pkg.MelSpec()
    with pytest.raises(ValueError):
        ms.collate([torch.zeros(4000), torch.zeros(3000)], sample_rates=rates)


def test_collate_rates_accepts_ints_lists_and_tensors():
    f = pkg.MelSpec._collate_rates
    assert f(None, 3) is None and f(16000, 2) == [16000, 16000] and f(44100.0, 1) == [44100]
    assert f(torch.tensor([16000, 48000]), 2) == [16000, 48000] and f(torch.tensor(22050), 2) == [22050, 22050]
    import numpy as np
    assert f(np.array([16000, 48000]), 2) == [16000, 48000] and f(np.int64(22050), 1) == [22050]


def test_tap_tables_stay_out_of_the_state_dict():
    """the tap tables a resampling collate caches are a non-persistent buffer: the state_dict keys are the reference's, and a new
    rate pair extends the table without renumbering the pairs already in it"""
    ms = pkg.MelSpec()
    keys = set(ms.state_dict())
    t1 = ms._rate_table([44100, 24000, 16000], 'cpu')
    assert set(ms.state_dict()) == keys and 'resample_taps' in dict(ms.named_buffers())
    t2 = ms._rate_table([48000], 'cpu')
    assert set(t2.index) == {(44100, 24000), (16000, 24000), (48000, 24000)} and t2.n_pairs == 3
    assert set(ms.state_dict()) == keys and ms._rate_table([16000], 'cpu') is t2 and t1 is not t2
    e = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), use_vocos=False)
    k0 = set(e.state_dict())
    e.mel_spec._rate_table([22050], 'cpu')
    assert set(e.state_dict()) == k0


def test_table_layout():
    """ResampleTable: pair words, phase words and fp32 tap bits in one int32 tensor, as b200_resample reads them"""
    t = pkg.ops.ResampleTable([(44100, 24000), (16000, 24000)])
    d = t.data
    P = pkg.ops.RESAMPLE_PAIR_WORDS
    assert t.n_pairs == 2 and d.dtype == torch.int32
    for p, (orig, new) in enumerate([(44100, 24000), (16000, 24000)]):
        o, n, width, first, count, taps = pkg.ops.resample_taps(orig, new)
        w = d[P * p:P * p + P].tolist()
        assert w[:3] == [o, n, width] and w[5] == taps.numel()
        ph = d[P * 2 + 3 * w[3]:P * 2 + 3 * (w[3] + n)].view(n, 3)
        assert torch.equal(ph[:, 0], first) and torch.equal(ph[:, 1], count)
        base = P * 2 + 3 * t.n_phases + w[4]
        for k in (0, n - 1):
            got = d[base + int(ph[k, 2]):base + int(ph[k, 2]) + int(ph[k, 1])].view(torch.float32)
            assert torch.equal(got, taps[int(ph[k, 2]):int(ph[k, 2]) + int(count[k])])
    assert t.max_pair_words == max(3 * 80 + pkg.ops.resample_taps(44100, 24000)[5].numel(), 3 * 3 + pkg.ops.resample_taps(16000, 24000)[5].numel())


def _abi_args(**kw):
    base = dict(wave=256, wave_lens=256, pair_idx=256, pairs=256, phases=256, taps=256, out=256, out_lens=256, B=2, nw=1000, nr=600,
                n_pairs=1, max_pair_words=100)
    return pkg.lib.make_args('b200_resample_args', **dict(base, **kw))


@pytest.mark.parametrize('kw,msg', [
    (dict(B=0), 'bad shape'), (dict(B=70000), 'bad shape'), (dict(nw=-1), 'bad shape'), (dict(nr=-5), 'bad shape'),
    (dict(n_pairs=-1), 'bad table'), (dict(max_pair_words=-1), 'bad table'), (dict(wave=None), 'null pointer'),
    (dict(out_lens=None), 'null pointer'), (dict(taps=None), 'null table pointer'),
])
def test_c_abi_refusals(kw, msg):
    """b200_resample refuses before any launch (placeholder pointers, never read)"""
    with pytest.raises(RuntimeError, match=msg):
        pkg.lib.call('b200_resample', _abi_args(**kw), None)


def test_banded_restatement_matches_full_convolution():
    """resample64 over the bands equals the full-table strided sum (every column, zeros included) in float64"""
    x = torch.randn(3001, generator=torch.Generator().manual_seed(5))
    full = taps_full(44100, 24000)
    o, n = reduced(44100, 24000)
    w = table_width(44100, 24000)
    xp = torch.nn.functional.pad(x.double(), (w, w + o))
    frames = xp.unfold(0, 2 * w + o, o)
    want = (frames @ full.double().T).flatten()[:out_length(3001, 44100, 24000)]
    got = resample64(x, 44100, 24000, *banded(full))
    assert float((got - want).abs().max()) < 1e-13
