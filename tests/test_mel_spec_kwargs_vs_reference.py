"""CPU: the reference's `mel_spec_kwargs` (e2_tts.py:249-260: win_length, center, power, normalize, norm, and filter_length off the
powers of two). The float64 restatement of tests/mel_kwargs_ref.py against what the original MelSpec computed with torchaudio
(tests/golden/reference/melspec_kwargs_*.pt, tools/make_melspec_kwargs_golden.py) and, where torchaudio imports, against
torchaudio directly on further settings; the package's buffers against the original's; and the refusals, in the module and in the
C ABI (before any launch)."""
import pytest
import torch

from mel_kwargs_ref import DEFAULTS, LOG_FLOOR, MEL_KWARGS_CASES, TA_NAMES, case_wave, mel_of_module, settings
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg


@pytest.mark.parametrize('name', list(MEL_KWARGS_CASES))
def test_restatement_vs_reference(name):
    """the original's fp32 log-mel lies within the element-wise bound the CUDA kernels are held to around the float64 restatement
    (it is an fp32 FFT too), and within 1e-4 absolute; the frame count is MelSpec.frames"""
    c = MEL_KWARGS_CASES[name]
    g = RC.load('melspec_kwargs_' + name)
    assert g['kw'] == c['kw']
    ms = pkg.MelSpec(**c['kw'])
    ref, bound = mel_of_module(ms, case_wave(c), bound=True)
    assert ref.shape == g['mel'].shape and ref.shape[-1] == ms.frames(c['nw'])
    d = (g['mel'].double() - ref).abs()
    assert bool((d <= bound).all()) and float(d.max()) < 1e-4, (float(d.max()), float((d / bound).max()))


def test_cases_reach_every_switch():
    """every switch alone, the 16 kHz front-end, a mixed-radix n_fft with a shorter window and valid framing, and all together"""
    kws = [settings(c['kw']) for c in MEL_KWARGS_CASES.values()]
    assert any(k['win_length'] < k['filter_length'] and (k['filter_length'] - k['win_length']) % 2 for k in kws)
    assert any(k['win_length'] < k['filter_length'] and (k['filter_length'] - k['win_length']) % 4 == 0 for k in kws)
    assert {True, False} == {k['center'] for k in kws} and {0.5, 1, 1.5, 2} <= {k['power'] for k in kws}
    assert {False, True, 'frame_length'} <= {k['normalize'] for k in kws} and {None, 'slaney'} == {k['norm'] for k in kws}
    assert any(k['filter_length'] & (k['filter_length'] - 1) for k in kws)
    assert any(sum(k[n] != DEFAULTS[n] for n in ('win_length', 'center', 'power', 'normalize', 'norm')) == 5 for k in kws)
    for name in MEL_KWARGS_CASES:
        assert RC.load('melspec_kwargs_' + name)['mel'].numel() > 0


@pytest.mark.parametrize('name', list(MEL_KWARGS_CASES))
def test_state_dict_matches_reference(name):
    """buffer names and shapes of the original (torchaudio's: spectrogram.window [win_length], mel_scale.fb [n_fft/2+1, n_mels])"""
    c = MEL_KWARGS_CASES[name]
    ms = pkg.MelSpec(**c['kw'])
    assert {k: tuple(v.shape) for k, v in ms.state_dict().items()} == RC.load('melspec_kwargs_' + name)['shapes']
    s = settings(c['kw'])
    assert ms.mel_stft.spectrogram.window.shape == (s['win_length'],)


FURTHER = [
    dict(filter_length=375, hop_length=100, win_length=300, n_mel_channels=40, sampling_rate=8000),          # odd n_fft, centred
    dict(filter_length=1536, hop_length=200, win_length=1001, n_mel_channels=128, power=0.5, norm='slaney', normalize='frame_length'),
    dict(filter_length=4000, hop_length=500, win_length=3999, n_mel_channels=100, center=False, power=2, normalize='window'),
    dict(filter_length=2187, hop_length=300, win_length=2187, n_mel_channels=90, sampling_rate=22050, center=False, power=1.5),
    dict(filter_length=64, hop_length=1, win_length=33, n_mel_channels=20, sampling_rate=16000, norm='slaney', normalize=True),
]


@pytest.mark.parametrize('kw', FURTHER, ids=[f'nfft{k["filter_length"]}' for k in FURTHER])
def test_restatement_vs_torchaudio(kw):
    """torchaudio.transforms.MelSpectrogram (float64, same buffers) on further seeded settings: odd and large n_fft, the other
    power / normalize combinations; buffers bit-identical to torchaudio's"""
    ta = pytest.importorskip('torchaudio')
    s = settings(kw)
    t = ta.transforms.MelSpectrogram(**{TA_NAMES[k]: v for k, v in s.items()}).double()
    ms = pkg.MelSpec(**kw)
    for k, v in t.state_dict().items():
        assert torch.equal(ms.mel_stft.state_dict()[k].double(), v), k
    wave = case_wave(dict(B=2, nw=s['filter_length'] + s['hop_length'] * 5 + 7, seed=s['filter_length']))
    want = t(wave.double()).clamp(min=LOG_FLOOR).log()   # the reference clamps in fp32: at fp32(1e-5)
    got = mel_of_module(ms, wave)
    assert got.shape == want.shape and got.shape[-1] == ms.frames(wave.shape[1])
    assert float((got - want).abs().max()) < 1e-9


@pytest.mark.parametrize('kw', [dict(filter_length=448), dict(filter_length=1000 + 7), dict(filter_length=32), dict(filter_length=8192),
                                dict(power=None)], ids=['nfft448', 'nfft1007', 'nfft32', 'nfft8192', 'power-none'])
def test_unsupported_settings_raise(kw):
    """what no kernel computes raises NotImplementedError at construction, naming the reference's line, in MelSpec and through
    E2TTS / DurationPredictor(mel_spec_kwargs=...)"""
    line = 'e2_tts.py:257' if 'power' in kw else 'e2_tts.py:251'
    with pytest.raises(NotImplementedError, match=line):
        pkg.MelSpec(**kw)
    with pytest.raises(NotImplementedError, match=line):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), mel_spec_kwargs=kw, use_vocos=False)
    with pytest.raises(NotImplementedError, match=line):
        pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2), mel_spec_kwargs=kw)


@pytest.mark.parametrize('kw', [dict(win_length=1025), dict(power=0), dict(power=-1), dict(normalize='energy'), dict(norm='htk')])
def test_invalid_settings_raise(kw):
    """what torch / torchaudio themselves refuse is a ValueError"""
    with pytest.raises(ValueError):
        pkg.MelSpec(**kw)


def test_model_takes_the_mel_count():
    """E2TTS / DurationPredictor take num_channels from n_mel_channels, so the stem and the prediction head follow it"""
    kw = dict(filter_length=400, hop_length=160, win_length=400, n_mel_channels=80, sampling_rate=16000)
    m = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), mel_spec_kwargs=kw, use_vocos=False)
    sd = m.state_dict()
    assert m.num_channels == 80 and m.sampling_rate == 16000
    assert sd['proj_in.weight'].shape == (128, 80) and sd['to_pred.weight'].shape == (80, 128)
    assert sd['mel_spec.mel_stft.mel_scale.fb'].shape == (201, 80) and sd['mel_spec.mel_stft.spectrogram.window'].shape == (400,)
    dp = pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2), mel_spec_kwargs=kw)
    assert dp.state_dict()['proj_in.weight'].shape == (128, 80)


def _abi_args(**kw):
    base = dict(wave=256, window=256, fb=256, out=256, ws_bands=256, B=1, nw=4096, n_fft=1024, hop=256, n_mels=100, win_length=1024,
                center=1, power=1.0, norm_scale=1.0)
    return pkg.lib.make_args('b200_melspec_args', **dict(base, **kw))


@pytest.mark.parametrize('kw,msg', [
    (dict(n_fft=448), 'prime factor'), (dict(n_fft=7 * 128), 'prime factor'), (dict(n_fft=32, win_length=32), r'\[64, 4096\]'),
    (dict(n_fft=8000, win_length=8000), r'\[64, 4096\]'), (dict(power=0.0), 'power'), (dict(power=-2.0), 'power'),
    (dict(win_length=1025), 'win_length'), (dict(win_length=0), 'win_length'), (dict(norm_scale=0.0), 'norm_scale'),
    (dict(center=0, nw=1023), 'at least n_fft'), (dict(center=1, nw=512), 'longer than n_fft/2'),
])
def test_c_abi_refusals(kw, msg):
    """b200_melspec_ex refuses before any launch (placeholder pointers, never read)"""
    with pytest.raises(RuntimeError, match=msg):
        pkg.lib.call('b200_melspec_ex', _abi_args(**kw), None)
