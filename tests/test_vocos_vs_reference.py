"""Vocos without a GPU: the restated 'same' ISTFT against torch.istft, the oracle sample path + the fp32 Vocos restatement against the
original's stored E2TTS(use_vocos=True) outputs (tests/golden/reference/vocos_*.pt, tools/make_vocos_golden.py), state_dict layout,
local-only loading and the refused config fields."""
import os
import socket
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vocos_ref as V  # noqa: E402
from oracle import e2tts_oracle as O  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402

import e2_tts_pytorch_b200 as pkg  # noqa: E402


@pytest.fixture
def no_network(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError('opened a socket')
    monkeypatch.setattr(socket, 'socket', refuse)
    monkeypatch.setattr(socket, 'create_connection', refuse)


@pytest.mark.parametrize('n_fft,hop', [(1024, 256), (256, 64), (64, 16)])
def test_istft_same_matches_torch_istft_center(n_fft, hop):
    """'same' output sample n is the centred ISTFT's sample n + n_fft/2 - pad on the overlap region"""
    g = torch.Generator().manual_seed(n_fft)
    T = 12
    spec = torch.randn(2, n_fft // 2 + 1, T, generator=g, dtype=torch.float64) + 1j * torch.randn(2, n_fft // 2 + 1, T, generator=g,
                                                                                                  dtype=torch.float64)
    spec[:, 0].imag = 0
    spec[:, -1].imag = 0
    w = torch.hann_window(n_fft, dtype=torch.float64)
    y = V.istft_same(spec.to(torch.complex64), w.float(), n_fft, hop)
    yc = torch.istft(spec, n_fft, hop, n_fft, w, center=True, length=(T - 1) * hop)
    pad, off = (n_fft - hop) // 2, n_fft // 2
    lo, hi = n_fft // 2, (T - 1) * hop - n_fft // 2     # every sample covered by n_fft / hop frames in both
    got = y[:, lo + off - pad:hi + off - pad].double()
    want = yc[:, lo:hi]
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())


@pytest.mark.parametrize('name', list(V.VOCOS_CASES))
def test_sample_audio_vs_reference(name):
    """the oracle's sample path, then DB_to_amplitude and the restated decode per item, reproduce the original's audio"""
    c = V.VOCOS_CASES[name]
    rec = RC.load('vocos_' + name)
    sd = V.full_state_dict(c)
    tsd = {k: v for k, v in sd.items() if not k.startswith('vocos.')}
    vsd = {k[len('vocos.'):]: v for k, v in sd.items() if k.startswith('vocos.')}
    cond = RC.randn((c['cond'][0], c['cond'][1], 100), c['seed'] + 1000)
    with torch.no_grad():
        mel = O.e2tts_sample(tsd, O.TransformerCfg(**RC.KW), cond, O.list_str_to_tensor(c['text']), duration=torch.tensor(c['duration']),
                             lens=torch.tensor(c['lens']), y0=RC.randn(rec['shape'], 3000 + c['seed']), steps=c['steps'])
        assert tuple(mel.shape) == rec['shape']
        assert RC.compact_rel_l2(mel, rec['mel']) < 1e-4
        hop = c['g']['hop_length']
        for b, n in enumerate(c['duration']):
            amp = torch.pow(torch.pow(10.0, 0.1 * mel[b, :n]), 0.5)   # torchaudio DB_to_amplitude(x, ref=1, power=0.5)
            audio = V.decode(vsd, c['g'], amp.t()[None])[0]
            assert audio.numel() == rec['audio_lens'][b] == n * hop
            assert RC.compact_rel_l2(audio, rec['audio'][b]) < 1e-3, (name, b)


@pytest.mark.parametrize('name', list(V.VOCOS_CASES))
def test_state_dict_matches_reference(name, tmp_path, no_network):
    c = V.VOCOS_CASES[name]
    V.write_checkpoint(str(tmp_path), c['g'], c['vseed'], c['opened'])
    m = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=True, pretrained_vocos_path=str(tmp_path))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == RC.load('vocos_' + name)['shapes']
    m.load_state_dict(V.full_state_dict(c), strict=True)
    assert m.vocos is not None and not m.vocos.training
    assert any(p is m.vocos.head.out.weight for p in m.parameters())


def test_from_pretrained_directory_and_hf_cache(tmp_path, monkeypatch, no_network):
    sd = V.write_checkpoint(str(tmp_path / 'ckpt'), V.SMALL, 3)
    m = pkg.Vocos.from_pretrained(str(tmp_path / 'ckpt'))
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items()) and m.state_dict().keys() == sd.keys()
    snap = tmp_path / 'hub' / 'models--someone--vocos-test' / 'snapshots' / 'abc123'
    V.write_checkpoint(str(snap), V.SMALL, 4)
    (tmp_path / 'hub' / 'models--someone--vocos-test' / 'refs').mkdir()
    (tmp_path / 'hub' / 'models--someone--vocos-test' / 'refs' / 'main').write_text('abc123')
    monkeypatch.setenv('HF_HUB_CACHE', str(tmp_path / 'hub'))
    m2 = pkg.Vocos.from_pretrained('someone/vocos-test')
    assert torch.equal(m2.head.out.weight, V.random_state_dict(V.SMALL, 4)['head.out.weight'])
    monkeypatch.delenv('HF_HUB_CACHE')
    monkeypatch.setenv('HF_HOME', str(tmp_path))
    assert pkg.Vocos.from_pretrained('someone/vocos-test').n_fft == V.SMALL['n_fft']
    with pytest.raises(FileNotFoundError):
        pkg.Vocos.from_pretrained('someone/not-there')


def test_unresolvable_vocos_refuses_before_the_ode_loop(tmp_path, monkeypatch, no_network):
    monkeypatch.setenv('HF_HUB_CACHE', str(tmp_path))
    m = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=True, pretrained_vocos_path='charactr/vocos-mel-24khz')
    assert m.vocos is None
    assert not any(k.startswith('vocos.') for k in m.state_dict())

    def never(*a, **k):
        raise AssertionError('the transformer ran')
    monkeypatch.setattr(m, 'transformer_with_pred_head', never)
    with pytest.raises(NotImplementedError, match='pretrained_vocos_path'):
        m.sample(torch.randn(1, 8, 100), text=['ab'], duration=12, steps=2)


@pytest.mark.parametrize('field,value', [('backbone.adanorm_num_embeddings', 4), ('feature_extractor.class_path', 'vocos.feature_extractors.EncodecFeatures'),
                                         ('head.padding', 'center'), ('head.n_fft', 1000), ('head.n_fft', 8192), ('head.n_fft', 32),
                                         ('head.hop_length', 255)])
def test_refused_config_fields(tmp_path, field, value):
    V.write_checkpoint(str(tmp_path), V.SMALL, 5, **{field: value})
    with pytest.raises(NotImplementedError, match=field.replace('.', r'\.')):
        pkg.Vocos.from_pretrained(str(tmp_path))
