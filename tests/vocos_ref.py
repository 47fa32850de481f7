"""Vocos (vocos-mel-24khz layout) restated in fp32 torch from the published vocos package, for the tests and the golden tool: the
mel VocosBackbone (embed Conv1d k 7, LayerNorm, ConvNeXt blocks, final LayerNorm) and the ISTFTHead with 'same' padding, read from a
state_dict in the published key layout. The vocos package is not a dependency of the project and no published checkpoint is used: the
restatement is a parity-unpinned leaf, like the x-transformers and hyper-connections leaves, and `write_checkpoint` makes seeded
random checkpoints (config.yaml + pytorch_model.bin) in a directory.

`RefVocos` has the vocos.Vocos surface the reference uses (from_pretrained, decode); tools/make_vocos_golden.py puts it in place of
`Vocos` while the reference's own e2_tts.py runs."""
import math
import os

import torch
import torch.nn.functional as F
import yaml

MEL_24KHZ = dict(input_channels=100, dim=512, intermediate_dim=1536, num_layers=8, n_fft=1024, hop_length=256, sample_rate=24000)
SMALL = dict(input_channels=100, dim=128, intermediate_dim=384, num_layers=2, n_fft=256, hop_length=64, sample_rate=24000)

# E2TTS(use_vocos=True) cases of tools/make_vocos_golden.py: name -> Vocos geometry, its seed and weight regime, the d128 depth-2 model's
# seed, prompt shape and lengths, per-item duration, text, ODE steps
VOCOS_CASES = {
    'mel24khz': dict(g=MEL_24KHZ, vseed=61, opened=False, seed=71, cond=(2, 20), lens=[20, 12], duration=[48, 31], text=['abc', 'de f'],
                     steps=3),
    'small': dict(g=SMALL, vseed=62, opened=True, seed=72, cond=(2, 16), lens=[16, 9], duration=[29, 40], text=['hello', 'xy'], steps=3),
}


def full_state_dict(c):
    """the seeded E2TTS(use_vocos=True) state_dict of a VOCOS_CASES entry, in the reference's key layout"""
    from oracle import reference_cases as RC
    sd = RC.state_dict('E2TTS', c['seed'], RC.KW)
    sd.update({'vocos.' + k: v for k, v in random_state_dict(c['g'], c['vseed'], c['opened']).items()})
    return sd


def config_yaml(g, **overrides):
    """The published config.yaml layout for geometry g; overrides: {'backbone.x': v, 'head.x': v, 'feature_extractor.class_path': v}"""
    cfg = {
        'feature_extractor': {'class_path': 'vocos.feature_extractors.MelSpectrogramFeatures',
                              'init_args': dict(sample_rate=g['sample_rate'], n_fft=g['n_fft'], hop_length=g['hop_length'],
                                                n_mels=g['input_channels'], padding='center')},
        'backbone': {'class_path': 'vocos.models.VocosBackbone',
                     'init_args': dict(input_channels=g['input_channels'], dim=g['dim'], intermediate_dim=g['intermediate_dim'],
                                       num_layers=g['num_layers'])},
        'head': {'class_path': 'vocos.heads.ISTFTHead', 'init_args': dict(dim=g['dim'], n_fft=g['n_fft'], hop_length=g['hop_length'],
                                                                          padding='same')},
    }
    for k, v in overrides.items():
        sec, key = k.split('.', 1)
        if key == 'class_path':
            cfg[sec]['class_path'] = v
        else:
            cfg[sec]['init_args'][key] = v
    return cfg


def random_state_dict(g, seed, opened=False):
    """Seeded weights in the published key layout. opened: head weights scaled so the log-magnitudes span about [-6, 6] (across the
    1e2 clip at log 4.6) and the phases several pi, gamma of order 1 instead of 1 / num_layers, non-trivial LayerNorm affines."""
    gen = torch.Generator().manual_seed(seed)

    def rn(*shape, s=1.):
        return torch.randn(*shape, generator=gen) * s

    C, d, I, L, n = g['input_channels'], g['dim'], g['intermediate_dim'], g['num_layers'], g['n_fft']
    sd = {}
    fb_n = n // 2 + 1
    sd['feature_extractor.mel_spec.spectrogram.window'] = torch.hann_window(n)
    sd['feature_extractor.mel_spec.mel_scale.fb'] = torch.rand(fb_n, C, generator=gen)
    sd['backbone.embed.weight'] = rn(d, C, 7, s=1 / math.sqrt(7 * C))
    sd['backbone.embed.bias'] = rn(d, s=0.02)

    def ln(name):
        sd[name + '.weight'] = 1 + rn(d, s=0.2 if opened else 0.)
        sd[name + '.bias'] = rn(d, s=0.1 if opened else 0.)

    ln('backbone.norm')
    for i in range(L):
        p = f'backbone.convnext.{i}.'
        sd[p + 'dwconv.weight'] = rn(d, 1, 7, s=1 / math.sqrt(7))
        sd[p + 'dwconv.bias'] = rn(d, s=0.02)
        ln(p + 'norm')
        sd[p + 'pwconv1.weight'] = rn(I, d, s=1 / math.sqrt(d))
        sd[p + 'pwconv1.bias'] = rn(I, s=0.02)
        sd[p + 'pwconv2.weight'] = rn(d, I, s=1 / math.sqrt(I))
        sd[p + 'pwconv2.bias'] = rn(d, s=0.02)
        sd[p + 'gamma'] = (0.5 + torch.rand(d, generator=gen)) if opened else torch.full((d,), 1 / L)
    ln('backbone.final_layer_norm')
    K = n // 2 + 1
    w = rn(n + 2, d, s=1 / math.sqrt(d))
    b = rn(n + 2, s=0.02)
    if opened:
        w[:K] *= 3.
        b[:K] -= 0.5
        w[K:] *= 12.
    sd['head.out.weight'], sd['head.out.bias'] = w, b
    sd['head.istft.window'] = torch.hann_window(n)
    return sd


def write_checkpoint(directory, g, seed, opened=False, **overrides):
    """config.yaml + pytorch_model.bin of a seeded random Vocos into `directory` (created); returns the state_dict"""
    os.makedirs(directory, exist_ok=True)
    with open(os.path.join(directory, 'config.yaml'), 'w') as f:
        yaml.safe_dump(config_yaml(g, **overrides), f)
    sd = random_state_dict(g, seed, opened)
    torch.save(sd, os.path.join(directory, 'pytorch_model.bin'))
    return sd


def istft_same(spec, window, n_fft, hop):
    """ISTFTHead('same'): complex spec [B, n_fft/2 + 1, T] -> [B, T * hop], in the dtype of `window` (float64 for the bound references)"""
    B, _, T = spec.shape
    pad = (n_fft - hop) // 2
    frames = torch.fft.irfft(spec, n_fft, dim=1, norm='backward') * window[None, :, None]
    size = (T - 1) * hop + n_fft
    y = F.fold(frames, output_size=(1, size), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0, pad:-pad]
    env = F.fold(window.square()[None, :, None].expand(1, -1, T), output_size=(1, size), kernel_size=(1, n_fft),
                 stride=(1, hop)).squeeze()[pad:-pad]
    return y / env


def head_spec(x):
    """head.out output [B, T, n_fft + 2] -> the complex spectrum [B, n_fft/2 + 1, T] of ISTFTHead.forward"""
    mag, p = x.transpose(1, 2).chunk(2, dim=1)
    mag = torch.exp(mag).clip(max=1e2)
    return mag * (torch.cos(p) + 1j * torch.sin(p))


def backbone(sd, g, x, round_bf16=False):
    """x [B, C, T] -> [B, T, dim]; round_bf16: round each stage output to bf16 as the kernels store them (the conditioning probe)"""
    r = (lambda t: t.to(torch.bfloat16).to(t.dtype)) if round_bf16 else (lambda t: t)
    d = g['dim']
    x = r(x)
    x = F.conv1d(x, sd['backbone.embed.weight'], sd['backbone.embed.bias'], padding=3).transpose(1, 2)
    x = r(x)
    x = r(F.layer_norm(x, (d,), sd['backbone.norm.weight'], sd['backbone.norm.bias'], 1e-6))
    for i in range(g['num_layers']):
        p = f'backbone.convnext.{i}.'
        h = F.conv1d(x.transpose(1, 2), sd[p + 'dwconv.weight'], sd[p + 'dwconv.bias'], padding=3, groups=d).transpose(1, 2)
        h = r(F.layer_norm(h, (d,), sd[p + 'norm.weight'], sd[p + 'norm.bias'], 1e-6))
        h = r(F.gelu(F.linear(h, sd[p + 'pwconv1.weight'], sd[p + 'pwconv1.bias'])))
        x = r(x + sd[p + 'gamma'] * F.linear(h, sd[p + 'pwconv2.weight'], sd[p + 'pwconv2.bias']))
    return r(F.layer_norm(x, (d,), sd['backbone.final_layer_norm.weight'], sd['backbone.final_layer_norm.bias'], 1e-6))


def decode(sd, g, features, round_bf16=False):
    """Vocos.decode: features [B, C, T] -> audio [B, T * hop] (fp32 unless the state_dict is float64)"""
    x = backbone(sd, g, features, round_bf16)
    x = F.linear(x, sd['head.out.weight'], sd['head.out.bias'])
    return istft_same(head_spec(x), sd['head.istft.window'], g['n_fft'], g['hop_length'])


def geometry_of(cfg):
    b, h = cfg['backbone']['init_args'], cfg['head']['init_args']
    return dict(input_channels=b['input_channels'], dim=b['dim'], intermediate_dim=b['intermediate_dim'], num_layers=b['num_layers'],
                n_fft=h['n_fft'], hop_length=h['hop_length'], sample_rate=cfg['feature_extractor']['init_args']['sample_rate'])


class RefVocos(torch.nn.Module):
    """vocos.Vocos surface for the reference's e2_tts.py: from_pretrained(dir) -> module with the checkpoint's keys, decode()"""

    def __init__(self, sd, g):
        super().__init__()
        self.g = g
        for k, v in sd.items():   # flat parameter holders under the published names, so state_dict() has exactly these keys
            mod = self
            *path, leaf = k.split('.')
            for part in path:
                if not hasattr(mod, part) or not isinstance(getattr(mod, part), torch.nn.Module):
                    mod.add_module(part, torch.nn.Module())
                mod = getattr(mod, part)
            if k.startswith('feature_extractor.') or k == 'head.istft.window':
                mod.register_buffer(leaf, v.clone())
            else:
                mod.register_parameter(leaf, torch.nn.Parameter(v.clone()))

    @classmethod
    def from_pretrained(cls, path):
        with open(os.path.join(path, 'config.yaml')) as f:
            g = geometry_of(yaml.safe_load(f))
        return cls(torch.load(os.path.join(path, 'pytorch_model.bin'), map_location='cpu', weights_only=True), g)

    def decode(self, features):
        return decode(dict(self.state_dict()), self.g, features)
