"""Vocos mel-spectrogram decoder (the reference's E2TTS(use_vocos=True): `Vocos.from_pretrained('charactr/vocos-mel-24khz')`,
e2_tts.py:1244, and the per-item decode of sample(), :1440-1451), restated from the published vocos package: a ConvNeXt backbone and
an inverse-STFT head with 'same' padding. Loads from local files only: a checkpoint directory, or a Hugging Face repo id already in the
local HF cache; nothing is downloaded. The parameters keep the published state_dict layout; `decode` runs on the sm_90a kernels.

Kernel launches per decode call, for any batch size: 3 per ConvNeXt block (dwconv + LayerNorm, pwconv1 with GELU, pwconv2 with the
gamma scale and the residual) and 8 more (weight pack, im2col, embed GEMM, LayerNorm, final LayerNorm, head GEMM, inverse STFT x 2).
"""
from __future__ import annotations

import os

import torch
from torch import nn
from torch.nn import Module, ModuleList

from . import ops
from .modules import _MelSTFT, _PackOwner

BF16, F32 = torch.bfloat16, torch.float32
MEL_FEATURES = 'vocos.feature_extractors.MelSpectrogramFeatures'


def _hub_cache():
    if os.environ.get('HF_HUB_CACHE'):
        return os.environ['HF_HUB_CACHE']
    if os.environ.get('HF_HOME'):
        return os.path.join(os.environ['HF_HOME'], 'hub')
    return os.path.join(os.path.expanduser('~'), '.cache', 'huggingface', 'hub')


def resolve_local(path_or_repo_id):
    """-> the directory holding config.yaml and pytorch_model.bin, or None: `path_or_repo_id` itself, else the repo id's snapshot in the
    local HF cache (models--{org}--{name}/refs/main -> snapshots/<rev>). Touches only the filesystem."""
    def complete(d):
        return os.path.isfile(os.path.join(d, 'config.yaml')) and os.path.isfile(os.path.join(d, 'pytorch_model.bin'))

    p = str(path_or_repo_id)
    if os.path.isdir(p):
        return p if complete(p) else None
    repo = os.path.join(_hub_cache(), 'models--' + p.replace('/', '--'))
    ref = os.path.join(repo, 'refs', 'main')
    if not os.path.isfile(ref):
        return None
    with open(ref) as f:
        snap = os.path.join(repo, 'snapshots', f.read().strip())
    return snap if complete(snap) else None


def _refuse(field, value, why):
    raise NotImplementedError(f'Vocos config {field}={value!r}: {why}; no CUDA kernel is built for it')


def parse_config(cfg):
    """config.yaml (dict) -> Vocos keyword arguments, refusing every field the kernels do not build."""
    fe, bb, hd = cfg['feature_extractor'], cfg['backbone'], cfg['head']
    if fe.get('class_path') != MEL_FEATURES:
        _refuse('feature_extractor.class_path', fe.get('class_path'), 'only mel-spectrogram features are decoded')
    b, h, f = bb.get('init_args', {}), hd.get('init_args', {}), fe.get('init_args', {})
    if b.get('adanorm_num_embeddings') is not None:
        _refuse('backbone.adanorm_num_embeddings', b['adanorm_num_embeddings'], 'AdaLayerNorm (the Encodec variant)')
    if h.get('padding', 'same') != 'same':
        _refuse('head.padding', h['padding'], "only the 'same' inverse STFT is built")
    n_fft, hop = int(h['n_fft']), int(h['hop_length'])
    if n_fft < 64 or n_fft > 4096 or n_fft & (n_fft - 1):
        _refuse('head.n_fft', n_fft, 'n_fft must be a power of two in [64, 4096]')
    if hop < 1 or hop > n_fft or (n_fft - hop) % 2:
        _refuse('head.hop_length', hop, 'hop must be in [1, n_fft] with n_fft - hop even')
    return dict(input_channels=int(b['input_channels']), dim=int(b['dim']), intermediate_dim=int(b['intermediate_dim']),
                num_layers=int(b['num_layers']), n_fft=n_fft, hop_length=hop, sample_rate=int(f.get('sample_rate', 24000)),
                fe_n_fft=int(f.get('n_fft', n_fft)), n_mels=int(f.get('n_mels', b['input_channels'])))


class _ConvNeXtBlock(Module):   # vocos/modules.py ConvNeXtBlock without AdaLayerNorm
    def __init__(self, dim, intermediate_dim, layer_scale_init_value):
        super().__init__()
        self.dwconv = nn.Conv1d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, intermediate_dim)
        self.pwconv2 = nn.Linear(intermediate_dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones(dim))


class _Backbone(Module):   # vocos/models.py VocosBackbone
    def __init__(self, input_channels, dim, intermediate_dim, num_layers):
        super().__init__()
        self.embed = nn.Conv1d(input_channels, dim, kernel_size=7, padding=3)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.convnext = ModuleList([_ConvNeXtBlock(dim, intermediate_dim, 1 / num_layers) for _ in range(num_layers)])
        self.final_layer_norm = nn.LayerNorm(dim, eps=1e-6)


class _ISTFT(Module):
    def __init__(self, n_fft):
        super().__init__()
        self.register_buffer('window', torch.hann_window(n_fft))


class _Head(Module):   # vocos/heads.py ISTFTHead
    def __init__(self, dim, n_fft):
        super().__init__()
        self.out = nn.Linear(dim, n_fft + 2)
        self.istft = _ISTFT(n_fft)


class _Features(Module):   # MelSpectrogramFeatures: its buffers only (decode never reads them; they keep the state_dict strict)
    def __init__(self, n_fft, n_mels, sample_rate):
        super().__init__()
        self.mel_spec = _MelSTFT(n_fft, n_fft, n_mels, sample_rate)


class Vocos(_PackOwner):
    """Vocos (mel features, ConvNeXt backbone, ISTFT head with 'same' padding). `from_pretrained(path_or_repo_id)` loads local files;
    `decode(features [B, C, T]) -> audio [B, T * hop]` runs on the GPU, inference only."""

    def __init__(self, input_channels=100, dim=512, intermediate_dim=1536, num_layers=8, n_fft=1024, hop_length=256, sample_rate=24000,
                 fe_n_fft=None, n_mels=None):
        super().__init__()
        self.input_channels, self.dim, self.intermediate_dim, self.num_layers = input_channels, dim, intermediate_dim, num_layers
        self.n_fft, self.hop_length = n_fft, hop_length
        if dim % 64 or dim > 1024:
            _refuse('backbone.dim', dim, 'the LayerNorm kernels take multiples of 64 up to 1024')
        if intermediate_dim % 8:
            _refuse('backbone.intermediate_dim', intermediate_dim, 'GEMM row pitches are multiples of 8')
        self.feature_extractor = _Features(fe_n_fft or n_fft, n_mels or input_channels, sample_rate)
        self.backbone = _Backbone(input_channels, dim, intermediate_dim, num_layers)
        self.head = _Head(dim, n_fft)

    @classmethod
    def from_pretrained(cls, path_or_repo_id):
        import yaml
        path = resolve_local(path_or_repo_id)
        if path is None:
            raise FileNotFoundError(f'{path_or_repo_id!r} is neither a directory with config.yaml and pytorch_model.bin nor a repo id in the '
                                    f'local Hugging Face cache ({_hub_cache()}); nothing is downloaded')
        with open(os.path.join(path, 'config.yaml')) as f:
            kw = parse_config(yaml.safe_load(f))
        model = cls(**kw)
        sd = torch.load(os.path.join(path, 'pytorch_model.bin'), map_location='cpu', weights_only=True)
        model.load_state_dict(sd, strict=True)
        return model.eval()

    def _add_weights(self, pack):
        bb, C, d = self.backbone, self.input_channels, self.dim
        lda = (7 * C + 7) // 8 * 8
        w = dict(lda=lda, embed=pack.buffer(d, lda), pw1=[], pw2=[], head=pack.buffer(self.n_fft + 2, d))
        pack.add(bb.embed.weight, w['embed'])   # [dim, C, 7] viewed [dim, 7C]: channel-major, tap-minor, like the im2col columns
        for blk in bb.convnext:
            w['pw1'].append(pack.buffer(*blk.pwconv1.weight.shape))
            w['pw2'].append(pack.buffer(*blk.pwconv2.weight.shape))
            pack.add(blk.pwconv1.weight, w['pw1'][-1])
            pack.add(blk.pwconv2.weight, w['pw2'][-1])
        pack.add(self.head.out.weight, w['head'])
        return w

    @torch.no_grad()
    def decode_padded(self, mel, lens, db_to_amp=False):
        """mel fp32 [B, T, C] with lens[b] valid frames per item -> audio fp32 [B, T * hop], item b decoded as if alone (lens[b] * hop
        samples, zeros after them). db_to_amp: decode 10^(mel / 20) (e2_tts.py:1444 DB_to_amplitude(ref=1, power=0.5))."""
        dev = next(self.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError('Vocos.decode runs on the CUDA kernels only: move the module to a GPU')
        B, T, C = mel.shape
        assert C == self.input_channels, f'expected {self.input_channels} mel channels, got {C}'
        lens = lens.to(device=dev, dtype=torch.int32).contiguous()
        if int(lens.min()) < 1 or int(lens.max()) > T:
            raise ValueError(f'Vocos.decode: item lengths must be in [1, {T}]')
        with torch.cuda.device(dev):
            w = self._packed_weights()
            bb, M, d = self.backbone, B * T, self.dim
            A = ops.vocos_im2col(mel.to(device=dev, dtype=F32).contiguous(), lens, w['lda'], db_to_amp)
            x = ops.gemm(A, w['embed'], M, d, 7 * C, lda=w['lda'], ldb=w['lda'], bias=bb.embed.bias)
            x = ops.vocos_ln(x, lens, bb.norm.weight, bb.norm.bias, bb.norm.eps, B, T, d)
            for i, blk in enumerate(bb.convnext):
                h = ops.vocos_ln(x, lens, blk.norm.weight, blk.norm.bias, blk.norm.eps, B, T, d, conv_w=blk.dwconv.weight,
                                 conv_b=blk.dwconv.bias)
                h = ops.gemm(h, w['pw1'][i], M, self.intermediate_dim, d, bias=blk.pwconv1.bias, act=ops.ACT_GELU)
                # x + gamma * pwconv2(h): the epilogue (z + bias) * colscale + resid with one colscale row for all M rows
                x = ops.gemm(h, w['pw2'][i], M, d, self.intermediate_dim, bias=blk.pwconv2.bias, colscale=blk.gamma, rows_per_batch=M,
                             resid=x, ldr=d)
            x = ops.vocos_ln(x, lens, bb.final_layer_norm.weight, bb.final_layer_norm.bias, bb.final_layer_norm.eps, B, T, d)
            spec = ops.gemm(x, w['head'], M, self.n_fft + 2, d, bias=self.head.out.bias, out_fp32=True)   # log-magnitudes stay fp32
            return ops.vocos_istft(spec, self.head.istft.window, lens, B, T, self.n_fft, self.hop_length)

    def decode(self, features):
        """features [B, C, T] (Vocos.decode's layout) -> audio fp32 [B, T * hop]."""
        B, C, T = features.shape
        return self.decode_padded(features.transpose(1, 2), torch.full((B,), T, dtype=torch.int32))
