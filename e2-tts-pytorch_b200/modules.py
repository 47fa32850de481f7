"""Host-side mirror of the reference's model classes for the hot path: same constructor / forward surface and
the same state_dict keys as /root/reference/e2_tts_pytorch/e2_tts.py (SURVEY Appendix B), with every forward
routed through the sm_90a kernels of libb200e2tts.so (ops.py). The nn.Modules below only HOLD parameters in
the reference's layout; the arithmetic lives in the CUDA library.
"""
from __future__ import annotations

import contextlib
import copy
import ctypes
import math
import numbers
import random as pyrandom
from collections import namedtuple
from functools import partial
from random import randrange
from typing import Callable

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn import Module, ModuleList

from . import lib, ode, ops

LossBreakdown = namedtuple('LossBreakdown', ['flow', 'velocity_consistency'])  # e2_tts.py:71
E2TTSReturn = namedtuple('E2TTS', ['loss', 'cond', 'pred_flow', 'pred_data', 'loss_breakdown'])  # e2_tts.py:73

BF16, F32 = torch.bfloat16, torch.float32
SOFTCLAMP = 50.0  # x-transformers logit_softclamp_value default (A.4)
SOFTCLAMP_MAX = 64.0  # largest clamp the clamped attention kernels take (include/b200_e2tts.h)
SUPPORTED_RESIDUAL_STREAMS = (1, 4)   # Transformer(num_residual_streams): 1 = plain residual, 4 = hyper-connections (the reference default)
SUPPORTED_DIM_HEADS = (64, 128)       # Transformer(dim_head, text_dim_head): head widths the attention kernels are built for
# x-transformers Attention keywords the kernels implement, with x-transformers' own defaults for a missing key
ATTN_KWARGS_DEFAULTS = dict(gate_value_heads=False, softclamp_logits=False, logit_softclamp_value=50.)
# x-transformers FeedForward keywords besides those the reference passes itself (dim, mult, glu, dropout), with x-transformers' defaults.
# The last five have no kernel and are refused unless set to their default.
FF_KWARGS_DEFAULTS = dict(swish=False, relu_squared=False, glu_mult_bias=False, no_bias=False, zero_init_output=False,
                          custom_activation=None, solu=False, post_act_ln=False, sublayer_dropout=0., dim_out=None)
GLU_GELU, GLU_SILU, GLU_RELU2 = ops.GLU_GELU, ops.GLU_SILU, ops.GLU_RELU2
# text sub-blocks of layer i+1 overlap the audio sub-blocks of layer i on a second CUDA stream (Transformer._run_layers);
# B200_TWO_STREAM=0 serialises them on the current stream (developer A/B switch)
import os as _os
TWO_STREAM = _os.environ.get('B200_TWO_STREAM', '1') != '0'
_SIDE_STREAMS = {}


def _side_stream(device):
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device)
    return _SIDE_STREAMS[key]


def exists(v):
    return v is not None


def default(v, d):
    return v if exists(v) else d


def _on_module_device(fn):
    """Run a public entry point with the CUDA device of the module's parameters current, so that the raw-pointer kernel launches
    (ops.py: torch.cuda.current_stream()) go to that device's stream even when the process-wide current device is another GPU.
    (Backward runs on the autograd engine's per-device threads, which set the device themselves.)"""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        dev = next(self.parameters()).device
        if dev.type != 'cuda' or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(self, *a, **k)
        with torch.cuda.device(dev):
            return fn(self, *a, **k)
    return wrapped


def _unsupported(name, value, ref):
    raise NotImplementedError(
        f'{name}={value!r} is a non-default research switch of the reference ({ref}) for which no CUDA kernel is built; '
        f'there is no fallback path (SURVEY.md §2 row 8)')


_ODE_REF = 'e2_tts.py:1122-1126'
# torchdiffeq methods without a solver here, and why
_ODE_REFUSED = {
    'dopri8': "its 13-stage tableau is not restated",
    'heun2': "only some torchdiffeq versions have it", 'heun3': "only some torchdiffeq versions have it",
    'explicit_adams': "a multistep method", 'implicit_adams': "a multistep method", 'fixed_adams': "a multistep method",
    'scipy_solver': "a host solver",
}


def _real(v):
    return isinstance(v, numbers.Real) and not isinstance(v, bool)


def _parse_odeint_kwargs(kw):
    """E2TTS(odeint_kwargs) -> dict(method, rtol, atol, options) for E2TTS.sample. 'midpoint' and 'euler' run the fixed-grid loop and
    take the other keys as they always did (ignored); a dict without 'method' keeps that midpoint loop. 'rk4' and the adaptive
    methods of ode.py take `atol` / `rtol` as Python floats (torchdiffeq's defaults 1e-9 / 1e-7 when missing) and `options` with only
    first_step, safety, ifactor, dfactor and max_num_steps (ignored by 'rk4', as torchdiffeq's fixed-grid solvers ignore them).
    Everything else raises NotImplementedError naming the key."""
    method = kw.get('method', 'midpoint')
    if method in ('midpoint', 'euler'):
        return dict(method=method)
    if method != 'rk4' and method not in ode.ADAPTIVE_METHODS:
        why = _ODE_REFUSED.get(method, 'not a torchdiffeq method this package solves') if isinstance(method, str) else 'not a method name'
        _unsupported("odeint_kwargs['method']", method, f'{_ODE_REF}; {why}')
    for key in kw:
        if key not in ('method', 'atol', 'rtol', 'options'):
            _unsupported(f'odeint_kwargs[{key!r}]', kw[key], _ODE_REF)
    out = dict(method=method)
    for key in ('rtol', 'atol'):
        v = kw.get(key, ode.DEFAULT_TOL[key])
        if not _real(v):
            _unsupported(f'odeint_kwargs[{key!r}]', v, f'{_ODE_REF}; a tolerance is a Python float here, not a tensor')
        if not (math.isfinite(v) and v >= 0):
            raise ValueError(f'odeint_kwargs[{key!r}]={v!r}: want a finite tolerance >= 0')
        out[key] = float(v)
    options = kw.get('options') or {}
    if not isinstance(options, dict):
        _unsupported("odeint_kwargs['options']", options, _ODE_REF)
    for key, v in options.items():
        if key not in ode.DEFAULT_OPTIONS:
            _unsupported(f'odeint_kwargs[\'options\'][{key!r}]', v, _ODE_REF)
        if key == 'max_num_steps':
            if not isinstance(v, numbers.Integral) or isinstance(v, bool) or v < 1:
                raise ValueError(f"odeint_kwargs['options']['max_num_steps']={v!r}: want an int >= 1")
        elif key == 'first_step' and v is None:
            continue
        elif not _real(v):
            _unsupported(f'odeint_kwargs[\'options\'][{key!r}]', v, f'{_ODE_REF}; a Python float here, not a tensor')
        elif not (math.isfinite(v) and v > 0):
            raise ValueError(f"odeint_kwargs['options'][{key!r}]={v!r}: want a finite value > 0")
    out['options'] = {k: (int(v) if k == 'max_num_steps' else v if v is None else float(v)) for k, v in options.items()}
    return out


# ----------------------------------------------------------------------------------------------------------------------
# helpers kept as tiny torch ops on (B,) / (B,N) integer / bool tensors (SURVEY §2 rows 6-7)


def list_str_to_tensor(text: list[str], padding_value=-1):  # e2_tts.py:128-135 (ignores padding_value like the reference)
    rows = [torch.tensor([*bytes(t, 'UTF-8')], dtype=torch.long) for t in text]
    n = max(r.numel() for r in rows)
    return torch.stack([F.pad(r, (0, n - r.numel()), value=-1) for r in rows])


def lens_to_mask(t, length=None):  # e2_tts.py:173-182
    if not exists(length):
        length = int(t.amax())
    return torch.arange(length, device=t.device)[None, :] < t[:, None]


def mask_from_frac_lengths(seq_len, frac_lengths, max_length):  # e2_tts.py:193-210 without the .item() host sync (:189)
    lengths = (frac_lengths * seq_len).long()
    max_start = seq_len - lengths
    rand = torch.rand_like(frac_lengths)
    start = (max_start * rand).long().clamp(min=0)
    end = start + lengths
    seq = torch.arange(max_length, device=seq_len.device)
    valid = seq[None] < seq_len.max()  # positions >= max(seq_len) are padding in the reference (pad_to_length :207-208)
    return (seq[None] >= start[:, None]) & (seq[None] < end[:, None]) & valid


# ----------------------------------------------------------------------------------------------------------------------
# parameter holders (names = SURVEY Appendix B)


class RMSNorm(Module):  # A.1
    def __init__(self, dim):
        super().__init__()
        self.g = nn.Parameter(torch.ones(dim))


class AdaptiveRMSNorm(Module):  # A.1
    def __init__(self, dim):
        super().__init__()
        self.to_gamma = nn.Linear(dim, dim, bias=False)
        nn.init.zeros_(self.to_gamma.weight)


class AdaLNZero(Module):  # e2_tts.py:332-351
    def __init__(self, dim, init_bias_value=-2.):
        super().__init__()
        self.to_gamma = nn.Linear(dim, dim)
        nn.init.zeros_(self.to_gamma.weight)
        nn.init.constant_(self.to_gamma.bias, init_bias_value)


class Identity(Module):
    pass


class DepthwiseConv(Module):  # e2_tts.py:295-328
    def __init__(self, dim, *, kernel_size):
        super().__init__()
        assert kernel_size % 2 == 1
        self.dw_conv1d = nn.Sequential(nn.Conv1d(dim, dim, kernel_size, groups=dim, padding=kernel_size // 2), nn.SiLU())


class Attention(Module):  # A.4
    def __init__(self, dim, heads, dim_head, learned_value_residual_mix, gate_value_heads=True):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_k = nn.Linear(dim, inner, bias=False)
        self.to_v = nn.Linear(dim, inner, bias=False)
        self.to_v_head_gate = None
        if gate_value_heads:
            self.to_v_head_gate = nn.Linear(dim, heads)
            nn.init.constant_(self.to_v_head_gate.weight, 0)
            nn.init.constant_(self.to_v_head_gate.bias, 10)
        self.to_value_residual_mix = nn.Sequential(nn.Linear(dim, heads), nn.Sigmoid()) if learned_value_residual_mix else None
        self.to_out = nn.Linear(inner, dim, bias=False)


class _GLU(Module):
    def __init__(self, dim_in, dim_out, mult_bias=False):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)   # x-transformers' GLU keeps this bias whatever no_bias says
        self.mult_bias = nn.Parameter(torch.ones(dim_out)) if mult_bias else None


class FeedForward(Module):  # A.2
    def __init__(self, dim, mult, dropout, act=GLU_GELU, glu_mult_bias=False, no_bias=False, zero_init_output=False):
        super().__init__()
        inner = int(dim * mult)
        self.act = act
        self.ff = nn.Sequential(_GLU(dim, inner, glu_mult_bias), nn.Dropout(dropout), nn.Linear(inner, dim, bias=not no_bias))
        if zero_init_output:
            nn.init.zeros_(self.ff[2].weight)
            if self.ff[2].bias is not None:
                nn.init.zeros_(self.ff[2].bias)


class TextAudioCrossCondition(Module):  # e2_tts.py:486-513
    def __init__(self, dim, dim_text, cond_audio_to_text=True):
        super().__init__()
        self.text_to_audio = nn.Linear(dim_text + dim, dim, bias=False)
        nn.init.zeros_(self.text_to_audio.weight)
        self.cond_audio_to_text = cond_audio_to_text
        if cond_audio_to_text:
            self.audio_to_text = nn.Linear(dim + dim_text, dim_text, bias=False)
            nn.init.zeros_(self.audio_to_text.weight)


class _HCNorm(Module):
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.zeros(dim))


class HyperConnections(Module):  # A.5
    def __init__(self, num_residual_streams, *, dim):
        super().__init__()
        S = num_residual_streams
        self.norm = _HCNorm(dim)
        self.static_beta = nn.Parameter(torch.ones(S))
        a0 = torch.zeros(S, 1)
        a0[randrange(S), 0] = 1.
        self.static_alpha = nn.Parameter(torch.cat([a0, torch.eye(S)], dim=1))
        self.dynamic_alpha_fn = nn.Parameter(torch.zeros(dim, S + 1))
        self.dynamic_alpha_scale = nn.Parameter(torch.ones(()) * 1e-2)
        self.dynamic_beta_fn = nn.Parameter(torch.zeros(dim))
        self.dynamic_beta_scale = nn.Parameter(torch.ones(()) * 1e-2)

    def params(self):
        return (self.norm.gamma, self.dynamic_alpha_fn, self.dynamic_alpha_scale, self.static_alpha, self.dynamic_beta_fn,
                self.dynamic_beta_scale, self.static_beta)


class Residual(Module):
    """The reference's disabled hyper-connection (num_residual_streams=1, e2_tts.py:607): a plain residual `out + residual`, without
    parameters. Kept in `hyper_conns` so that the module tree matches the reference's."""

    def __init__(self, num_residual_streams=1, *, dim=None):
        super().__init__()


class RandomFourierEmbed(Module):  # e2_tts.py:355-364
    def __init__(self, dim):
        super().__init__()
        assert dim % 2 == 0
        self.register_buffer('weights', torch.randn(dim // 2))


class RotaryEmbedding(Module):  # A.3 (buffer kept for state_dict compatibility; the kernels use a cos/sin table)
    def __init__(self, dim):
        super().__init__()
        self.register_buffer('inv_freq', 1. / (10000 ** (torch.arange(0, dim, 2).float() / dim)))


class CharacterEmbed(Module):  # e2_tts.py:390-412
    def __init__(self, dim, num_embeds=256):
        super().__init__()
        self.dim = dim
        self.embed = nn.Embedding(num_embeds + 1, dim)

    def ids(self, text, max_seq_len):
        """(b, nt) int64 with -1 padding -> (b, max_seq_len) int32 row indices (filler 0), e2_tts.py:407-410"""
        text = (text + 1)[:, :max_seq_len]
        if text.shape[1] < max_seq_len:
            text = F.pad(text, (0, max_seq_len - text.shape[1]), value=0)
        return text.to(torch.int32).contiguous()


class InterpolatedCharacterEmbed(Module):  # e2_tts.py:414-482 (E2TTS(interpolated_text=True), :1135, :1233)
    """Parameter holder with the reference's state_dict keys (`embed.weight`, `abs_pos_mlp.1.*`, `abs_pos_mlp.3.*`); the arithmetic is
    ops.InterpText. Character ids index the table directly (no +1 shift, :446) and padding (-1) is dropped per sample (:445)."""

    def __init__(self, dim, num_embeds=256):
        super().__init__()
        self.dim = dim
        self.embed = nn.Embedding(num_embeds, dim)
        self.abs_pos_mlp = nn.Sequential(nn.Identity(), nn.Linear(1, dim), nn.SiLU(), nn.Linear(dim, dim))   # index 0 = the reference's Rearrange

    @staticmethod
    def compact(text):
        """(b, nt) int64 with -1 padding anywhere -> (ids int32 (b, nt) with each row's valid characters first, in their original order;
        text_len int32 (b,)) — `one_text[one_text >= 0]` of e2_tts.py:445-446 for the whole batch."""
        valid = text >= 0
        order = torch.argsort((~valid).to(torch.int8), dim=1, stable=True)
        ids_c = torch.gather(text.clamp(min=0), 1, order).to(torch.int32).contiguous()
        return ids_c, valid.sum(dim=1).to(torch.int32)

    def embed_bf16(self, text, max_seq_len, mask, w2_packed):
        """text (b, nt) int64 with -1 padding, mask (b, n) bool | None, w2_packed: the bf16 copy of abs_pos_mlp[3].weight
        -> bf16 [b * n, dim] (rows of masked frames are zero)."""
        B = text.shape[0]
        ids_c, text_len = self.compact(text)
        if exists(mask):
            audio_len = mask.sum(dim=1).to(torch.int32)                           # :455-457
            mask_u8 = mask.to(torch.uint8).contiguous()
        else:
            audio_len = torch.full((B,), max_seq_len, device=text.device, dtype=torch.int32)
            mask_u8 = None
        lin1, lin2 = self.abs_pos_mlp[1], self.abs_pos_mlp[3]
        return ops.InterpText.apply(ids_c, text_len, audio_len, mask_u8, self.embed.weight, lin1.weight, lin1.bias, lin2.weight, w2_packed,
                                    lin2.bias, B, max_seq_len)


# ----------------------------------------------------------------------------------------------------------------------
# weight packing: one kernel launch per forward refreshes every bf16 GEMM operand from the fp32 parameters


class WeightPack:
    """The GEMM operands of one model: bf16 (or fp32) copies of its parameters in the layouts the kernels read, all written by
    ONE b200_pack_weights launch. The module whose forward the user calls (E2TTS, DurationPredictor, or a Transformer called
    directly) owns one pack and runs it at the start of every forward, so the operands always match the current parameters."""

    def __init__(self, device):
        self.device = device
        self.entries = []  # (param, dst, rows, cols, ld_dst, row_off, col_off, mode, out_fp32)
        self.dev_table = None
        self.ptrs = None
        self.frozen = False

    def buffer(self, *shape, dtype=BF16):
        """A zero-filled destination on the pack's device (padding that no entry writes stays 0)."""
        return torch.zeros(shape, device=self.device, dtype=dtype)

    def add(self, param, dst, *, ld=None, row_off=0, col_off=0, mode=0):
        p2 = param if param.dim() != 3 else param.reshape(param.shape[0], -1)
        rows, cols = (p2.shape[0], 1) if p2.dim() == 1 else p2.shape
        if ld is None:
            ld = dst.shape[-1] if dst.dim() > 1 else 1
        self.entries.append((param, dst, rows, cols, ld, row_off, col_off, mode, int(dst.dtype == F32)))

    def run(self):
        if self.frozen:
            return
        ptrs = tuple(e[0].data_ptr() for e in self.entries)
        if ptrs != self.ptrs:   # rebuilt only when a parameter gets new storage: a CUDA-graph capture never copies host to device
            Desc = lib.STRUCTS['b200_pack_desc']
            arr = (Desc * len(self.entries))()
            for i, (p, dst, rows, cols, ld, ro, co, mode, f32) in enumerate(self.entries):
                arr[i].src, arr[i].dst = p.data_ptr(), dst.data_ptr()
                arr[i].rows, arr[i].cols, arr[i].ld_dst, arr[i].row_off, arr[i].col_off, arr[i].mode, arr[i].out_fp32 = rows, cols, ld, ro, co, mode, f32
            raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
            self.dev_table = raw.to(self.device)
            self.ptrs = ptrs
        ops.pack_weights(self.dev_table, len(self.entries))

    @contextlib.contextmanager
    def freeze(self):
        """Pack now, then skip every run() inside the block: for a block in which the weights cannot change (sample()'s ODE solve)."""
        self.run()
        was, self.frozen = self.frozen, True
        try:
            yield
        finally:
            self.frozen = was


class _PackOwner(Module):
    """A module that can own a WeightPack. `_add_weights(pack)` lays out its operands and returns their handles. The pack and the
    rotary tables are derived device state: `_apply` (.to(), .cuda(), .float(), ...) drops them, and a deep copy (EMA(model))
    starts without them and without any attribute listed in `_NOT_COPIED`, so the copy never holds buffers that the original
    packs into."""
    _NOT_COPIED = ('_derived',)

    def __init__(self):
        super().__init__()
        self._derived = {}

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._derived = {}
        return out

    def __deepcopy__(self, memo):
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k in self._NOT_COPIED else copy.deepcopy(v, memo)
        new._derived = {}
        return new

    def _pack(self):
        """-> (this module's WeightPack, the handles `_add_weights` returned), built on first use."""
        if 'pack' not in self._derived:
            pack = WeightPack(next(self.parameters()).device)
            self._derived['pack'] = pack, self._add_weights(pack)
        return self._derived['pack']

    def _packed_weights(self):
        """Refresh the pack from the current parameters (one launch, none while frozen) and return its handles."""
        pack, handles = self._pack()
        pack.run()
        return handles


# ----------------------------------------------------------------------------------------------------------------------


class LinearFourierEmbed(Module):
    """e2_tts.py:368-386 — parameter holder (`linear.weight`, reference state_dict key `layers.{i}.0.4.linear.weight`); the arithmetic is
    ops.FourierLinear (wgmma GEMM + b200_fourier_feat_*)."""

    def __init__(self, dim, p=0.5):
        super().__init__()
        assert p <= 1.
        dim_fourier = int(p * dim)
        dim_rest = dim - (dim_fourier * 2)
        self.linear = nn.Linear(dim, dim_fourier + dim_rest, bias=False)
        self.split_dims = (dim_fourier, dim_rest)


def _parse_attn_kwargs(attn_kwargs):
    """x-transformers Attention keywords (e2_tts.py:548-551, passed to both the audio and the text attention) -> (gate_value_heads,
    softclamp or None). A missing key takes x-transformers' default, so dict() is attention without head gate and without clamp."""
    unknown = sorted(set(attn_kwargs) - set(ATTN_KWARGS_DEFAULTS))
    if unknown:
        _unsupported(f'attn_kwargs[{unknown[0]!r}]', attn_kwargs[unknown[0]], 'e2_tts.py:548-551')
    kw = {**ATTN_KWARGS_DEFAULTS, **attn_kwargs}
    if not kw['softclamp_logits']:
        return bool(kw['gate_value_heads']), None
    clamp = float(kw['logit_softclamp_value'])
    if not 0. < clamp <= SOFTCLAMP_MAX:
        raise NotImplementedError(
            f'attn_kwargs logit_softclamp_value={clamp!r}: the clamped attention kernels take a clamp in (0, {SOFTCLAMP_MAX:g}], because they '
            f'exponentiate the clamped logits without a running maximum; use softclamp_logits=False for attention without the clamp')
    return bool(kw['gate_value_heads']), clamp


def _parse_ff_kwargs(ff_kwargs):
    """x-transformers FeedForward keywords (e2_tts.py:552, passed to both the audio and the text FeedForward) -> the keyword arguments of
    FeedForward above. A missing key takes x-transformers' default; a refused switch set to its default value is accepted."""
    taken = sorted(set(ff_kwargs) & {'dim', 'mult', 'glu', 'dropout'})
    if taken:   # the reference passes these itself: its FeedForward(...) call fails the same way
        raise TypeError(f'FeedForward() got multiple values for keyword argument {taken[0]!r} (ff_kwargs, e2_tts.py:552)')
    unknown = sorted(set(ff_kwargs) - set(FF_KWARGS_DEFAULTS))
    if unknown:
        _unsupported(f'ff_kwargs[{unknown[0]!r}]', ff_kwargs[unknown[0]], 'e2_tts.py:552')
    kw = {**FF_KWARGS_DEFAULTS, **ff_kwargs}
    for key in ('custom_activation', 'solu', 'post_act_ln', 'sublayer_dropout', 'dim_out'):
        if kw[key] != FF_KWARGS_DEFAULTS[key]:
            _unsupported(f'ff_kwargs[{key!r}]', kw[key], 'e2_tts.py:552')
    act = GLU_RELU2 if kw['relu_squared'] else GLU_SILU if kw['swish'] else GLU_GELU   # x-transformers' precedence
    return dict(act=act, glu_mult_bias=bool(kw['glu_mult_bias']), no_bias=bool(kw['no_bias']),
                zero_init_output=bool(kw['zero_init_output']))


class Transformer(_PackOwner):
    """Multistream flow-matching backbone — constructor and forward signature of the reference's Transformer
    (e2_tts.py:518-952). Non-default research switches raise (no kernels, no fallback)."""
    _NOT_COPIED = ('_derived', '_seed_dev')   # the copy gets no GraphedTrainStep seed word of its own

    def __init__(
        self, *, dim, dim_text=None, depth=8, heads=8, dim_head=64, ff_mult=4, text_depth=None, text_heads=None, text_dim_head=None,
        text_ff_mult=None, has_freq_axis=False, freq_heads=None, freq_dim_head=None, cond_on_time=True, abs_pos_emb=True,
        max_seq_len=8192, kernel_size=31, dropout=0.1, num_registers=32, scale_residual=False, attn_laser=False,
        attn_laser_softclamp_value=15., attn_fourier_embed_input=False, attn_fourier_embed_input_frac=0.25, num_residual_streams=4,
        attn_kwargs: dict = dict(gate_value_heads=True, softclamp_logits=True), ff_kwargs: dict = dict(),
        checkpoint_activations: bool = False,
    ):
        super().__init__()
        assert depth % 2 == 0, 'depth needs to be even'
        if has_freq_axis:
            _unsupported('has_freq_axis', has_freq_axis, 'e2_tts.py:533')
        if attn_laser:
            _unsupported('attn_laser', attn_laser, 'e2_tts.py:543')
        gate_value_heads, self.softclamp = _parse_attn_kwargs(attn_kwargs)
        ff_kw = _parse_ff_kwargs(dict(ff_kwargs))
        if num_residual_streams not in SUPPORTED_RESIDUAL_STREAMS:
            raise NotImplementedError(
                f'num_residual_streams={num_residual_streams!r} (e2_tts.py:547): supported values are 1 (plain residual) and 4 '
                f'(hyper-connections; the kernels lay out 4 streams per token); there is no fallback path (SURVEY.md §2 row 8)')
        dim_text = default(dim_text, dim // 2)
        text_heads, text_dim_head = default(text_heads, heads), default(text_dim_head, dim_head)
        text_ff_mult, text_depth = default(text_ff_mult, ff_mult), default(text_depth, depth)
        for name, value in (('dim_head', dim_head), ('text_dim_head', text_dim_head)):
            if value not in SUPPORTED_DIM_HEADS:
                raise NotImplementedError(
                    f'{name}={value!r} (e2_tts.py:527, :531): supported head dims are 64 and 128, the widths the attention kernels are '
                    f'built for; there is no fallback path (SURVEY.md §2 row 8)')
        assert heads >= 1 and text_heads >= 1, 'heads and text_heads must be >= 1'
        assert 1 <= text_depth <= depth
        for name, width, line in (('dim', dim, ':523'), ('dim_text', dim_text, ':524, :566')):
            if width % 64 or width > 1024:
                raise NotImplementedError(
                    f'{name}={width!r} (e2_tts.py{line}): the kernels take model widths that are multiples of 64 up to 1024; there is no '
                    f'fallback path (SURVEY.md §2 row 8)')
        for name, width, mult, line in (('ff_mult', dim, ff_mult, ':646'), ('text_ff_mult', dim_text, text_ff_mult, ':692')):
            if int(width * mult) % 64:
                raise NotImplementedError(
                    f'{name}={mult!r} (e2_tts.py{line}): the feed-forward inner width int({width} * {mult!r}) = {int(width * mult)} is not a '
                    f'multiple of 64; the GLU kernels pack the hidden units in 64-column halves; there is no fallback path (SURVEY.md §2 row 8)')

        self.max_seq_len = max_seq_len
        self.abs_pos_emb = nn.Embedding(max_seq_len, dim) if abs_pos_emb else None
        self.dim, self.dim_text, self.depth, self.text_depth = dim, dim_text, depth, text_depth
        self.heads, self.dim_head = heads, dim_head
        self.text_heads, self.text_dim_head = text_heads, text_dim_head
        self.has_freq_axis = False
        self.dropout = dropout
        self.num_streams = num_residual_streams
        # Activation checkpointing (not a reference switch): a training forward under autograd keeps only each layer's boundary tensors
        # and recomputes the layer's sub-blocks in the backward (_run_layers, ops.Segment) — less memory for about one more forward
        # of the stack. The right choice depends on batch and clip length, so it is the user's; a plain attribute, read every forward.
        self.checkpoint_activations = bool(checkpoint_activations)

        self.num_registers = num_registers
        self.registers = nn.Parameter(torch.zeros(num_registers, dim))
        nn.init.normal_(self.registers, std=0.02)
        self.text_registers = nn.Parameter(torch.zeros(num_registers, dim_text))
        nn.init.normal_(self.text_registers, std=0.02)
        self.rotary_emb = RotaryEmbedding(dim_head)
        self.text_rotary_emb = RotaryEmbedding(text_dim_head)

        self.cond_on_time = cond_on_time
        norm_klass = AdaptiveRMSNorm if cond_on_time else RMSNorm
        post_klass = partial(AdaLNZero, dim) if cond_on_time else Identity
        self.time_cond_mlp = nn.Sequential(RandomFourierEmbed(dim), nn.Linear(dim + 1, dim), nn.SiLU()) if cond_on_time else Identity()

        layers, hyper_conns = [], []
        hc = partial(HyperConnections if num_residual_streams != 1 else Residual, num_residual_streams)   # :607, disable = S == 1
        for ind in range(depth):
            first, later_half, has_text = ind == 0, ind >= depth // 2, ind < text_depth
            speech = ModuleList([
                nn.Linear(dim * 2, dim, bias=False) if later_half else None,
                DepthwiseConv(dim, kernel_size=kernel_size),
                norm_klass(dim),
                Attention(dim, heads, dim_head, not first, gate_value_heads),
                LinearFourierEmbed(dim, p=attn_fourier_embed_input_frac) if attn_fourier_embed_input else nn.Identity(),   # :639
                post_klass(),
                norm_klass(dim),
                FeedForward(dim, ff_mult, dropout, **ff_kw),
                post_klass(),
                None, None, None,
            ])
            speech_hc = ModuleList([hc(dim=dim), hc(dim=dim), hc(dim=dim), None])
            text, text_hc = None, None
            if has_text:
                text = ModuleList([
                    DepthwiseConv(dim_text, kernel_size=kernel_size),
                    RMSNorm(dim_text),
                    Attention(dim_text, text_heads, text_dim_head, not first, gate_value_heads),
                    RMSNorm(dim_text),
                    FeedForward(dim_text, text_ff_mult, dropout, **ff_kw),
                    TextAudioCrossCondition(dim, dim_text, cond_audio_to_text=ind != text_depth - 1),
                ])
                text_hc = ModuleList([hc(dim=dim_text), hc(dim=dim_text), hc(dim=dim_text)])
            hyper_conns.append(ModuleList([speech_hc, text_hc]))
            layers.append(ModuleList([speech, text]))
        self.layers = ModuleList(layers)
        self.hyper_conns = ModuleList(hyper_conns)
        self.final_norm = RMSNorm(dim)

        # optional int64 device word added to every dropout seed when the kernels RUN (include/b200_e2tts.h "dropout seeds"):
        # set by GraphedTrainStep, whose captured graph would otherwise replay the same dropout masks on every step
        self._seed_dev = None

    # ------------------------------------------------------------------ packed operands
    def _add_weights(self, pack):
        """Add every per-layer GEMM operand and the stacked to_gamma weights to `pack`; -> dict(layers=[per-layer handles], cond=...)."""
        d, dt = self.dim, self.dim_text
        packed = []
        e = pack.buffer
        cond_rows = []
        for i, (speech, text) in enumerate(self.layers):
            L = {}
            for pre, mods, din in (('a', speech, d), ('t', text, dt)):
                if mods is None:
                    continue
                attn = mods[3] if pre == 'a' else mods[2]
                ff = mods[7] if pre == 'a' else mods[4]
                has_mix = attn.to_value_residual_mix is not None
                has_gate = attn.to_v_head_gate is not None
                H, I = attn.heads, attn.heads * attn.dim_head   # per stream: the text attention may have its own geometry
                qkv = e(3 * I + (int(has_gate) + int(has_mix)) * H, din)   # rows [q | k | v | gate | mix], gate and mix optional
                for j, lin in enumerate((attn.to_q, attn.to_k, attn.to_v)):
                    pack.add(lin.weight, qkv, row_off=j * I)
                if has_gate:
                    pack.add(attn.to_v_head_gate.weight, qkv, row_off=3 * I)
                if has_mix:
                    pack.add(attn.to_value_residual_mix[0].weight, qkv, row_off=3 * I + (H if has_gate else 0))
                out_w = e(din, I)
                pack.add(attn.to_out.weight, out_w)
                inner = ff.ff[2].weight.shape[1]
                w1, b1 = e(2 * inner, din), e(2 * inner, dtype=F32)
                pack.add(ff.ff[0].proj.weight, w1, mode=1)
                pack.add(ff.ff[0].proj.bias, b1, mode=1)
                w2 = e(din, inner)
                pack.add(ff.ff[2].weight, w2)
                L[pre] = dict(qkv=qkv, out=out_w, w1=w1, b1=b1, w2=w2)
            if isinstance(speech[4], LinearFourierEmbed):
                lfe = e(*speech[4].linear.weight.shape)
                pack.add(speech[4].linear.weight, lfe)
                L['a']['lfe'] = lfe
            if speech[0] is not None:
                L['skip'] = e(d, 2 * d)
                pack.add(speech[0].weight, L['skip'])
            if text is not None:
                cc = text[5]
                stack = e(d + (dt if cc.cond_audio_to_text else 0), d + dt)
                pack.add(cc.text_to_audio.weight, stack)
                if cc.cond_audio_to_text:
                    pack.add(cc.audio_to_text.weight, stack, row_off=d)
                L['cross'] = stack
            if self.cond_on_time:
                cond_rows += [speech[2].to_gamma, speech[5].to_gamma, speech[6].to_gamma, speech[8].to_gamma]
            packed.append(L)
        cond = None
        if self.cond_on_time:
            n = len(cond_rows) * d
            W_all, b_all = e(n, d, dtype=F32), e(n, dtype=F32)
            for j, lin in enumerate(cond_rows):
                pack.add(lin.weight, W_all, row_off=j * d)
                if lin.bias is not None:
                    pack.add(lin.bias, b_all, row_off=j * d)
            cond = dict(W=W_all, b=b_all, lins=cond_rows)
        return dict(layers=packed, cond=cond)

    def _rotary(self, Np, dim_head, dev):
        rot = self._derived.setdefault('rot', {})
        if (Np, dim_head) not in rot:
            rot[Np, dim_head] = ops.rotary_table(Np, dev, dim_head)
        return rot[Np, dim_head]

    # ------------------------------------------------------------------ conditioning vectors
    def _cond_gains(self, times, batch, c):
        """time_cond_mlp (:621-625, 778-789) and every per-layer to_gamma projection in ONE batched launch; `c` is the packed
        to_gamma stack. Returns a list [4 * depth] of contiguous fp32 [B, d]: (1 + gamma) for the adaptive norms, sigmoid gates for AdaLNZero."""
        if times.ndim == 0:
            times = times.expand(batch)
        times = times.to(F32).contiguous()
        four = ops.fourier_embed(times, self.time_cond_mlp[0].weights)
        lin = self.time_cond_mlp[1]
        cond = ops.SmallLinear.apply(four, lin.weight, lin.bias, 1, self.dim, False)
        weights = [l.weight for l in c['lins']]
        biases = [l.bias for l in c['lins'] if l.bias is not None]  # AdaLNZero gates sit on the odd d-wide segments
        W, b_full = ops.CondPack.apply(c['W'], c['b'], self.dim, len(weights), *weights, *biases)
        gains = ops.SmallLinear.apply(cond, W, b_full, 5, self.dim, True)
        return list(gains.unbind(0))

    # ------------------------------------------------------------------ the block stack
    def _run_layers(self, P, xs, ts, gains, mask_u8, B, Np, seed, Bt=None):
        """P: the per-layer packed operands; xs bf16 [T,S,d], ts bf16 [Tt,S,dt] | None -> final residual streams. Layer loop of e2_tts.py:825-939.
        Bt: the items that carry text, the first Bt of the B (Tt = Bt * Np; default all); the others pass the layers as without text."""
        # the audio and the text attention may differ in head count and width: each call takes both, and the rotary table, from its module
        rot = {dh: self._rotary(Np, dh, xs.device) for dh in {self.dim_head, self.text_dim_head}}
        p_drop = self.dropout if self.training else 0.0
        mbits = ops.attn_maskbits(mask_u8, B, Np, xs.device) if xs.is_cuda else None   # one key-mask bitmask for all 2 * depth attention calls
        # Hyper-connection plumbing of one stream: a sub-block returns its depth connection PENDING — (residual', branch_out, beta) — and
        # the next sub-block's width connection consumes it in one fused kernel (ops.HcDepthWidth) when the stream's rows allow it;
        # `close` materialises the streams where something else reads them (cross-conditioning, skip path, final norm).
        # (items, key mask, bitmask, fuse) of the audio and of the text stream: rows are item-major, so the text items' mask is a row
        # prefix, and each stream decides the fusion on its own rows, as a pass over its items alone would
        ageo = tgeo = (B, mask_u8, mbits, ops.hc_can_fuse(xs.shape[0], xs.shape[1]))
        if Bt is not None and Bt != B:
            tmask = mask_u8[:Bt] if mask_u8 is not None else None
            tgeo = (Bt, tmask, ops.attn_maskbits(tmask, Bt, Np, xs.device) if xs.is_cuda else None, ops.hc_can_fuse(Bt * Np, xs.shape[1]))
        skips = []
        v_first, tv_first = None, None
        nseed = [seed]

        def next_seed():
            nseed[0] = (nseed[0] * 6364136223846793005 + 1442695040888963407) & 0x7FFFFFFFFFFFFFFF
            return nseed[0]

        # num_residual_streams=1 (e2_tts.py:607, disable=True): every sub-block is x + branch(norm(x)). The width connection is then
        # the branch norm alone (the conv sub-block has none) and hands x on as `rest`; the branch's last launch (the conv kernel, the
        # to_out / FF-out GEMM epilogue) adds it, so the depth connection is nothing but a view back to [T, 1, D].
        plain = self.num_streams == 1

        def width(res, hcm, gain, mode, B):
            if plain:
                x2 = res.view(res.shape[0], res.shape[-1])
                if mode == 0:
                    return x2, x2, None
                br, xr = ops.BranchNorm.apply(x2, gain if mode == 1 else None, gain if mode == 2 else None, B, Np)
                return br, xr, None
            if isinstance(res, tuple):
                return ops.HcDepthWidth.apply(*res, *hcm.params(), gain, mode, Np)
            return ops.HcWidth.apply(res, *hcm.params(), gain, mode, Np)

        def depth(rest, y, beta, fuse):
            if plain:
                return y.view(y.shape[0], 1, y.shape[1])
            return (rest, y, beta) if fuse else ops.HcDepth.apply(rest, y, beta)

        def close(res):
            return ops.HcDepth.apply(*res) if isinstance(res, tuple) else res

        def sub_conv(res, hcm, conv, geo):
            B, mask_u8, _, fuse = geo
            br, rest, beta = width(res, hcm, None, 0, B)
            y = ops.DwConv.apply(br, conv.dw_conv1d[0].weight, conv.dw_conv1d[0].bias, mask_u8, B, Np, plain)
            return depth(rest, y, beta, fuse)

        def sub_attn(res, hcm, gain, mode, attn, pk, vf, colscale, seed, geo, lfe=None):
            B, mask_u8, mbits, fuse = geo
            br, rest, beta = width(res, hcm, gain, mode, B)
            if lfe is not None:   # attn_input_fourier_embed (:909): between the attention norm (fused into the width kernel) and the attention
                br = ops.FourierLinear.apply(br, lfe.linear.weight, pk['lfe'], *lfe.split_dims)
            mix, gate = attn.to_value_residual_mix, attn.to_v_head_gate
            cs, sn = rot[attn.dim_head]
            og, v = ops.Attention.apply(br, attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, gate.weight if gate is not None else None,
                                        gate.bias if gate is not None else None, mix[0].weight if mix is not None else None,
                                        mix[0].bias if mix is not None else None, vf if mix is not None else None,
                                        pk['qkv'], cs, sn, mask_u8, B, Np, attn.heads, p_drop, seed, self.softclamp, self._seed_dev, mbits,
                                        attn.dim_head)
            y = ops.OutProj.apply(og, attn.to_out.weight, pk['out'], colscale, mask_u8, B, Np, rest if plain else None)
            return depth(rest, y, beta, fuse), (v if vf is None else vf)

        def sub_ff(res, hcm, gain, mode, ff, pk, colscale, seed, geo):
            B, fuse = geo[0], geo[3]
            br, rest, beta = width(res, hcm, gain, mode, B)
            y = ops.FeedForward.apply(br, ff.ff[0].proj.weight, ff.ff[0].proj.bias, ff.ff[2].weight, ff.ff[2].bias,
                                      pk['w1'], pk['b1'], pk['w2'], colscale, B, Np, p_drop, seed, self._seed_dev,
                                      rest if plain else None, ff.act, ff.ff[0].mult_bias)
            return close(depth(rest, y, beta, fuse))

        def text_subblocks(i, ts, tvf, gains, seeds, pk):  # the three text sub-blocks of layer i (:853-882; no gains: plain RMSNorms)
            text, thc = self.layers[i][1], self.hyper_conns[i][1]
            ts = sub_conv(ts, thc[0], text[0], tgeo)
            ts, tvf = sub_attn(ts, thc[1], text[1].g, 1, text[2], pk, tvf, None, seeds[0], tgeo)
            return sub_ff(ts, thc[2], text[3].g, 1, text[4], pk, None, seeds[1], tgeo), tvf

        def audio_subblocks(i, xs, vf, gains4, seeds, pk):  # the three audio sub-blocks of layer i (:900-939)
            speech, shc = self.layers[i][0], self.hyper_conns[i][0]
            g_an, g_az, g_fn, g_fz = gains4
            mode = 2 if self.cond_on_time else 1
            xs = sub_conv(xs, shc[0], speech[1], ageo)  # :900-902
            xs, vf = sub_attn(xs, shc[1], g_an, mode, speech[3], pk, vf, g_az, seeds[0], ageo,
                              speech[4] if isinstance(speech[4], LinearFourierEmbed) else None)  # :906-916
            return sub_ff(xs, shc[2], g_fn, mode, speech[7], pk, g_fz, seeds[1], ageo), vf  # :936-939

        # Transformer(checkpoint_activations=True) under autograd: each layer's audio sub-blocks and each text block are one
        # ops.Segment, which keeps only its inputs and runs the sub-blocks again in the backward. The seeds are drawn here, in the
        # order of the plain path, and handed in, so the recompute draws the dropout masks of the forward.
        ckpt = self.checkpoint_activations and self.training and torch.is_grad_enabled()

        def segment(subblocks, i, res, vf, gains, seeds, pk):
            """subblocks(i, res, vf, gains, seeds, pk) -> (closed stream tensor, values), plain or as one ops.Segment"""
            if not ckpt:
                return subblocks(i, res, vf, gains, seeds, pk)
            keys, first = tuple(pk), vf is None

            def run(res, vf, *rest):
                gains, w = rest[:len(rest) - len(keys)], rest[len(rest) - len(keys):]
                out, v = subblocks(i, res, vf, gains, seeds, dict(zip(keys, w)))
                return (out, v) if first else (out,)
            outs = ops.Segment.apply(run, res, vf, *gains, *pk.values())
            return outs[0], (outs[1] if first else vf)

        def text_block(i, ts, tvf):
            seeds = next_seed(), next_seed()
            return segment(text_subblocks, i, ts, tvf, (), seeds, P[i]['t'])

        # The text sub-blocks of layer i+1 depend on the cross-conditioning of layer i only, not on layer i's audio sub-blocks
        # (:853-939): enqueue them on a second stream so that the half-width text kernels (K = dt GEMMs, D = dt token kernels)
        # fill the launch gaps and tile-quantisation tails of the audio kernels instead of serialising with them. The autograd
        # engine replays the same fork/join in backward (each node runs on its forward stream). Tensors that cross streams are
        # registered with the caching allocator (record_stream).
        has_text = lambda i: ts is not None and i < len(self.layers) and self.layers[i][1] is not None
        two = TWO_STREAM and has_text(0) and xs.is_cuda
        if two:
            main, side = torch.cuda.current_stream(xs.device), _side_stream(xs.device)
            for t in (*tgeo[1:3], *[x for pair in rot.values() for x in pair]):
                if t is not None:
                    t.record_stream(side)

            def fork_text(i, ts_in, tvf):
                side.wait_stream(main)
                ts_in.record_stream(side)
                with torch.cuda.stream(side):
                    return text_block(i, ts_in, tvf)
            ts, tv_first = fork_text(0, ts, tv_first)

        for i, ((speech, text), (shc, thc)) in enumerate(zip(self.layers, self.hyper_conns)):
            pk = P[i]
            if ts is not None and text is not None:  # :853-883
                if two:
                    main.wait_stream(side)      # join: text sub-blocks of this layer (enqueued one layer ago)
                    ts.record_stream(main)
                else:
                    ts, tv_first = text_block(i, ts, tv_first)
                cc = text[5]
                xs, ts = ops.CrossCondition.apply(xs, ts, cc.text_to_audio.weight,
                                                  cc.audio_to_text.weight if cc.cond_audio_to_text else None, pk['cross'])
                if two and has_text(i + 1):
                    ts, tv_first = fork_text(i + 1, ts, tv_first)
            if (i + 1) <= self.depth // 2:  # :887-896
                skips.append(xs)
            else:
                xs = ops.SkipProj.apply(xs, skips.pop(), speech[0].weight, pk['skip'])
            gains4 = tuple(gains[4 * i:4 * i + 4]) if self.cond_on_time else (speech[2].g, None, speech[6].g, None)
            seeds = next_seed(), next_seed()
            xs, v_first = segment(audio_subblocks, i, xs, v_first, gains4, seeds, pk['a'])
        assert not skips
        return xs

    def _prepare(self, B, N, mask):
        Np = N + self.num_registers
        assert N <= self.max_seq_len, f'{N} exceeds the set `max_seq_len` ({self.max_seq_len}) on Transformer'
        mask_u8 = None
        if exists(mask):
            mask_u8 = F.pad(mask, (self.num_registers, 0), value=True).to(torch.uint8).contiguous()
        return Np, mask_u8

    @_on_module_device
    def forward(self, x, times=None, mask=None, text_embed=None):
        """Reference signature (e2_tts.py:731-737): x (b, n, d) -> (b, n, d)."""
        assert x.ndim == 3, '`has_freq_axis` is not supported by this build'
        assert not (exists(times) ^ self.cond_on_time), '`times` must be passed in if `cond_on_time` is set to `True` and vice versa'
        B, N, d = x.shape
        if torch.is_grad_enabled():
            ops.zero_pool.begin(x.device)
        w = self._packed_weights()
        h = ops.CastRows.apply(x.reshape(B * N, d))
        te = ops.CastRows.apply(text_embed.reshape(B * N, -1)) if exists(text_embed) else None
        y = self._forward_from_h(w, h, B, N, times, mask, te_bf16=te)
        return y.view(B, N, d).to(x.dtype)

    def _forward_from_h(self, w, h, B, N, times, mask, text_ids=None, text_embed_module=None, te_bf16=None, text_items=None):
        """w: the handles of `_add_weights`, already packed; h bf16 [B*N, d] (already projected) -> final-normed bf16 [B*N, d].
        text_items: how many of the B items the text ids / embeddings are for (the first ones; default all). The other items run as
        without text — the text-dropped half of a batched classifier-free-guidance pass (E2TTS.cfg_pred_batched)."""
        S, R = self.num_streams, self.num_registers
        Bt = default(text_items, B)
        if Bt != B and torch.is_grad_enabled():
            raise NotImplementedError('text on a prefix of the items (text_items) is inference only: CrossCondition has no backward for it')
        Np, mask_u8 = self._prepare(B, N, mask)
        abs_w = self.abs_pos_emb.weight if exists(self.abs_pos_emb) else None
        xs = ops.Assemble.apply(h, abs_w, self.registers, B, N, S)
        ts = None
        if exists(text_ids):
            ts = ops.TextStem.apply(text_ids, text_embed_module.embed.weight, self.text_registers, Bt, N, S)
        elif exists(te_bf16):
            ts = ops.Assemble.apply(te_bf16, None, self.text_registers, Bt, N, S)
        gains = self._cond_gains(times, B, w['cond']) if self.cond_on_time else None
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if (self.training and self.dropout > 0) else 0
        xs = self._run_layers(w['layers'], xs, ts, gains, mask_u8, B, Np, seed, Bt)
        return ops.FinalNorm.apply(xs, self.final_norm.g, B, N, R)


# ----------------------------------------------------------------------------------------------------------------------
# MelSpec (e2_tts.py:248-290): parameter/buffer holder with torchaudio-compatible buffer names (Appendix B)


class _Spectrogram(Module):
    def __init__(self, win_length):
        super().__init__()
        self.register_buffer('window', torch.hann_window(win_length, periodic=True))   # [win_length], unpadded, as torchaudio keeps it


class _MelScale(Module):
    def __init__(self, n_freqs, n_mels, sample_rate, norm=None):
        super().__init__()
        self.register_buffer('fb', mel_filterbank(n_freqs, n_mels, sample_rate, norm=norm))


class _MelSTFT(Module):
    def __init__(self, n_fft, win_length, n_mels, sample_rate, norm=None):
        super().__init__()
        self.spectrogram = _Spectrogram(win_length)
        self.mel_scale = _MelScale(n_fft // 2 + 1, n_mels, sample_rate, norm)


def mel_filterbank(n_freqs, n_mels, sample_rate, f_min=0.0, f_max=None, norm=None):
    """HTK mel filterbank — what torchaudio.transforms.MelSpectrogram builds for the reference (:265-275); norm='slaney' scales
    filter i by 2 / (f[i+2] - f[i]) (torchaudio's melscale_fbanks), still on the HTK scale."""
    f_max = f_max if f_max is not None else sample_rate / 2
    hz2mel = lambda f: 2595.0 * math.log10(1.0 + f / 700.0)
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_pts = torch.linspace(hz2mel(f_min), hz2mel(f_max), n_mels + 2)
    f_pts = 700.0 * (10 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    fb = torch.clamp(torch.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]), min=0.0)
    if norm == 'slaney':
        fb *= (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels]))[None]
    return fb


MEL_NFFT_MIN, MEL_NFFT_MAX = 64, 4096


def _five_smooth(n):
    for p in (2, 3, 5):
        while n % p == 0:
            n //= p
    return n == 1


class MelSpec(Module):
    """The reference's MelSpec (e2_tts.py:248-290) with its full signature: torchaudio's MelSpectrogram semantics for win_length
    (a periodic Hann window of win_length <= n_fft taps, centred in the frame), center (reflect padding by n_fft // 2, or valid
    frames only), power > 0, normalize (True / 'window': divide X by sqrt(sum(window^2)); 'frame_length': by sqrt(n_fft)) and
    norm (None or 'slaney'), for any filter_length in [64, 4096] with no prime factor other than 2, 3 and 5."""

    def __init__(self, filter_length=1024, hop_length=256, win_length=1024, n_mel_channels=100, sampling_rate=24_000,
                 normalize=False, power=1, norm=None, center=True):
        super().__init__()
        win_length = filter_length if win_length is None else win_length
        if not (MEL_NFFT_MIN <= filter_length <= MEL_NFFT_MAX and _five_smooth(filter_length)):
            _unsupported('mel_spec_kwargs[\'filter_length\']', filter_length,
                         f'e2_tts.py:251 (the FFT kernels take n_fft in [{MEL_NFFT_MIN}, {MEL_NFFT_MAX}] with prime factors 2, 3 and 5 only)')
        if power is None:
            _unsupported('mel_spec_kwargs[\'power\']', power, 'e2_tts.py:257 (power=None is a complex spectrum, which the reference then takes the log of)')
        if not power > 0:
            raise ValueError(f'mel_spec_kwargs power must be positive (got {power!r})')
        if not 1 <= win_length <= filter_length:
            raise ValueError(f'mel_spec_kwargs win_length must be in [1, filter_length={filter_length}] (got {win_length}), as torch.stft requires')
        if normalize not in (False, True, 'window', 'frame_length'):
            raise ValueError(f"mel_spec_kwargs normalize must be a bool, 'window' or 'frame_length' (got {normalize!r})")
        if norm not in (None, 'slaney'):
            raise ValueError(f"mel_spec_kwargs norm must be None or 'slaney' (got {norm!r})")
        self.n_mel_channels, self.sampling_rate = n_mel_channels, sampling_rate
        self.n_fft, self.hop, self.win_length = filter_length, hop_length, win_length
        self.center, self.power = bool(center), float(power)
        self.mel_stft = _MelSTFT(filter_length, win_length, n_mel_channels, sampling_rate, norm)
        window = self.mel_stft.spectrogram.window.double()
        self.norm_scale = {False: 1.0, 'frame_length': filter_length ** -0.5}.get(normalize, float(window.square().sum().rsqrt()))
        self.register_buffer('dummy', torch.tensor(0), persistent=False)
        self._resample_table = None     # ops.ResampleTable of every rate pair collate() has met; its taps: buffer `resample_taps`

    def frames(self, n):
        """frames of n samples (int or tensor): 1 + n // hop centred (even n_fft), 1 + (n - n_fft) // hop without centring"""
        return ops.melspec_frames(n, self.n_fft, self.hop, self.center)

    def _melspec(self, waves, **kw):
        if waves.shape[1] < (self.n_fft // 2 + 1 if self.center else self.n_fft):
            raise ValueError(f'MelSpec: {waves.shape[1]} samples are too few for one frame of n_fft={self.n_fft} (center={self.center})')
        return ops.melspec(waves.to(F32).contiguous(), self.mel_stft.spectrogram.window, self.mel_stft.mel_scale.fb, self.n_fft, self.hop,
                           center=self.center, power=self.power, norm_scale=self.norm_scale, **kw)

    def forward(self, inp):
        if inp.ndim == 3:
            inp = inp[:, 0]
        assert inp.ndim == 2
        if self.dummy.device != inp.device:
            self.to(inp.device)
        return self._melspec(inp)

    def collate(self, waves, lens=None, sample_rates=None):
        """On-device data path (SURVEY §8f row 3): what the reference does per item on CPU workers — the resampling and `MelSpec` of
        HFDataset.__getitem__ (trainer.py:101-131) — and per batch in `collate_fn` (:61-82: zero-pad the mels to the longest,
        lengths) plus the trainer's `rearrange(batch['mel'], 'b d n -> b n d')` (:253), as at most two kernel launches over the
        ragged batch.
        waves: list of 1-D fp32 tensors or a zero-padded [B, nw_max] tensor with `lens` (samples per sequence).
        sample_rates: None (every item is at `sampling_rate`), an int, or a per-item list / 1-D tensor of positive integer rates.
        Items at another rate are resampled to `sampling_rate` first, as the dataset's torchaudio.transforms.Resample(rate,
        sampling_rate) does (same fp32 taps, same output length), all rates in one launch (ops.resample); items already at
        `sampling_rate` pass through unchanged, and a batch with no other rate takes no resampling launch at all.
        Returns dict(mel [B, n_frames_max, n_mels] fp32, mel_lengths [B] int64) — pass as
        `model(batch['mel'], text=..., lens=batch['mel_lengths'])`. A length past the padded wave counts as the padded length;
        an item too short for one frame — at most n_fft/2 samples centred (too short for the reflect padding: the reference's
        MelSpec raises on it), fewer than n_fft without centring — has zero frames and its mel_lengths entry is 0.
        n_frames_max is that of the longest resampled item with a list, and that of the padded width resampled at the slowest
        conversion present with a padded tensor."""
        B = len(waves) if isinstance(waves, (list, tuple)) else waves.shape[0]
        rates = self._collate_rates(sample_rates, B)
        if rates is not None and all(r == self.sampling_rate for r in rates):
            rates = None
        host_lens = [w.shape[-1] for w in waves] if isinstance(waves, (list, tuple)) else None
        if isinstance(waves, (list, tuple)):
            dev = self.dummy.device if self.dummy.device.type == 'cuda' else waves[0].device
            lens = torch.tensor([w.shape[-1] for w in waves], dtype=torch.int32)
            nmax = int(lens.max())
            padded = torch.zeros((len(waves), nmax), dtype=F32).pin_memory() if dev.type == 'cuda' and not waves[0].is_cuda else torch.zeros((len(waves), nmax), dtype=F32, device=waves[0].device)
            for i, w in enumerate(waves):
                padded[i, :w.shape[-1]] = w.reshape(-1)
            waves = padded.to(dev, non_blocking=True)
            lens = lens.to(dev, non_blocking=True)
        else:
            assert lens is not None and waves.ndim == 2
            lens = lens.to(device=waves.device, dtype=torch.int32)
        if self.dummy.device != waves.device:
            self.to(waves.device)
        if rates is not None:
            waves, lens = self._resample(waves.to(F32).contiguous(), lens.contiguous(), rates, host_lens)
        mel = self._melspec(waves, wave_lens=lens.contiguous(), out_bnd=True)
        lens = lens.long().clamp(max=waves.shape[1])      # the kernel clamps the same way
        long_enough = lens > self.n_fft // 2 if self.center else lens >= self.n_fft
        mel_lengths = torch.where(long_enough, self.frames(lens), 0)
        n_max = int(self.frames(waves.shape[1]))
        return dict(mel=mel[:, :n_max], mel_lengths=mel_lengths)

    @staticmethod
    def _collate_rates(sample_rates, B):
        """sample_rates -> a list of B ints, or None; what torchaudio refuses (a non-integer rate) or cannot mean (a rate <= 0) is a
        ValueError"""
        if sample_rates is None:
            return None
        if hasattr(sample_rates, 'ndim') and hasattr(sample_rates, 'tolist'):     # a tensor or a numpy array
            if sample_rates.ndim > 1:
                raise ValueError(f'sample_rates must be an int or a 1-D list / tensor of rates (got shape {tuple(sample_rates.shape)})')
            sample_rates = sample_rates.tolist()
        rates = list(sample_rates) if isinstance(sample_rates, (list, tuple)) else [sample_rates] * B
        if len(rates) != B:
            raise ValueError(f'sample_rates has {len(rates)} entries for a batch of {B}')
        out = []
        for r in rates:
            if isinstance(r, bool) or not isinstance(r, numbers.Real) or not math.isfinite(r) or int(r) != r or r <= 0:
                raise ValueError(f'sample rates must be positive integers (got {r!r}), as torchaudio.transforms.Resample requires')
            out.append(int(r))
        return out

    def _rate_table(self, rates, device):
        """the ops.ResampleTable of every rate pair met so far, rebuilt (host tap tables, one upload) when `rates` bring a new one;
        its data is the non-persistent buffer `resample_taps`, so it follows .to() and stays out of the state_dict"""
        pairs = {(r, self.sampling_rate) for r in rates if r != self.sampling_rate}
        table = self._resample_table
        if table is None or not pairs <= set(table.index):
            table = self._resample_table = ops.ResampleTable(sorted(pairs | set(table.index if table else ())), device=device)
            self.register_buffer('resample_taps', table.data, persistent=False)
        table.data = self.resample_taps
        return table

    def _resample(self, waves, lens, rates, host_lens):
        """one b200_resample launch to `sampling_rate` over the batch (items at that rate pass through) -> (waves [B, nr], lens)"""
        target = self.sampling_rate
        table = self._rate_table(rates, waves.device)
        nw = waves.shape[1]
        if host_lens is not None:
            nr = max(ops.resample_length(n, r, target) if r != target else n for n, r in zip(host_lens, rates))
        else:
            nr = max(ops.resample_length(nw, r, target) if r != target else nw for r in set(rates))
        idx = torch.tensor([table.index[(r, target)] if r != target else -1 for r in rates], dtype=torch.int32)
        if waves.is_cuda:
            idx = idx.pin_memory().to(waves.device, non_blocking=True)
        return ops.resample(waves, lens, idx, table, nr)


# ----------------------------------------------------------------------------------------------------------------------


class _HLGaussHead(Module):
    """hl-gauss-pytorch HLGaussLayer(dim, hl_gauss_loss, use_regression, regress_activation=Softplus()) (A.6; e2_tts.py:1035-1040):
    the regression head Linear(dim, 1) -> Softplus with the MSE loss, or with use_regression=False the classification head
    Linear(dim, num_bins) with the HL-Gauss loss. `hl_gauss_loss` is checked in both modes, as the reference builds its HLGaussLoss
    either way; the loss holds no parameters or buffers, so the state_dict is `to_pred.0.weight` / `.bias` in both."""

    def __init__(self, dim, hl_gauss_loss=None, use_regression=True):
        super().__init__()
        if not use_regression and hl_gauss_loss is None:
            raise ValueError('DurationPredictor: use_regression=False needs `hl_gauss_loss` (hl-gauss-pytorch HLGaussLayer asserts it)')
        self.spec = ops.HLGaussSpec(**hl_gauss_loss) if hl_gauss_loss is not None else None
        self.use_regression = bool(use_regression)
        if self.use_regression:
            self.to_pred = nn.Sequential(nn.Linear(dim, 1), nn.Softplus())
        else:
            if self.spec.num_bins > ops.HL_GAUSS_MAX_BINS:
                _unsupported('hl_gauss_loss num_bins', self.spec.num_bins,
                             f'e2_tts.py:966 (the HL-Gauss loss kernel takes at most {ops.HL_GAUSS_MAX_BINS} bins)')
            self.to_pred = nn.Sequential(nn.Linear(dim, self.spec.num_bins))

    def forward(self, pooled, target=None):
        """pooled fp32 [B, dim] -> the prediction [B] (target None) or the loss against target [B]"""
        lin = self.to_pred[0]
        if self.use_regression:
            pred = ops.SmallLinear.apply(pooled, lin.weight, lin.bias, 4, 1, False).squeeze(-1)
            if target is None:
                return pred
            return F.mse_loss(pred, target)  # (B,) scalar glue, :1111
        logits = ops.SmallLinear.apply(pooled, lin.weight, lin.bias, 0, 1, False)
        if target is None:
            return ops.hl_gauss_predict(logits, self.spec)
        return ops.HLGaussLoss.apply(logits, target, self.spec)


def _resolve_tokenizer(tokenizer, text_num_embeds):
    if callable(tokenizer):
        assert exists(text_num_embeds), '`text_num_embeds` must be given if supplying your own tokenizer encode function'
        return tokenizer, text_num_embeds
    if tokenizer == 'char_utf8':
        return list_str_to_tensor, 256
    if tokenizer == 'phoneme_en':
        _unsupported('tokenizer', tokenizer, 'e2_tts.py:141-166 (g2p_en is host-side preprocessing; pass a callable tokenizer instead)')
    raise ValueError(f'unknown tokenizer string {tokenizer}')


class DurationPredictor(_PackOwner):
    """Reference surface: e2_tts.py:956-1113."""

    def __init__(self, transformer: dict | Transformer, num_channels=None, mel_spec_kwargs: dict = dict(), char_embed_kwargs: dict = dict(),
                 text_num_embeds=None, num_freq_tokens=1, hl_gauss_loss: dict | None = None, use_regression=True,
                 tokenizer: str | Callable = 'char_utf8'):
        super().__init__()
        if num_freq_tokens != 1:
            _unsupported('num_freq_tokens', num_freq_tokens, 'e2_tts.py:965')
        self.num_freq_tokens, self.has_freq_axis = 1, False
        if isinstance(transformer, dict):
            transformer = dict(transformer)
            transformer.setdefault('has_freq_axis', False)
            transformer = Transformer(**transformer, cond_on_time=False)
        assert not transformer.has_freq_axis
        self.mel_spec = MelSpec(**mel_spec_kwargs)
        self.num_channels = default(num_channels, self.mel_spec.n_mel_channels)
        self.transformer = transformer
        self.dim = transformer.dim
        self.proj_in = nn.Linear(self.num_channels, self.dim)
        self.tokenizer, text_num_embeds = _resolve_tokenizer(tokenizer, text_num_embeds)
        self.embed_text = CharacterEmbed(transformer.dim_text, num_embeds=text_num_embeds, **char_embed_kwargs)
        self.hl_gauss_layer = _HLGaussHead(self.dim, hl_gauss_loss, use_regression)   # :1035-1040

    def _add_weights(self, pack):
        w = dict(tr=self.transformer._add_weights(pack), proj_in=pack.buffer(self.dim, (self.num_channels + 7) // 8 * 8))
        pack.add(self.proj_in.weight, w['proj_in'])
        return w

    @_on_module_device
    def forward(self, x, *, text=None, lens=None, return_loss=True):
        if x.ndim == 2:  # raw wave (:1052-1055; the reference's `== self.dim` assert is a known bug, Appendix C)
            x = self.mel_spec(x).transpose(1, 2)
        x = x.to(F32).contiguous()
        B, N, C = x.shape
        dev = x.device
        if torch.is_grad_enabled() and return_loss:
            ops.zero_pool.begin(dev)
        w = self._packed_weights()
        A = ops.cast_rows(x.reshape(B * N, C), B * N, C, w['proj_in'].shape[1])
        h = ops.StemLinear.apply(A, self.proj_in.weight, self.proj_in.bias, None, None, w['proj_in'])
        ids = None
        if exists(text):
            if isinstance(text, list):
                text = list_str_to_tensor(text).to(dev)  # :1067 (always the byte tokenizer, Appendix C)
                assert text.shape[0] == B
            ids = self.embed_text.ids(text, N)
        if not exists(lens):
            lens = torch.full((B,), N, device=dev)
        mask = lens_to_mask(lens, length=N)
        if return_loss:  # :1081-1086
            rand_frac_index = _rng.draw('duration_rand_frac', lambda: x.new_zeros(B).uniform_(0, 1))
            rand_index = (rand_frac_index * lens).long()
            mask = mask & (torch.arange(N, device=dev)[None] < rand_index[:, None])
        tr = self.transformer
        y = tr._forward_from_h(w['tr'], h, B, N, None, mask, text_ids=ids, text_embed_module=self.embed_text)
        pooled = ops.MaskedMean.apply(y, mask.to(torch.uint8).contiguous(), B, N)
        if not return_loss:
            return self.hl_gauss_layer(pooled)   # :1107
        return self.hl_gauss_layer(pooled, lens.float())   # :1111


class _RngOverride:
    """Test hook: replay the reference's random draws (x0, times, span mask, drop_text_cond, duration prefix) so that
    parity tests run all three implementations on identical (mel, text, t, noise) inputs (SURVEY §8c)."""

    def __init__(self):
        self.values = None

    def draw(self, name, fn):
        if self.values is not None and name in self.values:
            return self.values[name]
        return fn()


_rng = _RngOverride()


class inject_randomness:
    def __init__(self, **values):
        self.values = values

    def __enter__(self):
        _rng.values = self.values

    def __exit__(self, *a):
        _rng.values = None


class E2TTS(_PackOwner):
    """Reference surface: e2_tts.py:1115-1595 (constructor, forward, sample, transformer_with_pred_head,
    cfg_transformer_with_pred_head, device)."""

    def __init__(self, transformer: dict | Transformer = None, duration_predictor: dict | DurationPredictor | None = None,
                 odeint_kwargs: dict = dict(atol=1e-5, rtol=1e-5, method='midpoint'), cond_drop_prob=0.25, num_channels=None,
                 mel_spec_module: Module | None = None, num_freq_tokens=1, char_embed_kwargs: dict = dict(), mel_spec_kwargs: dict = dict(),
                 frac_lengths_mask: tuple[float, float] = (0.7, 1.), concat_cond=False, interpolated_text=False,
                 text_num_embeds: int | None = None, tokenizer: str | Callable = 'char_utf8', use_vocos=True,
                 pretrained_vocos_path='charactr/vocos-mel-24khz', sampling_rate: int | None = None, velocity_consistency_weight=0.):
        super().__init__()
        if num_freq_tokens != 1:
            _unsupported('num_freq_tokens', num_freq_tokens, 'e2_tts.py:1130')
        _parse_odeint_kwargs(odeint_kwargs)
        self.num_freq_tokens, self.has_freq_axis = 1, False
        if isinstance(transformer, dict):
            transformer = dict(transformer)
            transformer.setdefault('has_freq_axis', False)
            transformer = Transformer(**transformer, cond_on_time=True)
        assert not transformer.has_freq_axis
        self.transformer = transformer
        if isinstance(duration_predictor, dict):
            duration_predictor = DurationPredictor(**duration_predictor)
        dim, dim_text = transformer.dim, transformer.dim_text
        self.dim, self.dim_text = dim, dim_text
        self.frac_lengths_mask = frac_lengths_mask
        self.duration_predictor = duration_predictor
        self.odeint_kwargs = odeint_kwargs
        self.mel_spec = default(mel_spec_module, MelSpec(**mel_spec_kwargs))
        num_channels = default(num_channels, self.mel_spec.n_mel_channels)
        self.num_channels = num_channels
        self.sampling_rate = default(sampling_rate, getattr(self.mel_spec, 'sampling_rate', None))
        self.concat_cond = concat_cond
        if concat_cond:      # :1200-1204: one Linear on cat(cond, x) instead of two summed projections
            self.proj_in = nn.Linear(num_channels * 2, dim)
        else:
            self.proj_in = nn.Linear(num_channels, dim)
            self.cond_proj_in = nn.Linear(num_channels, dim)
        self.to_pred = nn.Linear(dim, num_channels)
        self.tokenizer, text_num_embeds = _resolve_tokenizer(tokenizer, text_num_embeds)
        self.cond_drop_prob = cond_drop_prob
        text_embed_klass = InterpolatedCharacterEmbed if interpolated_text else CharacterEmbed          # :1233
        self.embed_text = text_embed_klass(dim_text, num_embeds=text_num_embeds, **char_embed_kwargs)
        self.register_buffer('zero', torch.tensor(0.), persistent=False)
        self.velocity_consistency_weight = velocity_consistency_weight
        # Vocos (e2_tts.py:1244) is loaded from local files only: a checkpoint directory or a repo id already in the local HF cache.
        # When neither resolves, vocos stays None and sample() refuses to decode (nothing is downloaded).
        self.vocos = None
        self._use_vocos_requested = use_vocos
        if use_vocos:
            from .vocos import Vocos, resolve_local
            if resolve_local(pretrained_vocos_path) is not None:
                self.vocos = Vocos.from_pretrained(pretrained_vocos_path)

    @property
    def device(self):
        return next(self.parameters()).device

    def _add_weights(self, pack):
        C, d = self.num_channels, self.dim
        Cp = (C + 63) // 64 * 64
        w = dict(tr=self.transformer._add_weights(pack), Cp=Cp, stem=pack.buffer(d, 2 * Cp), pred=pack.buffer(C, d))
        pack.add(self.proj_in.weight, w['stem'])          # concat_cond: all 2C columns, matching stem_prepare's cat(cond, x) layout
        if not self.concat_cond:
            pack.add(self.cond_proj_in.weight, w['stem'], col_off=Cp)
        pack.add(self.to_pred.weight, w['pred'])
        if isinstance(self.embed_text, InterpolatedCharacterEmbed):
            w2 = self.embed_text.abs_pos_mlp[3].weight
            w['interp'] = pack.buffer(*w2.shape)
            pack.add(w2, w['interp'])
        return w

    def _embed(self, w, A, B, N, times, mask, text, drop_text_cond):
        if self.concat_cond:
            h = ops.StemLinear.apply(A, self.proj_in.weight, self.proj_in.bias, None, None, w['stem'])
        else:
            h = ops.StemLinear.apply(A, self.proj_in.weight, self.proj_in.bias, self.cond_proj_in.weight, self.cond_proj_in.bias, w['stem'])
        ids, te = None, None
        if exists(text) and not drop_text_cond:
            if isinstance(self.embed_text, InterpolatedCharacterEmbed):
                te = self.embed_text.embed_bf16(text, N, mask, w['interp'])      # :1283 embed_text(text, seq_len, mask = mask)
            else:
                ids = self.embed_text.ids(text, N)
        return self.transformer._forward_from_h(w['tr'], h, B, N, times, mask, text_ids=ids, text_embed_module=self.embed_text, te_bf16=te)

    @_on_module_device
    def transformer_with_pred_head(self, x, cond, times, mask=None, text=None, drop_text_cond=None, return_drop_text_cond=False):
        """e2_tts.py:1250-1301."""
        B, N, C = x.shape
        drop_text_cond = default(drop_text_cond, self.training and pyrandom.random() < self.cond_drop_prob)
        w = self._packed_weights()
        A, _ = ops.stem_prepare(B, N, C, w['Cp'], x_in=x.to(F32).contiguous(), cond_in=cond.to(F32).contiguous(), concat=self.concat_cond)
        if not torch.is_tensor(times):
            times = torch.tensor(times, device=x.device)
        y = self._embed(w, A, B, N, times.to(x.device), mask, text, drop_text_cond)
        pred = ops.PredHead.apply(y, self.to_pred.weight, self.to_pred.bias, w['pred']).view(B, N, C).to(x.dtype)
        if not return_drop_text_cond:
            return pred
        return pred, drop_text_cond

    def cfg_transformer_with_pred_head(self, *args, cfg_strength: float = 1., cfg_null_model=None, remove_parallel_component: bool = True,
                                       keep_parallel_frac: float = 0., **kwargs):
        """e2_tts.py:1303-1330 (CFG + APG projection in fp64, :113-124)."""
        pred = self.transformer_with_pred_head(*args, drop_text_cond=False, **kwargs)
        if cfg_strength < 1e-5:
            return pred
        null_drop = not exists(cfg_null_model)
        cfg_null_model = default(cfg_null_model, self)
        null_pred = cfg_null_model.transformer_with_pred_head(*args, drop_text_cond=null_drop, **kwargs)
        return ops.cfg_combine(pred, null_pred, float(cfg_strength), bool(remove_parallel_component), float(keep_parallel_frac))

    @_on_module_device
    def cfg_pred_batched(self, x, cond, times, mask2, text, cfg_strength: float = 1., remove_parallel_component: bool = True,
                         keep_parallel_frac: float = 0.):
        """cfg_transformer_with_pred_head without a cfg_null_model, as ONE transformer pass over 2B items: items 0..B-1 are
        (x, cond, text), items B..2B-1 the same x and cond with the text dropped. x, cond fp32 [B, N, C]; times a 0-dim tensor;
        mask2 bool [2B, N] (the mask of the B items, twice) or None; text ids [B, nt] or None. Inference only."""
        pred, null_pred = self._pred_pair(x, cond, times, mask2, text)
        return ops.cfg_combine(pred, null_pred, float(cfg_strength), bool(remove_parallel_component), float(keep_parallel_frac))

    def _pred_pair(self, x, cond, times, mask2, text):
        """-> (the conditional, the text-dropped prediction), each fp32 [B, N, C]: the two halves of one [2B, N, C] prediction, which
        cfg_combine reads in place. Rows are item-major, so the text stream covers a row prefix (Transformer._forward_from_h
        text_items). With text None both halves would be the same pass, so one pass over the B items serves as both."""
        B, N, C = x.shape
        w = self._packed_weights()
        A, _ = ops.stem_prepare(B, N, C, w['Cp'], x_in=x.to(F32).contiguous(), cond_in=cond.to(F32).contiguous(), concat=self.concat_cond)
        mask = mask2[:B] if exists(mask2) else None
        if not exists(text):
            y = self._embed(w, A, B, N, times, mask, None, True)
            pred = ops.PredHead.apply(y, self.to_pred.weight, self.to_pred.bias, w['pred']).view(B, N, C)
            return pred, pred
        bias = self.proj_in.bias if self.concat_cond else self.proj_in.bias + self.cond_proj_in.bias
        h = ops.stem_linear_twice(A, w['stem'], bias)     # both halves start from the same x and cond
        ids, te = None, None
        if isinstance(self.embed_text, InterpolatedCharacterEmbed):
            te = self.embed_text.embed_bf16(text, N, mask, w['interp'])
        else:
            ids = self.embed_text.ids(text, N)
        y = self.transformer._forward_from_h(w['tr'], h, 2 * B, N, times, mask2, text_ids=ids, text_embed_module=self.embed_text,
                                             te_bf16=te, text_items=B)
        pred = ops.PredHead.apply(y, self.to_pred.weight, self.to_pred.bias, w['pred']).view(2 * B, N, C)
        return pred[:B], pred[B:]

    def _check_decoder(self, vocoder, return_raw_output, save_to_filename=None):
        """sample()'s refusal to start an ODE solve whose output it could not decode"""
        no_vocos = self._use_vocos_requested and not exists(self.vocos)
        if not (exists(return_raw_output) and return_raw_output) and not exists(vocoder) and (no_vocos or exists(save_to_filename)):
            # fail BEFORE the ODE loop (124 transformer passes at the defaults), not after it
            raise NotImplementedError('Vocos decoding / audio saving needs the pretrained vocoder from the HF hub and is out of scope '
                                      '(SURVEY.md §2 row 10): call sample(..., return_raw_output=True), pass `vocoder=`, build '
                                      'E2TTS(use_vocos=False), or pass a local `pretrained_vocos_path`')

    def _sample_inputs(self, cond, text, lens, duration, max_duration):
        """sample()'s preparation ahead of the ODE (e2_tts.py:1356-1402): mel of a raw wave, tokens, lens = max(text lens, lens), the
        duration (predicted when None), clamped to [lens + 1, max_duration]. -> (cond fp32 [B, md, C] zero-padded, cond_mask bool
        [B, md, 1], text ids | None, duration [B]) with md = max(duration)."""
        if cond.ndim == 2:
            cond = self.mel_spec(cond).transpose(1, 2)
            assert cond.shape[-1] == self.num_channels
        cond = cond.to(F32)
        B, cond_seq_len, dev = *cond.shape[:2], cond.device
        if not exists(lens):
            lens = torch.full((B,), cond_seq_len, device=dev, dtype=torch.long)
        if isinstance(text, list):
            text = self.tokenizer(text).to(dev)
            assert text.shape[0] == B
        if exists(text):
            lens = torch.maximum((text != -1).sum(dim=-1), lens)
        cond_mask = lens_to_mask(lens)
        if exists(duration):
            if isinstance(duration, int):
                duration = torch.full((B,), duration, device=dev, dtype=torch.long)
        elif exists(self.duration_predictor):
            duration = self.duration_predictor(cond, text=text, lens=lens, return_loss=False).long()
        duration = torch.maximum(lens + 1, duration).clamp(max=max_duration)
        assert duration.shape[0] == B
        md = int(duration.amax())
        cond = F.pad(cond, (0, 0, 0, md - cond_seq_len), value=0.)
        cond_mask = F.pad(cond_mask, (0, md - cond_mask.shape[-1]), value=False)[..., None]
        return cond, cond_mask, text, duration

    def _sample_output(self, out, duration, vocoder, return_raw_output):
        """sample()'s return value from the solved mel `out` [B, md, C] (e2_tts.py:1430-1466)"""
        if exists(return_raw_output) and return_raw_output:
            return out
        if exists(vocoder):
            assert not exists(self.vocos), '`use_vocos` should not be turned on if you are passing in a custom `vocoder` on sampling'
            return vocoder(out.transpose(1, 2))
        if exists(self.vocos):   # :1440-1451, the whole ragged batch in one decode: item b is out[b, :duration[b]]
            audio = self.vocos.decode_padded(out, duration, db_to_amp=True)
            hop = self.vocos.hop_length
            return [audio[b, :int(n) * hop] for b, n in enumerate(duration.tolist())]
        return out

    @torch.no_grad()
    @_on_module_device
    def sample(self, cond, *, text=None, lens=None, duration=None, steps=32, cfg_strength=1., cfg_null_model=None, max_duration=4096,
               vocoder=None, return_raw_output=None, save_to_filename=None):
        """e2_tts.py:1332-1466. The ODE on t = linspace(0, 1, steps) with the torchdiffeq method of `odeint_kwargs` (SURVEY A.7): the
        fixed-grid midpoint / euler loop below, or rk4 and the adaptive Runge–Kutta methods of ode.py."""
        ode_kw = _parse_odeint_kwargs(self.odeint_kwargs)   # odeint_kwargs is a plain attribute: checked again before any work
        self.eval()
        self._check_decoder(vocoder, return_raw_output, save_to_filename)
        cond, cond_mask, text, duration = self._sample_inputs(cond, text, lens, duration, max_duration)
        dev = cond.device
        mask = lens_to_mask(duration)
        step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))  # step-invariant: hoisted out of fn (:1404)

        def fn(t, x):
            return self.cfg_transformer_with_pred_head(x, step_cond, times=t, text=text, mask=mask, cfg_strength=cfg_strength,
                                                       cfg_null_model=cfg_null_model)

        y = _rng.draw('y0', lambda: torch.randn_like(cond))
        ts_host = torch.linspace(0, 1, steps)          # fixed grid (torchdiffeq semantics); step sizes stay host floats: no device sync per step
        ts = ts_host.to(dev)
        method = ode_kw.pop('method')
        # weights are fixed for the whole solve: pack each model's operands once (fresh), not once per function evaluation
        freeze_null = cfg_null_model._pack()[0].freeze() if exists(cfg_null_model) else contextlib.nullcontext()
        with self._pack()[0].freeze(), freeze_null:
            fn_eval = fn   # (one function evaluation as a CUDA graph was measured: -1 % at cfg5, but re-capturing per call costs the e2e path 19 %;
                           #  GraphedSampler captures the whole solve once instead)
            if method not in ('midpoint', 'euler'):   # rk4 and the adaptive Runge–Kutta methods
                y = ode.odeint(fn_eval, y, steps, method, **ode_kw)
            else:
                for i in range(steps - 1):
                    t0, dt = ts[i], float(ts_host[i + 1] - ts_host[i])
                    if method == 'euler':
                        y = ops.axpy(y, fn_eval(t0, y), dt)
                    else:
                        half = 0.5 * dt
                        ymid = ops.axpy(y, fn_eval(t0, y), half)
                        y = ops.axpy(y, fn_eval(t0 + half, ymid), dt)
        return self._sample_output(torch.where(cond_mask, cond, y), duration, vocoder, return_raw_output)

    @_on_module_device
    def forward(self, inp, *, text=None, times=None, lens=None, velocity_consistency_model=None, velocity_consistency_delta=1e-5):
        """Flow-matching training objective, e2_tts.py:1468-1595. Returns E2TTSReturn(loss, cond, pred_flow, pred_data, breakdown)."""
        need_velocity_loss = exists(velocity_consistency_model) and self.velocity_consistency_weight > 0.
        if inp.ndim == 2:
            inp = self.mel_spec(inp).transpose(1, 2)
            assert inp.shape[-1] == self.num_channels
        x1 = inp.to(F32).contiguous()
        B, N, C = x1.shape
        dev = self.device
        if torch.is_grad_enabled():
            ops.zero_pool.begin(dev)
        if isinstance(text, list):
            text = self.tokenizer(text).to(dev)
            assert text.shape[0] == B
        if not exists(lens):
            lens = torch.full((B,), N, device=dev)
        mask = lens_to_mask(lens, length=N)
        # RNG draw order of the reference (Appendix C): frac_lengths, span start, x0, times, text drop
        def span():
            frac = torch.zeros((B,), device=dev).float().uniform_(*self.frac_lengths_mask)
            return mask_from_frac_lengths(lens, frac, N)
        rand_span_mask = _rng.draw('span_mask', span) & mask
        x0 = _rng.draw('x0', lambda: torch.randn_like(x1))
        times = _rng.draw('times', lambda: torch.rand((B,), dtype=x1.dtype, device=dev))
        drop_text_cond = _rng.draw('drop_text_cond', lambda: self.training and pyrandom.random() < self.cond_drop_prob)
        span_u8 = rand_span_mask.to(torch.uint8).contiguous()
        times = times.to(F32).contiguous()
        vel_target = None
        if need_velocity_loss:   # :1556-1576 — the EMA model's prediction at t + delta on the same (x0, x1, cond, text-drop coin), no grad
            vcm = velocity_consistency_model
            with torch.no_grad():
                t_d = times + velocity_consistency_delta
                vw = vcm._packed_weights()
                A_d, _ = ops.stem_prepare(B, N, C, vw['Cp'], x1=x1, x0=x0, times=t_d, span=span_u8, concat=velocity_consistency_model.concat_cond)
                y_d = vcm._embed(vw, A_d, B, N, t_d, mask, text, drop_text_cond)
                vel_target = ops.PredHead.apply(y_d, vcm.to_pred.weight, vcm.to_pred.bias, vw['pred'])
        w = self._packed_weights()
        A, cond = ops.stem_prepare(B, N, C, w['Cp'], x1=x1, x0=x0, times=times, span=span_u8, want_cond=True, concat=self.concat_cond)
        y = self._embed(w, A, B, N, times, mask, text, drop_text_cond)
        loss, pred, pred_data, parts = ops.FlowLossHead.apply(y, self.to_pred.weight, self.to_pred.bias, w['pred'], x1, x0, span_u8, vel_target,
                                                              float(self.velocity_consistency_weight) if need_velocity_loss else 0.0)
        breakdown = LossBreakdown(parts[0], parts[1] if need_velocity_loss else self.zero)
        return E2TTSReturn(loss, cond, pred.view(B, N, C), pred_data.view(B, N, C), breakdown)
