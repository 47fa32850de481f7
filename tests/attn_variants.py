"""Cases and oracle of the x-transformers `attn_kwargs` the model builds besides the reference's default (gate_value_heads=True,
softclamp_logits=True): no head gate, no logit soft-clamp, another clamp value. Shared by tests/test_attn_kwargs_vs_reference.py
(oracle against the original's stored outputs) and tests/test_gpu_attention_variants.py (kernels against the oracle).

The oracle of oracle/e2tts_oracle.py always clamps and always gates; `variant_oracle` swaps its attention leaf for the x-transformers
Attention of these switches (oracle/ref_leaves/x_transformers/x_transformers.py:93-143) for the duration of a `with` block."""
import contextlib

import torch

from oracle import e2tts_oracle as O

# x-transformers' defaults for a key missing from attn_kwargs
XT_DEFAULTS = dict(gate_value_heads=False, softclamp_logits=False, logit_softclamp_value=50.)

# name -> (attn_kwargs, model class, seed, mel shape, lens, text)
ATTN_KWARGS_CASES = {
    'plain': dict(attn_kwargs=dict(), cls='E2TTS', seed=51, mel=(2, 64), lens=[64, 45], text=['abc', 'defgh ij']),
    'gate_only': dict(attn_kwargs=dict(gate_value_heads=True), cls='E2TTS', seed=52, mel=(2, 64), lens=[64, 37], text=['abc', 'xy z']),
    'clamp30': dict(attn_kwargs=dict(softclamp_logits=True, logit_softclamp_value=30.), cls='E2TTS', seed=53, mel=(2, 64), lens=[64, 50],
                    text=['hello', 'abc']),
    'duration_plain': dict(attn_kwargs=dict(), cls='DurationPredictor', seed=54, mel=(3, 72), lens=[72, 50, 31],
                           text=['abc', 'hello world', 'x']),
}


def clamp_of(attn_kwargs):
    """the logit soft-clamp value of these kwargs, None without clamp"""
    kw = {**XT_DEFAULTS, **attn_kwargs}
    return float(kw['logit_softclamp_value']) if kw['softclamp_logits'] else None


def attention(sd, p, x, mask, freqs, value_residual, heads, dim_head, softclamp):
    """O.attention with the clamp optional (softclamp None) and the head gate optional (absent from sd)"""
    b, n, _ = x.shape
    split = lambda t: t.reshape(b, n, heads, dim_head).permute(0, 2, 1, 3)
    q, k, v = (split(x @ sd[p + f'.to_{c}.weight'].t()) for c in 'qkv')
    orig_v = v
    if value_residual is not None:
        mix = torch.sigmoid(x @ sd[p + '.to_value_residual_mix.0.weight'].t() + sd[p + '.to_value_residual_mix.0.bias'])
        mix = mix.permute(0, 2, 1)[..., None]
        v = v * mix + value_residual * (1.0 - mix)
    q, k = O.apply_rotary(q, freqs), O.apply_rotary(k, freqs)
    sim = torch.einsum('bhid,bhjd->bhij', q, k) * dim_head ** -0.5
    if softclamp is not None:
        sim = torch.tanh(sim / softclamp) * softclamp
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], -torch.finfo(sim.dtype).max)
    attn = O.drop(p + '.attn_dropout', torch.softmax(sim.float(), dim=-1).to(sim.dtype))
    out = torch.einsum('bhij,bhjd->bhid', attn, v)
    if p + '.to_v_head_gate.weight' in sd:
        gate = torch.sigmoid(x @ sd[p + '.to_v_head_gate.weight'].t() + sd[p + '.to_v_head_gate.bias'])
        out = out * gate.permute(0, 2, 1)[..., None]
    out = out.permute(0, 2, 1, 3).reshape(b, n, heads * dim_head) @ sd[p + '.to_out.weight'].t()
    if mask is not None:
        out = out * mask[..., None]
    return out, orig_v


@contextlib.contextmanager
def variant_oracle(attn_kwargs):
    """O.e2tts_forward / O.duration_forward / O.e2tts_sample run the attention of `attn_kwargs` inside the block"""
    clamp = clamp_of(attn_kwargs)
    orig = O.attention
    O.attention = lambda sd, p, x, mask, freqs, vr, heads, dim_head, _softclamp: attention(sd, p, x, mask, freqs, vr, heads, dim_head, clamp)
    try:
        yield
    finally:
        O.attention = orig
