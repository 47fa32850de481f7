"""CPU: the x-transformers `attn_kwargs` of Transformer (e2_tts.py:548-551) besides the reference's default — no head gate, no logit
soft-clamp, another clamp value. The oracle with the same attn_kwargs against what the original e2_tts.py computed on those settings
(tests/golden/reference/attn_kwargs_*.pt, oracle/make_reference_golden.py), the package's parameter layout against the original's,
the switches that still raise, and the C-ABI validation of the unclamped / no-gate fields."""
import pytest

from attn_variants import ATTN_KWARGS_CASES
from model_checks import check_case, oracle_case, state_dict_vs_reference
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg


@pytest.mark.parametrize('name', list(ATTN_KWARGS_CASES))
def test_oracle_vs_reference(name):
    """loss, prediction and gradient samples within the bounds of tests/test_oracle_vs_reference.py"""
    c, g = ATTN_KWARGS_CASES[name], RC.load('attn_kwargs_' + name)
    check_case(c, g, *oracle_case(c, g))


@pytest.mark.parametrize('name', list(ATTN_KWARGS_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model with the same attn_kwargs: its checkpoints load"""
    c = ATTN_KWARGS_CASES[name]
    got = state_dict_vs_reference(c, RC.load('attn_kwargs_' + name))
    has_gate = c['tkw']['attn_kwargs'].get('gate_value_heads', False)
    assert any(k.endswith('to_v_head_gate.weight') for k in got) == has_gate


@pytest.mark.parametrize('attn_kwargs,gate,clamp', [
    (dict(gate_value_heads=True, softclamp_logits=True), True, 50.0),
    (dict(gate_value_heads=True, softclamp_logits=True, logit_softclamp_value=50.), True, 50.0),
    (dict(), False, None),
    (dict(gate_value_heads=True), True, None),
    (dict(softclamp_logits=True, logit_softclamp_value=30.), False, 30.0),
    (dict(softclamp_logits=True, logit_softclamp_value=64.), False, 64.0),
    (dict(softclamp_logits=False, logit_softclamp_value=500.), False, None),
])
def test_attn_kwargs_parse(attn_kwargs, gate, clamp):
    """a missing key takes x-transformers' default; the reference's default dict keeps the module constant clamp"""
    t = pkg.Transformer(dim=128, depth=2, heads=2, attn_kwargs=attn_kwargs)
    assert t.softclamp == clamp == O.TransformerCfg(dim=128, attn_kwargs=attn_kwargs).softclamp
    if attn_kwargs.get('gate_value_heads') and attn_kwargs.get('softclamp_logits') and clamp == 50.0:
        assert t.softclamp == pkg.modules.SOFTCLAMP
    attn = t.layers[1][0][3]
    assert (attn.to_v_head_gate is not None) == gate
    assert (t.layers[1][1][2].to_v_head_gate is not None) == gate   # the text attention takes the same kwargs


def test_unsupported_attn_kwargs_raise():
    with pytest.raises(NotImplementedError, match='laser'):
        pkg.Transformer(dim=128, depth=2, heads=2, attn_kwargs=dict(laser=True))
    with pytest.raises(NotImplementedError, match='dropout'):
        pkg.Transformer(dim=128, depth=2, heads=2, attn_kwargs=dict(gate_value_heads=True, dropout=0.1))
    with pytest.raises(NotImplementedError, match='running maximum'):
        pkg.Transformer(dim=128, depth=2, heads=2, attn_kwargs=dict(softclamp_logits=True, logit_softclamp_value=100.))
    with pytest.raises(NotImplementedError, match='logit_softclamp_value'):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, attn_kwargs=dict(softclamp_logits=True, logit_softclamp_value=0.)),
                  use_vocos=False)


def test_cabi_unclamped_and_no_gate_validation_without_gpu():
    """the trailing unclamped / no_gate fields are checked before the device is touched (placeholder pointers, never read)"""
    ptrs = dict.fromkeys(('q', 'k', 'v', 'o', 'lse', 'ws_maskbits'), 256)
    shape = dict(B=1, H=1, Np=64, dim_head=64, scale=0.125)
    bwd = dict(d_og=256, ws_dO=256, ws_delta=256, dq=256, dk=256, dv=256)
    for name, extra in (('b200_attn_fwd', dict(og=256)), ('b200_attn_bwd', bwd)):
        args = name + '_args'
        # an ambiguous call: unclamped with a clamp value
        a = pkg.lib.make_args(args, **ptrs, **shape, **extra, softclamp=50.0, unclamped=1)
        with pytest.raises(RuntimeError, match='unclamped'):
            pkg.lib.call(name, a, None)
        # all-zero new field: today's refusals
        for clamp in (0.0, 100.0):
            a = pkg.lib.make_args(args, **ptrs, **shape, **extra, softclamp=clamp)
            with pytest.raises(RuntimeError, match='softclamp'):
                pkg.lib.call(name, a, None)
    # qkv_post: without no_gate the gate pointers are required; with it the row pitch may be 3I (+ H with the mix logits)
    q = dict(qkvg=256, rot_cos=256, rot_sin=256, q=256, k=256, v=256, B=1, H=8, Np=8, dim_head=64)   # I = 512
    a = pkg.lib.make_args('b200_qkv_post_args', ld=3 * 512 + 8, **q)
    with pytest.raises(RuntimeError, match='null pointer'):
        pkg.lib.call('b200_qkv_post_fwd', a, None)
    a = pkg.lib.make_args('b200_qkv_post_args', ld=3 * 512 + 8, gate_bias=256, gate=256, v_first=256, mix_bias=256, **q)
    with pytest.raises(RuntimeError, match='row pitch'):   # gate + mix need 3I + 2H columns
        pkg.lib.call('b200_qkv_post_fwd', a, None)
    a = pkg.lib.make_args('b200_qkv_post_args', ld=3 * 512 - 8, no_gate=1, **q)
    with pytest.raises(RuntimeError, match='row pitch'):
        pkg.lib.call('b200_qkv_post_fwd', a, None)
    a = pkg.lib.make_args('b200_qkv_post_args', ld=3 * 512, no_gate=1, dq=256, dk=256, dv=256, **q)
    with pytest.raises(RuntimeError, match='null pointer'):   # d_qkvg missing; d_gate is not needed
        pkg.lib.call('b200_qkv_post_bwd', a, None)
