"""CPU: the attention geometry knobs of Transformer (e2_tts.py:527-531) — 128-wide heads (dim_head, text_dim_head) and a text stream
with its own head count (text_heads). The oracle with the same geometry against what the original e2_tts.py computed with them
(tests/golden/reference/headdim_*.pt, oracle/make_reference_golden.py), the package's parameter layout against the original's, the head
dims that still raise, and the C-ABI validation of dim_head."""
import pytest

from headdim_variants import HEADDIM_CASES, HEADDIM_SAMPLE
from model_checks import check_case, oracle_case, sample_vs_reference, state_dict_vs_reference
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg


@pytest.mark.parametrize('name', list(HEADDIM_CASES))
def test_oracle_vs_reference(name):
    """loss, prediction and gradient samples within the bounds of tests/test_oracle_vs_reference.py"""
    c, g = HEADDIM_CASES[name], RC.load('headdim_' + name)
    check_case(c, g, *oracle_case(c, g))
    if c['drop']:   # the text stream is skipped: its parameters get no gradient
        assert g['grads']['transformer.layers.0.1.2.to_q.weight'] is None


def test_sample_vs_reference():
    sample_vs_reference(HEADDIM_SAMPLE, RC.load('headdim_sample'))


@pytest.mark.parametrize('name', list(HEADDIM_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model with the same geometry: its checkpoints load"""
    state_dict_vs_reference(HEADDIM_CASES[name], RC.load('headdim_' + name))


def test_geometry_is_recorded():
    t = pkg.Transformer(dim=256, depth=2, heads=2, dim_head=128, text_heads=1, text_dim_head=64)
    assert (t.heads, t.dim_head, t.text_heads, t.text_dim_head) == (2, 128, 1, 64)
    audio, text = t.layers[0][0][3], t.layers[0][1][2]
    assert (audio.heads, audio.dim_head, text.heads, text.dim_head) == (2, 128, 1, 64)
    assert audio.to_q.weight.shape == (256, 256) and text.to_q.weight.shape == (64, 128)


@pytest.mark.parametrize('kw', [dict(dim_head=32), dict(dim_head=96), dict(text_dim_head=32), dict(text_dim_head=96),
                                dict(dim_head=128, text_dim_head=256)])
def test_other_head_dims_raise(kw):
    name = next(iter(kw))
    with pytest.raises(NotImplementedError, match=f'{name}=.*supported head dims are 64 and 128'):
        pkg.Transformer(dim=128, depth=2, heads=2, **kw)
    with pytest.raises(NotImplementedError, match='supported head dims are 64 and 128'):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, **kw), use_vocos=False)


def test_cabi_dim_head_validation_without_gpu():
    """dim_head is checked before the device is touched (placeholder pointers, never read)"""
    ptrs = dict.fromkeys(('q', 'k', 'v', 'o', 'lse', 'ws_maskbits'), 256)
    bwd = dict(d_og=256, ws_dO=256, ws_delta=256, dq=256, dk=256, dv=256)
    for dh in (32, 96, 256):
        shape = dict(B=1, H=1, Np=64, dim_head=dh, scale=dh ** -0.5, softclamp=50.0)
        for name, extra in (('b200_attn_fwd', dict(og=256)), ('b200_attn_bwd', bwd)):
            a = pkg.lib.make_args(name + '_args', **ptrs, **shape, **extra)
            with pytest.raises(RuntimeError, match='dim_head must be 64 or 128'):
                pkg.lib.call(name, a, None)
        q = dict(qkvg=256, rot_cos=256, rot_sin=256, q=256, k=256, v=256, B=1, H=2, Np=8, dim_head=dh, ld=3 * 2 * 128 + 8, no_gate=1)
        a = pkg.lib.make_args('b200_qkv_post_args', **q)
        with pytest.raises(RuntimeError, match='dim_head must be 64 or 128'):
            pkg.lib.call('b200_qkv_post_fwd', a, None)
        a = pkg.lib.make_args('b200_qkv_post_args', **q, dq=256, dk=256, dv=256, d_qkvg=256)
        with pytest.raises(RuntimeError, match='dim_head must be 64 or 128'):
            pkg.lib.call('b200_qkv_post_bwd', a, None)
        with pytest.raises(RuntimeError, match='dim_head must be 64 or 128'):
            pkg.lib.call('b200_rotary_table', 256, 256, 8, dh, None)
    # the row pitch follows the head dim: 3 H dim_head columns (+ H per gate / mix logit)
    q = dict(qkvg=256, rot_cos=256, rot_sin=256, q=256, k=256, v=256, B=1, H=2, Np=8, dim_head=128, no_gate=1)
    a = pkg.lib.make_args('b200_qkv_post_args', ld=3 * 2 * 64, **q)
    with pytest.raises(RuntimeError, match='row pitch'):
        pkg.lib.call('b200_qkv_post_fwd', a, None)
