"""CPU: the model-shape knobs of Transformer (e2_tts.py:518-552) — depth 12, text_depth < depth, dim_text != dim // 2, ff_mult and
text_ff_mult != 4, num_registers 0 / 8 / 16, abs_pos_emb=False, kernel_size 1 / 5 / 7. The oracle against what the original e2_tts.py
computed with them (tests/golden/reference/geometry_*.pt, oracle/make_reference_golden.py), one negative control per knob, the package's
parameter layout against the original's, and the geometries that raise."""
import pytest
import torch

from geometry_variants import GEOMETRY_CASES, GEOMETRY_SAMPLE, reverted
from model_checks import check_case, oracle_case, sample_vs_reference, state_dict_vs_reference
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg


@pytest.mark.parametrize('name', list(GEOMETRY_CASES))
def test_oracle_vs_reference(name):
    """loss, prediction and gradient samples within the bounds of tests/test_oracle_vs_reference.py"""
    c, g = GEOMETRY_CASES[name], RC.load('geometry_' + name)
    check_case(c, g, *oracle_case(c, g))
    depth, text_depth = c['tkw']['depth'], c['tkw'].get('text_depth', c['tkw']['depth'])
    last = f'transformer.layers.{text_depth - 1}.1.'
    if c['drop']:   # the text stream is skipped: its parameters get no gradient
        assert g['grads'][last + '2.to_q.weight'] is None
    elif text_depth < depth:   # the text stream stops at text_depth: its last cross-condition conditions the audio only
        assert g['grads'][last + '2.to_q.weight'] is not None and last + '5.audio_to_text.weight' not in g['grads']
        assert not any(k.startswith(f'transformer.layers.{text_depth}.1.') for k in g['grads'])


@pytest.mark.parametrize('name,knob', [(n, k) for n, c in GEOMETRY_CASES.items() for k in c['knobs']])
def test_knob_reverted_misses_reference(name, knob):
    """negative control: the oracle with one knob back at the reference's default (on the case's own weights wherever the shapes
    allow) misses what the original computed, so no case passes whatever the knob does"""
    c = GEOMETRY_CASES[name]
    g = RC.load('geometry_' + name)
    tkw, sd = reverted(c, knob)
    with torch.no_grad():
        _, loss, pred = oracle_case(dict(c, tkw=tkw), g, sd=sd)
    if pred is not None:
        assert RC.compact_rel_l2(pred, g['pred']) > 1e-2
    else:
        assert abs(float(loss) - g['loss']) > 1e-3 * abs(g['loss'])


def test_sample_vs_reference():
    """4 midpoint steps, a per-element duration and a ragged prompt"""
    s, g = GEOMETRY_SAMPLE, RC.load('geometry_sample')
    sample_vs_reference(s, g, lens=torch.tensor(s['lens']))
    assert g['shape'] == (2, max(s['duration']), 100)


@pytest.mark.parametrize('name', list(GEOMETRY_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model with the same geometry: its checkpoints load"""
    state_dict_vs_reference(GEOMETRY_CASES[name], RC.load('geometry_' + name))


def test_geometry_is_recorded():
    t = pkg.Transformer(dim=192, depth=12, heads=3, dim_text=128, ff_mult=2, text_ff_mult=2.5, text_depth=5, num_registers=0,
                        abs_pos_emb=False, kernel_size=7)
    assert (t.dim, t.dim_text, t.depth, t.text_depth, t.num_registers) == (192, 128, 12, 5, 0)
    assert t.abs_pos_emb is None and t.registers.shape == (0, 192) and t.text_registers.shape == (0, 128)
    assert [t.layers[i][1] is not None for i in range(12)] == [True] * 5 + [False] * 7
    assert [t.layers[i][0][0] is not None for i in range(12)] == [False] * 6 + [True] * 6    # skip projections of the later half
    assert [t.layers[i][1][5].cond_audio_to_text for i in range(5)] == [True] * 4 + [False]
    assert t.layers[0][0][7].ff[2].weight.shape == (192, 384) and t.layers[0][1][4].ff[2].weight.shape == (128, 320)
    assert t.layers[0][0][1].dw_conv1d[0].weight.shape == (192, 1, 7)


@pytest.mark.parametrize('kw', [dict(kernel_size=4), dict(kernel_size=30)])
def test_even_kernel_size_raises(kw):
    """e2_tts.py:304 asserts an odd kernel size"""
    with pytest.raises(AssertionError):
        pkg.Transformer(dim=128, depth=2, heads=2, **kw)


@pytest.mark.parametrize('kw', [dict(text_depth=3), dict(text_depth=5, depth=4)])
def test_text_depth_past_depth_raises(kw):
    """e2_tts.py:574: 1 <= text_depth <= depth, in the package and in the oracle"""
    kw = dict(dict(depth=2), **kw)
    with pytest.raises(AssertionError):
        pkg.Transformer(dim=128, heads=2, **kw)
    with pytest.raises(AssertionError):
        O.TransformerCfg(dim=128, **kw)


@pytest.mark.parametrize('kw', [dict(dim=192), dict(dim=96, dim_text=64), dict(dim=1088, dim_text=512), dict(dim=128, dim_text=96)])
def test_width_off_64_raises(kw):
    """model widths the kernels do not take (dim 192 with its default dim_text 96 among them) are refused, naming the knob"""
    name = 'dim_text' if kw['dim'] in (192, 128) else 'dim'
    with pytest.raises(NotImplementedError, match=f'{name}=.*multiples of 64 up to 1024'):
        pkg.Transformer(depth=2, heads=2, **kw)


@pytest.mark.parametrize('kw,name,inner', [(dict(dim=192, dim_text=128, ff_mult=2.5), 'ff_mult', 480),(dict(dim=128, ff_mult=1.25), 'ff_mult', 160),
                                           (dict(dim=128, text_ff_mult=2.5), 'text_ff_mult', 160),
                                           (dict(dim=256, dim_text=64, text_ff_mult=1.5), 'text_ff_mult', 96)])
def test_ff_inner_width_off_64_raises(kw, name, inner):
    """the GLU kernels pack the hidden units in 64-column halves: an inner width int(dim * mult) that is not a multiple of 64 is
    refused when the model is built, naming the knob and the width (the reference builds it, e2_tts.py:646, :692)"""
    with pytest.raises(NotImplementedError, match=f'{name}=.*inner width .* = {inner} is not a multiple of 64'):
        pkg.Transformer(depth=2, heads=2, **kw)
    with pytest.raises(NotImplementedError, match='multiple of 64'):
        pkg.E2TTS(transformer=dict(depth=2, heads=2, **kw), use_vocos=False)
